"""Rotation averaging without a GPU: the fp64 oracle (tests/ra_oracle.py) on synthetic pose graphs with the bars of the
reference's rotation_averaging_test.cc, the exact per-axis split of the normal matrix that the GPU factors, the host
input checks of b200ra_solve, which refuse before any device work, and the ABI surface."""
import ctypes
import hashlib

import numpy as np
import pytest

import ra_oracle
from colmap_b200 import load_library
from colmap_b200.rotation_averaging import (ERR_INPUT, ERR_TOO_LARGE, UNDERDETERMINED, FlatRotationAveraging,
                                            RotationAveragingError, RotationEstimatorOptions, _bind, _COptions,
                                            solve_flat)
from colmap_b200.synthetic import synthesize_rotation_averaging


def block_rotations(flat, x):
    """The rotation matrix of every frame block of parameter vector x."""
    off = flat.param_offsets()
    Rs = []
    for f, d in enumerate(flat.frame_dof):
        o = off[f]
        Rs.append(ra_oracle.exp_so3(x[o:o + 3])[0] if d == 3 else ra_oracle.rot_y(x[o])[0])
    return np.stack(Rs)


def max_error_deg(flat, x, gt):
    """Largest angle between estimated and true frame rotations after removing the global rotation fixed by the
    gauge: the error of R_i R_g^T against the truth's."""
    Re, Rt = block_rotations(flat, x), block_rotations(flat, gt)
    g = flat.gauge_frame
    D = np.einsum("nij,kj->nik", Re, Re[g]) @ np.einsum("ij,nkj->nik", Rt[g], Rt)
    return np.degrees(np.linalg.norm(ra_oracle.log_so3(D), axis=1)).max()


@pytest.mark.parametrize("gravity", [0.0, 0.5])
def test_without_noise(gravity):
    flat, gt = synthesize_rotation_averaging(40, 8, noise_deg=0.0, outlier_ratio=0.0, seed=3, gravity_fraction=gravity)
    r = ra_oracle.solve(RotationEstimatorOptions(), flat)
    assert r.status == 0
    assert max_error_deg(flat, flat.rotations, gt) < 1e-2


def test_weighted_noise_free_matches_invariant():
    flat, gt = synthesize_rotation_averaging(40, 8, noise_deg=0.0, outlier_ratio=0.0, seed=4)
    a, b = flat.copy(), flat.copy()
    b.pair_reweighting = np.random.default_rng(0).uniform(0.1, 1.0, len(b.pair_frame1))
    ra_oracle.solve(RotationEstimatorOptions(), a)
    ra_oracle.solve(RotationEstimatorOptions(), b)
    assert max_error_deg(a, a.rotations, gt) < 1e-2 and max_error_deg(b, b.rotations, gt) < 1e-2


def test_weighted_reduces_error_with_noisy_low_match_edges():
    rng = np.random.default_rng(5)
    flat, gt = synthesize_rotation_averaging(40, 10, noise_deg=0.2, outlier_ratio=0.0, seed=5)
    P = len(flat.pair_frame1)
    bad = rng.uniform(size=P) < 0.3
    bad[np.arange(0, P, 7)] = False
    flat.pair_R[bad] = ra_oracle.exp_so3(rng.normal(0, np.radians(8.0), (bad.sum(), 3))) @ flat.pair_R[bad]
    opts = RotationEstimatorOptions(max_num_l1_iterations=0)
    uni, wei = flat.copy(), flat.copy()
    wei.pair_reweighting = np.where(bad, 0.05, 1.0)
    ra_oracle.solve(opts, uni)
    ra_oracle.solve(opts, wei)
    assert max_error_deg(wei, wei.rotations, gt) < max_error_deg(uni, uni.rotations, gt)


def test_noise_and_outliers():
    flat, gt = synthesize_rotation_averaging(50, 12, noise_deg=1.0, outlier_ratio=0.1, seed=6)
    r = ra_oracle.solve(RotationEstimatorOptions(), flat)
    assert r.status == 0
    assert max_error_deg(flat, flat.rotations, gt) < 3.0


def test_estimated_cameras_without_noise_stay_at_the_solution():
    """Estimated cam_from_rig blocks started where the reference's rig initialisation puts them on noise-free data
    (the truth): the solve keeps them there.  UpdateState's camera update averages the step over the camera's frames,
    which does not converge from far away on its own; the reference starts the final solve from the preliminary one."""
    flat, gt = synthesize_rotation_averaging(30, 10, noise_deg=0.0, outlier_ratio=0.0, seed=7, num_cameras=2,
                                            init_noise_deg=0.0)
    r = ra_oracle.solve(RotationEstimatorOptions(), flat)
    assert r.status == 0
    assert max_error_deg(flat, flat.rotations, gt) < 1e-2
    off = flat.param_offsets()[len(flat.frame_dof):]
    for o in off:
        R = ra_oracle.exp_so3(flat.rotations[o:o + 3])[0].T @ ra_oracle.exp_so3(gt[o:o + 3])[0]
        assert np.degrees(np.linalg.norm(ra_oracle.log_so3(R))) < 1e-2


def test_ridge_regularization_does_not_bias_solution():
    flat, gt = synthesize_rotation_averaging(40, 8, noise_deg=0.5, outlier_ratio=0.0, seed=8)
    a, b = flat.copy(), flat.copy()
    ra_oracle.solve(RotationEstimatorOptions(ridge_regularization=0.0), a)
    ra_oracle.solve(RotationEstimatorOptions(ridge_regularization=1e-9), b)
    Ra, Rb = block_rotations(a, a.rotations), block_rotations(b, b.rotations)
    d = np.linalg.norm(ra_oracle.log_so3(np.einsum("nji,njk->nik", Ra, Rb)), axis=1)
    assert np.degrees(d).max() < 1e-3


def test_disconnected_without_ridge_fails_factorisation():
    # frames 0-5 (with the gauge) and the pair 6-7 on its own: the L1 matrix of the pair's block is [[1, -1], [-1, 1]]
    # per axis, whose last pivot is 1 - 1 = 0 exactly
    flat, _ = synthesize_rotation_averaging(8, 6, noise_deg=0.0, outlier_ratio=0.0, seed=9, banded=True)
    keep = ~((flat.pair_frame1 <= 5) & (flat.pair_frame2 >= 6))
    for k in ("pair_frame1", "pair_frame2", "pair_dof", "pair_R"):
        setattr(flat, k, getattr(flat, k)[keep])
    before = flat.rotations.copy()
    r = ra_oracle.solve(RotationEstimatorOptions(ridge_regularization=0.0), flat)
    assert r.status == ra_oracle.FACTORIZATION_FAILED
    assert np.array_equal(flat.rotations, before)


@pytest.mark.parametrize("gravity", [False, True])
def test_normal_matrix_splits_by_axis(gravity):
    """blockdiag(M_xz, M_y, M_xz) after the permutation, exactly, with M_y = M_xz without 1-DOF frames."""
    flat, _ = synthesize_rotation_averaging(30, 8, seed=10, gravity_fraction=0.5 if gravity else 0.0, num_cameras=0 if gravity else 2,
                                            reweighting=True)
    w = np.random.default_rng(1).uniform(0.1, 2.0, len(flat.pair_frame1))
    M, xs, zs, ys = ra_oracle.axis_split(flat, w, 1e-9)
    perm = np.concatenate([xs, ys, zs])
    assert sorted(perm.tolist()) == list(range(M.shape[0]))
    Mp = M[np.ix_(perm, perm)]
    nx, ny = len(xs), len(ys)
    Mxz, My = M[np.ix_(xs, xs)], M[np.ix_(ys, ys)]
    expect = np.zeros_like(Mp)
    expect[:nx, :nx] = Mxz
    expect[nx:nx + ny, nx:nx + ny] = My
    expect[nx + ny:, nx + ny:] = Mxz
    assert np.array_equal(Mp, expect)
    assert np.array_equal(M[np.ix_(zs, zs)], Mxz)
    if not gravity:
        assert np.array_equal(My, Mxz)
    else:
        assert ny > nx


def test_empty_pose_graph():
    """A single frame and no pairs: the gauge alone, nothing moves."""
    flat = FlatRotationAveraging(frame_dof=[3], rotations=[0.1, 0.2, 0.3], pair_frame1=np.zeros(0), pair_frame2=np.zeros(0),
                                 pair_dof=np.zeros(0), pair_R=np.zeros((0, 3, 3)), gauge_rotation=[0.1, 0.2, 0.3])
    r = ra_oracle.solve(RotationEstimatorOptions(), flat)
    assert r.status == 0
    assert np.allclose(flat.rotations, [0.1, 0.2, 0.3], atol=1e-12)


# ------------------------------------------------------------------------------------------------ host checks (C-ABI)
def _small():
    return synthesize_rotation_averaging(8, 4, seed=11, gravity_fraction=0.5, num_cameras=1)[0]


def _break(flat, what):
    if what == "frame_range":
        flat.pair_frame2[0] = len(flat.frame_dof)
    elif what == "camera_range":
        flat.pair_cam1 = np.full(len(flat.pair_frame1), -1, np.int32)
        flat.pair_cam1[0] = 5
    elif what == "nonfinite_rotation":
        flat.rotations[0] = np.nan
    elif what == "nonfinite_R":
        p = int(np.nonzero(flat.pair_dof == 3)[0][0])
        flat.pair_R[p, 0, 0] = np.inf
    elif what == "one_dof_pair_on_three_dof_frame":
        p = int(np.nonzero((flat.frame_dof[flat.pair_frame1] == 3))[0][0])
        flat.pair_dof[p] = 1
        flat.pair_angle = np.zeros(len(flat.pair_frame1))
        flat.pair_xz_error = np.zeros(len(flat.pair_frame1))
    elif what == "bad_dof":
        flat.frame_dof[0] = 2
    elif what == "gauge_range":
        flat.gauge_frame = -1
    elif what == "negative_reweighting":
        flat.pair_reweighting = np.ones(len(flat.pair_frame1))
        flat.pair_reweighting[0] = -1
    elif what == "camera_without_frames":
        flat.cam_frame_start = np.array([0, 0], np.int32)
    return flat


@pytest.mark.parametrize("what", ["frame_range", "camera_range", "nonfinite_rotation", "nonfinite_R",
                                  "one_dof_pair_on_three_dof_frame", "bad_dof", "gauge_range", "negative_reweighting",
                                  "camera_without_frames"])
def test_host_checks_refuse(what):
    flat = _break(_small(), what)
    before = flat.rotations.copy()
    with pytest.raises(RotationAveragingError) as e:
        solve_flat(RotationEstimatorOptions(), flat)
    assert e.value.code == ERR_INPUT
    assert np.array_equal(flat.rotations, before, equal_nan=True)


def test_underdetermined_is_reported_before_device_work():
    flat = FlatRotationAveraging(frame_dof=[3, 3, 3], rotations=np.zeros(9), pair_frame1=[0], pair_frame2=[1],
                                 pair_dof=[3], pair_R=np.eye(3)[None])
    s = solve_flat(RotationEstimatorOptions(), flat)
    assert s.status == UNDERDETERMINED and s.l1_ms == 0.0
    assert np.array_equal(flat.rotations, np.zeros(9))


def test_refuses_above_dense_envelope_before_device_work():
    F = 32769
    flat = FlatRotationAveraging(frame_dof=np.full(F, 3), rotations=np.zeros(3 * F), pair_frame1=np.arange(F - 1),
                                 pair_frame2=np.arange(1, F), pair_dof=np.full(F - 1, 3), pair_R=np.tile(np.eye(3), (F - 1, 1, 1)))
    with pytest.raises(RotationAveragingError) as e:
        solve_flat(RotationEstimatorOptions(), flat)
    assert e.value.code == ERR_TOO_LARGE and "32768" in str(e.value)


def test_abi_surface():
    lib = _bind(load_library())
    o = _COptions()
    lib.b200ra_options_init(ctypes.byref(o))
    assert (o.max_num_l1_iterations, o.l1_step_convergence_threshold) == (5, 1e-3)
    assert (o.max_num_irls_iterations, o.irls_step_convergence_threshold) == (100, 1e-3)
    assert (o.irls_loss_parameter_sigma, o.ridge_regularization, o.weight_type, o.gpu_index) == (5.0, 1e-9, 0, -1)
    d = RotationEstimatorOptions()
    assert (d.max_num_l1_iterations, d.max_num_irls_iterations, d.irls_loss_parameter_sigma) == (5, 100, 5.0)
    assert lib.b200ra_solve(None, None, None) == ERR_INPUT
    assert b"null" in lib.b200ra_last_error()


# Fingerprints of synthesize_rotation_averaging's output before it took gravity_frames: the sha256 (first 16 hex
# digits) of the integer arrays and the gauge frame, and position-weighted sums of the float arrays and of the ground
# truth.  Every seeded test of rotation averaging depends on the generator drawing the same problem.  The sums are held
# to 1e-12 rather than bit for bit because numpy's sin and cos may round differently on another CPU's vector path; a
# shifted random stream changes them at order one.
GENERATOR_FINGERPRINTS = [
    (dict(num_frames=40, edges_per_frame=10, seed=0), "b14fb02df765afb1",
     [-36.70610160086049, -143.12507364371217, None, None, None, 6.836943981730275, -40.30174016915096]),
    (dict(num_frames=40, edges_per_frame=10, seed=4, gravity_fraction=0.5, reweighting=True), "340fbce35dbf0ac0",
     [57.509937664096704, 4.666506638549784, -137.91220028047866, 0.015874411227268525, 432.13480265498293,
      2.042467344288341, 73.46017945934442]),
    (dict(num_frames=40, edges_per_frame=10, seed=8, num_cameras=2), "451bd0199076fbf9",
     [-109.47876209816344, 42.05142967599167, None, None, None, 4.799817268449409, -137.79830597548076]),
    (dict(num_frames=300, edges_per_frame=12, seed=21, gravity_fraction=0.3, num_cameras=3), "908081079806de4e",
     [126.31189741057753, 501.38762674331446, 22.20029283174202, 0.1992239450052575, None, 5.612510932101304,
      59.195283003961485]),
    (dict(num_frames=8, edges_per_frame=6, noise_deg=0.0, outlier_ratio=0.0, seed=9, banded=True), "273ec9bb555e94ac",
     [-28.99511339041858, 102.66577459317047, None, None, None, -7.180252214228349, -24.870489115164464]),
    (dict(num_frames=200, edges_per_frame=20, seed=5, gravity_fraction=0.3, reweighting=True, banded=True),
     "9523d2f07442448d", [20.446003488378643, 626.184500360099, -69.31777356063616, 0.21922994939722318,
                          4099.673593695615, -4.440329584599022, 64.85640659222202]),
]
_INT_FIELDS = ("frame_dof", "pair_frame1", "pair_frame2", "pair_dof", "pair_cam1", "pair_cam2", "cam_frame_start", "cam_frames")
_FLOAT_FIELDS = ("rotations", "pair_R", "pair_angle", "pair_xz_error", "pair_reweighting", "gauge_rotation")


def _generator_fingerprint(flat, gt):
    h = hashlib.sha256()
    for k in _INT_FIELDS:
        a = getattr(flat, k)
        h.update(b"-" if a is None else np.ascontiguousarray(a).tobytes())
    h.update(str(flat.gauge_frame).encode())
    sums = []
    for a in [getattr(flat, k) for k in _FLOAT_FIELDS] + [gt]:
        sums.append(None if a is None else float(np.dot(a.reshape(-1), 1.0 + np.arange(a.size) % 7)))
    return h.hexdigest()[:16], sums


def _same_problem(a, b):
    for k in _INT_FIELDS + _FLOAT_FIELDS:
        x, y = getattr(a, k), getattr(b, k)
        assert (x is None) == (y is None), k
        if x is not None:
            assert x.dtype == y.dtype and np.array_equal(x.view(np.uint8), y.view(np.uint8)), k
    assert (a.gauge_frame, a.num_cameras) == (b.gauge_frame, b.num_cameras)


@pytest.mark.parametrize("case", range(len(GENERATOR_FINGERPRINTS)))
def test_generator_unchanged_by_gravity_frames(case):
    """The default draws the problem it drew before gravity_frames existed, and passing the mask the default would
    draw reproduces the default output bit for bit (the argument does not shift the random stream)."""
    kw, digest, sums = GENERATOR_FINGERPRINTS[case]
    flat, gt = synthesize_rotation_averaging(**kw)
    d, s = _generator_fingerprint(flat, gt)
    assert d == digest
    assert [x is None for x in s] == [x is None for x in sums]
    np.testing.assert_allclose([x for x in s if x is not None], [x for x in sums if x is not None], rtol=1e-12, atol=0)
    flat2, gt2 = synthesize_rotation_averaging(**kw, gravity_frames=flat.frame_dof == 1)
    _same_problem(flat, flat2)
    assert np.array_equal(gt.view(np.uint64), gt2.view(np.uint64))


def test_generator_gravity_frames_sets_exact_axis_sizes():
    F = 129
    mask = np.zeros(F, bool)
    mask[[0, 5, 64, 127, 128]] = True
    flat, _ = synthesize_rotation_averaging(F, 10, seed=1, gravity_frames=mask)
    assert np.array_equal(flat.frame_dof == 1, mask)
    assert flat.gauge_frame == 0
    one = mask[flat.pair_frame1] & mask[flat.pair_frame2]
    assert np.array_equal(flat.pair_dof == 1, one)
    allg, _ = synthesize_rotation_averaging(20, 6, seed=1, gravity_frames=np.ones(20, bool))
    assert (allg.frame_dof == 1).all() and (allg.pair_dof == 1).all() and allg.num_params == 20
    with pytest.raises(ValueError):
        synthesize_rotation_averaging(F, 10, seed=1, gravity_frames=mask[:-1])
