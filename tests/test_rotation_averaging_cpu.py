"""Rotation averaging without a GPU: the fp64 oracle (tests/ra_oracle.py) on synthetic pose graphs with the bars of the
reference's rotation_averaging_test.cc, the exact per-axis split of the normal matrix that the GPU factors, the host
input checks of b200ra_solve, which refuse before any device work, and the ABI surface."""
import ctypes

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
