"""Rotation averaging on the GPU against the fp64 oracle (tests/ra_oracle.py) at axis sizes past one 64-row tile of the
dense factorisation and triangular solves, with the bars of test_rotation_averaging_gpu.compare (the same iteration
and ADMM counts, average steps within 1e-8 relative, rotations within 1e-8 rad).  Each case asserts the axis sizes
n_xz (the x/z matrix: 3-DOF frames and cameras) and n_y (every block) it is meant to reach: multi-tile ADMM, the gravity
layout with two matrices of different padding, axes exactly at and one past a tile multiple, the y-only problem, the
CTA-strided camera average over more than 128 frames, rotations and 1-DOF residuals at the +-pi wrap, and failed
factorisations whose bad pivot lies past the first tile or only in the y matrix."""
import numpy as np
import pytest

import ra_oracle
from colmap_b200.rotation_averaging import (FACTORIZATION_FAILED, GEMAN_MCCLURE, HALF_NORM, SUCCESS,
                                            RotationEstimatorOptions, solve_flat)
from colmap_b200.synthetic import synthesize_rotation_averaging
from test_rotation_averaging_gpu import compare

pytestmark = pytest.mark.gpu


def opts(**kw):
    return RotationEstimatorOptions(gpu_index=0, **kw)


def gravity_mask(F, frames):
    m = np.zeros(F, bool)
    m[list(frames)] = True
    return m


def axis_sizes(flat):
    n_xz = int((flat.frame_dof == 3).sum()) + flat.num_cameras
    return n_xz, len(flat.frame_dof) + flat.num_cameras


def check(flat, n_xz, n_y, o=None, **bars):
    assert axis_sizes(flat) == (n_xz, n_y)
    s, g = compare(o or opts(), flat, **bars)
    assert (s.n_xz, s.n_y) == (n_xz, n_y)
    return s, g


def test_l1_and_irls_all_3dof_1000_frames():
    """16 tiles per axis, one matrix with 3 right-hand sides, through the ADMM phase."""
    flat, _ = synthesize_rotation_averaging(1000, 10, seed=31)
    s, _ = check(flat, 1000, 1000)
    assert s.num_l1_iterations >= 1 and len(s.admm_iterations) >= 1


def test_gravity_two_matrices_different_tile_counts():
    """Every other frame gravity-aligned: M_xz of 100 (2 tiles, 2 right-hand sides) and M_y of 200 (4 tiles, 1)."""
    flat, _ = synthesize_rotation_averaging(200, 12, seed=32, gravity_frames=np.arange(200) % 2 == 1)
    check(flat, 100, 200)


@pytest.mark.parametrize("F,n_gravity", [(65, 1), (192, 65)], ids=["xz64_y65", "xz127_y192"])
def test_gravity_at_exact_tile_edges(F, n_gravity):
    """One matrix exactly at a tile multiple (no padding) and the other one row past one (63 padding rows), or the other
    way round."""
    mask = gravity_mask(F, np.random.default_rng(F).choice(F, n_gravity, replace=False))
    flat, _ = synthesize_rotation_averaging(F, 12, seed=33, gravity_frames=mask)
    check(flat, F - n_gravity, F)


@pytest.mark.parametrize("F", [128, 129])
def test_same_y_at_exact_tile_edges(F):
    """All 3-DOF: an unpadded M_xz of 128 (the padding identity is not built) and one row past two tiles."""
    flat, _ = synthesize_rotation_averaging(F, 12, seed=34)
    check(flat, F, F)


def test_all_gravity_y_only():
    """Every frame 1-DOF: no x/z matrix at all (n_xz = 0), 3 tiles of M_y."""
    flat, _ = synthesize_rotation_averaging(150, 12, seed=35, gravity_frames=np.ones(150, bool))
    assert (flat.pair_dof == 1).all()
    check(flat, 0, 150)


def test_estimated_cameras_strided_average():
    """3 estimated cameras, each averaged over about 330 frames: three passes of the 128-thread CTA's strided loop."""
    flat, _ = synthesize_rotation_averaging(400, 20, seed=36, num_cameras=3)
    lengths = np.diff(flat.cam_frame_start)
    assert (lengths > 2 * 128).all(), lengths
    check(flat, 403, 403)


def test_camera_list_lengths():
    """Camera frame lists of exactly 1, 128, 129 and 257 frames: the one-frame average, one full pass, one frame into
    the second pass and one into the third.  The flat problem takes any list; the oracle reads the same one."""
    flat, _ = synthesize_rotation_averaging(300, 20, seed=37, num_cameras=4)
    rng = np.random.default_rng(37)
    lists = []
    for c, L in enumerate((1, 128, 129, 257)):
        linked = np.unique(np.concatenate([flat.pair_frame1[flat.pair_cam1 == c], flat.pair_frame2[flat.pair_cam2 == c]]))
        rest = np.setdiff1d(np.arange(300), linked)
        lists.append(np.sort(np.concatenate([linked, rng.permutation(rest)])[:L]))
    flat.cam_frame_start = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)
    flat.cam_frames = np.concatenate(lists).astype(np.int32)
    assert np.diff(flat.cam_frame_start).tolist() == [1, 128, 129, 257]
    check(flat, 304, 304)


# angle-axis vectors within 1e-7 rad of pi about x, y, z and a diagonal axis (Eigen's quaternion from a matrix of trace
# <= 0 takes the x, y or z branch), some just past pi; frame 0 is the gauge
_DIAG = np.array([1.0, 1.0, 1.0]) / np.sqrt(3.0)
NEAR_PI = {0: (np.pi - 2e-8) * np.array([1.0, -2.0, 0.5]) / np.sqrt(5.25),
           70: (np.pi - 1e-7) * np.array([1.0, 0.0, 0.0]), 71: (np.pi + 5e-8) * np.array([0.0, 1.0, 0.0]),
           140: (np.pi - 3e-8) * np.array([0.0, 0.0, 1.0]), 141: (np.pi + 1e-8) * np.array([0.0, 0.0, -1.0]),
           199: (np.pi - 1e-8) * _DIAG}


def test_rotations_near_pi():
    """Frames whose ground truth and initial rotation lie within 1e-7 rad of pi: UpdateState's R exp(-step) crosses pi
    (the angle-axis vector flips to the other side), and the residuals and the gauge take Eigen's trace <= 0 branches.
    The pairs are regenerated from the changed ground truth with 1 degree of noise."""
    flat, gt = synthesize_rotation_averaging(200, 12, seed=38)
    rng = np.random.default_rng(38)
    R = ra_oracle.exp_so3(gt.reshape(-1, 3))
    x0 = flat.rotations.reshape(-1, 3).copy()
    for f, w in NEAR_PI.items():
        R[f] = ra_oracle.exp_so3(w)[0]
        x0[f] = w
    f1, f2 = flat.pair_frame1, flat.pair_frame2
    flat.pair_R = ra_oracle.exp_so3(rng.normal(0, np.radians(1.0), (len(f1), 3))) @ R[f2] @ np.transpose(R[f1], (0, 2, 1))
    flat.rotations = x0.reshape(-1)
    flat.gauge_rotation = NEAR_PI[0].copy()
    assert flat.gauge_frame == 0
    traces = np.trace(ra_oracle.exp_so3(np.stack(list(NEAR_PI.values()))), axis1=1, axis2=2)
    assert (traces < -0.99).all()
    check(flat, 200, 200)


def test_1dof_residuals_near_pi():
    """1-DOF pairs whose initial residual remainder((a2 - a1) - angle, 2 pi) sits within 0.01 of +pi or -pi, on both
    sides of the wrap.  The reference jitters such residuals at random; neither the GPU nor the oracle does."""
    flat, _ = synthesize_rotation_averaging(200, 12, seed=39, gravity_frames=np.arange(200) % 2 == 0)
    one = np.nonzero(flat.pair_dof == 1)[0]
    off = flat.param_offsets()
    x = flat.rotations
    targets = [np.pi - 0.005, np.pi - 0.0005, -np.pi + 0.006, -np.pi + 0.001]
    picks = np.random.default_rng(39).choice(one, 4 * len(targets), replace=False)
    for k, p in enumerate(picks):
        t = targets[k % len(targets)] + (2 * np.pi if k % 8 >= 4 else 0.0)   # also the equivalent angle one turn away
        flat.pair_angle[p] = (x[off[flat.pair_frame2[p]]] - x[off[flat.pair_frame1[p]]]) - t
    pr = ra_oracle.Problem(flat)
    pr.compute_residuals()
    r = pr.res[pr.roff[picks]]
    assert (np.pi - np.abs(r) <= 0.01).all() and (r > 0).any() and (r < 0).any(), r
    check(flat, 100, 200)


def _isolated_pair(gravity_frames=None):
    """102 frames on a banded graph with the pair 100-101 cut off from the rest: with ridge 0 the L1 matrix of that pair
    is [[1, -1], [-1, 1]] per axis, whose second pivot is exactly 0 (row 101, in the second tile)."""
    flat, _ = synthesize_rotation_averaging(102, 6, noise_deg=0.0, outlier_ratio=0.0, seed=40, banded=True,
                                            gravity_frames=gravity_frames)
    keep = ~((flat.pair_frame1 <= 99) & (flat.pair_frame2 >= 100))
    for k in ("pair_frame1", "pair_frame2", "pair_dof", "pair_R", "pair_angle", "pair_xz_error"):
        if getattr(flat, k) is not None:
            setattr(flat, k, getattr(flat, k)[keep])
    return flat


def _fails_like_the_oracle(flat, o):
    before = flat.rotations.copy()
    s = solve_flat(o, flat)
    so = ra_oracle.solve(o, flat.copy())
    assert s.status == so.status == FACTORIZATION_FAILED
    assert np.array_equal(flat.rotations.view(np.uint64), before.view(np.uint64))
    return s


def test_factorisation_failure_past_tile_0():
    flat = _isolated_pair()
    s = _fails_like_the_oracle(flat, opts(ridge_regularization=0.0))
    assert (s.n_xz, s.n_y) == (102, 102)


def test_factorisation_failure_only_in_y():
    """Frames 0, 100 and 101 gravity-aligned: frame 0 is the gauge, the 1-DOF pair 100-101 lives only in M_y, so M_xz
    (the 99 3-DOF frames, anchored through frame 0's pairs) factors and M_y fails at its row 101."""
    flat = _isolated_pair(gravity_mask(102, (0, 100, 101)))
    assert flat.gauge_frame == 0
    M, xs, _, ys = ra_oracle.axis_split(flat, np.ones(len(flat.pair_frame1)), 0.0)
    np.linalg.cholesky(M[np.ix_(xs, xs)])                                         # M_xz is positive definite
    assert np.linalg.matrix_rank(M[np.ix_(ys, ys)]) == len(ys) - 1                # M_y is singular
    s = _fails_like_the_oracle(flat, opts(ridge_regularization=0.0))
    assert (s.n_xz, s.n_y) == (99, 102)


@pytest.mark.parametrize("weight", [GEMAN_MCCLURE, HALF_NORM])
def test_reweighting_and_weights_past_one_tile(weight):
    """Per-pair reweighting with 30% gravity frames.  HALF_NORM compares at most two IRLS iterations with the 1e-4 /
    1e-5 bars of test_gpu_matches_oracle, for the conditioning reason given there."""
    flat, _ = synthesize_rotation_averaging(200, 12, seed=41, gravity_fraction=0.3, reweighting=True)
    n_xz = int((flat.frame_dof == 3).sum())
    assert 64 < n_xz < 192
    tight = weight == GEMAN_MCCLURE
    o = opts(weight_type=weight, max_num_irls_iterations=100 if tight else 2)
    check(flat, n_xz, 200, o, step_rtol=1e-8 if tight else 1e-4, rot_tol=1e-8 if tight else 1e-5)


def test_half_norm_zero_residual_fails():
    """An exactly consistent 1-DOF pair with xz_error 0 has e2 = 0 and the HALF_NORM weight pow(0, -0.75) = inf.  The
    weight is not NaN, so both solves go on to factor.  On the GPU the inf pivot passes, the elimination turns its
    column into NaN (-inf * 0) and the next pivot fails; the oracle's SuperLU reports the matrix exactly singular.  Both
    report FACTORIZATION_FAILED and the rotations are kept."""
    flat, _ = synthesize_rotation_averaging(200, 12, seed=42, gravity_frames=np.arange(200) % 2 == 0)
    p = int(np.nonzero(flat.pair_dof == 1)[0][0])
    off = flat.param_offsets()
    flat.pair_angle[p] = flat.rotations[off[flat.pair_frame2[p]]] - flat.rotations[off[flat.pair_frame1[p]]]
    flat.pair_xz_error[p] = 0.0
    s = _fails_like_the_oracle(flat, opts(max_num_l1_iterations=0, weight_type=HALF_NORM))
    assert s.num_irls_iterations == 0 and (s.n_xz, s.n_y) == (100, 200)
