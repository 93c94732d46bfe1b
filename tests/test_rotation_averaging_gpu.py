"""Rotation averaging on the GPU against the fp64 oracle (tests/ra_oracle.py) from identical flat problems: the
iteration counts of both phases, the ADMM iterations, the average step of every iteration, the final rotations,
determinism, a failed factorisation, and one problem near the dense envelope."""
import itertools

import numpy as np
import pytest

import ra_oracle
from colmap_b200.rotation_averaging import (FACTORIZATION_FAILED, GEMAN_MCCLURE, HALF_NORM, SUCCESS,
                                            RotationEstimatorOptions, solve_flat)
from colmap_b200.synthetic import synthesize_rotation_averaging
from test_rotation_averaging_cpu import max_error_deg

pytestmark = pytest.mark.gpu

PHASES = {"l1": (5, 0), "irls": (0, 25), "both": (5, 25)}
KINDS = {"all3": {}, "gravity": {"gravity_fraction": 0.5}, "cameras": {"num_cameras": 2}}


def rotation_gap(flat, a, b):
    """Largest angle(R_a^T R_b) over all blocks (frames and cameras), in radians."""
    off = flat.param_offsets()
    d = np.concatenate([flat.frame_dof.astype(int), np.full(flat.num_cameras, 3)])
    gap = 0.0
    for k, o in enumerate(off):
        if d[k] == 1:
            gap = max(gap, abs(np.remainder(a[o] - b[o] + np.pi, 2 * np.pi) - np.pi))
        else:
            Ra, Rb = ra_oracle.exp_so3(a[o:o + 3])[0], ra_oracle.exp_so3(b[o:o + 3])[0]
            gap = max(gap, float(np.linalg.norm(ra_oracle.log_so3(Ra.T @ Rb))))
    return gap


def compare(opts, flat, step_rtol=1e-8, rot_tol=1e-8):
    g, o = flat.copy(), flat.copy()
    sg = solve_flat(opts, g)
    so = ra_oracle.solve(opts, o)
    assert sg.status == so.status == SUCCESS
    assert (sg.num_l1_iterations, sg.num_irls_iterations) == (so.num_l1_iterations, so.num_irls_iterations)
    assert sg.admm_iterations.tolist() == list(so.admm_iterations)
    np.testing.assert_allclose(sg.step_history, so.step_history, rtol=step_rtol, atol=0)
    gap = rotation_gap(flat, g.rotations, o.rotations)
    assert gap < rot_tol, gap
    return sg, g


@pytest.mark.parametrize("phase,kind", list(itertools.product(PHASES, KINDS)))
@pytest.mark.parametrize("weight,reweight,ridge", list(itertools.product((GEMAN_MCCLURE, HALF_NORM), (False, True), (0.0, 1e-9))))
def test_gpu_matches_oracle(phase, kind, weight, reweight, ridge):
    l1, irls = PHASES[phase]
    flat, _ = synthesize_rotation_averaging(40, 10, noise_deg=1.0, outlier_ratio=0.1, seed=3 * list(PHASES).index(phase) + list(KINDS).index(kind),
                                            reweighting=reweight, **KINDS[kind])
    if weight == HALF_NORM:
        irls = min(irls, 2)
    opts = RotationEstimatorOptions(max_num_l1_iterations=l1, max_num_irls_iterations=irls, weight_type=weight,
                                    ridge_regularization=ridge, gpu_index=0)
    # HALF_NORM weights |r|^-1.5 span several orders of magnitude between inlier and outlier pairs, so the weighted
    # normal matrix is far worse conditioned than with GEMAN_MCCLURE; a different summation order (dense per-axis
    # matrices here, SuperLU on the full matrix in the oracle) then moves the small late steps by up to a few 1e-6
    # relative (3.0e-6 measured on an H100), hence the wider bars for that weight.  As the solve proceeds the spread
    # grows (an inlier's residual goes to zero and its weight to infinity): after an L1 phase the fifth IRLS step
    # differed by up to 4e-2 relative on an H100, so half-norm cases compare at most two IRLS iterations.
    tight = weight == GEMAN_MCCLURE or irls == 0   # without an IRLS phase the weight type is not used
    s, _ = compare(opts, flat, step_rtol=1e-8 if tight else 1e-4, rot_tol=1e-8 if tight else 1e-5)
    assert s.n_y == len(flat.frame_dof) + flat.num_cameras
    assert s.n_xz == int((flat.frame_dof == 3).sum()) + flat.num_cameras


def test_repeated_solves_are_bit_identical():
    flat, _ = synthesize_rotation_averaging(300, 12, seed=21, gravity_fraction=0.3, num_cameras=3)
    opts = RotationEstimatorOptions(max_num_irls_iterations=10, gpu_index=0)
    outs = []
    for _ in range(2):
        f = flat.copy()
        s = solve_flat(opts, f)
        outs.append((f.rotations, s.step_history))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])


def test_factorisation_failure_leaves_rotations_untouched():
    # frames 0-5 (with the gauge) and the pair 6-7 on its own: the L1 matrix of the pair's block is [[1, -1], [-1, 1]]
    # per axis, whose last pivot is 1 - 1 = 0 exactly
    flat, _ = synthesize_rotation_averaging(8, 6, noise_deg=0.0, outlier_ratio=0.0, seed=9, banded=True)
    keep = ~((flat.pair_frame1 <= 5) & (flat.pair_frame2 >= 6))
    for k in ("pair_frame1", "pair_frame2", "pair_dof", "pair_R"):
        setattr(flat, k, getattr(flat, k)[keep])
    before = flat.rotations.copy()
    s = solve_flat(RotationEstimatorOptions(ridge_regularization=0.0, gpu_index=0), flat)
    assert s.status == FACTORIZATION_FAILED
    assert np.array_equal(flat.rotations.view(np.uint64), before.view(np.uint64))


def test_recovers_ground_truth():
    flat, gt = synthesize_rotation_averaging(500, 20, noise_deg=1.0, outlier_ratio=0.1, seed=22)
    s = solve_flat(RotationEstimatorOptions(gpu_index=0), flat)
    assert s.status == SUCCESS
    assert max_error_deg(flat, flat.rotations, gt) < 3.0


def test_near_the_envelope():
    """32,000 frames (n = 32,000 per axis) over two IRLS iterations.  The banded graph keeps the oracle's sparse
    factorisation small; the GPU factors the dense 32,000 x 32,000 matrix."""
    flat, _ = synthesize_rotation_averaging(32000, 20, noise_deg=1.0, outlier_ratio=0.1, seed=23, banded=True)
    opts = RotationEstimatorOptions(max_num_l1_iterations=0, max_num_irls_iterations=2, gpu_index=0)
    s, _ = compare(opts, flat)
    assert s.n_xz == s.n_y == 32000
