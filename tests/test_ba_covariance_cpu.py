"""Bundle-adjustment covariance on the CPU: the two oracle statements (tests/oracle_cov.py) against each other on the
reference's covariance test grid (covariance_test.cc:64-323), the block sizes of masked poses, and the Rigid3d
uncertainty-propagation helpers (rigid3_test.cc:160-274)."""
import numpy as np
import pytest

import oracle_ba
import oracle_cov
from colmap_b200.bundle_adjustment import (FULL_OPENCV, RAD_TAN_THIN_PRISM_FISHEYE, BundleAdjustmentConfig, BundleAdjustmentOptions,
                                           GetCovarianceForComposedRigid3d,
                                           GetCovarianceForRelativeRigid3d, GetCovarianceForRigid3dInverse, flatten_reconstruction,
                                           rigid3d_adjoint, rigid3d_adjoint_inverse, rigid3d_inverse)
from colmap_b200.synthetic import synthesize_ba_problem, synthesize_rig_reconstruction

# (params, fixed_points, fixed_cam_poses, fixed_cam_intrinsics): the seven cases of the reference's test
GRID = [(oracle_cov.ALL, False, False, False), (oracle_cov.ALL, True, False, False), (oracle_cov.ALL, False, False, True),
        (oracle_cov.ALL, False, True, False), (oracle_cov.POINTS, False, False, False), (oracle_cov.POSES, False, False, False),
        (oracle_cov.POSES_AND_POINTS, False, False, False)]


def reference_scene(fixed_points, fixed_cam_poses, fixed_cam_intrinsics, solve=None):
    """The reference test's scene (1 rig, 1 camera, 7 frames, 200 points, 0.01 px noise, 3 constant points), flattened and
    solved (by the oracle unless `solve` is given)."""
    rec = synthesize_rig_reconstruction(1, 1, 7, 200, point2D_stddev=0.01, seed=3)
    cfg = BundleAdjustmentConfig()
    for image_id, im in rec.images.items():
        cfg.AddImage(image_id)
        if fixed_cam_poses:
            cfg.SetConstantRigFromWorldPose(im.frame_id)
        if fixed_cam_intrinsics:
            cfg.SetConstantCamIntrinsics(im.camera_id)
    for n, pid in enumerate(sorted(rec.points3D)):
        if n < 3 or fixed_points:
            cfg.AddConstantPoint(pid)
    options = BundleAdjustmentOptions()
    flat = flatten_reconstruction(options, cfg, rec)[0]
    (solve or oracle_ba.solve)(options, flat)
    return options, flat


@pytest.mark.parametrize("case", GRID, ids=lambda c: f"params{c[0]}-pts{int(c[1])}-poses{int(c[2])}-intr{int(c[3])}")
def test_oracle_statements_agree(case):
    params, fp, fpose, fint = case
    options, flat = reference_scene(fp, fpose, fint)
    est, msg = oracle_cov.estimate(options, flat, params)
    assert est is not None, msg
    ref = oracle_cov.ceres_semantics(options, flat, params)
    assert set(est) == set(ref)
    kinds = {k[0] for k in est}
    assert ("point" in kinds) == (params != oracle_cov.POSES and not fp)
    assert ("pose" in kinds) == (params != oracle_cov.POINTS and not fpose)
    assert ("camera" in kinds) == (params == oracle_cov.ALL and not fint)
    for k in est:
        assert est[k].shape == ref[k].shape
        assert np.abs(est[k] - ref[k]).max() <= 1e-8, (k, np.abs(est[k] - ref[k]).max())
    if ("pose", 0) in est:
        assert est[("pose", 0)].shape == (6, 6)
    if ("point", 10) in est:
        assert est[("point", 10)].shape == (3, 3)


def test_masked_pose_sizes():
    """A two-cams gauge pose has 5 tangent dimensions, a pose under constant_rig_from_world_rotation 3; constant blocks
    have none."""
    gt, flat = synthesize_ba_problem(6, 150, 4, seed=7)
    flat.pose_constant = flat.pose_constant.copy(); flat.pose_fixed_dim = flat.pose_fixed_dim.copy()
    flat.pose_constant[0] = 1
    flat.pose_fixed_dim[1] = 2
    est, msg = oracle_cov.estimate(BundleAdjustmentOptions(), flat, oracle_cov.ALL)
    assert est is not None, msg
    assert ("pose", 0) not in est and est[("pose", 1)].shape == (5, 5) and est[("pose", 2)].shape == (6, 6)
    assert est[("cross", 1, 2)].shape == (5, 6)
    o = BundleAdjustmentOptions(constant_rig_from_world_rotation=True)
    flat.pose_fixed_dim[1] = -1
    est, msg = oracle_cov.estimate(o, flat, oracle_cov.POSES)
    assert est is not None, msg
    assert est[("pose", 1)].shape == (3, 3) and ("camera", 1) not in est


def weak_intrinsics_scene(name, solve):
    """(options, flat): wide-model scenes, solved by `solve`, under a two-cams gauge, whose intrinsics are weakly
    determined (FULL_OPENCV: k1 against the rational k4) while the poses are not.  The reference eliminates the intrinsics
    and rank-tests only the reduced pose matrix, so the POSES modes are estimable and ALL is not."""
    if name == "full_opencv":
        _, flat = synthesize_ba_problem(12, 600, 6, models=(FULL_OPENCV,), seed=11, point2D_stddev=0.5)
        options = BundleAdjustmentOptions()
    else:
        _, flat = synthesize_ba_problem(16, 1200, 8, models=(RAD_TAN_THIN_PRISM_FISHEYE,), seed=11, point2D_stddev=0.5)
        options = BundleAdjustmentOptions(refine_principal_point=True)
    flat.pose_constant = flat.pose_constant.copy(); flat.pose_fixed_dim = flat.pose_fixed_dim.copy()
    flat.pose_constant[0] = 1
    flat.pose_fixed_dim[1] = int(np.argmax(np.abs(flat.poses[1, 4:] - flat.poses[0, 4:])))
    solve(options, flat)
    return options, flat


def test_weak_intrinsics_scene_still_tests_the_rank_test_rows():
    """Keeps the FULL_OPENCV scene of the GPU POSES-mode tests a case where the rows of the rank test matter: the
    reference estimates the pose covariances, while a rank test over all rows of S in the [others | poses] order (damping
    on the others) would stop at an intrinsics pivot <= 1e-6."""
    options, flat = weak_intrinsics_scene("full_opencv", oracle_ba.solve)
    jac = oracle_cov.jacobian(options, flat)
    est, msg = oracle_cov.estimate(options, flat, oracle_cov.POSES, jac=jac)
    assert est is not None, msg
    S, npose = oracle_cov.reduced_matrix(jac)
    order = np.r_[npose:len(S), :npose]
    S = S[np.ix_(order, order)]
    no = len(S) - npose
    S[np.arange(no), np.arange(no)] += 1e-8
    pivots = np.diag(np.linalg.cholesky(S)) ** 2
    assert pivots[:no].min() <= 1e-6 and pivots[no:].min() > 1e-6, (pivots[:no].min(), pivots[no:].min())


def test_unfixed_gauge_not_estimable():
    gt, flat = synthesize_ba_problem(6, 150, 4, seed=7)
    est, msg = oracle_cov.estimate(BundleAdjustmentOptions(), flat, oracle_cov.ALL)
    assert est is None and msg


# ---- Rigid3d helpers (rigid3_test.cc:160-274)
def _random_rigid(rng):
    q = rng.normal(size=4)
    return np.concatenate([q / np.linalg.norm(q), rng.normal(size=3)])


def _random_cov(rng, n):
    A = rng.uniform(-1, 1, (n, n))
    return A @ A.T


def test_rigid3d_adjoint():
    rng = np.random.default_rng(0)
    b_from_a = _random_rigid(rng)
    assert np.allclose(rigid3d_adjoint(b_from_a) @ rigid3d_adjoint_inverse(b_from_a), np.eye(6), atol=1e-6)
    assert np.allclose(rigid3d_adjoint_inverse(b_from_a), rigid3d_adjoint(rigid3d_inverse(b_from_a)), atol=1e-6)


def test_covariance_for_inverse():
    rng = np.random.default_rng(1)
    b_from_a, cov = _random_rigid(rng), _random_cov(rng, 6)
    back = GetCovarianceForRigid3dInverse(rigid3d_inverse(b_from_a), GetCovarianceForRigid3dInverse(b_from_a, cov))
    assert np.allclose(back, cov, atol=1e-6)


def test_covariance_for_relative_perfect_correlation():
    rng = np.random.default_rng(2)
    world_from_a, world_from_b, sub = _random_rigid(rng), _random_rigid(rng), _random_cov(rng, 6)
    cov_world = np.block([[sub, sub], [sub, sub]])
    J0 = np.zeros((12, 12))
    J0[:6, :6] = -rigid3d_adjoint_inverse(world_from_a)
    J0[6:, 6:] = -rigid3d_adjoint_inverse(world_from_b)
    rel = GetCovarianceForRelativeRigid3d(rigid3d_inverse(world_from_a), rigid3d_inverse(world_from_b), J0 @ cov_world @ J0.T)
    assert np.linalg.norm(rel) < 1e-6


def test_covariance_for_relative_matches_right_convention():
    rng = np.random.default_rng(3)
    a_from_world, b_from_world, cov = _random_rigid(rng), _random_rigid(rng), _random_cov(rng, 12)
    ours = GetCovarianceForRelativeRigid3d(a_from_world, b_from_world, cov)
    J0 = np.zeros((12, 12))
    J0[:6, :6] = -rigid3d_adjoint_inverse(a_from_world)
    J0[6:, 6:] = np.eye(6)
    J = np.hstack([rigid3d_adjoint(b_from_world), np.eye(6)])
    assert np.allclose(ours, J @ (J0 @ cov @ J0.T) @ J.T, atol=1e-6)


def test_covariance_composed_vs_relative():
    rng = np.random.default_rng(4)
    a_from_b, b_from_c, cov = _random_rigid(rng), _random_rigid(rng), _random_cov(rng, 12)
    composed = GetCovarianceForComposedRigid3d(a_from_b, cov)
    J0 = np.zeros((12, 12))
    J0[6:, :6] = np.eye(6)
    J0[:6, 6:] = -rigid3d_adjoint_inverse(b_from_c)
    relative = GetCovarianceForRelativeRigid3d(rigid3d_inverse(b_from_c), a_from_b, J0 @ cov @ J0.T)
    assert np.allclose(composed, relative, atol=1e-6)
