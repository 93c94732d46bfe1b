"""b200ba_estimate_covariance on the GPU against the CPU restatement of covariance.cc (tests/oracle_cov.py), on the same
parameter arrays: the reference's test grid, wide models (camera-block widths DC = 14, 18, 22 and 28) with robust
losses, rigs with variable, constant and unrefined sensors, a two-cams gauge, constant rotations, tracks of 1 to 300
observations, a non-default damping, POSES modes whose eliminated intrinsics are weakly determined or span several
tiles, dense dimensions around the 64-row tile of the factorisation, a multi-tile problem, the not-estimable path and
the Python interface."""
import dataclasses

import numpy as np
import pytest

import oracle_ba
import oracle_cov
from colmap_b200.bundle_adjustment import (CAUCHY, HUBER, OPENCV, SIMPLE_PINHOLE, SIMPLE_RADIAL, SOFT_L1, THIN_PRISM_FISHEYE,
                                           BACovarianceOptions, BundleAdjustmentConfig, BundleAdjustmentOptions,
                                           CovarianceNotEstimable, CreateDefaultBundleAdjuster, EstimateBACovariance,
                                           GetCovarianceForRelativeRigid3d, estimate_covariance_flat, solve_flat)
from colmap_b200.synthetic import synthesize_ba_problem, synthesize_rig_problem, synthesize_rig_reconstruction
from test_ba_covariance_cpu import GRID, reference_scene, weak_intrinsics_scene

pytestmark = pytest.mark.gpu
WORST = {"abs": 0.0, "rel": 0.0}


def _gpu_blocks(cov, keys):
    out = {}
    for k in keys:
        if k[0] == "pose": out[k] = cov.pose(k[1])
        elif k[0] == "point": out[k] = cov.point(k[1])
        elif k[0] == "camera": out[k] = cov.camera(k[1])
        elif k[0] == "sensor": out[k] = cov.sensor(k[1])
        else: out[k] = cov.pose_cross(k[1], k[2])
    return out


def compare(options, flat, params, abs_tol=1e-8, rel_tol=1e-9, cross_every=1, damping=1e-8):
    ref, msg = oracle_cov.estimate(options, flat, params, damping=damping)
    assert ref is not None, msg
    cov = estimate_covariance_flat(options, BACovarianceOptions(params, damping), flat, raise_not_estimable=True)
    keys = [k for k in ref if k[0] != "cross" or (k[1] + k[2]) % cross_every == 0]
    got = _gpu_blocks(cov, keys)
    worst_abs, worst_rel = (0.0, None), (0.0, None)
    for k in keys:
        assert got[k] is not None, k
        assert got[k].shape == ref[k].shape, (k, got[k].shape, ref[k].shape)
        err = np.abs(got[k] - ref[k]).max()
        rel = np.linalg.norm(got[k] - ref[k]) / max(np.linalg.norm(ref[k]), 1e-300)
        worst_abs, worst_rel = max(worst_abs, (err, k), key=lambda t: t[0]), max(worst_rel, (rel, k), key=lambda t: t[0])
    WORST["abs"], WORST["rel"] = max(WORST["abs"], worst_abs[0]), max(WORST["rel"], worst_rel[0])
    print(f"worst block error: {worst_abs[0]:.3g} absolute at {worst_abs[1]}, {worst_rel[0]:.3g} relative at {worst_rel[1]}")
    assert worst_abs[0] <= abs_tol and worst_rel[0] <= rel_tol, (worst_abs, worst_rel)
    # the bulk read-back agrees with the single getters
    poses, size = cov.poses_all()
    for i in range(len(flat.poses)):
        b = cov.pose(i)
        assert (b is None and size[i] == 0) or (size[i] == b.shape[0] and np.array_equal(poses[i, :size[i], :size[i]], b))
    pts, valid = cov.points_all()
    for k in range(0, len(flat.points), 7):
        b = cov.point(k)
        assert (b is None and not valid[k]) or (valid[k] and np.array_equal(pts[k], b))
    # what the reference reports as nullopt
    assert cov.pose(-1) is None and cov.pose(len(flat.poses)) is None and cov.point(len(flat.points)) is None
    for i in np.nonzero(flat.pose_constant)[0]:
        assert cov.pose(int(i)) is None
    return cov


@pytest.mark.parametrize("case", GRID, ids=lambda c: f"params{c[0]}-pts{int(c[1])}-poses{int(c[2])}-intr{int(c[3])}")
def test_reference_grid(case):
    params, fp, fpose, fint = case
    options, flat = reference_scene(fp, fpose, fint, solve=lambda o, f: solve_flat(BundleAdjustmentOptions(gpu_index=0), f))
    compare(options, flat, params)


def _two_cams_gauge(flat):
    flat.pose_constant = flat.pose_constant.copy(); flat.pose_fixed_dim = flat.pose_fixed_dim.copy()
    flat.pose_constant[0] = 1
    flat.pose_fixed_dim[1] = int(np.argmax(np.abs(flat.poses[1, 4:] - flat.poses[0, 4:])))
    return flat


def test_wide_model_cauchy():
    # OPENCV (6 variable intrinsics per camera); FULL_OPENCV's rational coefficients are not estimable on this scene
    _, flat = synthesize_ba_problem(12, 600, 6, models=(OPENCV,), seed=11, point2D_stddev=0.5)
    o = BundleAdjustmentOptions(gpu_index=0, loss_function_type=CAUCHY, loss_function_scale=1.0)
    _two_cams_gauge(flat)
    solve_flat(o, flat)
    for params in (oracle_cov.ALL, oracle_cov.POSES):
        compare(o, flat, params, abs_tol=1e-6)


def test_rig_sensor_blocks():
    _, flat = synthesize_rig_problem(8, 3, 400, 5, seed=5, point2D_stddev=0.5)
    _two_cams_gauge(flat)
    o = BundleAdjustmentOptions(gpu_index=0)
    solve_flat(o, flat)
    cov = compare(o, flat, oracle_cov.ALL, abs_tol=1e-6)
    assert cov.sensor(0).shape == (6, 6) and cov.sensor(1).shape == (6, 6) and cov.pose(1).shape == (5, 5)


def _tile_problem(num_images, num_const_cams):
    """Only focal lengths and poses vary: n = 5 + 6 (num_images - 2) + num_images - num_const_cams under a two-cams gauge."""
    _, flat = synthesize_ba_problem(num_images, 40 * num_images, 5, models=(SIMPLE_PINHOLE,), seed=num_images, point2D_stddev=0.5)
    _two_cams_gauge(flat)
    flat.cam_constant = flat.cam_constant.copy()
    flat.cam_constant[:num_const_cams] = 1
    return flat


@pytest.mark.parametrize("n,images,const", [(1, None, None), (63, 10, 0), (64, 11, 6), (65, 11, 5), (129, 20, 4)])
def test_tile_boundaries(n, images, const):
    o = BundleAdjustmentOptions(gpu_index=0, refine_extra_params=False)
    if images is None:      # one variable focal length, every pose constant
        flat = _tile_problem(6, 0)
        flat.pose_constant = np.ones(len(flat.poses), np.uint8)
        flat.cam_constant = np.ones(len(flat.cam_model), np.uint8); flat.cam_constant[2] = 0
    else:
        flat = _tile_problem(images, const)
    cov = compare(o, flat, oracle_cov.ALL)
    assert cov.info()[0] == n


def test_multi_tile():
    """300 SIMPLE_RADIAL cameras (f, k variable) and 30k points: n = 2393, 38 tiles."""
    _, flat = synthesize_ba_problem(300, 30000, 6, models=(SIMPLE_RADIAL,), seed=9, point2D_stddev=0.5)
    _two_cams_gauge(flat)
    o = BundleAdjustmentOptions(gpu_index=0)
    cov = compare(o, flat, oracle_cov.ALL, cross_every=97)
    n, ms = cov.info()
    assert n == 2393
    print(f"n = {n}: {ms}; worst margin so far: {WORST}")


@pytest.mark.parametrize("params", [oracle_cov.POSES, oracle_cov.POSES_AND_POINTS])
@pytest.mark.parametrize("scene", ["full_opencv", "rad_tan_thin_prism"])
def test_poses_mode_weak_intrinsics(scene, params):
    """Intrinsics pivots of S near the damping (DC = 18 and 22): the POSES modes eliminate the intrinsics and rank-test
    only the poses, as the reference does; ALL mode is not estimable on either side."""
    options, flat = weak_intrinsics_scene(scene, oracle_ba.solve)
    o = dataclasses.replace(options, gpu_index=0)
    # The damped S_oo has condition ~1e15-1e16 (its smallest pivots are the 1e-8 damping), so eps kappa(S_oo) gives no
    # usable bound.  The weak directions barely couple to the poses: the measured block errors on one H100 are at most
    # 3.0e-6 absolute and 2.3e-4 relative (the rounding of S, summed in another order, through the elimination).  The
    # bars keep a margin of 33x or more and stay far below the O(1) error of a wrong row range or a wrong elimination.
    ref, msg = oracle_cov.estimate(o, flat, params)
    if ref is None:
        # FULL_OPENCV: the smallest eigenvalues of S_oo + damping I are at the rounding level of S, so whether an LLT of
        # it succeeds depends on the summation order (the CPU restatement's did at other solved parameters).  The
        # poses are still determined: they must come back as symmetric positive definite blocks.
        assert msg == "others not positive definite", msg
        cov = estimate_covariance_flat(o, BACovarianceOptions(params), flat, raise_not_estimable=True)
        poses, size = cov.poses_all()
        assert size.sum() > 0
        for i in np.nonzero(size)[0]:
            b = poses[i, :size[i], :size[i]]
            assert np.allclose(b, b.T, rtol=1e-9, atol=0) and np.linalg.eigvalsh(b).min() > 0
    else:
        compare(o, flat, params, abs_tol=1e-4, rel_tol=1e-2)
    assert oracle_cov.estimate(o, flat, oracle_cov.ALL)[0] is None
    with pytest.raises(CovarianceNotEstimable, match="intrinsics of camera"):
        estimate_covariance_flat(o, BACovarianceOptions(oracle_cov.ALL), flat, raise_not_estimable=True)


def test_rig_wide_poses_mode():
    """A THIN_PRISM_FISHEYE rig with the principal point refined: camera blocks of 6 + 12 columns, DC = 28."""
    _, flat = synthesize_rig_problem(10, 3, 800, 8, models=(THIN_PRISM_FISHEYE,), seed=75, point2D_stddev=0.5)
    _two_cams_gauge(flat)
    o = BundleAdjustmentOptions(gpu_index=0, refine_principal_point=True)
    solve_flat(o, flat)
    # S has condition ~2e18 here (the thin-prism coefficients are weakly determined and are eliminated in POSES mode);
    # measured on one H100: 3.6e-9 absolute, 1.7e-7 relative (a small cross block).  Bars 28x and 58x above that.
    compare(o, flat, oracle_cov.POSES, abs_tol=1e-7, rel_tol=1e-5)


def test_track_lengths():
    """Tracks of 1, 2, 33, 200 and 300 observations in one problem (the point kernel's lane loop and its L x L pair
    loop past one warp), constant points, two constant poses."""
    lens = [1] * 30 + [2] * 30 + [33] * 20 + [200] * 3 + [300] * 3 + [8] * 4000
    _, flat = synthesize_ba_problem(320, len(lens), 8, models=(SIMPLE_RADIAL,), seed=17, point2D_stddev=0.5, track_lengths=lens)
    _two_cams_gauge(flat)
    flat.pose_constant[5] = 1
    flat.point_constant = flat.point_constant.copy()
    flat.point_constant[[1, 31, 61, 81, 84, 200]] = 1    # one of each track length
    o = BundleAdjustmentOptions(gpu_index=0)
    solve_flat(o, flat)
    # A point seen once has a rank-2 H_pp, so H_pp + damping I has condition ||H_pp|| / damping ~ 1e13; its inverse
    # (LAPACK in the oracle, cofactors in the kernel) is accurate to ~eps kappa, and through the Schur complement that
    # error reaches every block of S^-1.  Bar: 10 eps kappa relative (measured on one H100: 2.5e-3 relative, at
    # kappa = 1.3e13, i.e. 0.9 eps kappa), and the same fraction of the largest block absolute (5.6e4 at a 1e8 block).
    J, columns = oracle_cov.jacobian(o, flat)
    kappa = np.linalg.cond(oracle_cov.point_blocks(J, columns, [k for k in columns if k[0] == "point"], 1e-8)[1]).max()
    rel = 10 * np.finfo(np.float64).eps * kappa
    big = max(np.abs(b).max() for b in oracle_cov.estimate(o, flat, oracle_cov.POINTS, jac=(J, columns))[0].values())
    print(f"max cond(H_pp + damping I) = {kappa:.3g}")
    compare(o, flat, oracle_cov.ALL, abs_tol=rel * big, rel_tol=rel, cross_every=97)


@pytest.mark.parametrize("loss", [SOFT_L1, HUBER])
def test_robust_losses(loss):
    """SOFT_L1 and HUBER with 2 % outliers of 20 px, so that the loss weights vary across observations."""
    _, flat = synthesize_ba_problem(12, 600, 6, models=(SIMPLE_RADIAL,), seed=19, point2D_stddev=0.5)
    _two_cams_gauge(flat)
    flat.obs_xy[::50] += 20.0
    o = BundleAdjustmentOptions(gpu_index=0, loss_function_type=loss, loss_function_scale=1.0)
    solve_flat(o, flat)
    for params in (oracle_cov.ALL, oracle_cov.POSES):
        compare(o, flat, params)


@pytest.mark.parametrize("case", ["rotation_constant", "sensor_constant", "sensor_not_refined"])
def test_pose_and_sensor_options(case):
    if case == "rotation_constant":     # 3 x 3 pose blocks, 2 x 2 for the two-cams gauge pose
        _, flat = synthesize_ba_problem(10, 500, 6, models=(SIMPLE_RADIAL,), seed=21, point2D_stddev=0.5)
        _two_cams_gauge(flat)
        o, params = BundleAdjustmentOptions(gpu_index=0, constant_rig_from_world_rotation=True), oracle_cov.POSES
    else:
        _, flat = synthesize_rig_problem(8, 3, 400, 5, seed=5, point2D_stddev=0.5)
        _two_cams_gauge(flat)
        o, params = BundleAdjustmentOptions(gpu_index=0), oracle_cov.ALL
        if case == "sensor_constant":
            flat.sensor_constant = np.array([1, 0], np.uint8)
        else:
            o = dataclasses.replace(o, refine_sensor_from_rig=False)
    solve_flat(o, flat)
    cov = compare(o, flat, params)
    if case == "rotation_constant":
        assert cov.pose(1).shape == (2, 2) and cov.pose(2).shape == (3, 3)
    else:
        assert cov.sensor(0) is None and (cov.sensor(1) is None) == (case == "sensor_not_refined")


def test_damping():
    _, flat = synthesize_ba_problem(12, 600, 6, models=(OPENCV,), seed=23, point2D_stddev=0.5)
    _two_cams_gauge(flat)
    o = BundleAdjustmentOptions(gpu_index=0)
    solve_flat(o, flat)
    compare(o, flat, oracle_cov.POSES_AND_POINTS, damping=1e-4)


def test_multi_tile_poses_mode():
    """POSES mode whose eliminated intrinsics span several tiles: 40 OPENCV cameras, 240 intrinsics rows first."""
    _, flat = synthesize_ba_problem(40, 2000, 6, models=(OPENCV,), seed=29, point2D_stddev=0.5)
    _two_cams_gauge(flat)
    o = BundleAdjustmentOptions(gpu_index=0)
    solve_flat(o, flat)
    cov = compare(o, flat, oracle_cov.POSES, cross_every=7)
    assert cov.info()[0] == 240 + 6 * 38 + 5


def test_not_estimable_then_ok():
    _, flat = synthesize_ba_problem(6, 150, 4, seed=7)
    o = BundleAdjustmentOptions(gpu_index=0)
    with pytest.raises(CovarianceNotEstimable, match="pivot"):
        estimate_covariance_flat(o, BACovarianceOptions(), flat, raise_not_estimable=True)
    assert estimate_covariance_flat(o, BACovarianceOptions(), flat) is None
    compare(o, _two_cams_gauge(flat), oracle_cov.ALL, abs_tol=1e-6)


def test_python_interface():
    rec = synthesize_rig_reconstruction(1, 1, 7, 200, point2D_stddev=0.01, seed=3)
    cfg = BundleAdjustmentConfig()
    for image_id in rec.images:
        cfg.AddImage(image_id)
    for pid in sorted(rec.points3D)[:3]:
        cfg.AddConstantPoint(pid)
    ba = CreateDefaultBundleAdjuster(BundleAdjustmentOptions(gpu_index=0), cfg, rec)
    assert ba.Solve().IsSolutionUsable()
    cov = EstimateBACovariance(BACovarianceOptions(), rec, ba)
    flat = ba.flat_problem()[0]
    ref, _ = oracle_cov.estimate(ba.Options(), flat, oracle_cov.ALL)
    ids = sorted(rec.images)
    assert np.abs(cov.GetCamCovFromWorld(ids[1]) - ref[("pose", 1)]).max() <= 1e-8
    assert np.abs(cov.GetCamCrossCovFromWorld(ids[1], ids[2]) - ref[("cross", 1, 2)]).max() <= 1e-8
    cam = rec.cameras[rec.images[ids[0]].camera_id]
    assert np.abs(cov.GetOtherParamsCov(cam.params) - ref[("camera", 0)]).max() <= 1e-8
    assert cov.GetOtherParamsCov(cam.params.copy()) is None
    pid = sorted(rec.points3D)[10]
    assert np.abs(cov.GetPointCov(pid) - ref[("point", 10)]).max() <= 1e-8
    assert cov.GetPointCov(sorted(rec.points3D)[0]) is None and cov.GetPointCov(10 ** 9) is None
    assert cov.GetCamCovFromWorld(10 ** 9) is None
    c1, c2 = rec.images[ids[1]].cam_from_world, rec.images[ids[2]].cam_from_world
    full = np.block([[ref[("pose", 1)], ref[("cross", 1, 2)]], [ref[("cross", 1, 2)].T, ref[("pose", 2)]]])
    rel = cov.GetCam2CovFromCam1(ids[1], c1, ids[2], c2)
    assert np.abs(rel - GetCovarianceForRelativeRigid3d(c1, c2, full)).max() <= 1e-8
    print(f"worst margin over the file: {WORST}")
