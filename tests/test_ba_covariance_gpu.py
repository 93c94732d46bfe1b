"""b200ba_estimate_covariance on the GPU against the CPU restatement of covariance.cc (tests/oracle_cov.py), on the same
parameter arrays: the reference's test grid, a wide model with a robust loss, a rig, a two-cams gauge, dense dimensions
around the 64-row tile of the factorisation, a multi-tile problem, the not-estimable path and the Python interface."""
import numpy as np
import pytest

import oracle_cov
from colmap_b200.bundle_adjustment import (CAUCHY, OPENCV, SIMPLE_PINHOLE, SIMPLE_RADIAL, BACovarianceOptions,
                                           BundleAdjustmentConfig, BundleAdjustmentOptions, CovarianceNotEstimable,
                                           CreateDefaultBundleAdjuster, EstimateBACovariance, GetCovarianceForRelativeRigid3d,
                                           estimate_covariance_flat, solve_flat)
from colmap_b200.synthetic import synthesize_ba_problem, synthesize_rig_problem, synthesize_rig_reconstruction
from test_ba_covariance_cpu import GRID, reference_scene

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


def compare(options, flat, params, abs_tol=1e-8, rel_tol=1e-9, cross_every=1):
    ref, msg = oracle_cov.estimate(options, flat, params)
    assert ref is not None, msg
    cov = estimate_covariance_flat(options, BACovarianceOptions(params), flat, raise_not_estimable=True)
    keys = [k for k in ref if k[0] != "cross" or (k[1] + k[2]) % cross_every == 0]
    got = _gpu_blocks(cov, keys)
    for k in keys:
        assert got[k] is not None, k
        assert got[k].shape == ref[k].shape, (k, got[k].shape, ref[k].shape)
        err = np.abs(got[k] - ref[k]).max()
        rel = np.linalg.norm(got[k] - ref[k]) / max(np.linalg.norm(ref[k]), 1e-300)
        WORST["abs"], WORST["rel"] = max(WORST["abs"], err), max(WORST["rel"], rel)
        assert err <= abs_tol and rel <= rel_tol, (k, err, rel)
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
