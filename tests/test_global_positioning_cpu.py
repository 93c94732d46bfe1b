"""Global positioning without a GPU: the set-up of GlobalPositioner solved by the fp64 oracle on the reference's three
scenarios (global_positioning_test.cc), the host camera rays of all eighteen models, and the host input checks of
b200gp_solve, which refuse before any device work."""
import ctypes
import itertools

import numpy as np
import pytest

import gp_oracle
from colmap_b200 import load_library
from colmap_b200.bundle_adjustment import MODEL_NUM_PARAMS, _quat_to_R
from colmap_b200.global_positioning import (ERR_INPUT, ERR_TOO_LARGE, FlatGlobalPositioning, GlobalPositioner,
                                            GlobalPositionerOptions, GlobalPositioningError, PoseGraph,
                                            cam_ray_from_img, solve_flat)
from colmap_b200.synthetic import _MODEL_DEFAULTS, _project, synthesize_rig_reconstruction


class OraclePositioner(GlobalPositioner):
    def _solve_flat(self, flat):
        o = self.options_
        r = gp_oracle.solve(flat, o.max_num_iterations, o.optimize_positions, o.optimize_points, o.optimize_scales,
                            o.loss_function_scale, o.function_tolerance, o.gradient_tolerance, o.parameter_tolerance)

        class S:
            termination_type = r.termination_type
            def IsSolutionUsable(self): return r.termination_type in (0, 1)
        return S()


def scenario(num_rigs, cams, frames, seed=0):
    gt = synthesize_rig_reconstruction(num_rigs, cams, frames, 200, seed=seed)
    rec = synthesize_rig_reconstruction(num_rigs, cams, frames, 200, seed=seed)
    for fr in rec.frames.values():
        fr.rig_from_world[4:] = 0.0
    GlobalPositioner._sync_image_poses(rec)
    edges = list(itertools.combinations(sorted(rec.images), 2))
    return gt, rec, PoseGraph(edges)


def centers(rec):
    return np.array([-_quat_to_R(rec.images[i].cam_from_world[:4]).T @ rec.images[i].cam_from_world[4:] for i in sorted(rec.images)])


def similarity_error(a, b):
    """max distance between b and the similarity transform of a that best fits it (Umeyama)."""
    ma, mb = a.mean(0), b.mean(0)
    A, B = a - ma, b - mb
    U, S, Vt = np.linalg.svd(B.T @ A)
    d = np.sign(np.linalg.det(U @ Vt))
    D = np.diag([1, 1, d])
    R = U @ D @ Vt
    s = np.trace(np.diag(S) @ D) / np.sum(A * A)
    return np.max(np.linalg.norm(s * A @ R.T - B, axis=1))


@pytest.mark.parametrize("rigs,cams,frames", [(1, 1, 10), (2, 3, 5)], ids=["Nominal", "MultiCameraRig"])
def test_oracle_recovers_ground_truth(rigs, cams, frames):
    gt, rec, pg = scenario(rigs, cams, frames)
    assert OraclePositioner(GlobalPositionerOptions(random_seed=42)).Solve(pg, rec)
    assert similarity_error(centers(rec), centers(gt)) < 0.5   # max_proj_center_error of the reference test


def test_refine_sensor_from_rig_false_preserves_rig():
    gt, rec, pg = scenario(2, 3, 5)
    snap = {(r, c): v.copy() for r, rig in rec.rigs.items() for c, v in rig.sensors.items()}
    assert snap
    assert OraclePositioner(GlobalPositionerOptions(random_seed=42, refine_sensor_from_rig=False)).Solve(pg, rec)
    for (r, c), v in snap.items():
        assert np.array_equal(rec.rigs[r].sensors[c].view(np.uint64), v.view(np.uint64))


def test_nan_sensor_translation_needs_refine_sensor_from_rig():
    _, rec, pg = scenario(1, 2, 4)
    next(iter(rec.rigs.values())).sensors[2][4:] = np.nan
    with pytest.raises(ValueError, match="refine_sensor_from_rig"):
        OraclePositioner(GlobalPositionerOptions(random_seed=1, refine_sensor_from_rig=False)).Solve(pg, rec)
    pos = OraclePositioner(GlobalPositionerOptions(random_seed=1))
    assert pos.Solve(pg, rec)
    f = pos.flat_problem
    assert len(f.cams_in_rig) == 1 and (f.obs_sensor >= 0).any()
    assert np.all(np.isfinite(next(iter(rec.rigs.values())).sensors[2]))


def test_setup_quirks():
    _, rec, _ = scenario(1, 1, 6)
    # frame 6 only in the pose graph (its image's observations dropped): randomised centre written back anyway
    for p in rec.points3D.values():
        p.track = [t for t in p.track if t[0] != 6]
    pos = OraclePositioner(GlobalPositionerOptions(random_seed=3))
    assert pos.Solve(PoseGraph([(1, 6)]), rec)
    assert len(pos.flat_problem.frame_centers) == 6 and 5 not in set(pos.flat_problem.obs_frame.tolist())
    c6 = centers(rec)[5]
    assert np.allclose(c6, pos.flat_problem.frame_centers[5], atol=1e-9) and np.abs(c6).max() > 1.0
    # short tracks are skipped; generate_scales=False derives the scales from the initial positions
    for pid in list(rec.points3D)[:10]:
        rec.points3D[pid].track = rec.points3D[pid].track[:2]
    pos = OraclePositioner(GlobalPositionerOptions(random_seed=3, generate_scales=False, max_num_iterations=0))
    pos.Solve(PoseGraph(), rec)
    f = pos.flat_problem
    assert len(f.points) == 190
    t = f.points[f.obs_point] - f.frame_centers[f.obs_frame]
    assert np.allclose(f.obs_scale, np.maximum(1e-5, np.sum(f.obs_ray * t, 1) / np.sum(t * t, 1)))
    assert np.all(f.obs_loss_weight == 0.5)
    rec.cameras[1].has_prior_focal_length = True
    pos.Solve(PoseGraph(), rec)
    assert np.all(pos.flat_problem.obs_loss_weight == 1.0)


def test_seed_is_reproducible():
    a = [OraclePositioner(GlobalPositionerOptions(random_seed=7, max_num_iterations=0)) for _ in range(2)]
    for p in a:
        _, rec, pg = scenario(1, 1, 4)
        p.Solve(pg, rec)
    assert np.array_equal(a[0].flat_problem.frame_centers, a[1].flat_problem.frame_centers)


@pytest.mark.parametrize("model", range(18))
def test_cam_ray_round_trips_img_from_cam(model):
    prm = np.asarray(_MODEL_DEFAULTS[model], np.float64)
    assert len(prm) == MODEL_NUM_PARAMS[model]
    rng = np.random.default_rng(model)
    d = np.concatenate([rng.uniform(-0.35, 0.35, (40, 2)), np.ones((40, 1))], 1)
    if model == 17:
        d[:10, 2] = -1.0   # the equirectangular ray also covers the back hemisphere
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    xy = _project(model, np.broadcast_to(prm, (len(d), len(prm))), d)
    for k in range(len(d)):
        ray = cam_ray_from_img(model, prm, xy[k])
        assert ray is not None
        assert np.abs(ray - d[k]).max() < 1e-9, (model, k, ray, d[k])


def test_cam_ray_failures():
    assert cam_ray_from_img(16, [1280.0, 1270.0, 512.0, 384.0, 0.8, 3.0], [1e5, 1e5]) is None   # EUCM outside its domain
    assert cam_ray_from_img(99, [1.0], [0.0, 0.0]) is None


def small_flat(N=6):
    rng = np.random.default_rng(0)
    return FlatGlobalPositioning(frame_centers=rng.normal(size=(2, 3)), points=rng.normal(size=(3, 3)),
                                 obs_frame=np.arange(N) % 2, obs_point=np.arange(N) % 3,
                                 obs_ray=rng.normal(size=(N, 3)), obs_scale=np.ones(N))


@pytest.mark.parametrize("breakage", ["frame", "point", "sensor", "ray", "scale", "weight", "nan_centre", "no_refine", "no_rotation"])
def test_host_checks_refuse(breakage):
    f = small_flat()
    o = GlobalPositionerOptions()
    if breakage == "frame": f.obs_frame[2] = 5
    if breakage == "point": f.obs_point[1] = -1
    if breakage == "sensor": f.obs_sensor = np.array([0, -1, -1, -1, -1, -1], np.int32)
    if breakage == "ray": f.obs_ray[3, 1] = np.inf
    if breakage == "scale": f.obs_scale[4] = 1e-6
    if breakage == "weight": f.obs_loss_weight = np.array([1, 1, 0, 1, 1, 1], np.float64)
    if breakage == "nan_centre": f.frame_centers[1, 0] = np.nan
    if breakage in ("no_refine", "no_rotation"):
        f.cams_in_rig = np.zeros((1, 3)); f.obs_sensor = np.array([0, -1, -1, -1, -1, -1], np.int32)
        if breakage == "no_refine":
            f.world_from_rig = np.tile(np.eye(3), (2, 1, 1)); o.refine_sensor_from_rig = False
    with pytest.raises(GlobalPositioningError) as e:
        solve_flat(o, f)
    assert e.value.code == ERR_INPUT


def test_refuses_above_dense_envelope_before_device_work():
    F = 32768 // 3 + 1
    f = FlatGlobalPositioning(frame_centers=np.zeros((F, 3)), points=np.zeros((1, 3)), obs_frame=np.arange(F),
                              obs_point=np.zeros(F, np.int32), obs_ray=np.tile([0.0, 0.0, 1.0], (F, 1)), obs_scale=np.ones(F))
    with pytest.raises(GlobalPositioningError, match="dense limit") as e:
        solve_flat(GlobalPositionerOptions(), f)
    assert e.value.code == ERR_TOO_LARGE


def test_abi_surface():
    lib = load_library()
    for name in ("b200gp_solve", "b200gp_options_init", "b200gp_cam_ray_from_img", "b200gp_last_error"):
        assert hasattr(lib, name)
    from colmap_b200.global_positioning import _CProblem, _COptions, _CSummary
    assert ctypes.sizeof(_COptions) == 4 * 4 + 8 + 8 + 8 * 9 + 8 and ctypes.sizeof(_CSummary) == 5 * 4 + 4 + 3 * 8 + 8 + 8
    assert ctypes.sizeof(_CProblem) == 16 * 8
