"""CPU tier for the bundle-adjustment path: the oracle against the reference's known answers and properties,
the product's host-compiled arithmetic against the oracle, the C-ABI surface.  No GPU compute."""
import ctypes
import os
import re

import numpy as np
import pytest

import oracle_ba
from colmap_b200 import load_library
from colmap_b200.bundle_adjustment import (DENSE_SCHUR, ITERATIVE_SCHUR, PINHOLE, RADIAL, RADIAL_FISHEYE, SIMPLE_PINHOLE,
                                           SIMPLE_RADIAL_FISHEYE,
                                           SIMPLE_RADIAL, SOFT_L1, BundleAdjustmentOptions, _CConfig, _CCovOptions, _CProblem,
                                           _COptions, _CScene, _bind, _bind_cov, _f64p, _i8p, _i32p, _u8p)
from colmap_b200.synthetic import synthesize_ba_problem

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDENTITY_POSE = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)


# ---------------------------------------------------------------- reference known answers
def test_reprojection_known_answers():
    """cost_functions/reprojection_error_test.cc:41-71 (SIMPLE_PINHOLE {1,0,0}, identity pose, point (0,0,1)):
    observation (0,0) -> residual (0,0); (0,1) -> (0,-1); f = 2 and point (0,1,1)... ; behind camera -> 0."""
    ok, res, *_ = oracle_ba.reproj(SIMPLE_PINHOLE, [0, 0, 1], IDENTITY_POSE, [1, 0, 0], [0, 0])
    assert ok and np.allclose(res, [0, 0])
    ok, res, *_ = oracle_ba.reproj(SIMPLE_PINHOLE, [0, 0, 1], IDENTITY_POSE, [1, 0, 0], [0, 1])
    assert ok and np.allclose(res, [0, -1])
    ok, res, *_ = oracle_ba.reproj(SIMPLE_PINHOLE, [0, 1, 1], IDENTITY_POSE, [2, 0, 0], [0, 0])
    assert ok and np.allclose(res, [0, 2])
    # point behind / on the camera plane: residual and Jacobians are zero (reprojection_error.h:101-116)
    for z in (-1.0, 0.0):
        ok, res, Jpt, Jps, Jpr = oracle_ba.reproj(SIMPLE_PINHOLE, [0, 0, z], IDENTITY_POSE, [1, 0, 0], [3, 4])
        assert not ok and np.all(res == 0) and np.all(Jpt == 0) and np.all(Jps == 0) and np.all(Jpr == 0)


@pytest.mark.parametrize("model,params", [(SIMPLE_PINHOLE, [600., 320, 240]), (PINHOLE, [600., 610, 320, 240]),
                                          (SIMPLE_RADIAL, [600., 320, 240, 0.08]), (RADIAL, [600., 320, 240, 0.08, -0.02]),
                                          (SIMPLE_RADIAL_FISHEYE, [600., 320, 240, 0.08]),
                                          (RADIAL_FISHEYE, [600., 320, 240, 0.08, -0.02])])
def test_analytic_jacobians_match_finite_differences(model, params):
    """The property reprojection_error_test.cc:211-323 pins with autodiff (tolerance 1e-4), restated with
    central differences over a grid of points and a non-trivial pose."""
    rng = np.random.default_rng(0)
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    pose = np.concatenate([q, [0.1, -0.2, 4.0]])
    params = np.asarray(params, np.float64)
    for _ in range(20):
        pt = rng.uniform(-1, 1, 3)
        ok, res, Jpt, Jps, Jpr = oracle_ba.reproj(model, pt, pose, params, [1.0, 2.0])
        assert ok

        def f(pt_, pose_, prm_):
            return oracle_ba.reproj(model, pt_, pose_, prm_, [1.0, 2.0])[1]
        h = 1e-6
        for k in range(3):
            d = np.zeros(3); d[k] = h
            assert np.allclose((f(pt + d, pose, params) - f(pt - d, pose, params)) / (2 * h), Jpt[:, k], atol=1e-4, rtol=1e-6)
        for k in range(7):
            d = np.zeros(7); d[k] = h
            assert np.allclose((f(pt, pose + d, params) - f(pt, pose - d, params)) / (2 * h), Jps[:, k], atol=1e-4, rtol=1e-6)
        for k in range(len(params)):
            d = np.zeros(len(params)); d[k] = h * max(1.0, abs(params[k]))
            assert np.allclose((f(pt, pose, params + d) - f(pt, pose, params - d)) / (2 * d[k]), Jpr[:, k], atol=1e-4, rtol=1e-5)


def test_quaternion_plus_is_a_rotation_update():
    L = oracle_ba.lib()
    rng = np.random.default_rng(1)
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    out = np.zeros(4)
    L.ba_oracle_quat_plus(q.ctypes.data_as(_f64p), np.zeros(3).ctypes.data_as(_f64p), out.ctypes.data_as(_f64p))
    assert np.array_equal(out, q)
    d = np.array([0.01, -0.02, 0.03])
    L.ba_oracle_quat_plus(q.ctypes.data_as(_f64p), d.ctypes.data_as(_f64p), out.ctypes.data_as(_f64p))
    assert abs(np.linalg.norm(out) - 1) < 1e-14
    # first-order: out ~ q + PlusJacobian * d  (ceres EigenQuaternionManifold)
    x, y, z, w = q
    PJ = np.array([[w, z, -y], [-z, w, x], [y, -x, w], [-x, -y, -z]])
    assert np.allclose(out, q + PJ @ d, atol=1e-3)


# ---------------------------------------------------------------- oracle solver behaviour (bundle_adjustment_test.cc)
def _gauge(flat):
    flat.pose_constant = flat.pose_constant.copy(); flat.pose_fixed_dim = flat.pose_fixed_dim.copy()
    flat.pose_constant[0] = 1
    base = flat.poses[1, 4:] - flat.poses[0, 4:]
    flat.pose_fixed_dim[1] = int(np.argmax(np.abs(base)))
    return flat


def test_oracle_nominal_recovers_ground_truth():
    """bundle_adjustment_test.cc:303-352 (Nominal): 10 frames, 200 points, noise (0.5 px, 0.1, 0.5 deg, 0.1):
    ground truth recovered to 0.1 units / 0.1 deg after aligning; here: reprojection RMSE back to the noise
    floor and exact residual count."""
    gt, noisy = synthesize_ba_problem(10, 200, 10, models=(SIMPLE_RADIAL,), shared_camera=True, seed=1,
                                      point2D_stddev=0.5, point3D_stddev=0.1, translation_stddev=0.1, rotation_stddev_deg=0.5)
    _gauge(noisy)
    s = oracle_ba.solve(BundleAdjustmentOptions(), noisy)
    assert s.termination_type == 0
    assert s.num_residuals == 2 * 200 * 10
    rmse = np.sqrt(2 * s.final_cost / (s.num_residuals / 2))
    assert rmse < 0.5 * np.sqrt(2) * 1.05          # noise floor (0.5 px per coordinate)
    assert s.final_cost < 1e-3 * s.initial_cost
    # relative geometry: compare camera centres / points up to the similarity the gauge leaves: use distances
    c_gt = gt.points[:50]; c_es = noisy.points[:50]
    d_gt = np.linalg.norm(c_gt[:, None] - c_gt[None], axis=-1); d_es = np.linalg.norm(c_es[:, None] - c_es[None], axis=-1)
    scale = d_es.sum() / d_gt.sum()
    assert np.abs(d_es / scale - d_gt).max() < 0.1


def test_oracle_constant_blocks_are_bit_identical_and_counts():
    """bundle_adjustment_test.cc:354-411: constant points stay bit-identical; num_residuals only counts
    observations that touch a variable block."""
    gt, noisy = synthesize_ba_problem(6, 60, 4, models=(PINHOLE,), shared_camera=True, seed=2)
    _gauge(noisy)
    noisy.point_constant = noisy.point_constant.copy(); noisy.point_constant[:10] = 1
    before = noisy.copy()
    s = oracle_ba.solve(BundleAdjustmentOptions(), noisy)
    assert s.termination_type in (0, 1)
    assert np.array_equal(noisy.points[:10], before.points[:10])
    assert np.array_equal(noisy.poses[0], before.poses[0])                   # gauge-fixed frame
    assert noisy.cam_params[2] == before.cam_params[2] and noisy.cam_params[3] == before.cam_params[3]  # principal point
    assert not np.array_equal(noisy.points[10:], before.points[10:])
    assert s.num_residuals == 2 * 60 * 4
    # everything constant except the points: residuals of constant points drop out
    o = BundleAdjustmentOptions(refine_rig_from_world=False, refine_focal_length=False, refine_extra_params=False)
    f2 = before.copy(); f2.point_constant = noisy.point_constant; f2.pose_constant = noisy.pose_constant; f2.pose_fixed_dim = noisy.pose_fixed_dim
    s2 = oracle_ba.solve(o, f2)
    assert s2.num_residuals == 2 * 50 * 4


def test_oracle_dense_and_iterative_schur_agree():
    gt, noisy = synthesize_ba_problem(12, 300, 6, models=(SIMPLE_RADIAL,), seed=3)
    _gauge(noisy)
    a, b = noisy.copy(), noisy.copy()
    for f in (a, b):
        f.pose_constant, f.pose_fixed_dim = noisy.pose_constant, noisy.pose_fixed_dim
    sa = oracle_ba.solve(BundleAdjustmentOptions(linear_solver_type=DENSE_SCHUR), a)
    sb = oracle_ba.solve(BundleAdjustmentOptions(linear_solver_type=ITERATIVE_SCHUR), b)
    assert sa.termination_type == 0 and sb.termination_type == 0
    assert abs(sa.final_cost - sb.final_cost) < 1e-6 * sa.final_cost
    assert np.allclose(a.poses, b.poses, atol=1e-6) and np.allclose(a.points, b.points, atol=1e-6)
    assert sb.num_linear_solver_iterations > 0 and sa.num_linear_solver_iterations == 0


def test_oracle_robust_loss_downweights_outliers():
    gt, noisy = synthesize_ba_problem(8, 150, 5, models=(PINHOLE,), shared_camera=True, seed=4)
    _gauge(noisy)
    rng = np.random.default_rng(0)
    bad = rng.choice(len(noisy.obs_xy), 30, replace=False)
    noisy.obs_xy[bad] += rng.normal(0, 80, (30, 2))
    a, b = noisy.copy(), noisy.copy()
    for f in (a, b):
        f.pose_constant, f.pose_fixed_dim = noisy.pose_constant, noisy.pose_fixed_dim
    oracle_ba.solve(BundleAdjustmentOptions(), a)
    oracle_ba.solve(BundleAdjustmentOptions(loss_function_type=SOFT_L1, loss_function_scale=1.0), b)
    err = lambda f: np.median(np.linalg.norm(f.points - gt.points, axis=1))
    assert err(b) < err(a)


# ---------------------------------------------------------------- product host side vs oracle
def test_library_exports_every_declared_ba_symbol():
    lib = load_library()
    hdr = open(os.path.join(ROOT, "include", "b200_bundle_adjustment.h")).read()
    names = set(re.findall(r"\b(b200ba_[a-z_0-9]+)\s*\(", hdr))
    assert names == {"b200ba_options_init", "b200ba_fix_gauge_two_cams_from_world", "b200ba_solve", "b200ba_last_error",
                     "b200ba_comm_unique_id", "b200ba_comm_init", "b200ba_comm_destroy", "b200ba_comm_peer_memory", "b200ba_solve_sharded",
                     "b200ba_assemble", "b200ba_assembly_problem", "b200ba_assembly_free"}
    for n in names:
        assert hasattr(lib, n), n


def test_options_init_matches_reference_defaults():
    lib = _bind(load_library())
    o = _COptions()
    lib.b200ba_options_init(ctypes.byref(o))
    d = BundleAdjustmentOptions().to_c()
    for f, _ in _COptions._fields_:
        assert getattr(o, f) == getattr(d, f), f
    assert (o.max_num_iterations, o.max_linear_solver_iterations, o.gradient_tolerance, o.function_tolerance) == (100, 200, 1e-4, 0.0)


def test_product_reprojection_arithmetic_matches_oracle():
    lib = load_library()
    lib.b200ba_test_reproj.argtypes = [ctypes.c_int] + [_f64p] * 8
    rng = np.random.default_rng(5)
    prm = {0: [600., 320, 240], 1: [600., 610, 320, 240], 2: [600., 320, 240, 0.08], 3: [600., 320, 240, 0.08, -0.02],
           8: [600., 320, 240, 0.08], 9: [600., 320, 240, 0.08, -0.02]}
    for model in prm:
        for _ in range(50):
            q = rng.normal(size=4); q /= np.linalg.norm(q)
            pose = np.concatenate([q, rng.uniform(-1, 1, 2), [4.0]])
            pt = rng.uniform(-1, 1, 3); xy = rng.uniform(0, 500, 2); params = np.asarray(prm[model])
            ok, res, Jpt, Jps, Jpr = oracle_ba.reproj(model, pt, pose, params, xy)
            r2 = np.zeros(2); a = np.zeros((2, 3)); b = np.zeros((2, 7)); c = np.zeros((2, len(params)))
            ok2 = lib.b200ba_test_reproj(model, pt.ctypes.data_as(_f64p), pose.ctypes.data_as(_f64p), params.ctypes.data_as(_f64p),
                                         xy.ctypes.data_as(_f64p), r2.ctypes.data_as(_f64p), a.ctypes.data_as(_f64p),
                                         b.ctypes.data_as(_f64p), c.ctypes.data_as(_f64p))
            assert ok == ok2
            for u, v in ((res, r2), (Jpt, a), (Jps, b), (Jpr, c)):
                assert np.allclose(u, v, rtol=1e-13, atol=1e-13)


def test_gauge_two_cams_from_world():
    """FixGaugeWithTwoCamsFromWorld (bundle_adjustment_ceres.cc:308-417): first image constant, the second frame
    with a non-degenerate baseline gets its largest baseline coordinate fixed; nothing to do if two are fixed."""
    lib = _bind(load_library())
    gt, noisy = synthesize_ba_problem(5, 20, 3, models=(PINHOLE,), shared_camera=True, seed=6)
    # make pose 1 coincide with pose 0 -> degenerate baseline, must be skipped
    noisy.poses[1] = noisy.poses[0]
    cp, co = noisy.to_c(), BundleAdjustmentOptions().to_c()
    pc = np.zeros(5, np.uint8); fd = np.zeros(5, np.int8)
    assert lib.b200ba_fix_gauge_two_cams_from_world(ctypes.byref(cp), ctypes.byref(co), pc.ctypes.data_as(_u8p), fd.ctypes.data_as(_i8p)) == 0
    assert pc.tolist() == [1, 0, 0, 0, 0]
    assert fd[1] == -1 and fd[2] in (0, 1, 2) and (fd[3:] == -1).all()
    # expected dimension: largest |baseline| of (T0 * T2^-1).translation
    from colmap_b200.synthetic import _quat_rotate
    q0, t0, q2, t2 = noisy.poses[0, :4], noisy.poses[0, 4:], noisy.poses[2, :4], noisy.poses[2, 4:]
    q2inv = q2 * np.array([-1, -1, -1, 1])
    c2 = -_quat_rotate(q2inv, t2)
    base = _quat_rotate(q0, c2) + t0
    assert fd[2] == int(np.argmax(np.abs(base)))
    # two frames already constant -> untouched
    noisy.pose_constant = np.array([0, 1, 0, 1, 0], np.uint8)
    cp = noisy.to_c()
    assert lib.b200ba_fix_gauge_two_cams_from_world(ctypes.byref(cp), ctypes.byref(co), pc.ctypes.data_as(_u8p), fd.ctypes.data_as(_i8p)) == 0
    assert pc.tolist() == [0, 1, 0, 1, 0] and (fd == -1).all()


def test_point_sharding_covers_and_balances():
    from colmap_b200.bundle_adjustment import shard_flat_problem
    gt, noisy = synthesize_ba_problem(20, 3000, 6, models=(SIMPLE_RADIAL,), seed=8)
    for world in (2, 3, 8):
        shards = [shard_flat_problem(noisy, r, world) for r in range(world)]
        ids = np.concatenate([s.point_ids for s in shards])
        assert np.array_equal(ids, np.arange(3000))
        nobs = [len(s.obs_pose) for s in shards]
        assert sum(nobs) == len(noisy.obs_pose) and max(nobs) - min(nobs) <= 0.05 * len(noisy.obs_pose)
        for s in shards:   # local indices are consistent and every observation of a local point is present
            assert s.obs_point.min() >= 0 and s.obs_point.max() < len(s.points)
            assert np.array_equal(s.points, noisy.points[s.point_ids])
            assert len(s.obs_pose) == np.isin(noisy.obs_point, s.point_ids).sum()
            assert np.array_equal(s.poses, noisy.poses)


# ---------------------------------------------------------------- host flattening of the product (no GPU needed)
def _pack(flat, options=None):
    """b200ba_test_pack: the slot layout b200ba_solve builds on the host before anything touches the GPU."""
    lib = _bind(load_library())
    i32p, i64p = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)
    lib.b200ba_test_pack.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CProblem), ctypes.c_int64, i32p, i32p, i32p, i32p,
                                     i32p, i32p, i64p]
    co, cp = (options or BundleAdjustmentOptions(linear_solver_type=ITERATIVE_SCHUR)).to_c(), flat.to_c()
    info = np.zeros(10, np.int64)
    assert lib.b200ba_test_pack(ctypes.byref(co), ctypes.byref(cp), 0, None, None, None, None, None, None, info.ctypes.data_as(i64p)) == 0
    n, nvpt = int(info[0]), int(info[1])
    a = {k: np.empty(n, np.int32) for k in ("s_obs", "s_lpt", "s_seg")}
    v = {k: np.empty(max(nvpt, 1), np.int32) for k in ("vpt_s0", "vpt_s1", "vpt_point")}
    p = lambda x: x.ctypes.data_as(i32p)
    assert lib.b200ba_test_pack(ctypes.byref(co), ctypes.byref(cp), n, p(a["s_obs"]), p(a["s_lpt"]), p(a["s_seg"]), p(v["vpt_s0"]),
                                p(v["vpt_s1"]), p(v["vpt_point"]), info.ctypes.data_as(i64p)) == 0
    return dict(a, **{k: x[:nvpt] for k, x in v.items()}, nslots=n, nvpt=nvpt, nblocks_warp=int(info[2]), nblocks_var=int(info[3]),
                nblocks_giant0=int(info[4]), nblocks_giant1=int(info[5]), nc=int(info[6]), dkmax=int(info[7]),
                num_residuals=int(info[8]), num_effective_parameters=int(info[9]))


def test_product_slot_packing_invariants():
    """Tracks of <= 32 observations never cross a 32-slot warp (with the head / last lane recorded for the segmented
    shuffle reductions), tracks of <= 256 never cross a block, longer ones are contiguous; every observation that
    touches a variable block sits in exactly one slot; observations of constant points follow the variable blocks."""
    rng = np.random.default_rng(4)
    lens = np.concatenate([rng.integers(2, 12, 4000), rng.integers(33, 200, 30), [300, 700]])
    gt, noisy = synthesize_ba_problem(900, len(lens), 0, models=(SIMPLE_RADIAL,), shared_camera=True, seed=9, track_lengths=lens)
    _gauge(noisy)
    noisy.point_constant = noisy.point_constant.copy(); noisy.point_constant[:50] = 1     # some constant points
    L = _pack(noisy)
    s_obs, s_lpt, s_seg = L["s_obs"], L["s_lpt"], L["s_seg"]
    assert L["nslots"] % 256 == 0
    valid = s_obs >= 0
    assert np.array_equal(np.sort(s_obs[valid]), np.arange(len(noisy.obs_pose)))           # every observation exactly once
    assert np.all(s_lpt[~valid] == -1)
    # slot -> point consistency
    pt_of_slot = noisy.obs_point[s_obs[valid]]
    lpt = s_lpt[valid]
    const_slots = lpt < 0
    assert np.all(noisy.point_constant[pt_of_slot[const_slots]] == 1) and np.all(noisy.point_constant[pt_of_slot[~const_slots]] == 0)
    assert np.array_equal(L["vpt_point"][lpt[~const_slots]], pt_of_slot[~const_slots])
    assert L["nvpt"] == int((noisy.point_constant == 0).sum())
    slots = np.arange(L["nslots"])
    for n in range(L["nvpt"]):
        s0, s1 = int(L["vpt_s0"][n]), int(L["vpt_s1"][n])
        assert np.all(s_lpt[s0:s1] == n) and s1 - s0 == lens[L["vpt_point"][n]]
        blk0, blk1 = s0 // 256, (s1 - 1) // 256
        if s1 - s0 <= 32:
            assert blk0 < L["nblocks_warp"] and s0 // 32 == (s1 - 1) // 32                # inside one warp
            assert np.all((s_seg[s0:s1] & 0xff) == s0 % 32) and np.all((s_seg[s0:s1] >> 8) == (s1 - 1) % 32)
        elif s1 - s0 <= 256:
            assert L["nblocks_warp"] <= blk0 == blk1 < L["nblocks_giant0"]                # inside one block
        else:
            assert L["nblocks_giant0"] <= blk0 and blk1 < L["nblocks_giant1"]
    # constant-point observations sit behind the variable blocks
    assert np.all(slots[valid][const_slots] >= L["nblocks_giant1"] * 256) and L["nblocks_var"] == L["nblocks_giant0"]
    # the length-bucket packing wastes little: >= 95 % of the warp-packed slots carry an observation
    warp_region = valid[:L["nblocks_warp"] * 256]
    assert warp_region.mean() > 0.95
    assert L["nc"] == 6 * 899 + 2 and L["dkmax"] == 2          # 899 variable poses (the gauge-fixed coordinate is masked, the block stays 6 wide) + f, k of the shared camera


def test_product_rejects_unsupported_inputs_without_a_gpu():
    gt, noisy = synthesize_ba_problem(4, 30, 3, models=(SIMPLE_RADIAL,), seed=1)
    bad = noisy.copy(); bad.cam_model = noisy.cam_model.copy(); bad.cam_model[0] = 18      # beyond CameraModelId (0..17)
    lib = _bind(load_library())
    info = np.zeros(10, np.int64)
    lib.b200ba_test_pack.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CProblem), ctypes.c_int64] + [ctypes.c_void_p] * 6 + [ctypes.POINTER(ctypes.c_int64)]
    co, cp = BundleAdjustmentOptions().to_c(), bad.to_c()
    assert lib.b200ba_test_pack(ctypes.byref(co), ctypes.byref(cp), 0, None, None, None, None, None, None,
                                info.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))) == -2
    assert b"unknown camera model" in lib.b200ba_last_error()
    bad2 = noisy.copy(); bad2.obs_pose = noisy.obs_pose.copy(); bad2.obs_pose[0] = 99
    cp = bad2.to_c()
    assert lib.b200ba_test_pack(ctypes.byref(co), ctypes.byref(cp), 0, None, None, None, None, None, None,
                                info.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))) == -2


def test_assembly_covariance_and_solve_errors_reach_b200ba_last_error():
    # the problem assembly, the covariance estimate and the solve are separate translation units with one error string
    lib = _bind_cov(_bind(load_library()))
    lib.b200ba_assemble.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CScene), ctypes.POINTER(_CConfig), ctypes.POINTER(ctypes.c_void_p)]
    co, h = BundleAdjustmentOptions().to_c(), ctypes.c_void_p()
    image_camera = np.array([1], np.int32)
    sc = _CScene(num_images=1, image_camera=image_camera.ctypes.data_as(_i32p), num_cameras=1)
    assert lib.b200ba_assemble(ctypes.byref(co), ctypes.byref(sc), ctypes.byref(_CConfig()), ctypes.byref(h)) == -2
    assert lib.b200ba_last_error() == b"image references a camera outside the scene"
    cov = _CCovOptions(7, 1e-8)
    assert lib.b200ba_estimate_covariance(ctypes.byref(co), ctypes.byref(cov), ctypes.byref(_CProblem()), ctypes.byref(h)) == -2
    assert lib.b200ba_last_error() == b"unknown covariance mode"
    assert lib.b200ba_solve(None, None, None) == -1
    assert lib.b200ba_last_error() == b"null argument"



# ---------------------------------------------------------------- C++ problem assembly == the Python mirror's
def _apply_two_cams_gauge(options, config, flat, image_ids):
    """what BundleAdjuster.Solve does after flatten_reconstruction (gauge search over the config's images)."""
    from colmap_b200.bundle_adjustment import FlatProblem, TWO_CAMS_FROM_WORLD
    if not (config.FixedGauge() == TWO_CAMS_FROM_WORLD and options.refine_rig_from_world):
        return flat
    lib = _bind(load_library())
    in_cfg = np.array([1 if i in config.Images() else 0 for i in image_ids], np.uint8)
    sub = FlatProblem(flat.poses[in_cfg == 1], flat.pose_constant[in_cfg == 1], flat.pose_fixed_dim[in_cfg == 1], flat.cam_model,
                      flat.cam_off, flat.cam_params, flat.cam_constant, flat.points, flat.point_constant, np.zeros(0, np.int32),
                      np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros((0, 2)))
    out_c = np.zeros(len(sub.poses), np.uint8); out_d = -np.ones(len(sub.poses), np.int8)
    co, csub = options.to_c(), sub.to_c()
    lib.b200ba_fix_gauge_two_cams_from_world(ctypes.byref(csub), ctypes.byref(co), out_c.ctypes.data_as(_u8p), out_d.ctypes.data_as(_i8p))
    idx = np.nonzero(in_cfg)[0]
    flat.pose_constant = flat.pose_constant.copy(); flat.pose_fixed_dim = flat.pose_fixed_dim.copy()
    flat.pose_constant[idx] = out_c; flat.pose_fixed_dim[idx] = out_d
    return flat


@pytest.mark.parametrize("case", ["all_images", "subset_with_config_points", "constants_and_ignored", "min_track_length", "no_points_refined"])
def test_cpp_assembly_equals_the_python_mirror(case):
    from colmap_b200.bundle_adjustment import (BundleAdjustmentConfig, TWO_CAMS_FROM_WORLD, assemble_reconstruction,
                                               flatten_reconstruction)
    from colmap_b200.synthetic import flat_to_reconstruction
    gt, noisy = synthesize_ba_problem(7, 90, 4, models=(SIMPLE_RADIAL, PINHOLE), seed=6)
    rec = flat_to_reconstruction(noisy)
    cfg = BundleAdjustmentConfig()
    o = BundleAdjustmentOptions()
    ids = sorted(rec.images)
    if case == "all_images":
        for i in ids: cfg.AddImage(i)
        cfg.FixGauge(TWO_CAMS_FROM_WORLD)
    elif case == "subset_with_config_points":
        for i in ids[:4]: cfg.AddImage(i)
        for p in list(rec.points3D)[:10]: cfg.AddVariablePoint(p)
        for p in list(rec.points3D)[10:15]: cfg.AddConstantPoint(p)
        cfg.FixGauge(TWO_CAMS_FROM_WORLD)
    elif case == "constants_and_ignored":
        for i in ids: cfg.AddImage(i)
        cfg.SetConstantRigFromWorldPose(ids[2]); cfg.SetConstantCamIntrinsics(rec.images[ids[1]].camera_id)
        for p in list(rec.points3D)[:7]: cfg.IgnorePoint(p)
        cfg.FixGauge(TWO_CAMS_FROM_WORLD)
    elif case == "min_track_length":
        for i in ids: cfg.AddImage(i)
        o = BundleAdjustmentOptions(min_track_length=5)        # tracks have 4 observations: nothing is left
    else:
        for i in ids[1:]: cfg.AddImage(i)
        o = BundleAdjustmentOptions(refine_points3D=False, refine_rig_from_world=False)
        cfg.FixGauge(TWO_CAMS_FROM_WORLD)
    a, ia, ca, pa = assemble_reconstruction(o, cfg, rec)
    b, ib, cb, pb = flatten_reconstruction(o, cfg, rec)
    b = _apply_two_cams_gauge(o, cfg, b, ib)
    assert (ia, ca, pa) == (ib, cb, pb)
    for name in ("poses", "pose_constant", "pose_fixed_dim", "cam_model", "cam_off", "cam_params", "cam_constant", "points",
                 "point_constant", "obs_pose", "obs_cam", "obs_point", "obs_xy"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name
    if case == "min_track_length":
        assert len(a.obs_pose) == 0
    if case == "subset_with_config_points":
        assert np.any(~np.isin(a.obs_pose, [0, 1, 2, 3]))       # observations brought in by the config points
    # the assembled problem is what the solver's host flattening accepts
    if len(a.obs_pose):
        L = _pack(a, o)
        assert L["nslots"] >= len(a.obs_pose) or (L["s_obs"] >= 0).sum() <= len(a.obs_pose)


# ---------------------------------------------------------------- camera models with > 5 parameters (groundwork, SURVEY 8f-4)
_WIDE = {4: [600., 610., 320., 240., 0.08, -0.02, 0.001, -0.0015],                                    # OPENCV
         5: [600., 610., 320., 240., 0.05, -0.01, 0.004, -0.001],                                      # OPENCV_FISHEYE
         6: [600., 610., 320., 240., 0.08, -0.02, 0.001, -0.0015, 0.004, 0.03, -0.01, 0.002],          # FULL_OPENCV
         7: [600., 610., 320., 240., 0.9],                                                             # FOV
         10: [600., 610., 320., 240., 0.05, -0.01, 0.001, -0.0015, 0.004, -0.001, 0.002, -0.003],      # THIN_PRISM_FISHEYE
         11: [600., 610., 320., 240., 0.05, -0.01, 0.004, -0.001, 0.0005, -0.0002, 0.001, -0.0015, 0.002, -0.001, 0.0015, 0.0007],  # RAD_TAN_THIN_PRISM_FISHEYE
         12: [600., 320., 240., -0.05],                                                                # SIMPLE_DIVISION
         13: [600., 610., 320., 240., -0.05],                                                          # DIVISION
         14: [600., 320., 240.],                                                                       # SIMPLE_FISHEYE
         15: [600., 610., 320., 240.],                                                                 # FISHEYE
         16: [600., 610., 320., 240., 0.6, 1.2],                                                       # EUCM
         17: [1000., 500.]}                                                                            # EQUIRECTANGULAR


def _project_wide(fn, model, params, uvw):
    P = len(params)
    xy, Juvw, Jp = np.zeros(2), np.zeros((2, 3)), np.zeros((2, P))
    prm, p3 = np.ascontiguousarray(params, np.float64), np.ascontiguousarray(uvw, np.float64)
    rc = fn(model, prm.ctypes.data_as(_f64p), p3.ctypes.data_as(_f64p), xy.ctypes.data_as(_f64p), Juvw.ctypes.data_as(_f64p),
            Jp.ctypes.data_as(_f64p))
    return rc, xy, Juvw, Jp


@pytest.mark.parametrize("model", sorted(_WIDE))
def test_wide_models_dual_numbers_vs_complex_step_oracle(model):
    """Product: formulas + forward-mode dual numbers (ba_models.cuh); oracle: the same models over complex numbers with
    complex-step derivatives; plus central finite differences of the product's own value.  Known answer: with all
    distortion parameters zero OPENCV / FULL_OPENCV reduce to PINHOLE (sensor/models.h:1513-1543)."""
    lib = load_library()
    lib.b200ba_test_project_wide.argtypes = [ctypes.c_int] + [_f64p] * 5
    ol = oracle_ba.lib()
    ol.ba_oracle_project_wide.argtypes = [ctypes.c_int] + [_f64p] * 5
    rng = np.random.default_rng(model)
    params = np.asarray(_WIDE[model])
    cases = [rng.uniform(-1.2, 1.2, 3) * [1, 1, 0] + [0, 0, rng.uniform(2, 6)] for _ in range(40)]
    cases += [np.array([1e-9, -1e-9, 3.0]), np.array([0.0, 0.0, 2.0])]        # r -> 0 branches
    if model == 7:
        cases += [np.array([0.001, 0.002, 1.0])]                              # FOV small-radius branch
    for uvw in cases:
        rc, xy, Juvw, Jp = _project_wide(lib.b200ba_test_project_wide, model, params, uvw)
        rc2, xy2, Juvw2, Jp2 = _project_wide(ol.ba_oracle_project_wide, model, params, uvw)
        assert rc == rc2 == 1
        assert np.allclose(xy, xy2, rtol=1e-13, atol=1e-10)
        tol = 1e-6 if model == 17 else 1e-9          # the equirectangular oracle differentiates numerically
        assert np.allclose(Juvw, Juvw2, rtol=tol, atol=tol) and np.allclose(Jp, Jp2, rtol=tol, atol=tol)
        if np.hypot(uvw[0], uvw[1]) > 1e-3:       # finite differences (away from the non-smooth point of sqrt)
            for k in range(3):
                e = np.zeros(3); e[k] = 1e-6
                fd = (_project_wide(lib.b200ba_test_project_wide, model, params, uvw + e)[1] -
                      _project_wide(lib.b200ba_test_project_wide, model, params, uvw - e)[1]) / 2e-6
                assert np.allclose(Juvw[:, k], fd, rtol=1e-5, atol=1e-4)
            for k in range(len(params)):
                e = np.zeros(len(params)); e[k] = 1e-6 * max(1.0, abs(params[k]))
                fd = (_project_wide(lib.b200ba_test_project_wide, model, params + e, uvw)[1] -
                      _project_wide(lib.b200ba_test_project_wide, model, params - e, uvw)[1]) / (2 * e[k])
                assert np.allclose(Jp[:, k], fd, rtol=1e-5, atol=1e-4)
    # depth guard and unknown ids
    if model not in (12, 13, 17):                 # the division and equirectangular models have no depth guard
        assert _project_wide(lib.b200ba_test_project_wide, model, params, [0.1, 0.1, 0.0])[0] == 0
        assert _project_wide(ol.ba_oracle_project_wide, model, params, [0.1, 0.1, -1.0])[0] == 0
    if model == 17:
        assert _project_wide(lib.b200ba_test_project_wide, model, params, [0.0, 0.0, 0.0])[0] == 0
        assert _project_wide(lib.b200ba_test_project_wide, model, params, [0.3, 0.2, -1.0])[0] == 1      # behind the camera is fine on a sphere
    if model in (12, 13):
        pos = list(params); pos[-1] = 0.5
        assert _project_wide(lib.b200ba_test_project_wide, model, pos, [3.0, 3.0, 1.0])[0] == 0          # negative discriminant
    assert _project_wide(lib.b200ba_test_project_wide, 99, params, [0, 0, 1.0])[0] == -1
    if model in (4, 6):
        zero = params.copy(); zero[4:] = 0.0
        uvw = np.array([0.3, -0.2, 2.0])
        xy = _project_wide(lib.b200ba_test_project_wide, model, zero, uvw)[1]
        assert np.allclose(xy, [zero[0] * 0.15 + zero[2], zero[1] * -0.1 + zero[3]], rtol=1e-15)


def test_three_points_gauge_assembly_and_oracle_solve():
    """FixGaugeWithThreePoints (bundle_adjustment_ceres.cc:270-306): C++ assembly == Python mirror; already-constant points
    count first; collinear-with-origin candidates are skipped; the oracle converges under that gauge."""
    from colmap_b200.bundle_adjustment import (BundleAdjustmentConfig, THREE_POINTS, assemble_reconstruction, fix_gauge_three_points,
                                               flatten_reconstruction)
    from colmap_b200.synthetic import flat_to_reconstruction
    gt, noisy = synthesize_ba_problem(6, 80, 4, models=(PINHOLE,), shared_camera=True, seed=12)
    noisy.points[1] = 2.0 * noisy.points[0]            # same direction as point 0: adds no rank
    rec = flat_to_reconstruction(noisy)
    ids = sorted(rec.points3D)
    cfg = BundleAdjustmentConfig()
    for i in rec.images: cfg.AddImage(i)
    cfg.AddConstantPoint(ids[5])                       # an explicit constant point is used first
    cfg.FixGauge(THREE_POINTS)
    o = BundleAdjustmentOptions(max_num_iterations=50)
    a = assemble_reconstruction(o, cfg, rec)[0]
    b = flatten_reconstruction(o, cfg, rec)[0]
    assert fix_gauge_three_points(b) == 3
    assert np.array_equal(a.point_constant, b.point_constant)
    fixed = np.nonzero(a.point_constant)[0]
    assert list(fixed) == [0, 2, 5]                    # 5 (already constant), then 0, skip collinear 1, then 2
    assert np.linalg.matrix_rank(a.points[fixed].T) == 3
    assert not a.pose_constant.any() and np.all(a.pose_fixed_dim == -1)      # no camera is touched by this gauge
    before = a.points[fixed].copy()
    s = oracle_ba.solve(o, a)
    assert s.termination_type in (0, 1) and s.final_cost < 1e-2 * s.initial_cost
    assert np.array_equal(a.points[fixed], before)
    assert s.num_effective_parameters == 6 * 6 + 2 + 3 * (80 - 3)             # fx, fy of the shared camera


def test_two_cams_gauge_falls_back_to_three_points():
    """One image in the config: no second camera exists, so the reference fixes three points instead
    (bundle_adjustment_ceres.cc:386-394)."""
    from colmap_b200.bundle_adjustment import BundleAdjustmentConfig, TWO_CAMS_FROM_WORLD, assemble_reconstruction
    from colmap_b200.synthetic import flat_to_reconstruction
    gt, noisy = synthesize_ba_problem(3, 40, 3, models=(PINHOLE,), seed=2)
    rec = flat_to_reconstruction(noisy)
    cfg = BundleAdjustmentConfig()
    cfg.AddImage(sorted(rec.images)[0])
    cfg.FixGauge(TWO_CAMS_FROM_WORLD)
    a = assemble_reconstruction(BundleAdjustmentOptions(), cfg, rec)[0]
    assert a.pose_constant[0] == 0 and np.all(a.pose_fixed_dim == -1)
    # points observed only partly inside the config are constant anyway (ParameterizePoints): the gauge is already held
    assert a.point_constant.sum() >= 3


# ---------------------------------------------------------------- rigs + the twelve wide camera models (SURVEY 8a / 8f-4)
ALL_MODELS = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17]


def _product_reproj_rig(model, point, rig, sensor, params, xy):
    lib = _bind(load_library())
    f = ctypes.POINTER(ctypes.c_double)
    lib.b200ba_test_reproj_rig.argtypes = [ctypes.c_int, f, f, f, f, f, f, f, f, f, f]
    d = lambda a: np.ascontiguousarray(a, np.float64)
    point, rig, params, xy = d(point), d(rig), d(params), d(xy)
    sp = d(sensor).ctypes.data_as(f) if sensor is not None else None
    res = np.zeros(2); Jpt = np.zeros((2, 3)); Jr = np.zeros((2, 7)); Js = np.zeros((2, 7)); Jp = np.zeros((2, len(params)))
    ok = lib.b200ba_test_reproj_rig(model, point.ctypes.data_as(f), rig.ctypes.data_as(f), sp, params.ctypes.data_as(f), xy.ctypes.data_as(f),
                                    res.ctypes.data_as(f), Jpt.ctypes.data_as(f), Jr.ctypes.data_as(f), Js.ctypes.data_as(f), Jp.ctypes.data_as(f))
    return ok, res, Jpt, Jr, Js, Jp


@pytest.mark.parametrize("model", ALL_MODELS)
@pytest.mark.parametrize("with_sensor", [False, True])
def test_rig_reprojection_all_models_product_vs_oracle_vs_finite_differences(model, with_sensor):
    """RigReprojErrorCostFunctor (reprojection_error.h:344-420) with analytic derivatives for every camera model: the
    product's device code (evaluated on the host), the oracle (independent: complex step for the wide models) and central
    differences of the residual must agree - the reference's own property test (reprojection_error_test.cc:211-323:
    analytic == autodiff to 1e-4... here 1e-6 relative)."""
    import oracle_ba
    from colmap_b200.synthetic import _MODEL_DEFAULTS
    rng = np.random.default_rng(100 + model)
    params = np.array(_MODEL_DEFAULTS[model], np.float64)
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    rig = np.r_[q, rng.normal(size=3) * 0.1]
    X = np.array([0.2, -0.1, 0.3])
    # put the point ~4 in front of the camera
    qs = rng.normal(size=4) * 0.05 + np.array([0, 0, 0, 1.0]); qs /= np.linalg.norm(qs)
    sensor = np.r_[qs, rng.normal(size=3) * 0.1] if with_sensor else None
    rig[4:] += np.array([0, 0, 4.0])
    xy = np.array([500.0, 400.0])
    ok_p, res_p, Jpt_p, Jr_p, Js_p, Jp_p = _product_reproj_rig(model, X, rig, sensor, params, xy)
    ok_o, res_o, Jpt_o, Jr_o, Js_o, Jp_o = oracle_ba.reproj_rig(model, X, rig, sensor, params, xy)
    assert ok_p == 1 and ok_o == 1
    for a, b in ((res_p, res_o), (Jpt_p, Jpt_o), (Jr_p, Jr_o), (Js_p, Js_o), (Jp_p, Jp_o)):
        assert np.allclose(a, b, rtol=1e-7, atol=1e-7 * max(1.0, np.abs(b).max()))
    # central differences of the product's residual
    def resid(Xv, rv, sv, pv):
        return _product_reproj_rig(model, Xv, rv, sv, pv, xy)[1]
    def fd(fun, v, h=1e-6):
        J = np.zeros((2, len(v)))
        for k in range(len(v)):
            hk = h * max(1.0, abs(v[k]))
            a, b = v.copy(), v.copy(); a[k] += hk; b[k] -= hk
            J[:, k] = (fun(a) - fun(b)) / (2 * hk)
        return J
    tol = dict(rtol=2e-5, atol=2e-4)
    assert np.allclose(Jpt_p, fd(lambda v: resid(v, rig, sensor, params), X), **tol)
    assert np.allclose(Jr_p, fd(lambda v: resid(X, v, sensor, params), rig), **tol)
    if with_sensor:
        assert np.allclose(Js_p, fd(lambda v: resid(X, rig, v, params), sensor), **tol)
    else:
        assert not Js_p.any()
    assert np.allclose(Jp_p, fd(lambda v: resid(X, rig, sensor, v), params), **tol)


def test_oracle_recovers_ground_truth_with_rig_and_wide_models():
    """bundle_adjustment_ceres_test.cc rig scenarios in spirit (synthetic rig, noise, solve, compare with the ground truth):
    one rig of three sensors (OPENCV, SIMPLE_RADIAL, FISHEYE), 8 frames; rig poses, sensor_from_rig poses, intrinsics and
    points variable; the oracle must bring the reprojection RMSE back to the noise floor and the sensor_from_rig poses to
    the truth."""
    import oracle_ba
    from colmap_b200.synthetic import synthesize_rig_problem
    gt, noisy = synthesize_rig_problem(8, 3, 600, 8, models=(4, 2, 15), seed=3, point2D_stddev=0.5)
    noisy.pose_constant = noisy.pose_constant.copy(); noisy.pose_fixed_dim = noisy.pose_fixed_dim.copy()
    noisy.pose_constant[0] = 1
    noisy.pose_fixed_dim[1] = int(np.argmax(np.abs(noisy.poses[1, 4:] - noisy.poses[0, 4:])))
    s = oracle_ba.solve(BundleAdjustmentOptions(), noisy)
    assert s.termination_type in (0, 1) and s.num_residuals == 2 * 600 * 8
    assert s.num_effective_parameters == 6 * 7 - 1 + 6 * 2 + (6 + 2 + 2) + 3 * 600       # poses (gauge), sensors, intrinsics, points
    rmse = np.sqrt(2 * s.final_cost / (600 * 8))
    assert rmse < 0.5 * np.sqrt(2) * 1.1
    assert np.abs(noisy.sensors[:, 4:] - gt.sensors[:, 4:]).max() < 5e-3
    dq = np.abs(np.sum(noisy.sensors[:, :4] * gt.sensors[:, :4], axis=1))
    assert np.all(dq > 1 - 1e-5)


def _noisy_rig_reconstruction(seed=4):
    """NominalMultiCameraRig's scene (bundle_adjustment_ceres_test.cc:183-220): 2 rigs x 3 cameras x 5 frames, 200 points, noise
    0.5 px / 0.1 (points) / 0.5 deg + 0.1 (rig_from_world).  Returns (ground truth, noisy) reconstructions."""
    import copy
    from colmap_b200.synthetic import _quat_mul, synthesize_rig_reconstruction
    gt = synthesize_rig_reconstruction(2, 3, 5, 200, model=SIMPLE_RADIAL, seed=seed, point2D_stddev=0.5)
    noisy = copy.deepcopy(gt)
    rng = np.random.default_rng(seed + 100)
    for p in noisy.points3D.values():
        p.xyz += rng.normal(0, 0.1, 3)
    for f in noisy.frames.values():
        a = np.deg2rad(rng.normal(0, 0.5))
        f.rig_from_world[:4] = _quat_mul(f.rig_from_world[None, :4], np.array([[0, 0, np.sin(a / 2), np.cos(a / 2)]]))[0]
        f.rig_from_world[4:] += rng.normal(0, 0.1, 3)
    return gt, noisy


def test_rig_assembly_with_images_outside_the_config_and_oracle_solve():
    """A local-BA-shaped rig problem: only the images of two frames are in the config, two config points bring in their
    observations from images outside it.  Those observations sit on CONSTANT copies of their frames' poses appended after
    the frame poses (the reference bakes them with a constant pose, bundle_adjustment_ceres.cc:846-878), their cameras
    become constant (:880-884); the C++ assembly equals the Python mirror; the oracle's solve leaves every constant
    block bit-identical and moves the variable ones."""
    import oracle_ba
    from colmap_b200.bundle_adjustment import (BundleAdjustmentConfig, TWO_CAMS_FROM_WORLD, assemble_reconstruction,
                                               flatten_reconstruction)
    gt, rec = _noisy_rig_reconstruction()
    cfg = BundleAdjustmentConfig()
    in_cfg = [i for i, im in rec.images.items() if im.frame_id in (1, 2)]      # rig 1, frames 1 and 2: images 1..6
    for i in in_cfg:
        cfg.AddImage(i)
    cfg.AddVariablePoint(7); cfg.AddConstantPoint(9)
    cfg.FixGauge(TWO_CAMS_FROM_WORLD)
    o = BundleAdjustmentOptions(max_num_iterations=10)
    flat_py, frame_ids, camera_ids, point_ids = flatten_reconstruction(o, cfg, rec)
    flat = assemble_reconstruction(o, cfg, rec)[0]
    for name in ("poses", "pose_constant", "pose_fixed_dim", "cam_constant", "point_constant", "obs_pose", "obs_cam", "obs_point",
                 "obs_xy", "sensors", "sensor_constant", "cam_sensor"):
        assert np.array_equal(getattr(flat, name), getattr(flat_py, name)), name
    n_out = len(rec.images) - len(in_cfg)
    assert len(flat.poses) == len(frame_ids) + n_out                      # one constant pose per outside image
    assert np.all(flat.pose_constant[len(frame_ids):] == 1)
    assert len(flat.obs_pose) == 200 * len(in_cfg) + 2 * n_out            # every point from the six images + 2 points from the others
    # points other than 7 have part of their track outside the problem: constant; 7 is fully inside now: variable; 9 constant
    assert flat.point_constant[point_ids.index(7)] == 0 and flat.point_constant[point_ids.index(9)] == 1
    assert int((flat.point_constant == 0).sum()) == 1
    assert np.all(flat.cam_constant[3:] == 1) and np.all(flat.cam_constant[:3] == 0)     # rig 2's cameras: outside images only
    before = flat.copy()
    s = oracle_ba.solve(o, flat)
    # point 9 is constant: its 15 observations from rig 2 (constant cameras, baked poses, sensors that are no parameter blocks)
    # touch nothing variable and do not count (bundle_adjustment.h:66-68)
    assert s.termination_type in (0, 1) and s.num_residuals == 2 * (len(flat.obs_pose) - 15)
    assert s.num_effective_parameters == (12 - 7) + 2 * 6 + 3 * 2 + 3          # frames 1, 2 minus the gauge, rig 1's sensors, cameras 1-3, point 7
    assert np.array_equal(flat.poses[2:], before.poses[2:])               # frames 3.. and the outside copies untouched
    assert np.array_equal(flat.poses[0], before.poses[0])                 # gauge: frame 1 fixed
    assert not np.array_equal(flat.poses[1], before.poses[1])
    assert not np.array_equal(flat.sensors[:2], before.sensors[:2]) and np.array_equal(flat.sensors[2:], before.sensors[2:])
    moved = np.nonzero(np.any(flat.points != before.points, axis=1))[0]
    assert [point_ids[k] for k in moved] == [7]
    assert s.final_cost < s.initial_cost
