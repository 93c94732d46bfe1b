"""GPU tier of the pose-prior bundle adjustment: b200ba_solve_with_position_priors against the CPU oracle
(tests/ba_prior_oracle.c) on the same inputs, over every solve regime of test_ba_paths_gpu.py, the prior losses, full and
fallback covariances, rigs with priors on non-reference sensors and constant blocks; zero priors bit-identical to
b200ba_solve; the reference's five pose-prior tests restated through CreatePosePriorBundleAdjuster; B3 with priors."""
import copy
import dataclasses

import numpy as np
import pytest

import oracle_prior
from colmap_b200.bundle_adjustment import (CAUCHY, DENSE_SCHUR, HUBER, ITERATIVE_SCHUR, SIMPLE_RADIAL, SOFT_L1, TRIVIAL,
                                           TWO_CAMS_FROM_WORLD, BundleAdjustmentConfig, BundleAdjustmentOptions,
                                           FlatPositionPriors, PosePriorBundleAdjustmentOptions, RANSACOptions,
                                           CreatePosePriorBundleAdjuster, solve_flat, solve_flat_with_position_priors)
from colmap_b200.synthetic import synthesize_ba_problem, synthesize_noise, synthesize_rig_reconstruction
from prior_cases import flat_priors, reconstruction_near
from test_ba_gpu import _gauge
from test_ba_paths_gpu import DENSE, ITER, SEAMS, _problem, regime

pytestmark = pytest.mark.gpu


def _both(options, noisy, priors):
    a, b = noisy.copy(), noisy.copy()
    for f in (a, b):
        f.pose_constant, f.pose_fixed_dim, f.point_constant, f.cam_constant = (noisy.pose_constant, noisy.pose_fixed_dim,
                                                                                noisy.point_constant, noisy.cam_constant)
        f.sensor_constant = noisy.sensor_constant
    sg = solve_flat_with_position_priors(options, a, priors)
    sr = oracle_prior.solve(options, b, priors)
    return a, sg, b, sr


def _groups(a, b):
    g = [(a.poses, b.poses), (a.points, b.points), (a.cam_params, b.cam_params)]
    return g + [(a.sensors, b.sensors)] if len(b.sensors) else g


def _msg(sg, sr):
    return (f"gpu cost {sg.initial_cost!r} -> {sg.final_cost!r} ({sg.num_successful_steps}+{sg.num_unsuccessful_steps}, "
            f"{sg.num_linear_solver_iterations} PCG) oracle {sr.initial_cost!r} -> {sr.final_cost!r} "
            f"({sr.num_successful_steps}+{sr.num_unsuccessful_steps}, {sr.num_linear_solver_iterations} PCG)")


def _arithmetic(options, noisy, priors, iters=3, cam_rel=1e-5, cost_rel=1e-6, param_rel=1e-5):
    """The bar of test_ba_paths_gpu.py: cost 1e-6, parameters 1e-5, equal step and (ITERATIVE_SCHUR) PCG counts."""
    a, sg, b, sr = _both(dataclasses.replace(options, max_num_iterations=iters), noisy, priors)
    msg = _msg(sg, sr)
    assert sg.num_residuals == sr.num_residuals and sg.num_effective_parameters == sr.num_effective_parameters, msg
    assert abs(sg.initial_cost - sr.initial_cost) <= 1e-9 * sr.initial_cost, msg
    assert sg.num_successful_steps == sr.num_successful_steps and sg.num_unsuccessful_steps == sr.num_unsuccessful_steps, msg
    assert abs(sg.final_cost - sr.final_cost) <= cost_rel * sr.final_cost, msg
    for u, v in _groups(a, b):
        rel = cam_rel if u is a.cam_params else param_rel
        assert np.allclose(u, v, rtol=rel, atol=rel * max(1.0, np.abs(v).max())), f"{msg}; max |diff| {np.abs(u - v).max():.3g}"
    if options.linear_solver_type == ITERATIVE_SCHUR and iters <= 3:
        assert sg.num_linear_solver_iterations == sr.num_linear_solver_iterations, msg
    return a, sg, b, sr


def _full(options, noisy, priors, iters=100):
    """A full run: both usable, cost 1e-5, parameters 1e-4."""
    a, sg, b, sr = _both(dataclasses.replace(options, max_num_iterations=iters), noisy, priors)
    msg = _msg(sg, sr)
    assert sg.termination_type in (0, 1) and sr.termination_type in (0, 1), msg
    assert abs(sg.final_cost - sr.final_cost) <= 1e-5 * sr.final_cost, msg
    for u, v in _groups(a, b):
        assert np.allclose(u, v, rtol=1e-4, atol=1e-4 * max(1.0, np.abs(v).max())), f"{msg}; max |diff| {np.abs(u - v).max():.3g}"


@pytest.fixture
def clean_env(monkeypatch):
    for k in SEAMS:
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


# (problem of test_ba_paths_gpu.py, options, environment, expected path)
REGIMES = [
    ("nc256", DENSE, (), "dense"),
    ("seam_narrow", ITER, (), "staged"),
    ("seam_narrow", ITER, (("B200BA_MID_PLAIN", "1"),), "mid_smem"),
    ("seam_narrow", ITER, (("B200BA_MID_PLAIN", "1"), ("B200BA_MID_GLOBAL", "1")), "mid_global"),
    ("seam_narrow", ITER, (("B200BA_PCG_MULTI", "1"),), "multi"),
    ("nc256", DENSE, (("B200BA_NO_DENSE", "1"),), "staged"),
    ("rig_opencv", ITER, (), "staged"),
    ("rig_rad_tan_thin_prism", dataclasses.replace(DENSE, refine_principal_point=True), (), "dense"),
    ("rig_rad_tan_thin_prism", dataclasses.replace(ITER, refine_principal_point=True), (), "staged"),
]


@pytest.mark.parametrize("problem,options,env,path", REGIMES, ids=[f"{p}-{w}-{i}" for i, (p, _, _, w) in enumerate(REGIMES)])
def test_parity_every_regime(problem, options, env, path, clean_env):
    for k, v in env:
        clean_env.setenv(k, v)
    noisy = _problem(problem)
    r = regime(noisy, options, dict(env))
    assert r["path"] == path, r
    if problem.startswith("rig_rad"):
        assert r["DC"] == 28
    priors = flat_priors(noisy, seed=5)
    cam_rel = 1e-4 if (problem.startswith("rig_rad") and path != "dense") else 1e-5
    _arithmetic(options, noisy, priors, cam_rel=cam_rel)


@pytest.mark.parametrize("loss", [TRIVIAL, CAUCHY, HUBER, SOFT_L1])
@pytest.mark.parametrize("cov", ["full", "fallback"])
def test_parity_losses_and_covariances(loss, cov, clean_env):
    noisy = _problem("seam_narrow")
    # priors tighter than the scene noise, so the robust losses see residuals on both sides of their scale
    priors = flat_priors(noisy, seed=7, stddev=0.02, cov=cov, loss=loss, loss_scale=1.0)
    _arithmetic(ITER, noisy, priors)
    _full(ITER, noisy, priors)


@pytest.mark.parametrize("case", ["sensor_variable", "sensor_constant", "rig_constant", "constant_rotation",
                                  "no_sensor_refine"])
def test_parity_rigs_and_constant_blocks(case, clean_env):
    noisy = _problem("rig_opencv").copy()
    noisy.pose_constant, noisy.pose_fixed_dim = _problem("rig_opencv").pose_constant.copy(), _problem("rig_opencv").pose_fixed_dim.copy()
    noisy.sensor_constant = noisy.sensor_constant.copy()
    options = ITER
    if case == "sensor_constant":
        noisy.sensor_constant[:] = 1
    elif case == "rig_constant":
        noisy.pose_constant[:] = 1          # only the sensor blocks carry the priors of the non-reference cameras
    elif case == "constant_rotation":
        options = dataclasses.replace(ITER, constant_rig_from_world_rotation=True)
    elif case == "no_sensor_refine":
        options = dataclasses.replace(ITER, refine_sensor_from_rig=False)
    priors = flat_priors(noisy, seed=9)
    # with the frame rotations constant the sensor rotations carry the orientation alone and are weakly determined: the
    # GPU (fp32-stored Jacobians) and the oracle agree to 2.5e-7 in cost with equal PCG counts, while the sensor_from_rig
    # parameters differ by up to 1.8e-5 (measured), so that case compares them at 1e-4
    a, sg, b, sr = _arithmetic(options, noisy, priors, param_rel=1e-4 if case == "constant_rotation" else 1e-5)
    if case == "rig_constant":      # the reference-sensor priors have every block constant and are skipped
        assert sg.num_residuals == 2 * len(noisy.obs_pose) + 3 * len(noisy.poses) * len(noisy.sensors)


def test_zero_priors_is_the_plain_solve(clean_env):
    """num_priors == 0 takes b200ba_solve's code path (the entry drops the priors before anything else): the same
    residuals and the same result up to the run-to-run spread of the fp64 atomics, at the parity bar.  (On the rig
    problems two plain b200ba_solve runs already differ by a few PCG iterations and 1e-5 in the points after five LM
    iterations, so they are not a fair probe of this.)"""
    for problem, options in (("seam_narrow", ITER), ("nc256", DENSE)):
        noisy = _problem(problem)
        a, b = noisy.copy(), noisy.copy()
        for f in (a, b):
            f.pose_constant, f.pose_fixed_dim = noisy.pose_constant, noisy.pose_fixed_dim
        sa = solve_flat(dataclasses.replace(options, max_num_iterations=5), a)
        sb = solve_flat_with_position_priors(dataclasses.replace(options, max_num_iterations=5), b,
                                             FlatPositionPriors(np.zeros(0), np.zeros(0), np.zeros((0, 3)), np.zeros((0, 3, 3))))
        assert sa.num_residuals == sb.num_residuals and sa.num_effective_parameters == sb.num_effective_parameters
        assert sa.num_successful_steps == sb.num_successful_steps
        assert abs(sa.initial_cost - sb.initial_cost) <= 1e-12 * sa.initial_cost
        assert abs(sa.final_cost - sb.final_cost) <= 1e-6 * sa.final_cost
        for u, v in _groups(a, b):
            assert np.allclose(u, v, rtol=1e-5, atol=1e-5 * max(1.0, np.abs(v).max()))


# ---------------------------------------------------------------- the reference's pose-prior tests
def _scene(num_frames, num_points, seed, **noise):
    gt, priors = synthesize_rig_reconstruction(1, 1, num_frames, num_points, seed=seed, prior_position=True)
    rec = copy.deepcopy(gt)
    synthesize_noise(rec, priors, seed=seed + 1, **noise)
    config = BundleAdjustmentConfig()
    for i in rec.images:
        config.AddImage(i)
    return gt, rec, priors, config


def _prior_options(**kw):
    return PosePriorBundleAdjustmentOptions(alignment_ransac_options=RANSACOptions(random_seed=0, **kw))


def test_nominal():
    """bundle_adjustment_test.cc:423-481"""
    gt, rec, priors, config = _scene(7, 100, 21, point2D_stddev=0.5, point3D_stddev=0.1, rig_from_world_rotation_stddev=0.5,
                                     rig_from_world_translation_stddev=0.1, prior_position_stddev=0.05)
    ba = CreatePosePriorBundleAdjuster(BundleAdjustmentOptions(), _prior_options(), config, priors, rec)
    assert ba.Config().NumImages() == 7
    s = ba.Solve()
    assert s.IsSolutionUsable() and s.num_residuals > 0
    ok, msg = reconstruction_near(gt, rec, 0.1, 0.1)
    assert ok, msg


def test_alignment_robust_to_outliers():
    """bundle_adjustment_ceres_test.cc:1461-1512"""
    gt, rec, priors, config = _scene(7, 50, 23, point3D_stddev=0.2, rig_from_world_rotation_stddev=1.0,
                                     rig_from_world_translation_stddev=0.2, prior_position_stddev=0.05)
    priors[0].position = priors[0].position + 10; priors[0].position_covariance = np.eye(3) * 1e6
    priors[1].position = priors[1].position + 1; priors[1].position_covariance = np.eye(3) * 1e2
    s = CreatePosePriorBundleAdjuster(BundleAdjustmentOptions(), _prior_options(max_error=0.0), config, priors, rec).Solve()
    assert s.IsSolutionUsable()
    ok, msg = reconstruction_near(gt, rec, 0.1, 0.1)
    assert ok, msg


def test_insufficient_priors_use_two_camera_gauge():
    """bundle_adjustment_ceres_test.cc:1514-1548"""
    gt, rec, priors, config = _scene(3, 50, 25)
    ba = CreatePosePriorBundleAdjuster(BundleAdjustmentOptions(), _prior_options(), config, priors[:2], rec)
    assert ba.Config().FixedGauge() == TWO_CAMS_FROM_WORLD
    assert ba.Solve().IsSolutionUsable()


def test_missing_position_cov():
    """bundle_adjustment_ceres_test.cc:1550-1596: priors without a covariance use the fallback stddev"""
    gt, rec, priors, config = _scene(7, 50, 27, point3D_stddev=0.1, rig_from_world_rotation_stddev=0.5,
                                     rig_from_world_translation_stddev=0.1, prior_position_stddev=0.05)
    for pp in priors:
        pp.position_covariance = np.full((3, 3), np.nan)
    s = CreatePosePriorBundleAdjuster(BundleAdjustmentOptions(), _prior_options(), config, priors, rec).Solve()
    assert s.IsSolutionUsable()
    ok, msg = reconstruction_near(gt, rec, 0.1, 0.1)
    assert ok, msg


def test_optimization_robust_to_outliers():
    """bundle_adjustment_ceres_test.cc:1598-1648: a Cauchy prior loss keeps one gross outlier prior from pulling"""
    gt, rec, priors, config = _scene(7, 50, 29, point3D_stddev=0.1, rig_from_world_rotation_stddev=0.5,
                                     rig_from_world_translation_stddev=0.1, prior_position_stddev=0.05)
    priors[3].position = priors[3].position + 5.0
    po = _prior_options()
    po.prior_position_loss_function_type = CAUCHY
    s = CreatePosePriorBundleAdjuster(BundleAdjustmentOptions(), po, config, priors, rec).Solve()
    assert s.IsSolutionUsable()
    ok, msg = reconstruction_near(gt, rec, 0.1, 0.1)
    assert ok, msg


def test_b3_with_priors_parity():
    """B3 (500 SIMPLE_RADIAL cameras, 300k points, 2M observations, ITERATIVE_SCHUR) with a noisy prior on every image:
    10 LM iterations against the oracle at the large-problem bar of the B3 test (cost 1e-5, parameters 1e-4)."""
    gt, noisy = synthesize_ba_problem(500, 300000, 7, models=(SIMPLE_RADIAL,), seed=42, num_obs=2000000)
    _gauge(noisy)
    priors = flat_priors(noisy, seed=3, stddev=0.05)
    a, sg, b, sr = _both(dataclasses.replace(ITER, max_num_iterations=10), noisy, priors)
    msg = _msg(sg, sr)
    assert sg.num_residuals == 4000000 + 3 * 499, msg      # pose 0 holds the gauge: its prior has no variable block
    assert sg.num_successful_steps + sg.num_unsuccessful_steps == sr.num_successful_steps + sr.num_unsuccessful_steps, msg
    assert abs(sg.final_cost - sr.final_cost) <= 1e-5 * sr.final_cost, msg
    for u, v in _groups(a, b):
        assert np.allclose(u, v, rtol=1e-4, atol=1e-4 * max(1.0, np.abs(v).max())), msg
