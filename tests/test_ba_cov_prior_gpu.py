"""b200ba_estimate_covariance_with_position_priors on the GPU against the covariance oracle with the prior rows appended
(tests/oracle_cov_prior.py), on the same parameter arrays and with no gauge fixed (the priors fix it): the three modes
that form S, the four prior losses, full and fallback prior covariances, priors on every image and on three, a narrow
and a wide camera model, constant rotations, a rig with priors on non-reference sensors, a prior on a constant pose;
estimability with no, non-collinear and collinear priors; zero priors and POINTS mode against the plain estimate; and
EstimateBACovariance through CreatePosePriorBundleAdjuster before and after Solve()."""
import copy

import numpy as np
import pytest

import oracle_cov
import oracle_cov_prior
import oracle_prior
from colmap_b200.bundle_adjustment import (CAUCHY, HUBER, OPENCV, SIMPLE_RADIAL, SOFT_L1, TRIVIAL, TWO_CAMS_FROM_WORLD,
                                           BACovarianceOptions, BundleAdjustmentConfig, BundleAdjustmentOptions,
                                           CovarianceNotEstimable, CreateDefaultBundleAdjuster, CreatePosePriorBundleAdjuster,
                                           EstimateBACovariance, FlatPositionPriors, PosePriorBundleAdjustmentOptions,
                                           RANSACOptions, _quat_to_R, estimate_covariance_flat, solve_flat_with_position_priors)
from colmap_b200.synthetic import synthesize_ba_problem, synthesize_noise, synthesize_rig_problem, synthesize_rig_reconstruction
from prior_cases import flat_priors, random_spd
from test_ba_covariance_gpu import _gpu_blocks

pytestmark = pytest.mark.gpu
WORST = {"abs": 0.0, "rel": 0.0}
MODES = (oracle_cov.ALL, oracle_cov.POSES, oracle_cov.POSES_AND_POINTS)


def _bars(jac, ref):
    """The bars of test_ba_covariance_gpu.py, 1e-8 absolute and 1e-9 relative, unless the conditioning of S calls for
    more.  The Cholesky factorisation and inverse are invariant under diagonal scaling, so the relevant condition number
    is that of D^-1/2 S D^-1/2 (kappa_s): with priors on every image it is 3e4-2e5 and 10 eps kappa_s stays below 1e-9;
    with only three priors the gauge directions rest on nine prior rows and kappa_s reaches 1.7e7 after the solve (a wide
    model with a Cauchy prior loss) and 1.4e8 at unsolved parameters.  There the relative bar is 10 eps kappa_s, and the
    absolute bar the same fraction of the largest block.  Measured on one H100: at most 0.65 eps kappa_s relative there
    (9.5e-9 at kappa_s = 1.4e8), and 1.5e-10 absolute, 6.1e-11 relative where the default bars apply."""
    S, _ = oracle_cov.reduced_matrix(jac)
    d = 1.0 / np.sqrt(np.diag(S))
    kappa_s = np.linalg.cond(S * d[:, None] * d[None, :])
    rel = max(1e-9, 10 * np.finfo(np.float64).eps * kappa_s)
    big = max(np.abs(b).max() for b in ref.values())
    return max(1e-8, rel * big), rel, kappa_s


def compare(options, flat, priors, params, jac=None):
    """GPU blocks against oracle_cov.estimate on the prior-augmented Jacobian, at the bars of _bars."""
    jac = jac if jac is not None else oracle_cov_prior.jacobian(options, flat, priors)
    ref, msg = oracle_cov.estimate(options, flat, params, jac=jac)
    assert ref is not None, msg
    abs_tol, rel_tol, kappa_s = _bars(jac, ref)
    cov = estimate_covariance_flat(options, BACovarianceOptions(params), flat, raise_not_estimable=True, priors=priors)
    got = _gpu_blocks(cov, list(ref))
    worst_abs, worst_rel = (0.0, None), (0.0, None)
    for k in ref:
        assert got[k] is not None and got[k].shape == ref[k].shape, (k, got[k], ref[k].shape)
        err = np.abs(got[k] - ref[k]).max()
        rel = np.linalg.norm(got[k] - ref[k]) / max(np.linalg.norm(ref[k]), 1e-300)
        worst_abs, worst_rel = max(worst_abs, (err, k), key=lambda t: t[0]), max(worst_rel, (rel, k), key=lambda t: t[0])
    WORST["abs"], WORST["rel"] = max(WORST["abs"], worst_abs[0]), max(WORST["rel"], worst_rel[0])
    print(f"params {params}: worst block error {worst_abs[0]:.3g} absolute at {worst_abs[1]}, {worst_rel[0]:.3g} relative "
          f"at {worst_rel[1]}; kappa_s {kappa_s:.3g}, {worst_rel[0] / (np.finfo(np.float64).eps * kappa_s):.3g} eps kappa_s; "
          f"over the file {WORST}")
    assert worst_abs[0] <= abs_tol and worst_rel[0] <= rel_tol, (worst_abs, worst_rel)
    return cov


def _subset(priors, keep):
    return FlatPositionPriors(priors.pose_idx[keep], priors.sensor_idx[keep], priors.position[keep], priors.covariance[keep],
                              priors.loss_function_type, priors.loss_function_scale)


def _scene(model, seed):
    """12 images, no gauge fixed; narrow (SIMPLE_RADIAL) or wide (OPENCV, camera blocks of 6 + 6 columns)."""
    _, flat = synthesize_ba_problem(12, 600, 6, models=(model,), seed=seed, point2D_stddev=0.5)
    return flat


# images 0, 4 and 8 of the 12 are not collinear in every scene used here
THREE = np.array([0, 4, 8])


@pytest.mark.parametrize("model", [SIMPLE_RADIAL, OPENCV], ids=["narrow", "wide"])
@pytest.mark.parametrize("which", ["every", "three"])
@pytest.mark.parametrize("cov", ["full", "fallback"])
@pytest.mark.parametrize("loss", [TRIVIAL, CAUCHY, HUBER, SOFT_L1], ids=["trivial", "cauchy", "huber", "soft_l1"])
def test_grid(loss, cov, which, model):
    flat = _scene(model, seed=31 + model)
    # priors tighter than the scene noise and a loss scale of 1, so the robust losses act on some priors and not others
    priors = flat_priors(flat, seed=7, stddev=0.02, cov=cov, loss=loss, loss_scale=1.0)
    if which == "three":
        priors = _subset(priors, THREE)
    o = BundleAdjustmentOptions(gpu_index=0)
    solve_flat_with_position_priors(o, flat, priors)
    jac = oracle_cov_prior.jacobian(o, flat, priors)
    for params in MODES:
        compare(o, flat, priors, params, jac=jac)


def test_constant_rotation():
    flat = _scene(SIMPLE_RADIAL, seed=41)
    o = BundleAdjustmentOptions(gpu_index=0, constant_rig_from_world_rotation=True)
    priors = flat_priors(flat, seed=11, stddev=0.02)
    solve_flat_with_position_priors(o, flat, priors)
    jac = oracle_cov_prior.jacobian(o, flat, priors)
    for params in MODES:
        cov = compare(o, flat, priors, params, jac=jac)
        assert cov.pose(3).shape == (3, 3)


@pytest.mark.parametrize("loss", [TRIVIAL, CAUCHY], ids=["trivial", "cauchy"])
def test_rig_sensor_priors(loss):
    """Priors on every (frame, sensor) of a three-sensor rig: the non-reference ones add pose-sensor cross terms to S."""
    _, flat = synthesize_rig_problem(8, 3, 400, 5, seed=5, point2D_stddev=0.5)
    o = BundleAdjustmentOptions(gpu_index=0)
    priors = flat_priors(flat, seed=13, stddev=0.02, loss=loss, loss_scale=1.0)
    assert (priors.sensor_idx >= 0).sum() == 2 * len(flat.poses)
    solve_flat_with_position_priors(o, flat, priors)
    jac = oracle_cov_prior.jacobian(o, flat, priors)
    for params in MODES:
        cov = compare(o, flat, priors, params, jac=jac)
        if params == oracle_cov.ALL:
            assert cov.sensor(0).shape == (6, 6) and cov.sensor(1).shape == (6, 6)


def test_prior_on_constant_pose_is_skipped():
    flat = _scene(SIMPLE_RADIAL, seed=43)
    flat.pose_constant = flat.pose_constant.copy()
    flat.pose_constant[0] = 1
    o = BundleAdjustmentOptions(gpu_index=0)
    priors = flat_priors(flat, seed=17, stddev=0.02)
    solve_flat_with_position_priors(o, flat, priors)
    J, columns = oracle_cov.jacobian(o, flat)
    assert oracle_cov_prior.prior_rows(o, flat, priors, columns, J.shape[1])[1] == len(flat.poses) - 1
    cov = compare(o, flat, priors, oracle_cov.ALL)
    assert cov.pose(0) is None


# ---------------------------------------------------------------- estimability
def _collinear(flat, images):
    """Moves the projection centre of images[2] onto the line through those of images[0] and images[1]."""
    c = [-_quat_to_R(flat.poses[i, :4]).T @ flat.poses[i, 4:] for i in images]
    R = _quat_to_R(flat.poses[images[2], :4])
    flat.poses[images[2], 4:] = -R @ (c[0] + 0.5 * (c[1] - c[0]))


def _pivot(msg):
    return float(msg.split("pivot ")[1].split(" ")[0])


def test_estimability():
    """No gauge fixed: not estimable without priors, estimable with three non-collinear ones, not estimable with three
    collinear ones (rotation about their line is free).  The GPU and the oracle agree in each case."""
    flat = _scene(SIMPLE_RADIAL, seed=47)
    o = BundleAdjustmentOptions(gpu_index=0)
    empty = FlatPositionPriors(np.zeros(0), np.zeros(0), np.zeros((0, 3)), np.zeros((0, 3, 3)))
    with pytest.raises(CovarianceNotEstimable) as e:
        estimate_covariance_flat(o, BACovarianceOptions(), flat, raise_not_estimable=True, priors=empty)
    print(f"no priors: {e.value}")
    assert oracle_cov.estimate(o, flat, oracle_cov.ALL, jac=oracle_cov_prior.jacobian(o, flat, empty))[0] is None
    three = _subset(flat_priors(flat, seed=19, stddev=0.05), THREE)
    compare(o, flat, three, oracle_cov.ALL)
    _collinear(flat, THREE)
    for params in (oracle_cov.ALL, oracle_cov.POSES):
        with pytest.raises(CovarianceNotEstimable) as e:
            estimate_covariance_flat(o, BACovarianceOptions(params), flat, raise_not_estimable=True, priors=three)
        print(f"collinear priors, params {params}: {e.value}")
        assert _pivot(str(e.value)) <= 1e-6
        ref, msg = oracle_cov.estimate(o, flat, params, jac=oracle_cov_prior.jacobian(o, flat, three))
        assert ref is None, "the oracle finds the collinear case estimable"


# ---------------------------------------------------------------- identities
def _all_blocks(cov, flat):
    poses, size = cov.poses_all()
    pts, valid = cov.points_all()
    cams = [cov.camera(c) for c in range(len(flat.cam_model))]
    return [poses, size, pts, valid] + [c for c in cams if c is not None]


def _same_estimate(a, b, label):
    """Two estimates of one problem by the same code path.  S is summed with fp64 atomics, whose order varies from run to
    run, so two plain b200ba_estimate_covariance calls already differ in the last bits (measured on one H100: up to
    3.3e-12 of a block's largest entry).  Held per block at 1e-10 of its largest entry, far below the effect of one prior
    row."""
    worst = 0.0
    for x, y in zip(a, b):
        assert x.shape == y.shape
        if x.dtype.kind != "f":
            assert np.array_equal(x, y)
            continue
        for xb, yb in zip(x.reshape(len(x), -1), y.reshape(len(y), -1)):
            scale = np.abs(yb).max()
            if scale > 0:
                worst = max(worst, np.abs(xb - yb).max() / scale)
    print(f"{label}: largest difference {worst:.3g} of a block's largest entry")
    assert worst <= 1e-10


def test_zero_priors_is_the_plain_estimate():
    """num_priors == 0 takes b200ba_estimate_covariance's code path (the entry drops the priors before anything else)."""
    flat = _scene(SIMPLE_RADIAL, seed=53)
    flat.pose_constant = flat.pose_constant.copy(); flat.pose_fixed_dim = flat.pose_fixed_dim.copy()
    flat.pose_constant[0] = 1
    flat.pose_fixed_dim[1] = int(np.argmax(np.abs(flat.poses[1, 4:] - flat.poses[0, 4:])))
    o = BundleAdjustmentOptions(gpu_index=0)
    empty = FlatPositionPriors(np.zeros(0), np.zeros(0), np.zeros((0, 3)), np.zeros((0, 3, 3)))
    for params in (oracle_cov.ALL, oracle_cov.POSES):
        a1 = _all_blocks(estimate_covariance_flat(o, BACovarianceOptions(params), flat), flat)
        a2 = _all_blocks(estimate_covariance_flat(o, BACovarianceOptions(params), flat), flat)
        b = _all_blocks(estimate_covariance_flat(o, BACovarianceOptions(params), flat, priors=empty), flat)
        _same_estimate(a1, a2, f"params {params}, two plain runs")
        _same_estimate(b, a1, f"params {params}, zero priors against plain")


def test_points_mode_ignores_priors():
    flat = _scene(SIMPLE_RADIAL, seed=59)
    o = BundleAdjustmentOptions(gpu_index=0)
    priors = flat_priors(flat, seed=23, stddev=0.02)
    solve_flat_with_position_priors(o, flat, priors)
    a = estimate_covariance_flat(o, BACovarianceOptions(oracle_cov.POINTS), flat).points_all()
    b = estimate_covariance_flat(o, BACovarianceOptions(oracle_cov.POINTS), flat, priors=priors).points_all()
    assert np.array_equal(a[1], b[1]) and a[1].sum() > 0
    assert np.array_equal(a[0].view(np.uint64), b[0].view(np.uint64))


# ---------------------------------------------------------------- end to end
def _pp_scene(seed, full_cov=True):
    gt, priors = synthesize_rig_reconstruction(1, 1, 7, 100, seed=seed, prior_position=True)
    rec = copy.deepcopy(gt)
    synthesize_noise(rec, priors, seed=seed + 1, point2D_stddev=0.5, point3D_stddev=0.1, rig_from_world_rotation_stddev=0.5,
                     rig_from_world_translation_stddev=0.1, prior_position_stddev=0.05)
    rng = np.random.default_rng(seed)
    if full_cov:
        for pp in priors:
            pp.position_covariance = random_spd(rng, 0.05)
    config = BundleAdjustmentConfig()
    for i in rec.images:
        config.AddImage(i)
    return rec, priors, config


def _prior_options():
    return PosePriorBundleAdjustmentOptions(alignment_ransac_options=RANSACOptions(random_seed=0))


def _oracle_priors(rec, pose_ids, pose_priors, to_frame, fallback_stddev):
    """The priors of the reconstruction's images in the frame `to_frame` maps the metric positions to (a translation)."""
    frame_of = {f: k for k, f in enumerate(pose_ids)}
    pos, covs, idx = [], [], []
    for pp in pose_priors:
        idx.append(frame_of[rec.images[pp.image_id].frame_id])
        pos.append(to_frame(pp.position))
        covs.append(pp.position_covariance if pp.HasPositionCov() else fallback_stddev ** 2 * np.eye(3))
    return FlatPositionPriors(idx, -np.ones(len(idx)), pos, covs)


def _check_against_oracle(ba, rec, pose_priors, to_frame):
    flat, pose_ids, camera_ids, point_ids = ba.flat_problem()
    po = ba.prior_options_
    priors = _oracle_priors(rec, pose_ids, pose_priors, to_frame, po.prior_position_fallback_stddev)
    ref, msg = oracle_cov.estimate(ba.Options(), flat, oracle_cov.ALL, jac=oracle_cov_prior.jacobian(ba.Options(), flat, priors))
    assert ref is not None, msg
    cov = EstimateBACovariance(BACovarianceOptions(), rec, ba)
    frame_of = {f: k for k, f in enumerate(pose_ids)}
    worst = 0.0
    for i, im in rec.images.items():
        k = frame_of[im.frame_id]
        got = cov.GetCamCovFromWorld(i)
        worst = max(worst, np.linalg.norm(got - ref[("pose", k)]) / np.linalg.norm(ref[("pose", k)]))
    for k in range(0, len(point_ids), 9):
        got = cov.GetPointCov(point_ids[k])
        worst = max(worst, np.linalg.norm(got - ref[("point", k)]) / np.linalg.norm(ref[("point", k)]))
    cam = rec.cameras[camera_ids[0]]
    worst = max(worst, np.linalg.norm(cov.GetOtherParamsCov(cam.params) - ref[("camera", 0)]) / np.linalg.norm(ref[("camera", 0)]))
    print(f"worst relative block error {worst:.3g}")
    assert worst <= 1e-9
    return cov, flat, pose_ids


def test_pose_prior_adjuster_before_and_after_solve():
    rec, pose_priors, config = _pp_scene(61)
    ba = CreatePosePriorBundleAdjuster(BundleAdjustmentOptions(gpu_index=0), _prior_options(), config, pose_priors, rec)
    assert ba.use_prior_position_ and ba.Config().FixedGauge() != TWO_CAMS_FROM_WORLD
    # after the constructor the reconstruction is in the normalized frame
    _check_against_oracle(ba, rec, pose_priors, lambda c: ba.normalized_from_metric_ * c)
    assert ba.Solve().IsSolutionUsable()
    # after Solve() it is back in the metric frame: the priors as given
    cov, flat, pose_ids = _check_against_oracle(ba, rec, pose_priors, lambda c: np.asarray(c, np.float64))
    # no parameter is more certain a priori than a posteriori: the projection-centre covariance is at most the prior's
    for pp in pose_priors:
        im = rec.images[pp.image_id]
        _, Jr, _ = oracle_prior.prior_position(im.cam_from_world, None, pp.position)   # d(c - centre) / d tangent
        post = Jr @ cov.GetCamCovFromWorld(pp.image_id) @ Jr.T
        gap = np.linalg.eigvalsh(pp.position_covariance - post)
        assert gap.min() >= -1e-9 * np.abs(pp.position_covariance).max(), (pp.image_id, gap)


def test_pose_prior_adjuster_fallback_is_the_plain_adjuster():
    """Two priors: the adjuster fixes the TWO_CAMS_FROM_WORLD gauge and holds no priors."""
    rec, pose_priors, config = _pp_scene(67, full_cov=False)
    ba = CreatePosePriorBundleAdjuster(BundleAdjustmentOptions(gpu_index=0), _prior_options(), config, pose_priors[:2], rec)
    assert ba.Config().FixedGauge() == TWO_CAMS_FROM_WORLD
    assert ba.Solve().IsSolutionUsable()
    assert len(ba.flat_priors(*ba.flat_problem()[:2], normalized=ba.in_normalized_frame_)) == 0
    plain = CreateDefaultBundleAdjuster(BundleAdjustmentOptions(gpu_index=0), config, rec)
    a = EstimateBACovariance(BACovarianceOptions(), rec, ba)
    b = EstimateBACovariance(BACovarianceOptions(), rec, plain)
    flat = ba.flat_problem()[0]
    _same_estimate(_all_blocks(a.flat_cov, flat), _all_blocks(b.flat_cov, flat), "fallback adjuster against plain")
