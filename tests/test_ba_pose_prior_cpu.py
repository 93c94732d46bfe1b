"""Pose-prior bundle adjustment without a GPU: the residual and its Jacobians (CPU oracle against finite differences, the
product's host-compiled device function against the oracle), the covariance weighting and its refusals, the alignment
and normalisation mirror, the prior filter, the gauge choice, and the oracle's own convergence on the reference's
Nominal scene."""
import copy
import ctypes

import numpy as np
import pytest

import oracle_prior
from colmap_b200 import load_library
from colmap_b200.bundle_adjustment import (TWO_CAMS_FROM_WORLD, UNSPECIFIED_GAUGE, BundleAdjustmentConfig,
                                           BundleAdjustmentError, BundleAdjustmentOptions, FlatPositionPriors, PosePrior,
                                           PosePriorBundleAdjustmentOptions, RANSACOptions, Sim3d, _bind_prior, _f64p,
                                           _R_to_quat, _rigid_compose, automatic_alignment_max_error,
                                           CreatePosePriorBundleAdjuster, estimate_sim3_robust, estimate_sim3_umeyama,
                                           filter_pose_priors, normalization_centroid, normalize_reconstruction,
                                           projection_center, solve_flat_with_position_priors, transform_reconstruction)
from colmap_b200.synthetic import _quat_mul, synthesize_noise, synthesize_rig_problem, synthesize_rig_reconstruction
from prior_cases import random_spd, reconstruction_near


def _rand_pose(rng, t=2.0):
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    return np.concatenate([q, rng.normal(0, t, 3)])


def _plus(T, d):
    n = np.linalg.norm(d[:3])
    dq = np.concatenate([np.sin(n) / n * d[:3], [np.cos(n)]]) if n > 0 else np.array([0, 0, 0, 1.0])
    return np.concatenate([_quat_mul(dq[None], T[None, :4])[0], T[4:] + d[3:]])


def _residual(rig, sensor, c):
    T = _rigid_compose(sensor, rig) if sensor is not None else rig
    from colmap_b200.bundle_adjustment import _quat_to_R
    return c + _quat_to_R(T[:4]).T @ T[4:]


def _product(rig, sensor, c):
    lib = _bind_prior(load_library())
    d = lambda a: np.ascontiguousarray(a, np.float64)
    rig, c = d(rig), d(c)
    res, Jr, Js = np.zeros(3), np.zeros((3, 6)), np.zeros((3, 6))
    lib.b200ba_test_prior_position(rig.ctypes.data_as(_f64p), d(sensor).ctypes.data_as(_f64p) if sensor is not None else None,
                                   c.ctypes.data_as(_f64p), res.ctypes.data_as(_f64p), Jr.ctypes.data_as(_f64p),
                                   Js.ctypes.data_as(_f64p))
    return res, Jr, Js


@pytest.mark.parametrize("rig_sensor", [False, True])
def test_residual_and_jacobians(rig_sensor):
    """Oracle (complex step through the ambient parameters and the PlusJacobian) against central differences through the
    manifold's Plus; the product's host-compiled device function against the oracle.  Random poses, sensors, positions."""
    rng = np.random.default_rng(3 + rig_sensor)
    for _ in range(25):
        rig, c = _rand_pose(rng), rng.normal(0, 3, 3)
        sensor = _rand_pose(rng, 0.3) if rig_sensor else None
        r, Jr, Js = oracle_prior.prior_position(rig, sensor, c)
        assert np.allclose(r, _residual(rig, sensor, c), atol=1e-12)
        h = 1e-6
        for blk, J in ((0, Jr), (1, Js)):
            Jn = np.zeros((3, 6))
            for j in range(6):
                d = np.zeros(6); d[j] = h
                f = (lambda dd: _residual(_plus(rig, dd), sensor, c)) if blk == 0 else \
                    (lambda dd: _residual(rig, _plus(sensor, dd), c) if sensor is not None else np.zeros(3))
                Jn[:, j] = (f(d) - f(-d)) / (2 * h)
            assert np.abs(Jn - J).max() <= 1e-7 * max(1.0, np.abs(J).max())
        rp, Jrp, Jsp = _product(rig, sensor, c)
        assert np.allclose(rp, r, rtol=0, atol=1e-12)
        assert np.allclose(Jrp, Jr, rtol=0, atol=1e-11 * max(1.0, np.abs(Jr).max()))
        assert np.allclose(Jsp, Js, rtol=0, atol=1e-11 * max(1.0, np.abs(Js).max()))
        if sensor is None:
            assert not Jsp.any()


def test_constant_rotation_columns():
    """constant_rig_from_world_rotation masks the rotation columns in the solve; the translation columns are R^T."""
    rng = np.random.default_rng(9)
    rig = _rand_pose(rng)
    _, Jr, _ = _product(rig, None, np.zeros(3))
    from colmap_b200.bundle_adjustment import _quat_to_R
    assert np.allclose(Jr[:, 3:], _quat_to_R(rig[:4]).T, atol=1e-14)


def test_covariance_weight_matches_numpy():
    lib = _bind_prior(load_library())
    rng = np.random.default_rng(1)
    for k in range(40):
        C = random_spd(rng, 10.0 ** rng.uniform(-3, 2))
        W = np.zeros((3, 3))
        assert lib.b200ba_test_prior_weight(np.ascontiguousarray(C).ctypes.data_as(_f64p), W.ctypes.data_as(_f64p)) == 0
        ref = np.linalg.cholesky(np.linalg.inv(C)).T
        assert np.allclose(W, ref, rtol=1e-10, atol=1e-12 * np.abs(ref).max())
        assert np.allclose(W.T @ W, np.linalg.inv(C), rtol=1e-9, atol=1e-12 * np.abs(np.linalg.inv(C)).max())
    for bad in (np.diag([1.0, -1.0, 1.0]), np.array([[1.0, 2.0, 0], [2.0, 1.0, 0], [0, 0, 1.0]]), np.zeros((3, 3)),
                np.full((3, 3), np.nan), np.array([[1.0, 0.5, 0], [0.0, 1.0, 0], [0, 0, 1.0]])):
        W = np.zeros((3, 3))
        assert lib.b200ba_test_prior_weight(np.ascontiguousarray(bad).ctypes.data_as(_f64p), W.ctypes.data_as(_f64p)) < 0


def _small_flat():
    gt, noisy = synthesize_rig_problem(4, 2, 60, 4, seed=3)
    return noisy


@pytest.mark.parametrize("what,msg", [
    ("pose", "pose_idx out of range"), ("sensor", "sensor_idx out of range"), ("nan_position", "position is not finite"),
    ("nan_cov", "covariance is not finite"), ("not_spd", "not symmetric positive definite"),
    ("asymmetric", "not symmetric positive definite")])
def test_bad_priors_are_refused(what, msg):
    """Refused on the host before any device work: an error, not a crash (this runs without a GPU)."""
    flat = _small_flat()
    pose, sens, pos, cov = [0, 1], [-1, 0], np.zeros((2, 3)), np.stack([np.eye(3)] * 2)
    if what == "pose":
        pose[1] = len(flat.poses)
    elif what == "sensor":
        sens[1] = len(flat.sensors)
    elif what == "nan_position":
        pos[1, 2] = np.nan
    elif what == "nan_cov":
        cov[1, 0, 0] = np.inf
    elif what == "not_spd":
        cov[1] = np.diag([1.0, 1.0, -1e-3])
    else:
        cov[1, 0, 1] = 0.5
    with pytest.raises(BundleAdjustmentError, match=msg):
        solve_flat_with_position_priors(BundleAdjustmentOptions(), flat, FlatPositionPriors(pose, sens, pos, cov))


# ---------------------------------------------------------------- the alignment and normalisation mirror
def test_umeyama_recovers_a_known_sim3():
    rng = np.random.default_rng(0)
    R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    R *= np.sign(np.linalg.det(R))
    T = Sim3d(1.7, _R_to_quat(R), np.array([1.0, -2.0, 0.5]))
    src = rng.normal(size=(20, 3))
    E = estimate_sim3_umeyama(src, T * src)
    assert abs(E.scale - T.scale) < 1e-12
    assert np.allclose(E.R(), T.R(), atol=1e-12) and np.allclose(E.translation, T.translation, atol=1e-12)


def test_robust_fit_with_outliers():
    rng = np.random.default_rng(1)
    R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    R *= np.sign(np.linalg.det(R))
    T = Sim3d(0.8, _R_to_quat(R), np.array([3.0, 0.0, -1.0]))
    src = rng.normal(0, 5, size=(50, 3))
    tgt = T * src + rng.normal(0, 0.01, (50, 3))
    out = rng.choice(50, 15, replace=False)      # 30 % outliers
    tgt[out] += rng.normal(0, 20, (15, 3))
    E, mask = estimate_sim3_robust(src, tgt, RANSACOptions(max_error=0.05, random_seed=0))
    assert E is not None
    assert not mask[out].any() and mask.sum() == 35
    assert abs(E.scale - T.scale) < 1e-3 and np.allclose(E.R(), T.R(), atol=1e-3)
    assert np.allclose(E.translation, T.translation, atol=2e-2)
    E2, mask2 = estimate_sim3_robust(src, tgt, RANSACOptions(max_error=0.05, random_seed=0))
    assert np.array_equal(mask, mask2) and E2.scale == E.scale   # seeded: reproducible


def test_automatic_max_error():
    assert automatic_alignment_max_error([0.04, 0.01, 0.09], 1.0) == pytest.approx(np.sqrt(7.814727903251179 * 0.04))
    assert automatic_alignment_max_error([0.04, 0.01], 1.0) == pytest.approx(np.sqrt(7.814727903251179 * 0.025))
    assert automatic_alignment_max_error([], 2.0) == pytest.approx(np.sqrt(7.814727903251179 * 4.0))


def test_normalize_fixed_scale_matches_percentiles():
    rec = synthesize_rig_reconstruction(1, 1, 11, 20, seed=4)
    centers = np.array([projection_center(rec, i) for i in sorted(rec.images)])
    n = len(centers)
    lo, hi = int(np.floor(0.1 * (n - 1))), int(np.ceil(0.9 * (n - 1)))
    want = np.array([np.sort(centers[:, a])[lo:hi + 1].mean() for a in range(3)])
    assert np.allclose(normalization_centroid(centers), want, atol=1e-15)
    T = normalize_reconstruction(rec, fixed_scale=True)
    assert T.scale == 1.0 and np.allclose(T.translation, -want)
    after = np.array([projection_center(rec, i) for i in sorted(rec.images)])
    assert np.allclose(after, centers - want, atol=1e-12)


@pytest.mark.parametrize("cams_per_rig", [1, 3])
def test_transform_round_trip_with_rigs(cams_per_rig):
    rng = np.random.default_rng(2)
    rec = synthesize_rig_reconstruction(2, cams_per_rig, 3, 15, seed=5)
    ref = copy.deepcopy(rec)
    R = np.linalg.qr(rng.normal(size=(3, 3)))[0]; R *= np.sign(np.linalg.det(R))
    T = Sim3d(2.5, _R_to_quat(R), rng.normal(0, 3, 3))
    c0 = {i: projection_center(rec, i) for i in rec.images}
    transform_reconstruction(rec, T)
    for i in rec.images:   # every camera centre (rig sensors included) moves with the similarity
        assert np.allclose(projection_center(rec, i), T * c0[i], atol=1e-9)
    for r in rec.rigs.values():
        for c, S in r.sensors.items():
            assert np.allclose(S[4:], 2.5 * ref.rigs[r.rig_id].sensors[c][4:])
    transform_reconstruction(rec, T.inverse())
    for f in rec.frames:
        a, b = rec.frames[f].rig_from_world, ref.frames[f].rig_from_world
        assert np.allclose(a[4:], b[4:], atol=1e-9) and abs(abs(a[:4] @ b[:4]) - 1) < 1e-12
    for p in rec.points3D:
        assert np.allclose(rec.points3D[p].xyz, ref.points3D[p].xyz, atol=1e-12)
    for r in rec.rigs.values():
        for c, S in r.sensors.items():
            assert np.allclose(S[4:], ref.rigs[r.rig_id].sensors[c][4:], atol=1e-15)


def test_filter_rules():
    rec, priors = synthesize_rig_reconstruction(1, 1, 6, 20, seed=1, prior_position=True)
    config = BundleAdjustmentConfig()
    for i in sorted(rec.images)[:-1]:
        config.AddImage(i)
    priors[0].position = np.full(3, np.nan)            # no position
    priors[1].sensor_type = "IMU"                       # not a camera
    kept = filter_pose_priors(priors, config)
    assert [p.image_id for p in kept] == [3, 4, 5]      # image 6 is not in the config
    # a non-parameterized image (no observation in the problem) and an image whose blocks are all constant get no residual
    for im in rec.images.values():
        if im.image_id == 3:
            for p2 in im.points2D:
                p2.point3D_id = -1
    config.SetConstantRigFromWorldPose(rec.images[4].frame_id)
    ba = CreatePosePriorBundleAdjuster(BundleAdjustmentOptions(), PosePriorBundleAdjustmentOptions(), config,
                                       [PosePrior(i, projection_center(rec, i), 0.01 * np.eye(3)) for i in range(1, 7)], rec)
    flat, pose_ids, _, _ = ba.flat_problem()
    fp = ba.flat_priors(flat, pose_ids)
    kept_frames = sorted(pose_ids[k] for k in fp.pose_idx)
    assert kept_frames == [rec.images[i].frame_id for i in (1, 2, 4, 5)]   # 3: not parameterized; 6: not in the config
    assert flat.pose_constant[pose_ids.index(rec.images[4].frame_id)] == 1   # its prior reaches the library, which skips it


def test_insufficient_priors_use_two_camera_gauge():
    """Host half of the reference's InsufficientPriorsUseTwoCameraGauge: fewer than three priors -> TWO_CAMS_FROM_WORLD."""
    rec, priors = synthesize_rig_reconstruction(1, 1, 3, 50, seed=2, prior_position=True)
    config = BundleAdjustmentConfig()
    for i in rec.images:
        config.AddImage(i)
    assert config.FixedGauge() == UNSPECIFIED_GAUGE
    ba = CreatePosePriorBundleAdjuster(BundleAdjustmentOptions(), PosePriorBundleAdjustmentOptions(), config, priors[:2], rec)
    assert ba.Config().FixedGauge() == TWO_CAMS_FROM_WORLD and not ba.use_prior_position_
    config2 = BundleAdjustmentConfig()
    for i in rec.images:
        config2.AddImage(i)
    ba2 = CreatePosePriorBundleAdjuster(BundleAdjustmentOptions(), PosePriorBundleAdjustmentOptions(
        alignment_ransac_options=RANSACOptions(random_seed=0)), config2, priors, rec)
    assert ba2.Config().FixedGauge() == UNSPECIFIED_GAUGE and ba2.use_prior_position_


def test_options_check():
    assert PosePriorBundleAdjustmentOptions().Check()
    assert not PosePriorBundleAdjustmentOptions(prior_position_fallback_stddev=0.0).Check()
    assert not PosePriorBundleAdjustmentOptions(prior_position_loss_scale=0.0).Check()


def test_oracle_converges_on_the_nominal_scene():
    """The CPU oracle alone on the reference's Nominal scene (1 rig, 1 camera, 7 frames, 100 points; noise 0.5 px,
    0.1 points, 0.5 deg / 0.1 poses, 0.05 priors): within 0.1 deg and 0.1 of the ground truth."""
    gt, priors = synthesize_rig_reconstruction(1, 1, 7, 100, seed=11, prior_position=True)
    rec = copy.deepcopy(gt)
    synthesize_noise(rec, priors, point2D_stddev=0.5, point3D_stddev=0.1, rig_from_world_rotation_stddev=0.5,
                     rig_from_world_translation_stddev=0.1, prior_position_stddev=0.05, seed=12)
    config = BundleAdjustmentConfig()
    for i in rec.images:
        config.AddImage(i)
    ba = CreatePosePriorBundleAdjuster(BundleAdjustmentOptions(), PosePriorBundleAdjustmentOptions(
        alignment_ransac_options=RANSACOptions(random_seed=0)), config, priors, rec)
    ba._solve_flat = lambda flat, pose_ids: oracle_prior.solve(ba.Options(), flat, ba.flat_priors(flat, pose_ids))
    s = ba.Solve()
    assert s.IsSolutionUsable() and s.num_residuals == 2 * 700 + 3 * 7
    ok, msg = reconstruction_near(gt, rec, 0.1, 0.1)
    assert ok, msg
