"""Shared helpers of the pose-prior tests: priors for flat problems, the ReconstructionNear restatement."""
import numpy as np

from colmap_b200.bundle_adjustment import (FlatPositionPriors, TRIVIAL, _quat_to_R, _rigid_compose, estimate_sim3_umeyama,
                                           projection_center)


def random_spd(rng, scale):
    """A full anisotropic covariance: random rotation, eigenvalues scale^2 * [0.3, 3]."""
    A = rng.normal(size=(3, 3))
    Q, _ = np.linalg.qr(A)
    return scale ** 2 * (Q @ np.diag(rng.uniform(0.3, 3.0, 3)) @ Q.T)


def flat_priors(flat, seed, stddev=0.05, cov="full", loss=TRIVIAL, loss_scale=float(np.sqrt(7.814727903251179)), sensors=True):
    """One prior per (pose, sensor) of `flat`: the noisy projection centre of cam_from_world plus Gaussian noise.  cov:
    "full" (random anisotropic), "fallback" (stddev^2 I).  sensors=False: priors on the reference sensor only."""
    rng = np.random.default_rng(seed)
    pose_idx, sensor_idx, pos, covs = [], [], [], []
    sens = [-1] + (list(range(len(flat.sensors))) if sensors else [])
    for i in range(len(flat.poses)):
        for s in sens:
            T = flat.poses[i] if s < 0 else _rigid_compose(flat.sensors[s], flat.poses[i])
            C = random_spd(rng, stddev) if cov == "full" else stddev ** 2 * np.eye(3)
            pose_idx.append(i); sensor_idx.append(s)
            pos.append(-_quat_to_R(T[:4]).T @ T[4:] + rng.multivariate_normal(np.zeros(3), C))
            covs.append(C)
    return FlatPositionPriors(pose_idx, sensor_idx, pos, covs, loss, loss_scale)


def rotation_error_deg(qa, qb):
    R = _quat_to_R(qa) @ _quat_to_R(qb).T
    return float(np.degrees(np.arccos(np.clip((np.trace(R) - 1) / 2, -1.0, 1.0))))


def reconstruction_near(gt, rec, max_rotation_error_deg, max_proj_center_error):
    """ReconstructionNear (scene/reconstruction_matchers.h:87-217) for the images: align `rec` to `gt` by a Sim3 over the
    projection centres, then compare every image's rotation (degrees) and projection centre.  Returns the worst errors and
    a message; asserts nothing."""
    ids = sorted(gt.images)
    src = np.array([projection_center(rec, i) for i in ids]); tgt = np.array([projection_center(gt, i) for i in ids])
    T = estimate_sim3_umeyama(src, tgt)
    worst_rot = worst_c = 0.0
    from colmap_b200.bundle_adjustment import _image_cam_from_world
    for k, i in enumerate(ids):
        a = _image_cam_from_world(rec, i)
        Ra = _quat_to_R(a[:4]) @ T.R().T
        b = _image_cam_from_world(gt, i)
        Rrel = Ra @ _quat_to_R(b[:4]).T
        worst_rot = max(worst_rot, float(np.degrees(np.arccos(np.clip((np.trace(Rrel) - 1) / 2, -1.0, 1.0)))))
        worst_c = max(worst_c, float(np.linalg.norm(T * src[k] - tgt[k])))
    ok = worst_rot <= max_rotation_error_deg and worst_c <= max_proj_center_error
    return ok, f"worst rotation error {worst_rot:.4g} deg, worst projection-centre error {worst_c:.4g}"
