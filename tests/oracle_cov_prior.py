"""The prior rows of a pose-prior bundle adjustment appended to the covariance oracle's Jacobian (tests/oracle_cov.py), for
``oracle_cov.estimate(..., jac=...)``.  Test infrastructure.

Each kept prior adds three rows W (c + R^T t) on its pose's unmasked tangent columns and, for a non-reference sensor, the
sensor's.  The weight W = chol(cov^-1)^T is formed here with scipy, the derivatives come from the complex-step oracle
(oracle_prior.prior_position, in the same [rotation (quaternion Plus), translation] tangent as oracle_cov), and the ceres
Corrector of the priors' loss uses oracle_cov._loss."""
import numpy as np
import scipy.linalg
import scipy.sparse

import oracle_cov
import oracle_prior
from colmap_b200.bundle_adjustment import TRIVIAL


def weight(C):
    """chol(C^-1)^T (upper triangular)."""
    return scipy.linalg.cholesky(np.linalg.inv(np.asarray(C, np.float64)), lower=True).T


def _pose_dims(options, flat, i):
    """oracle_cov.jacobian's rule for the unmasked tangent dimensions of a variable pose."""
    return np.array([d for d in range(6) if not (options.constant_rig_from_world_rotation and d < 3)
                     and not (flat.pose_fixed_dim[i] >= 0 and d == 3 + flat.pose_fixed_dim[i])], np.int64)


def prior_rows(options, flat, priors, columns, ncols):
    """(rows as scipy.sparse.csr_matrix with ncols columns, number of priors kept)."""
    rows, cols, vals, kept = [], [], [], 0
    for k in range(len(priors)):
        i, s = int(priors.pose_idx[k]), int(priors.sensor_idx[k])
        pose_key, sens_key = ("pose", i), ("sensor", s)
        pose_var, sens_var = pose_key in columns, s >= 0 and sens_key in columns
        if not (pose_var or sens_var):
            continue        # every block of the prior is constant: no residual
        rig = np.array(flat.poses[i], np.float64)
        if pose_var:
            rig[:4] /= np.linalg.norm(rig[:4])
        sen = None
        if s >= 0:
            sen = np.array(flat.sensors[s], np.float64)
            if sens_var:
                sen[:4] /= np.linalg.norm(sen[:4])
        res, Jr, Js = oracle_prior.prior_position(rig, sen, priors.position[k])
        W = weight(priors.covariance[k])
        rw = W @ res
        block_cols, block_J = [], []
        if pose_var:
            block_cols.append(columns[pose_key]); block_J.append((W @ Jr)[:, _pose_dims(options, flat, i)])
        if sens_var:
            block_cols.append(columns[sens_key]); block_J.append(W @ Js)
        Jo, co = np.hstack(block_J), np.concatenate(block_cols)
        if priors.loss_function_type != TRIVIAL:     # ceres Corrector
            sq = float(rw @ rw)
            r1, r2 = oracle_cov._loss(priors.loss_function_type, priors.loss_function_scale, sq)
            alpha_sq_norm = 0.0
            if sq != 0.0 and r2 > 0.0:
                alpha_sq_norm = (1.0 - np.sqrt(1.0 + 2.0 * sq * r2 / r1)) / sq
            Jo = np.sqrt(r1) * (Jo - alpha_sq_norm * np.outer(rw, rw @ Jo))
        rows.append(np.repeat(3 * kept + np.arange(3), len(co))); cols.append(np.tile(co, 3)); vals.append(Jo.reshape(-1))
        kept += 1
    J = scipy.sparse.csr_matrix((np.concatenate(vals) if vals else np.zeros(0),
                                 (np.concatenate(rows) if rows else np.zeros(0, np.int64),
                                  np.concatenate(cols) if cols else np.zeros(0, np.int64))), shape=(3 * kept, ncols))
    return J, kept


def jacobian(options, flat, priors):
    """oracle_cov.jacobian(options, flat) with the prior rows appended: (J, columns) for oracle_cov.estimate(jac=...)."""
    J, columns = oracle_cov.jacobian(options, flat)
    P, _ = prior_rows(options, flat, priors, columns, J.shape[1])
    return scipy.sparse.vstack([J, P]).tocsr(), columns
