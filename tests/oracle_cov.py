"""Two independent CPU statements of the bundle-adjustment covariance, on the Jacobian built from the BA oracle's
per-observation reprojection derivatives (ba_oracle_reproj_rig): loss-corrected, unscaled, in the tangent space.
Test infrastructure.

* ``jacobian``: the problem's variable blocks as the oracle's flattening decides them (refine flags, constant flags,
  gauge masks, "used" blocks, observations connected to a variable block), the ambient derivatives of every observation
  from the oracle, the quaternion (x) R^3 tangent map and the ceres Corrector of the robust loss.
* ``estimate``: a restatement of EstimateBACovarianceFromProblem (src/colmap/estimators/covariance.cc) with scipy.sparse
  and dense LAPACK: Schur elimination of the points with damping, elimination of the others (intrinsics, sensor_from_rig)
  with damping in the POSES modes, the LDL^T rank test (|D_i| <= 1e-6: not estimable), L^-1 and blocks of L^-T L^-1.
* ``ceres_semantics``: what ceres::Covariance returns in the reference's covariance test: blocks of (J^T J)^-1 over all
  variable tangent dimensions for poses and others, (J_p^T J_p)^-1 per point with everything else held constant.

Both return dicts {("pose", i) | ("camera", c) | ("sensor", s) | ("point", k): block, ("cross", i, j): block}, with
masked (constant) dimensions omitted."""
import ctypes

import numpy as np
import scipy.linalg
import scipy.sparse

import oracle_ba
from colmap_b200.bundle_adjustment import CAUCHY, HUBER, MODEL_NUM_PARAMS, SOFT_L1, TRIVIAL, _f64p

POSES, POINTS, POSES_AND_POINTS, ALL = 0, 1, 2, 3
_SINGLE_FOCAL = (0, 2, 3, 8, 9, 12, 14)      # models whose parameters start f, cx, cy


def _param_group(model, k):
    """0 focal, 1 principal point, 2 extra, 3 never refined (models.h focal / principal point / extra indices)."""
    if model == 17:         # EQUIRECTANGULAR {width, height}: sensor metadata
        return 3
    if model in _SINGLE_FOCAL:
        return 0 if k == 0 else (1 if k < 3 else 2)
    return 0 if k < 2 else (1 if k < 4 else 2)


def _loss(kind, a, s):
    """ceres SoftLOneLoss / CauchyLoss / HuberLoss: (rho', rho'') at s = |r|^2."""
    b, c = a * a, 1.0 / (a * a)
    if kind == SOFT_L1:
        sm = 1.0 + s * c
        r1 = max(2.2250738585072014e-308, 1.0 / np.sqrt(sm))
        return r1, -(c * r1) / (2.0 * sm)
    if kind == CAUCHY:
        inv = 1.0 / (1.0 + s * c)
        return max(2.2250738585072014e-308, inv), -c * inv * inv
    if kind == HUBER and s > b:
        r1 = max(2.2250738585072014e-308, a / np.sqrt(s))
        return r1, -r1 / (2.0 * s)
    return 1.0, 0.0


def _plus_jacobian(q):
    """PlusJacobian (4 x 3) of EigenQuaternionManifold at delta = 0, q = (x, y, z, w)."""
    x, y, z, w = q
    return np.array([[w, z, -y], [-z, w, x], [y, -x, w], [-x, -y, -z]])


def _normalized(q):
    return q / np.linalg.norm(q)


def jacobian(options, flat):
    """(J as scipy.sparse.csr_matrix, columns) with columns = dict of index arrays per variable block:
    ("pose", i) -> unmasked pose columns [rotation, translation], ("sensor", s), ("camera", c), ("point", k)."""
    o = options
    npose, ncam, npt, nobs = len(flat.poses), len(flat.cam_model), len(flat.points), len(flat.obs_pose)
    cam_sensor = flat.cam_sensor if len(flat.cam_sensor) == ncam else -np.ones(ncam, np.int32)
    pose_used, cam_used, pt_used = np.zeros(npose, bool), np.zeros(ncam, bool), np.zeros(npt, bool)
    pose_used[flat.obs_pose] = True; cam_used[flat.obs_cam] = True; pt_used[flat.obs_point] = True
    columns, nc = {}, 0
    pose_var, pose_dims = np.zeros(npose, bool), {}
    for i in range(npose):
        if not o.refine_rig_from_world or flat.pose_constant[i] or not pose_used[i]:
            continue
        dims = [d for d in range(6) if not (o.constant_rig_from_world_rotation and d < 3)
                and not (flat.pose_fixed_dim[i] >= 0 and d == 3 + flat.pose_fixed_dim[i])]
        pose_var[i] = True
        pose_dims[i] = np.array(dims, np.int64)
        columns[("pose", i)] = nc + pose_dims[i]; nc += 6
    sens_var = np.zeros(len(flat.sensors), bool)
    for s in range(len(flat.sensors)):
        used = any(cam_used[c] and cam_sensor[c] == s for c in range(ncam))
        if o.refine_sensor_from_rig and not flat.sensor_constant[s] and used:
            sens_var[s] = True
            columns[("sensor", s)] = nc + np.arange(6); nc += 6
    cam_var = []
    for c in range(ncam):
        m = int(flat.cam_model[c])
        refine = {0: o.refine_focal_length, 1: o.refine_principal_point, 2: o.refine_extra_params, 3: False}
        var = [k for k in range(MODEL_NUM_PARAMS[m]) if refine[_param_group(m, k)]] if (cam_used[c] and not flat.cam_constant[c]) else []
        cam_var.append(var)
        if var:
            columns[("camera", c)] = nc + np.arange(len(var)); nc += len(var)
    pt_var = -np.ones(npt, np.int64)
    nvpt = 0
    for k in range(npt):
        if o.refine_points3D and not flat.point_constant[k] and pt_used[k]:
            pt_var[k] = nvpt; columns[("point", k)] = nc + 3 * nvpt + np.arange(3); nvpt += 1
    poses = flat.poses.copy()
    sensors = flat.sensors.copy()
    for i in np.nonzero(pose_var)[0]:
        poses[i, :4] = _normalized(poses[i, :4])
    for s in np.nonzero(sens_var)[0]:
        sensors[s, :4] = _normalized(sensors[s, :4])
    # ambient derivatives of every effective observation from the oracle (buffers reused across calls)
    L = oracle_ba.lib()
    res, Jpt, Jr, Js = np.zeros(2), np.zeros((2, 3)), np.zeros((2, 7)), np.zeros((2, 7))
    xy = np.zeros(2)
    ptr = lambda a: a.ctypes.data_as(_f64p)
    rows, cols, vals = [], [], []
    nrow = 0
    for j in range(nobs):
        pi, ci, ti = int(flat.obs_pose[j]), int(flat.obs_cam[j]), int(flat.obs_point[j])
        si = int(cam_sensor[ci])
        sv = si >= 0 and sens_var[si]
        if not (pose_var[pi] or cam_var[ci] or pt_var[ti] >= 0 or sv):
            continue
        m = int(flat.cam_model[ci])
        prm = np.ascontiguousarray(flat.cam_params[flat.cam_off[ci]:flat.cam_off[ci] + MODEL_NUM_PARAMS[m]])
        pt, rig = np.ascontiguousarray(flat.points[ti]), np.ascontiguousarray(poses[pi])
        xy[:] = flat.obs_xy[j]
        sen = np.ascontiguousarray(sensors[si]) if si >= 0 else None
        Jp_params = np.zeros((2, len(prm)))
        L.ba_oracle_reproj_rig(m, ptr(pt), ptr(rig), ptr(sen) if sen is not None else None, ptr(prm), ptr(xy), ptr(res),
                               ptr(Jpt), ptr(Jr), ptr(Js), ptr(Jp_params))
        block_cols, block_J = [], []
        if pose_var[pi]:
            block_cols.append(columns[("pose", pi)])
            Jt = np.hstack([Jr[:, :4] @ _plus_jacobian(rig[:4]), Jr[:, 4:]])
            block_J.append(Jt[:, pose_dims[pi]])
        if sv:
            block_cols.append(columns[("sensor", si)])
            block_J.append(np.hstack([Js[:, :4] @ _plus_jacobian(sen[:4]), Js[:, 4:]]))
        if cam_var[ci]:
            block_cols.append(columns[("camera", ci)])
            block_J.append(Jp_params[:, cam_var[ci]])
        if pt_var[ti] >= 0:
            block_cols.append(columns[("point", ti)])
            block_J.append(Jpt.copy())
        Jo = np.hstack(block_J)
        co = np.concatenate(block_cols)
        if o.loss_function_type != TRIVIAL:     # ceres Corrector
            sq = float(res @ res)
            r1, r2 = _loss(o.loss_function_type, o.loss_function_scale, sq)
            sqrt_r1, alpha_sq_norm = np.sqrt(r1), 0.0
            if sq != 0.0 and r2 > 0.0:
                alpha = 1.0 - np.sqrt(1.0 + 2.0 * sq * r2 / r1)
                alpha_sq_norm = alpha / sq
            Jo = sqrt_r1 * (Jo - alpha_sq_norm * np.outer(res, res @ Jo))
        rows.append(np.repeat([nrow, nrow + 1], len(co))); cols.append(np.tile(co, 2)); vals.append(Jo.reshape(-1))
        nrow += 2
    J = scipy.sparse.csr_matrix((np.concatenate(vals) if vals else np.zeros(0),
                                 (np.concatenate(rows) if rows else np.zeros(0, np.int64), np.concatenate(cols) if cols else np.zeros(0, np.int64))),
                                shape=(nrow, nc + 3 * nvpt))
    return J, columns


def _order(columns, kind):
    return [key for key in columns if key[0] == kind]


def point_blocks(J, columns, points, damping):
    """(H_pp + damping I)^-1 per point (H_pp is block diagonal: 3 x 3 per point)."""
    p_cols = np.concatenate([columns[k] for k in points]) if points else np.zeros(0, np.int64)
    Jp = J[:, p_cols].tocsc()
    Hpp = (Jp.T @ Jp).tocoo()
    blocks = np.zeros((len(points), 3, 3))
    blocks[Hpp.row // 3, Hpp.row % 3, Hpp.col % 3] = Hpp.data
    return Jp, (np.linalg.inv(blocks + damping * np.eye(3)) if points else blocks)


def reduced_matrix(jac, damping=1e-8):
    """(S, npose): the Schur complement of the points (with damping) over [poses | others], npose pose rows first."""
    J, columns = jac
    poses, points = _order(columns, "pose"), _order(columns, "point")
    a_keys = poses + _order(columns, "sensor") + _order(columns, "camera")
    a_cols = np.concatenate([columns[k] for k in a_keys]) if a_keys else np.zeros(0, np.int64)
    Ja = J[:, a_cols].tocsc()
    Jp, Hpp_inv = point_blocks(J, columns, points, damping)
    S = (Ja.T @ Ja).toarray()
    if points:
        Hap = (Ja.T @ Jp).tocsr()
        r = np.arange(3 * len(points)).reshape(-1, 3)
        Hi = scipy.sparse.csr_matrix((Hpp_inv.reshape(-1), (np.repeat(r, 3, axis=1).reshape(-1), np.tile(r, (1, 3)).reshape(-1))),
                                     shape=(r.size, r.size))
        S = S - (Hap @ Hi @ Hap.T).toarray()
    return S, sum(len(columns[k]) for k in poses)


def estimate(options, flat, params=ALL, damping=1e-8, cross=True, jac=None):
    """covariance.cc restated.  Returns (blocks, None) or (None, message) when not estimable.  cross=False: no
    pose-pair blocks; jac: the (J, columns) of jacobian(options, flat), when already formed."""
    J, columns = jac if jac is not None else jacobian(options, flat)
    poses, points = _order(columns, "pose"), _order(columns, "point")
    others = _order(columns, "sensor") + _order(columns, "camera")
    want_points, want_poses, want_others = params != POSES, params != POINTS, params == ALL
    out = {}
    a_keys = poses + others
    if want_points:
        Hpp_inv = point_blocks(J, columns, points, damping)[1]
        for n, key in enumerate(points):
            out[key] = Hpp_inv[n]
    if not want_poses:
        return out, None
    S, npose = reduced_matrix((J, columns), damping)
    starts, at = {}, 0
    for k in a_keys:
        starts[k] = (at, len(columns[k])); at += len(columns[k])
    if not want_others and npose < len(S):      # SchurEliminateOtherParams: an LLT of S_oo + damping I
        S_cc, S_co, S_oo = S[:npose, :npose], S[:npose, npose:], S[npose:, npose:].copy()
        S_oo[np.diag_indices_from(S_oo)] += damping
        try:
            Y = scipy.linalg.solve_triangular(np.linalg.cholesky(S_oo), S_co.T, lower=True)
        except np.linalg.LinAlgError:
            return None, "others not positive definite"
        S = S_cc - Y.T @ Y
    elif not want_others:
        S = S[:npose, :npose]
    n = S.shape[0]
    if n == 0:
        return out, None
    # LDL^T in natural order: D = squared Cholesky diagonal; a failed Cholesky has a pivot <= 0
    try:
        C = np.linalg.cholesky(S)
    except np.linalg.LinAlgError:
        return None, "not positive definite"
    D = np.diag(C) ** 2
    if (np.abs(D) <= 1e-6).any():
        return None, f"rank {int((np.abs(D) > 1e-6).sum())} < {n}"
    L_inv = scipy.linalg.solve_triangular(C, np.eye(n), lower=True)
    block = lambda k1, k2: L_inv[:, starts[k1][0]:starts[k1][0] + starts[k1][1]].T @ L_inv[:, starts[k2][0]:starts[k2][0] + starts[k2][1]]
    for k in poses:
        out[k] = block(k, k)
        for k2 in (poses if cross else []):
            out[("cross", k[1], k2[1])] = block(k, k2)
    if want_others:
        for k in others:
            out[k] = block(k, k)
    return out, None


def ceres_semantics(options, flat, params=ALL):
    """ceres::Covariance as the reference's covariance test uses it (no damping anywhere)."""
    J, columns = jacobian(options, flat)
    poses, points = _order(columns, "pose"), _order(columns, "point")
    others = _order(columns, "sensor") + _order(columns, "camera")
    out = {}
    if params != POINTS and (poses or others):
        keys = poses + others + points
        cols = np.concatenate([columns[k] for k in keys])
        H = (J[:, cols].T @ J[:, cols]).toarray()
        Hinv = np.linalg.inv(H)
        starts, at = {}, 0
        for k in keys:
            starts[k] = slice(at, at + len(columns[k])); at += len(columns[k])
        for k in poses:
            out[k] = Hinv[starts[k], starts[k]]
            for k2 in poses:
                out[("cross", k[1], k2[1])] = Hinv[starts[k], starts[k2]]
        if params == ALL:
            for k in others:
                out[k] = Hinv[starts[k], starts[k]]
    if params != POSES:
        for k in points:
            Jk = J[:, columns[k]]
            out[k] = np.linalg.inv((Jk.T @ Jk).toarray())
    return out
