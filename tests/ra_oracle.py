"""fp64 CPU oracle of rotation averaging (b200ra_solve): RotationAveragingProblem's residuals and UpdateState,
RotationAveragingSolver's L1 and IRLS phases and LeastAbsoluteDeviationSolver's ADMM, restated with numpy and
scipy.sparse on the full, unsplit constraint matrix A (rows: pairs in order, then the gauge; columns: every parameter
component).  The normal matrices are factored with SuperLU; a singular or indefinite matrix is a failed factorisation.

It reads the same flat problem as the C-ABI (colmap_b200.rotation_averaging.FlatRotationAveraging), so agreement with
the GPU also checks the GPU's per-axis split of A^T D A.  Rotations follow geometry/pose.cc and Eigen:
AngleAxisToRotationMatrix with its 1e-12 small-angle branch, RotationMatrixToAngleAxis through Eigen's quaternion, and
AverageQuaternions as the principal eigenvector of the mean of q q^T.  The reference's random jitter of 1-DOF residuals
within 0.01 of +-pi is not restated, as on the GPU."""
import math

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

SUCCESS, FACTORIZATION_FAILED, NAN_STEP, NAN_WEIGHT, UNDERDETERMINED = 0, 1, 2, 3, 4
RHO, ALPHA, ABS_TOL, REL_TOL = 1.0, 1.0, 1e-4, 1e-2


class Result:
    pass


def exp_so3(w):
    """AngleAxisToRotationMatrix of every row of w [n, 3] -> [n, 3, 3]."""
    w = np.asarray(w, np.float64).reshape(-1, 3)
    th = np.linalg.norm(w, axis=1)
    R = np.empty((len(w), 3, 3))
    big = th > 1e-12
    if big.any():
        a = w[big] / th[big, None]
        s, c = np.sin(th[big]), np.cos(th[big])
        K = np.zeros((len(a), 3, 3))
        K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -a[:, 2], a[:, 1], -a[:, 0]
        K[:, 1, 0], K[:, 2, 0], K[:, 2, 1] = a[:, 2], -a[:, 1], a[:, 0]
        R[big] = c[:, None, None] * np.eye(3) + (1 - c)[:, None, None] * a[:, :, None] * a[:, None, :] + s[:, None, None] * K
    sm = ~big
    if sm.any():
        v = w[sm]
        S = np.tile(np.eye(3), (len(v), 1, 1))
        S[:, 1, 0], S[:, 2, 0], S[:, 0, 1] = v[:, 2], -v[:, 1], -v[:, 2]
        S[:, 2, 1], S[:, 0, 2], S[:, 1, 2] = v[:, 0], v[:, 1], -v[:, 0]
        R[sm] = S
    return R


def quat_from_R(R):
    """Eigen's Quaternion(Matrix3d) of every matrix -> [n, 4] as (x, y, z, w)."""
    R = np.asarray(R).reshape(-1, 3, 3)
    q = np.empty((len(R), 4))
    t = R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2]
    pos = t > 0
    if pos.any():
        Rp = R[pos]
        s = np.sqrt(t[pos] + 1.0)
        w = 0.5 * s
        s = 0.5 / s
        q[pos] = np.stack([(Rp[:, 2, 1] - Rp[:, 1, 2]) * s, (Rp[:, 0, 2] - Rp[:, 2, 0]) * s,
                           (Rp[:, 1, 0] - Rp[:, 0, 1]) * s, w], 1)
    for n in np.nonzero(~pos)[0]:
        M = R[n]
        i = 0
        if M[1, 1] > M[0, 0]:
            i = 1
        if M[2, 2] > M[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(M[i, i] - M[j, j] - M[k, k] + 1.0)
        q[n, i] = 0.5 * s
        s = 0.5 / s
        q[n, 3] = (M[k, j] - M[j, k]) * s
        q[n, j] = (M[j, i] + M[i, j]) * s
        q[n, k] = (M[k, i] + M[i, k]) * s
    return q


def log_quat(q):
    q = np.asarray(q).reshape(-1, 4)
    n = np.linalg.norm(q[:, :3], axis=1)
    out = np.zeros((len(q), 3))
    nz = n != 0
    ang = 2 * np.arctan2(n[nz], np.abs(q[nz, 3]))
    f = np.where(q[nz, 3] < 0, -ang, ang) / n[nz]
    out[nz] = f[:, None] * q[nz, :3]
    return out


def log_so3(R):
    """RotationMatrixToAngleAxis of every matrix -> [n, 3]."""
    return log_quat(quat_from_R(R))


def rot_y(a):
    a = np.asarray(a, np.float64).reshape(-1)
    return exp_so3(np.stack([np.zeros_like(a), a, np.zeros_like(a)], 1))


class Problem:
    """The flat problem with its constraint matrix (RotationAveragingProblem after construction)."""

    def __init__(self, flat):
        self.flat = flat
        F, C = len(flat.frame_dof), flat.num_cameras
        self.F, self.C = F, C
        self.dof = np.concatenate([flat.frame_dof.astype(int), np.full(C, 3, int)])
        self.off = flat.param_offsets()
        self.np = int(self.dof.sum())
        P = len(flat.pair_frame1)
        self.P = P
        pd = flat.pair_dof.astype(int)
        self.roff = np.concatenate([[0], np.cumsum(pd)[:-1]]).astype(int) if P else np.zeros(0, int)
        self.gdof = int(self.dof[flat.gauge_frame])
        self.m = int(pd.sum()) + self.gdof
        cam1 = flat.pair_cam1 if flat.pair_cam1 is not None else np.full(P, -1)
        cam2 = flat.pair_cam2 if flat.pair_cam2 is not None else np.full(P, -1)
        self.cam1 = np.where(cam1 >= 0, F + cam1, -1)
        self.cam2 = np.where(cam2 >= 0, F + cam2, -1)
        rows, cols, vals = [], [], []
        for p in range(P):
            r = self.roff[p]
            if pd[p] == 1:
                rows += [r, r]; cols += [self.off[flat.pair_frame1[p]], self.off[flat.pair_frame2[p]]]; vals += [-1.0, 1.0]
                continue
            for b, sgn in ((flat.pair_frame1[p], -1.0), (flat.pair_frame2[p], 1.0), (self.cam1[p], -1.0), (self.cam2[p], 1.0)):
                if b < 0:
                    continue
                if self.dof[b] == 3:
                    for i in range(3):
                        rows.append(r + i); cols.append(self.off[b] + i); vals.append(sgn)
                else:
                    rows.append(r + 1); cols.append(self.off[b]); vals.append(sgn)
        g = flat.gauge_frame
        for i in range(self.gdof):
            rows.append(self.m - self.gdof + i); cols.append(self.off[g] + i); vals.append(1.0)
        self.A = sp.csr_matrix((vals, (rows, cols)), shape=(self.m, self.np))   # duplicates are summed
        rw = flat.pair_reweighting
        self.rw_pair = np.ones(P) if rw is None else rw.astype(np.float64)
        self.rw_row = np.ones(self.m)
        for p in range(P):
            self.rw_row[self.roff[p]:self.roff[p] + pd[p]] = self.rw_pair[p]
        self.reweighted = rw is not None
        self.rot = flat.rotations.astype(np.float64).copy()
        self.res = np.zeros(self.m)

    def frame_R(self, b):
        x = self.rot[self.off[b]:self.off[b] + self.dof[b]]
        return exp_so3(x)[0] if self.dof[b] == 3 else rot_y(x[0])[0]

    def block_Rs(self):
        """The rotation of every block [nb, 3, 3] (a 1-DOF frame: AngleAxisToRotationMatrix((0, angle, 0)))."""
        W = np.zeros((len(self.dof), 3))
        three = self.dof == 3
        idx = self.off[three][:, None] + np.arange(3)[None, :]
        W[three] = self.rot[idx]
        W[~three, 1] = self.rot[self.off[~three]]
        return exp_so3(W)

    def compute_residuals(self):
        fl = self.flat
        if self.P:
            Rb = self.block_Rs()
            f1, f2 = fl.pair_frame1.astype(int), fl.pair_frame2.astype(int)
            R1, R2 = Rb[f1], Rb[f2]
            m1, m2 = self.cam1 >= 0, self.cam2 >= 0
            R1[m1] = Rb[self.cam1[m1]] @ R1[m1]
            R2[m2] = Rb[self.cam2[m2]] @ R2[m2]
            three = fl.pair_dof == 3
            E = np.transpose(R2[three], (0, 2, 1)) @ fl.pair_R[three] @ R1[three]
            idx = self.roff[three][:, None] + np.arange(3)[None, :]
            self.res[idx] = -log_so3(E)
            for p in np.nonzero(~three)[0]:
                self.res[self.roff[p]] = math.remainder(
                    (self.rot[self.off[f2[p]]] - self.rot[self.off[f1[p]]]) - fl.pair_angle[p], 2 * math.pi)
        g = fl.gauge_frame
        if self.gdof == 1:
            self.res[-1] = self.rot[self.off[g]] - fl.gauge_rotation[1]
        else:
            self.res[-3:] = log_so3(exp_so3(fl.gauge_rotation)[0].T @ exp_so3(self.rot[self.off[g]:self.off[g] + 3])[0])[0]

    def update_state(self, step):
        F = self.F
        three = np.nonzero(self.dof[:F] == 3)[0]
        one = np.nonzero(self.dof[:F] == 1)[0]
        self.rot[self.off[one]] -= step[self.off[one]]
        idx = self.off[three][:, None] + np.arange(3)[None, :]
        self.rot[idx] = log_so3(exp_so3(self.rot[idx]) @ exp_so3(-step[idx]))
        fl = self.flat
        for c in range(self.C):
            b = self.F + c
            o = self.off[b]
            Rc, Ru = exp_so3(self.rot[o:o + 3])[0], exp_so3(-step[o:o + 3])[0]
            frames = fl.cam_frames[fl.cam_frame_start[c]:fl.cam_frame_start[c + 1]]
            Q = quat_from_R(np.stack([Rc @ self.frame_R(f) @ Ru @ self.frame_R(f).T for f in frames]))
            Q /= np.linalg.norm(Q, axis=1, keepdims=True)
            M = Q.T @ Q / len(Q)
            _, V = np.linalg.eigh(M)
            q = V[:, -1] / np.linalg.norm(V[:, -1])
            self.rot[o:o + 3] = log_quat(q)[0]

    def average_step(self, step):
        tot = 0.0
        for f in range(self.F):
            o = self.off[f]
            tot += abs(step[o]) if self.dof[f] == 1 else float(np.linalg.norm(step[o:o + 3]))
        return tot / self.F


def _factor(M):
    try:
        lu = spla.splu(sp.csc_matrix(M))
    except RuntimeError:
        return None
    d = lu.U.diagonal()
    if not np.all(np.isfinite(d)) or np.any(d == 0):
        return None
    return lu


def normal_matrix(A, w, ridge):
    M = (A.T @ sp.diags(w) @ A).tocsc()
    if ridge > 0:
        M = M + ridge * sp.identity(A.shape[1], format="csc")
    return M


def admm(A, lu, b, max_iter):
    """LeastAbsoluteDeviationSolver::Solve; returns (x, iterations run)."""
    m, n = A.shape
    z, u = np.zeros(m), np.zeros(m)
    b_norm = np.linalg.norm(b)
    eps_pri0, eps_dual0 = math.sqrt(m) * ABS_TOL, math.sqrt(n) * ABS_TOL
    x = np.zeros(n)
    it = 0
    for i in range(max_iter):
        it = i + 1
        x = lu.solve(A.T @ (b + z - u))
        Ax = A @ x
        Ax_hat = ALPHA * Ax + (1 - ALPHA) * (z + b)
        z_old = z
        a = Ax_hat - b + u
        z = np.minimum(a + 1 / RHO, 0) + np.maximum(a - 1 / RHO, 0)
        u = u + Ax_hat - z - b
        r_norm = np.linalg.norm(Ax - z - b)
        s_norm = np.linalg.norm(-RHO * (A.T @ (z - z_old)))
        eps_pri = eps_pri0 + REL_TOL * max(b_norm, max(np.linalg.norm(Ax), np.linalg.norm(z)))
        eps_dual = eps_dual0 + REL_TOL * np.linalg.norm(RHO * (A.T @ u))
        if r_norm < eps_pri and s_norm < eps_dual:
            break
    return x, it


def solve(options, flat, problem=None):
    """RotationAveragingSolver::Solve on the flat problem; flat.rotations is updated in place on success.  The result
    carries status, num_l1_iterations, num_irls_iterations, admm_iterations and step_history as the GPU summary does."""
    pr = problem or Problem(flat)
    res = Result()
    res.status, res.num_l1_iterations, res.num_irls_iterations = SUCCESS, 0, 0
    res.admm_iterations, res.step_history = [], []
    res.problem = pr
    ridge = options.ridge_regularization
    if options.max_num_l1_iterations > 0:
        if pr.m < pr.np:
            res.status = UNDERDETERMINED
            return res
        Aw = sp.diags(pr.rw_row) @ pr.A
        lu = _factor(normal_matrix(Aw, np.ones(pr.m), ridge))
        if lu is None:
            res.status = FACTORIZATION_FAILED
            return res
        prev_norm = curr_norm = 0.0
        max_admm = 10
        it = 0
        while it < options.max_num_l1_iterations:
            pr.compute_residuals()
            step, k = admm(Aw, lu, pr.rw_row * pr.res, max_admm)
            res.admm_iterations.append(k)
            prev_norm = curr_norm
            if np.isnan(step).any():
                res.status = NAN_STEP
                res.num_l1_iterations = it
                return res
            curr_norm = float(np.linalg.norm(step))
            pr.update_state(step)
            avg = pr.average_step(step)
            res.step_history.append(avg)
            it += 1
            if avg < options.l1_step_convergence_threshold or abs(prev_norm - curr_norm) < 1e-12:
                break
            max_admm = min(max_admm * 2, 100)
        res.num_l1_iterations = it
    if options.max_num_irls_iterations > 0:
        sigma = math.radians(options.irls_loss_parameter_sigma)
        it = 0
        while it < options.max_num_irls_iterations:
            pr.compute_residuals()
            w = np.ones(pr.m)
            if pr.P:
                pd = flat.pair_dof.astype(int)
                r0 = pr.res[pr.roff]
                e2 = np.where(pd == 1, r0 * r0 + (flat.pair_xz_error if flat.pair_xz_error is not None else 0.0), 0.0)
                three = pd == 3
                idx = pr.roff[three][:, None] + np.arange(3)[None, :]
                e2[three] = np.sum(pr.res[idx] ** 2, axis=1)
                with np.errstate(divide="ignore", invalid="ignore"):
                    if options.weight_type == 1:
                        wp = np.power(e2, (0.5 - 2) / 2)
                    else:
                        t = e2 + sigma * sigma
                        wp = sigma * sigma / (t * t)
                if np.isnan(wp).any():
                    res.status = NAN_WEIGHT
                    res.num_irls_iterations = it
                    return res
                w[:pr.m - pr.gdof] = np.repeat(wp, pd)
            w *= pr.rw_row
            lu = _factor(normal_matrix(pr.A, w, ridge))
            if lu is None:
                res.status = FACTORIZATION_FAILED
                res.num_irls_iterations = it
                return res
            step = lu.solve(pr.A.T @ (w * pr.res))
            if np.isnan(step).any():
                res.status = NAN_STEP
                res.num_irls_iterations = it
                return res
            pr.update_state(step)
            avg = pr.average_step(step)
            res.step_history.append(avg)
            it += 1
            if avg < options.irls_step_convergence_threshold:
                break
        res.num_irls_iterations = it
    flat.rotations[:] = pr.rot
    return res


def axis_split(flat, w_pair, ridge):
    """The permutation of the normal matrix the GPU factors: returns (full M, M_xz, M_y, xz column indices of the
    x and z components, y column indices), with w_pair the weight of every pair and gauge weight 1."""
    pr = Problem(flat)
    w = np.ones(pr.m)
    for p in range(pr.P):
        w[pr.roff[p]:pr.roff[p] + flat.pair_dof[p]] = w_pair[p]
    M = normal_matrix(pr.A, w, ridge).toarray()
    xs = [pr.off[b] for b in range(len(pr.dof)) if pr.dof[b] == 3]
    zs = [pr.off[b] + 2 for b in range(len(pr.dof)) if pr.dof[b] == 3]
    ys = [pr.off[b] + (1 if pr.dof[b] == 3 else 0) for b in range(len(pr.dof))]
    return M, np.array(xs, int), np.array(zs, int), np.array(ys, int)
