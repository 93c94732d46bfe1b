"""fp64 CPU oracle of the global positioner's LM solve (b200gp_solve): the same trust-region rules on the full,
un-eliminated normal equations, assembled with scipy.sparse and solved directly (SuperLU).

Independent of the product's formulas: the residual is written once, r = d - s (X - c + t), and every Jacobian is taken
from it by complex step (the residual is polynomial in the parameters, so the complex step is exact to rounding).
Rules shared with the product and with oracle/ba_oracle.c: Huber corrector (rho'' <= 0, so residual and Jacobian scale by
sqrt(rho')), times the loss weight; Jacobi scaling 1 / (1 + ||J_col||) from the first Jacobian; LM diagonal
clamp(diag(J^T J), 1e-6, 1e32) / radius; rho = (cost - new cost) / model change; radius / max(1/3, 1 - (2 rho - 1)^3)
on success and / 2, 4, 8, ... on failure; parameter and function tolerances checked on every valid step; the projected
gradient under the scale bound; candidates clamped to the bound while the model change uses the unclamped step."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

LB = 1e-5


class Result:
    pass


def _residual(flat, c, X, q, s, sen):
    f, p = flat.obs_frame, flat.obs_point
    t = np.zeros((len(f), 3), dtype=c.dtype)
    if flat.obs_rig_offset is not None:
        t = t + flat.obs_rig_offset
    m = sen >= 0
    if m.any():
        t[m] = -np.einsum("nij,nj->ni", flat.world_from_rig[f[m]], q[sen[m]])
    return flat.obs_ray - s[:, None] * (X[p] - c[f] + t)


def solve(flat, max_num_iterations=100, optimize_positions=True, optimize_points=True, optimize_scales=True,
          loss_function_scale=0.1, function_tolerance=1e-5, gradient_tolerance=1e-10, parameter_tolerance=1e-8,
          initial_radius=1e4, max_radius=1e16, min_radius=1e-32, min_relative_decrease=1e-3, min_diag=1e-6, max_diag=1e32):
    """Solves `flat` (a FlatGlobalPositioning) in place; returns a Result with the cost history and counters."""
    a = loss_function_scale
    F, P, N, S = len(flat.frame_centers), len(flat.points), len(flat.obs_frame), len(flat.cams_in_rig)
    sen = flat.obs_sensor if flat.obs_sensor is not None else -np.ones(N, np.int32)
    w = flat.obs_loss_weight if flat.obs_loss_weight is not None else np.ones(N)
    fconst = flat.frame_constant if flat.frame_constant is not None else np.zeros(F, np.uint8)
    fused = np.zeros(F, bool); fused[flat.obs_frame] = True
    pused = np.zeros(P, bool); pused[flat.obs_point] = True
    sused = np.zeros(S, bool); sused[sen[sen >= 0]] = True
    fvar = fused & optimize_positions & (fconst == 0)
    pvar = pused & optimize_points
    svar = np.full(N, bool(optimize_scales)); svar[:1] = False
    # column layout: frames | sensors | points | scales (variable blocks only)
    fcol = -np.ones(F, np.int64); fcol[fvar] = 3 * np.arange(fvar.sum())
    o = 3 * int(fvar.sum())
    qcol = -np.ones(S, np.int64); qcol[sused] = o + 3 * np.arange(sused.sum())
    o += 3 * int(sused.sum())
    pcol = -np.ones(P, np.int64); pcol[pvar] = o + 3 * np.arange(pvar.sum())
    o += 3 * int(pvar.sum())
    scol = -np.ones(N, np.int64); scol[svar] = o + np.arange(svar.sum())
    ncol = o + int(svar.sum())

    c, X, q, s = flat.frame_centers.copy(), flat.points.copy(), flat.cams_in_rig.copy(), flat.obs_scale.copy()

    def evaluate(c, X, q, s):
        r = _residual(flat, c, X, q, s, sen)
        s2 = np.sum(r * r, axis=1)
        out = s2 > a * a
        rr = np.sqrt(s2)
        rho0 = np.where(out, 2 * a * rr - a * a, s2)
        rho1 = np.where(out, np.maximum(np.finfo(float).tiny, a / np.where(out, rr, 1.0)), 1.0)
        return r, 0.5 * w * rho0, np.sqrt(w * rho1)

    def jacobian(c, X, q, s, sw):
        h = 1e-30
        rows, cols, vals = [], [], []
        base = np.arange(N) * 3
        blocks = [(c, fcol[flat.obs_frame], flat.obs_frame, 3), (X, pcol[flat.obs_point], flat.obs_point, 3)]
        for which, (_, colidx, _, dim) in enumerate(blocks):
            for k in range(dim):
                r = _residual_perturbed(flat, c.astype(complex), X.astype(complex), q.astype(complex), s.astype(complex), sen, which, k, h)
                d = (r.imag / h) * sw[:, None]
                m = colidx >= 0
                for mm in range(3):
                    rows.append(base[m] + mm); cols.append(colidx[m] + k); vals.append(d[m, mm])
        m = sen >= 0
        if m.any():
            qc = qcol[np.where(m, sen, 0)]
            for k in range(3):
                r = _residual_perturbed(flat, c.astype(complex), X.astype(complex), q.astype(complex), s.astype(complex), sen, 2, k, h)
                d = (r.imag / h) * sw[:, None]
                mm_ = m & (qc >= 0)
                for mm in range(3):
                    rows.append(base[mm_] + mm); cols.append(qc[mm_] + k); vals.append(d[mm_, mm])
        r = _residual_perturbed(flat, c.astype(complex), X.astype(complex), q.astype(complex), s.astype(complex), sen, 3, 0, h)
        d = (r.imag / h) * sw[:, None]
        for mm in range(3):
            rows.append(base[svar] + mm); cols.append(scol[svar]); vals.append(d[svar, mm])
        rows, cols, vals = np.concatenate(rows), np.concatenate(cols), np.concatenate(vals)
        return sp.csr_matrix((vals, (rows, cols)), shape=(3 * N, ncol))

    def state_vec(c, X, q, s):
        v = np.zeros(ncol)
        for arr, col, msk in ((c, fcol, fvar), (q, qcol, sused), (X, pcol, pvar)):
            for k in range(3):
                v[col[msk] + k] = arr[msk, k]
        v[scol[svar]] = s[svar]
        return v

    def apply(c, X, q, s, dx):
        c2, X2, q2, s2 = c.copy(), X.copy(), q.copy(), s.copy()
        for arr, col, msk in ((c2, fcol, fvar), (q2, qcol, sused), (X2, pcol, pvar)):
            for k in range(3):
                arr[msk, k] += dx[col[msk] + k]
        s2[svar] = np.maximum(s[svar] + dx[scol[svar]], LB)
        return c2, X2, q2, s2

    res = Result()
    r, cst, sw = evaluate(c, X, q, s)
    cost = cst.sum()
    res.initial_cost = cost
    hist = [cost]
    J = jacobian(c, X, q, s, sw)
    rt = (r * sw[:, None]).reshape(-1)
    D = 1.0 / (1.0 + np.sqrt(np.asarray(J.multiply(J).sum(axis=0)).ravel()))
    radius, dec = initial_radius, 2.0
    it, res.num_successful_steps, res.num_unsuccessful_steps = 0, 0, 0
    res.termination_type = 1

    def grad_norm(J, rt, s):
        g = J.T @ rt
        gp = g.copy()
        sc = scol[svar]
        gp[sc] = s[svar] - np.maximum(s[svar] - g[sc], LB)
        return np.max(np.abs(gp)) if len(gp) else 0.0

    gnorm = grad_norm(J, rt, s)
    done = False
    while not done:
        if gnorm <= gradient_tolerance:
            res.termination_type = 0
            break
        x_norm = np.linalg.norm(state_vec(c, X, q, s))
        Js = J @ sp.diags(D)
        JtJ = (Js.T @ Js).tocsc()
        g = Js.T @ rt
        diag = JtJ.diagonal()
        while True:
            if it >= max_num_iterations:
                done = True
                break
            it += 1
            A = JtJ + sp.diags(np.clip(diag, min_diag, max_diag) / radius)
            dx = spla.spsolve(A.tocsc(), -g, permc_spec="MMD_AT_PLUS_A") if ncol else np.zeros(0)
            ok = np.all(np.isfinite(dx))
            y = Js @ dx
            model = -float(y @ (rt + 0.5 * y))
            accepted = False
            if ok and model > 0:
                c2, X2, q2, s2 = apply(c, X, q, s, D * dx)
                _, cst2, _ = evaluate(c2, X2, q2, s2)
                new_cost = cst2.sum()
                rho = (cost - new_cost) / model
                step = np.linalg.norm(state_vec(c2, X2, q2, s2) - state_vec(c, X, q, s))
                if step / (x_norm + parameter_tolerance) <= parameter_tolerance or abs(cost - new_cost) <= function_tolerance * cost:
                    res.termination_type = 0
                    hist.append(cost)
                    done = True
                    break
                if rho > min_relative_decrease:
                    accepted = True
            if accepted:
                res.num_successful_steps += 1
                c, X, q, s = c2, X2, q2, s2
                r, cst, sw = evaluate(c, X, q, s)
                cost = cst.sum()
                J = jacobian(c, X, q, s, sw)
                rt = (r * sw[:, None]).reshape(-1)
                gnorm = grad_norm(J, rt, s)
                t = 2.0 * rho - 1.0
                radius = min(max_radius, radius / max(1.0 / 3.0, 1.0 - t ** 3))
                dec = 2.0
                hist.append(cost)
                break
            res.num_unsuccessful_steps += 1
            radius /= dec
            dec *= 2.0
            hist.append(cost)
            if radius < min_radius:
                res.termination_type = 0
                done = True
                break
    res.final_cost = cost
    res.cost_history = np.asarray(hist)
    flat.frame_centers[fvar] = c[fvar]
    flat.points[pvar] = X[pvar]
    if S:
        flat.cams_in_rig[sused] = q[sused]
    flat.obs_scale[svar] = s[svar]
    return res


def _residual_perturbed(flat, c, X, q, s, sen, which, k, h):
    """The residual with the k-th coordinate of each observation's own block `which` (0 frame, 1 point, 2 sensor,
    3 scale) shifted by i h: per observation, so every row gets the derivative wrt its own block."""
    f, p = flat.obs_frame, flat.obs_point
    N = len(f)
    cf, Xp = c[f].copy(), X[p].copy()
    qs = q[np.where(sen >= 0, sen, 0)].copy() if len(q) else np.zeros((N, 3), complex)
    ss = s.copy()
    if which == 0:
        cf[:, k] += 1j * h
    elif which == 1:
        Xp[:, k] += 1j * h
    elif which == 2:
        qs[:, k] += 1j * h
    else:
        ss = ss + 1j * h
    t = np.zeros((N, 3), complex)
    if flat.obs_rig_offset is not None:
        t = t + flat.obs_rig_offset
    m = sen >= 0
    if m.any():
        t[m] = -np.einsum("nij,nj->ni", flat.world_from_rig[f[m]], qs[m])
    return flat.obs_ray - ss[:, None] * (Xp - cf + t)
