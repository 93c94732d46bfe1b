"""Float64 restatement of the per-hypothesis math of COLMAP's PatchMatchCuda, for tests.

Written from the reference (src/colmap/mvs/), independently of oracle/pm_oracle.c and of the CUDA kernels:
  patch_match_cuda.cu       ComposeHomography :271-332, PhotoConsistencyCostComputer::Compute :489-593,
                            ComputeGeomConsistencyCost :601-667, ComputeViewingAngles :241-269,
                            ComputePointAtDepth :198-205, LikelihoodComputer :698-832,
                            backward messages :976-989, forward messages + selection probability :1184-1207,
                            filter decision :1209-1276
  gpu_mat_ref_image.{h,cu}  BilateralWeightComputer gpu_mat_ref_image.h:70-90, FilterKernel gpu_mat_ref_image.cu:39-82
  image.cc                  ComputeRelativePose :97-112, ComposeProjectionMatrix :114-123,
                            ComposeInverseProjectionMatrix :125-135, ComputeProjectionCenter :137-142

It works in the ORIGINAL orientation only, from the problem's own inputs (K, R, T, grey bitmaps, source depth maps):
no rotated pose tables and no frame maps.  The reference evaluates sweeps 1-3 in a rotated frame; every quantity
modelled here is invariant under that rotation (the tap grid -r, -r+s, ..., r maps onto itself, bilateral weights
depend on |offset| only, angles and reprojection distances are Euclidean), so an error in the rotated set-up of the
product shows up as a disagreement with this model.

Accepted simplifications: exact bilinear weights (the reference's texture unit uses 9-bit weights) and no fast-math.
`Variant` switches on deliberately wrong readings of the reference; the tests require each to be rejected.
"""
import math
from dataclasses import dataclass

import numpy as np

K_MIN_VAR = 1e-5          # PhotoConsistencyCostComputer::Compute, :577
K_MAX_COST = 2.0          # :466
K_NO_CHANGE = 0.99999     # ComputeMessage, :808
K_UNIFORM = 0.5           # :807
U32 = 2.0 ** -24          # unit roundoff of fp32


@dataclass
class Variant:
    """Deliberately wrong readings of the reference (all off = the model)."""
    texel_shift: float = 0.0          # sample at p + shift (forgetting the +0.5 of tex2DLayered: 0.5)
    sigma_spatial_plus1: bool = False  # sigma_spatial = radius + 1 instead of radius
    grid_start_plus1: bool = False     # tap grid -r+1, -r+1+s, ... (wrong for step 2)
    behind_camera_border: bool = False  # z <= 0 samples the zero border (the clamp of an older spec)
    swap_change: bool = False          # kChangeProb and kNoChangeProb swapped
    backward_reversed_frame: int = -1  # frame whose backward chain is walked in the forward direction


def _taps(radius, step, variant):
    start = -radius + (1 if variant.grid_start_plus1 else 0)
    offs = np.arange(start, radius + 1, step, dtype=np.float64)
    dy, dx = np.meshgrid(offs, offs, indexing="ij")
    return dy.ravel(), dx.ravel()


class Model:
    """fp64 model of one PatchMatch problem.  `options` is a PatchMatchOptions, `problem` a Problem."""

    def __init__(self, options, problem, variant=None):
        self.v = variant or Variant()
        self.o = options
        ims = problem.images
        ref = ims[problem.ref_image_idx]
        self.srcs = [ims[i] for i in problem.src_image_idxs]
        self.N = len(self.srcs)
        self.H, self.W = ref.bitmap.shape
        self.r, self.s = int(options.window_radius), int(options.window_step)
        sig_s = float(options.sigma_spatial) if options.sigma_spatial > 0 else float(self.r)  # patch_match.cc:436-438
        if self.v.sigma_spatial_plus1:
            sig_s = float(self.r + 1)
        self.spatial_norm = 1.0 / (2.0 * sig_s * sig_s)
        self.color_norm = 1.0 / (2.0 * float(options.sigma_color) ** 2)
        self.tap_dy, self.tap_dx = _taps(self.r, self.s, self.v)
        K = np.asarray(ref.K, np.float64)
        self.fx, self.cx, self.fy, self.cy = K[0, 0], K[0, 2], K[1, 1], K[1, 2]
        R1, T1 = np.asarray(ref.R, np.float64), np.asarray(ref.T, np.float64)
        self.rel = []
        for s in self.srcs:
            # ComputeRelativePose: R = R2 R1^T, T = T2 - R T1; P = K [R | T]; C = -R^T T
            R2, T2 = np.asarray(s.R, np.float64), np.asarray(s.T, np.float64)
            R = R2 @ R1.T
            T = T2 - R @ T1
            Ks = np.asarray(s.K, np.float64)
            P = Ks @ np.hstack([R, T[:, None]])
            P4 = np.vstack([P, [0, 0, 0, 1]])
            self.rel.append(dict(R=R, T=T, K=Ks, P=P, invP=np.linalg.inv(P4)[:3], C=-R.T @ T,
                                 img=np.asarray(s.bitmap, np.float64) / 255.0))
        self.src_depth = None
        if options.geom_consistency and problem.depth_maps is not None:
            self.src_depth = [np.asarray(problem.depth_maps[i], np.float64) for i in problem.src_image_idxs]
        self._filter_ref(np.asarray(ref.bitmap))
        # LikelihoodComputer constants (:700-707, ComputeNCCCostNormFactor :796-802)
        sig = float(options.ncc_sigma)
        self.inv_ncc_sigma_sq = -0.5 / (sig * sig)
        self.ncc_norm = 2.0 / (math.sqrt(2.0 * math.pi) * sig * math.erf(2.0 / (sig * math.sqrt(2.0))))
        self.k_nochange = 1.0 - K_NO_CHANGE if self.v.swap_change else K_NO_CHANGE
        self.k_change = 1.0 - self.k_nochange

    # ---------------------------------------------------------------------------------------------------------
    # reference image: FilterKernel (gpu_mat_ref_image.cu:39-82)
    # ---------------------------------------------------------------------------------------------------------
    def _bilateral(self, dy, dx, c1, c2):
        """BilateralWeightComputer::Compute (gpu_mat_ref_image.h:80-87)."""
        return np.exp(-(dy * dy + dx * dx) * self.spatial_norm - (c1 - c2) ** 2 * self.color_norm)

    def _ref_color(self, img, rows, cols):
        """point-sampled, border -> 0 (texture in cudaAddressModeBorder)."""
        inside = (rows >= 0) & (cols >= 0) & (rows < self.H) & (cols < self.W)
        rr = np.clip(rows, 0, self.H - 1).astype(np.int64)
        cc = np.clip(cols, 0, self.W - 1).astype(np.int64)
        return np.where(inside, img[rr, cc], 0.0)

    def _filter_ref(self, gray):
        g = gray.astype(np.float64) / 255.0
        rows, cols = np.mgrid[0:self.H, 0:self.W].astype(np.float64)
        cs = np.zeros_like(g); cq = np.zeros_like(g); ws = np.zeros_like(g)
        for dy, dx in zip(self.tap_dy, self.tap_dx):
            c = self._ref_color(g, rows + dy, cols + dx)
            w = self._bilateral(dy, dx, g, c)
            cs += w * c; cq += w * c * c; ws += w
        self.ref_sum = cs / ws
        self.ref_sqsum = cq / ws
        self.ref_wsum_taps = ws
        # image.Set(row, col, uint8(255 * centre)) in fp32: the image the NCC reads back
        c32 = (gray.astype(np.float32) / np.float32(255.0)).astype(np.float32)
        self.ref_img = (np.float32(255.0) * c32).astype(np.uint8).astype(np.float64) / 255.0

    # ---------------------------------------------------------------------------------------------------------
    # geometry
    # ---------------------------------------------------------------------------------------------------------
    def ray(self, row, col):
        """K_ref^-1 (col, row, 1) (ComputePointAtDepth :198-205 without the depth)."""
        return np.stack([(col - self.cx) / self.fx, (row - self.cy) / self.fy, np.ones_like(np.asarray(col, float))], -1)

    def homography(self, i, row, col, depth, normal):
        """ComposeHomography (:271-332): H = K_src (R + T n^T / dist) K_ref^-1, dist = depth n . ray.
        Returns H [P,3,3] and the entrywise magnitude bound |K_src| (|R| + c |T| |n|^T / |dist|) |K_ref^-1| with c
        the condition number of dist (for the fp32 error estimate)."""
        e = self.rel[i]
        ray = self.ray(row, col)
        nr = normal * ray
        dist = depth * nr.sum(-1)
        cond = np.abs(nr).sum(-1) / np.maximum(np.abs(nr.sum(-1)), 1e-300)
        Ks = np.array([[e["K"][0, 0], 0, e["K"][0, 2]], [0, e["K"][1, 1], e["K"][1, 2]], [0, 0, 1]])
        Kinv = np.array([[1 / self.fx, 0, -self.cx / self.fx], [0, 1 / self.fy, -self.cy / self.fy], [0, 0, 1]])
        M = e["R"][None] + e["T"][None, :, None] * (normal / dist[:, None])[:, None, :]
        Ma = np.abs(e["R"])[None] + np.abs(e["T"])[None, :, None] * (np.abs(normal) * (cond / np.abs(dist))[:, None])[:, None, :]
        return Ks @ M @ Kinv, np.abs(Ks) @ Ma @ np.abs(Kinv)

    # ---------------------------------------------------------------------------------------------------------
    # NCC: PhotoConsistencyCostComputer::Compute (:489-593)
    # ---------------------------------------------------------------------------------------------------------
    def _sample(self, i, px, py):
        """tex2DLayered at (p + 0.5) with linear filtering and border 0: texel centres at integers."""
        img = self.rel[i]["img"]
        Hs, Ws = img.shape
        px = px + self.v.texel_shift
        py = py + self.v.texel_shift
        ok = np.isfinite(px) & np.isfinite(py)
        px = np.where(ok, np.clip(px, -4.0, Ws + 4.0), -4.0)
        py = np.where(ok, np.clip(py, -4.0, Hs + 4.0), -4.0)
        fx, fy = np.floor(px), np.floor(py)
        wx, wy = px - fx, py - fy
        ix, iy = fx.astype(np.int64), fy.astype(np.int64)
        pad = np.zeros((Hs + 14, Ws + 14))   # zero apron wide enough for the clipped range and the 4x4 block
        pad[6:6 + Hs, 6:6 + Ws] = img
        a = pad[iy + 6, ix + 6]; b = pad[iy + 6, ix + 7]; c = pad[iy + 7, ix + 6]; d = pad[iy + 7, ix + 7]
        val = (a * (1 - wx) + b * wx) * (1 - wy) + (c * (1 - wx) + d * wx) * wy
        # max - min over the 4x4 texels around the cell bounds |dI/dx| + |dI/dy| on a segment of length < 1 texel
        blk = np.stack([pad[iy + 6 + u, ix + 6 + t] for u in (-1, 0, 1, 2) for t in (-1, 0, 1, 2)], 0)
        grad = blk.max(0) - blk.min(0)
        return val, grad

    def ncc(self, i, row, col, depth, normal):
        """Cost 1 - NCC of hypotheses (depth[P], normal[P,3]) at pixels (row[P], col[P]) in source i.
        Returns dict(cost, ref_var, src_var, bound): `bound` is an fp32 error bound of an implementation that follows
        the reference in fp32 (see error_bound)."""
        row = np.asarray(row, np.float64); col = np.asarray(col, np.float64)
        depth = np.asarray(depth, np.float64); normal = np.asarray(normal, np.float64)
        Hm, Ha = self.homography(i, row, col, depth, normal)
        x = col[:, None] + self.tap_dx[None]
        y = row[:, None] + self.tap_dy[None]
        X = Hm[:, 0, 0, None] * x + Hm[:, 0, 1, None] * y + Hm[:, 0, 2, None]
        Y = Hm[:, 1, 0, None] * x + Hm[:, 1, 1, None] * y + Hm[:, 1, 2, None]
        Z = Hm[:, 2, 0, None] * x + Hm[:, 2, 1, None] * y + Hm[:, 2, 2, None]
        with np.errstate(divide="ignore", invalid="ignore"):
            px, py = X / Z, Y / Z       # 1 / z with its sign kept (:526-535)
            if self.v.behind_camera_border:
                px = np.where(Z > 0, px, -1e30); py = np.where(Z > 0, py, -1e30)
        s, grad = self._sample(i, px, py)
        rc = self._ref_color(self.ref_img, y, x)
        cc = self._ref_color(self.ref_img, row, col)[:, None]
        w = self._bilateral(self.tap_dy[None], self.tap_dx[None], cc, rc)
        arg = (self.tap_dy ** 2 + self.tap_dx ** 2)[None] * self.spatial_norm + (cc - rc) ** 2 * self.color_norm
        W = w.sum(1)
        m1 = (w * s).sum(1) / W
        m2 = (w * s * s).sum(1) / W
        m3 = (w * s * rc).sum(1) / W
        rs = self.ref_sum[row.astype(np.int64), col.astype(np.int64)]
        rq = self.ref_sqsum[row.astype(np.int64), col.astype(np.int64)]
        vr = rq - rs * rs
        vs = m2 - m1 * m1
        cov = m3 - rs * m1
        with np.errstate(divide="ignore", invalid="ignore"):
            ncc = cov / np.sqrt(vr * vs)
        low = (vr < K_MIN_VAR) | (vs < K_MIN_VAR)
        cost = np.where(low, K_MAX_COST, np.clip(1.0 - ncc, 0.0, K_MAX_COST))
        # fp32 error of the sample position: |H| magnitudes bound the rounding of X, Y, Z
        ax, ay = np.abs(x), np.abs(y)
        dX = Ha[:, 0, 0, None] * ax + Ha[:, 0, 1, None] * ay + Ha[:, 0, 2, None]
        dY = Ha[:, 1, 0, None] * ax + Ha[:, 1, 1, None] * ay + Ha[:, 1, 2, None]
        dZ = Ha[:, 2, 0, None] * ax + Ha[:, 2, 1, None] * ay + Ha[:, 2, 2, None]
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            dpos = (dX + dY + (np.abs(px) + np.abs(py)) * dZ) / np.abs(Z)
        dpos = np.where(np.isfinite(dpos), dpos, np.inf)
        ds = np.minimum(grad * dpos * 8 * U32, grad)     # colour error from the position error (8 ulp)
        return dict(cost=cost, ncc=ncc, ref_var=vr, src_var=vs, ref_sum=rs, ref_sqsum=rq, m1=m1, m2=m2, m3=m3,
                    wsum=W, low=low, ds=ds, w=w, s=s, rc=rc, z=Z, arg=arg)

    def error_bound(self, d):
        """fp32 error bound of 1 - NCC, from the fp64 magnitudes of one evaluation (d = ncc(...)).

        u = 2^-24, n = ntaps, t = w, w s, w s^2 or w s r per tap (all >= 0), a = the argument of the tap's exp:
          e_w    = (2 |a| + 4) u          relative error of a tap weight (exp of an argument rounded to ~2 ulp)
          dS     = (n / 8 + 3) u sum t + sum t (e_w + 4 u)   each tap sum (8 interleaved partial sums; 4 ulp of the
                                          bilinear sample), W the same with n / 32 + 5
          dm_k   = (dS_k + m_k dW) / W + u m_k
          dvs    = dm2 + 2 m1 dm1 + u (m2 + m1^2);  dvr = (n + 5) u (rq + 2 rs^2) + u (rq + rs^2)  (sequential filter sums)
          dcov   = dm3 + rs dm1 + (n + 5) u rs m1 + u (m3 + rs m1)
          ds     = |grad I| |dp|          colour error of a tap from the fp32 error of its sample position:
                   |dp| <= 8 u (|dX| + |dY| + (|px| + |py|) |dZ|) / |Z|, |dX|.. = |H| (|x|, |y|, 1), |H| from
                   homography() (cancellation in the plane distance included); |grad I| <= max - min of the 4x4 texels
          dpos   = sum_t |d ncc / d s_t| ds_t,  d ncc / d s_t = w_t / W ((r_t - rs) / sqrt(vr vs) - ncc (s_t - m1) / vs)
          dcost <= 2 (dcov / sqrt(vr vs) + |ncc| (dvr / 2 vr + dvs / 2 vs) + dpos + 4 u)      (factor 2: margin)
        """
        w, s, rc = d["w"], d["s"], d["rc"]
        n = w.shape[1]
        ew = (2 * np.abs(d["arg"]) + 8) * U32
        W = d["wsum"]
        dW = (n / 32.0 + 5) * U32 * W + (w * ew).sum(1)
        def dmean(t):
            S = t.sum(1)
            dS = (n / 8.0 + 3) * U32 * S + (t * ew).sum(1)
            return (dS + S / W * dW) / W + U32 * S / W
        dm1, dm2, dm3 = dmean(w * s), dmean(w * s * s), dmean(w * s * rc)
        m1, rs, rq = d["m1"], d["ref_sum"], d["ref_sqsum"]
        e_ref = (n + 5) * U32
        dvs = dm2 + 2 * m1 * dm1 + U32 * (d["m2"] + m1 * m1)
        dvr = e_ref * (rq + 2 * rs * rs) + U32 * (rq + rs * rs)
        dcov = dm3 + rs * dm1 + e_ref * rs * m1 + U32 * (d["m3"] + rs * m1)
        vr, vs = d["ref_var"], d["src_var"]
        with np.errstate(divide="ignore", invalid="ignore"):
            sens = w / W[:, None] * ((rc - rs[:, None]) / np.sqrt(vr * vs)[:, None]
                                     - d["ncc"][:, None] * (s - m1[:, None]) / vs[:, None])
            dpos = (np.abs(sens) * d["ds"]).sum(1)
            b = 2 * (dcov / np.sqrt(vr * vs) + np.abs(d["ncc"]) * (dvr / (2 * vr) + dvs / (2 * vs)) + dpos + 4 * U32)
        return dict(bound=np.where(np.isfinite(b), b, np.inf), dvr=dvr, dvs=dvs)

    # ---------------------------------------------------------------------------------------------------------
    # geometric consistency: ComputeGeomConsistencyCost (:601-667)
    # ---------------------------------------------------------------------------------------------------------
    def geom_cost(self, i, row, col, depth, max_cost):
        """Returns (cost, error-before-clamp, hit) - hit False where the depth texel is 0 (or outside)."""
        e = self.rel[i]
        pt = depth[:, None] * self.ray(row, col)
        P, iP = e["P"], e["invP"]
        f = pt @ P[:, :3].T + P[:, 3]
        sc, sr = f[:, 0] / f[:, 2], f[:, 1] / f[:, 2]
        dm = self.src_depth[i]
        Hs, Ws = dm.shape
        cx, cy = np.floor(sc + 0.5), np.floor(sr + 0.5)    # point sample at (p + 0.5): nearest texel, border 0
        inside = np.isfinite(cx) & np.isfinite(cy) & (cx >= 0) & (cy >= 0) & (cx < Ws) & (cy < Hs)
        sd = np.where(inside, dm[np.clip(cy, 0, Hs - 1).astype(np.int64) * inside,
                                 np.clip(cx, 0, Ws - 1).astype(np.int64) * inside], 0.0)
        hit = sd != 0.0
        b = np.stack([sc * sd, sr * sd, sd], -1) @ iP[:, :3].T + iP[:, 3]
        with np.errstate(divide="ignore", invalid="ignore"):
            bc = (self.fx * b[:, 0] + self.cx * b[:, 2]) / b[:, 2]
            br = (self.fy * b[:, 1] + self.cy * b[:, 2]) / b[:, 2]
            err = np.sqrt((col - bc) ** 2 + (row - br) ** 2)
        err = np.where(hit, err, np.inf)
        return np.minimum(err, max_cost), err, hit, np.stack([sc, sr], -1)

    # ---------------------------------------------------------------------------------------------------------
    # viewing angles (:241-269) and the filter decision (:1209-1276)
    # ---------------------------------------------------------------------------------------------------------
    def viewing_angles(self, i, row, col, depth, normal):
        pt = depth[:, None] * self.ray(row, col)
        SX = self.rel[i]["C"][None] - pt
        sxn = np.linalg.norm(SX, axis=1)
        cos_inc = (SX * normal).sum(1) / sxn
        cos_tri = -(SX * pt).sum(1) / (np.linalg.norm(pt, axis=1) * sxn)
        return cos_tri, cos_inc

    def ncc_prob(self, cost):
        """ComputeNCCProb (:739-741)."""
        return np.exp(np.asarray(cost, np.float64) ** 2 * self.inv_ncc_sigma_sq) * self.ncc_norm

    def filter_terms(self, i, row, col, depth, normal, sel_prob):
        """The three tests of the filter for one source: returns dict of fp64 margins (positive = passes)."""
        o = self.o
        ct, ci = self.viewing_angles(i, row, col, depth, normal)
        tri = math.cos(math.radians(o.filter_min_triangulation_angle)) - ct    # skip if cos_tri > cos_min
        inc = ci                                                                # skip if cos_inc <= 0
        ncc = np.asarray(sel_prob, np.float64) - float(self.ncc_prob(1.0 - o.filter_min_ncc))
        out = dict(tri=tri, inc=inc, ncc=ncc)
        if o.geom_consistency:
            g, err, _, _ = self.geom_cost(i, row, col, depth, o.geom_consistency_max_cost)
            out["geom"] = o.filter_geom_consistency_max_cost - g
            out["geom_err"] = o.filter_geom_consistency_max_cost - err   # the clamp at max_cost is exact: no band
        return out

    # ---------------------------------------------------------------------------------------------------------
    # messages of one sweep: ComputeMessage (:804-826), ComputeSelProb (:724-731), :976-989, :1184-1207
    # ---------------------------------------------------------------------------------------------------------
    def forward_message(self, cost, prev):
        em = self.ncc_prob(cost)
        zn0 = (prev * self.k_change + (1 - prev) * self.k_nochange) * K_UNIFORM
        zn1 = (prev * self.k_nochange + (1 - prev) * self.k_change) * em
        return zn1 / (zn0 + zn1)

    def backward_message(self, cost, prev):
        em = self.ncc_prob(cost)
        zn0 = prev * em * self.k_change + (1 - prev) * K_UNIFORM * self.k_nochange
        zn1 = prev * em * self.k_nochange + (1 - prev) * K_UNIFORM * self.k_change
        return zn1 / (zn0 + zn1)

    def sweep_sel_prob(self, frame, cost_before, cost_after, sel_before, prev_weight):
        """Selection probability after one sweep in `frame` (0-3), all maps [N,H,W] in the original orientation.

        The sweep runs down the rows of the frame rotated `frame` times by the reference's Rotate (cuda_rotate.h:57-75,
        out(row = W-1-x, col = y) = in(row = y, col = x), pinned by test_rotate_convention_matches_reference_gpu_mat_test):
        that is np.rot90(A, frame).  The backward chain (bottom to top) reads the costs before the sweep; the forward
        chain (top to bottom) the costs after it, because a row's cost is final before its forward message."""
        rot = lambda a: np.rot90(np.asarray(a, np.float64), frame, axes=(1, 2))
        cb, ca, sp = rot(cost_before), rot(cost_after), rot(sel_before)
        N, h, w = cb.shape
        beta = np.empty_like(cb)
        b = np.full((N, w), K_UNIFORM)
        rows = range(h) if frame == self.v.backward_reversed_frame else range(h - 1, -1, -1)
        for r in rows:
            b = self.backward_message(cb[:, r], b)
            beta[:, r] = b
        out = np.empty_like(cb)
        cond = np.empty_like(cb)
        a = np.full((N, w), K_UNIFORM)
        for r in range(h):
            a = self.forward_message(ca[:, r], a)
            bt = beta[:, r]
            zn0 = (1 - a) * (1 - bt)
            zn1 = a * bt
            curr = zn1 / (zn0 + zn1)
            out[:, r] = prev_weight * sp[:, r] + (1 - prev_weight) * curr
            # fp32 1 - alpha and 1 - beta carry an absolute error of a few u: relative 1 / (1 - alpha) etc. in curr
            cond[:, r] = (1 - prev_weight) * curr * (1 - curr) * (1 / a + 1 / (1 - a) + 1 / bt + 1 / (1 - bt))
        self.last_msg_cond = np.rot90(cond, -frame, axes=(1, 2))
        return np.rot90(out, -frame, axes=(1, 2))


# -------------------------------------------------------------------------------------------------------------
# checks shared by tests/test_pm_fp64_cpu.py (the oracle) and tests/test_pm_fp64_gpu.py (the kernels)
# -------------------------------------------------------------------------------------------------------------
VAR_BAND = 0.05            # relative band around kMinVar where the 2.0-versus-finite decision may differ
MAX_EXCLUDED = 0.01        # at most this fraction of pairs may fall in that band
# |sel_prob - fp64| <= MSG_ULP u (cond + 1), cond from Model.sweep_sel_prob.  The messages are fp32 recurrences along a
# whole column, and each step evaluates 1 - prev with the same conditioning, so the error grows with the chain: on the
# 64x48 scene the oracle reaches 3400 u (cond + 1); the two wrong message variants exceed 1.2e7 u (cond + 1).
MSG_ULP = 8192


def pixel_grid(H, W):
    rows, cols = np.mgrid[0:H, 0:W]
    return rows.ravel().astype(np.float64), cols.ravel().astype(np.float64)


def check_costs(model, depth, normal, cost, sample=None):
    """cost[i] (N,H,W fp32) must be the NCC of each pixel's hypothesis (depth (H,W), normal (3,H,W)) in source i.
    `sample`: optional (pixel indices, source indices) to compare instead of every pair.  Returns counts."""
    H, W = depth.shape
    rows, cols = pixel_grid(H, W)
    d = depth.ravel().astype(np.float64)
    n = normal.reshape(3, -1).T.astype(np.float64)
    stats = dict(pairs=0, excluded=0, decided=0, behind=0)
    for i in range(model.N):
        idx = np.arange(H * W) if sample is None else sample[0][sample[1] == i]
        if idx.size == 0:
            continue
        for chunk in np.array_split(idx, max(1, idx.size * model.tap_dx.size // 1_000_000)):
            r = model.ncc(i, rows[chunk], cols[chunk], d[chunk], n[chunk])
            b = model.error_bound(r)["bound"]
            got = cost[i].ravel()[chunk].astype(np.float64)
            band = ((np.abs(r["ref_var"] / K_MIN_VAR - 1) < VAR_BAND) | (np.abs(r["src_var"] / K_MIN_VAR - 1) < VAR_BAND))
            two = got == K_MAX_COST
            bad_dec = (two != r["low"]) & ~band
            assert not bad_dec.any(), (
                f"source {i}: 2.0-versus-finite decision differs at {int(bad_dec.sum())} pairs, e.g. pixel "
                f"{int(chunk[bad_dec][0])}: got {got[bad_dec][0]}, fp64 {r['cost'][bad_dec][0]} "
                f"(vars {r['ref_var'][bad_dec][0]:.3g}, {r['src_var'][bad_dec][0]:.3g})")
            cmp = ~band & ~two & ~r["low"]
            diff = np.abs(got - r["cost"])
            out = cmp & ~(diff <= b)
            assert not out.any(), (
                f"source {i}: {int(out.sum())} of {int(cmp.sum())} costs outside their fp32 bound, worst pixel "
                f"{int(chunk[out][np.argmax((diff / b)[out])])}: got {got[out][np.argmax((diff / b)[out])]}, fp64 "
                f"{r['cost'][out][np.argmax((diff / b)[out])]}, bound {b[out][np.argmax((diff / b)[out])]:.3g}")
            stats["pairs"] += chunk.size
            stats["excluded"] += int(band.sum())
            stats["decided"] += int((two & r["low"]).sum())
            stats["behind"] += int((r["z"] <= 0).any(1).sum())
    assert stats["excluded"] <= MAX_EXCLUDED * stats["pairs"], stats
    return stats


def check_messages(model, frame, cost_before, cost_after, sel_before, sel_after, prev_weight):
    """sel_after must be the selection probability of one sweep in `frame` from the three maps."""
    want = model.sweep_sel_prob(frame, cost_before, cost_after, sel_before, prev_weight)
    diff = np.abs(sel_after.astype(np.float64) - want)
    tol = MSG_ULP * U32 * (model.last_msg_cond + 1.0)
    worst = np.unravel_index(np.argmax(diff / tol), diff.shape)
    assert (diff <= tol).all(), (f"frame {frame}: {int((diff > tol).sum())} selection probabilities outside their "
                                 f"bound, worst at {worst}: off by {diff[worst]:.3g}, bound {tol[worst]:.3g}")
    return float((diff / tol).max())


def check_filter(model, depth, normal, sel_prob, mask, bands=None):
    """The consistency mask of the last sweep against the fp64 filter decision (:1209-1276)."""
    bands = bands or dict(tri=1e-5, inc=1e-5, ncc=1e-6, geom_err=1e-3)
    o = model.o
    H, W = depth.shape
    kept = depth.ravel() != 0
    filtered = ~kept
    assert (normal.reshape(3, -1)[:, filtered] == 0).all() and (mask.reshape(model.N, -1)[:, filtered] == 0).all()
    rows, cols = pixel_grid(H, W)
    rows, cols = rows[kept], cols[kept]
    d = depth.ravel()[kept].astype(np.float64)
    n = normal.reshape(3, -1).T[kept].astype(np.float64)
    m = mask.reshape(model.N, -1)[:, kept]
    assert (m.sum(0) >= o.filter_min_num_consistent).all()
    compared = excluded = 0
    for i in range(model.N):
        t = model.filter_terms(i, rows, cols, d, n, sel_prob[i].ravel()[kept])
        near = np.zeros(d.shape, bool)
        for k in ("tri", "inc", "ncc", "geom_err"):
            if k in t:
                near |= np.abs(t[k]) < bands[k] * (1.0 if k != "ncc" else max(1.0, float(model.ncc_prob(0.0))))
        if o.geom_consistency:
            _, _, _, pos = model.geom_cost(i, rows, cols, d, o.geom_consistency_max_cost)
            frac = np.abs((pos + 0.5) - np.round(pos + 0.5))
            near |= (frac < 1e-3).any(1)       # the nearest depth texel is ambiguous
        want = (t["tri"] >= 0) & (t["inc"] > 0) & (t["ncc"] >= 0)
        if o.geom_consistency:
            want &= t["geom"] >= 0
        bad = (want != (m[i] != 0)) & ~near
        assert not bad.any(), f"source {i}: {int(bad.sum())} mask entries differ from the fp64 filter decision"
        compared += int((~near).sum())
        excluded += int(near.sum())
    assert excluded <= MAX_EXCLUDED * (compared + excluded), (excluded, compared)
    return compared, excluded


def forward_source(scene, k, frac=0.5):
    """Move source image k onto the reference's optical axis, `frac` of the way to the scene, looking the same way:
    the hypotheses nearer than that lie behind it, and their taps mirror through its centre into the image."""
    ref = scene["images"][0]
    im = scene["images"][k]
    R = np.asarray(ref.R, np.float64)
    C = -R.T @ np.asarray(ref.T, np.float64)
    C = C + frac * (scene["depth_min"] + scene["depth_max"]) * R[2]
    im.R = R.astype(np.float32)
    im.T = (-R @ C).astype(np.float32)
    return scene
