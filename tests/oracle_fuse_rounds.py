"""CPU model of a deterministic parallel schedule for stereo fusion, the round schedule of DESIGN.md section 6c: pure
Python with numpy float32 scalars, one traversal at a time.  It is the reference for any parallel fusion built on that
schedule; DESIGN.md records why the GPU version measured so far was not shipped.

A traversal is the reference's Fuse(image, row, col) (src/colmap/mvs/fusion.cc:369-560) against a given visited mask;
its claim set is every pixel it marks.  For each seed image (FindNextImage order) the pending seeds are its unmasked
pixels whose depth is not <= 0, ranked by raster index.  Each round admits the lowest-ranked pending seed of every
TILE x TILE tile and runs each admitted seed against the mask of the round start; an admitted seed commits iff no
lower-ranked admitted seed claimed a pixel of its claim set.  Committed seeds mark their claims and emit their point;
the rest stay pending unless their seed pixel is now masked.

The per-pixel arithmetic is that of oracle/ws_oracle.py (same fp32 operations in the same order); medians are
Percentile(., 50) with -0 ordered before +0."""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
from ws_oracle import F, _dot3, _round_half_away  # noqa: E402

TILE = 4


def _views(images):
    """P = K [R | T] (fp32), invP = [R^T K^-1 | -R^T T] (double, rounded once), invR = R^T, K scaled to the map size."""
    V, used = [None] * len(images), [False] * len(images)
    for i, im in enumerate(images):
        if not im["used"]:
            continue
        used[i] = True
        h, w = im["depth"].shape
        sx, sy = F(F(w) / F(im["image_width"])), F(F(h) / F(im["image_height"]))
        K = np.array(im["K"], np.float32).reshape(3, 3).copy()
        K[0, 0] = F(K[0, 0] * sx); K[0, 2] = F(K[0, 2] * sx); K[1, 1] = F(K[1, 1] * sy); K[1, 2] = F(K[1, 2] * sy)
        R = np.asarray(im["R"], np.float32).reshape(3, 3); T = np.asarray(im["T"], np.float32).reshape(3)
        M = np.concatenate([R, T[:, None]], 1)
        P = np.empty((3, 4), np.float32)
        for r in range(3):
            for c in range(4):
                P[r, c] = _dot3(K[r, 0], K[r, 1], K[r, 2], M[0, c], M[1, c], M[2, c])
        k = K.astype(np.float64).reshape(9)
        det = k[0] * (k[4] * k[8] - k[5] * k[7]) - k[1] * (k[3] * k[8] - k[5] * k[6]) + k[2] * (k[3] * k[7] - k[4] * k[6])
        iK = [(k[4] * k[8] - k[5] * k[7]) / det, (k[2] * k[7] - k[1] * k[8]) / det, (k[1] * k[5] - k[2] * k[4]) / det,
              (k[5] * k[6] - k[3] * k[8]) / det, (k[0] * k[8] - k[2] * k[6]) / det, (k[2] * k[3] - k[0] * k[5]) / det,
              (k[3] * k[7] - k[4] * k[6]) / det, (k[1] * k[6] - k[0] * k[7]) / det, (k[0] * k[4] - k[1] * k[3]) / det]
        Rd, Td = R.astype(np.float64), T.astype(np.float64)
        invP = np.empty((3, 4), np.float32)
        for r in range(3):
            for c in range(3):
                invP[r, c] = F((Rd[0, r] * iK[c] + Rd[1, r] * iK[3 + c]) + Rd[2, r] * iK[6 + c])
            invP[r, 3] = F(-((Rd[0, r] * Td[0] + Rd[1, r] * Td[1]) + Rd[2, r] * Td[2]))
        V[i] = dict(P=P, invP=invP, invR=R.T.copy(), sx=sx, sy=sy, w=w, h=h)
    return V, used


def _median(values):
    v = sorted((float(x) for x in values), key=lambda x: (x, math.copysign(1.0, x) > 0))
    idx = 0.5 * (len(v) - 1)
    lo, hi = int(math.floor(idx)), int(math.ceil(idx))
    if lo == hi:
        return v[hi]
    return (hi - idx) * v[lo] + (idx - lo) * v[hi]


class Fusion:
    """Inputs in the dict form of ws_oracle.fuse.  `masks[i]` is the visited mask of image i (bool, h x w)."""

    def __init__(self, opt, images, overlap):
        self.opt, self.images, self.overlap = opt, images, overlap
        self.V, self.used = _views(images)
        self.max_sq = F(opt["max_reproj_error"] * opt["max_reproj_error"])
        self.min_cos = F(math.cos(opt["max_normal_error"] * 0.017453292519943295))
        self.max_derr = F(opt["max_depth_error"])
        self.masks = [None if v is None else (np.zeros((v["h"], v["w"]), bool) if images[i].get("mask") is None
                                               else (np.asarray(images[i]["mask"]) != 0).copy())
                      for i, v in enumerate(self.V)]
        self.fused = [False] * len(images)

    def traverse(self, image0, row0, col0, masks=None):
        """Fuse(image0, row0, col0) against `masks` (default: the current ones), which it does not change.  Returns
        (claims, point): claims in claim order as (image, row, col); point = (xyz, normal, rgb, vis) or None."""
        masks = self.masks if masks is None else masks
        opt, images, V = self.opt, self.images, self.V
        own = set()
        claims = []
        queue = [(image0, row0, col0, 0)]
        ref_p, ref_n = np.zeros(4, np.float32), np.zeros(3, np.float32)
        px, py, pz, nx, ny, nz, cr, cg, cb, vis = [], [], [], [], [], [], [], [], [], set()
        while queue:
            i, row, col, td = queue.pop()
            im, v = images[i], V[i]
            if masks[i][row, col] or (i, row, col) in own:
                continue
            depth = F(im["depth"][row, col])
            if depth <= 0:
                continue
            P = v["P"]
            if td > 0:
                proj = [F(F(F(F(P[r, 0] * ref_p[0]) + F(P[r, 1] * ref_p[1])) + F(P[r, 2] * ref_p[2])) + F(P[r, 3] * ref_p[3])) for r in range(3)]
                if F(abs(F(F(proj[2] - depth) / depth))) > self.max_derr:
                    continue
                cd, rd = F(F(proj[0] / proj[2]) - F(col)), F(F(proj[1] / proj[2]) - F(row))
                if F(F(cd * cd) + F(rd * rd)) > self.max_sq:
                    continue
            nm = im["normal"]
            n0, n1, n2 = F(nm[0, row, col]), F(nm[1, row, col]), F(nm[2, row, col])
            iR = v["invR"]
            normal = [_dot3(iR[r, 0], iR[r, 1], iR[r, 2], n0, n1, n2) for r in range(3)]
            if td > 0 and _dot3(ref_n[0], ref_n[1], ref_n[2], normal[0], normal[1], normal[2]) < self.min_cos:
                continue
            hv = [F(F(col) * depth), F(F(row) * depth), depth, F(1)]
            iP = v["invP"]
            xyz = [F(F(F(F(iP[r, 0] * hv[0]) + F(iP[r, 1] * hv[1])) + F(iP[r, 2] * hv[2])) + F(iP[r, 3] * hv[3])) for r in range(3)]
            xx, yy = int(_round_half_away(float(F(F(col) / v["sx"])))), int(_round_half_away(float(F(F(row) / v["sy"]))))
            H, W = im["rgb"].shape[:2]
            color = tuple(int(c) for c in im["rgb"][yy, xx]) if 0 <= xx < W and 0 <= yy < H else (0, 0, 0)
            own.add((i, row, col))
            claims.append((i, row, col))
            if any(xyz[k] < F(opt["bbox_min"][k]) or xyz[k] > F(opt["bbox_max"][k]) for k in range(3)):
                continue
            px.append(xyz[0]); py.append(xyz[1]); pz.append(xyz[2]); nx.append(normal[0]); ny.append(normal[1]); nz.append(normal[2])
            cr.append(color[0]); cg.append(color[1]); cb.append(color[2]); vis.add(i)
            if td == 0:
                ref_p = np.array([xyz[0], xyz[1], xyz[2], 1], np.float32); ref_n = np.array(normal, np.float32)
            if len(px) >= opt["max_num_pixels"]:
                break
            if td >= opt["max_traversal_depth"] - 1:
                continue
            for nxt in self.overlap[i]:
                if nxt < 0:
                    break
                if not self.used[nxt] or self.fused[nxt]:
                    continue
                Pn = V[nxt]["P"]
                q = [F(F(F(F(Pn[r, 0] * xyz[0]) + F(Pn[r, 1] * xyz[1])) + F(Pn[r, 2] * xyz[2])) + Pn[r, 3]) for r in range(3)]
                fc, fr = float(F(q[0] / q[2])), float(F(q[1] / q[2]))
                if not (math.isfinite(fc) and math.isfinite(fr)):
                    continue
                nc, nr = int(_round_half_away(fc)), int(_round_half_away(fr))
                if nc < 0 or nr < 0 or nc >= V[nxt]["w"] or nr >= V[nxt]["h"]:
                    continue
                queue.append((nxt, nr, nc, td + 1))
        if len(px) < opt["min_num_pixels"] or not px:
            return claims, None
        fn = [F(_median(nx)), F(_median(ny)), F(_median(nz))]
        norm = F(np.sqrt(F(F(F(fn[0] * fn[0]) + F(fn[1] * fn[1])) + F(fn[2] * fn[2]))))
        if norm < np.finfo(np.float32).eps:
            return claims, None
        point = ([F(_median(px)), F(_median(py)), F(_median(pz))], [F(fn[0] / norm), F(fn[1] / norm), F(fn[2] / norm)],
                 [min(255, max(0, int(_round_half_away(float(F(_median(c))))))) for c in (cr, cg, cb)], sorted(vis))
        return claims, point

    def image_order(self):
        n = len(self.images)
        image = 0 if n else -1
        while image >= 0:
            yield image
            self.fused[image] = True
            nxt = next((c for c in self.overlap[image] if c >= 0 and self.used[c] and not self.fused[c]), -1)
            if nxt < 0:
                nxt = next((i for i in range(n) if self.used[i] and not self.fused[i]), -1)
            image = nxt

    def pending(self, image):
        v = self.V[image]
        d = self.images[image]["depth"]
        return [r * v["w"] + c for r in range(v["h"]) for c in range(v["w"])
                if not self.masks[image][r, c] and not F(d[r, c]) <= 0]


def fuse_rounds(opt, images, overlap):
    """Returns (xyz, normal, rgb, visibility, stats); stats holds rounds, traversals, per-image round counts and, per
    round, the committed seeds with their claim sets."""
    f = Fusion(opt, images, overlap)
    out = []
    stats = dict(rounds=0, traversals=0, image_rounds=[], committed=[])
    for image in f.image_order():
        if not f.used[image]:
            continue
        w = f.V[image]["w"]
        pending = f.pending(image)
        points, nrounds = [], 0
        while pending:
            nrounds += 1
            admitted, tiles = [], set()
            for rank in pending:                      # ascending: the first of a tile is its lowest-ranked
                t = (rank // w // TILE, rank % w // TILE)
                if t not in tiles:
                    tiles.add(t)
                    admitted.append(rank)
            stats["traversals"] += len(admitted)
            runs = {rank: f.traverse(image, rank // w, rank % w) for rank in admitted}
            owner = {}
            for rank in admitted:
                for c in runs[rank][0]:
                    owner.setdefault(c, rank)
            committed = [rank for rank in admitted if all(owner[c] == rank for c in runs[rank][0])]
            stats["committed"].append([(rank, runs[rank][0]) for rank in committed])
            for rank in committed:
                claims, point = runs[rank]
                for (i, r, c) in claims:
                    f.masks[i][r, c] = True
                if point is not None:
                    points.append((rank, point))
            pending = [rank for rank in pending if not f.masks[image][rank // w, rank % w]]
        stats["rounds"] += nrounds
        stats["image_rounds"].append(nrounds)
        out += [p for _, p in sorted(points, key=lambda t: t[0])]
    xyz = np.array([p[0] for p in out], np.float32).reshape(-1, 3)
    nrm = np.array([p[1] for p in out], np.float32).reshape(-1, 3)
    rgb = np.array([p[2] for p in out], np.uint8).reshape(-1, 3)
    return xyz, nrm, rgb, [p[3] for p in out], stats
