"""Time SIFT feature matching on one GPU: one 8192 x 8192 pair (the scan kernel by CUDA events, the whole call's device
time, and Match end to end with both uploads), an exhaustive block of 50 images x 8192 features (1,225 pairs) through
MatchPairs, and the CPU oracle (tests/sm_oracle.c, a restatement of the rule, not the reference's code) on all host
cores.  Prints the card's name and power limit beside the numbers, and one JSON line at the end.

With --guided it times guided matching instead: one 8192 x 8192 pair per filter (E, F, H) with cross-check, the
exhaustive block under F, and the guided CPU oracle (tests/sm_guided_oracle.c) on one E pair.

  python tools/sm_time.py [--reps 20] [--block 50] [--oracle-pairs 3] [--guided]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

from colmap_b200.feature_matching import (CreateSiftFeatureMatcher, FeatureMatcherImage,  # noqa: E402
                                          FeatureMatchingOptions, SiftMatchingOptions)
from colmap_b200.synthetic import make_sift_view_pair  # noqa: E402

U8_DENSE_TOPS = 1979.0      # H100 SXM data sheet, INT8 dense (700 W)
N = 8192


def block_images(num_images, n, seed=0):
    """Views of one scene: each image holds noisy copies of 70% of its rows drawn from a shared pool."""
    rng = np.random.default_rng(seed)
    pool, own, _ = make_sift_view_pair(4 * n, num_images * n, overlap=0.0, seed=seed)
    images = []
    for k in range(num_images):
        shared = int(0.7 * n)
        rows = np.concatenate([pool[rng.choice(len(pool), shared, replace=False)], own[k * n:k * n + n - shared]])
        noisy = np.clip(rows.astype(np.int16) + rng.integers(-12, 13, rows.shape, dtype=np.int16), 0, 255)
        images.append(FeatureMatcherImage(k, noisy.astype(np.uint8)[rng.permutation(n)]))
    return images


def stats(v):
    return float(np.min(v)), float(np.median(v))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--block", type=int, default=50)
    ap.add_argument("--oracle-pairs", type=int, default=3)
    ap.add_argument("--guided", action="store_true")
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    card = smi.splitlines()[0] if smi else "unknown"
    print("GPU:", card, flush=True)
    out = {"gpu": card}
    if args.guided:
        guided(args, out)
        print(json.dumps(out))
        return

    d1, d2, _ = make_sift_view_pair(N, N, seed=1)
    for cc in (True, False):
        o = FeatureMatchingOptions(gpu_index="0", sift=SiftMatchingOptions(cross_check=cc))
        with CreateSiftFeatureMatcher(o) as m:
            a, b = FeatureMatcherImage(1, d1), FeatureMatcherImage(2, d2)
            for _ in range(3):
                res = m.Match(a, b)
            scan, total = [], []
            for _ in range(args.reps):
                m.Match(a, b)
                s, t = m.LastTiming()
                scan.append(s); total.append(t)
            e2e = []
            for r in range(args.reps):     # new image ids: both images are uploaded again
                a2, b2 = FeatureMatcherImage(100 + 2 * r, d1), FeatureMatcherImage(101 + 2 * r, d2)
                t0 = time.perf_counter()
                m.Match(a2, b2)
                e2e.append((time.perf_counter() - t0) * 1e3)
        ways = 2 if cc else 1
        smin, smed = stats(scan)
        tops = 2.0 * N * N * 128 * ways / (smin * 1e-3) / 1e12
        dots = N * N * ways / (smin * 1e-3)
        floor_ms = 2.0 * N * N * 128 * ways / (U8_DENSE_TOPS * 1e12) * 1e3
        key = "cross_check" if cc else "one_way"
        out[key] = {"matches": int(len(res)), "scan_ms_min": smin, "scan_ms_median": smed,
                    "call_device_ms_median": stats(total)[1], "match_with_upload_ms_median": stats(e2e)[1],
                    "u8_tops": tops, "share_of_u8_dense_peak": tops / U8_DENSE_TOPS, "dots_per_s": dots,
                    "tensor_floor_ms": floor_ms}
        print(f"8192 x 8192, {key}: {len(res)} matches; scan kernel {smin:.3f} ms min / {smed:.3f} ms median "
              f"(CUDA events, {args.reps} reps), whole call on the device {stats(total)[1]:.3f} ms, Match with "
              f"both uploads {stats(e2e)[1]:.3f} ms (host clock, median)", flush=True)
        print(f"  {tops:.1f} u8 TOPS = {100 * tops / U8_DENSE_TOPS:.1f}% of the data sheet's {U8_DENSE_TOPS:.0f} dense; "
              f"{dots / 1e9:.1f} G dots/s through the top-2 epilogue; the product alone at the data-sheet rate would "
              f"take {floor_ms * 1e3:.1f} us, so the kernel is {'epilogue' if smin > 3 * floor_ms else 'tensor'}-bound",
              flush=True)

    images = block_images(args.block, N, seed=2)
    pairs = [(i, j) for i in range(len(images)) for j in range(i + 1, len(images))]
    with CreateSiftFeatureMatcher(FeatureMatchingOptions(gpu_index="0")) as m:
        t0 = time.perf_counter()
        res = m.MatchPairs(images, pairs)     # includes the uploads
        first = time.perf_counter() - t0
        wall = []
        for _ in range(3):
            t0 = time.perf_counter()
            res = m.MatchPairs(images, pairs)
            wall.append(time.perf_counter() - t0)
            s, t = m.LastTiming()
    nm = sum(len(r) for r in res)
    out["block"] = {"images": args.block, "pairs": len(pairs), "matches": int(nm), "first_call_s": first,
                    "call_s_min": min(wall), "pairs_per_s": len(pairs) / min(wall), "scan_ms": s, "device_ms": t}
    print(f"exhaustive block {args.block} x {N}: {len(pairs)} pairs, {nm} matches; {len(pairs) / min(wall):.0f} pairs/s "
          f"({min(wall) * 1e3:.1f} ms per MatchPairs call, host clock; scan kernels {s:.1f} ms, device work {t:.1f} ms); "
          f"first call with the uploads {first * 1e3:.1f} ms", flush=True)

    if args.oracle_pairs:
        import oracle_sm
        oracle_sm.match(d1[:64], d2[:64])
        t0 = time.perf_counter()
        for k in range(args.oracle_pairs):
            ref = oracle_sm.match(images[k].descriptors, images[k + 1].descriptors)
        per = (time.perf_counter() - t0) / args.oracle_pairs
        ok = bool(np.array_equal(ref, res[pairs.index((args.oracle_pairs - 1, args.oracle_pairs))]))
        out["cpu_restatement"] = {"cores": os.cpu_count(), "s_per_pair": per, "equal_to_gpu": ok}
        print(f"CPU restatement of the rule (tests/sm_oracle.c, OpenMP, {os.cpu_count()} cores): {per:.2f} s per "
              f"8192 x 8192 pair with cross-check; GPU matches identical: {ok}", flush=True)
    print(json.dumps(out))


def guided(args, out):
    from colmap_b200.feature_matching import TwoViewGeometry
    from colmap_b200.synthetic import make_guided_view_pair
    s = make_guided_view_pair(N, N, model_id=0, plane=True, seed=1)
    a = FeatureMatcherImage(1, s["desc1"], s["camera1"], s["xy1"])
    b = FeatureMatcherImage(2, s["desc2"], s["camera2"], s["xy2"])
    configs = {"E": TwoViewGeometry.CALIBRATED, "F": TwoViewGeometry.UNCALIBRATED, "H": TwoViewGeometry.PLANAR}
    with CreateSiftFeatureMatcher(FeatureMatchingOptions(gpu_index="0")) as m:
        for kind, config in configs.items():
            g = TwoViewGeometry(config=config)
            setattr(g, kind, s[kind])
            for _ in range(3):
                m.MatchGuided(4.0, a, b, g)
            scan, total = [], []
            for _ in range(args.reps):
                m.MatchGuided(4.0, a, b, g)
                sc, t = m.LastTiming()
                scan.append(sc); total.append(t)
            out["guided_" + kind] = {"matches": int(len(g.inlier_matches)), "scan_ms_min": stats(scan)[0],
                                     "scan_ms_median": stats(scan)[1], "call_device_ms_median": stats(total)[1]}
            print(f"guided {kind}, 8192 x 8192 with cross-check: {len(g.inlier_matches)} matches; guided scan "
                  f"{stats(scan)[0]:.3f} ms min / {stats(scan)[1]:.3f} ms median, whole call on the device "
                  f"{stats(total)[1]:.3f} ms (CUDA events, {args.reps} reps)", flush=True)

    rng = np.random.default_rng(3)
    images = [FeatureMatcherImage(im.image_id, im.descriptors, s["camera1"],
                                  rng.uniform([0, 0], [640, 480], (N, 2)).astype(np.float32))
              for im in block_images(args.block, N, seed=2)]
    pairs = [(i, j) for i in range(len(images)) for j in range(i + 1, len(images))]
    geos = [TwoViewGeometry(config=TwoViewGeometry.UNCALIBRATED, F=s["F"]) for _ in pairs]
    with CreateSiftFeatureMatcher(FeatureMatchingOptions(gpu_index="0")) as m:
        m.MatchGuidedPairs(images, pairs, geos, 4.0)
        wall = []
        for _ in range(3):
            t0 = time.perf_counter()
            res = m.MatchGuidedPairs(images, pairs, geos, 4.0)
            wall.append(time.perf_counter() - t0)
            sc, t = m.LastTiming()
    nm = sum(len(r) for r in res)
    out["guided_block_F"] = {"images": args.block, "pairs": len(pairs), "matches": int(nm), "call_s_min": min(wall),
                             "pairs_per_s": len(pairs) / min(wall), "scan_ms": sc, "device_ms": t}
    print(f"guided block {args.block} x {N} under F: {len(pairs)} pairs, {nm} matches; {len(pairs) / min(wall):.0f} "
          f"pairs/s ({min(wall) * 1e3:.1f} ms per MatchGuidedPairs call, host clock; guided scans {sc:.1f} ms, device "
          f"work {t:.1f} ms)", flush=True)

    if args.oracle_pairs:
        import oracle_smg
        g1, g2 = oracle_smg.geo(s["camera1"], s["xy1"]), oracle_smg.geo(s["camera2"], s["xy2"])
        t0 = time.perf_counter()
        ref = oracle_smg.match(s["desc1"], s["desc2"], s["xy1"], s["xy2"], oracle_smg.E, s["E"], 4.0, g1, g2)
        per = time.perf_counter() - t0
        with CreateSiftFeatureMatcher(FeatureMatchingOptions(gpu_index="0")) as m:
            g = TwoViewGeometry(config=TwoViewGeometry.CALIBRATED, E=s["E"])
            m.MatchGuided(4.0, a, b, g)
        ok = bool(np.array_equal(ref, g.inlier_matches))
        out["guided_cpu_restatement"] = {"cores": os.cpu_count(), "s_per_pair_E": per, "equal_to_gpu": ok}
        print(f"CPU restatement of the guided rule (tests/sm_guided_oracle.c, OpenMP, {os.cpu_count()} cores): "
              f"{per:.2f} s per 8192 x 8192 E pair with cross-check; GPU matches identical: {ok}", flush=True)


if __name__ == "__main__":
    main()
