"""Cost of the position priors in the covariance estimate: B3 (500 SIMPLE_RADIAL cameras, 300k points, 2M observations)
solved under the two-cams gauge, then estimated in ALL mode with and without a prior on every image (pose 0 is constant,
so 499 priors are kept), the two alternating in one process.  Reports the device time of each b200ba_covariance_info
phase (set-up is host time), minimum and median over the repeats, and the card's name and power limit.

  python tools/ba_cov_prior_time.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

from colmap_b200.bundle_adjustment import (ITERATIVE_SCHUR, SIMPLE_RADIAL, BACovarianceOptions,  # noqa: E402
                                           BundleAdjustmentOptions, estimate_covariance_flat, solve_flat)
from colmap_b200.synthetic import synthesize_ba_problem  # noqa: E402
from prior_cases import flat_priors  # noqa: E402

PHASES = ("setup", "build", "factorize", "inverse")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    print("GPU:", smi.strip().splitlines()[0] if smi.strip() else "unknown", flush=True)
    o = BundleAdjustmentOptions(linear_solver_type=ITERATIVE_SCHUR, gpu_index=0)
    _, b3 = synthesize_ba_problem(500, 300000, 7, models=(SIMPLE_RADIAL,), seed=42, num_obs=2000000)
    b3.pose_constant = b3.pose_constant.copy(); b3.pose_fixed_dim = b3.pose_fixed_dim.copy()
    b3.pose_constant[0] = 1
    b3.pose_fixed_dim[1] = int(np.argmax(np.abs(b3.poses[1, 4:] - b3.poses[0, 4:])))
    s = solve_flat(o, b3)
    print(f"B3 solved: {s.num_successful_steps + s.num_unsuccessful_steps} LM iterations", flush=True)
    priors = flat_priors(b3, seed=3, stddev=0.05)
    runs = {"without": [], "with": []}
    for rep in range(args.reps + 1):              # the first pair warms up
        for label, pr in (("without", None), ("with", priors)):
            cov = estimate_covariance_flat(o, BACovarianceOptions(BACovarianceOptions.ALL), b3, raise_not_estimable=True, priors=pr)
            n, ms = cov.info()
            cov.close()
            if rep:
                runs[label].append(ms)
    for label, rs in runs.items():
        row = {"config": f"B3 ALL {label} priors", "n": n, "num_priors": len(priors) if label == "with" else 0}
        for p in PHASES:
            v = np.array([r[p] for r in rs])
            row[f"{p}_ms_min"], row[f"{p}_ms_median"] = round(float(v.min()), 3), round(float(np.median(v)), 3)
        print(json.dumps(row), flush=True)
    d = np.array([a["build"] for a in runs["with"]]) - np.array([b["build"] for b in runs["without"]])
    print(f"build phase, with minus without priors, pair by pair: median {np.median(d):.3f} ms, "
          f"range [{d.min():.3f}, {d.max():.3f}] ms", flush=True)


if __name__ == "__main__":
    main()
