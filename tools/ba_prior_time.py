"""Cost of the pose priors in the GPU LM solve: B3 (500 SIMPLE_RADIAL cameras, 300k points, 2M observations,
ITERATIVE_SCHUR) with a noisy prior on every image, TRIVIAL and CAUCHY prior loss, and a mapper-sized problem (50 images,
DENSE_SCHUR; its camera side of 394 columns is above the dense factorisation's 256, so it runs the exact PCG).  Solves with and without priors alternate in one process; LM iterations/s from the solve's device
time; the prior kernels' device time per LM iteration from a separate torch.profiler run.  Prints one JSON line per
configuration and the card's name and power limit.

  python tools/ba_prior_time.py [--reps 3] [--iters 20]
"""
import argparse
import dataclasses
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

from colmap_b200.bundle_adjustment import (CAUCHY, DENSE_SCHUR, ITERATIVE_SCHUR, SIMPLE_RADIAL, TRIVIAL,  # noqa: E402
                                           BundleAdjustmentOptions, solve_flat, solve_flat_with_position_priors)
from colmap_b200.synthetic import synthesize_ba_problem  # noqa: E402
from prior_cases import flat_priors  # noqa: E402


def _gauge(flat):
    flat.pose_constant = flat.pose_constant.copy(); flat.pose_fixed_dim = flat.pose_fixed_dim.copy()
    flat.pose_constant[0] = 1
    flat.pose_fixed_dim[1] = int(np.argmax(np.abs(flat.poses[1, 4:] - flat.poses[0, 4:])))
    return flat


def _fresh(noisy):
    f = noisy.copy()
    f.pose_constant, f.pose_fixed_dim = noisy.pose_constant, noisy.pose_fixed_dim
    return f


def _prior_kernel_ms(options, noisy, priors):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s = solve_flat_with_position_priors(options, _fresh(noisy), priors)
        torch.cuda.synchronize()
    total = sum(e.device_time_total for e in prof.key_averages() if "ba_prior" in e.key) / 1e3
    return total, s.num_successful_steps + s.num_unsuccessful_steps


def run(name, options, noisy, loss, reps):
    priors = flat_priors(noisy, seed=3, stddev=0.05, loss=loss)
    rows = {"without": [], "with": []}
    for _ in range(reps + 1):              # the first round warms up
        for key in ("without", "with"):
            f = _fresh(noisy)
            s = solve_flat(options, f) if key == "without" else solve_flat_with_position_priors(options, f, priors)
            lm = s.num_successful_steps + s.num_unsuccessful_steps
            rows[key].append((lm / (s.solve_ms / 1e3), s.solve_ms / lm, s.kernel_launches, s.num_linear_solver_iterations, lm))
    rows = {k: v[1:] for k, v in rows.items()}
    ms, lm = _prior_kernel_ms(options, noisy, priors)
    out = {"config": name, "prior_loss": {TRIVIAL: "TRIVIAL", CAUCHY: "CAUCHY"}[loss], "priors": len(priors),
           "lm_it_per_s_without": [round(r[0], 2) for r in rows["without"]],
           "lm_it_per_s_with": [round(r[0], 2) for r in rows["with"]],
           "ms_per_lm_it_without": round(float(np.median([r[1] for r in rows["without"]])), 4),
           "ms_per_lm_it_with": round(float(np.median([r[1] for r in rows["with"]])), 4),
           "launches_without": rows["without"][0][2], "launches_with": rows["with"][0][2],
           "pcg_without": rows["without"][0][3], "pcg_with": rows["with"][0][3],
           "lm_its_without": rows["without"][0][4], "lm_its_with": rows["with"][0][4],
           "prior_kernels_ms_per_lm_it": round(ms / max(lm, 1), 4)}
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)
    gt, b3 = synthesize_ba_problem(500, 300000, 7, models=(SIMPLE_RADIAL,), seed=42, num_obs=2000000)
    _gauge(b3)
    it = BundleAdjustmentOptions(linear_solver_type=ITERATIVE_SCHUR, max_num_iterations=a.iters, gpu_index=0)
    for loss in (TRIVIAL, CAUCHY):
        run("B3", it, b3, loss, a.reps)
    gt, m50 = synthesize_ba_problem(50, 4000, 6, models=(SIMPLE_RADIAL,), seed=7)
    _gauge(m50)
    dense = BundleAdjustmentOptions(linear_solver_type=DENSE_SCHUR, max_num_iterations=a.iters, gpu_index=0)
    for loss in (TRIVIAL, CAUCHY):
        run("mapper_50_images_exact", dense, m50, loss, a.reps)


if __name__ == "__main__":
    main()
