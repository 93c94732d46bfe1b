"""LM iterations per second of the global positioner (b200gp_solve, device time from CUDA events) on synthetic BATA
problems, and the fp64 oracle (tests/gp_oracle.py, a scipy port of the same LM, not Ceres) beside it where it fits.

    python tools/gp_time.py [--iters 10] [--oracle-max-obs 20000]

Prints one JSON line per size with the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from colmap_b200.global_positioning import GlobalPositionerOptions, solve_flat  # noqa: E402
from colmap_b200.synthetic import synthesize_global_positioning  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--oracle-max-obs", type=int, default=0, help="also time the oracle up to this many observations")
    a = ap.parse_args()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:
        card = "unknown"
    sizes = [(1000, 300000, 2100000), (100, 3000, 21000), (2000, 100000, 700000), (5000, 200000, 1400000),
             (10900, 300000, 2100000)]
    for F, P, N in sizes:
        flat = synthesize_global_positioning(F, P, N)
        o = GlobalPositionerOptions(max_num_iterations=a.iters, function_tolerance=0.0, parameter_tolerance=0.0)
        solve_flat(o, flat.copy())   # warm-up: module load and allocations
        g = flat.copy()
        s = solve_flat(o, g)
        it = len(s.cost_history) - 1
        row = dict(frames=F, points=P, observations=len(flat.obs_frame), reduced_dim=s.reduced_dim, iterations=it,
                   successful_steps=s.num_successful_steps, unsuccessful_steps=s.num_unsuccessful_steps,
                   initial_cost=s.initial_cost, final_cost=s.final_cost,
                   device_ms=round(s.solve_ms, 2), gpu_iters_per_s=round(it / (s.solve_ms / 1e3), 2), card=card)
        if len(flat.obs_frame) <= a.oracle_max_obs:
            import gp_oracle
            r = flat.copy()
            t0 = time.perf_counter()
            sr = gp_oracle.solve(r, a.iters, function_tolerance=0.0, parameter_tolerance=0.0)
            dt = time.perf_counter() - t0
            row.update(oracle_port_iters_per_s=round((len(sr.cost_history) - 1) / dt, 3), oracle_threads=os.cpu_count(),
                       final_cost_rel_diff=float(abs(s.final_cost - sr.final_cost) / sr.final_cost))
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
