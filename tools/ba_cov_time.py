"""Bundle-adjustment covariance timing (b200ba_estimate_covariance): B3 solved first, then estimated in ALL, POSES and
POINTS mode, with the device time of every phase, the factorisation + inverse rate (n^3 flops) against the H100 SXM
data-sheet fp64 tensor-core rate (67 TFLOP/s dense), the bulk read-back and the CPU route (tests/oracle_cov.py: scipy.sparse
+ LAPACK on the same problem; the Jacobian, which that module forms observation by observation in Python, is timed
apart).  Then a B5-sized camera set (2000 SIMPLE_RADIAL cameras, 200k points, n = 15993), estimated at its synthetic
parameters.  Prints the card and its power limit."""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from colmap_b200.bundle_adjustment import (ITERATIVE_SCHUR, SIMPLE_RADIAL, BACovarianceOptions, BundleAdjustmentOptions,
                                           estimate_covariance_flat, solve_flat)
from colmap_b200.synthetic import synthesize_ba_problem

PEAK_FP64_TC = 67e12


def gauge(flat):
    flat.pose_constant = flat.pose_constant.copy(); flat.pose_fixed_dim = flat.pose_fixed_dim.copy()
    flat.pose_constant[0] = 1
    flat.pose_fixed_dim[1] = int(np.argmax(np.abs(flat.poses[1, 4:] - flat.poses[0, 4:])))
    return flat


def run(name, o, flat, modes, repeats=3):
    for mode, label in modes:
        best = None
        for _ in range(repeats):
            t = time.time()
            cov = estimate_covariance_flat(o, BACovarianceOptions(mode), flat, raise_not_estimable=True)
            wall = (time.time() - t) * 1e3
            n, ms = cov.info()
            t = time.time(); cov.poses_all(); cov.points_all(); readback = (time.time() - t) * 1e3
            cov.close()
            if best is None or ms["factorize"] + ms["inverse"] < best[1]["factorize"] + best[1]["inverse"]:
                best = (n, ms, wall, readback)
        n, ms, wall, readback = best
        fi = ms["factorize"] + ms["inverse"]
        rate = n ** 3 / (fi * 1e-3) / 1e12 if fi > 0 else 0.0
        print(f"{name} {label:5s} n={n:6d}: setup {ms['setup']:.1f} ms, build {ms['build']:.2f} ms, factorize {ms['factorize']:.2f} ms, "
              f"inverse {ms['inverse']:.2f} ms, bulk read-back {readback:.1f} ms, call {wall:.1f} ms; "
              f"factorize + inverse {rate:.2f} TFLOP/s = {100 * rate * 1e12 / PEAK_FP64_TC:.1f}% of 67", flush=True)


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    print("GPU:", smi.strip().splitlines()[0] if smi.strip() else "unknown")
    o = BundleAdjustmentOptions(linear_solver_type=ITERATIVE_SCHUR, gpu_index=0)
    _, b3 = synthesize_ba_problem(500, 300000, 7, models=(SIMPLE_RADIAL,), seed=42, num_obs=2000000)
    gauge(b3)
    s = solve_flat(o, b3)
    print(f"B3 solved: {s.num_successful_steps + s.num_unsuccessful_steps} LM iterations, cost {s.final_cost:.6f}")
    run("B3", o, b3, [(BACovarianceOptions.ALL, "ALL"), (BACovarianceOptions.POSES, "POSES"), (BACovarianceOptions.POINTS, "POINTS")])
    if "--no-cpu" not in sys.argv:
        import oracle_cov
        t = time.time()
        jac = oracle_cov.jacobian(o, b3)
        t_jac = time.time() - t
        t = time.time()
        est, msg = oracle_cov.estimate(o, b3, oracle_cov.ALL, cross=False, jac=jac)
        print(f"B3 CPU route (oracle_cov.estimate, ALL, diagonal blocks only): {time.time() - t:.1f} s of sparse / dense "
              f"algebra after {t_jac:.1f} s forming the Jacobian observation by observation in Python", flush=True)
    _, b5 = synthesize_ba_problem(2000, 200000, 6, models=(SIMPLE_RADIAL,), seed=7, point2D_stddev=0.5)
    gauge(b5)
    run("B5-sized", o, b5, [(BACovarianceOptions.ALL, "ALL")], repeats=2)


if __name__ == "__main__":
    main()
