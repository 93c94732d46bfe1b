"""Time b200ra_solve (rotation averaging, L1 then IRLS) on synthetic pose graphs: about 20 pairs per frame, 1 degree of
noise, 10 % outliers.  For each size: the iteration counts of both phases and the device time of each phase, split into
matrix builds, factorisations and triangular solves (CUDA events inside the library), and the wall time of the fp64
scipy oracle where it fits.  Prints the card's name and power limit with the numbers.

    python tools/ra_time.py [--frames 1000 5000 10000 30000] [--oracle-max 2000]
"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from colmap_b200.rotation_averaging import RotationEstimatorOptions, solve_flat  # noqa: E402
from colmap_b200.synthetic import synthesize_rotation_averaging  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        return "unknown card"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[1000, 5000, 10000, 30000])
    ap.add_argument("--edges-per-frame", type=int, default=20)
    ap.add_argument("--oracle-max", type=int, default=2000, help="time the scipy oracle up to this many frames")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    print(f"card: {card()}")
    opts = RotationEstimatorOptions(gpu_index=0)
    warm, _ = synthesize_rotation_averaging(200, a.edges_per_frame, seed=a.seed)
    solve_flat(opts, warm)   # module load and first launches
    print(f"{'frames':>7} {'pairs':>8} {'n':>6} {'L1 it':>5} {'ADMM it':>7} {'IRLS it':>7} {'L1 ms':>9} {'IRLS ms':>9} "
          f"{'build ms':>9} {'factor ms':>10} {'solve ms':>9} {'wall s':>7} {'oracle s':>9}")
    for F in a.frames:
        flat, _ = synthesize_rotation_averaging(F, a.edges_per_frame, noise_deg=1.0, outlier_ratio=0.1, seed=a.seed)
        f = flat.copy()
        t0 = time.perf_counter()
        s = solve_flat(opts, f)
        wall = time.perf_counter() - t0
        orc = "-"
        if F <= a.oracle_max:
            import ra_oracle
            t0 = time.perf_counter()
            ra_oracle.solve(opts, flat.copy())
            orc = f"{time.perf_counter() - t0:.1f}"
        print(f"{F:>7} {len(flat.pair_frame1):>8} {s.n_y:>6} {s.num_l1_iterations:>5} {int(s.admm_iterations.sum()):>7} "
              f"{s.num_irls_iterations:>7} {s.l1_ms:>9.1f} {s.irls_ms:>9.1f} {s.build_ms:>9.1f} {s.factor_ms:>10.1f} "
              f"{s.solve_ms:>9.1f} {wall:>7.2f} {orc:>9}  status {s.status}", flush=True)


if __name__ == "__main__":
    main()
