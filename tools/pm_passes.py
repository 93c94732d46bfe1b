"""Per-rotation pass times of a PatchMatch run: R|M (rand and msg side by side, then R and M alone), P (pixel) and S
(serial), averaged over the sweeps of each frame (frames 0 and 2 walk W columns of H rows, frames 1 and 3 walk H columns
of W rows), plus the part of the run before the first sweep (patch store + initial cost).  CUDA events inside the
library, one line per configuration.
usage: pm_passes.py [W H N] ["K1=V1 K2=V2" ...]   (defaults: the bench.py C2 shape 1920 1080 8; each quoted argument is
one set of environment settings, e.g. "B200PM_PATCH_STORE=0"; none: the defaults)"""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from colmap_b200.patch_match import PatchMatch, PatchMatchOptions
from colmap_b200.synthetic import make_patch_match_scene

args = sys.argv[1:]
w, h, n = (int(v) for v in args[:3]) if len(args) >= 3 and args[0].isdigit() else (1920, 1080, 8)
configs = (args[3:] if len(args) >= 3 and args[0].isdigit() else args) or [""]
REPS = 3
PASSES = 5   # last_sweep_pass_ms indices: R|M, P, S, R alone, M alone
sc = make_patch_match_scene(w, h, n, seed=0)
o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False, window_radius=5,
                      window_step=1, num_samples=15, num_iterations=5, gpu_index="0")
sweeps = 4 * o.num_iterations
for cfg in configs:
    env = dict(kv.split("=") for kv in cfg.split())
    os.environ.update(env)
    pm = PatchMatch(o, sc["problem"])
    pm.Run()   # warm-up
    run_ms, pre_ms = [], []
    per = np.zeros((4, PASSES))
    for _ in range(REPS):
        pm.RunOnly()
        run_ms.append(pm.last_run_ms())
        pre_ms.append(pm.last_run_ms() - pm.last_sweep_ms())
        for t in range(sweeps):
            for k in range(PASSES):
                per[t % 4, k] += pm.last_sweep_pass_ms(t, k)
    store = pm.patch_store_bytes()
    pm.close()
    for k in env:
        os.environ.pop(k, None)
    per /= REPS * (sweeps // 4)
    print(f"[{cfg or 'defaults'}] {w}x{h} N={n}: run {np.mean(run_ms):.1f} ms (min {np.min(run_ms):.1f}), before the sweeps "
          f"{np.mean(pre_ms):.2f} ms, patch store {store / 1e9:.2f} GB", flush=True)
    for r in range(4):
        cols = h if r & 1 else w
        print(f"  frame {r} ({cols:4d} columns): R|M {per[r, 0]:6.2f} (R {per[r, 3]:5.2f}, M {per[r, 4]:5.2f})  "
              f"P {per[r, 1]:6.2f}  S {per[r, 2]:6.2f}  sweep {per[r, :3].sum():6.2f} ms", flush=True)
