"""Timing of the PatchMatch run, split into the rand(+msg) / pixel / serial passes, under sets of environment settings
(the B200PM_WPC / B200PM_PRUNE / B200PM_PRUNE_FROM schedule seams): one line per configuration.
usage: pm_time.py W H N "K1=V1 K2=V2" "K1=V3" ...   (each quoted argument is one configuration; none: the defaults)"""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from colmap_b200.patch_match import PatchMatch, PatchMatchOptions
from colmap_b200.synthetic import make_patch_match_scene

w, h, n = (int(v) for v in sys.argv[1:4])
configs = sys.argv[4:] or [""]
sc = make_patch_match_scene(w, h, n, seed=0)
o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False, gpu_index="0")
for cfg in configs:
    env = dict(kv.split("=") for kv in cfg.split())
    for k, v in env.items():
        os.environ[k] = v
    pm = PatchMatch(o, sc["problem"])
    pm.Run()
    ms = []
    for _ in range(2):
        pm.RunOnly()
        ms.append((pm.last_run_ms(), pm.last_pass_ms(0), pm.last_pass_ms(1), pm.last_pass_ms(2)))
    d = pm.GetDepthMap()
    pm.close()
    for k in env:
        os.environ.pop(k, None)
    m = np.mean(ms, axis=0)
    print(f"{cfg:60s} run {m[0]:7.1f} ms = {w * h / 1e3 / m[0]:.3f} Mpx/s  rand+msg {m[1]:6.1f} pixel {m[2]:6.1f} serial-tail {m[3]:6.1f}  checksum {float(np.abs(d).sum()):.3f}", flush=True)
