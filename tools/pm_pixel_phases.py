"""Where the pixel pass (pm_pixel_kernel) spends its time: compiles patch_match.cu with -DPM_PIXEL_PHASES into a scratch
library (a temporary directory; the other objects are the ones build() left in colmap_b200/lib), runs one PatchMatch
problem and prints, for the unpruned first sweep and for the pruned sweeps, the share of lane 0's clock() cycles in each
phase of the pass and the cycles per pixel, and per pixel the NCCs the pixel pass evaluated, its rounds, the share of
its group slots left empty and the NCCs the serial pass evaluated itself (pm_pixel4_kernel, N <= 8).  The clock reads
change the schedule a little: the P time of the instrumented run is printed next to the shares so it can be set against
an uninstrumented run (tools/pm_passes.py).
usage: pm_pixel_phases.py [W H N]   (default: the bench.py C2 shape 1920 1080 8)"""
import ctypes
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import colmap_b200._lib as _lib
from colmap_b200.patch_match import PatchMatch, PatchMatchOptions
from colmap_b200.synthetic import make_patch_match_scene

PHASES = ["patch copy wait", "set-up (priors, CDF, prediction)", "pair selection", "tap loops",
          "NCC finalize (+ homography)", "bound update", "other (loop, input loads)"]
COUNTS = ["pixel-pass NCCs", "pixel-pass rounds", "serial-pass NCCs"]


def build_scratch(tmp):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    libdir = os.path.join(ROOT, "colmap_b200", "lib")
    objs = [os.path.join(libdir, f) for f in sorted(os.listdir(libdir)) if f.endswith(".o") and f != "patch_match.o"]
    if not objs:
        raise RuntimeError("colmap_b200/lib has no objects: run __graft_entry__.build() first")
    common = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17"]
    obj = os.path.join(tmp, "patch_match_phases.o")
    subprocess.check_call(common + ["-Xcompiler", "-fPIC,-ffp-contract=off", "-fmad=false", "-DPM_PIXEL_PHASES", "-c",
                                    os.path.join(ROOT, "colmap_b200", "csrc", "patch_match.cu"), "-o", obj])
    so = os.path.join(tmp, "libcolmap_b200_phases.so")
    subprocess.check_call(common + ["-shared", "-o", so, obj] + objs)
    return so


def main():
    args = sys.argv[1:]
    w, h, n = (int(v) for v in args[:3]) if len(args) >= 3 else (1920, 1080, 8)
    with tempfile.TemporaryDirectory() as tmp:
        lib = ctypes.CDLL(build_scratch(tmp), mode=ctypes.RTLD_GLOBAL)
        _lib._LIB = lib   # every PatchMatch below binds the instrumented library
        lib.b200pm_debug_pixel_phases.argtypes = [ctypes.POINTER(ctypes.c_ulonglong)]
        lib.b200pm_debug_pool_counts.argtypes = [ctypes.POINTER(ctypes.c_ulonglong)]
        nph = len(PHASES)
        buf = (ctypes.c_ulonglong * (2 * nph))()
        cbuf = (ctypes.c_ulonglong * (2 * len(COUNTS)))()
        sc = make_patch_match_scene(w, h, n, seed=0)
        o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                              window_radius=5, window_step=1, num_samples=15, num_iterations=5, gpu_index="0")
        sweeps = 4 * o.num_iterations
        pm = PatchMatch(o, sc["problem"])
        pm.Run()   # warm-up
        if lib.b200pm_debug_pixel_phases(buf) != nph:
            raise RuntimeError("phase count of the library and the tool differ")
        if lib.b200pm_debug_pool_counts(cbuf) != len(COUNTS):
            raise RuntimeError("counter count of the library and the tool differ")
        pm.RunOnly()
        p_ms = [pm.last_sweep_pass_ms(t, 1) for t in range(sweeps)]
        s_ms = [pm.last_sweep_pass_ms(t, 2) for t in range(sweeps)]
        lib.b200pm_debug_pixel_phases(buf)
        lib.b200pm_debug_pool_counts(cbuf)
        pm.close()
    cyc = np.array(buf[:], dtype=np.float64).reshape(2, nph)
    cnt = np.array(cbuf[:], dtype=np.float64).reshape(2, len(COUNTS))
    print(f"{w}x{h} N={n}: instrumented P {p_ms[0]:.2f} ms (sweep 0, unpruned), "
          f"{np.mean(p_ms[1:]):.2f} ms per pruned sweep (mean of {sweeps - 1}); S {s_ms[0]:.2f} / {np.mean(s_ms[1:]):.2f} ms")
    for k, name, nsw in ((0, "unpruned first sweep", 1), (1, "pruned sweeps", sweeps - 1)):
        tot = cyc[k].sum()
        print(f"  {name}: {tot / (w * h * nsw):.0f} cycles per pixel (lane 0 of its warp)")
        for j in range(nph):
            print(f"    {PHASES[j]:34s} {100.0 * cyc[k, j] / tot:5.1f} %")
        npx = w * h * nsw
        ncc_p, rounds, ncc_s = cnt[k]
        empty = 100.0 * (1.0 - ncc_p / (4.0 * rounds)) if rounds else 0.0
        print(f"    per pixel: P {ncc_p / npx:.2f} NCCs in {rounds / npx:.2f} rounds ({empty:.1f} % of group slots empty), "
              f"S {ncc_s / npx:.3f} NCCs")


if __name__ == "__main__":
    main()
