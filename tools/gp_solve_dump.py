"""Solve two seeded global-positioning problems with b200gp_solve and save every output array, so that two builds of
the library (for example before and after a change to the dense solves) can be compared bit for bit:

    python tools/gp_solve_dump.py out_a.npz            # with one build
    python tools/gp_solve_dump.py out_b.npz            # with the other
    python tools/gp_solve_dump.py --compare out_a.npz out_b.npz

Problems: synthesize_global_positioning seed 0 with 300 frames, 3,000 points, 30,000 observations, and seed 1 with
1,000 frames, 4,000 points, 40,000 observations; up to 30 LM iterations each.  Saved: frame centres, points, scales and the
cost history of each.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [(0, 300, 3000, 30000), (1, 1000, 4000, 40000)]


def dump(path):
    from colmap_b200.global_positioning import GlobalPositionerOptions, solve_flat
    from colmap_b200.synthetic import synthesize_global_positioning
    out = {}
    for seed, F, P, N in CASES:
        flat = synthesize_global_positioning(F, P, N, seed=seed)
        s = solve_flat(GlobalPositionerOptions(gpu_index=0, max_num_iterations=30), flat)
        print(f"seed {seed}: {s.num_successful_steps + s.num_unsuccessful_steps} iterations, final cost {s.final_cost!r}")
        out.update({f"centers{seed}": flat.frame_centers, f"points{seed}": flat.points, f"scales{seed}": flat.obs_scale,
                    f"costs{seed}": s.cost_history})
    np.savez(path, **out)


def compare(a, b):
    A, B = np.load(a), np.load(b)
    same = True
    for k in A.files:
        eq = A[k].shape == B[k].shape and np.array_equal(A[k].view(np.uint64), B[k].view(np.uint64))
        same &= eq
        print(f"{k} {A[k].shape}: {'bit-identical' if eq else 'DIFFERENT'}")
    return 0 if same else 1


if __name__ == "__main__":
    if sys.argv[1] == "--compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    dump(sys.argv[1])
