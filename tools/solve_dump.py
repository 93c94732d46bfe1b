"""Solve seeded global-positioning (b200gp_solve) and rotation-averaging (b200ra_solve) problems and save every output,
so that two builds of the library (for example before and after a change to the solves) can be compared bit for bit:

    python tools/solve_dump.py out_a.npz            # with one build
    python tools/solve_dump.py out_b.npz            # with the other
    python tools/solve_dump.py --compare out_a.npz out_b.npz

Global positioning: synthesize_global_positioning seed 0 with 300 frames, 3,000 points, 30,000 observations, and seed 1
with 1,000 frames, 4,000 points, 40,000 observations; up to 30 LM iterations each.  Saved: frame centres, points, scales,
the cost history, the initial and final costs and the summary counts.

Rotation averaging, default options (L1 then IRLS): synthesize_rotation_averaging(1000, seed=0), all frames 3-DOF (one
axis matrix, three right-hand sides, 16 tiles), and synthesize_rotation_averaging(600, gravity_fraction=0.3,
num_cameras=8, reweighting=True, seed=1) (two axis matrices, estimated cameras, reweighting).  Saved: rotations, the
step history, the ADMM iteration counts, and the status, iteration counts, axis sizes and residual count.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GP_CASES = [(0, 300, 3000, 30000), (1, 1000, 4000, 40000)]
RA_CASES = [(0, 1000, {}), (1, 600, dict(gravity_fraction=0.3, num_cameras=8, reweighting=True))]


def dump(path):
    from colmap_b200.global_positioning import GlobalPositionerOptions, solve_flat as gp_solve
    from colmap_b200.rotation_averaging import RotationEstimatorOptions, solve_flat as ra_solve
    from colmap_b200.synthetic import synthesize_global_positioning, synthesize_rotation_averaging
    out = {}
    for seed, F, P, N in GP_CASES:
        flat = synthesize_global_positioning(F, P, N, seed=seed)
        s = gp_solve(GlobalPositionerOptions(gpu_index=0, max_num_iterations=30), flat)
        print(f"gp seed {seed}: {s.num_successful_steps + s.num_unsuccessful_steps} iterations, final cost {s.final_cost!r}")
        out.update({f"centers{seed}": flat.frame_centers, f"points{seed}": flat.points, f"scales{seed}": flat.obs_scale,
                    f"costs{seed}": s.cost_history,
                    f"gp_cost_ends{seed}": np.array([s.initial_cost, s.final_cost]),
                    f"gp_counts{seed}": np.array([s.termination_type, s.num_successful_steps, s.num_unsuccessful_steps,
                                                  s.num_residuals, s.reduced_dim], np.int64)})
    for seed, F, kw in RA_CASES:
        flat, _ = synthesize_rotation_averaging(F, seed=seed, **kw)
        s = ra_solve(RotationEstimatorOptions(gpu_index=0), flat)
        print(f"ra seed {seed}: status {s.status}, {s.num_l1_iterations} L1 and {s.num_irls_iterations} IRLS iterations, "
              f"n_xz {s.n_xz}, n_y {s.n_y}")
        out.update({f"ra_rotations{seed}": flat.rotations, f"ra_steps{seed}": s.step_history,
                    f"ra_admm{seed}": s.admm_iterations,
                    f"ra_counts{seed}": np.array([s.status, s.num_l1_iterations, s.num_irls_iterations, s.n_xz, s.n_y,
                                                  s.num_residuals], np.int64)})
    np.savez(path, **out)


def compare(a, b):
    A, B = np.load(a), np.load(b)
    same = set(A.files) == set(B.files)
    for k in sorted(set(A.files) | set(B.files)):
        eq = (k in A.files and k in B.files and A[k].dtype == B[k].dtype and A[k].shape == B[k].shape
              and A[k].tobytes() == B[k].tobytes())
        same &= eq
        shape = A[k].shape if k in A.files else B[k].shape
        print(f"{k} {shape}: {'bit-identical' if eq else 'DIFFERENT'}")
    return 0 if same else 1


if __name__ == "__main__":
    if sys.argv[1] == "--compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    dump(sys.argv[1])
