"""Solve the bundle-adjustment problems of tests/test_ba_paths_gpu.py, one with position priors, and B3 of bench.py, and
save every output, so that two builds of the library (for example before and after a change to the PCG kernels) can be
compared bit for bit:

    python tools/ba_solve_dump.py out_a.npz                          # with the library of this checkout
    python tools/ba_solve_dump.py --tree OTHER_CHECKOUT out_b.npz    # with the library built in another checkout
    python tools/ba_solve_dump.py --compare out_a.npz out_b.npz

Cases: every natural-size case of test_ba_paths_gpu.py (one per PCG form: staged, mid with r in shared memory and in
global memory, multi-kernel), the seam_narrow cases (every B200BA_* seam, ITERATIVE_SCHUR and exact PCG), the
full_opencv cases (blocks wider than 11 columns through the staged, mid and multi-kernel forms), seam_narrow with one
position prior per pose, each for 10 LM iterations, and B3 (500 cameras, 2M observations) for up to 100.  Saved per
case: poses, intrinsics, points, rig sensors, initial and final cost, and the PCG, step and termination counts.

Each case is solved twice.  A case whose two solves differ is marked not reproducible: the reduced camera system is
accumulated with fp64 atomics (red.add) in an order that changes from run to run, so its last bits, and those of
everything downstream, drift between two solves of one build.  --compare fails on any difference in a reproducible
case; for the others it prints the largest relative difference of the cost and of the parameters and whether the PCG
and LM counts agree, to be read against the drift between two solves of one build.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LM_ITERATIONS = 10


def _cases():
    import dataclasses
    from test_ba_paths_gpu import NATURAL, SEAM, WIDE, _problem
    for c in NATURAL + [c for c in SEAM if c.problem == "seam_narrow"] + [c for c in WIDE if c.problem == "full_opencv"]:
        yield c.id, _problem(c.problem), dataclasses.replace(c.options, max_num_iterations=LM_ITERATIONS), dict(c.env), None
    from prior_cases import flat_priors
    from test_ba_paths_gpu import ITER
    noisy = _problem("seam_narrow")
    yield ("seam_narrow-iter-priors", noisy, dataclasses.replace(ITER, max_num_iterations=LM_ITERATIONS), {},
           flat_priors(noisy, seed=5))
    from bench import _b3_problem
    from colmap_b200.bundle_adjustment import ITERATIVE_SCHUR, BundleAdjustmentOptions
    yield "b3", _b3_problem(), BundleAdjustmentOptions(linear_solver_type=ITERATIVE_SCHUR), {}, None


def _solve(flat, options, env, priors):
    from colmap_b200.bundle_adjustment import solve_flat, solve_flat_with_position_priors
    from test_ba_paths_gpu import SEAMS
    f = flat.copy()
    f.pose_constant, f.pose_fixed_dim, f.point_constant, f.cam_constant = (flat.pose_constant, flat.pose_fixed_dim,
                                                                            flat.point_constant, flat.cam_constant)
    for k in SEAMS:
        os.environ.pop(k, None)
    os.environ.update(env)
    try:
        s = solve_flat_with_position_priors(options, f, priors) if priors is not None else solve_flat(options, f)
    finally:
        for k in env:
            os.environ.pop(k)
    return dict(poses=f.poses, cam_params=f.cam_params, points=f.points, sensors=f.sensors,
                costs=np.array([s.initial_cost, s.final_cost]),
                counts=np.array([s.num_linear_solver_iterations, s.num_successful_steps, s.num_unsuccessful_steps,
                                 s.termination_type], np.int64))


def dump(path, tree):
    for p in (os.path.join(ROOT, "tests"), ROOT, tree):   # colmap_b200 (and its library) from `tree`, cases from here
        sys.path.insert(0, p)
    import colmap_b200
    print(f"library {colmap_b200.__file__}")
    out = {}
    for name, flat, options, env, priors in _cases():
        runs = [_solve(flat, options, env, priors) for _ in range(2)]
        same = all(runs[0][k].tobytes() == runs[1][k].tobytes() for k in runs[0])
        c = runs[0]["counts"]
        print(f"{name}: {c[0]} PCG iterations, {c[1]}+{c[2]} LM steps, final cost {runs[0]['costs'][1]!r}"
              f"{'' if same else ', NOT reproducible'}")
        out.update({f"{name}/{k}": v for k, v in runs[0].items()})
        out[f"{name}/reproducible"] = np.array(same)
    np.savez(path, **out)


def compare(a, b):
    A, B = np.load(a), np.load(b)
    names = sorted({k.rsplit("/", 1)[0] for k in A.files} | {k.rsplit("/", 1)[0] for k in B.files})
    failed = 0
    for n in names:
        keys = sorted(k for k in set(A.files) | set(B.files) if k.startswith(n + "/") and not k.endswith("/reproducible"))
        diff = [k.rsplit("/", 1)[1] for k in keys
                if not (k in A.files and k in B.files and A[k].dtype == B[k].dtype and A[k].shape == B[k].shape
                        and A[k].tobytes() == B[k].tobytes())]
        rep = all(bool(X[f"{n}/reproducible"]) for X in (A, B) if f"{n}/reproducible" in X.files)
        if not diff:
            print(f"{n}: bit-identical")
        elif rep:
            failed += 1
            print(f"{n}: DIFFERENT ({', '.join(diff)})")
        else:
            cost = abs(A[f"{n}/costs"][1] - B[f"{n}/costs"][1]) / abs(A[f"{n}/costs"][1])
            par = max(np.abs(A[f"{n}/{g}"] - B[f"{n}/{g}"]).max(initial=0.0) / max(1.0, np.abs(A[f"{n}/{g}"]).max(initial=0.0))
                      for g in ("poses", "points", "cam_params", "sensors"))
            counts = "equal" if "counts" not in diff else f"{A[f'{n}/counts'].tolist()} vs {B[f'{n}/counts'].tolist()}"
            print(f"{n}: not reproducible within one build; final cost {cost:.1e}, parameters {par:.1e} relative, "
                  f"counts {counts}")
    print(f"{failed} reproducible case(s) differ")
    return 1 if failed else 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    ap.add_argument("--tree", default=ROOT, help="checkout whose colmap_b200 and built library solve (default: this one)")
    ap.add_argument("out", nargs="?")
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if not args.out:
        ap.error("an output file, or --compare A B")
    dump(args.out, os.path.abspath(args.tree))
