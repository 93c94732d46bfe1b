"""Every solve path of b200ba_solve against the fp64 CPU oracle (oracle/ba_oracle.c).

The solver picks its reduced-system kernels from the shape of the problem: nc, the camera-side dimension (6 per
variable pose, the variable intrinsics, 6 per refined rig sensor), and dkmax, the widest camera block, which sets DC,
the template width every LM kernel is instantiated for.  The small problems of test_ba_gpu.py only reach the dense
solve, the staged PCG step and the shared-memory SpMV.  This file puts one problem into every other regime, pairs of
problems on both sides of each shared-memory boundary, the exact solves, every B200BA_* seam and the wide (> 11
columns, DC = 28) camera blocks.

`test_every_case_lands_in_its_regime` needs no GPU: it runs the host flattening (b200ba_test_pack) on every case, so a
case that drifts out of the regime it is named for fails before any GPU is involved.

The checks:
  * arithmetic, every case: a 3-iteration solve from the same start takes the same steps on both sides, so the cost
    agrees to 1e-6 and the parameters to 1e-5 (test_wide_model_grid_parity, step 1; the intrinsics of exact PCG on
    the wide problems at 1e-4, see EXACT_WIDE_CAM_REL).  Under ITERATIVE_SCHUR the PCG
    iteration counts agree too: a preconditioner or dot-product bug costs iterations before it costs accuracy.  Exact
    solves must stop on the residual test, not on the iteration cap.
  * convergence, natural sizes, exact solves and the narrow seam problem: a 10-iteration solve at the large-problem bar
    of the B3 test (cost 1e-5, parameters 1e-4, the same number of LM steps).
"""
import dataclasses
import functools

import numpy as np
import pytest

from colmap_b200.bundle_adjustment import (AUTO, DENSE_SCHUR, FULL_OPENCV, ITERATIVE_SCHUR, OPENCV, PINHOLE, RADIAL,
                                           RAD_TAN_THIN_PRISM_FISHEYE, SIMPLE_RADIAL, SPARSE_SCHUR, THIN_PRISM_FISHEYE,
                                           BundleAdjustmentOptions)
from colmap_b200.synthetic import synthesize_ba_problem, synthesize_rig_problem
from test_ba_cpu import _pack
from test_ba_gpu import _assert_parity, _both, _gauge

# ---------------------------------------------------------------- the thresholds of colmap_b200/csrc: ba_common.cuh (DENSE_MAX,
# SPMV_SMEM_MAX, NARROW_MODELS) and bundle_adjustment.cu (the PCG step: PCG_FUSED_MAX, MID_STAGED_MAX, MID_SMEM_MAX)
DENSE_MAX = 256                  # BA_DENSE_MAX: exact requests up to this nc factorise the reduced matrix densely
PCG_FUSED_MAX = 65536            # BA_PCG_FUSED_MAX: single-CTA PCG vector step between SpMVs; above: five kernels
MID_STAGED_MAX = 1024 * 5        # BA_PCG_T * BA_MID_EPT: ba_pcg_mid_staged_kernel
MID_SMEM_MAX = 160 * 1024 // 8   # the 160 KB dynamic shared memory of ba_pcg_mid_kernel: r in shared memory
SPMV_SMEM_MAX = 72 * 1024 // 8   # BA_SPMV_SMEM_MAX: SpMV pass 1 with p in shared memory
NARROW_MODELS = (0, 1, 2, 3, 8, 9)   # ba_model_is_narrow: hand-written Jacobians, DC = 6 + dkmax
SEAMS = ("B200BA_NO_DENSE", "B200BA_PCG_MULTI", "B200BA_MID_GLOBAL", "B200BA_MID_PLAIN", "B200BA_SPMV_SMEM")



def regime(flat, options, env=None):
    """nc, dkmax, DC and the kernels b200ba_solve runs for (flat, options) under the environment `env`."""
    env = env or {}
    L = _pack(flat, options)
    nc, dkmax = L["nc"], L["dkmax"]
    wide = len(flat.sensors) > 0 or any(int(m) not in NARROW_MODELS for m in flat.cam_model)
    DC = (14 if dkmax <= 8 else 18 if dkmax <= 12 else 22 if dkmax <= 16 else 28) if wide else 6 + dkmax
    lst = options.linear_solver_type
    if lst == AUTO:
        nimg = flat.num_config_images or len(np.unique(flat.obs_pose))
        lst = DENSE_SCHUR if nimg <= 50 else (SPARSE_SCHUR if nimg <= 1000 else ITERATIVE_SCHUR)
    exact = lst != ITERATIVE_SCHUR
    r = dict(nc=nc, dkmax=dkmax, DC=DC, lst=lst, exact=exact, spmv=None)
    if exact and nc <= DENSE_MAX and "B200BA_NO_DENSE" not in env:
        r["path"] = "dense"
        return r
    fused = nc <= PCG_FUSED_MAX and "B200BA_PCG_MULTI" not in env
    if not fused:
        r["path"] = "multi"
    elif nc <= MID_STAGED_MAX and "B200BA_MID_PLAIN" not in env:
        r["path"] = "staged"
    else:
        r["path"] = "mid_smem" if nc <= MID_SMEM_MAX and "B200BA_MID_GLOBAL" not in env else "mid_global"
    if L["nblocks_warp"] == 0:      # no track of <= 32 observations: pass 1 runs ba_schur_spmv_kernel only
        r["spmv"] = "block"
    else:
        r["spmv"] = "smem" if env.get("B200BA_SPMV_SMEM", "1") != "0" and nc <= SPMV_SMEM_MAX else "global"
    return r


# ---------------------------------------------------------------- problems
# Exact PCG on the wide problems (seam_wide: single-image OPENCV / FULL_OPENCV cameras with the principal point refined;
# the thin-prism rigs) leaves some intrinsics nearly undetermined: the costs of the GPU and the oracle agree to 1e-9 while
# the intrinsics move along that flat valley.  There the deterministic dense solve lands within 0.2-0.4 of the 1e-5 bar,
# and ITERATIVE_SCHUR within 0.3-0.75 of it, the same on every run.  PCG run to the 1e-12 residual (170-280 iterations per
# solve on the rigs, about 630 on seam_wide, far below max_cg) lands within 0.05-1.11 of it, differently on every run:
# the fp64 atomics sum in a different order each time, and the fp32 rounding of the SpMV's per-observation intermediate
# then differs.  Poses, points and sensors stay within 0.01 of their 1e-5 bar.  So the intrinsics of exact PCG on these
# problems are compared at 1e-4, everything else at 1e-5.
EXACT_WIDE_CAM_REL = 1e-4
PTS_PER_CAM = 20        # tracks of 6: about 120 observations per camera
WIDE_NOISE = dict(point2D_stddev=0.3, point3D_stddev=0.02, rotation_stddev_deg=0.3)


def _natural(ncam, models, seed):
    gt, noisy = synthesize_ba_problem(ncam, ncam * PTS_PER_CAM, 6, models=models, seed=seed)
    return _gauge(noisy)


def _sized(nc, seed):
    """Own-intrinsics SIMPLE_RADIAL cameras (8 columns each; the first camera RADIAL when nc is odd) with pose 0 fixed
    and up to three constant cameras, so that the camera side has exactly `nc` columns."""
    odd = nc % 2
    ncam = -(-(nc + 6 - odd) // 8)
    drop = (8 * ncam - 6 + odd - nc) // 2
    models = ((RADIAL,) if odd else ()) + (SIMPLE_RADIAL,) * (ncam - odd)
    noisy = _natural(ncam, models, seed)
    noisy.cam_constant = noisy.cam_constant.copy()
    noisy.cam_constant[1:1 + drop] = 1
    return noisy


def _rig(model, seed):
    gt, noisy = synthesize_rig_problem(10, 3, 800, 8, models=(model,), seed=seed, point2D_stddev=0.5)
    return _gauge(noisy)


PROBLEMS = {
    # A: natural sizes
    "staged_ept5": lambda: _natural(600, (SIMPLE_RADIAL,), 31),
    "mid_smem_spmv_smem": lambda: _natural(1000, (PINHOLE, SIMPLE_RADIAL), 32),
    "b5_shape": lambda: _natural(2000, (PINHOLE, SIMPLE_RADIAL), 33),
    "mid_global": lambda: _natural(2600, (SIMPLE_RADIAL,), 34),
    "multi": lambda: _natural(8300, (RADIAL,), 35),
    # B: both sides of every shared-memory boundary
    **{f"nc{n}": functools.partial(_sized, n, 40 + k) for k, n in enumerate(
        (4096, 4097, 5120, 5121, 9216, 9217, 20480, 20481, 65536, 65537))},
    # C: exact solves
    "auto_100": lambda: _natural(100, (SIMPLE_RADIAL,), 51),
    "nc256": functools.partial(_sized, 256, 52),
    "nc257": functools.partial(_sized, 257, 53),
    # D: the seams
    "seam_narrow": lambda: _natural(60, (SIMPLE_RADIAL,), 61),
    "seam_wide": lambda: _gauge(synthesize_ba_problem(60, 60 * PTS_PER_CAM, 6, models=(OPENCV, FULL_OPENCV), seed=62,
                                                      **WIDE_NOISE)[1]),
    # E: wide camera blocks
    "full_opencv": lambda: _gauge(synthesize_ba_problem(16, 1200, 8, models=(FULL_OPENCV,), seed=71, **WIDE_NOISE)[1]),
    "rad_tan_thin_prism": lambda: _gauge(synthesize_ba_problem(16, 1200, 8, models=(RAD_TAN_THIN_PRISM_FISHEYE,), seed=72,
                                                               **WIDE_NOISE)[1]),
    "rig_opencv": lambda: _rig(OPENCV, 73),
    "rig_rad_tan_thin_prism": lambda: _rig(RAD_TAN_THIN_PRISM_FISHEYE, 74),
    "rig_thin_prism": lambda: _rig(THIN_PRISM_FISHEYE, 75),
}


@functools.lru_cache(maxsize=None)
def _problem(name):
    return PROBLEMS[name]()


ITER = BundleAdjustmentOptions(linear_solver_type=ITERATIVE_SCHUR)
DENSE = BundleAdjustmentOptions(linear_solver_type=DENSE_SCHUR)
PP = dict(refine_principal_point=True)


@dataclasses.dataclass(frozen=True)
class Case:
    problem: str
    options: BundleAdjustmentOptions
    env: tuple = ()          # (name, value) pairs
    expect: tuple = ()       # (key, value) pairs the regime must show
    cam_rel: float = 1e-5    # bar of the intrinsics in the arithmetic check (see EXACT_WIDE_CAM_REL)

    @property
    def id(self):
        mode = {ITERATIVE_SCHUR: "iter", DENSE_SCHUR: "dense", SPARSE_SCHUR: "sparse", AUTO: "auto"}[self.options.linear_solver_type]
        return "-".join([self.problem, mode] + [f"{k[7:].lower()}={v}" for k, v in self.env])


def _c(problem, options, env=(), cam_rel=1e-5, **expect):
    return Case(problem, options, tuple(env), tuple(expect.items()), cam_rel)


NATURAL = [
    _c("staged_ept5", ITER, path="staged", spmv="smem", nc=4794),
    _c("mid_smem_spmv_smem", ITER, path="mid_smem", spmv="smem", nc=7994),
    _c("b5_shape", ITER, path="mid_smem", spmv="global", nc=15994),
    _c("mid_global", ITER, path="mid_global", spmv="global", nc=20794),
    _c("multi", ITER, path="multi", spmv="global", nc=74694),
]
BOUNDARY = [
    _c("nc4096", ITER, path="staged", spmv="smem", nc=4096),
    _c("nc4097", ITER, path="staged", spmv="smem", nc=4097),
    _c("nc5120", ITER, path="staged", spmv="smem", nc=5120),
    _c("nc5121", ITER, path="mid_smem", spmv="smem", nc=5121),
    _c("nc9216", ITER, path="mid_smem", spmv="smem", nc=9216),
    _c("nc9217", ITER, path="mid_smem", spmv="global", nc=9217),
    _c("nc20480", ITER, path="mid_smem", spmv="global", nc=20480),
    _c("nc20481", ITER, path="mid_global", spmv="global", nc=20481),
    _c("nc65536", ITER, path="mid_global", spmv="global", nc=65536),
    _c("nc65537", ITER, path="multi", spmv="global", nc=65537),
]
EXACT = [
    _c("auto_100", BundleAdjustmentOptions(), path="staged", lst=SPARSE_SCHUR, exact=True, nc=794),
    _c("nc256", DENSE, path="dense", nc=256),
    _c("nc256", DENSE, (("B200BA_NO_DENSE", "1"),), path="staged", exact=True, nc=256),   # same system, PCG to 1e-12
    _c("nc257", DENSE, path="staged", exact=True, nc=257),
]
_SEAM_SETTINGS = [
    ((), dict(path="staged", spmv="smem")),
    ((("B200BA_MID_PLAIN", "1"),), dict(path="mid_smem", spmv="smem")),
    ((("B200BA_MID_PLAIN", "1"), ("B200BA_MID_GLOBAL", "1")), dict(path="mid_global", spmv="smem")),
    ((("B200BA_PCG_MULTI", "1"),), dict(path="multi", spmv="smem")),
    ((("B200BA_SPMV_SMEM", "0"),), dict(path="staged", spmv="global")),
]
# Each problem runs every setting under ITERATIVE_SCHUR and exact (DENSE_SCHUR with the dense factorisation off), so in
# one process every variable is set after a solve without it and unset after a solve with it.
SEAM = [
    _c(problem, dataclasses.replace(options, **kw), env + ((("B200BA_NO_DENSE", "1"),) if options is DENSE else ()),
       exact=options is DENSE, cam_rel=EXACT_WIDE_CAM_REL if options is DENSE and problem == "seam_wide" else 1e-5, **exp)
    for problem, kw in (("seam_narrow", {}), ("seam_wide", PP))
    for options in (ITER, DENSE)
    for env, exp in _SEAM_SETTINGS
]
_WIDE_PCG_SETTINGS = [((), "staged"), ((("B200BA_MID_PLAIN", "1"),), "mid_smem"), ((("B200BA_PCG_MULTI", "1"),), "multi")]
WIDE = [
    _c(problem, dataclasses.replace(ITER, **kw), env, path=path, dkmax=dk)
    for problem, kw, dk in (("full_opencv", PP, 12), ("rad_tan_thin_prism", PP, 16), ("rig_opencv", {}, 12))
    for env, path in _WIDE_PCG_SETTINGS
] + [
    _c(problem, dataclasses.replace(options, **PP), env, path=path, dkmax=dk, DC=28, cam_rel=cam_rel)
    for problem, dk in (("rig_rad_tan_thin_prism", 22), ("rig_thin_prism", 18))
    for options, env, path, cam_rel in ((DENSE, (), "dense", 1e-5), (ITER, (), "staged", 1e-5),
                                        (DENSE, (("B200BA_NO_DENSE", "1"),), "staged", EXACT_WIDE_CAM_REL))
]
ALL = NATURAL + BOUNDARY + EXACT + SEAM + WIDE


def _regime(case):
    return regime(_problem(case.problem), case.options, dict(case.env))


def test_every_case_lands_in_its_regime():
    """Host only: every case below runs the path it is named for (the thresholds above, the layout of b200ba_test_pack)."""
    rows, bad, regimes = [], [], [_regime(case) for case in ALL]
    for case, r in zip(ALL, regimes):
        rows.append(f"{case.id:62s} nc {r['nc']:6d}  dkmax {r['dkmax']:2d}  DC {r['DC']:2d}  {r['path']:10s} spmv {r['spmv']}")
        if any(r[k] != v for k, v in case.expect):
            bad.append(f"{case.id}: expected {dict(case.expect)}, got {r}")
    print("\n" + "\n".join(rows))
    assert not bad, "\n".join(bad)
    # every regime of the table is covered
    seen = {(r["path"], r["spmv"]) for r in regimes}
    for want in (("dense", None), ("staged", "smem"), ("staged", "global"), ("mid_smem", "smem"), ("mid_smem", "global"),
                 ("mid_global", "global"), ("mid_global", "smem"), ("multi", "global"), ("multi", "smem")):
        assert want in seen, want
    assert max(r["dkmax"] for r in regimes) > 16


# ---------------------------------------------------------------- the GPU checks
def _set_env(monkeypatch, case):
    for k in SEAMS:
        monkeypatch.delenv(k, raising=False)
    for k, v in case.env:
        monkeypatch.setenv(k, v)


def _msg(sg, sr):
    return (f"gpu cost {sg.initial_cost!r} -> {sg.final_cost!r} ({sg.num_successful_steps}+{sg.num_unsuccessful_steps} steps, "
            f"{sg.num_linear_solver_iterations} PCG) oracle {sr.initial_cost!r} -> {sr.final_cost!r} "
            f"({sr.num_successful_steps}+{sr.num_unsuccessful_steps} steps, {sr.num_linear_solver_iterations} PCG)")


def _groups(a, b):
    g = [(a.poses, b.poses), (a.points, b.points), (a.cam_params, b.cam_params)]
    return g + [(a.sensors, b.sensors)] if len(b.sensors) else g


def _arithmetic(case, iters=3):
    """Same start, same steps: cost to 1e-6, parameters to 1e-5; under ITERATIVE_SCHUR the PCG counts agree."""
    noisy = _problem(case.problem)
    a, sg, b, sr = _both(dataclasses.replace(case.options, max_num_iterations=iters), noisy)
    msg = f"{case.id}: {_msg(sg, sr)}"
    assert sg.num_residuals == sr.num_residuals and sg.num_effective_parameters == sr.num_effective_parameters, msg
    assert sg.linear_solver_type_used == sr.linear_solver_type_used == _regime(case)["lst"], msg
    assert abs(sg.initial_cost - sr.initial_cost) <= 1e-9 * sr.initial_cost, msg
    assert sg.num_successful_steps == sr.num_successful_steps and sg.num_unsuccessful_steps == sr.num_unsuccessful_steps, msg
    assert abs(sg.final_cost - sr.final_cost) <= 1e-6 * sr.final_cost, msg
    for u, v in _groups(a, b):
        rel = case.cam_rel if u is a.cam_params else 1e-5
        err = np.abs(u - v).max()
        assert np.allclose(u, v, rtol=rel, atol=rel * max(1.0, np.abs(v).max())), f"{msg}; max |diff| {err:.3g}"
    lm = sr.num_successful_steps + sr.num_unsuccessful_steps
    if case.options.linear_solver_type == ITERATIVE_SCHUR:
        assert sr.num_linear_solver_iterations > lm, msg
        assert sg.num_linear_solver_iterations == sr.num_linear_solver_iterations, msg
    else:
        _assert_exact_pcg_stops_on_the_residual(case, sg, lm, msg)
    return sg, sr


def _assert_exact_pcg_stops_on_the_residual(case, sg, lm, msg):
    r = _regime(case)
    if r["path"] == "dense":
        assert sg.num_linear_solver_iterations == 0, msg
    else:   # a solve that never reaches the 1e-12 residual runs max_cg iterations on its own, so a total below one max_cg
            # shows that every solve stopped on the residual (the wide rig problems take about 2 nc per solve, the
            # narrow ones less than nc)
        max_cg = max(10 * r["nc"] + 100, case.options.max_linear_solver_iterations)
        assert 0 < sg.num_linear_solver_iterations < max_cg, msg


def _converged(case, iters=10):
    """10 LM iterations at the large-problem bar: cost 1e-5, parameters 1e-4, the same number of LM steps.  A solve
    that reaches the gradient tolerance first sits at the noise floor of the cost, where the GPU's gradient (from
    fp32-stored Jacobians) may stay above the tolerance and take a few more, rejected, steps: the step counts are
    compared where both solves run to the iteration limit."""
    a, sg, b, sr = _both(dataclasses.replace(case.options, max_num_iterations=iters), _problem(case.problem))
    msg = f"{case.id}: {_msg(sg, sr)}"
    if sg.termination_type == sr.termination_type == 1:
        assert sg.num_successful_steps + sg.num_unsuccessful_steps == sr.num_successful_steps + sr.num_unsuccessful_steps, msg
    _assert_parity(a, sg, b, sr, param_rel=1e-4)


@pytest.mark.gpu
def test_pcg_counts_on_the_staged_path():
    """The trusted staged path (the medium problem of test_ba_gpu.py): the GPU and the oracle count the same PCG
    iterations over 1 and 3 LM iterations.  (Over three runs of every ITERATIVE_SCHUR case below the counts were equal
    every time, so every case asserts equality.)"""
    gt, noisy = synthesize_ba_problem(60, 12000, 6, models=(SIMPLE_RADIAL,), seed=21)
    _gauge(noisy)
    for iters in (1, 3):
        a, sg, b, sr = _both(BundleAdjustmentOptions(linear_solver_type=ITERATIVE_SCHUR, max_num_iterations=iters), noisy)
        lm = sr.num_successful_steps + sr.num_unsuccessful_steps
        assert lm == iters and sr.num_linear_solver_iterations > lm, _msg(sg, sr)
        assert sg.num_linear_solver_iterations == sr.num_linear_solver_iterations, _msg(sg, sr)


@pytest.mark.gpu
@pytest.mark.parametrize("case", NATURAL, ids=lambda c: c.id)
def test_natural_size_regimes(case, monkeypatch):
    _set_env(monkeypatch, case)
    _arithmetic(case)
    _converged(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", BOUNDARY, ids=lambda c: c.id)
def test_shared_memory_boundaries(case, monkeypatch):
    _set_env(monkeypatch, case)
    _arithmetic(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", EXACT, ids=lambda c: c.id)
def test_exact_solves(case, monkeypatch):
    """DENSE_/SPARSE_SCHUR: the GPU's dense Cholesky (nc <= 256) or PCG to a 1e-12 relative residual against the
    oracle's dense Cholesky of the explicit reduced matrix.  One LM iteration takes the oracle's step to 5e-6: the GPU
    forms the reduced system from fp32-stored Jacobians (relative rounding 6e-8), and its PCG's SpMV also rounds the
    per-observation intermediate to fp32.  The conditioning of these systems amplifies that to about 5e-7 (dense
    Cholesky) and 2.2e-6 (PCG on the same nc = 256 system) in the pose block of the step."""
    _set_env(monkeypatch, case)
    noisy = _problem(case.problem)
    a, sg, b, sr = _both(dataclasses.replace(case.options, max_num_iterations=1), noisy)
    msg = f"{case.id}: {_msg(sg, sr)}"
    assert sg.linear_solver_type_used == sr.linear_solver_type_used == _regime(case)["lst"], msg
    assert sg.num_successful_steps == sr.num_successful_steps == 1, msg
    _assert_exact_pcg_stops_on_the_residual(case, sg, 1, msg)
    for (u, v), x0 in zip(_groups(a, b), _groups(noisy, noisy)):
        du, dv = u - x0[0], v - x0[0]
        err = np.linalg.norm(du - dv) / np.linalg.norm(dv)
        assert err <= 5e-6, f"{msg}; relative step difference {err:.3g}"
    assert abs(sg.final_cost - sr.final_cost) <= 1e-6 * sr.final_cost, msg
    _arithmetic(case)
    _converged(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", SEAM, ids=lambda c: c.id)
def test_seams(case, monkeypatch):
    _set_env(monkeypatch, case)
    _arithmetic(case)
    if case.problem == "seam_narrow":
        _converged(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", WIDE, ids=lambda c: c.id)
def test_wide_camera_blocks(case, monkeypatch):
    _set_env(monkeypatch, case)
    _arithmetic(case)
