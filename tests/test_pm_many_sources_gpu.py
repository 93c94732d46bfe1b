"""PatchMatch with 9 to 32 source images, the source counts of the C4 workspace (20 sources per reference image), held
to the oracle bit for bit.  Above N = 8 the sweep runs code that N <= 8 never reaches:
  * the pixel pass is pm_pixel_kernel (pm_pixel4_kernel only takes N <= 8): its 3 N pair loop, the sentinel fill over
    3 N entries, nmask (N = 31 by the shift, N = 32 the full-warp case), the multiplicity key over 32 lanes and the
    geometric costs of lanes 8..31;
  * the sequential-shuffle branches of pm_cdf_lanes and pm_sample_image;
  * the serial pass's phase B over more images than groups, tab1[32], the sampled / m2..m4 masks and evaluate() on
    images >= 8, and the filter's vote over up to 32 lanes against filter_min_num_consistent;
  * the per-image offset tables (quad_off, depth_off, pitch) past image 8, with mixed source sizes and geometric maps;
  * the [pixel][N] exports and the consistency list with more than 8 images.
Every case compares depth, normal, selection probability and, where the filter runs, the consistency mask and
GetConsistentImageIdxs with the oracle, bit for bit.  The schedules, the pruned tab3 invariant, passes R and M, the
fp64 model of the reference and a C4-shaped two-phase run are covered at N = 20 and N = 32."""
import os

import numpy as np
import pytest

import oracle_pm
import pm_fp64
from colmap_b200.patch_match import PatchMatch, PatchMatchOptions, consistency_list_from_mask
from colmap_b200.synthetic import make_patch_match_scene, make_workspace_scene
from test_pm_fp64_gpu import _compare
from test_pm_pixel_pool_gpu import _check_invariant
from test_pm_rand_msg_gpu import _assert_same, _rand_msg

pytestmark = pytest.mark.gpu

_KNOBS = ("B200PM_WPC", "B200PM_PRUNE", "B200PM_PRUNE_FROM", "B200PM_PATCH_STORE", "B200PM_MAX_SWEEPS")


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _scene(w, h, n, seed, geom=False, crops=(), shuffle=False):
    """make_patch_match_scene with, optionally: geometric maps from the perturbed ground truth with holes in the source
    maps (as the geom case of test_pm_fp64_cpu.py), sources cropped ((source lane, height, width): the principal point
    stays), and src_image_idxs in shuffled order.  Returns (scene, problem)."""
    sc = make_patch_match_scene(w, h, n, seed=seed, with_gt_maps=geom)
    prob = sc["problem"]
    if geom:
        rng = np.random.default_rng(seed + 1000)
        prob.depth_maps = [(d * (1 + 0.01 * rng.standard_normal(d.shape))).astype(np.float32) for d in sc["depth_maps"]]
        for d in prob.depth_maps[1:]:
            d[rng.random(d.shape) < 0.1] = 0.0
        prob.normal_maps = [nm.astype(np.float32) for nm in sc["normal_maps"]]
    for lane, ch, cw in crops:
        k = prob.src_image_idxs[lane]
        sc["images"][k].bitmap = np.ascontiguousarray(sc["images"][k].bitmap[:ch, :cw])
        if geom:
            prob.depth_maps[k] = np.ascontiguousarray(prob.depth_maps[k][:ch, :cw])
    if shuffle:
        prob.src_image_idxs = [int(i) for i in np.random.default_rng(seed).permutation(prob.src_image_idxs)]
    return sc, prob


def _opts(sc, **kw):
    base = dict(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False, num_iterations=1)
    base.update(kw)
    return PatchMatchOptions(**base)


def _run_cuda(o, problem, env=None):
    """Whole run with exactly the given schedule knobs set (None: unset); the environment is restored afterwards."""
    old = {name: os.environ.get(name) for name in _KNOBS}
    for name in _KNOBS:
        os.environ.pop(name, None)
    os.environ.update({name: str(v) for name, v in (env or {}).items() if v is not None})
    try:
        pm = PatchMatch(o, problem)
        pm.Run()
        out = dict(depth=pm.GetDepthMap(), normal=pm.GetNormalMap(), sel_prob=pm.GetSelProbMap(),
                   store_bytes=pm.patch_store_bytes())
        if o.filter:
            out["mask"] = pm.GetConsistencyMask()
            out["list"] = pm.GetConsistentImageIdxs()
        pm.close()
    finally:
        for name, v in old.items():
            if v is None:
                os.environ.pop(name, None)
            else:
                os.environ[name] = v
    return out


_ORACLE = {}


def _oracle(key, o, problem):
    """oracle_pm.run, once per case key (the schedule cases share one oracle run per scene)."""
    if key not in _ORACLE:
        _ORACLE[key] = oracle_pm.run(o, problem)
    return _ORACLE[key]


def _assert_exact(got, ref, problem, what=""):
    for key in ("depth", "normal", "sel_prob"):
        eq = _bits(got[key]) == _bits(ref[key])
        assert eq.all(), f"{what}{key}: {(~eq).sum()} of {eq.size} values differ, first at {np.argwhere(~eq)[:4].tolist()}"
    if "mask" in got:
        diff = got["mask"] != ref["mask"]
        assert not diff.any(), f"{what}mask: {diff.sum()} entries differ, first at {np.argwhere(diff)[:4].tolist()}"
        assert np.array_equal(got["list"], consistency_list_from_mask(ref["mask"], problem.src_image_idxs)), \
            f"{what}consistency list"


# ---------------------------------------------------------------- 1. source counts
@pytest.mark.parametrize("n,w,h", [
    (9, 45, 37), (12, 53, 41), (16, 43, 58), (20, 57, 39), (24, 41, 47),
    (31, 50, 43),   # the largest N whose image mask is computed by the shift
    (32, 55, 42),   # the full-warp image mask
])
def test_source_count_grid(n, w, h):
    """Two iterations, so all four sweep frames run twice, with the default filter."""
    sc, prob = _scene(w, h, n, seed=100 + n)
    o = _opts(sc, num_iterations=2)
    got = _run_cuda(o, prob)
    _assert_exact(got, oracle_pm.run(o, prob), prob)
    assert (got["depth"] > 0).mean() > 0.5


# ---------------------------------------------------------------- 2. schedules
def _schedule_case(n, geom):
    sc, prob = _scene(47, 38, n, seed=7 + n, geom=geom)
    o = _opts(sc, geom_consistency=geom, num_iterations=2)
    return o, prob, _oracle(("schedule", n, geom), o, prob)


@pytest.mark.parametrize("prune,prune_from", [(0, 0), (1, 0), (1, 3), (2, 0)])
@pytest.mark.parametrize("store", [0, 1])
@pytest.mark.parametrize("n", [20, 32])
def test_schedules(n, store, prune, prune_from):
    """Serial-pass warps per column 1, 2, 4 and automatic, every pixel-pass early-out schedule (PRUNE_FROM = 3: the
    first three sweeps unpruned, the other five pruned), with and without the reference-patch store."""
    o, prob, ref = _schedule_case(n, False)
    for wpc in (1, 2, 4, None):
        env = dict(B200PM_WPC=wpc, B200PM_PRUNE=prune, B200PM_PRUNE_FROM=prune_from, B200PM_PATCH_STORE=store)
        got = _run_cuda(o, prob, env)
        _assert_exact(got, ref, prob, f"{env}: ")
        assert (got["store_bytes"] > 0) == bool(store)


@pytest.mark.parametrize("prune", [1, 2])
@pytest.mark.parametrize("n", [20, 32])
def test_schedules_geometric(n, prune):
    o, prob, ref = _schedule_case(n, True)
    for wpc in (1, 2, 4, None):
        env = dict(B200PM_WPC=wpc, B200PM_PRUNE=prune, B200PM_PRUNE_FROM=0)
        _assert_exact(_run_cuda(o, prob, env), ref, prob, f"{env}: ")


# ---------------------------------------------------------------- 3. options
@pytest.mark.parametrize("ns", [1, 15, 40])   # 40: more samples than lanes, the serial pass's second block of 32
@pytest.mark.parametrize("n", [20, 32])
def test_num_samples(n, ns):
    sc, prob = _scene(46, 39, n, seed=20 + n + ns)
    o = _opts(sc, num_samples=ns, num_iterations=2)
    _assert_exact(_run_cuda(o, prob), oracle_pm.run(o, prob), prob)


@pytest.mark.parametrize("n,r,s", [
    (20, 1, 1), (20, 5, 2),
    (20, 20, 1), (32, 20, 1),   # 1681 taps: the pixel and serial passes' dynamic shared memory is above 48 KB
])
def test_windows(n, r, s):
    sc, prob = _scene(43, 35, n, seed=30 + n + r)
    o = _opts(sc, window_radius=r, window_step=s)
    _assert_exact(_run_cuda(o, prob), oracle_pm.run(o, prob), prob)


# sources 8, 11, 15 and 19 (and 27 at N = 32) cropped to four different sizes, smaller and narrower than the reference:
# their quad tables, pitches and depth maps sit at offsets only images past the eighth have
_CROPS = ((8, 30, 35), (11, 41, 29), (15, 22, 47), (19, 33, 33), (27, 41, 40))


@pytest.mark.parametrize("geom", [False, True])
@pytest.mark.parametrize("n", [20, 32])
def test_mixed_source_sizes(n, geom):
    sc, prob = _scene(47, 41, n, seed=40 + n, geom=geom, crops=[c for c in _CROPS if c[0] < n])
    o = _opts(sc, geom_consistency=geom, num_iterations=2)
    _assert_exact(_run_cuda(o, prob), oracle_pm.run(o, prob), prob)


@pytest.mark.parametrize("n", [12, 20, 32])
def test_geometric_with_holes(n):
    sc, prob = _scene(49, 37, n, seed=50 + n, geom=True)
    o = _opts(sc, geom_consistency=True, num_iterations=2, num_samples=21)
    _assert_exact(_run_cuda(o, prob), oracle_pm.run(o, prob), prob)


# ---------------------------------------------------------------- 4. a filter that decides
@pytest.mark.parametrize("geom", [False, True])
@pytest.mark.parametrize("n,seed,min_consistent", [(20, 3, 13), (32, 5, 16), (12, 4, 6)])
def test_filter_that_decides(n, seed, min_consistent, geom):
    """A 9-degree triangulation threshold and a vote near the middle: the filter zeroes a sizeable share of the pixels,
    and among the sources past the eighth some are mostly consistent and some mostly not.  src_image_idxs are shuffled,
    so the consistency list's global indices are not the lane order.  At N = 20 the decision is also held to the fp64
    model of the reference."""
    sc, prob = _scene(48, 36, n, seed=seed, geom=geom, shuffle=True)
    o = _opts(sc, geom_consistency=geom, filter_min_triangulation_angle=9, filter_min_num_consistent=min_consistent)
    got = _run_cuda(o, prob)
    _assert_exact(got, oracle_pm.run(o, prob), prob)
    kept = got["depth"] > 0
    assert 0.1 < 1 - kept.mean() < 0.9, f"{1 - kept.mean():.3f} of the pixels zeroed"
    frac = got["mask"][:, kept].mean(axis=1)
    assert (frac[8:] > 0.5).any() and (frac[8:] < 0.5).any(), np.round(frac, 2).tolist()
    assert (got["mask"][:, kept].sum(axis=0) >= min_consistent).all()
    if n == 20:
        compared, _ = pm_fp64.check_filter(pm_fp64.Model(o, prob), got["depth"], got["normal"], got["sel_prob"],
                                           got["mask"])
        assert compared > 0


# ---------------------------------------------------------------- 5. pruned pixel pass
@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("n,w,h", [(20, 45, 34), (32, 39, 41)])
def test_pruned_tab3_is_sentinel_or_exact(n, w, h, k):
    """Every tab3 entry the pruned pixel pass left is PM_NOT_EVALUATED or the unpruned run's entry, bit for bit, and
    the pruned pass does skip entries."""
    sc, prob = _scene(w, h, n, seed=60 + n)
    o = _opts(sc, window_radius=2, num_samples=11)
    _check_invariant(o, prob, k)


# ---------------------------------------------------------------- 6. passes R and M
@pytest.mark.parametrize("k", [0, 1, 2, 3])
@pytest.mark.parametrize("n,ns,geom", [(20, 15, False), (32, 15, False), (32, 40, False), (20, 9, True)])
def test_rand_msg_bit_exact_vs_column_serial(n, ns, geom, k):
    sc, prob = _scene(37, 45, n, seed=70 + n, geom=geom)
    host, gpu, _ = _rand_msg(_opts(sc, geom_consistency=geom, window_radius=2, num_samples=ns), prob, k)
    _assert_same(host, gpu)


# ---------------------------------------------------------------- 7. the fp64 model of the reference
@pytest.mark.parametrize("k", [1, 2])
def test_fp64_costs_and_messages_at_20_sources(k):
    """After k sweeps the partial run is the oracle's bit for bit (cost map included), every (pixel, source) cost is the
    fp64 NCC of the pixel's hypothesis within its fp32 bound, and sweep k's selection probability follows from the
    messages."""
    sc, prob = _scene(48, 36, 20, seed=80)
    st = _compare(_opts(sc, filter=False), prob, k, messages=True)
    assert st["pairs"] == 20 * 48 * 36


def test_fp64_costs_geometric_at_20_sources():
    sc, prob = _scene(48, 36, 20, seed=81, geom=True)
    st = _compare(_opts(sc, geom_consistency=True, filter=False), prob, 1)
    assert st["pairs"] == 20 * 48 * 36


# ---------------------------------------------------------------- 8. C4-shaped two-phase run
def test_c4_shaped_two_phase_run_equals_the_oracle():
    """22 views of one scene, each with its 20 nearest views as sources (chosen as bench.py's C4 leg does), photometric
    then geometric phase with the filter.  The resident path (device-to-device exports, maps handed over as device
    pointers) gives each image's final depth and normal maps bit for bit as the same schedule run by the oracle."""
    import torch
    from colmap_b200.workspace import run_two_phase
    sc = make_workspace_scene(48, 36, 22, seed=7)
    cen = sc["centers"]
    srcs = []
    for i in range(len(cen)):
        order = np.argsort(np.linalg.norm(cen - cen[i], axis=1), kind="stable")
        srcs.append([int(j) for j in order if j != i][:20])
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=True, window_radius=5,
                          num_samples=15, num_iterations=1, gpu_index="0")

    def oracle_runner(opt, problem):
        out = oracle_pm.run(opt, problem)
        return out["depth"], out["normal"]

    dev = run_two_phase(sc["images"], srcs, o, 0, 1, device=torch.device("cuda", 0))
    ref = run_two_phase(sc["images"], srcs, o, 0, 1, runner=oracle_runner)
    assert sorted(dev) == sorted(ref) == list(range(22))
    for i in range(22):
        for m, name in ((0, "depth"), (1, "normal")):
            eq = _bits(dev[i][m]) == _bits(ref[i][m])
            assert eq.all(), f"image {i}: {name} differs at {(~eq).sum()} of {eq.size}"
        assert (dev[i][0] > 0).mean() > 0.5, f"image {i}: {(dev[i][0] > 0).mean():.3f} of the pixels kept"
