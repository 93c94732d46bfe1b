"""The PatchMatch kernels against the float64 model of the reference (tests/pm_fp64.py), at the shapes, windows and
schedules where kernels go wrong.  Each case stops a run after k sweeps (B200PM_MAX_SWEEPS), first checks that the
partial-run exports (depth, normal, selection probability, cost) are the oracle's partial run bit for bit, then holds
the cost map, the selection probability and the filter decision to the model (the checks of test_pm_fp64_cpu.py)."""
import ctypes
import os

import numpy as np
import pytest

import oracle_pm
import pm_fp64
from colmap_b200.patch_match import PatchMatch, PatchMatchOptions, _f32p
from colmap_b200.synthetic import make_patch_match_scene

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _run_cuda(o, problem, k, env=None):
    """Maps after k sweeps (k < 0: the whole run), original orientation."""
    env = dict(env or {})
    if k >= 0:
        env["B200PM_MAX_SWEEPS"] = k
    old = {name: os.environ.get(name) for name in env}
    os.environ.update({name: str(v) for name, v in env.items()})
    try:
        pm = PatchMatch(o, problem)
        pm.Run()
        h, w, n = pm._dims
        cost = np.empty((n, h, w), np.float32)
        pm._lib.b200pm_debug_get_cost.argtypes = [ctypes.c_void_p, _f32p]
        assert pm._lib.b200pm_debug_get_cost(pm._h, cost.ctypes.data_as(_f32p)) == 0
        out = dict(depth=pm.GetDepthMap(), normal=pm.GetNormalMap(), sel_prob=pm.GetSelProbMap(), cost=cost,
                   mask=pm.GetConsistencyMask())
        pm.close()
    finally:
        for name, v in old.items():
            if v is None:
                os.environ.pop(name, None)
            else:
                os.environ[name] = v
    return out


def _compare(o, prob, k, env=None, messages=False):
    got = _run_cuda(o, prob, k, env)
    ref = oracle_pm.run(o, prob, stop_after_sweeps=k)
    for key in ("depth", "normal", "sel_prob", "cost"):
        eq = _bits(got[key]) == _bits(ref[key])
        assert eq.all(), f"partial run after {k} sweeps: {key} differs from the oracle at {(~eq).sum()} of {eq.size}"
    model = pm_fp64.Model(o, prob)
    st = pm_fp64.check_costs(model, got["depth"], got["normal"], got["cost"])
    if messages and k >= 1:
        before = _run_cuda(o, prob, k - 1, env)
        pm_fp64.check_messages(model, k - 1, before["cost"], got["cost"], before["sel_prob"], got["sel_prob"],
                               (k - 1) / (4.0 * o.num_iterations))
    return st


def _opts(sc, **kw):
    base = dict(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False, num_iterations=1,
                filter=False)
    base.update(kw)
    return PatchMatchOptions(**base)


@pytest.mark.parametrize("r,s", [(1, 2), (1, 1), (3, 2), (5, 1), (14, 1), (20, 1), (20, 2)])
@pytest.mark.parametrize("k", [0, 1])
def test_windows(r, s, k):
    """(14, 1): 841 taps, more than 48 KB of shared memory per CTA; (20, *): the largest window."""
    sc = make_patch_match_scene(48, 36, 3, seed=1)
    _compare(_opts(sc, window_radius=r, window_step=s), sc["problem"], k)


@pytest.mark.parametrize("store", [0, 1])
@pytest.mark.parametrize("prune", [0, 1, 2])
@pytest.mark.parametrize("wpc", [1, 2, 4])
def test_schedules(store, prune, wpc):
    sc = make_patch_match_scene(56, 40, 3, seed=2)
    _compare(_opts(sc), sc["problem"], 2, dict(B200PM_PATCH_STORE=store, B200PM_PRUNE=prune, B200PM_PRUNE_FROM=0,
                                              B200PM_WPC=wpc))


@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_messages_each_frame(k):
    sc = make_patch_match_scene(64, 48, 3, seed=0)
    _compare(_opts(sc), sc["problem"], k, messages=True)


@pytest.mark.parametrize("w,h", [(37, 53), (71, 29)])
def test_ragged_and_portrait_sizes(w, h):
    sc = make_patch_match_scene(w, h, 3, seed=5)
    for k in (1, 2):
        _compare(_opts(sc), sc["problem"], k)


def test_cropped_sources_put_footprints_on_the_apron():
    sc = make_patch_match_scene(64, 48, 3, seed=7)
    for im, (y, x) in zip(sc["images"][1:], [(30, 40), (48, 20), (12, 64)]):
        im.bitmap = np.ascontiguousarray(im.bitmap[:y, :x])
    for k in (0, 1):
        _compare(_opts(sc), sc["problem"], k)


def test_textureless_and_saturated_bands():
    """A flat band in the reference and in one source (variances under kMinVar) and a saturated band."""
    sc = make_patch_match_scene(64, 48, 3, seed=8)
    sc["images"][0].bitmap[10:22, :] = 128
    sc["images"][2].bitmap[:, 20:40] = 90
    sc["images"][1].bitmap[30:40, :] = 255
    for k in (0, 1):
        st = _compare(_opts(sc), sc["problem"], k)
        assert st["decided"] > 0


def test_geometric_mode_with_holes():
    sc = make_patch_match_scene(56, 40, 3, seed=4, with_gt_maps=True)
    prob = sc["problem"]
    rng = np.random.default_rng(2)
    prob.depth_maps = [(d * (1 + 0.01 * rng.standard_normal(d.shape))).astype(np.float32) for d in sc["depth_maps"]]
    for d in prob.depth_maps[1:]:
        d[rng.random(d.shape) < 0.1] = 0.0
    prob.normal_maps = [n.astype(np.float32) for n in sc["normal_maps"]]
    o = _opts(sc, geom_consistency=True)
    for k in (0, 1, 3):
        _compare(o, prob, k)


def test_taps_behind_a_source_camera_at_k0():
    sc = pm_fp64.forward_source(make_patch_match_scene(64, 48, 3, seed=0), 2)
    st = _compare(_opts(sc), sc["problem"], 0)
    assert st["behind"] > 0.1 * st["pairs"] / 3, st


@pytest.mark.parametrize("geom,filter_geom_max", [(False, 1.0), (True, 0.5), (True, 3.0)])
def test_filter_decision(geom, filter_geom_max):
    sc = make_patch_match_scene(56, 40, 4, seed=6, with_gt_maps=geom)
    prob = sc["problem"]
    if geom:
        rng = np.random.default_rng(3)
        prob.depth_maps = [(d * (1 + 0.003 * rng.standard_normal(d.shape))).astype(np.float32) for d in sc["depth_maps"]]
        for d in prob.depth_maps[1:]:
            d[rng.random(d.shape) < 0.05] = 0.0
        prob.normal_maps = [n.astype(np.float32) for n in sc["normal_maps"]]
    o = _opts(sc, geom_consistency=geom, filter=True, filter_geom_consistency_max_cost=filter_geom_max)
    got = _run_cuda(o, prob, -1)
    compared, _ = pm_fp64.check_filter(pm_fp64.Model(o, prob), got["depth"], got["normal"], got["sel_prob"],
                                       got["mask"])
    assert compared > 0 and got["mask"].any()


def test_c2_size_one_sweep_sampled():
    """1920x1080, 8 sources, after one sweep: a seeded sample of 120k (pixel, source) pairs against the model."""
    sc = make_patch_match_scene(1920, 1080, 8, seed=0)
    o = _opts(sc)
    got = _run_cuda(o, sc["problem"], 1)
    rng = np.random.default_rng(0)
    npairs = 120_000
    pix = rng.integers(0, 1920 * 1080, npairs)
    src = rng.integers(0, 8, npairs)
    st = pm_fp64.check_costs(pm_fp64.Model(o, sc["problem"]), got["depth"], got["normal"], got["cost"],
                             sample=(pix, src))
    assert st["pairs"] == npairs
