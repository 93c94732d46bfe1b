"""GPU tier for the reference-patch store: every pass either copies each pixel's bilateral reference patch from the store
that pm_patch_kernel builds once per run, or builds it inline (B200PM_PATCH_STORE=0, or a store over its budget).  Both
paths must give the same bits in every output, in every sweep frame and serial-pass schedule."""
import os

import numpy as np
import pytest

import oracle_pm
from colmap_b200.patch_match import PatchMatch, PatchMatchOptions
from colmap_b200.synthetic import make_patch_match_scene

pytestmark = pytest.mark.gpu

BUDGET = 3 << 30   # PM_PATCH_STORE_BUDGET in patch_match.cu


def _run(o, problem, store, wpc=None):
    os.environ["B200PM_PATCH_STORE"] = "1" if store else "0"
    if wpc is not None:
        os.environ["B200PM_WPC"] = str(wpc)
    try:
        pm = PatchMatch(o, problem)
        pm.Run()
        out = dict(depth=pm.GetDepthMap(), normal=pm.GetNormalMap(), sel_prob=pm.GetSelProbMap(),
                   store_bytes=pm.patch_store_bytes())
        if o.filter:
            out["mask"] = pm.GetConsistencyMask()
        pm.close()
    finally:
        os.environ.pop("B200PM_PATCH_STORE", None)
        os.environ.pop("B200PM_WPC", None)
    return out


def _assert_same(a, b, keys):
    for k in keys:
        x, y = np.ascontiguousarray(a[k]), np.ascontiguousarray(b[k])
        if x.dtype == np.float32:
            x, y = x.view(np.uint32), y.view(np.uint32)
        eq = x == y
        assert eq.all(), f"{k}: {(~eq).sum()} of {eq.size} values differ"


def _store_bytes(w, h, radius, step):
    ntaps = ((2 * radius) // step + 1) ** 2
    return w * h * (8 * ((ntaps + 1) & ~1) + 16)


@pytest.mark.parametrize("wpc", [1, 2, 4])
def test_store_equals_inline_every_serial_schedule(wpc):
    """Two iterations: all four sweep frames, each with its own tap permutation and weight-sum order, and the filter."""
    sc = make_patch_match_scene(96, 72, 4, seed=0)
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False, num_iterations=2)
    got = _run(o, sc["problem"], True, wpc)
    inl = _run(o, sc["problem"], False, wpc)
    assert got["store_bytes"] == _store_bytes(96, 72, 5, 1) and inl["store_bytes"] == 0
    _assert_same(got, inl, ("depth", "normal", "sel_prob", "mask"))
    ref = oracle_pm.run(o, sc["problem"])
    _assert_same(got, ref, ("depth", "normal", "sel_prob", "mask"))


@pytest.mark.parametrize("w,h,n,radius,step", [
    (64, 80, 8, 4, 2),     # window step 2, odd tap count (25): the stored blocks carry one padding tap
    (64, 48, 3, 5, 2),     # window step 2, even tap count (36)
    (30, 24, 2, 14, 1),    # 841 taps: more than 48 KB of dynamic shared memory in the pixel pass
])
def test_store_equals_inline_window_grid(w, h, n, radius, step):
    sc = make_patch_match_scene(w, h, n, seed=11)
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                          num_iterations=1, window_radius=radius, window_step=step)
    got = _run(o, sc["problem"], True, 1)
    inl = _run(o, sc["problem"], False, 1)
    assert got["store_bytes"] == _store_bytes(w, h, radius, step)
    _assert_same(got, inl, ("depth", "normal", "sel_prob", "mask"))


def test_store_equals_inline_mixed_source_sizes():
    sc = make_patch_match_scene(80, 60, 3, seed=2)
    img = sc["images"][2]
    img.bitmap = np.ascontiguousarray(img.bitmap[:50, :70])
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                          num_iterations=1, filter=False)
    for wpc in (1, 2):
        got = _run(o, sc["problem"], True, wpc)
        inl = _run(o, sc["problem"], False, wpc)
        assert got["store_bytes"] > 0
        _assert_same(got, inl, ("depth", "normal", "sel_prob"))


def test_store_equals_inline_geometric():
    sc = make_patch_match_scene(80, 60, 4, seed=4, with_gt_maps=True)
    prob = sc["problem"]
    rng = np.random.default_rng(0)
    prob.depth_maps = [(d * (1 + 0.002 * rng.standard_normal(d.shape))).astype(np.float32) for d in sc["depth_maps"]]
    prob.normal_maps = [n.copy() for n in sc["normal_maps"]]
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=True, num_iterations=1)
    for wpc in (1, 2, 4):
        got = _run(o, prob, True, wpc)
        inl = _run(o, prob, False, wpc)
        assert got["store_bytes"] > 0
        _assert_same(got, inl, ("depth", "normal", "sel_prob", "mask"))


def test_over_budget_takes_the_inline_path():
    """Radius 20 (1681 taps, 13.5 KB per pixel) at 640x400 needs more than the budget: no store, and the run completes."""
    w, h = 640, 400
    assert _store_bytes(w, h, 20, 1) > BUDGET
    sc = make_patch_match_scene(w, h, 2, seed=5)
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                          num_iterations=1, window_radius=20, window_step=1, filter=False)
    got = _run(o, sc["problem"], True)
    assert got["store_bytes"] == 0
    assert np.isfinite(got["depth"]).all() and (got["depth"] > 0).mean() > 0.9
