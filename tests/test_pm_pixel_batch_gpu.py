"""The pixel pass in batches of four pixels per warp (pm_pixel4_kernel, N <= 8): set-up of the four pixels on all 32
lanes, four split reference patches per warp, NCC rounds pixel after pixel.  Every case is compared bit for bit with
the oracle: source counts on both sides of the N <= 8 limit (N = 9 runs pm_pixel_kernel), frames whose pixel count is
not a multiple of four (the last batch of every sweep is partial) and frames one pixel wide or high (every batch
straddles rows), every early-out schedule, geometric mode, a step-2 window, and the largest windows on the inline
patch build (radius 20 with step 2 runs the batched kernel, with step 1 its four split patches do not fit a CTA and
pm_pixel_kernel runs)."""
import os

import numpy as np
import pytest

import oracle_pm
from colmap_b200.patch_match import PatchMatch, PatchMatchOptions
from colmap_b200.synthetic import make_patch_match_scene

pytestmark = pytest.mark.gpu


def _run(o, problem, env):
    for k, v in env.items():
        os.environ[k] = str(v)
    try:
        pm = PatchMatch(o, problem)
        pm.Run()
        out = dict(depth=pm.GetDepthMap(), normal=pm.GetNormalMap(), sel_prob=pm.GetSelProbMap())
        if o.filter:
            out["mask"] = pm.GetConsistencyMask()
        pm.close()
    finally:
        for k in env:
            os.environ.pop(k, None)
    return out


def _assert_bit_exact(got, ref):
    for k in ("depth", "normal", "sel_prob"):
        eq = np.ascontiguousarray(got[k], np.float32).view(np.uint32) == np.ascontiguousarray(ref[k], np.float32).view(np.uint32)
        assert eq.all(), f"{k}: {(~eq).sum()} of {eq.size} values differ"
    if "mask" in got:
        assert np.array_equal(got["mask"], ref["mask"])


SCHEDULES = [dict(B200PM_PRUNE=0), dict(B200PM_PRUNE=1), dict(B200PM_PRUNE=2),
             dict(B200PM_PRUNE=1, B200PM_PRUNE_FROM=0), dict(B200PM_PRUNE=1, B200PM_PRUNE_FROM=3)]


@pytest.mark.parametrize("w,h,n", [
    (37, 29, 1),   # 1073 pixels: one pixel in the last batch
    (30, 27, 3),   # 810 pixels: two
    (23, 21, 8),   # 483 pixels: three; N = 8 fills every lane of a segment
    (22, 19, 9),   # N = 9: pm_pixel_kernel
])
def test_source_counts_partial_batches_every_schedule(w, h, n):
    sc = make_patch_match_scene(w, h, n, seed=31 + n)
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                          num_iterations=1, window_radius=2, window_step=1, num_samples=11)
    ref = oracle_pm.run(o, sc["problem"])
    for env in SCHEDULES:
        _assert_bit_exact(_run(o, sc["problem"], env), ref)


@pytest.mark.parametrize("w,h", [(1, 23), (19, 1)])
def test_one_pixel_wide_frame(w, h):
    """Frames 1 and 3 (or 0 and 2) walk one-pixel rows: every batch of four spans four rows."""
    sc = make_patch_match_scene(w, h, 3, seed=7)
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                          num_iterations=1, window_radius=2, window_step=1, num_samples=9)
    ref = oracle_pm.run(o, sc["problem"])
    for env in SCHEDULES[:3]:
        _assert_bit_exact(_run(o, sc["problem"], env), ref)


def test_geometric_mode_partial_batches():
    sc = make_patch_match_scene(35, 26, 4, seed=9, with_gt_maps=True)
    prob = sc["problem"]
    rng = np.random.default_rng(3)
    prob.depth_maps = [(d * (1 + 0.002 * rng.standard_normal(d.shape))).astype(np.float32) for d in sc["depth_maps"]]
    prob.normal_maps = [nm.copy() for nm in sc["normal_maps"]]
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=True,
                          num_iterations=1, window_radius=2, window_step=1, num_samples=9)
    ref = oracle_pm.run(o, prob)
    for env in SCHEDULES[:3]:
        _assert_bit_exact(_run(o, prob, env), ref)


def test_window_step_2():
    sc = make_patch_match_scene(33, 25, 5, seed=12)
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                          num_iterations=1, window_radius=4, window_step=2, num_samples=9)
    ref = oracle_pm.run(o, sc["problem"])
    for store in (1, 0):
        _assert_bit_exact(_run(o, sc["problem"], dict(B200PM_PATCH_STORE=store)), ref)


@pytest.mark.parametrize("step", [2, 1])
def test_radius_20_inline_patch(step):
    sc = make_patch_match_scene(27, 21, 2, seed=5)
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                          num_iterations=1, window_radius=20, window_step=step, num_samples=5)
    ref = oracle_pm.run(o, sc["problem"])
    _assert_bit_exact(_run(o, sc["problem"], dict(B200PM_PATCH_STORE=0)), ref)
