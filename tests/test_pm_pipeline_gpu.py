"""Edges of the pipelined NCC tap loop (pm_ncc_group: each lane walks its own taps sub, sub + 8, ... with the next
taps' gathers in flight, the look-ahead clamped to the lane's last tap).  Every case is compared bit for bit with the
oracle: tap counts below the pipeline depth, lanes without taps, no ragged tail, the largest window on the inline
patch build, every pixel-pass early-out schedule, geometric mode, and source images of other sizes whose footprints
are clamped at the zero apron."""
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


@pytest.mark.parametrize("radius,step", [
    (1, 2),   # 4 taps: half the lanes of a group have none, the others one (fewer than the pipeline depth)
    (1, 1),   # 9 taps: one full round of 8 and a tail of one
    (3, 2),   # 16 taps: two full rounds, no tail
])
def test_small_windows_every_early_out_schedule(radius, step):
    sc = make_patch_match_scene(56, 44, 3, seed=21)
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                          num_iterations=1, window_radius=radius, window_step=step, num_samples=9)
    ref = oracle_pm.run(o, sc["problem"])
    for prune in (0, 1, 2):
        _assert_bit_exact(_run(o, sc["problem"], dict(B200PM_PRUNE=prune)), ref)


def test_radius_20_inline_patch():
    """1681 taps (210 full rounds and a tail of one) with the reference patch built inline in every pass."""
    sc = make_patch_match_scene(26, 22, 2, seed=5)
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                          num_iterations=1, window_radius=20, window_step=1, num_samples=5)
    ref = oracle_pm.run(o, sc["problem"])
    _assert_bit_exact(_run(o, sc["problem"], dict(B200PM_PATCH_STORE=0)), ref)


def test_geometric_mode_small_window():
    sc = make_patch_match_scene(48, 40, 3, seed=8, with_gt_maps=True)
    prob = sc["problem"]
    rng = np.random.default_rng(2)
    prob.depth_maps = [(d * (1 + 0.002 * rng.standard_normal(d.shape))).astype(np.float32) for d in sc["depth_maps"]]
    prob.normal_maps = [n.copy() for n in sc["normal_maps"]]
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=True,
                          num_iterations=1, window_radius=1, window_step=1, num_samples=9)
    ref = oracle_pm.run(o, prob)
    _assert_bit_exact(_run(o, prob, {}), ref)


def test_mixed_source_sizes_footprints_at_the_apron():
    """Two source images cropped well inside the reference's view: many footprints leave the image and are clamped
    onto the zero apron, on both patch paths."""
    sc = make_patch_match_scene(64, 48, 3, seed=13)
    sc["images"][1].bitmap = np.ascontiguousarray(sc["images"][1].bitmap[:30, :41])
    sc["images"][3].bitmap = np.ascontiguousarray(sc["images"][3].bitmap[:47, :22])
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                          num_iterations=2, window_radius=3, window_step=1, num_samples=9)
    ref = oracle_pm.run(o, sc["problem"])
    for store in (1, 0):
        _assert_bit_exact(_run(o, sc["problem"], dict(B200PM_PATCH_STORE=store)), ref)
