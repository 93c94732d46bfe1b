"""The pixel pass's pooled rounds (pm_pixel4_kernel, N <= 8): the four group slots of a round take pairs of any of the
batch's four pixels, so a result that lands in the wrong pixel's tab3 row, or a wrong hypothesis or image, can be
masked in the final maps when the serial pass re-evaluates the entry or the entry loses anyway.  The invariant checked
here sees it: a run stopped after k sweeps (B200PM_MAX_SWEEPS) under the pruned schedule and under B200PM_PRUNE=0
starts its last sweep from the same state (the maps are bit-exact whatever the pixel pass evaluates), so every tab3
entry of the pruned run is either PM_NOT_EVALUATED or bit-equal to the unpruned run's entry.  N = 9 runs
pm_pixel_kernel, where the same invariant holds.  A bit-exact oracle case covers batches that only pooling makes
different: pixels that are done early next to a pixel that runs long, and one pixel extending a surviving hypothesis to
every image."""
import ctypes
import os

import numpy as np
import pytest

import oracle_pm
from colmap_b200.patch_match import PatchMatch, PatchMatchOptions, _f32p
from colmap_b200.synthetic import make_patch_match_scene

pytestmark = pytest.mark.gpu

NOT_EVALUATED = np.float32(-1.0)


def _run(o, problem, env):
    """Run with the given environment; returns (depth, normal, sel_prob, tab3 [pixel][3][N] of the last sweep)."""
    for k, v in env.items():
        os.environ[k] = str(v)
    try:
        pm = PatchMatch(o, problem)
        pm.Run()
        n = len(problem.src_image_idxs)
        h, w = problem.images[problem.ref_image_idx].bitmap.shape[:2]
        tab3 = np.empty((h * w, 3, n), np.float32)
        pm._lib.b200pm_debug_get_tab3.argtypes = [ctypes.c_void_p, _f32p]
        assert pm._lib.b200pm_debug_get_tab3(pm._h, tab3.ctypes.data_as(_f32p)) == 0
        out = dict(depth=pm.GetDepthMap(), normal=pm.GetNormalMap(), sel_prob=pm.GetSelProbMap(), tab3=tab3)
        pm.close()
    finally:
        for k in env:
            os.environ.pop(k, None)
    return out


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _check_invariant(o, problem, k, min_real=0.05):
    pruned = _run(o, problem, dict(B200PM_MAX_SWEEPS=k, B200PM_PRUNE=1))
    full = _run(o, problem, dict(B200PM_MAX_SWEEPS=k, B200PM_PRUNE=0))
    for key in ("depth", "normal", "sel_prob"):   # the same state: the premise of the comparison below
        assert np.array_equal(_bits(pruned[key]), _bits(full[key])), key
    t, ref = pruned["tab3"], full["tab3"]
    assert not (ref == NOT_EVALUATED).any(), "the unpruned pixel pass left an entry out"
    skipped = t == NOT_EVALUATED
    wrong = ~skipped & (_bits(t) != _bits(ref))
    assert not wrong.any(), f"{wrong.sum()} evaluated tab3 entries differ, first at {np.argwhere(wrong)[:4].tolist()}"
    real = (~skipped).mean()
    assert real >= min_real, f"only {real:.3f} of the entries were evaluated: the check is close to vacuous"
    if t.shape[2] > 1:   # (one image: every hypothesis takes its one image, nothing is left out)
        assert skipped.any(), "the pruned pixel pass evaluated every entry: nothing was pruned"
    return pruned


@pytest.mark.parametrize("k", [2, 3])   # the last sweep walks frame 1 (columns of H rows), then frame 2
@pytest.mark.parametrize("w,h,n", [
    (37, 29, 1),   # 1073 pixels: one pixel in the last batch
    (30, 27, 3),   # 810 pixels: two
    (23, 21, 8),   # 483 pixels: three
    (22, 19, 9),   # N = 9: pm_pixel_kernel
    (1, 23, 3),    # one pixel wide: every batch of frames 0 and 2 spans four rows
])
def test_pruned_tab3_is_sentinel_or_exact(w, h, n, k):
    sc = make_patch_match_scene(w, h, n, seed=40 + n + w)
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                          num_iterations=1, window_radius=2, window_step=1, num_samples=11)
    _check_invariant(o, sc["problem"], k)


@pytest.mark.parametrize("k", [2, 3])
def test_pruned_tab3_geometric(k):
    sc = make_patch_match_scene(35, 26, 4, seed=9, with_gt_maps=True)
    prob = sc["problem"]
    rng = np.random.default_rng(5)
    prob.depth_maps = [(d * (1 + 0.002 * rng.standard_normal(d.shape))).astype(np.float32) for d in sc["depth_maps"]]
    prob.normal_maps = [nm.copy() for nm in sc["normal_maps"]]
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=True,
                          num_iterations=1, window_radius=2, window_step=1, num_samples=9)
    _check_invariant(o, prob, k)


def _batches(tab3, w0, h0, rot):
    """tab3 rows in the sweep order of frame `rot`, cut into the pixel pass's batches of four (the tail dropped)."""
    fw, fh = (h0, w0) if rot & 1 else (w0, h0)
    q = np.arange(fw * fh)
    r, c = q // fw, q % fw
    if rot == 0:
        r0, c0 = r, c
    elif rot == 1:
        r0, c0 = c, w0 - 1 - r
    elif rot == 2:
        r0, c0 = h0 - 1 - r, w0 - 1 - c
    else:
        r0, c0 = h0 - 1 - c, r
    t = tab3[r0 * w0 + c0]
    nb = len(q) // 4
    return t[:4 * nb].reshape(nb, 4, 3, -1)


def _assert_bit_exact(got, ref):
    for key in ("depth", "normal", "sel_prob"):
        eq = _bits(got[key]) == _bits(ref[key])
        assert eq.all(), f"{key}: {(~eq).sum()} of {eq.size} values differ"


def test_batches_of_mixed_lengths_bit_exact():
    """A whole run (four sweeps) against the oracle, on a scene whose last sweep has batches where a pixel is done
    after at most one image per hypothesis while another pixel of the batch evaluates a hypothesis on every image, and
    batches where exactly one pixel extends a survivor to every image.  (A pixel that samples no image starts its
    batch with no hypothesis left, as does a position past the frame's end in the partial batches above.)"""
    w, h, n = 41, 33, 8
    sc = make_patch_match_scene(w, h, n, seed=77)
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                          num_iterations=1, window_radius=2, window_step=1, num_samples=5)
    got = _run(o, sc["problem"], {})
    _assert_bit_exact(got, oracle_pm.run(o, sc["problem"]))
    b = _batches(got["tab3"], w, h, 3)
    ev = (b != NOT_EVALUATED)
    nev = ev.sum(axis=(2, 3))                  # [batch][pixel] entries evaluated
    full_row = ev.all(axis=3).any(axis=2)      # [batch][pixel] a hypothesis evaluated on every image
    mixed = ((nev <= 3).any(axis=1) & full_row.any(axis=1)).sum()
    lone = (full_row.sum(axis=1) == 1).sum()
    assert mixed > 0, f"no batch with a short pixel next to a long one ({(nev <= 3).sum()} short pixels)"
    assert lone > 0, f"no batch where exactly one pixel extends a hypothesis to every image ({full_row.sum()} such pixels)"
