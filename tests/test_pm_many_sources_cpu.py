"""The 32-source limit of the PatchMatch path, on both sides: the library's problem check (b200pm_check, reached through
PatchMatch.Check) accepts 32 source images and refuses 33 with its message, and the oracle refuses 33 as well, so a
GPU comparison above the limit cannot pass by both sides quietly doing something.  The oracle's consistency decision at
N = 20, with a filter that keeps some sources and drops others, is held to the fp64 model of the reference.  No GPU
needed: nothing here creates a handle."""
import numpy as np
import pytest

import oracle_pm
import pm_fp64
from colmap_b200.patch_match import PatchMatch, PatchMatchError, PatchMatchOptions
from colmap_b200.synthetic import make_patch_match_scene


def _opts(sc, **kw):
    return PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                             num_iterations=1, **kw)


def test_check_accepts_32_sources_and_refuses_33():
    sc = make_patch_match_scene(14, 11, 33, seed=0)
    prob = sc["problem"]
    prob.src_image_idxs = list(range(1, 33))
    PatchMatch(_opts(sc), prob).Check()
    prob.src_image_idxs = list(range(1, 34))
    with pytest.raises(PatchMatchError, match="more than 32 source images are not supported"):
        PatchMatch(_opts(sc), prob).Check()


def test_oracle_runs_32_sources_and_refuses_33():
    sc = make_patch_match_scene(14, 11, 33, seed=1)
    prob = sc["problem"]
    o = _opts(sc, window_radius=2)
    prob.src_image_idxs = list(range(1, 33))
    out = oracle_pm.run(o, prob)
    assert out["sel_prob"].shape == (32, 11, 14) and np.isfinite(out["sel_prob"]).all()
    prob.src_image_idxs = list(range(1, 34))
    with pytest.raises(RuntimeError, match=r"pm_oracle_run_partial -> -1"):
        oracle_pm.run(o, prob)


def test_oracle_filter_decision_at_20_sources_is_the_fp64_one():
    """filter_min_triangulation_angle = 9 and 13 of 20 sources required: about a quarter of the pixels are zeroed and
    the sources with index >= 8 split into mostly consistent and mostly not; every mask entry is the fp64 decision."""
    sc = make_patch_match_scene(48, 36, 20, seed=3)
    o = _opts(sc, filter_min_triangulation_angle=9, filter_min_num_consistent=13)
    out = oracle_pm.run(o, sc["problem"])
    kept = out["depth"] > 0
    assert 0.1 < 1 - kept.mean() < 0.9
    frac = out["mask"][:, kept].mean(axis=1)
    assert (frac[8:] > 0.5).any() and (frac[8:] < 0.5).any()
    compared, _ = pm_fp64.check_filter(pm_fp64.Model(o, sc["problem"]), out["depth"], out["normal"], out["sel_prob"],
                                       out["mask"])
    assert compared > 0
