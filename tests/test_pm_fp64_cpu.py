"""The PatchMatch oracle (oracle/pm_oracle.c) against the float64 model of the reference (tests/pm_fp64.py).

The oracle is bit-identical to the CUDA kernels (tests/test_pm_gpu.py), so this is where what both compute is tied to
the reference's definition: costs after k sweeps within an fp32 error bound per pair, the selection probability of one
sweep from its three input maps, and the filter decision of the last sweep.  Each check is also run against
deliberately wrong readings of the reference and must reject every one of them.  No GPU needed."""
import numpy as np
import pytest

import oracle_pm
import pm_fp64
from colmap_b200.patch_match import PatchMatchOptions
from colmap_b200.synthetic import make_patch_match_scene


def _case(name):
    """(options, problem) of the named case."""
    if name == "forward":    # one source camera on the optical axis: hypotheses nearer than it lie behind it
        sc = pm_fp64.forward_source(make_patch_match_scene(64, 48, 3, seed=0), 2)
        return PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                                 num_iterations=1, filter=False), sc["problem"]
    if name == "geom":       # geometric mode from a perturbed ground truth, with holes in the source depth maps
        sc = make_patch_match_scene(56, 40, 3, seed=4, with_gt_maps=True)
        prob = sc["problem"]
        rng = np.random.default_rng(2)
        prob.depth_maps = [(d * (1 + 0.01 * rng.standard_normal(d.shape))).astype(np.float32) for d in sc["depth_maps"]]
        for d in prob.depth_maps[1:]:
            d[rng.random(d.shape) < 0.1] = 0.0
        prob.normal_maps = [n.astype(np.float32) for n in sc["normal_maps"]]
        return PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=True,
                                 num_iterations=1, filter=False), prob
    r, s = dict(r5s1=(5, 1), r3s2=(3, 2))[name]
    sc = make_patch_match_scene(64, 48, 3, seed=0)
    return PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=False,
                             num_iterations=1, filter=False, window_radius=r, window_step=s), sc["problem"]


_RUNS = {}


def _run(name, k):
    if (name, k) not in _RUNS:
        o, prob = _case(name)
        _RUNS[(name, k)] = oracle_pm.run(o, prob, stop_after_sweeps=k)
    return _RUNS[(name, k)]


def _check_costs(name, k, variant=None):
    o, prob = _case(name)
    out = _run(name, k)
    return pm_fp64.check_costs(pm_fp64.Model(o, prob, variant), out["depth"], out["normal"], out["cost"])


def _check_messages(name, k, variant=None):
    o, prob = _case(name)
    a, b = _run(name, k - 1), _run(name, k)
    return pm_fp64.check_messages(pm_fp64.Model(o, prob, variant), k - 1, a["cost"], b["cost"], a["sel_prob"],
                                  b["sel_prob"], (k - 1) / (4.0 * o.num_iterations))


@pytest.mark.parametrize("k", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("name", ["r5s1", "r3s2"])
def test_cost_map_is_the_fp64_ncc_after_k_sweeps(name, k):
    """After the initial cost (k = 0) and after one sweep in each frame, every (pixel, source) cost is the NCC of the
    pixel's current hypothesis, within its fp32 bound; frames 1-3 run in rotated buffers, the model does not."""
    st = _check_costs(name, k)
    assert st["pairs"] == 3 * 64 * 48


@pytest.mark.parametrize("k", [0, 2])
def test_geometric_mode_cost_map_holds_the_photometric_term(k):
    _check_costs("geom", k)


def test_taps_behind_a_source_camera_sample_its_mirror_image():
    """k = 0 with a source camera in front of the reference: about a third of its pairs have taps behind it."""
    st = _check_costs("forward", 0)
    assert st["behind"] > 0.1 * st["pairs"] / 3, st


@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_selection_probability_follows_from_the_messages(k):
    _check_messages("r5s1", k)


def _filter_case(geom, filter_geom_max):
    sc = make_patch_match_scene(56, 40, 4, seed=6, with_gt_maps=geom)
    prob = sc["problem"]
    if geom:
        rng = np.random.default_rng(3)
        prob.depth_maps = [(d * (1 + 0.003 * rng.standard_normal(d.shape))).astype(np.float32) for d in sc["depth_maps"]]
        for d in prob.depth_maps[1:]:
            d[rng.random(d.shape) < 0.05] = 0.0
        prob.normal_maps = [n.astype(np.float32) for n in sc["normal_maps"]]
    o = PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=geom,
                          num_iterations=1, filter=True, filter_geom_consistency_max_cost=filter_geom_max)
    return o, prob


@pytest.mark.parametrize("geom,filter_geom_max", [(False, 1.0), (True, 0.5), (True, 1.0), (True, 3.0)])
def test_consistency_mask_is_the_fp64_filter_decision(geom, filter_geom_max):
    o, prob = _filter_case(geom, filter_geom_max)
    out = oracle_pm.run(o, prob)
    model = pm_fp64.Model(o, prob)
    compared, _ = pm_fp64.check_filter(model, out["depth"], out["normal"], out["sel_prob"], out["mask"])
    assert compared > 0 and out["mask"].any()
    if geom and filter_geom_max < o.geom_consistency_max_cost:
        # the geometric test decides both ways: some pairs pass every other test and fail on it
        H, W = out["depth"].shape
        rows, cols = pm_fp64.pixel_grid(H, W)
        kept = out["depth"].ravel() != 0
        fails = 0
        for i in range(model.N):
            t = model.filter_terms(i, rows[kept], cols[kept], out["depth"].ravel()[kept].astype(np.float64),
                                   out["normal"].reshape(3, -1).T[kept].astype(np.float64),
                                   out["sel_prob"][i].ravel()[kept])
            fails += int(((t["tri"] >= 0) & (t["inc"] > 0) & (t["ncc"] >= 0) & (t["geom"] < 0)).sum())
        assert fails > 0


@pytest.mark.parametrize("variant,check", [
    (pm_fp64.Variant(texel_shift=0.5), ("r5s1", 1, "costs")),
    (pm_fp64.Variant(sigma_spatial_plus1=True), ("r5s1", 1, "costs")),
    (pm_fp64.Variant(grid_start_plus1=True), ("r3s2", 1, "costs")),
    (pm_fp64.Variant(behind_camera_border=True), ("forward", 0, "costs")),
    (pm_fp64.Variant(swap_change=True), ("r5s1", 1, "messages")),
    (pm_fp64.Variant(backward_reversed_frame=1), ("r5s1", 2, "messages")),
], ids=["texel_centre", "sigma_spatial", "step2_grid", "behind_camera_border", "swapped_change", "backward_frame1"])
def test_wrong_model_variants_are_rejected(variant, check):
    """A tolerance loose enough to let any of these readings of the reference through would be too loose."""
    name, k, what = check
    with pytest.raises(AssertionError):
        (_check_costs if what == "costs" else _check_messages)(name, k, variant)
