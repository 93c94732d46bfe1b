"""Global positioning on the GPU against the fp64 oracle (tests/gp_oracle.py) from identical initial states: the cost
of every iteration, the final parameters, determinism, and the reference's scenarios end to end."""
import itertools

import numpy as np
import pytest

import gp_oracle
from colmap_b200.global_positioning import GlobalPositioner, GlobalPositionerOptions, PoseGraph, solve_flat
from colmap_b200.synthetic import synthesize_global_positioning, synthesize_rig_reconstruction
from test_global_positioning_cpu import OraclePositioner, centers, scenario, similarity_error

pytestmark = pytest.mark.gpu


def flat_of(rigs, cams, frames, seed=0, nan_sensor=False, prior_focal=(), points=200):
    rec = synthesize_rig_reconstruction(rigs, cams, frames, points, seed=seed, point2D_stddev=0.5)
    for fr in rec.frames.values():
        fr.rig_from_world[4:] = 0.0
    if nan_sensor:
        for rig in rec.rigs.values():
            for v in rig.sensors.values():
                v[4:] = np.nan
    GlobalPositioner._sync_image_poses(rec)
    for c in prior_focal:
        rec.cameras[c].has_prior_focal_length = True
    pos = OraclePositioner(GlobalPositionerOptions(random_seed=seed, max_num_iterations=0))
    pos.Solve(PoseGraph(), rec)
    return pos.flat_problem


def compare(flat, opts, iters=40, rtol_cost=1e-8, rtol_par=1e-6):
    opts.max_num_iterations = iters
    g, r = flat.copy(), flat.copy()
    sg = solve_flat(opts, g)
    sr = gp_oracle.solve(r, iters, opts.optimize_positions, opts.optimize_points, opts.optimize_scales)
    assert sg.termination_type == sr.termination_type
    assert len(sg.cost_history) == len(sr.cost_history), (sg.cost_history, sr.cost_history)
    # relative, with a floor at fp64 rounding of the initial cost
    tol = rtol_cost * np.abs(sr.cost_history) + 1e-14 * sr.cost_history[0]
    assert np.all(np.abs(sg.cost_history - sr.cost_history) <= tol), \
        np.abs(sg.cost_history - sr.cost_history) / sr.cost_history
    assert (sg.num_successful_steps, sg.num_unsuccessful_steps) == (sr.num_successful_steps, sr.num_unsuccessful_steps)
    for a, b in ((g.frame_centers, r.frame_centers), (g.points, r.points), (g.cams_in_rig, r.cams_in_rig), (g.obs_scale, r.obs_scale)):
        if b.size:
            assert np.abs(a - b).max() <= rtol_par * max(1.0, np.abs(b).max())
    return sg, g


@pytest.mark.parametrize("pos,pts,scl", list(itertools.product([True, False], repeat=3)))
def test_optimize_flags(pos, pts, scl):
    compare(flat_of(1, 1, 8), GlobalPositionerOptions(optimize_positions=pos, optimize_points=pts, optimize_scales=scl))


def test_constant_rig_and_mixed_calibration():
    compare(flat_of(2, 3, 4, prior_focal=(1, 5)), GlobalPositionerOptions())


def test_variable_rig():
    f = flat_of(2, 3, 4, nan_sensor=True, seed=2)
    assert len(f.cams_in_rig) == 4
    compare(f, GlobalPositionerOptions())


def test_scale_bound_active():
    f = flat_of(1, 1, 6, seed=4)
    f.obs_ray[1::7] *= -1.0   # rays pointing away: their scales are pushed to the bound
    f.obs_scale[1::7] = 2e-5
    s, g = compare(f, GlobalPositionerOptions())
    assert np.any(g.obs_scale == 1e-5)


def test_no_reduced_system():
    f = flat_of(1, 1, 6)
    s, _ = compare(f, GlobalPositionerOptions(optimize_positions=False))
    assert s.reduced_dim == 0


def test_medium_case_and_determinism():
    f = flat_of(1, 1, 30, points=1000, seed=5)
    s, g = compare(f, GlobalPositionerOptions(), iters=10)
    g2 = f.copy()
    solve_flat(GlobalPositionerOptions(max_num_iterations=10), g2)
    for a, b in ((g.frame_centers, g2.frame_centers), (g.points, g2.points), (g.obs_scale, g2.obs_scale)):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


def test_large_reduced_system():
    """1,000 frames (n = 3,000: 47 tiles of the dense factorisation and the triangular solves, the reduced size of the
    timed 2.1M-observation case), first 10 iterations.  The tracks are 30,000 points x 7 views: the full-normal-equation
    oracle needs about two minutes per iteration at 2.1M observations, so the observation count is a tenth of that."""
    f = synthesize_global_positioning(1000, 30000, 210000, seed=11)
    s, _ = compare(f, GlobalPositionerOptions(), iters=10)
    assert s.reduced_dim == 3000
    assert s.num_successful_steps >= 5 and s.final_cost < 1e-2 * s.initial_cost


@pytest.mark.parametrize("frames,dim", [(21, 63), (22, 66), (64, 192), (65, 195)])
def test_reduced_system_at_tile_edges(frames, dim):
    """Reduced sizes around the 64-row tile of the dense factorisation and triangular solves: one padding row (63),
    three rows into the second tile (66), exactly three tiles without padding (192), one row past them (195)."""
    f = synthesize_global_positioning(frames, 300, 2100, seed=frames)
    s, _ = compare(f, GlobalPositionerOptions())
    assert s.reduced_dim == dim


def test_variable_rig_sensors_in_a_later_tile():
    """2 rigs x 3 cameras x 30 frames: the 60 frame blocks fill rows 0-179 (tiles 0 to 2) and the 4 variable
    camera-in-rig blocks, after the frames, rows 180-191 of tile 2, so most of each sensor's frames lie in other tiles."""
    f = flat_of(2, 3, 30, nan_sensor=True, seed=3, points=60)
    assert len(f.cams_in_rig) == 4
    s, _ = compare(f, GlobalPositionerOptions())
    assert s.reduced_dim == 192


@pytest.mark.parametrize("rigs,cams,frames,refine", [(1, 1, 10, True), (2, 3, 5, True), (2, 3, 5, False)],
                         ids=["Nominal", "MultiCameraRig", "RefineSensorFromRigFalsePreservesRig"])
def test_reference_scenarios(rigs, cams, frames, refine):
    gt, rec, pg = scenario(rigs, cams, frames)
    snap = {(r, c): v.copy() for r, rig in rec.rigs.items() for c, v in rig.sensors.items()}
    pos = GlobalPositioner(GlobalPositionerOptions(random_seed=42, refine_sensor_from_rig=refine))
    assert pos.Solve(pg, rec)
    assert similarity_error(centers(rec), centers(gt)) < 0.5
    if not refine:
        for (r, c), v in snap.items():
            assert np.array_equal(rec.rigs[r].sensors[c].view(np.uint64), v.view(np.uint64))
