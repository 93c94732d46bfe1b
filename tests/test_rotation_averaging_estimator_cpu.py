"""RotationEstimator / RunRotationAveraging on the Python mirror without a GPU: the reference's scenarios of
rotation_averaging_test.cc solved with the fp64 oracle behind the estimator's _solve_flat hook, with the reference's
bars, and the data-model additions they rely on (PoseGraph edges, PosePrior gravity, registered frames)."""
import copy

import numpy as np
import pytest

import ra_oracle
from colmap_b200.bundle_adjustment import PosePrior, Reconstruction, _quat_to_R
from colmap_b200.global_positioning import PoseGraph, PoseGraphEdge
from colmap_b200.rotation_averaging import (InitializeRigRotationsFromImages, RotationAveragingReweighting,
                                            RotationEstimator, RotationEstimatorOptions, RunRotationAveraging,
                                            _R_to_aa)
from colmap_b200.synthetic import synthesize_pose_graph, synthesize_rig_reconstruction


class OracleEstimator(RotationEstimator):
    def _solve_flat(self, flat):
        return ra_oracle.solve(self.options_, flat)


def make(rigs, cams, frames, noise=0.0, outliers=0.0, seed=0, gravity=False, unknown_rig=False, gravity_fraction=1.0):
    """(gt, rec, pose_graph, priors): rec is gt with every frame pose unknown (and, with unknown_rig, every non-reference
    cam_from_rig unknown)."""
    gt = synthesize_rig_reconstruction(rigs, cams, frames, 10, seed=seed)
    pg, priors = synthesize_pose_graph(gt, noise, outliers, seed=seed + 1, gravity=gravity)
    priors = priors[:int(round(gravity_fraction * len(priors)))]
    rec = copy.deepcopy(gt)
    for fr in rec.frames.values():
        fr.rig_from_world = None
    if unknown_rig:
        for rig in rec.rigs.values():
            for c in rig.sensors:
                rig.sensors[c] = None
    return gt, rec, pg, priors


def max_rotation_error_deg(gt, rec):
    """ExpectEqualRotations: the largest angle between estimated and true relative rotations R_i R_0^T of all images."""
    ids = sorted(gt.images)
    Rg = {i: _quat_to_R(gt.images[i].cam_from_world[:4]) for i in ids}
    Re = {i: _quat_to_R(rec.images[i].cam_from_world[:4]) for i in ids}
    i0 = ids[0]
    err = 0.0
    for i in ids:
        D = (Re[i] @ Re[i0].T).T @ (Rg[i] @ Rg[i0].T)
        err = max(err, np.degrees(np.linalg.norm(_R_to_aa(D))))
    return err


def run(options, pg, rec, priors, estimator=OracleEstimator):
    """RunRotationAveraging with the oracle behind the hook (estimator=None: the GPU solve)."""
    return RunRotationAveraging(options, pg, rec, priors, estimator=estimator or RotationEstimator)


@pytest.mark.parametrize("use_gravity,fraction", [(False, 1.0), (True, 1.0), (True, 0.6)])
def test_without_noise(use_gravity, fraction):
    """fraction 0.6: gravity priors on part of the frames, so the stratified 1-DOF subset solve runs first."""
    gt, rec, pg, priors = make(1, 1, 10, seed=1, gravity=use_gravity, gravity_fraction=fraction)
    assert run(RotationEstimatorOptions(use_gravity=use_gravity), pg, rec, priors)
    assert max_rotation_error_deg(gt, rec) < 1e-2
    assert sorted(rec.RegFrameIds()) == sorted(rec.frames)


def test_weighted_noise_free_matches_invariant():
    gt, rec, pg, priors = make(1, 1, 10, seed=2)
    rec2, pg2 = copy.deepcopy(rec), copy.deepcopy(pg)
    assert run(RotationEstimatorOptions(), pg, rec, priors)
    assert run(RotationEstimatorOptions(reweighting=RotationAveragingReweighting.INLIER_MATCH_COUNT), pg2, rec2, priors)
    assert max_rotation_error_deg(gt, rec) < 1e-2 and max_rotation_error_deg(gt, rec2) < 1e-2
    assert max_rotation_error_deg(rec, rec2) < 1e-2


def test_weighted_reduces_error_with_noisy_low_match_edges():
    gt, rec, pg, priors = make(1, 1, 12, noise=0.2, seed=3)
    rng = np.random.default_rng(4)
    for (i1, i2), e in pg.Edges().items():
        if rng.uniform() < 0.3:
            n = rng.normal(0, np.radians(8.0), 3)
            from colmap_b200.synthetic import _exp_so3
            from colmap_b200.rotation_averaging import _R_to_quat
            e.cam2_from_cam1[:4] = _R_to_quat(_exp_so3(n)[0] @ _quat_to_R(e.cam2_from_cam1[:4]))
            e.num_matches = 20
        else:
            e.num_matches = 500
    rec2, pg2 = copy.deepcopy(rec), copy.deepcopy(pg)
    o = RotationEstimatorOptions(max_rotation_error_deg=0)
    assert run(o, pg, rec, priors)
    assert run(RotationEstimatorOptions(max_rotation_error_deg=0, reweighting=RotationAveragingReweighting.INLIER_MATCH_COUNT),
               pg2, rec2, priors)
    assert max_rotation_error_deg(gt, rec2) < max_rotation_error_deg(gt, rec)


def test_without_noise_with_non_trivial_known_rig():
    gt, rec, pg, priors = make(1, 2, 6, seed=5)
    assert run(RotationEstimatorOptions(), pg, rec, priors)
    assert max_rotation_error_deg(gt, rec) < 1e-2


def test_without_noise_with_non_trivial_unknown_rig():
    gt, rec, pg, priors = make(1, 2, 6, seed=6, unknown_rig=True)
    assert run(RotationEstimatorOptions(), pg, rec, priors)
    assert max_rotation_error_deg(gt, rec) < 1e-2
    for c, T in rec.rigs[1].sensors.items():
        D = _quat_to_R(T[:4]).T @ _quat_to_R(gt.rigs[1].sensors[c][:4])
        assert np.degrees(np.linalg.norm(_R_to_aa(D))) < 1e-2
        assert np.isnan(T[4:]).all()


def test_with_noise_and_outliers():
    gt, rec, pg, priors = make(1, 1, 20, noise=1.0, outliers=0.1, seed=7)
    assert run(RotationEstimatorOptions(), pg, rec, priors)
    assert max_rotation_error_deg(gt, rec) < 3.0


def test_with_noise_and_outliers_with_non_trivial_known_rigs():
    gt, rec, pg, priors = make(2, 2, 8, noise=1.0, outliers=0.1, seed=8)
    assert run(RotationEstimatorOptions(), pg, rec, priors)
    assert max_rotation_error_deg(gt, rec) < 2.0


def test_ridge_regularization_does_not_bias_solution():
    gt, rec, pg, priors = make(1, 1, 10, seed=9)
    rec2, pg2 = copy.deepcopy(rec), copy.deepcopy(pg)
    assert run(RotationEstimatorOptions(ridge_regularization=0.0), pg, rec, priors)
    assert run(RotationEstimatorOptions(ridge_regularization=1e-9), pg2, rec2, priors)
    assert max_rotation_error_deg(rec, rec2) < 1e-6


def test_empty_pose_graph():
    gt, rec, _, priors = make(1, 1, 5, seed=10)
    assert not run(RotationEstimatorOptions(), PoseGraph(), rec, priors)


def test_gravity_with_unknown_rig_sensors_returns_false():
    """Through RotationEstimator directly, as the reference's test does: RunRotationAveraging takes the expanded path
    for unknown rig sensors, whose singleton rigs pass the calibration check."""
    gt, rec, pg, priors = make(1, 2, 4, seed=11, gravity=True, unknown_rig=True)
    before = copy.deepcopy(rec)
    assert not OracleEstimator(RotationEstimatorOptions(use_gravity=True)).EstimateRotations(pg, priors, set(rec.images), rec)
    assert all(fr.rig_from_world is None for fr in rec.frames.values()) and rec.rigs[1].sensors == before.rigs[1].sensors


def test_multi_image_rig_frame_deregister_does_not_crash_on_second_visit():
    gt, rec, pg, priors = make(1, 2, 4, seed=12)
    isolated = max(rec.frames)
    iso_images = {i for i, im in rec.images.items() if im.frame_id == isolated}
    for i1, i2 in list(pg.Edges()):
        if i1 in iso_images or i2 in iso_images:
            pg.DeleteEdge(i1, i2)
    rec.frames[isolated].rig_from_world = gt.frames[isolated].rig_from_world.copy()
    rec.RegisterFrame(isolated)
    assert run(RotationEstimatorOptions(max_rotation_error_deg=1.0), pg, rec, priors)
    assert rec.frames[isolated].rig_from_world is None and isolated not in rec.RegFrameIds()
    for f in sorted(rec.frames)[:-1]:
        assert rec.frames[f].rig_from_world is not None and f in rec.RegFrameIds()


def test_relative_rotation_filter_invalidates_outlier_edges():
    gt, rec, pg, priors = make(1, 1, 12, noise=0.5, outliers=0.1, seed=13)
    assert run(RotationEstimatorOptions(max_rotation_error_deg=5.0), pg, rec, priors)
    bad = [k for k, e in pg.Edges().items() if not e.valid]
    assert bad, "the outlier edges are invalidated"


def test_initialize_rig_rotations_from_images():
    gt, rec, _, _ = make(1, 3, 4, seed=14, unknown_rig=True)
    cams = {i: _quat_to_R(im.cam_from_world[:4]) for i, im in gt.images.items()}
    assert InitializeRigRotationsFromImages(cams, rec, True)
    for c, T in rec.rigs[1].sensors.items():
        D = _quat_to_R(T[:4]).T @ _quat_to_R(gt.rigs[1].sensors[c][:4])
        assert np.linalg.norm(_R_to_aa(D)) < 1e-12
    for f, fr in rec.frames.items():
        D = _quat_to_R(fr.rig_from_world[:4]).T @ _quat_to_R(gt.frames[f].rig_from_world[:4])
        assert np.linalg.norm(_R_to_aa(D)) < 1e-12


def test_data_model_additions_keep_old_behaviour():
    pg = PoseGraph(edges=[(1, 2), (2, 3)])
    assert pg.ValidEdges() == [(1, 2), (2, 3)]
    pg.AddEdge(5, 4, PoseGraphEdge(np.array([0.0, 0.0, np.sin(0.1), np.cos(0.1), 1.0, 0.0, 0.0]), 7))
    assert (4, 5) in pg.Edges() and pg.Edges()[(4, 5)].num_matches == 7
    assert np.allclose(pg.GetEdge(5, 4).cam2_from_cam1[:4], [0.0, 0.0, np.sin(0.1), np.cos(0.1)])
    pg.SetInvalidEdge(2, 1)
    assert pg.ValidEdges() == [(2, 3), (4, 5)]
    assert not PosePrior(1).HasGravity() and PosePrior(1, gravity=np.array([0.0, 1.0, 0.0])).HasGravity()
    rec = Reconstruction()
    assert rec.RegFrameIds() == []
