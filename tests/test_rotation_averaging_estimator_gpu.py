"""RunRotationAveraging end to end on the GPU: the reference's scenarios of rotation_averaging_test.cc through the
Python mirror with the flat solves on the GPU, held to the reference's bars and to the same pipeline with the fp64
oracle behind the _solve_flat hook."""
import copy

import pytest

from colmap_b200.rotation_averaging import RotationAveragingReweighting, RotationEstimatorOptions
from test_rotation_averaging_estimator_cpu import make, max_rotation_error_deg, run

pytestmark = pytest.mark.gpu

SCENARIOS = {   # name: (make arguments, options, bar against the truth in degrees)
    "without_noise": (dict(rigs=1, cams=1, frames=10, seed=1), {}, 1e-2),
    "without_noise_gravity": (dict(rigs=1, cams=1, frames=10, seed=1, gravity=True), dict(use_gravity=True), 1e-2),
    "without_noise_stratified": (dict(rigs=1, cams=1, frames=10, seed=1, gravity=True, gravity_fraction=0.6),
                                 dict(use_gravity=True), 1e-2),
    "weighted_noise_free": (dict(rigs=1, cams=1, frames=10, seed=2),
                            dict(reweighting=RotationAveragingReweighting.INLIER_MATCH_COUNT), 1e-2),
    "known_rig": (dict(rigs=1, cams=2, frames=6, seed=5), {}, 1e-2),
    "unknown_rig": (dict(rigs=1, cams=2, frames=6, seed=6, unknown_rig=True), {}, 1e-2),
    "noise_and_outliers": (dict(rigs=1, cams=1, frames=20, noise=1.0, outliers=0.1, seed=7), {}, 3.0),
    "noise_and_outliers_known_rigs": (dict(rigs=2, cams=2, frames=8, noise=1.0, outliers=0.1, seed=8), {}, 2.0),
}


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_run_rotation_averaging_on_the_gpu(name):
    args, opts, bar = SCENARIOS[name]
    gt, rec, pg, priors = make(**args)
    rec_o, pg_o = copy.deepcopy(rec), copy.deepcopy(pg)
    assert run(RotationEstimatorOptions(gpu_index=0, **opts), pg, rec, priors, estimator=None)
    assert run(RotationEstimatorOptions(**opts), pg_o, rec_o, priors)
    assert max_rotation_error_deg(gt, rec) < bar
    assert max_rotation_error_deg(rec_o, rec) < 1e-6
    assert rec.RegFrameIds() == rec_o.RegFrameIds()
    assert [e.valid for e in pg.Edges().values()] == [e.valid for e in pg_o.Edges().values()]
