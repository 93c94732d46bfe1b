"""Host side of b200ba_estimate_covariance_with_position_priors: the exports of b200_ba_covariance.h, and the refusal of bad
priors before any device work (on a machine without a GPU the call still reaches the prior checks, which come first)."""
import ctypes
import os
import re

import numpy as np
import pytest

from colmap_b200 import load_library
from colmap_b200.bundle_adjustment import (BACovarianceOptions, BundleAdjustmentError, BundleAdjustmentOptions,
                                           FlatPositionPriors, estimate_covariance_flat)
from colmap_b200.synthetic import synthesize_ba_problem

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_covariance_symbol():
    lib = load_library()
    hdr = open(os.path.join(ROOT, "include", "b200_ba_covariance.h")).read()
    names = set(re.findall(r"\b(b200ba_[a-z_0-9]+)\s*\(", hdr))
    assert "b200ba_estimate_covariance_with_position_priors" in names and "b200ba_estimate_covariance" in names
    for n in names:
        assert hasattr(lib, n), n


def _priors(flat, **change):
    n = len(flat.poses)
    pos = np.array([-flat.poses[i, 4:] for i in range(n)])
    cov = np.repeat(0.01 * np.eye(3)[None], n, axis=0)
    pose_idx, sensor_idx = np.arange(n), -np.ones(n)
    k = change.get("at", 1)
    if "position" in change:
        pos[k] = change["position"]
    if "covariance" in change:
        cov[k] = change["covariance"]
    if "pose_idx" in change:
        pose_idx[k] = change["pose_idx"]
    if "sensor_idx" in change:
        sensor_idx[k] = change["sensor_idx"]
    return FlatPositionPriors(pose_idx, sensor_idx, pos, cov)


@pytest.mark.parametrize("change,message", [
    (dict(covariance=np.diag([1.0, -1.0, 1.0])), "prior 1: covariance is not symmetric positive definite"),
    (dict(covariance=np.array([[1.0, 0.5, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])), "prior 1: covariance is not symmetric"),
    (dict(covariance=np.full((3, 3), np.inf)), "prior 1: covariance is not finite"),
    (dict(position=[0.0, np.nan, 0.0]), "prior 1: position is not finite"),
    (dict(pose_idx=99), "prior 1: pose_idx out of range"),
    (dict(pose_idx=-1), "prior 1: pose_idx out of range"),
    (dict(sensor_idx=0), "prior 1: sensor_idx out of range"),
])
def test_bad_priors_refused_before_device_work(change, message):
    _, flat = synthesize_ba_problem(6, 150, 4, seed=7)
    with pytest.raises(BundleAdjustmentError, match=r"b200ba_estimate_covariance_with_position_priors failed \(-2\): " + re.escape(message)):
        estimate_covariance_flat(BundleAdjustmentOptions(), BACovarianceOptions(), flat, priors=_priors(flat, **change))


def test_bad_prior_loss_refused():
    _, flat = synthesize_ba_problem(6, 150, 4, seed=7)
    pr = _priors(flat)
    pr.loss_function_type = 99
    with pytest.raises(BundleAdjustmentError, match="unknown prior loss function type"):
        estimate_covariance_flat(BundleAdjustmentOptions(), BACovarianceOptions(), flat, priors=pr)
