"""ctypes driver of the pose-prior CPU oracle (tests/ba_prior_oracle.c).  Test infrastructure.

The oracle is compiled on first use into a per-user temporary directory keyed by the hash of its sources, so the
repository tree is never written."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from colmap_b200.bundle_adjustment import BundleAdjustmentSummary, _COptions, _CPositionPriors, _CProblem, _CSummary, _f64p

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(_ROOT, "tests", "ba_prior_oracle.c")
_DEPS = [_SRC, os.path.join(_ROOT, "oracle", "ba_oracle.c"), os.path.join(_ROOT, "include", "b200_bundle_adjustment.h"),
         os.path.join(_ROOT, "include", "b200_ba_pose_prior.h")]
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        h = hashlib.sha256()
        for d in _DEPS:
            with open(d, "rb") as f:
                h.update(f.read())
        out_dir = os.path.join(tempfile.gettempdir(), f"colmap_b200_oracle_{os.getuid()}")
        os.makedirs(out_dir, exist_ok=True)
        path = os.path.join(out_dir, f"ba_prior_oracle_{h.hexdigest()[:16]}.so")
        if not os.path.exists(path):
            tmp = path + f".{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-O2", "-fopenmp", "-shared", "-fPIC", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, path)
        L = ctypes.CDLL(path)
        L.ba_oracle_solve_with_position_priors.argtypes = [ctypes.POINTER(_COptions), ctypes.POINTER(_CProblem),
                                                           ctypes.POINTER(_CPositionPriors), ctypes.POINTER(_CSummary)]
        L.ba_oracle_prior_position.argtypes = [_f64p, _f64p, _f64p, _f64p, _f64p, _f64p]
        L.ba_oracle_prior_position.restype = None
        _LIB = L
    return _LIB


def solve(options, flat, priors):
    """Runs the oracle on `flat` in place with `priors` (FlatPositionPriors); returns BundleAdjustmentSummary."""
    co, cp, cpr, cs = options.to_c(), flat.to_c(), priors.to_c(), _CSummary()
    rc = lib().ba_oracle_solve_with_position_priors(ctypes.byref(co), ctypes.byref(cp), ctypes.byref(cpr), ctypes.byref(cs))
    if rc != 0:
        raise RuntimeError(f"ba_oracle_solve_with_position_priors -> {rc}")
    return BundleAdjustmentSummary.from_c(cs)


def prior_position(rig, sensor, position):
    """ba_oracle_prior_position: residual (3) and tangent Jacobians (3x6) of the rig and sensor blocks."""
    d = lambda a: np.ascontiguousarray(a, np.float64)
    rig, position = d(rig), d(position)
    sp = d(sensor).ctypes.data_as(_f64p) if sensor is not None else None
    res, Jr, Js = np.zeros(3), np.zeros((3, 6)), np.zeros((3, 6))
    lib().ba_oracle_prior_position(rig.ctypes.data_as(_f64p), sp, position.ctypes.data_as(_f64p), res.ctypes.data_as(_f64p),
                                   Jr.ctypes.data_as(_f64p), Js.ctypes.data_as(_f64p))
    return res, Jr, Js
