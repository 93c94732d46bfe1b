"""ctypes driver of the guided SIFT matching CPU oracle (tests/sm_guided_oracle.c).  Test infrastructure.

The oracle is compiled on first use into a per-user temporary directory keyed by the hash of its source, so the
repository tree is never written.  Rays and Jacobians are inputs: `geo` builds them with the library's
CamRayFromImgWithJac, which the CPU tests hold to finite differences on its own."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(_ROOT, "tests", "sm_guided_oracle.c")
_LIB = None
_u8p = ctypes.POINTER(ctypes.c_uint8)
_u32p = ctypes.POINTER(ctypes.c_uint32)
_f32p = ctypes.POINTER(ctypes.c_float)
_f64p = ctypes.POINTER(ctypes.c_double)

NONE, E, F, H = 0, 1, 2, 3


def lib():
    global _LIB
    if _LIB is None:
        with open(_SRC, "rb") as f:
            digest = hashlib.sha256(f.read()).hexdigest()[:16]
        out_dir = os.path.join(tempfile.gettempdir(), f"colmap_b200_oracle_{os.getuid()}")
        os.makedirs(out_dir, exist_ok=True)
        path = os.path.join(out_dir, f"sm_guided_oracle_{digest}.so")
        if not os.path.exists(path):
            tmp = path + f".{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-o", tmp, _SRC,
                                   "-lm"])
            os.replace(tmp, path)
        L = ctypes.CDLL(path)
        L.smg_oracle_match.argtypes = [_u8p, ctypes.c_int64, _u8p, ctypes.c_int64, _f32p, _f32p, _f64p, _f64p,
                                       ctypes.c_int, _f64p, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                       ctypes.c_int, ctypes.c_int64, _u32p]
        L.smg_oracle_match.restype = ctypes.c_int64
        _LIB = L
    return _LIB


def geo(camera, xy):
    """(n, 10) float64 rows: ray, row-major 3 x 2 Jacobian, 1 for a valid ray (0 and zeros where the reference's
    CamRayFromImgWithJac returns nullopt)."""
    from colmap_b200.feature_matching import CamRayFromImgWithJac
    xy = np.asarray(xy, np.float32).reshape(-1, 2)
    out = np.zeros((len(xy), 10), np.float64)
    for k, p in enumerate(xy.astype(np.float64)):
        r = CamRayFromImgWithJac(camera, p)
        if r is not None:
            out[k, :3], out[k, 3:9], out[k, 9] = r[0], r[1].ravel(), 1.0
    return out


def match(desc1, desc2, xy1, xy2, type, M, max_error, geo1=None, geo2=None, max_ratio=0.8, max_distance=0.7,
          cross_check=True, max_num_matches=32768):
    """Guided matches under filter `type` (E, F, H or NONE) with the 3 x 3 matrix M; (k, 2) uint32."""
    a = np.ascontiguousarray(desc1, np.uint8).reshape(-1, 128)
    b = np.ascontiguousarray(desc2, np.uint8).reshape(-1, 128)
    k1 = np.ascontiguousarray(np.asarray(xy1, np.float32).reshape(len(a), 2))
    k2 = np.ascontiguousarray(np.asarray(xy2, np.float32).reshape(len(b), 2))
    g1 = np.ascontiguousarray(geo1 if geo1 is not None else np.zeros((len(a), 10)), np.float64)
    g2 = np.ascontiguousarray(geo2 if geo2 is not None else np.zeros((len(b), 10)), np.float64)
    m = np.ascontiguousarray(np.zeros(9) if M is None else np.asarray(M, np.float64).reshape(9))
    n1, n2 = min(len(a), max_num_matches), min(len(b), max_num_matches)
    out = np.zeros((max(min(n1, n2) if cross_check else n1, 1), 2), np.uint32)
    k = lib().smg_oracle_match(a.ctypes.data_as(_u8p), len(a), b.ctypes.data_as(_u8p), len(b), k1.ctypes.data_as(_f32p),
                               k2.ctypes.data_as(_f32p), g1.ctypes.data_as(_f64p), g2.ctypes.data_as(_f64p), int(type),
                               m.ctypes.data_as(_f64p), float(max_error), max_ratio, max_distance,
                               1 if cross_check else 0, max_num_matches, out.ctypes.data_as(_u32p))
    if k < 0:
        raise MemoryError("smg_oracle_match")
    return out[:k].copy()
