"""ctypes driver of the SIFT matching CPU oracle (tests/sm_oracle.c).  Test infrastructure.

The oracle is compiled on first use into a per-user temporary directory keyed by the hash of its source, so the
repository tree is never written."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(_ROOT, "tests", "sm_oracle.c")
_LIB = None
_u8p = ctypes.POINTER(ctypes.c_uint8)
_u32p = ctypes.POINTER(ctypes.c_uint32)


def lib():
    global _LIB
    if _LIB is None:
        with open(_SRC, "rb") as f:
            digest = hashlib.sha256(f.read()).hexdigest()[:16]
        out_dir = os.path.join(tempfile.gettempdir(), f"colmap_b200_oracle_{os.getuid()}")
        os.makedirs(out_dir, exist_ok=True)
        path = os.path.join(out_dir, f"sm_oracle_{digest}.so")
        if not os.path.exists(path):
            tmp = path + f".{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, path)
        L = ctypes.CDLL(path)
        L.sm_oracle_match.argtypes = [_u8p, ctypes.c_int64, _u8p, ctypes.c_int64, ctypes.c_double, ctypes.c_double,
                                      ctypes.c_int, ctypes.c_int64, _u32p]
        L.sm_oracle_match.restype = ctypes.c_int64
        _LIB = L
    return _LIB


def _desc(d):
    d = np.ascontiguousarray(d, dtype=np.uint8).reshape(-1, 128)
    return d, d.ctypes.data_as(_u8p)


def match(desc1, desc2, max_ratio=0.8, max_distance=0.7, cross_check=True, max_num_matches=32768):
    """FindBestMatchesBruteForce on the first max_num_matches rows of each image; (k, 2) uint32 matches."""
    a, pa = _desc(desc1)
    b, pb = _desc(desc2)
    n1, n2 = min(len(a), max_num_matches), min(len(b), max_num_matches)
    out = np.zeros((max(min(n1, n2) if cross_check else n1, 1), 2), np.uint32)
    k = lib().sm_oracle_match(pa, len(a), pb, len(b), max_ratio, max_distance, 1 if cross_check else 0,
                              max_num_matches, out.ctypes.data_as(_u32p))
    if k < 0:
        raise MemoryError("sm_oracle_match")
    return out[:k].copy()
