"""SIFT feature matching without a GPU: the CPU oracle (tests/sm_oracle.c) against an independent numpy statement of
FindBestMatchesBruteForce, the reference's matcher test scenarios restated on the oracle, and the C ABI's surface,
defaults and refusals (every refusal here happens before any device work)."""
import ctypes
import ctypes.util
import os
import re

import numpy as np
import pytest

import oracle_sm
from colmap_b200.synthetic import (CreateRandomFeatureDescriptors, FeatureDescriptorsToUnsignedByte,
                                   make_sift_view_pair)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200_sift_matching.h")

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.acosf.argtypes = [ctypes.c_float]
_libm.acosf.restype = ctypes.c_float


def libm_acosf(x):
    """The C library's acosf (what std::acos(float) calls) elementwise; numpy's float32 arccos is a different
    function."""
    x = np.asarray(x, np.float32)
    u, inv = np.unique(x, return_inverse=True)
    return np.array([_libm.acosf(float(v)) for v in u], np.float32)[inv].reshape(x.shape)


def numpy_one_way(D, max_ratio, max_distance):
    """FindBestMatchesOneWayBruteForce on an int64 dot matrix: best = the largest dot floored at 0, its first column
    (np.argmax returns the first maximum), second = the largest dot once one copy of best is removed, floored at 0."""
    n1, n2 = D.shape
    m = np.full(n1, -1, np.int64)
    if n1 == 0 or n2 == 0:
        return m
    idx = np.argmax(D, axis=1)
    best = np.maximum(D[np.arange(n1), idx], 0)
    E = D.copy()
    E[np.arange(n1), idx] = -1
    second = np.maximum(E.max(axis=1), 0) if n2 > 1 else np.zeros(n1, np.int64)
    inv = np.float32(1.0 / 262144.0)
    d1 = libm_acosf(np.minimum(best.astype(np.float32) * inv, np.float32(1)))
    d2 = libm_acosf(np.minimum(second.astype(np.float32) * inv, np.float32(1)))
    ok = (best > 0) & ~(d1 > np.float32(max_distance)) & ~(d1 >= np.float32(max_ratio) * d2)
    m[ok] = idx[ok]
    return m


def numpy_match(d1, d2, max_ratio=0.8, max_distance=0.7, cross_check=True, max_num_matches=32768):
    a = np.asarray(d1, np.int64)[:max_num_matches]
    b = np.asarray(d2, np.int64)[:max_num_matches]
    D = a @ b.T
    m12 = numpy_one_way(D, max_ratio, max_distance)
    keep = m12 >= 0
    if cross_check and keep.any():
        m21 = numpy_one_way(D.T, max_ratio, max_distance)
        keep &= np.where(keep, m21[np.maximum(m12, 0)] == np.arange(len(a)), False)
    i1 = np.nonzero(keep)[0]
    return np.stack([i1, m12[i1]], axis=1).astype(np.uint32).reshape(-1, 2)


def test_libm_acosf_is_not_numpy_arccos_nor_rounded_double_acos():
    """Why the spec tabulates the C library's acosf: over the 2^18 + 1 arguments k * 2^-18 it differs from the
    correctly rounded arccos on many of them (this only documents the premise; the matcher uses acosf throughout)."""
    x = (np.arange(0, 262145, 97, dtype=np.float64) / 262144.0).astype(np.float32)
    f = libm_acosf(x)
    cr = np.arccos(x.astype(np.float64)).astype(np.float32)
    assert np.all(np.abs(f.astype(np.float64) - cr) <= 2 * np.spacing(cr))
    assert np.any(f != cr)


@pytest.mark.parametrize("kind", ["ties", "view"])
@pytest.mark.parametrize("cross_check", [True, False])
@pytest.mark.parametrize("ratio_distance", [(0.8, 0.7), (0.4, 0.7), (1.0, 1.2), (0.95, 0.9)])
def test_oracle_equals_numpy_statement(kind, cross_check, ratio_distance):
    r, dmax = ratio_distance
    if kind == "ties":
        a, b = CreateRandomFeatureDescriptors(300, seed=1), CreateRandomFeatureDescriptors(257, seed=2)
        b[100:140] = a[:40]          # exact copies: best ties with other near-copies and identical seconds
        b[200] = b[199]               # a duplicated column: best == second
    else:
        a, b, _ = make_sift_view_pair(400, 333, seed=3)
    ref = numpy_match(a, b, r, dmax, cross_check)
    got = oracle_sm.match(a, b, r, dmax, cross_check)
    assert np.array_equal(got, ref)
    assert len(ref) > 0


def test_oracle_clamps_rows_to_max_num_matches():
    a, b, _ = make_sift_view_pair(300, 300, seed=4)
    assert np.array_equal(oracle_sm.match(a, b, max_num_matches=120), numpy_match(a[:120], b[:120]))
    assert np.array_equal(oracle_sm.match(a, b, max_num_matches=120), oracle_sm.match(a[:120], b[:120]))


# ---- the scenarios of the reference's feature/sift_test.cc, restated with our generator --------------------------
def _normalized_u8(row):
    r = row.astype(np.float32)
    return FeatureDescriptorsToUnsignedByte(r / np.linalg.norm(r))


def ratio_scenario():
    """MatchSiftFeaturesCPUvsGPU's ratio check (sift_test.cc:1332-1360): row 49 of image 2 becomes a perturbed copy of
    row 0, and row 0 is perturbed too (uint8 arithmetic wraps as in the reference)."""
    d1 = CreateRandomFeatureDescriptors(50)
    d2 = d1.copy()
    d2[49] = d2[0]
    d2[0, 0] = np.uint8((int(d2[0, 0]) + 50) % 256)
    d2[0] = _normalized_u8(d2[0])
    d2[49, 0] = np.uint8((int(d2[49, 0]) + 100) % 256)
    d2[49] = _normalized_u8(d2[49])
    return d1, d2


def reference_scenarios(match):
    """Runs the scenarios through `match(d1, d2, **options)`; returns nothing, asserts the reference's outcomes."""
    empty = np.zeros((0, 128), np.uint8)
    two = CreateRandomFeatureDescriptors(2)
    assert match(empty, two[::-1]).shape == (0, 2)
    assert match(two, empty).shape == (0, 2)
    assert match(empty, empty).shape == (0, 2)
    assert np.array_equal(match(two, two[::-1]), np.array([[0, 1], [1, 0]], np.uint32))
    d50 = CreateRandomFeatureDescriptors(50)
    rev = match(d50, d50[::-1])
    assert len(rev) == 50 and np.array_equal(rev[:, 1], 49 - rev[:, 0])
    same = match(d50, d50.copy())
    assert len(same) == 50 and np.array_equal(same[:, 0], same[:, 1])
    d1, d2 = ratio_scenario()
    assert len(match(d1[:49], d2, max_ratio=0.4)) == 48
    assert len(match(d1, d2, max_ratio=0.6)) == 49


def test_reference_scenarios_on_the_oracle():
    reference_scenarios(oracle_sm.match)


def test_reference_scenarios_on_the_numpy_statement():
    reference_scenarios(numpy_match)


# ---- the C ABI ------------------------------------------------------------------------------------------------------
def _lib():
    from colmap_b200.feature_matching import _lib as bound
    return bound()


def test_library_exports_every_declared_sift_matching_symbol():
    with open(HEADER) as f:
        hdr = f.read()
    names = set(re.findall(r"\b(b200sm_[a-z_0-9]+)\s*\(", hdr))
    assert {"b200sm_create", "b200sm_set_descriptors", "b200sm_match_pairs", "b200sm_destroy", "b200sm_last_error",
            "b200sm_options_init"} <= names
    L = _lib()
    for n in sorted(names):
        assert hasattr(L, n), n


def test_options_init_gives_the_reference_defaults():
    from colmap_b200.feature_matching import FeatureMatchingOptions, SiftMatchingOptions, _COptions
    c = _COptions()
    _lib().b200sm_options_init(ctypes.byref(c))
    assert (c.max_ratio, c.max_distance, c.cross_check, c.max_num_matches, c.gpu_index) == (0.8, 0.7, 1, 32768, -1)
    s, f = SiftMatchingOptions(), FeatureMatchingOptions()
    assert (s.max_ratio, s.max_distance, s.cross_check) == (0.8, 0.7, True)
    assert (f.max_num_matches, f.gpu_index) == (32768, "-1")
    m = f.to_c()
    assert (m.max_ratio, m.max_distance, m.cross_check, m.max_num_matches, m.gpu_index) == (0.8, 0.7, 1, 32768, -1)


def _create(**kw):
    from colmap_b200.feature_matching import _COptions
    L = _lib()
    c = _COptions()
    L.b200sm_options_init(ctypes.byref(c))
    num_slots = kw.pop("num_slots", 2)
    for k, v in kw.items():
        setattr(c, k, v)
    h = ctypes.c_void_p(1234)
    rc = L.b200sm_create(ctypes.byref(c), num_slots, ctypes.byref(h))
    return rc, h


@pytest.mark.parametrize("kw, code", [
    (dict(max_ratio=0.0), -1), (dict(max_ratio=-0.5), -1), (dict(max_distance=0.0), -1), (dict(max_distance=-1.0), -1),
    (dict(max_ratio=float("nan")), -1), (dict(max_num_matches=-1), -1), (dict(num_slots=0), -1),
    (dict(gpu_index=-2), -1), (dict(max_num_matches=(1 << 22) + 1), -2), (dict(num_slots=(1 << 20) + 1), -2)])
def test_create_refuses_before_device_work(kw, code):
    rc, h = _create(**kw)
    assert rc == code
    assert not h.value
    assert _lib().b200sm_last_error().decode()


def test_null_arguments_are_refused():
    from colmap_b200.feature_matching import _COptions
    L = _lib()
    c = _COptions()
    L.b200sm_options_init(ctypes.byref(c))
    assert L.b200sm_create(None, 2, ctypes.byref(ctypes.c_void_p())) == -1
    assert L.b200sm_create(ctypes.byref(c), 2, None) == -1
    d = np.zeros((4, 128), np.uint8)
    assert L.b200sm_set_descriptors(None, 0, 4, d.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))) == -1
    s = np.zeros(1, np.int32)
    sp = s.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    off = np.zeros(2, np.uint64)
    assert L.b200sm_match_capacity(None, 1, sp, sp) == -1
    assert L.b200sm_match_pairs(None, 1, sp, sp, off.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), None, 0) == -1
    L.b200sm_destroy(None)


@pytest.mark.parametrize("bad", [np.zeros((4, 64), np.uint8), np.zeros((4, 129), np.uint8), np.zeros(128, np.uint8),
                                 np.zeros((4, 128), np.float32), np.zeros((4, 128), np.int16)])
def test_descriptors_other_than_uint8_rows_of_128_are_refused(bad):
    from colmap_b200.feature_matching import FeatureMatcherImage, FeatureMatchingError
    with pytest.raises(FeatureMatchingError):
        FeatureMatcherImage(1, bad)


@pytest.mark.parametrize("opts", [dict(max_ratio=0.0), dict(max_distance=-0.1), dict(max_num_matches=0)])
def test_matcher_refuses_invalid_options(opts):
    from colmap_b200.feature_matching import (CreateSiftFeatureMatcher, FeatureMatchingError, FeatureMatchingOptions,
                                              SiftMatchingOptions)
    s = SiftMatchingOptions(**{k: v for k, v in opts.items() if k != "max_num_matches"})
    f = FeatureMatchingOptions(sift=s, **{k: v for k, v in opts.items() if k == "max_num_matches"})
    assert not f.Check()
    with pytest.raises(FeatureMatchingError):
        CreateSiftFeatureMatcher(f)


def test_gpu_index_lists_are_refused():
    from colmap_b200.feature_matching import FeatureMatchingError, FeatureMatchingOptions
    with pytest.raises(FeatureMatchingError):
        FeatureMatchingOptions(gpu_index="0,1").to_c()
