"""Guided SIFT matching without a GPU: the CPU oracle (tests/sm_guided_oracle.c) against an independent numpy statement
of the rule, the reference's MatchGuidedSiftFeaturesCPU.Nominal scenario, CamRayFromImgWithJac for all eighteen camera
models, model selection for every configuration, and the C ABI's refusals (all before any device work)."""
import ctypes
import os
import re

import numpy as np
import pytest

import oracle_smg
from colmap_b200.bundle_adjustment import Camera
from colmap_b200.synthetic import CreateRandomFeatureDescriptors, make_guided_view_pair

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = np.float32, np.float64


# ---- an independent statement of the rule -------------------------------------------------------------------------
def numpy_reject(typ, M, max_error, xy1, xy2, geo1, geo2):
    """(n1, n2) bool: the filter of every candidate, in float32 (F, H) or float64 (E) numpy elementwise operations in
    the pinned order (numpy does not contract a * b + c)."""
    if typ == oracle_smg.E:
        E = np.asarray(M, F64)
        r1, r2 = geo1[:, :3], geo2[:, :3]
        J1, J2 = geo1[:, 3:9], geo2[:, 3:9]
        e = [(E[r, 0] * r1[:, 0] + E[r, 1] * r1[:, 1] + E[r, 2] * r1[:, 2])[:, None] for r in range(3)]
        t = [(E[0, c] * r2[:, 0] + E[1, c] * r2[:, 1] + E[2, c] * r2[:, 2])[None, :] for c in range(3)]
        num = r2[None, :, 0] * e[0] + r2[None, :, 1] * e[1] + r2[None, :, 2] * e[2]
        gx = J1[:, None, 0] * t[0] + J1[:, None, 2] * t[1] + J1[:, None, 4] * t[2]
        gy = J1[:, None, 1] * t[0] + J1[:, None, 3] * t[1] + J1[:, None, 5] * t[2]
        hx = J2[None, :, 0] * e[0] + J2[None, :, 2] * e[1] + J2[None, :, 4] * e[2]
        hy = J2[None, :, 1] * e[0] + J2[None, :, 3] * e[1] + J2[None, :, 5] * e[2]
        den = (gx * gx + gy * gy) + (hx * hx + hy * hy)
        with np.errstate(all="ignore"):
            err = np.where(den == 0, np.finfo(F64).max, num * num / np.where(den == 0, 1, den))
            rej = err > max_error * max_error
        return rej | (geo1[:, None, 9] == 0) | (geo2[None, :, 9] == 0)
    M = np.asarray(M, F64).astype(F32)
    thr = F32(max_error * max_error)
    x1, y1 = xy1[:, 0:1], xy1[:, 1:2]
    x2, y2 = xy2[None, :, 0], xy2[None, :, 1]
    a = [M[r, 0] * x1 + M[r, 1] * y1 + M[r, 2] for r in range(3)]
    with np.errstate(all="ignore"):
        if typ == oracle_smg.F:
            b0 = M[0, 0] * x2 + M[1, 0] * y2 + M[2, 0]
            b1 = M[0, 1] * x2 + M[1, 1] * y2 + M[2, 1]
            nom = x2 * a[0] + y2 * a[1] + a[2]
            den = a[0] * a[0] + a[1] * a[1] + b0 * b0 + b1 * b1
            return nom * nom > thr * den
        dx, dy = a[0] / a[2] - x2, a[1] / a[2] - y2
        return dx * dx + dy * dy > thr


def numpy_one_way(D, max_ratio, max_distance):
    n1, n2 = D.shape
    m = np.full(n1, -1, np.int64)
    if n1 == 0 or n2 == 0:
        return m
    idx = np.argmin(D, axis=1)
    best = D[np.arange(n1), idx]
    Dm = D.copy()
    Dm[np.arange(n1), idx] = np.inf
    second = Dm.min(axis=1).astype(F32) if n2 > 1 else np.full(n1, np.finfo(F32).max, F32)
    second = np.minimum(second, np.finfo(F32).max)
    md, mr = F32(max_distance), F32(max_ratio)
    ok = ~(best > F32(262144.0) * md * md) & ~(np.sqrt(best) >= mr * np.sqrt(second))
    m[ok] = idx[ok]
    return m


def numpy_match(d1, d2, xy1, xy2, typ, M, max_error, geo1=None, geo2=None, max_ratio=0.8, max_distance=0.7,
                cross_check=True, max_num_matches=32768):
    a = np.asarray(d1, np.int64)[:max_num_matches]
    b = np.asarray(d2, np.int64)[:max_num_matches]
    n1, n2 = len(a), len(b)
    if typ == oracle_smg.NONE or n1 == 0 or n2 == 0:
        return np.zeros((0, 2), np.uint32)
    L2 = ((a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2 * a @ b.T).astype(F32)
    g1 = None if geo1 is None else geo1[:n1]
    g2 = None if geo2 is None else geo2[:n2]
    rej = numpy_reject(typ, M, max_error, np.asarray(xy1, F32)[:n1], np.asarray(xy2, F32)[:n2], g1, g2)
    D = np.where(rej, F32(262144.0), L2)
    m12 = numpy_one_way(D, max_ratio, max_distance)
    keep = m12 >= 0
    if cross_check and keep.any():
        m21 = numpy_one_way(D.T, max_ratio, max_distance)
        keep &= np.where(keep, m21[np.maximum(m12, 0)] == np.arange(n1), False)
    i1 = np.nonzero(keep)[0]
    return np.stack([i1, m12[i1]], axis=1).astype(np.uint32).reshape(-1, 2)


def _scene(kind, n1=300, n2=260, seed=3):
    s = make_guided_view_pair(n1, n2, model_id=0, plane=True, seed=seed)
    if kind == "ties":    # duplicated rows and keypoints: equal distances and equal filter outcomes
        s["desc2"][100:140] = s["desc1"][:40]
        s["desc2"][200] = s["desc2"][199]
        s["xy2"][200] = s["xy2"][199]
    return s


@pytest.mark.parametrize("kind", ["view", "ties"])
@pytest.mark.parametrize("typ", [oracle_smg.E, oracle_smg.F, oracle_smg.H])
@pytest.mark.parametrize("cross_check", [True, False])
@pytest.mark.parametrize("rd", [(0.8, 0.7), (0.4, 0.7), (1.0, 1.2)])
def test_oracle_equals_numpy_statement(kind, typ, cross_check, rd):
    s = _scene(kind)
    g1, g2 = oracle_smg.geo(s["camera1"], s["xy1"]), oracle_smg.geo(s["camera2"], s["xy2"])
    M = {oracle_smg.E: s["E"], oracle_smg.F: s["F"], oracle_smg.H: s["H"]}[typ]
    args = (s["desc1"], s["desc2"], s["xy1"], s["xy2"], typ, M, 3.0, g1, g2)
    ref = numpy_match(*args, max_ratio=rd[0], max_distance=rd[1], cross_check=cross_check)
    got = oracle_smg.match(*args, max_ratio=rd[0], max_distance=rd[1], cross_check=cross_check)
    assert np.array_equal(got, ref)
    assert len(ref) > 0


def test_oracle_returns_rejected_candidate_with_max_distance_above_one():
    """With max_distance >= 1 a rejected candidate (distance 512^2) passes the distance test: a row whose only
    candidate is rejected, against one other far row, is returned as a match."""
    d1 = CreateRandomFeatureDescriptors(1, seed=5)
    d2 = np.zeros((2, 128), np.uint8)
    d2[1, :] = 255                      # L2 from any descriptor row far above 512^2
    xy1 = np.array([[0, 0]], F32)
    xy2 = np.array([[500, 500], [0, 0]], F32)
    H = np.eye(3)
    got = oracle_smg.match(d1, d2, xy1, xy2, oracle_smg.H, H, 1.0, max_ratio=1.0, max_distance=1.2, cross_check=False)
    # column 0 is rejected (262144), column 1 is real and larger: best is the rejected one
    assert np.array_equal(got, np.array([[0, 0]], np.uint32))
    assert np.array_equal(got, numpy_match(d1, d2, xy1, xy2, oracle_smg.H, H, 1.0, max_ratio=1.0, max_distance=1.2,
                                           cross_check=False))


# ---- the reference's MatchGuidedSiftFeaturesCPU.Nominal (sift_test.cc:591-645) -----------------------------------
def nominal_scenario(match):
    """match(d1, xy1, d2, xy2) -> matches under identity H, PLANAR_OR_PANORAMIC, max_error 1."""
    d1 = CreateRandomFeatureDescriptors(2)
    kp1 = np.array([[1, 0], [2, 0]], F32)
    d2, kp2 = d1[::-1].copy(), np.array([[2, 0], [1, 0]], F32)
    d3, kp3 = CreateRandomFeatureDescriptors(2), np.array([[100, 0], [2, 0]], F32)   # the generator's fixed seed
    d0, kp0 = np.zeros((0, 128), np.uint8), np.zeros((0, 2), F32)
    assert np.array_equal(match(d1, kp1, d2, kp2), np.array([[0, 1], [1, 0]], np.uint32))
    assert np.array_equal(match(d3, kp3, d2, kp2), np.array([[1, 0]], np.uint32))
    assert match(d0, kp0, d2, kp2).shape == (0, 2)
    assert match(d1, kp1, d0, kp0).shape == (0, 2)
    assert match(d0, kp0, d0, kp0).shape == (0, 2)


def test_nominal_scenario_on_the_oracle():
    nominal_scenario(lambda a, ka, b, kb: oracle_smg.match(a, b, ka, kb, oracle_smg.H, np.eye(3), 1.0))


def test_nominal_scenario_on_the_numpy_statement():
    nominal_scenario(lambda a, ka, b, kb: numpy_match(a, b, ka, kb, oracle_smg.H, np.eye(3), 1.0))


# ---- CamRayFromImgWithJac ------------------------------------------------------------------------------------------
MODELS = {
    0: [500, 320, 240], 1: [500, 480, 320, 240], 2: [500, 320, 240, -0.05], 3: [500, 320, 240, -0.05, 0.01],
    4: [500, 480, 320, 240, -0.05, 0.01, 0.001, -0.002], 5: [300, 290, 320, 240, 0.02, -0.01, 0.003, -0.001],
    6: [500, 480, 320, 240, -0.05, 0.01, 0.001, -0.002, 0.001, 0.01, 0.002, 0.001],
    7: [500, 480, 320, 240, 0.8], 8: [300, 320, 240, 0.02], 9: [300, 320, 240, 0.02, -0.005],
    10: [300, 290, 320, 240, 0.02, -0.01, 0.001, -0.002, 0.001, 0.001, 0.001, -0.001],
    11: [300, 290, 320, 240, 0.02, -0.01, 0.003, -0.001, 0.0005, 0.0001, 0.001, -0.002, 0.001, 0.0005, -0.001, 0.0003],
    12: [500, 320, 240, -0.1], 13: [500, 480, 320, 240, -0.1], 14: [300, 320, 240], 15: [300, 290, 320, 240],
    16: [400, 390, 320, 240, 0.6, 1.1], 17: [1024, 512]}


@pytest.mark.parametrize("model_id", sorted(MODELS))
def test_ray_jacobian_against_finite_differences(model_id):
    from colmap_b200.feature_matching import CamRayFromImgWithJac
    from colmap_b200.global_positioning import cam_ray_from_img
    cam = Camera(1, model_id, np.array(MODELS[model_id], F64))
    for xy in ([100.5, 80.25], [320.0, 240.0], [500.0, 400.0], [37.0, 300.0]):
        r = CamRayFromImgWithJac(cam, xy)
        assert r is not None, (model_id, xy)
        ray, J = r
        assert np.allclose(ray, cam_ray_from_img(model_id, cam.params, np.array(xy, F64)), rtol=0, atol=1e-15)
        assert abs(np.linalg.norm(ray) - 1) < 1e-12
        h = 1e-4
        fd = np.zeros((3, 2))
        for c in range(2):
            e = np.zeros(2); e[c] = h
            fd[:, c] = (cam_ray_from_img(model_id, cam.params, np.array(xy, F64) + e)
                        - cam_ray_from_img(model_id, cam.params, np.array(xy, F64) - e)) / (2 * h)
        assert np.allclose(J, fd, rtol=1e-5, atol=1e-9 * np.abs(J).max()), (model_id, xy, J, fd)
        assert np.all(np.abs(ray @ J) <= 1e-12 * np.abs(J).max())   # both columns tangent to the sphere


def test_ray_jacobian_invalid_cases():
    from colmap_b200.feature_matching import CamRayFromImgWithJac
    # EUCM outside its domain: the unprojection's radicand is negative
    eucm = Camera(1, 16, np.array([100, 100, 0, 0, 0.9, 2.0], F64))
    assert CamRayFromImgWithJac(eucm, [400.0, 400.0]) is None
    # the relative alpha test: a division model at the edge of its image circle, where the Jacobian is singular
    div = Camera(1, 12, np.array([100, 0, 0, 0.25], F64))
    assert CamRayFromImgWithJac(div, [1e-3, 0.0]) is not None
    assert CamRayFromImgWithJac(div, [200.0, 0.0]) is None
    from colmap_b200.feature_matching import FeatureMatchingError
    with pytest.raises(FeatureMatchingError):
        CamRayFromImgWithJac(Camera(1, 18, np.zeros(16)), [0.0, 0.0])


# ---- model selection ----------------------------------------------------------------------------------------------
def _img(model_id=0):
    from colmap_b200.feature_matching import FeatureMatcherImage
    return FeatureMatcherImage(1, np.zeros((1, 128), np.uint8), camera=Camera(1, model_id, np.array(MODELS[model_id], F64)),
                               keypoints=np.zeros((1, 2), F32))


@pytest.mark.parametrize("config", range(10))
@pytest.mark.parametrize("have", ["", "E", "F", "H", "EFH", "E+cam", "EF+cam"])
def test_model_selection(config, have):
    from colmap_b200.feature_matching import GUIDED_E, GUIDED_F, GUIDED_H, GUIDED_NONE, SelectGuidedModel, TwoViewGeometry
    g = TwoViewGeometry(config=config)
    for k in "EFH":
        if k in have:
            setattr(g, k, np.eye(3))
    if "cam" in have:
        g.camera2 = Camera(2, 1, np.array(MODELS[1], F64))
    typ, M, c1, c2 = SelectGuidedModel(g, _img(), _img())
    e = "E" in have and (config in (2, 9) or (config == 3 and "cam" in have))
    f = not e and config == 3 and "F" in have
    h = config in (4, 5, 6) and "H" in have
    assert typ == (GUIDED_E if e else GUIDED_F if f else GUIDED_H if h else GUIDED_NONE)
    assert c2.model_id == (1 if "cam" in have else 0)


def test_homography_with_spherical_camera_is_refused():
    from colmap_b200.feature_matching import FeatureMatchingError, SelectGuidedModel, TwoViewGeometry
    g = TwoViewGeometry(config=TwoViewGeometry.PLANAR, H=np.eye(3))
    with pytest.raises(FeatureMatchingError):
        SelectGuidedModel(g, _img(17), _img())
    SelectGuidedModel(TwoViewGeometry(config=TwoViewGeometry.CALIBRATED, E=np.eye(3)), _img(17), _img(17))


def test_guided_images_need_camera_keypoints_and_equal_counts():
    from colmap_b200.feature_matching import FeatureMatcherImage, FeatureMatchingError, _check_guided_image
    with pytest.raises(FeatureMatchingError):
        FeatureMatcherImage(1, np.zeros((2, 128), np.uint8), keypoints=np.zeros((2, 3), F32))
    with pytest.raises(FeatureMatchingError):
        _check_guided_image(FeatureMatcherImage(1, np.zeros((2, 128), np.uint8)))
    with pytest.raises(FeatureMatchingError):
        _check_guided_image(FeatureMatcherImage(1, np.zeros((2, 128), np.uint8), camera=Camera(1, 0, np.ones(3)),
                                                keypoints=np.zeros((3, 2), F32)))


# ---- the C ABI ----------------------------------------------------------------------------------------------------
def _lib():
    from colmap_b200.feature_matching import _lib as bound
    return bound()


def test_library_exports_the_guided_entry_points():
    with open(os.path.join(ROOT, "include", "b200_sift_matching.h")) as f:
        names = set(re.findall(r"\b(b200sm_[a-z_0-9]+)\s*\(", f.read()))
    new = {"b200sm_set_keypoints", "b200sm_set_camera", "b200sm_cam_ray_from_img_with_jac", "b200sm_match_guided_pairs"}
    assert new <= names
    for n in new:
        assert hasattr(_lib(), n)


def test_guided_calls_refuse_null_handles_and_arguments():
    from colmap_b200.feature_matching import _CGuided
    L = _lib()
    xy = np.zeros((2, 2), F32)
    prm = np.zeros(16)
    f32p, f64p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)
    assert L.b200sm_set_keypoints(None, 0, 2, xy.ctypes.data_as(f32p)) == -1
    assert L.b200sm_set_camera(None, 0, 0, prm.ctypes.data_as(f64p)) == -1
    out = np.zeros(9)
    assert L.b200sm_cam_ray_from_img_with_jac(0, None, prm.ctypes.data_as(f64p), out.ctypes.data_as(f64p)) == -1
    assert L.b200sm_cam_ray_from_img_with_jac(-1, prm.ctypes.data_as(f64p), prm.ctypes.data_as(f64p),
                                              out.ctypes.data_as(f64p)) == -1
    s = np.zeros(1, np.int32)
    sp = s.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    off = np.zeros(2, np.uint64)
    g = (_CGuided * 1)()
    assert L.b200sm_match_guided_pairs(None, 1, sp, sp, g, off.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)),
                                       None, 0) == -1
    assert L.b200sm_last_error().decode()


def test_selection_without_a_camera_is_refused():
    from colmap_b200.feature_matching import (FeatureMatcherImage, FeatureMatchingError, GUIDED_F, SelectGuidedModel,
                                              TwoViewGeometry)
    bare = FeatureMatcherImage(1, np.zeros((1, 128), np.uint8), keypoints=np.zeros((1, 2), F32))
    for g in (TwoViewGeometry(config=TwoViewGeometry.PLANAR, H=np.eye(3)),
              TwoViewGeometry(config=TwoViewGeometry.CALIBRATED, E=np.eye(3))):
        with pytest.raises(FeatureMatchingError):
            SelectGuidedModel(g, bare, _img())
        with pytest.raises(FeatureMatchingError):
            SelectGuidedModel(g, _img(), bare)
    assert SelectGuidedModel(TwoViewGeometry(config=TwoViewGeometry.UNCALIBRATED, F=np.eye(3)), bare, bare)[0] == GUIDED_F


# ---- rays against known answers ------------------------------------------------------------------------------------
_RAYS = np.array([[0.0, 0.0, 1.0], [0.1, -0.05, 1.0], [-0.3, 0.2, 1.0], [0.25, 0.3, 1.0], [-0.05, -0.4, 1.0]])


@pytest.mark.parametrize("model_id", sorted(MODELS))
def test_rays_invert_the_projection(model_id):
    """Known rays projected by the projection of bundle adjustment (numpy for the radial pinhole and fisheye family,
    the wide models' own host formulas otherwise), which the BA tests hold to the reference; the pixel must unproject
    to the same unit ray.  Independent of the unprojection code (cam_rays.cuh)."""
    from colmap_b200.feature_matching import CamRayFromImgWithJac
    from colmap_b200.synthetic import _project
    prm = np.array(MODELS[model_id], F64)
    xy = _project(model_id, np.tile(prm, (len(_RAYS), 1)), _RAYS)
    cam = Camera(1, model_id, prm)
    for ray, p in zip(_RAYS, xy):
        r = CamRayFromImgWithJac(cam, p)
        assert r is not None, (model_id, p)
        assert np.allclose(r[0], ray / np.linalg.norm(ray), rtol=0, atol=1e-9), (model_id, r[0], ray)


def test_rays_known_answers_in_closed_form():
    """Closed-form rays: EQUIRECTANGULAR (azimuth and elevation), SIMPLE_FISHEYE (equidistant: the angle to the axis is
    the pixel radius over f), SIMPLE_DIVISION (models.h: (x, 1 + k |x|^2) is the homogeneous ray)."""
    from colmap_b200.feature_matching import CamRayFromImgWithJac
    eq = Camera(1, 17, np.array([1024.0, 512.0]))
    for x, y in ((512.0, 256.0), (768.0, 128.0), (100.0, 400.0), (1000.0, 30.0)):
        th, ph = 2 * np.pi * (x / 1024 - 0.5), np.pi * (0.5 - y / 512)
        ref = np.array([np.cos(ph) * np.sin(th), -np.sin(ph), np.cos(ph) * np.cos(th)])
        assert np.allclose(CamRayFromImgWithJac(eq, [x, y])[0], ref, rtol=0, atol=1e-14)
    fe = Camera(1, 14, np.array([300.0, 320.0, 240.0]))
    for x, y in ((320.0, 240.0), (500.0, 240.0), (100.0, 50.0), (620.0, 470.0)):
        u, v = (x - 320) / 300, (y - 240) / 300
        r = np.hypot(u, v)
        ref = np.array([0, 0, 1.0]) if r == 0 else np.array([np.sin(r) * u / r, np.sin(r) * v / r, np.cos(r)])
        assert np.allclose(CamRayFromImgWithJac(fe, [x, y])[0], ref, rtol=0, atol=1e-12)
    dv = Camera(1, 12, np.array([500.0, 320.0, 240.0, -0.1]))
    for x, y in ((320.0, 240.0), (600.0, 100.0), (30.0, 420.0)):
        u, v = (x - 320) / 500, (y - 240) / 500
        ref = np.array([u, v, 1 - 0.1 * (u * u + v * v)])
        assert np.allclose(CamRayFromImgWithJac(dv, [x, y])[0], ref / np.linalg.norm(ref), rtol=0, atol=1e-12)
