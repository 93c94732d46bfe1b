"""Guided SIFT matching on the GPU, held to the CPU oracle (tests/sm_guided_oracle.c) bit for bit: a size grid around
the 128-row strips and 128-column tiles for E, F and H, with and without cross-check, at three threshold settings;
crafted cases at the edges of the rule; a mixed batch checked three ways; and unguided matching on the same handle
before and after guided calls."""
import numpy as np
import pytest

import oracle_sm
import oracle_smg
from colmap_b200.bundle_adjustment import Camera
from colmap_b200.feature_matching import (CreateSiftFeatureMatcher, FeatureMatcherImage, FeatureMatchingOptions,
                                          SiftMatchingOptions, TwoViewGeometry)
from colmap_b200.synthetic import CreateRandomFeatureDescriptors, make_guided_view_pair

pytestmark = pytest.mark.gpu
F32 = np.float32
KIND = {"E": (oracle_smg.E, TwoViewGeometry.CALIBRATED), "F": (oracle_smg.F, TwoViewGeometry.UNCALIBRATED),
        "H": (oracle_smg.H, TwoViewGeometry.PLANAR)}


def _matcher(r=0.8, d=0.7, cc=True, max_num_matches=32768):
    return CreateSiftFeatureMatcher(FeatureMatchingOptions(gpu_index="0", max_num_matches=max_num_matches,
                                                           sift=SiftMatchingOptions(r, d, cc)))


def _geometry(kind, M):
    g = TwoViewGeometry(config=KIND[kind][1])
    setattr(g, kind, M)
    return g


def _images(s, id1=1, id2=2):
    return (FeatureMatcherImage(id1, s["desc1"], camera=s["camera1"], keypoints=s["xy1"]),
            FeatureMatcherImage(id2, s["desc2"], camera=s["camera2"], keypoints=s["xy2"]))


def _oracle(s, kind, M, max_error, r=0.8, d=0.7, cc=True, max_num_matches=32768):
    g1 = g2 = None
    if kind == "E":
        g1, g2 = oracle_smg.geo(s["camera1"], s["xy1"]), oracle_smg.geo(s["camera2"], s["xy2"])
    return oracle_smg.match(s["desc1"], s["desc2"], s["xy1"], s["xy2"], KIND[kind][0], M, max_error, g1, g2,
                            max_ratio=r, max_distance=d, cross_check=cc, max_num_matches=max_num_matches)


_SCENES = {}


def _scene(n, plane=True, model_id=0):
    key = (n, plane, model_id)
    if key not in _SCENES:
        _SCENES[key] = make_guided_view_pair(n, n, model_id=model_id, plane=plane, seed=n)
    return _SCENES[key]


@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 127, 129, 1000, 8192])
@pytest.mark.parametrize("kind", ["E", "F", "H"])
def test_size_grid_equals_oracle(n, kind):
    s = _scene(n)
    M = s[kind]
    for cc in (True, False):
        for r, d in ((0.8, 0.7), (0.4, 0.7), (1.0, 1.2)):
            if n == 8192 and (r, d) != (0.8, 0.7):
                continue                       # the oracle's time: one setting per direction mode at 8192
            with _matcher(r, d, cc) as m:
                g = _geometry(kind, M)
                m.MatchGuided(4.0, *_images(s), g)
            ref = _oracle(s, kind, M, 4.0, r, d, cc)
            assert np.array_equal(g.inlier_matches, ref), (n, kind, cc, r, d, len(g.inlier_matches), len(ref))
            if n >= 129:
                assert len(ref) > 0


@pytest.mark.parametrize("model_id", [2, 8, 17])
def test_essential_filter_on_distorted_fisheye_and_spherical_cameras(model_id):
    s = make_guided_view_pair(700, 600, model_id=model_id, seed=11)
    with _matcher() as m:
        g = _geometry("E", s["E"])
        m.MatchGuided(3.0, *_images(s), g)
    ref = _oracle(s, "E", s["E"], 3.0)
    assert len(ref) > 50 and np.array_equal(g.inlier_matches, ref)


def _crafted(n1, n2, seed):
    rng = np.random.default_rng(seed)
    s = {"desc1": CreateRandomFeatureDescriptors(n1, seed=seed), "desc2": CreateRandomFeatureDescriptors(n2, seed=seed + 1),
         "xy1": rng.uniform(0, 64, (n1, 2)).astype(F32), "xy2": rng.uniform(0, 64, (n2, 2)).astype(F32),
         "camera1": Camera(1, 0, np.array([50.0, 32, 32])), "camera2": Camera(2, 0, np.array([50.0, 32, 32]))}
    return s


def _check(s, kind, M, max_error, **kw):
    r, d, cc = kw.get("r", 0.8), kw.get("d", 0.7), kw.get("cc", True)
    with _matcher(r, d, cc) as m:
        g = _geometry(kind, M)
        m.MatchGuided(max_error, *_images(s), g)
    ref = _oracle(s, kind, M, max_error, r, d, cc)
    assert np.array_equal(g.inlier_matches, ref), (kind, len(g.inlier_matches), len(ref))
    return ref


def test_residuals_exactly_at_the_threshold():
    """Keypoints on an integer grid and H a pure integer shift: transfer errors are exact integers, and max_error 2
    puts many at exactly 4 == max_error^2 (not rejected)."""
    s = _crafted(300, 300, 1)
    s["xy1"] = np.random.default_rng(2).integers(0, 6, (300, 2)).astype(F32)
    s["xy2"] = np.random.default_rng(3).integers(0, 6, (300, 2)).astype(F32)
    s["desc2"][:150] = s["desc1"][:150]
    H = np.array([[1, 0, 1.0], [0, 1, -1.0], [0, 0, 1]])
    for cc in (True, False):
        for d in (0.7, 1.2):
            _check(s, "H", H, 2.0, cc=cc, d=d, r=0.95)
    F = np.array([[0, 0, 0], [0, 0, -1.0], [0, 1.0, 0]])   # horizontal epipolar lines: the error is (y2 - y1)^2 / 2
    _check(s, "F", F, 1.0, r=0.95)


def test_nan_filters_do_not_reject():
    """F with both epipoles at keypoints (den == 0, nom == 0: 0 > 0 is false) and H with hz == 0 (NaN residuals)."""
    s = _crafted(200, 200, 4)
    s["xy1"][::3] = 0
    s["xy2"][::3] = 0
    s["desc2"][:100] = s["desc1"][:100]
    F = np.array([[0, 0, 0], [0, 0, -1.0], [0, 1.0, 0]])
    _check(s, "F", F, 0.5)
    H = np.array([[1, 0, 0], [0, 1, 0], [1.0, 0, 0]])     # hz == x1: zero where x1 == 0
    ref = _check(s, "H", H, 0.5, d=1.2, r=1.0)
    assert len(ref) > 0


def test_invalid_rays_are_rejected():
    s = _crafted(250, 250, 5)
    eucm = Camera(1, 16, np.array([20.0, 20, 32, 32, 0.9, 2.0]))    # outside the EUCM domain far from the centre
    s["camera1"] = s["camera2"] = eucm
    s["desc2"][:120] = s["desc1"][:120]
    s["xy2"][:120] = s["xy1"][:120]
    assert (oracle_smg.geo(eucm, s["xy1"])[:, 9] == 0).any()
    _check(s, "E", np.array([[0, 0, 0], [0, 0, -1.0], [0, 1.0, 0]]), 5.0)


def test_rejected_candidates_win_best_and_second():
    """Real distances above 512^2 (rows of 255 against rows of 0) so that rejected candidates (512^2) become best and
    second; with max_distance 1.2 a rejected candidate is returned as a match."""
    rng = np.random.default_rng(6)
    s = _crafted(200, 300, 6)
    s["desc1"][:100] = 255
    s["desc2"][:150] = 0
    s["desc2"][150:] = rng.integers(0, 256, (150, 128), dtype=np.uint8)
    H = np.eye(3)
    for cc in (True, False):
        _check(s, "H", H, 3.0, cc=cc)
        _check(s, "H", H, 3.0, cc=cc, d=1.2, r=1.0)
    # one rejected column per row (keypoint far away), every other column accepted and farther than 512^2 in L2 from
    # the rows of 255: the rejected column is best, and max_distance 1.2 returns it
    s["xy1"][:] = 0
    s["xy2"][:] = 0
    s["xy2"][0] = 500
    ref = _check(s, "H", H, 3.0, cc=False, d=1.2, r=1.0)
    assert np.array_equal(ref[:100], np.stack([np.arange(100), np.zeros(100)], axis=1).astype(np.uint32))
    _check(s, "H", H, 3.0, cc=True, d=1.2, r=1.0)


def test_distances_on_both_sides_of_the_distance_threshold():
    """L2 on both sides of 262144 * 0.7f * 0.7f: rows built at distances spread around 128450."""
    rng = np.random.default_rng(7)
    n = 256
    base = rng.integers(0, 40, (n, 128)).astype(np.int32)
    other = base.copy()
    target = rng.integers(126000, 131000, n)
    for k in range(n):   # raise dimensions until the squared distance reaches the target
        rem, j = int(target[k]), 0
        while rem > 0 and j < 128:
            step = min(int(np.sqrt(rem)), 215)
            other[k, j] = base[k, j] + step
            rem -= step * step
            j += 1
    s = _crafted(n, n, 7)
    s["desc1"], s["desc2"] = base.astype(np.uint8), other.astype(np.uint8)
    s["xy2"] = s["xy1"].copy()
    _check(s, "H", np.eye(3), 1.0, r=0.99)
    _check(s, "H", np.eye(3), 1.0, r=0.99, cc=False)


def test_ties_across_strips_and_tiles_and_padding_columns():
    """Exact copies placed across 128-row strips and 128-column tiles (best ties resolve to the smallest column), and
    rows of zeros whose L2 to zero padding would be 0 if padding columns were not masked."""
    s = _crafted(300, 300, 8)
    s["desc2"][5] = s["desc2"][133] = s["desc2"][261] = s["desc1"][7]
    s["desc2"][140] = s["desc2"][260] = s["desc1"][200]
    s["desc1"][250:] = 0
    s["xy1"][:] = s["xy2"][:] = 10.0
    for cc in (True, False):
        _check(s, "H", np.eye(3), 1.0, cc=cc, r=1.0, d=1.2)
        _check(s, "H", np.eye(3), 1.0, cc=cc)


def test_one_column():
    s = _crafted(200, 1, 9)
    s["desc2"][0] = s["desc1"][17]
    for cc in (True, False):
        _check(s, "H", np.eye(3), 100.0, cc=cc, r=1.0)
        _check(s, "F", np.array([[0, 0, 0], [0, 0, -1.0], [0, 1.0, 0]]), 100.0, cc=cc)


def test_mixed_batch_three_ways_shuffled_and_repeated():
    rng = np.random.default_rng(10)
    sc = [make_guided_view_pair(n, n + 37 * k, model_id=0, plane=True, seed=20 + k)
          for k, n in enumerate([300, 129, 500, 64, 400])]
    images, pairs, geos = [], [], []
    for k, s in enumerate(sc):
        a, b = _images(s, 10 * k + 1, 10 * k + 2)
        images += [a, b]
    images.append(FeatureMatcherImage(99, np.zeros((0, 128), np.uint8), camera=sc[0]["camera1"],
                                      keypoints=np.zeros((0, 2), F32)))
    specs = [(0, "E"), (1, "F"), (2, "H"), (3, "E"), (4, "F"), (0, "H"), (2, None), (4, "E")]
    for k, kind in specs:
        pairs.append((2 * k, 2 * k + 1))
        g = TwoViewGeometry(config=KIND[kind][1] if kind else TwoViewGeometry.DEGENERATE)
        if kind:
            setattr(g, kind, sc[k][kind])
        geos.append(g)
    # E with per-pair estimated cameras: the same images under a different focal length
    g = TwoViewGeometry(config=TwoViewGeometry.UNCALIBRATED, E=sc[1]["E"], camera1=Camera(1, 0, np.array([480.0, 320, 240])))
    pairs.append((2, 3)); geos.append(g)
    pairs.append((10, 1)); geos.append(_geometry("H", sc[0]["H"]))          # an empty image
    pairs.append((0, 10)); geos.append(_geometry("F", sc[0]["F"]))
    refs = []
    for (i, j), g in zip(pairs, geos):
        with _matcher(max_num_matches=450) as m:        # the 500-row scene is above max_num_matches
            gg = TwoViewGeometry(g.config, g.E, g.F, g.H, g.camera1, g.camera2)
            m.MatchGuided(4.0, images[i], images[j], gg)
        refs.append(gg.inlier_matches)
    for (i, j), g, r in zip(pairs, geos, refs):
        typ, M, c1, c2 = __import__("colmap_b200.feature_matching", fromlist=["x"]).SelectGuidedModel(g, images[i], images[j])
        kind = {oracle_smg.E: "E", oracle_smg.F: "F", oracle_smg.H: "H"}.get(typ)
        if kind is None:
            assert len(r) == 0
            continue
        s = {"desc1": images[i].descriptors, "desc2": images[j].descriptors, "xy1": images[i].keypoints,
             "xy2": images[j].keypoints, "camera1": c1, "camera2": c2}
        assert np.array_equal(r, _oracle(s, kind, M, 4.0, max_num_matches=450))
    assert sum(len(r) for r in refs) > 100
    with _matcher(max_num_matches=450) as m:
        for rep in range(3):
            order = rng.permutation(len(pairs))
            out = m.MatchGuidedPairs(images, [pairs[k] for k in order], [geos[k] for k in order], 4.0)
            for k, o in zip(order, out):
                assert np.array_equal(o, refs[k]), (rep, k)
                assert np.array_equal(geos[k].inlier_matches, refs[k])


def test_unguided_match_on_the_same_handle_before_and_after_guided():
    s = _scene(1000)
    a, b = _images(s)
    plain = oracle_sm.match(s["desc1"], s["desc2"])
    with _matcher() as m:
        assert np.array_equal(m.Match(a, b), plain)
        g = _geometry("F", s["F"])
        m.MatchGuided(4.0, a, b, g)
        assert np.array_equal(g.inlier_matches, _oracle(s, "F", s["F"], 4.0))
        assert np.array_equal(m.Match(a, b), plain)
        g = _geometry("E", s["E"])
        m.MatchGuided(4.0, b, a, g)
        s2 = {"desc1": s["desc2"], "desc2": s["desc1"], "xy1": s["xy2"], "xy2": s["xy1"], "camera1": s["camera2"],
              "camera2": s["camera1"]}
        assert np.array_equal(g.inlier_matches, _oracle(s2, "E", s["E"], 4.0))
        assert np.array_equal(m.Match(a, b), plain)
        assert np.array_equal(m.Match(b, a), oracle_sm.match(s["desc2"], s["desc1"]))


def test_guided_call_after_a_refused_one_equals_oracle():
    """A call refused as too large (more than B200SM_MAX_ROWS_PER_CALL rows) must leave every slot as it was: the next
    guided call on the same handle, with slots whose descriptor norms were never computed (slots 0 and 1) or belong to
    an earlier descriptor set (slot 1 after a new upload), equals the oracle."""
    import ctypes
    from colmap_b200.feature_matching import _CGuided, _lib
    L = _lib()
    s = _scene(1000)
    big = CreateRandomFeatureDescriptors(65536, seed=3)
    big_img = FeatureMatcherImage(50, big, camera=s["camera1"], keypoints=np.zeros((65536, 2), F32))
    a, b = _images(s)
    c = make_guided_view_pair(1300, 1300, model_id=0, plane=True, seed=77)
    b2 = FeatureMatcherImage(3, c["desc2"], camera=c["camera2"], keypoints=c["xy2"])

    def refuse(m):
        P = 1 + 16385                                  # 16385 x (65536 + 65536) rows > 2^31
        s1 = np.array([0] + [2] * (P - 1), np.int32)
        s2 = np.array([1] + [3] * (P - 1), np.int32)
        g = (_CGuided * P)()
        for k in range(P):
            g[k].type, g[k].max_error = 2, 4.0
            g[k].M[:] = np.asarray(s["F"], np.float64).ravel().tolist()
        i32p = ctypes.POINTER(ctypes.c_int)
        cap = L.b200sm_match_capacity(m._h, P, s1.ctypes.data_as(i32p), s2.ctypes.data_as(i32p))
        off = np.zeros(P + 1, np.uint64)
        out = np.zeros(2, np.uint32)                   # refused before anything is written
        rc = L.b200sm_match_guided_pairs(m._h, P, s1.ctypes.data_as(i32p), s2.ctypes.data_as(i32p), g,
                                         off.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)),
                                         out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), cap)
        assert rc == -2, L.b200sm_last_error()

    with _matcher(max_num_matches=65536) as m:
        m._reserve(4)
        for k, im in enumerate((a, b, big_img, big_img)):
            m._upload_guided(k, im, None)
        refuse(m)
        g = _geometry("F", s["F"])
        m.MatchGuided(4.0, a, b, g)
        assert len(g.inlier_matches) > 0
        assert np.array_equal(g.inlier_matches, _oracle(s, "F", s["F"], 4.0))
        m._upload_guided(1, b2, None)                  # a new, longer descriptor set in slot 1
        refuse(m)
        g = _geometry("F", s["F"])
        m.MatchGuided(4.0, a, b2, g)
        s2 = {"desc1": s["desc1"], "desc2": c["desc2"], "xy1": s["xy1"], "xy2": c["xy2"]}
        assert np.array_equal(g.inlier_matches, _oracle(s2, "F", s["F"], 4.0))
