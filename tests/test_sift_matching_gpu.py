"""SIFT feature matching on the GPU, held to exact equality with the CPU oracle (tests/sm_oracle.c): a grid of image
sizes across the kernel's 128-row strips and 128-column tiles, both cross-check settings, several thresholds and four
kinds of descriptors; crafted dot products on the acosf arguments that decide the distance and ratio tests and on exact
ties at tile and strip boundaries; shuffled and repeated batches; the reference's matcher scenarios."""
import ctypes

import numpy as np
import pytest

import oracle_sm
from colmap_b200.feature_matching import (CreateSiftFeatureMatcher, FeatureMatcherImage, FeatureMatchingOptions,
                                          SiftMatchingOptions, _COptions, _lib)
from colmap_b200.synthetic import CreateRandomFeatureDescriptors, make_sift_view_pair
from test_sift_matching_cpu import libm_acosf, reference_scenarios

pytestmark = pytest.mark.gpu

SIZES = [1, 2, 63, 64, 65, 127, 129, 1000, 8192]


def _options(max_ratio=0.8, max_distance=0.7, cross_check=True, max_num_matches=32768):
    return FeatureMatchingOptions(gpu_index="0", max_num_matches=max_num_matches,
                                  sift=SiftMatchingOptions(max_ratio, max_distance, cross_check))


def _pair(kind, n1, n2, seed):
    if kind == "ties":
        a, b = CreateRandomFeatureDescriptors(n1, seed=seed), CreateRandomFeatureDescriptors(n2, seed=seed + 7919)
        k = min(n1, n2) // 3
        b[:k] = a[n1 - k:][::-1]          # exact copies in other positions: ties between copies and their near twins
        return a, b
    a, b, _ = make_sift_view_pair(n1, n2, seed=seed)
    rng = np.random.default_rng(seed + 1)
    if kind == "zeros":                   # all-zero rows in both images: dot 0 with everything, never a match
        a[rng.random(n1) < 0.3] = 0
        b[rng.random(n2) < 0.3] = 0
    elif kind == "clamp":                 # brightened rows whose dot with their copy exceeds 2^18: acos argument 1
        sel = rng.random(n1) < 0.5
        a[sel] = np.minimum(a[sel].astype(np.int32) * 2, 255).astype(np.uint8)
        sel = rng.random(n2) < 0.5
        b[sel] = np.minimum(b[sel].astype(np.int32) * 2, 255).astype(np.uint8)
    return a, b


_GRID_CACHE = {}


def _grid_images(kind):
    if kind not in _GRID_CACHE:
        images, pairs = [], []
        for i, n1 in enumerate(SIZES):
            for j, n2 in enumerate(SIZES):
                a, b = _pair(kind, n1, n2, seed=100 * i + j)
                images += [FeatureMatcherImage(len(images), a), FeatureMatcherImage(len(images) + 1, b)]
                pairs.append((len(images) - 2, len(images) - 1))
        _GRID_CACHE[kind] = (images, pairs)
    return _GRID_CACHE[kind]


@pytest.mark.parametrize("kind", ["ties", "view", "zeros", "clamp"])
@pytest.mark.parametrize("cross_check", [True, False])
@pytest.mark.parametrize("ratio_distance", [(0.8, 0.7), (0.4, 0.7), (1.0, 1.2)])
def test_grid_equals_oracle(kind, cross_check, ratio_distance):
    r, dmax = ratio_distance
    images, pairs = _grid_images(kind)
    with CreateSiftFeatureMatcher(_options(r, dmax, cross_check)) as m:
        got = m.MatchPairs(images, pairs)
    total = 0
    for (i, j), g in zip(pairs, got):
        ref = oracle_sm.match(images[i].descriptors, images[j].descriptors, r, dmax, cross_check)
        assert np.array_equal(g, ref), (kind, len(images[i].descriptors), len(images[j].descriptors))
        total += len(ref)
    assert total > 0


def test_clamp_kind_reaches_the_clamp():
    a, b = _pair("clamp", 1000, 1000, seed=5)
    D = a.astype(np.int64) @ b.astype(np.int64).T
    assert (D.max(axis=1) > 262144).sum() > 100


# ---- crafted dot products -------------------------------------------------------------------------------------------
Q = np.full(128, 255, np.uint8)
Q[0] = 1


def row_with_dot(v):
    """A row y with dot(Q, y) == v exactly: y[0] = v mod 255, and v // 255 spread over the other components."""
    y = np.zeros(128, np.uint8)
    y[0] = v % 255
    s = v // 255
    assert s <= 127 * 255
    full, rem = divmod(s, 255)
    y[1:1 + full] = 255
    if rem:
        y[1 + full] = rem
    return y


def _column_image(n, values):
    """n zero rows (dot 0) with row p set to reach dot values[p]."""
    b = np.zeros((n, 128), np.uint8)
    for p, v in values.items():
        b[p] = row_with_dot(v)
    return b


def _acos_tables():
    k = np.arange(262145)
    x = (k.astype(np.float64) / 262144.0).astype(np.float32)
    return libm_acosf(x), np.arccos(x.astype(np.float64)).astype(np.float32)


def crafted_cases(max_ratio=0.8, max_distance=0.7):
    """Single-row queries whose best and second dot products sit where the distance and ratio tests are decided:
    best on the arguments around max_distance (and on the arguments within 2000 of it where acosf and the correctly
    rounded arccos disagree), and every (best, second) within 3 arguments of d1 == max_ratio * d2 whose decision differs
    between acosf and the rounded double arccos.  Returns the cases ({column: dot}) and the number of such flips."""
    f, cr = _acos_tables()
    disagree = np.nonzero(f != cr)[0]
    r, dm = np.float32(max_ratio), np.float32(max_distance)
    cases = []
    thr = int(np.searchsorted(-f, -dm))
    near = np.union1d(disagree[np.abs(disagree - thr) <= 2000], np.arange(thr - 3, thr + 4))
    for b in near:
        cases.append({3: int(b), 9: 1000})
    s = np.arange(1, 262145)
    c = np.searchsorted(-f, -(r * f[s]))
    flips = []
    for d in range(-3, 4):
        b = np.clip(c + d, 1, 262144)
        flip = ((f[b] >= r * f[s]) != (cr[b] >= r * cr[s])) & (b > s) & ~(f[b] > dm)
        flips += list(zip(b[flip], s[flip]))
    for b, s2 in flips:
        cases.append({5: int(b), 130: int(s2)})          # best and second in different column tiles
    return cases, len(flips)


def _run_cases(cases, n2=300, **opts):
    images, pairs = [], []
    for c in cases:
        images += [FeatureMatcherImage(len(images), Q[None].copy()), FeatureMatcherImage(len(images) + 1, _column_image(n2, c))]
        pairs.append((len(images) - 2, len(images) - 1))
    with CreateSiftFeatureMatcher(_options(**opts)) as m:
        got = m.MatchPairs(images, pairs)
    for (i, j), g in zip(pairs, got):
        ref = oracle_sm.match(images[i].descriptors, images[j].descriptors, opts.get("max_ratio", 0.8),
                              opts.get("max_distance", 0.7), opts.get("cross_check", True))
        assert np.array_equal(g, ref), cases[i // 2]
    return got


@pytest.mark.parametrize("cross_check", [True, False])
@pytest.mark.parametrize("max_distance", [0.7, 1.6])
def test_crafted_thresholds_where_acosf_decides(cross_check, max_distance):
    cases, flips = crafted_cases(max_distance=max_distance)
    assert flips > 0      # some of these decisions would differ with a correctly rounded arccos
    got = _run_cases(cases, max_distance=max_distance, cross_check=cross_check)
    assert 0 < sum(len(g) for g in got) < len(cases)


@pytest.mark.parametrize("p, q", [(127, 128), (128, 127), (255, 256), (256, 255), (0, 299), (128, 256), (1, 2)])
def test_crafted_exact_ties_across_tiles_take_the_first_column(p, q):
    """best tied at columns p and q (in different 128-column tiles but for (1, 2)): second == best, so only a
    max_ratio above 1 accepts the row, and then the match is the first of the tied columns."""
    v = 250000
    for cc in (False, True):
        got = _run_cases([{p: v, q: v}, {p: v, q: v, 40: v}, {p: v, q: v, 290: 1000}], max_ratio=1.5,
                         max_distance=1.6, cross_check=cc)
        for g, first in zip(got, (min(p, q), min(p, q, 40), min(p, q))):
            assert np.array_equal(g, np.array([[0, first]], np.uint32))
    got = _run_cases([{p: v, q: v}], max_ratio=1.0, max_distance=1.6, cross_check=False)
    assert len(got[0]) == 0            # d1 >= 1.0 * d2 when best == second


@pytest.mark.parametrize("p, q", [(127, 128), (255, 256), (0, 383), (126, 129)])
def test_crafted_exact_ties_across_row_strips_take_the_first_row(p, q):
    """The transposed direction: query rows p and q (in different 128-row strips) are identical, so every column ties
    between them; without cross-check both rows match the same column, with it only the first row p survives (a
    max_ratio above 1 lets the tied column through its own ratio test)."""
    a = np.zeros((400, 128), np.uint8)
    a[p] = a[q] = row_with_dot(200000)
    b = np.zeros((10, 128), np.uint8)
    b[4] = Q
    b[7] = row_with_dot(300)          # a weak second column for rows p and q
    for cc in (False, True):
        with CreateSiftFeatureMatcher(_options(max_ratio=1.5, max_distance=1.6, cross_check=cc)) as m:
            got = m.Match(FeatureMatcherImage(1, a), FeatureMatcherImage(2, b))
        ref = oracle_sm.match(a, b, 1.5, 1.6, cc)
        assert np.array_equal(got, ref)
        want = [[p, 4]] if cc else [[p, 4], [q, 4]]
        assert np.array_equal(got, np.array(want, np.uint32))


# ---- batches ----------------------------------------------------------------------------------------------------------
def _block(seed=11):
    """About 20 views of one scene of unequal sizes, one empty: each holds noisy copies of a random subset of a shared
    pool of rows plus rows of its own."""
    rng = np.random.default_rng(seed)
    sizes = [int(n) for n in rng.integers(1, 1500, 18)] + [0, 1300]
    rng.shuffle(sizes)
    pool, own, _ = make_sift_view_pair(1500, 3000, overlap=0.0, seed=seed)
    images = []
    for k, n in enumerate(sizes):
        shared = int(n * 0.7)
        rows = np.concatenate([pool[rng.choice(1500, shared, replace=False)], own[rng.choice(3000, n - shared, replace=False)]])
        noisy = rows.astype(np.int32) + rng.integers(-12, 13, rows.shape)
        d = np.clip(noisy, 0, 255).astype(np.uint8)[rng.permutation(n)]
        images.append(FeatureMatcherImage(1000 + k, d))
    return images


def test_exhaustive_block_equals_per_pair_match_and_oracle_in_any_order():
    images = _block()
    pairs = [(i, j) for i in range(len(images)) for j in range(i + 1, len(images))]
    mnm = 1000                          # one image holds more rows than max_num_matches
    assert max(len(im.descriptors) for im in images) > mnm and min(len(im.descriptors) for im in images) == 0
    with CreateSiftFeatureMatcher(_options(max_num_matches=mnm)) as m:
        got = m.MatchPairs(images, pairs)
        again = m.MatchPairs(images, pairs)
        perm = np.random.default_rng(1).permutation(len(pairs))
        shuffled = m.MatchPairs(images, [pairs[k] for k in perm])
        single = [m.Match(images[i], images[j]) for (i, j) in pairs[::7]]
    total = 0
    for k, (i, j) in enumerate(pairs):
        ref = oracle_sm.match(images[i].descriptors, images[j].descriptors, max_num_matches=mnm)
        assert np.array_equal(got[k], ref), (i, j)
        assert np.array_equal(again[k], ref)
        total += len(ref)
    for k, pk in enumerate(perm):
        assert np.array_equal(shuffled[k], got[pk])
    for g, k in zip(single, range(0, len(pairs), 7)):
        assert np.array_equal(g, got[k])
    assert total > 0


def test_match_reuploads_only_when_the_image_id_changes():
    a, b, _ = make_sift_view_pair(500, 400, seed=21)
    c = CreateRandomFeatureDescriptors(300, seed=5)
    with CreateSiftFeatureMatcher(_options()) as m:
        first = m.Match(FeatureMatcherImage(1, a), FeatureMatcherImage(2, b))
        # same ids: the cached descriptors are used (as SiftGPUFeatureMatcher::Match does)
        cached = m.Match(FeatureMatcherImage(1, c), FeatureMatcherImage(2, b))
        fresh = m.Match(FeatureMatcherImage(3, c), FeatureMatcherImage(2, b))
    assert np.array_equal(first, oracle_sm.match(a, b)) and np.array_equal(cached, first)
    assert np.array_equal(fresh, oracle_sm.match(c, b))


def test_reference_scenarios_on_the_gpu():
    def match(d1, d2, **kw):
        with CreateSiftFeatureMatcher(_options(**kw)) as m:
            return m.Match(FeatureMatcherImage(1, np.ascontiguousarray(d1)), FeatureMatcherImage(2, np.ascontiguousarray(d2)))
    reference_scenarios(match)


# ---- refusals that need a handle ----------------------------------------------------------------------------------------
def test_slot_out_of_range_and_short_capacity_are_refused_and_the_handle_stays_usable():
    L = _lib()
    c = _COptions()
    L.b200sm_options_init(ctypes.byref(c))
    c.gpu_index = 0
    h = ctypes.c_void_p()
    assert L.b200sm_create(ctypes.byref(c), 2, ctypes.byref(h)) == 0
    try:
        a, b, _ = make_sift_view_pair(300, 200, seed=2)
        u8 = ctypes.POINTER(ctypes.c_uint8)
        assert L.b200sm_set_descriptors(h, 2, len(a), a.ctypes.data_as(u8)) == -1
        assert L.b200sm_set_descriptors(h, -1, len(a), a.ctypes.data_as(u8)) == -1
        assert L.b200sm_set_descriptors(h, 0, 5, None) == -1
        assert L.b200sm_set_descriptors(h, 0, len(a), a.ctypes.data_as(u8)) == 0
        assert L.b200sm_set_descriptors(h, 1, len(b), b.ctypes.data_as(u8)) == 0
        i32 = ctypes.POINTER(ctypes.c_int)
        s1, s2, bad = np.array([0, 1], np.int32), np.array([1, 0], np.int32), np.array([0, 2], np.int32)
        off = np.zeros(3, np.uint64)
        out = np.zeros((400, 2), np.uint32)
        offp, outp = off.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32))
        assert L.b200sm_match_capacity(h, 2, s1.ctypes.data_as(i32), s2.ctypes.data_as(i32)) == 400
        assert L.b200sm_match_pairs(h, 2, s1.ctypes.data_as(i32), bad.ctypes.data_as(i32), offp, outp, 400) == -1
        assert "slot" in L.b200sm_last_error().decode()
        assert L.b200sm_match_pairs(h, 2, s1.ctypes.data_as(i32), s2.ctypes.data_as(i32), offp, outp, 399) == -1
        assert "capacity" in L.b200sm_last_error().decode()
        assert not off.any() and not out.any()
        assert L.b200sm_match_pairs(h, 2, s1.ctypes.data_as(i32), s2.ctypes.data_as(i32), offp, outp, 400) == 0
        k = int(off[1])
        assert np.array_equal(out[:k], oracle_sm.match(a, b)) and np.array_equal(out[k:int(off[2])], oracle_sm.match(b, a))
    finally:
        L.b200sm_destroy(h)
