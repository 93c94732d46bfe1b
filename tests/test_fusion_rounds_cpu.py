"""The round schedule for a parallel stereo fusion (DESIGN.md section 6c), checked on its CPU model
(tests/oracle_fuse_rounds.py) against the serial oracle (oracle/ws_oracle.py: fuse): equality where no traversal can
conflict, the disjointness that makes the committed seeds a serial execution, the fact that marking pixels outside a
traversal's claim set does not change it, and the fused cloud on the rendered scenes of test_fusion_cpu.py."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ws_oracle  # noqa: E402

import oracle_fuse_rounds as rounds  # noqa: E402
from colmap_b200.mvs_fusion import StereoFusionOptions  # noqa: E402
from test_fusion_cpu import _oracle_inputs, _scene  # noqa: E402

OPTION_SETS = [(0, 0.0, {}), (1, 0.002, dict(min_num_pixels=2, max_traversal_depth=3)),
               (2, 0.004, dict(min_num_pixels=2, max_num_pixels=4, max_normal_error=25.0, max_depth_error=0.02))]


def _same(a, b):
    xyz, nrm, rgb, vis = a[:4]
    exyz, enrm, ergb, evis = b[:4]
    assert len(xyz) == len(exyz)
    assert np.array_equal(xyz.view(np.uint32), exyz.view(np.uint32))
    assert np.array_equal(nrm.view(np.uint32), enrm.view(np.uint32))
    assert np.array_equal(rgb, ergb) and [list(v) for v in vis] == [list(v) for v in evis]


@pytest.mark.parametrize("seed,noise,kw", OPTION_SETS)
def test_model_is_the_serial_oracle_when_traversals_cannot_conflict(seed, noise, kw):
    # max_traversal_depth = 1: every traversal claims its seed pixel only
    images, overlap = _scene(40, 30, 3, seed, noise)
    o = StereoFusionOptions(**{**kw, "max_traversal_depth": 1, "min_num_pixels": 1})
    opt, ims = _oracle_inputs(o, images)
    got = rounds.fuse_rounds(opt, ims, overlap)
    _same(got, ws_oracle.fuse(opt, ims, overlap))
    assert len(got[0]) > 1000 and got[4]["image_rounds"] == [rounds.TILE ** 2] * 4    # one seed per tile per round
    # a single used image: nothing to traverse to
    for k in range(1, 4):
        images[k].used = False
    o = StereoFusionOptions(**{**kw, "min_num_pixels": 1})
    opt, ims = _oracle_inputs(o, images)
    got = rounds.fuse_rounds(opt, ims, overlap)
    _same(got, ws_oracle.fuse(opt, ims, overlap))
    assert len(got[0]) > 1000 and got[4]["rounds"] == rounds.TILE ** 2


@pytest.mark.parametrize("seed,noise,kw", OPTION_SETS)
def test_committed_seeds_form_a_serial_execution(seed, noise, kw):
    images, overlap = _scene(40, 30, 3, seed, noise)
    opt, ims = _oracle_inputs(StereoFusionOptions(**kw), images)
    stats = rounds.fuse_rounds(opt, ims, overlap)[4]
    assert stats["rounds"] > 4                             # there were conflicts to resolve
    for committed in stats["committed"]:
        assert committed                                   # the lowest-ranked pending seed always commits
        seen = set()
        for rank, claims in committed:                     # pairwise disjoint claim sets
            assert rank == committed[0][0] or claims       # a committed seed claims at least its seed pixel
            assert seen.isdisjoint(claims)
            seen.update(claims)


def test_marks_outside_the_claim_set_do_not_change_a_traversal():
    images, overlap = _scene(40, 30, 3, 1, 0.002)
    opt, ims = _oracle_inputs(StereoFusionOptions(min_num_pixels=2), images)
    f = rounds.Fusion(opt, ims, overlap)
    rng = np.random.default_rng(7)
    shapes = [m.shape for m in f.masks]
    checked = 0
    for _ in range(40):
        base = [rng.random(s) < 0.3 for s in shapes]
        row, col = int(rng.integers(2, 30)), int(rng.integers(0, 40))
        base[0][row, col] = False
        claims, point = f.traverse(0, row, col, base)
        if len(claims) < 2:
            continue
        C = set(claims)
        # marking any pixels outside C leaves the traversal as it was (marks are only ever added)
        other = [m.copy() for m in base]
        for i, m in enumerate(other):
            add = rng.random(m.shape) < 0.5
            for (j, r, c) in C:
                if j == i:
                    add[r, c] = False
            m |= add
        assert f.traverse(0, row, col, other) == (claims, point)
        # masking one pixel of C changes it
        j, r, c = claims[int(rng.integers(0, len(claims)))]
        inside = [m.copy() for m in base]
        inside[j][r, c] = True
        assert f.traverse(0, row, col, inside)[0] != claims
        checked += 1
    assert checked >= 20


@pytest.mark.parametrize("seed,noise,kw", OPTION_SETS)
def test_model_fuses_like_the_serial_oracle_on_the_rendered_scenes(seed, noise, kw):
    """The round schedule is the serial algorithm on another seed order, so the clouds differ but should be alike.
    Measured on the three scenes: point counts -16.4 %, -2.5 %, +0.26 % against the serial oracle (the noiseless scene
    groups its pixels into fewer, larger points when the seeds start on the 4 x 4 lattice), median surface error
    0.90x, 0.98x, 0.97x the serial one (rounds per seed image 18/13/12/8, 16/14/8/8, 16/9/8/13).  Bars: 20 % and 1.5x."""
    images, overlap = _scene(40, 30, 3, seed, noise)
    o = StereoFusionOptions(**kw)
    opt, ims = _oracle_inputs(o, images)
    got = rounds.fuse_rounds(opt, ims, overlap)
    ser = ws_oracle.fuse(opt, ims, overlap)
    assert abs(len(got[0]) - len(ser[0])) <= 0.20 * len(ser[0])
    im0 = images[0]

    def surface_error(xyz):
        pc = (np.asarray(im0.R, np.float64) @ xyz.T.astype(np.float64)).T + np.asarray(im0.T, np.float64)
        uv = (np.asarray(im0.K, np.float64) @ pc.T).T
        u, v = np.round(uv[:, 0] / uv[:, 2]).astype(int), np.round(uv[:, 1] / uv[:, 2]).astype(int)
        ok = (u >= 0) & (v >= 2) & (u < 40) & (v < 30)
        assert ok.mean() > 0.5
        return np.median(np.abs(pc[ok, 2] - im0.depth_map[v[ok], u[ok]]) / pc[ok, 2])

    assert surface_error(got[0]) <= 1.5 * surface_error(ser[0]) + 1e-6
    assert np.allclose(np.linalg.norm(got[1], axis=1), 1.0, atol=1e-6)
