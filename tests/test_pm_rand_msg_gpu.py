"""Passes R (pm_rand_kernel) and M (pm_msg_kernel) against their column-serial statement.  R runs one warp per column:
lane 0 walks the column's XORWOW stream and leaves each row's start state in a 32-row ring, from which lane k computes
row k.  M runs the backward and forward recurrences interleaved, with each step's likelihood computed ahead of the
chain.  A run stopped after k sweeps (B200PM_MAX_SWEEPS) leaves the state sweep k starts from: b200pm_debug_rand_msg
runs that sweep's R and M on the GPU, and b200pm_test_rand_msg runs the column-serial loops on the host over the same
state.  The random hypotheses, Monte-Carlo uniforms, backward and forward messages and RNG border slots must agree bit
for bit.  A lane restarted from the wrong row of the ring, or a step fed the wrong row's cost, shows here even where the
final maps would hide it (a random hypothesis that loses, a uniform that picks the same image)."""
import ctypes
import os

import numpy as np
import pytest

from colmap_b200.patch_match import PatchMatch, PatchMatchOptions
from colmap_b200.synthetic import make_patch_match_scene

pytestmark = pytest.mark.gpu

KEYS = ("rand_hyp", "usamp", "sel", "fwd", "rng")


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _buffers(w, h, n, ns):
    return dict(rand_hyp=np.full((h * w, 4), np.nan, np.float32), usamp=np.full((h * w, ns), np.nan, np.float32),
                sel=np.full((h * w, n), np.nan, np.float32), fwd=np.full((h * w, n), np.nan, np.float32),
                rng=np.zeros((2 * w + 2 * h, 6), np.uint32))


def _rand_msg(o, problem, k):
    """R and M of sweep k on the GPU and on the host, from the state a run stopped after k sweeps left."""
    h, w = problem.images[problem.ref_image_idx].bitmap.shape[:2]
    n = len(problem.src_image_idxs)
    os.environ["B200PM_MAX_SWEEPS"] = str(k)
    try:
        pm = PatchMatch(o, problem)
        pm.Run()
    finally:
        os.environ.pop("B200PM_MAX_SWEEPS", None)
    try:
        lib = pm._lib
        lib.b200pm_test_rand_msg.argtypes = [ctypes.c_void_p] * 7
        lib.b200pm_debug_rand_msg.argtypes = [ctypes.c_void_p] * 6
        host, gpu = _buffers(w, h, n, o.num_samples), _buffers(w, h, n, o.num_samples)
        rounds = np.zeros(h * w, np.uint8)
        assert lib.b200pm_test_rand_msg(pm._h, *(_ptr(host[key]) for key in KEYS), _ptr(rounds)) == 0   # reads only
        assert lib.b200pm_debug_rand_msg(pm._h, *(_ptr(gpu[key]) for key in KEYS)) == 0
    finally:
        pm.close()
    return host, gpu, rounds


def _assert_same(host, gpu):
    for key in KEYS:
        a, b = host[key].view(np.uint32), gpu[key].view(np.uint32)
        diff = a != b
        assert not diff.any(), f"{key}: {diff.sum()} of {diff.size} words differ, first at {np.argwhere(diff)[:4].tolist()}"


def _options(sc, ns, geom=False):
    return PatchMatchOptions(depth_min=sc["depth_min"], depth_max=sc["depth_max"], geom_consistency=geom,
                             num_iterations=1, window_radius=2, window_step=1, num_samples=ns)


# k even: the sweep walks frame 0 or 2 (W columns of H rows); k odd: frame 1 or 3 (H columns of W rows)
@pytest.mark.parametrize("k", [0, 1, 2, 3])
@pytest.mark.parametrize("w,h,n,ns", [
    (37, 29, 3, 15),   # 29 / 37 rows: one partial ring block, then one full block and a partial one
    (70, 45, 1, 15),   # N = 1; 45 / 70 rows: two and three ring blocks
    (1, 23, 3, 15),    # one pixel wide: one column of 23 rows, then 23 columns of one row
    (23, 21, 8, 1),    # one Monte-Carlo sample per row
    (22, 19, 9, 40),   # N = 9; more samples per row than a warp has lanes
    (33, 34, 8, 15),   # one column and one row past a multiple of 32
])
def test_rand_msg_bit_exact_vs_column_serial(w, h, n, ns, k):
    sc = make_patch_match_scene(w, h, n, seed=60 + n + w)
    host, gpu, _ = _rand_msg(_options(sc, ns), sc["problem"], k)
    _assert_same(host, gpu)


@pytest.mark.parametrize("k", [0, 1])
def test_rand_msg_every_rounds_count(k):
    """An early sweep (perturbation 1 and 2^-1/4): PerturbNormal rejects often enough that every row length occurs,
    1 to 4 rounds of three draws, so lane 0's walk and the lanes' restarts meet every stream offset a row can have."""
    sc = make_patch_match_scene(70, 45, 3, seed=71)
    host, gpu, rounds = _rand_msg(_options(sc, 15), sc["problem"], k)
    _assert_same(host, gpu)
    seen = set(np.unique(rounds).tolist())
    assert seen == {1, 2, 3, 4}, f"rounds seen: {sorted(seen)}"


@pytest.mark.parametrize("k", [0, 1, 2, 3])
def test_rand_msg_geometric(k):
    sc = make_patch_match_scene(35, 26, 4, seed=9, with_gt_maps=True)
    prob = sc["problem"]
    rng = np.random.default_rng(5)
    prob.depth_maps = [(d * (1 + 0.002 * rng.standard_normal(d.shape))).astype(np.float32) for d in sc["depth_maps"]]
    prob.normal_maps = [nm.copy() for nm in sc["normal_maps"]]
    host, gpu, _ = _rand_msg(_options(sc, 9, geom=True), prob, k)
    _assert_same(host, gpu)
