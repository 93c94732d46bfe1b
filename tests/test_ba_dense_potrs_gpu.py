"""The fp64 tiled triangular solves (ba_dense_potrs in colmap_b200/csrc/ba_dense_f64.cu) on their own, through the
library's test hook b200ba_test_dense_potrs (ba_dense_potrf, then ba_dense_potrs on nrhs device columns), against
LAPACK's Cholesky solve (scipy.linalg.cho_solve) up to n = 4,097 and closed-form products at n = 32,768.

* Accuracy: the SPD inputs Q diag(s) Q^T of tests/test_ba_dense_f64_gpu.py (kappa 1 to 1e12), padded to a multiple of
  64 with an identity block, at every size around the 64-row tile (1 to 3 tiles and every ragged tail), n = 1,000 and
  4,097, with 1, 2 and 3 right-hand sides.  Bars: backward error ||A x - b|| / (||A|| ||x|| + ||b||) <= C n eps and
  forward error ||x - x_ref|| / ||x_ref|| <= C n eps kappa per column, C = 1 (see C_BAR).  Every case also holds the
  layout: the strict upper triangle goes in as NaN with a payload and the scratch W goes in as the same NaN, and the
  solution must be finite (neither is read before it is written); the padding rows of B go in as zero and must come back
  exactly zero.
* Right-hand sides: column j of a 3-column solve is bit-identical to the 1-column solve of that column and to the same
  column solved in a permuted order, with column magnitudes 1e-150, 1 and 1e150 so any mixing between columns shows;
  two repeated solves are bit-identical.
* Failed factorisation: a bad pivot in the first tile or in a later one sets the flag, and every launch of the solve
  returns at once: B and W come back bit-identical.
* Envelope: the closed-form A = diag(d) + G G^T of test_envelope_32768 at n = 32,768 (512 tiles) with 3 right-hand
  sides, and at n = 32,700 padded to N = 32,704, against ||A x - b||_max <= C n eps kappa ||x||_max."""
import ctypes
import functools

import numpy as np
import pytest
import scipy.linalg
import torch

from colmap_b200._lib import load_library
from test_ba_dense_f64_gpu import NAN_PAYLOAD, _ldl, _padded, _spd, to_device

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
# Measured on one H100 80GB HBM3 (700 W) over every case here, worst error / bar scale: backward 0.11 (n eps), forward
# 0.016 (n eps kappa), envelope residual 6.8e-5 (n eps kappa ||x||_max).  C = 1 keeps a margin of 9x or more.
C_BAR = 1.0
NAN = NAN_PAYLOAD.view(np.float64)
WORST = {}


def _hook():
    lib = load_library()
    f = lib.b200ba_test_dense_potrs
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                  ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)]
    f.restype = ctypes.c_int
    lib.b200ba_last_error.restype = ctypes.c_char_p
    return lib, f


def potrs(T, n_check, B, W):
    """ba_dense_potrf on the device matrix T, then ba_dense_potrs on the device columns B [nrhs, N] (in place) with
    scratch W [nrhs, N] -> (rc, bad_row, bad_pivot)."""
    lib, f = _hook()
    assert B.shape == W.shape and B.shape[1] == T.shape[0] and B.is_contiguous() and W.is_contiguous()
    row, piv = ctypes.c_int(-1), ctypes.c_double(0.0)
    rc = f(T.data_ptr(), T.shape[0], n_check, B.shape[0], B.data_ptr(), W.data_ptr(), ctypes.byref(row), ctypes.byref(piv))
    assert rc in (0, 1), (rc, lib.b200ba_last_error().decode())
    return rc, row.value, piv.value


def _columns(b, N):
    """Right-hand sides b [n, nrhs] as the device's [nrhs, N] columns, padding rows zero."""
    out = np.zeros((b.shape[1], N))
    out[:, :b.shape[0]] = b.T
    return torch.from_numpy(out).cuda()


def _nan_scratch(shape):
    return torch.from_numpy(np.full(shape, NAN)).cuda()


def solve(M, n, b):
    """Solve with the padded matrix M (order N) and right-hand sides b [n, nrhs] -> the device's [nrhs, N] result."""
    N = M.shape[0]
    B = _columns(b, N)
    rc = potrs(to_device(M), n, B, _nan_scratch(B.shape))
    assert rc == (0, 0, 0.0)
    return B.cpu().numpy()


def _note(name, value):
    WORST[name] = max(WORST.get(name, 0.0), float(value))


@functools.lru_cache(maxsize=4)
def _case(n, kappa):
    A = _spd(n, kappa, np.random.default_rng(n))
    return A, scipy.linalg.cho_factor(A, lower=True)


SIZES = [(n, kappa) for n in (1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 1000, 4097) for kappa in (1.0, 1e4, 1e12)]


@pytest.mark.parametrize("n,kappa", SIZES, ids=lambda v: f"{v:g}")
def test_solve_accuracy_and_layout(n, kappa):
    A, cho = _case(n, kappa)
    N = -(-n // 64) * 64
    M = _padded(A, N)
    Al = A.astype(np.longdouble)
    normA = 1.0                        # ||A||_2: the largest of the eigenvalues set by _spd
    rng = np.random.default_rng(10 * n + 1)
    for nrhs in (1, 2, 3):
        b = rng.standard_normal((n, nrhs))
        X = solve(M, n, b)
        assert np.isfinite(X).all(), "upper triangle or scratch read before written"
        assert (X[:, n:] == 0).all(), "padding rows"
        x = X[:, :n].T
        x_ref = scipy.linalg.cho_solve(cho, b)
        r = (Al @ x.astype(np.longdouble) - b).astype(np.float64)   # the residual in extended precision
        for j in range(nrhs):
            back = np.linalg.norm(r[:, j]) / (normA * np.linalg.norm(x[:, j]) + np.linalg.norm(b[:, j]))
            fwd = np.linalg.norm(x[:, j] - x_ref[:, j]) / np.linalg.norm(x_ref[:, j])
            _note("backward / (n eps)", back / (n * EPS))
            _note("forward / (n eps kappa)", fwd / (n * EPS * kappa))
            assert back <= C_BAR * n * EPS, (nrhs, j, back, C_BAR * n * EPS)
            assert fwd <= C_BAR * n * EPS * kappa, (nrhs, j, fwd, C_BAR * n * EPS * kappa)


@pytest.mark.parametrize("n", [65, 193, 1000])
def test_right_hand_sides_are_independent(n):
    A, _ = _case(n, 1e4)
    N = -(-n // 64) * 64
    M = _padded(A, N)
    b = np.random.default_rng(n + 7).standard_normal((n, 3)) * np.array([1e-150, 1.0, 1e150])
    X3 = solve(M, n, b)
    assert np.isfinite(X3).all()
    bits = X3.view(np.int64)
    assert np.array_equal(solve(M, n, b).view(np.int64), bits), "repeated solve"
    for j in range(3):
        assert np.array_equal(solve(M, n, b[:, j:j + 1]).view(np.int64)[0], bits[j]), f"column {j} alone"
    perm = [2, 0, 1]
    Xp = solve(M, n, b[:, perm]).view(np.int64)
    for k, j in enumerate(perm):
        assert np.array_equal(Xp[k], bits[j]), f"column {j} in position {k}"


@pytest.mark.parametrize("row", [10, 130])
def test_failed_factorisation_leaves_b_and_w(row):
    """A bad pivot in tile 0 or tile 2 of a 256-row matrix: the flag is set and no solve launch touches B or W."""
    N = 256
    D = np.ones(N)
    D[row] = -1.0
    T = to_device(_ldl(N, D, np.random.default_rng(row)))
    B0 = np.random.default_rng(1).standard_normal((3, N))
    W0 = np.random.default_rng(2).standard_normal((3, N))
    B, W = torch.from_numpy(B0.copy()).cuda(), torch.from_numpy(W0.copy()).cuda()
    rc, bad_row, piv = potrs(T, 200, B, W)
    assert (rc, bad_row) == (1, row) and piv == pytest.approx(-1.0, rel=1e-6)
    assert np.array_equal(B.cpu().numpy().view(np.int64), B0.view(np.int64))
    assert np.array_equal(W.cpu().numpy().view(np.int64), W0.view(np.int64))


@pytest.mark.parametrize("n,N", [(32768, 32768), (32700, 32704)])
def test_envelope(n, N):
    """A = diag(d) + G G^T as in test_envelope_32768 (an 8.6 GB matrix), padded to N with an identity block, 3
    right-hand sides; A x costs two thin products.  kappa is bounded by (max d + ||G||_2^2) / min d."""
    dev = "cuda"
    idx = torch.arange(n, device=dev)
    i = idx.to(torch.float64)
    d = 1.0 + (idx % 7).to(torch.float64) / 7.0
    G = torch.stack([np.sqrt(2.0 * s / n) * torch.cos(w * i + p)
                     for s, w, p in ((8.0, 1e-3, 0.1), (4.0, 7.3e-3, 1.3), (2.0, 0.0517, 2.1), (1.0, 0.731, 0.4))], 1)
    kappa = (d.max() + torch.linalg.eigvalsh(G.T @ G).max()).item() / d.min().item()
    g = torch.Generator(device=dev).manual_seed(n)
    b = torch.randn((3, n), dtype=torch.float64, device=dev, generator=g) * torch.tensor([[1e-3], [1.0], [1e3]], device=dev,
                                                                                          dtype=torch.float64)
    B = torch.zeros((3, N), dtype=torch.float64, device=dev)
    B[:, :n] = b
    W = torch.full((3, N), float("nan"), dtype=torch.float64, device=dev)
    try:
        T = torch.zeros((N, N), dtype=torch.float64, device=dev)
        for r0 in range(0, n, 2048):            # symmetric: row block r of T = rows of A
            r1 = min(n, r0 + 2048)
            T[r0:r1, :n] = G[r0:r1] @ G.T
        T.diagonal()[:n].add_(d)
        T.diagonal()[n:] = 1.0
        assert potrs(T, n, B, W) == (0, 0, 0.0)
    finally:
        T = None
        torch.cuda.empty_cache()
    assert (B[:, n:] == 0).all(), "padding rows"
    x = B[:, :n].T
    R = d[:, None] * x + G @ (G.T @ x) - b.T
    for j in range(3):
        res, xm = R[:, j].abs().max().item(), x[:, j].abs().max().item()
        _note("envelope residual / (n eps kappa ||x||)", res / (n * EPS * kappa * xm))
        assert res <= C_BAR * n * EPS * kappa * xm, (j, res, kappa, xm)


def test_report_margins():
    print(f"worst error ratios (bar: {C_BAR}): {WORST}")
