"""The fp64 tiled Cholesky and SPD inverse (colmap_b200/csrc/ba_dense_f64.cu) on their own, through the library's test
hook b200ba_test_dense_f64, against LAPACK (numpy) up to n = 4,097 and cuBLAS fp64 products at n = 32,768.

* Accuracy: SPD inputs Q diag(s) Q^T with a set condition number kappa (1 to 1e12), padded to a multiple of 64 with an
  identity block, at every size around the 64-row tile (1 to 3 tiles, the first trailing-update grids of 1 and 3 tiles,
  every ragged tail), n = 1,000 and 4,097, and one closed-form matrix at the documented envelope n = 32,768 (512 tiles,
  trailing-update grids up to 130,816 CTAs).  Bars: backward error ||A - L L^T||_F / ||A||_F <= C n eps, forward error
  of L and of X = A^-1, and ||A X - I||_max, all <= C n eps kappa.  C = 1 (see C_BAR).  A dropped K chunk, a wrong
  mask or a misplaced tile gives errors of order one, far above every bar that is asserted.
* Upper triangle: the strict upper triangle goes in as NaN with a payload.  The results must be finite (no kernel reads
  it), and outside the 64 x 64 diagonal tiles every NaN must come back bit-identical (no kernel writes it).
* Pivot flag: A = L0 D L0^T with a unit lower L0 and D = 1 except at chosen rows; the first failing row and its pivot
  are reported, rows at or past n_check are not tested, rows before n_test0 fail only on a pivot <= 0, and a failed
  factorisation turns the inverse into a no-op."""
import ctypes

import numpy as np
import pytest
import torch

from colmap_b200._lib import load_library

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
# Measured on one H100 over every case here, worst error / bar scale: factor backward 0.0625 (n eps), factor forward
# 3.4e-5, inverse residual 0.10, inverse forward 0.031 (n eps kappa).  C = 1 keeps a 10x margin above the worst of them.
C_BAR = 1.0
NAN_PAYLOAD = np.int64(0x7FF8_0000_DEAD_BEEF)
WORST = {}


def _hook():
    lib = load_library()
    f = lib.b200ba_test_dense_f64
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int,
                  ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double)]
    f.restype = ctypes.c_int
    lib.b200ba_last_error.restype = ctypes.c_char_p
    return lib, f


def dense_f64(T, n_check, pivot_min=0.0, invert=False, n_test0=0):
    """ba_dense_potrf (+ ba_dense_potri) in place on the device matrix T -> (rc, bad_row, bad_pivot)."""
    lib, f = _hook()
    row, piv = ctypes.c_int(-1), ctypes.c_double(0.0)
    rc = f(T.data_ptr(), T.shape[0], n_test0, n_check, pivot_min, int(invert), ctypes.byref(row), ctypes.byref(piv))
    assert rc in (0, 1), (rc, lib.b200ba_last_error().decode())
    return rc, row.value, piv.value


# The kernels' layout is column-major: element (i, j) at [j * N + i], i.e. the row-major tensor holds M^T.
def to_device(M):
    return torch.from_numpy(np.ascontiguousarray(M.T)).cuda()


def from_device(T):
    return T.cpu().numpy().T


def _mm(a, b):
    """fp64 product on the GPU (cuBLAS): only the residuals, never the references, go through it."""
    return (torch.from_numpy(np.ascontiguousarray(a)).cuda() @ torch.from_numpy(np.ascontiguousarray(b)).cuda()).cpu().numpy()


def _spd(n, kappa, rng):
    """Q diag(s) Q^T, s log-spaced from 1 down to 1 / kappa (||A||_2 = 1, ||A^-1||_2 = kappa)."""
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = (Q * np.logspace(0.0, -np.log10(kappa), n)) @ Q.T
    return (A + A.T) / 2


def _padded(A, N):
    """A in the top-left corner of the identity of order N, the strict upper triangle NaN with a payload."""
    M = np.eye(N)
    M[:A.shape[0], :A.shape[0]] = A
    M[np.triu_indices(N, 1)] = NAN_PAYLOAD.view(np.float64)
    return M


def _note(name, value):
    WORST[name] = max(WORST.get(name, 0.0), float(value))


SIZES = [(n, kappa) for n in (1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193) for kappa in (1.0, 1e4, 1e12)]
SIZES += [(1000, 1e6), (4097, 1e6)]


@pytest.mark.parametrize("n,kappa", SIZES, ids=lambda v: f"{v:g}")
def test_factor_and_inverse(n, kappa):
    A = _spd(n, kappa, np.random.default_rng(n))
    N = -(-n // 64) * 64
    M = _padded(A, N)
    up = np.triu_indices(N, 1)
    off_tile = up[0] // 64 != up[1] // 64
    L_ref = np.linalg.cholesky(A)
    X_ref = np.linalg.inv(A)
    for invert in (False, True):
        T = to_device(M)
        assert dense_f64(T, n, invert=invert) == (0, 0, 0.0)
        out = from_device(T)
        assert np.array_equal(out.view(np.int64)[up][off_tile], np.full(int(off_tile.sum()), NAN_PAYLOAD)), "upper triangle written"
        low = np.tril(out)
        assert np.isfinite(low).all(), "upper triangle read"
        assert np.array_equal(low[n:], np.eye(N)[n:]), "padding block"   # exactly: its factor and inverse are the identity
        X = low[:n, :n]
        bar = C_BAR * n * EPS * kappa
        if not invert:
            back = np.linalg.norm(A - _mm(X, X.T)) / np.linalg.norm(A)
            fwd = np.linalg.norm(X - L_ref) / np.linalg.norm(L_ref)
            _note("factor backward / (n eps)", back / (n * EPS))
            _note("factor forward / (n eps kappa)", fwd / (n * EPS * kappa))
            assert back <= C_BAR * n * EPS, (back, C_BAR * n * EPS)
            assert fwd <= bar, (fwd, bar)
        else:
            res = np.abs(_mm(A, X + np.tril(X, -1).T) - np.eye(n)).max()
            fwd = np.abs(X - np.tril(X_ref)).max() / np.abs(X_ref).max()
            _note("inverse residual / (n eps kappa)", res / (n * EPS * kappa))
            _note("inverse forward / (n eps kappa)", fwd / (n * EPS * kappa))
            assert res <= bar, (res, bar)
            assert fwd <= bar, (fwd, bar)


def test_envelope_32768():
    """n = 32,768 in one 8.6 GB matrix A = diag(d) + G G^T (G: n x 4 cosines, so any tile is regenerated from its
    indices and A x costs two thin products); 64 columns of X = A^-1, among them the first and last of the first and last
    tiles, against ||A X[:, c] - e_c||_max <= C n eps kappa, kappa bounded by (max d + ||G||_2^2) / min d."""
    n, dev = 32768, "cuda"
    idx = torch.arange(n, device=dev)
    i = idx.to(torch.float64)
    d = 1.0 + (idx % 7).to(torch.float64) / 7.0
    G = torch.stack([np.sqrt(2.0 * s / n) * torch.cos(w * i + p)
                     for s, w, p in ((8.0, 1e-3, 0.1), (4.0, 7.3e-3, 1.3), (2.0, 0.0517, 2.1), (1.0, 0.731, 0.4))], 1)
    kappa = (d.max() + torch.linalg.eigvalsh(G.T @ G).max()).item() / d.min().item()
    try:
        T = torch.empty((n, n), dtype=torch.float64, device=dev)
        for r0 in range(0, n, 2048):            # symmetric: row block r of T = rows of A
            T[r0:r0 + 2048] = G[r0:r0 + 2048] @ G.T
        T.diagonal().add_(d)
        assert dense_f64(T, n, invert=True) == (0, 0, 0.0)
        rng = np.random.default_rng(32768)
        cols = np.unique(np.concatenate([[0, 63, 64, n - 65, n - 64, n - 1], rng.choice(n, 58, replace=False)]))
        c = torch.from_numpy(cols).to(dev)
        Xc = torch.where(idx[:, None] < c[None, :], T[:, c], T[c, :].T)   # lower triangle: X(i, c) at [c * n + i], i >= c
        del T
        torch.cuda.empty_cache()
        R = d[:, None] * Xc + G @ (G.T @ Xc)
        R[c, torch.arange(len(cols), device=dev)] -= 1.0
        res = R.abs().max().item()
    finally:
        T = None
        torch.cuda.empty_cache()
    _note("inverse residual / (n eps kappa)", res / (n * EPS * kappa))
    assert res <= C_BAR * n * EPS * kappa, (res, kappa)


def _ldl(n, D, rng):
    """A = L0 diag(D) L0^T, L0 unit lower with entries of at most 0.5 / sqrt(n) below the diagonal; a non-finite D[r]
    spreads only into A[r:, r:] (the pivots before r stay exact)."""
    L0 = np.eye(n) + np.tril(rng.uniform(-0.5, 0.5, (n, n)), -1) / np.sqrt(n)
    good = np.where(np.isfinite(D), D, 0.0)
    A = (L0 * good) @ L0.T
    for r in np.nonzero(~np.isfinite(D))[0]:
        A[r:, r:] += D[r] * np.outer(L0[r:, r], L0[r:, r])
    return A


N_PIV, NCHK_PIV = 256, 200


def _pivot_case(bad, n_check=NCHK_PIV, n_test0=0, invert=False, seed=0):
    D = np.ones(N_PIV)
    for r, v in bad.items():
        D[r] = v
    A = _ldl(N_PIV, D, np.random.default_rng(seed))
    T = to_device(A)
    return dense_f64(T, n_check, pivot_min=1e-6, invert=invert, n_test0=n_test0), A, T


@pytest.mark.parametrize("row", [0, 63, 64, 130, NCHK_PIV - 1])
@pytest.mark.parametrize("pivot", [1e-7, -1.0, np.nan])
def test_pivot_flag_row(row, pivot):
    (rc, bad_row, bad_pivot), _, _ = _pivot_case({row: pivot})
    assert rc == 1 and bad_row == row
    if np.isnan(pivot):
        assert np.isnan(bad_pivot)
    else:
        assert bad_pivot == pytest.approx(pivot, rel=1e-6)


def test_pivot_flag_passes_and_orders():
    (rc, _, _), A, T = _pivot_case({130: 2e-6})
    assert rc == 0
    L = np.tril(from_device(T))
    assert np.linalg.norm(A - L @ L.T) / np.linalg.norm(A) <= C_BAR * N_PIV * EPS
    assert _pivot_case({64: 1e-7, 130: -1.0})[0][:2] == (1, 64)         # the first failing row is reported
    assert _pivot_case({130: -1.0, 199: 1e-7})[0][:2] == (1, 130)


@pytest.mark.parametrize("pivot", [1e-7, -1.0])
def test_pivot_flag_past_n_check(pivot):
    assert _pivot_case({NCHK_PIV: pivot})[0][0] == 0
    assert _pivot_case({N_PIV - 1: pivot})[0][0] == 0
    assert _pivot_case({130: pivot}, n_check=130)[0][0] == 0


def test_pivot_flag_before_n_test0():
    """Rows before n_test0 are eliminated, not rank-tested: a small positive pivot passes, a non-positive one fails."""
    assert _pivot_case({64: 1e-7}, n_test0=100)[0][0] == 0
    assert _pivot_case({99: 1e-7}, n_test0=100)[0][0] == 0
    assert _pivot_case({100: 1e-7}, n_test0=100)[0][:2] == (1, 100)
    (rc, row, piv), _, _ = _pivot_case({64: -1.0}, n_test0=100)
    assert (rc, row) == (1, 64) and piv == pytest.approx(-1.0, rel=1e-6)
    assert _pivot_case({64: 0.0}, n_test0=100)[0][:2] == (1, 64)


def test_failed_factorisation_skips_inverse_then_recovers():
    (rc0, _, _), _, T0 = _pivot_case({130: -1.0}, invert=False)
    (rc1, row, _), _, T1 = _pivot_case({130: -1.0}, invert=True)
    assert rc0 == rc1 == 1 and row == 130
    assert np.array_equal(T0.cpu().numpy().view(np.int64), T1.cpu().numpy().view(np.int64)), "inverse ran after a failed pivot"
    (rc, _, _), A, T = _pivot_case({}, invert=True, seed=1)
    assert rc == 0
    assert np.abs(np.tril(from_device(T)) - np.tril(np.linalg.inv(A))).max() <= C_BAR * N_PIV * EPS * np.linalg.cond(A)


def test_report_margins():
    print(f"worst error ratios (bar: {C_BAR}): {WORST}")
