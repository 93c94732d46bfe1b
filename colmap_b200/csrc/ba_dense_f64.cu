// ba_dense_f64.cu — tiled fp64 Cholesky (POTRF) and SPD inverse (TRTRI + LAUUM) for sm_90a, see ba_dense_f64.h.
//
// Every off-diagonal tile operation is one 64 x 64 output tile per CTA, accumulated over a range of 64-wide K tiles by
// one shared routine (ba_tile_kernel): operands staged through shared memory in 16-column chunks, products on the fp64
// tensor cores (mma.sync.aligned.m16n8k4 .f64, DMMA), four warps of 32 x 32.  The six operations differ only in where
// the two operands come from and where the result goes (the MODE template argument).  The diagonal tiles are factorised
// and inverted by one CTA each in shared memory (ba_tile_potrf_kernel); the panel solve then multiplies by that inverse
// on the tensor cores, as does TRTRI.  The triangular solves with the factor (ba_dense_potrs) run one 64-wide tile per
// launch on those inverted diagonal tiles.
#include "ba_dense_f64.h"

#include <math.h>

#define T BA_TILE
#define KC 16          // K columns staged per chunk
#define TT 128         // threads of a tile CTA: 2 x 2 warps of 32 x 32

enum { TM_SYRK = 0,    // POTRF trailing update: A(i, j) -= L(i, k) L(j, k)^T, k < j <= i
       TM_TRSM = 1,    // POTRF panel: L(i, k) = A(i, k) inv(L(k, k))^T
       TM_TRMM = 2,    // TRTRI step j: P_i = sum_{k = j+1..i} X(i, k) L(k, j)   (X = L^-1 below and right of (j, j))
       TM_SCALE = 3,   // TRTRI step j: X(i, j) = -P_i inv(L(j, j)); one extra CTA stores inv(L(j, j)) as X(j, j)
       TM_LAUUM = 4,   // LAUUM step i: R(i, j) = sum_{k >= i} X(k, i)^T X(k, j), j < i
       TM_LAUUM_D = 5 };  // LAUUM step i, the diagonal tile (a separate launch: the others read X(i, i))

struct BaTileArgs {
  double* A;
  int N, nt, step;
  const double* dinv;
  double* panel;
  const BaDenseFlag* flag;
};

__device__ __forceinline__ void ba_dmma(double* c, double a0, double a1, double b0) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5}, {%6}, {%0, %1, %2, %3};\n"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a0), "d"(a1), "d"(b0));
}

// operand A (64 x KC chunk, element (r, kk) of K tile kt) and B (element (kk, c)); masks keep the triangular tiles triangular
template <int MODE>
__device__ __forceinline__ double ba_tile_a(const BaTileArgs& a, int ti, int kt, int r, int kk) {
  const long long N = a.N;
  if (MODE == TM_SYRK || MODE == TM_TRSM) return a.A[(long long)(kt * T + kk) * N + ti * T + r];
  if (MODE == TM_TRMM) return (kt == ti && kk > r) ? 0.0 : a.A[(long long)(kt * T + kk) * N + ti * T + r];
  if (MODE == TM_SCALE) return a.panel[(long long)kk * N + ti * T + r];
  return (kt == ti && kk < r) ? 0.0 : a.A[(long long)(ti * T + r) * N + kt * T + kk];   // X(kt, ti)^T
}
template <int MODE>
__device__ __forceinline__ double ba_tile_b(const BaTileArgs& a, int tj, int kt, int kk, int c) {
  const long long N = a.N;
  if (MODE == TM_SYRK) return a.A[(long long)(kt * T + kk) * N + tj * T + c];           // L(j, k)^T
  if (MODE == TM_TRSM) return a.dinv[(long long)kt * T * T + kk * T + c];               // inv(L(k, k))^T
  if (MODE == TM_TRMM) return a.A[(long long)(tj * T + c) * N + kt * T + kk];           // L(k, j)
  if (MODE == TM_SCALE) return a.dinv[(long long)tj * T * T + c * T + kk];              // inv(L(j, j))
  return (kt == tj && kk < c) ? 0.0 : a.A[(long long)(tj * T + c) * N + kt * T + kk];   // X(k, j)
}

template <int MODE>
__global__ void __launch_bounds__(TT) ba_tile_kernel(const BaTileArgs a) {
  if (a.flag->bad) return;
  const int s = a.step;
  int ti, tj, k0, k1;
  if (MODE == TM_SYRK) {       // lower-triangular tile list of the trailing matrix
    const int t = blockIdx.x;
    int ip = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
    while (ip * (ip + 1) / 2 > t) --ip;
    while ((ip + 1) * (ip + 2) / 2 <= t) ++ip;
    ti = s + 1 + ip; tj = s + 1 + (t - ip * (ip + 1) / 2); k0 = s; k1 = s + 1;
  } else if (MODE == TM_TRSM) {
    ti = s + 1 + blockIdx.x; tj = s; k0 = s; k1 = s + 1;
  } else if (MODE == TM_TRMM) {
    ti = s + 1 + blockIdx.x; tj = s; k0 = s + 1; k1 = ti + 1;
  } else if (MODE == TM_SCALE) {
    ti = s + 1 + blockIdx.x; tj = s; k0 = 0; k1 = 1;
    if (ti == a.nt) {          // the extra CTA: X(j, j) = inv(L(j, j))
      for (int e = threadIdx.x; e < T * T; e += TT) {
        const int r = e % T, c = e / T;
        a.A[(long long)(s * T + c) * a.N + s * T + r] = a.dinv[(long long)s * T * T + c * T + r];
      }
      return;
    }
  } else if (MODE == TM_LAUUM) {
    ti = s; tj = blockIdx.x; k0 = s; k1 = a.nt;
  } else {
    ti = s; tj = s; k0 = s; k1 = a.nt;
  }
  __shared__ double As[T][KC + 1];
  __shared__ double Bs[KC][T + 1];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, g = lane >> 2, tg = lane & 3;
  const int wr = (w >> 1) * 32, wc = (w & 1) * 32;
  double acc[2][4][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[mi][ni][q] = 0.0;
  constexpr bool a_r_fast = MODE != TM_LAUUM && MODE != TM_LAUUM_D;   // which index is contiguous in memory
  constexpr bool b_c_fast = MODE == TM_SYRK || MODE == TM_TRSM;
  for (int kt = k0; kt < k1; ++kt) {
    for (int kc = 0; kc < T; kc += KC) {
#pragma unroll
      for (int q = 0; q < T * KC / TT; ++q) {
        const int e = tid + q * TT;
        const int r = a_r_fast ? (e % T) : (e / KC), kk = a_r_fast ? (e / T) : (e % KC);
        As[r][kk] = ba_tile_a<MODE>(a, ti, kt, r, kc + kk);
        const int c = b_c_fast ? (e % T) : (e / KC), kb = b_c_fast ? (e / T) : (e % KC);
        Bs[kb][c] = ba_tile_b<MODE>(a, tj, kt, kc + kb, c);
      }
      __syncthreads();
#pragma unroll
      for (int ks = 0; ks < KC; ks += 4) {
        double af[2][2], bf[4];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) { af[mi][0] = As[wr + mi * 16 + g][ks + tg]; af[mi][1] = As[wr + mi * 16 + g + 8][ks + tg]; }
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) bf[ni] = Bs[ks + tg][wc + ni * 8 + g];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
          for (int ni = 0; ni < 4; ++ni) ba_dmma(acc[mi][ni], af[mi][0], af[mi][1], bf[ni]);
      }
      __syncthreads();
    }
  }
  const long long N = a.N;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int r = wr + mi * 16 + g + (q >> 1) * 8, c = wc + ni * 8 + 2 * tg + (q & 1);
        const double v = acc[mi][ni][q];
        if (MODE == TM_TRMM) { a.panel[(long long)c * N + ti * T + r] = v; continue; }
        double* dst = a.A + (long long)(tj * T + c) * N + ti * T + r;
        if (MODE == TM_SYRK) *dst -= v;
        else if (MODE == TM_SCALE) *dst = -v;
        else *dst = v;
      }
}

// Diagonal tile k: unblocked Cholesky in shared memory with the pivot test, then the inverse of the factor (one column
// per thread, forward substitution) into dinv[k].  The factor goes back with a zero upper triangle.
#define PT 256
__global__ void __launch_bounds__(PT) ba_tile_potrf_kernel(double* A, int N, int k, int n_test0, int n_check, double pivot_min,
                                                           double* dinv, BaDenseFlag* flag) {
  if (flag->bad) return;
  __shared__ double s[T][T + 1];   // s[c][r]: column-major
  __shared__ int s_bad;
  const int tid = threadIdx.x;
  double* D = A + (long long)(k * T) * N + k * T;
  for (int e = tid; e < T * T; e += PT) { const int r = e % T, c = e / T; s[c][r] = r >= c ? D[(long long)c * N + r] : 0.0; }
  if (tid == 0) s_bad = 0;
  __syncthreads();
  for (int c = 0; c < T; ++c) {
    if (tid == 0) {
      const double d = s[c][c];
      const int row = k * T + c;
      if (row < n_check && !(d > (row < n_test0 ? 0.0 : pivot_min))) {
        s_bad = 1;
        flag->row = row; flag->pivot = d; __threadfence(); flag->bad = 1;
      } else {
        s[c][c] = sqrt(d);
      }
    }
    __syncthreads();
    if (s_bad) return;
    const double inv = 1.0 / s[c][c];
    for (int r = c + 1 + tid; r < T; r += PT) s[c][r] *= inv;
    __syncthreads();
    for (int e = tid; e < T * T; e += PT) {
      const int r = e % T, cc = e / T;
      if (cc > c && r >= cc) s[cc][r] -= s[c][r] * s[c][cc];
    }
    __syncthreads();
  }
  double* X = dinv + (long long)k * T * T;   // column-major inverse of the factor
  if (tid < T) {
    const int c = tid;
    for (int r = 0; r < c; ++r) X[c * T + r] = 0.0;
    X[c * T + c] = 1.0 / s[c][c];
    for (int r = c + 1; r < T; ++r) {
      double acc = 0.0;
      for (int m = c; m < r; ++m) acc += s[m][r] * X[c * T + m];
      X[c * T + r] = -acc / s[r][r];
    }
  }
  for (int e = tid; e < T * T; e += PT) { const int r = e % T, c = e / T; D[(long long)c * N + r] = r >= c ? s[c][r] : 0.0; }
}

cudaError_t ba_dense_potrf(double* A, int N, int n_test0, int n_check, double pivot_min, double* dinv, BaDenseFlag* flag,
                           cudaStream_t st) {
  const int nt = N / T;
  BaTileArgs a{A, N, nt, 0, dinv, nullptr, flag};
  for (int k = 0; k < nt; ++k) {
    ba_tile_potrf_kernel<<<1, PT, 0, st>>>(A, N, k, n_test0, n_check, pivot_min, dinv, flag);
    const int m = nt - 1 - k;
    if (!m) continue;
    a.step = k;
    ba_tile_kernel<TM_TRSM><<<m, TT, 0, st>>>(a);
    ba_tile_kernel<TM_SYRK><<<m * (m + 1) / 2, TT, 0, st>>>(a);
  }
  return cudaGetLastError();
}

cudaError_t ba_dense_potri(double* A, int N, const double* dinv, double* panel, const BaDenseFlag* flag, cudaStream_t st) {
  const int nt = N / T;
  BaTileArgs a{A, N, nt, 0, dinv, panel, flag};
  for (int j = nt - 1; j >= 0; --j) {   // TRTRI: block columns right to left, X(j+1.., j+1..) already inverted
    const int m = nt - 1 - j;
    a.step = j;
    if (m) ba_tile_kernel<TM_TRMM><<<m, TT, 0, st>>>(a);
    ba_tile_kernel<TM_SCALE><<<m + 1, TT, 0, st>>>(a);
  }
  for (int i = 0; i < nt; ++i) {        // LAUUM: block rows top to bottom, row i reads only rows >= i
    a.step = i;
    if (i) ba_tile_kernel<TM_LAUUM><<<i, TT, 0, st>>>(a);
    ba_tile_kernel<TM_LAUUM_D><<<1, TT, 0, st>>>(a);
  }
  return cudaGetLastError();
}

// L L^T X = B with L from ba_dense_potrf, one 64-wide tile per launch and every launch spread over the GPU; blockIdx.y
// is the right-hand side, and every right-hand side sees the same arithmetic in the same order.  Forward, tile k:
// y_k = Linv_kk b_k, then b_r -= L_rk y_k for every row below the tile (one thread per row, coalesced down the
// columns).  Backward, tile k (last first): x_k = Linv_kk^T u_k, then u_c -= L_kc^T x_k for every column left of the
// tile (one warp per column, the tile's 64 entries of a column are contiguous).  Every CTA recomputes the tile's
// 64-vector from the tile's inputs, which no launch writes, and CTA 0 stores it.
#define TB 256
__global__ void __launch_bounds__(TB) ba_trsv_fwd(const double* A, const double* dinv, int N, int k, double* B, double* Y,
                                                  const BaDenseFlag* flag) {
  if (flag->bad) return;
  __shared__ double t[T], yk[T];
  const int tid = threadIdx.x;
  double* b = B + (long long)blockIdx.y * N;
  double* y = Y + (long long)blockIdx.y * N;
  const double* X = dinv + (long long)k * T * T;
  if (tid < T) t[tid] = b[k * T + tid];
  __syncthreads();
  if (tid < T) { double s = 0; for (int c = 0; c <= tid; ++c) s += X[c * T + tid] * t[c]; yk[tid] = s; }
  __syncthreads();
  if (blockIdx.x == 0 && tid < T) y[k * T + tid] = yk[tid];
  const int r = (k + 1) * T + blockIdx.x * TB + tid;
  if (r >= N) return;
  const double* col = A + (long long)k * T * N + r;
  double s = 0;
  for (int c = 0; c < T; ++c) s += col[(long long)c * N] * yk[c];
  b[r] -= s;
}

__global__ void __launch_bounds__(TB) ba_trsv_bwd(const double* A, const double* dinv, int N, int k, double* U, double* B,
                                                  const BaDenseFlag* flag) {
  if (flag->bad) return;
  __shared__ double t[T], xk[T];
  const int tid = threadIdx.x;
  double* u = U + (long long)blockIdx.y * N;
  double* x = B + (long long)blockIdx.y * N;
  const double* X = dinv + (long long)k * T * T;
  if (tid < T) t[tid] = u[k * T + tid];
  __syncthreads();
  if (tid < T) { double s = 0; for (int r = tid; r < T; ++r) s += X[tid * T + r] * t[r]; xk[tid] = s; }
  __syncthreads();
  if (blockIdx.x == 0 && tid < T) x[k * T + tid] = xk[tid];
  const int warp = tid / 32, lane = tid % 32;
  const int c = blockIdx.x * (TB / 32) + warp;
  if (c >= k * T) return;
  const double* L = A + (long long)c * N + k * T;
  double s = L[lane] * xk[lane] + L[lane + 32] * xk[lane + 32];
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) u[c] -= s;
}

static inline unsigned ba_blocks(long long n, int t) { return (unsigned)(n > 0 ? (n + t - 1) / t : 1); }

cudaError_t ba_dense_potrs(const double* A, int N, const double* dinv, int nrhs, double* B, double* W, const BaDenseFlag* flag,
                           cudaStream_t st) {
  const int nt = N / T;
  for (int k = 0; k < nt; ++k)
    ba_trsv_fwd<<<dim3(ba_blocks(N - (long long)(k + 1) * T, TB), nrhs), TB, 0, st>>>(A, dinv, N, k, B, W, flag);
  for (int k = nt - 1; k >= 0; --k)
    ba_trsv_bwd<<<dim3(ba_blocks((long long)k * T, TB / 32), nrhs), TB, 0, st>>>(A, dinv, N, k, W, B, flag);
  return cudaGetLastError();
}
