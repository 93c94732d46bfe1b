// ba_dense_backsub.cu — DENSE_SCHUR and the back-substitution of the point steps.
// DENSE_SCHUR: the reduced camera matrix S = H_cc + D_c^2 - H_cp (H_pp + D_p^2)^-1 H_pc formed explicitly and factorised
// (ceres DENSE_SCHUR = SchurEliminator + dense Cholesky; COLMAP picks it for <= 50 images, bundle_adjustment_ceres.cc:
// 202-206).  Built from the same fp32-stored scaled Jacobians the implicit operator of the PCG path reads.
#include "ba_common.cuh"

template <int DC>
__device__ __forceinline__ void ba_slot_rows(const BaDev& D, long long s, float* J0, float* J1, int* idx) {
  const int4 pk = __ldg(D.s_pack + s);
  const unsigned pky = (unsigned)pk.y;
  const int po = pk.x;
  int co, nv;
  ba_unpack_cam(pky, DC > 11 ? D.wide : 0, co, nv);
#pragma unroll
  for (int c = 0; c < DC; ++c) { J0[c] = D.Jc[BA_JC(c, s)]; J1[c] = D.Jc[BA_JC(DC + c, s)]; }
#pragma unroll
  for (int c = 0; c < DC; ++c) idx[c] = (c < 6) ? (po >= 0 ? po + c : -1) : ((co >= 0 && c - 6 < nv) ? co + c - 6 : -1);
  if (pk.w < 0) {
#pragma unroll
    for (int c = 0; c < DC; ++c) idx[c] = -1;
  }
}
// S += J_c^T J_c, one thread per observation slot (pose block, intrinsics block and their coupling)
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_dense_gram_kernel(const BaDev D) {
  const long long s = (long long)blockIdx.x * BA_BLOCK + threadIdx.x;
  float J0[DC], J1[DC];
  int idx[DC];
  ba_slot_rows<DC>(D, s, J0, J1, idx);
#pragma unroll
  for (int r = 0; r < DC; ++r) {
    if (idx[r] < 0) continue;
#pragma unroll
    for (int c = 0; c < DC; ++c)
      if (idx[c] >= 0 && idx[r] >= idx[c])   // lower triangle only: element (i, j), i >= j, lives at Sd[j * nc + i]
        atomicAdd(&D.Sd[(long long)idx[c] * D.nc + idx[r]], (double)J0[r] * (double)J0[c] + (double)J1[r] * (double)J1[c]);
  }
}
// S -= sum over the pairs (i, j) of a track of W_i^T Hinv W_j with W_o = J_p(o)^T J_c(o); one warp per variable point
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_dense_schur_kernel(const BaDev D) {
  const int k = blockIdx.x * (BA_BLOCK / 32) + (threadIdx.x >> 5);
  if (k >= D.nvpt) return;
  const int lane = threadIdx.x & 31;
  const int s0 = D.vpt_s0[k], L = D.vpt_s1[k] - s0;
  const double* I = D.Hpp_inv + 6 * (long long)k;
  const double Hi[9] = {I[0], I[1], I[2], I[1], I[3], I[4], I[2], I[4], I[5]};
  for (long long t = lane; t < (long long)L * L; t += 32) {
    const int i = (int)(t / L), j = (int)(t - (long long)i * L);
    float A0[DC], A1[DC], B0[DC], B1[DC];
    int ia[DC], ib[DC];
    ba_slot_rows<DC>(D, s0 + i, A0, A1, ia);
    ba_slot_rows<DC>(D, s0 + j, B0, B1, ib);
    double pa[6], pb[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) { pa[c] = D.Jp[BA_JP(c, s0 + i)]; pb[c] = D.Jp[BA_JP(c, s0 + j)]; }
    // G = Hinv W_j (3 x DC)
    double G[3][DC];
#pragma unroll
    for (int c = 0; c < DC; ++c) {
      const double w0 = pb[0] * B0[c] + pb[3] * B1[c], w1 = pb[1] * B0[c] + pb[4] * B1[c], w2 = pb[2] * B0[c] + pb[5] * B1[c];
      G[0][c] = Hi[0] * w0 + Hi[1] * w1 + Hi[2] * w2;
      G[1][c] = Hi[3] * w0 + Hi[4] * w1 + Hi[5] * w2;
      G[2][c] = Hi[6] * w0 + Hi[7] * w1 + Hi[8] * w2;
    }
#pragma unroll
    for (int r = 0; r < DC; ++r) {
      if (ia[r] < 0) continue;
      const double v0 = pa[0] * A0[r] + pa[3] * A1[r], v1 = pa[1] * A0[r] + pa[4] * A1[r], v2 = pa[2] * A0[r] + pa[5] * A1[r];
#pragma unroll
      for (int c = 0; c < DC; ++c)
        if (ib[c] >= 0 && ia[r] >= ib[c]) atomicAdd(&D.Sd[(long long)ib[c] * D.nc + ia[r]], -(v0 * G[0][c] + v1 * G[1][c] + v2 * G[2][c]));
    }
  }
}
// S += D_c^2 on the diagonal, Cholesky S = L L^T in place (lower triangle, left-looking, one CTA), then L L^T x = rhs.
// The matrix is symmetric, so "row i" is read as column i: consecutive threads touch consecutive addresses.
#define BA_DENSE_T 1024
__global__ void __launch_bounds__(BA_DENSE_T) ba_dense_solve_kernel(const BaDev D) {
  __shared__ double s_d;
  __shared__ int s_bad;
  const int n = D.nc, tid = threadIdx.x;
  double* S = D.Sd;
  // element (i, j), i >= j, of the lower triangle lives at S[j * n + i]
  if (tid == 0) s_bad = 0;
  for (int i = tid; i < n; i += BA_DENSE_T) S[(long long)i * n + i] += D.Dc2[i];
  __syncthreads();
  for (int j = 0; j < n; ++j) {
    // column j: L(i, j) = (S(i, j) - sum_{k < j} L(i, k) L(j, k)) / L(j, j), i = j .. n - 1
    for (int i = j + tid; i < n; i += BA_DENSE_T) {
      double acc = S[(long long)j * n + i];
      for (int k = 0; k < j; ++k) acc -= S[(long long)k * n + i] * S[(long long)k * n + j];
      S[(long long)j * n + i] = acc;
    }
    __syncthreads();
    if (tid == 0) { const double d = S[(long long)j * n + j]; if (!(d > 0.0)) { s_bad = 1; s_d = 1.0; } else s_d = sqrt(d); }
    __syncthreads();
    const double inv = 1.0 / s_d;
    for (int i = j + tid; i < n; i += BA_DENSE_T) S[(long long)j * n + i] = (i == j) ? s_d : S[(long long)j * n + i] * inv;
    __syncthreads();
  }
  if (s_bad) { if (tid == 0) D.ctl->fail = 1; return; }
  // forward: L y = b (column-oriented), then backward: L^T x = y
  double* x = D.x;
  for (int i = tid; i < n; i += BA_DENSE_T) x[i] = D.rhs[i];
  __syncthreads();
  for (int j = 0; j < n; ++j) {
    if (tid == 0) x[j] = x[j] / S[(long long)j * n + j];
    __syncthreads();
    const double xj = x[j];
    for (int i = j + 1 + tid; i < n; i += BA_DENSE_T) x[i] -= S[(long long)j * n + i] * xj;
    __syncthreads();
  }
  for (int j = n - 1; j >= 0; --j) {
    // x_j = (y_j - sum_{i > j} L(i, j) x_i) / L(j, j): a dot product over column j
    double acc = 0.0;
    for (int i = j + 1 + tid; i < n; i += BA_DENSE_T) acc += S[(long long)j * n + i] * x[i];
    __shared__ double red[33];
    const double tot = ba_cta_allsum(acc, red);
    if (tid == 0) x[j] = (x[j] - tot) / S[(long long)j * n + j];
    __syncthreads();
  }
}

// d_p = Hinv (-g_p - H_pc d_c); also the model cost change -(Jd)^T (r + Jd/2), one thread per slot block-wise
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_backsub_model_kernel(const BaDev D, int blk0) {
  __shared__ double sy[2][BA_BLOCK];
  __shared__ double sw[3][BA_BLOCK];
  __shared__ double sm[8];
  const int blk = blockIdx.x + blk0;
  if (blk >= D.nblocks_giant0 && blk < D.nblocks_giant1) return;
  const long long s = (long long)blk * BA_BLOCK + threadIdx.x;
  const int pi = D.s_pose[s];
  double y0 = 0.0, y1 = 0.0;
  if (pi >= 0) {
    const int ci = D.s_cam[s];
    const int po = D.pose_off[pi], co = D.cam_off[ci], nv = D.cam_width[ci];
    if (po >= 0) for (int c = 0; c < 6; ++c) { const double v = D.x[po + c]; y0 += D.Jc[BA_JC(c, s)] * v; y1 += D.Jc[BA_JC((DC + c), s)] * v; }
    if (co >= 0) for (int c = 0; c < nv; ++c) { const double v = D.x[co + c]; y0 += D.Jc[BA_JC((6 + c), s)] * v; y1 += D.Jc[BA_JC((DC + 6 + c), s)] * v; }
  }
  if (blk < D.nblocks_var) {
    sy[0][threadIdx.x] = y0; sy[1][threadIdx.x] = y1;
    __syncthreads();
    if (threadIdx.x < D.blk_npt[blk]) {
      const int k = D.blk_pt0[blk] + threadIdx.x;
      double t0 = -D.gp[3 * (long long)k], t1 = -D.gp[3 * (long long)k + 1], t2 = -D.gp[3 * (long long)k + 2];
      for (int t = D.vpt_s0[k]; t < D.vpt_s1[k]; ++t) {
        const int l = t - blk * BA_BLOCK;
        const double a0 = sy[0][l], a1 = sy[1][l];
        t0 -= D.Jp[BA_JP(0, t)] * a0 + D.Jp[BA_JP(3, t)] * a1;
        t1 -= D.Jp[BA_JP(1, t)] * a0 + D.Jp[BA_JP(4, t)] * a1;
        t2 -= D.Jp[BA_JP(2, t)] * a0 + D.Jp[BA_JP(5, t)] * a1;
      }
      const double* I = D.Hpp_inv + 6 * (long long)k;
      const double d0 = I[0] * t0 + I[1] * t1 + I[2] * t2, d1 = I[1] * t0 + I[3] * t1 + I[4] * t2, d2 = I[2] * t0 + I[4] * t1 + I[5] * t2;
      D.dp[3 * (long long)k] = d0; D.dp[3 * (long long)k + 1] = d1; D.dp[3 * (long long)k + 2] = d2;
      sw[0][threadIdx.x] = d0; sw[1][threadIdx.x] = d1; sw[2][threadIdx.x] = d2;
    }
    __syncthreads();
    const int lp = (pi >= 0) ? D.s_lpt[s] : -1;
    if (lp >= 0) {
      const int lt = lp - D.blk_pt0[blk];
      const double w0 = sw[0][lt], w1 = sw[1][lt], w2 = sw[2][lt];
      y0 += D.Jp[BA_JP(0, s)] * w0 + D.Jp[BA_JP(1, s)] * w1 + D.Jp[BA_JP(2, s)] * w2;
      y1 += D.Jp[BA_JP(3, s)] * w0 + D.Jp[BA_JP(4, s)] * w1 + D.Jp[BA_JP(5, s)] * w2;
    }
  }
  double m = 0.0;
  if (pi >= 0) m = -(y0 * (D.r[s] + 0.5 * y0) + y1 * (D.r[D.nslots + s] + 0.5 * y1));
  const double t = ba_block_sum(m, sm);
  if (threadIdx.x == 0) atomicAdd(&D.ctl->model, t);
}

// Warp-packed blocks (tracks of <= 32 observations): the same step with the per-track sums as segmented shuffle
// reductions (cf. ba_spmv_slot) — no shared-memory exchange, no per-track serial loop.
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_backsub_warp_kernel(const BaDev D) {
  __shared__ double sm[8];
  const long long s = (long long)blockIdx.x * BA_BLOCK + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const int4 pk = __ldg(D.s_pack + s);
  const unsigned pky = (unsigned)pk.y;
  const int po = pk.x;
  int co, nv;
  ba_unpack_cam(pky, DC > 11 ? D.wide : 0, co, nv);
  const int lp = pk.z;
  const long long cp = pk.w;
  float J0[DC], J1[DC], jp[6];
#pragma unroll
  for (int c = 0; c < DC; ++c) { J0[c] = D.Jc[BA_JC(c, s)]; J1[c] = D.Jc[BA_JC(DC + c, s)]; }
#pragma unroll
  for (int c = 0; c < 6; ++c) jp[c] = D.Jp[BA_JP(c, s)];
  const double r0 = D.r[s], r1 = D.r[D.nslots + s];
  int head = lane, last = lane;
  double y0 = 0.0, y1 = 0.0;
  if (cp >= 0) {
    head = (int)((pky >> 22) & 31u); last = (int)((pky >> 27) & 31u);
    if (po >= 0) {
#pragma unroll
      for (int c = 0; c < 6; ++c) { const double v = D.x[po + c]; y0 += (double)J0[c] * v; y1 += (double)J1[c] * v; }
    }
    if (co >= 0) {
#pragma unroll
      for (int c = 0; c < DC - 6; ++c) if (c < nv) { const double v = D.x[co + c]; y0 += (double)J0[6 + c] * v; y1 += (double)J1[6 + c] * v; }
    }
  }
  double z0 = (double)jp[0] * y0 + (double)jp[3] * y1, z1 = (double)jp[1] * y0 + (double)jp[4] * y1, z2 = (double)jp[2] * y0 + (double)jp[5] * y1;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const double t0 = ba_shfl_down_f64(z0, off), t1 = ba_shfl_down_f64(z1, off), t2 = ba_shfl_down_f64(z2, off);
    if (lane + off <= last) { z0 += t0; z1 += t1; z2 += t2; }
  }
  double d0 = 0.0, d1 = 0.0, d2 = 0.0;
  if (lane == head && lp >= 0 && cp >= 0) {
    const double t0 = -D.gp[3 * (long long)lp] - z0, t1 = -D.gp[3 * (long long)lp + 1] - z1, t2 = -D.gp[3 * (long long)lp + 2] - z2;
    const double* I = D.Hpp_inv + 6 * (long long)lp;
    d0 = I[0] * t0 + I[1] * t1 + I[2] * t2; d1 = I[1] * t0 + I[3] * t1 + I[4] * t2; d2 = I[2] * t0 + I[4] * t1 + I[5] * t2;
    D.dp[3 * (long long)lp] = d0; D.dp[3 * (long long)lp + 1] = d1; D.dp[3 * (long long)lp + 2] = d2;
  }
  d0 = ba_shfl_f64(d0, head); d1 = ba_shfl_f64(d1, head); d2 = ba_shfl_f64(d2, head);
  double m = 0.0;
  if (cp >= 0) {
    if (lp >= 0) {
      y0 += (double)jp[0] * d0 + (double)jp[1] * d1 + (double)jp[2] * d2;
      y1 += (double)jp[3] * d0 + (double)jp[4] * d1 + (double)jp[5] * d2;
    }
    m = -(y0 * (r0 + 0.5 * y0) + y1 * (r1 + 0.5 * y1));
  }
  const double t = ba_block_sum(m, sm);
  if (threadIdx.x == 0) atomicAdd(&D.ctl->model, t);
}

// dense path: the full J^T J (pose-sensor cross block included) into the lower triangle of S (element (i, j), i >= j, at
// Sd[j * nc + i])
__global__ void ba_prior_dense_kernel(const BaDev D, const BaPrior P) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= P.n) return;
  const int4 ix = P.idx[k];
  const double* J = P.J + 36 * (long long)k;
  for (int a = 0; a < 12; ++a) {
    const int ia = ba_prior_col(ix, a);
    if (ia < 0) continue;
    for (int b = 0; b < 12; ++b) {
      const int ib = ba_prior_col(ix, b);
      if (ib >= 0 && ia >= ib) atomicAdd(&D.Sd[(long long)ib * D.nc + ia], J[a] * J[b] + J[12 + a] * J[12 + b] + J[24 + a] * J[24 + b]);
    }
  }
}
template <int DC>
static void ba_launch_dense_dc(const BaDev& D, const BaPrior& P, cudaStream_t s) {
  cudaMemsetAsync(D.Sd, 0, sizeof(double) * (size_t)D.nc * D.nc, s);
  ba_dense_gram_kernel<DC><<<D.nblocks, BA_BLOCK, 0, s>>>(D);
  if (D.nvpt) ba_dense_schur_kernel<DC><<<(D.nvpt + BA_BLOCK / 32 - 1) / (BA_BLOCK / 32), BA_BLOCK, 0, s>>>(D);
  if (P.n) ba_prior_dense_kernel<<<(P.n + 255) / 256, 256, 0, s>>>(D, P);
  ba_dense_solve_kernel<<<1, BA_DENSE_T, 0, s>>>(D);
}
template <int DC>
static void ba_launch_backsub_dc(const BaDev& D, cudaStream_t s) {
  if (D.nblocks_warp) ba_backsub_warp_kernel<DC><<<D.nblocks_warp, BA_BLOCK, 0, s>>>(D);
  if (D.nblocks > D.nblocks_warp) ba_backsub_model_kernel<DC><<<D.nblocks - D.nblocks_warp, BA_BLOCK, 0, s>>>(D, D.nblocks_warp);
  if (D.nblocks_giant1 > D.nblocks_giant0) {
    cudaMemsetAsync(D.zg, 0, sizeof(double) * 3 * (size_t)D.nvpt, s);
    ba_giant_accumulate_kernel<1><<<D.nblocks_giant1 - D.nblocks_giant0, BA_BLOCK, 0, s>>>(D, D.x);
    ba_giant_finish_kernel<1><<<D.nblocks_giant1 - D.nblocks_giant0, BA_BLOCK, 0, s>>>(D, D.x);
  }
}
void ba_launch_dense(const BaDev& D, const BaPrior& P, cudaStream_t s) { BA_DISPATCH_DC(ba_launch_dense_dc, D, P, s); }
void ba_launch_backsub(const BaDev& D, cudaStream_t s) { BA_DISPATCH_DC(ba_launch_backsub_dc, D, s); }
