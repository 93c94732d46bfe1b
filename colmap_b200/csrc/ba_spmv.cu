// ba_spmv.cu — the implicit Schur-complement product S p of the PCG: the slot pass and the camera-order pass.
#include "ba_common.cuh"

// Warp-packed variant of pass 1 (tracks of <= 32 observations, i.e. almost all of them): the track never crosses
// a warp, so the point-block elimination is a segmented shuffle reduction — no shared memory, no block barrier,
// every lane stays busy.  Same arithmetic as ba_schur_spmv_kernel below.
template <int DC>
__device__ __forceinline__ void ba_spmv_slot(const BaDev& D, const long long s, const int lane, const double* __restrict__ pvec) {
  const int4 pk = __ldg(D.s_pack + s);          // all per-slot indices in one coalesced 16-byte load
  const unsigned pky = (unsigned)pk.y;
  const int po = pk.x;
  int co, nv;
  ba_unpack_cam(pky, DC > 11 ? D.wide : 0, co, nv);
  const int lp = pk.z;
  const long long cp = pk.w;                     // -1 on padding slots
  int head = lane, last = lane;
  double y0 = 0.0, y1 = 0.0;
  // the Jacobian rows are fetched unconditionally (padding slots hold zeros) so that their loads are in flight
  // together with the index load instead of behind it
  float J0[DC], J1[DC], jp[6];
#pragma unroll
  for (int c = 0; c < DC; ++c) { J0[c] = D.Jc[BA_JC(c, s)]; J1[c] = D.Jc[BA_JC(DC + c, s)]; }
#pragma unroll
  for (int c = 0; c < 6; ++c) jp[c] = D.Jp[BA_JP(c, s)];
  if (cp >= 0) {
    head = (int)((pky >> 22) & 31u); last = (int)((pky >> 27) & 31u);
    if (po >= 0) {   // pose blocks are 6 doubles wide: the offset is 16-byte aligned -> three 128-bit loads
      const double2* v2 = reinterpret_cast<const double2*>(pvec + po);
      const double2 va = v2[0], vb = v2[1], vc = v2[2];
      const double v[6] = {va.x, va.y, vb.x, vb.y, vc.x, vc.y};
#pragma unroll
      for (int c = 0; c < 6; ++c) { y0 += (double)J0[c] * v[c]; y1 += (double)J1[c] * v[c]; }
    }
    if (co >= 0) {
#pragma unroll
      for (int c = 0; c < DC - 6; ++c) if (c < nv) { const double v = pvec[co + c]; y0 += (double)J0[6 + c] * v; y1 += (double)J1[6 + c] * v; }
    }
  }
  double z0 = (double)jp[0] * y0 + (double)jp[3] * y1, z1 = (double)jp[1] * y0 + (double)jp[4] * y1, z2 = (double)jp[2] * y0 + (double)jp[5] * y1;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const double t0 = ba_shfl_down_f64(z0, off), t1 = ba_shfl_down_f64(z1, off), t2 = ba_shfl_down_f64(z2, off);
    if (lane + off <= last) { z0 += t0; z1 += t1; z2 += t2; }
  }
  double w0 = 0.0, w1 = 0.0, w2 = 0.0;
  if (lane == head && lp >= 0) {
    const double2* I2 = reinterpret_cast<const double2*>(D.Hpp_inv + 6 * (long long)lp);   // 48-byte records: 16-byte aligned
    const double2 ia = I2[0], ib = I2[1], ic = I2[2];
    w0 = ia.x * z0 + ia.y * z1 + ib.x * z2;
    w1 = ia.y * z0 + ib.y * z1 + ic.x * z2;
    w2 = ib.x * z0 + ic.x * z1 + ic.y * z2;
  }
  w0 = ba_shfl_f64(w0, head); w1 = ba_shfl_f64(w1, head); w2 = ba_shfl_f64(w2, head);
  if (cp >= 0) {
    if (lp >= 0) {
      y0 -= (double)jp[0] * w0 + (double)jp[1] * w1 + (double)jp[2] * w2;
      y1 -= (double)jp[3] * w0 + (double)jp[4] * w1 + (double)jp[5] * w2;
    }
    D.u[cp] = make_float2((float)y0, (float)y1);   // one 8-byte scattered store per observation
  }
}

template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_schur_spmv_warp_kernel(const BaDev D, const double* __restrict__ pvec) {
  if (D.ctl->done) return;
  ba_spmv_slot<DC>(D, (long long)blockIdx.x * BA_BLOCK + threadIdx.x, threadIdx.x & 31, pvec);
}
// Persistent form with the camera-side vector staged in shared memory: the per-lane gathers p[pose], p[camera] (every
// lane of a warp looks at a different camera) cost one L1 wavefront per lane and instruction from global memory, a few
// bank-conflict cycles from shared memory.  Grid = SMs x resident CTAs, each CTA loads p once and walks the slot blocks.
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_schur_spmv_warp_smem_kernel(const BaDev D, const double* __restrict__ pvec) {
  extern __shared__ double2 ba_sp2[];
  double* sp = reinterpret_cast<double*>(ba_sp2);
  if (D.ctl->done) return;
  for (int i = threadIdx.x; i < D.nc; i += BA_BLOCK) sp[i] = pvec[i];
  __syncthreads();
  for (int blk = blockIdx.x; blk < D.nblocks_warp; blk += gridDim.x)
    ba_spmv_slot<DC>(D, (long long)blk * BA_BLOCK + threadIdx.x, threadIdx.x & 31, sp);
}

// THE ROOFLINE KERNEL, pass 1 of 2: u_o = J_c p - J_p (H_pp + D_p^2)^-1 sum_track J_p^T J_c p per observation.
// One thread per observation slot; a block holds whole tracks, so the point-block elimination
// (z_p = sum J_p^T y, w_p = Hinv z_p) is a shared-memory exchange.  u is written in camera-sorted order and
// reduced per camera-side block by ba_cam_stream_loop_kernel.
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_schur_spmv_kernel(const BaDev D, const double* __restrict__ pvec,
                                                                 double* __restrict__ qvec) {
  __shared__ double sy[2][BA_BLOCK];
  __shared__ double sw[3][BA_BLOCK];
  if (D.ctl->done) return;
  const int blk = blockIdx.x + D.nblocks_warp;   // blocks after the warp-packed region
  if (blk >= D.nblocks_giant0 && blk < D.nblocks_giant1) return;   // tracks longer than a block: generic path
  const long long s = (long long)blk * BA_BLOCK + threadIdx.x;
  const int pi = D.s_pose[s];
  int po = -1, co = -1, nv = 0;
  double J0[DC], J1[DC], y0 = 0.0, y1 = 0.0;
  if (pi >= 0) {
    const int ci = D.s_cam[s];
    po = D.pose_off[pi]; co = D.cam_off[ci]; nv = D.cam_width[ci];
#pragma unroll
    for (int c = 0; c < DC; ++c) { J0[c] = D.Jc[BA_JC(c, s)]; J1[c] = D.Jc[BA_JC((DC + c), s)]; }
    if (po >= 0) {
#pragma unroll
      for (int c = 0; c < 6; ++c) { const double v = pvec[po + c]; y0 += J0[c] * v; y1 += J1[c] * v; }
    }
    if (co >= 0) {
#pragma unroll
      for (int c = 0; c < DC - 6; ++c) if (c < nv) { const double v = pvec[co + c]; y0 += J0[6 + c] * v; y1 += J1[6 + c] * v; }
    }
  }
  const bool var_block = blk < D.nblocks_var;
  if (var_block) {
    sy[0][threadIdx.x] = y0; sy[1][threadIdx.x] = y1;
    __syncthreads();
    // one thread per track of this block
    if (threadIdx.x < D.blk_npt[blk]) {
      const int k = D.blk_pt0[blk] + threadIdx.x;
      const int s0 = D.vpt_s0[k], s1 = D.vpt_s1[k];
      double z0 = 0, z1 = 0, z2 = 0;
      for (int t = s0; t < s1; ++t) {
        const int l = t - blk * BA_BLOCK;
        const double a0 = sy[0][l], a1 = sy[1][l];
        z0 += D.Jp[BA_JP(0, t)] * a0 + D.Jp[BA_JP(3, t)] * a1;
        z1 += D.Jp[BA_JP(1, t)] * a0 + D.Jp[BA_JP(4, t)] * a1;
        z2 += D.Jp[BA_JP(2, t)] * a0 + D.Jp[BA_JP(5, t)] * a1;
      }
      const double* I = D.Hpp_inv + 6 * (long long)k;
      sw[0][threadIdx.x] = I[0] * z0 + I[1] * z1 + I[2] * z2;
      sw[1][threadIdx.x] = I[1] * z0 + I[3] * z1 + I[4] * z2;
      sw[2][threadIdx.x] = I[2] * z0 + I[4] * z1 + I[5] * z2;
    }
    __syncthreads();
    const int lp = (pi >= 0) ? D.s_lpt[s] : -1;
    if (lp >= 0) {
      const int lt = lp - D.blk_pt0[blk];
      const double w0 = sw[0][lt], w1 = sw[1][lt], w2 = sw[2][lt];
      y0 -= D.Jp[BA_JP(0, s)] * w0 + D.Jp[BA_JP(1, s)] * w1 + D.Jp[BA_JP(2, s)] * w2;
      y1 -= D.Jp[BA_JP(3, s)] * w0 + D.Jp[BA_JP(4, s)] * w1 + D.Jp[BA_JP(5, s)] * w2;
    }
  }
  if (pi >= 0) {
    const long long cp = D.s2c[s];
    D.u[cp] = make_float2((float)y0, (float)y1);   // one 8-byte scattered store per observation
  }
}

// Warp-reduces the per-lane sums of one (camera, pose) run and adds them to the run's pose / camera blocks of out.
template <int DC>
__device__ __forceinline__ void ba_cam_stream_flush(double* acc, int run, const BaDev& D, double* __restrict__ out, int lane) {
  if (run < 0) return;
  const int4 rd = D.runs[run];
  double mine = 0.0;
#pragma unroll
  for (int c = 0; c < DC; ++c) {
    double t = acc[c];
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == c) mine = t;
    acc[c] = 0.0;
  }
  if (lane < 6) { if (rd.x >= 0) atomicAdd(&out[rd.x + lane], mine); }
  else if (lane < 6 + rd.z) { if (rd.y >= 0) atomicAdd(&out[rd.y + lane - 6], mine); }
}
// Second SpMV pass (streaming): out[block] += sum over the block's observations of J_c^T u, observations in camera
// order.  A warp walks a contiguous range of 32-observation tiles (fully coalesced tile lines); the next tile's loads
// are issued before the current tile is accumulated (register double buffer).  The products are accumulated per lane
// while the tiles stay inside one (camera, pose) run — runs are thousands of observations long — and reduced with
// shuffles only when the run changes or the range ends: 6 + nv red.adds per run a warp touches.  No shared memory, no barrier.
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_cam_stream_loop_kernel(const BaDev D, double* __restrict__ out, int respect_done,
                                                                      int tiles_per_warp) {
  if (respect_done && D.ctl->done) return;
  const int lane = threadIdx.x & 31;
  const long long ntiles = (D.nobs_c + 31) >> 5;
  long long t = ((long long)blockIdx.x * (BA_BLOCK / 32) + (threadIdx.x >> 5)) * tiles_per_warp;
  const long long t1 = (t + tiles_per_warp < ntiles) ? t + tiles_per_warp : ntiles;
  if (t >= t1) return;
  int run_c;
  float j0c[DC], j1c[DC], u0c, u1c;
  {
    const long long k = t * 32 + lane;
    run_c = D.c_run[k];
#pragma unroll
    for (int c = 0; c < DC; ++c) { j0c[c] = D.JcC[BA_JC(c, k)]; j1c[c] = D.JcC[BA_JC(DC + c, k)]; }
    { const float2 uu = D.u[k]; u0c = uu.x; u1c = uu.y; }
  }
  double acc[DC];
#pragma unroll
  for (int c = 0; c < DC; ++c) acc[c] = 0.0;
  int cur = -1;
  for (; t < t1; ++t) {
    int run_n = -1;
    float j0n[DC], j1n[DC], u0n = 0.f, u1n = 0.f;
    if (t + 1 < t1) {
      const long long k = (t + 1) * 32 + lane;
      run_n = D.c_run[k];
#pragma unroll
      for (int c = 0; c < DC; ++c) { j0n[c] = D.JcC[BA_JC(c, k)]; j1n[c] = D.JcC[BA_JC(DC + c, k)]; }
      { const float2 uu = D.u[k]; u0n = uu.x; u1n = uu.y; }
    } else {
#pragma unroll
      for (int c = 0; c < DC; ++c) { j0n[c] = 0.f; j1n[c] = 0.f; }
    }
    const int r0 = __shfl_sync(0xffffffffu, run_c, 0);
    const bool uniform = __all_sync(0xffffffffu, run_c == r0);
    if (uniform) {
      if (r0 != cur) { ba_cam_stream_flush<DC>(acc, cur, D, out, lane); cur = r0; }
      if (r0 >= 0) {
#pragma unroll
        for (int c = 0; c < DC; ++c) acc[c] += (double)j0c[c] * (double)u0c + (double)j1c[c] * (double)u1c;
      }
    } else {  // the tile straddles a run boundary (or is the ragged tail): per-observation adds (rare)
      ba_cam_stream_flush<DC>(acc, cur, D, out, lane); cur = -1;
      if (run_c >= 0) {
        const int4 rd = D.runs[run_c];
#pragma unroll
        for (int c = 0; c < DC; ++c) {
          const double v = (double)j0c[c] * (double)u0c + (double)j1c[c] * (double)u1c;
          if (c < 6) { if (rd.x >= 0) atomicAdd(&out[rd.x + c], v); }
          else if (c < 6 + rd.z) { if (rd.y >= 0) atomicAdd(&out[rd.y + c - 6], v); }
        }
      }
    }
    run_c = run_n; u0c = u0n; u1c = u1n;
#pragma unroll
    for (int c = 0; c < DC; ++c) { j0c[c] = j0n[c]; j1c[c] = j1n[c]; }
  }
  ba_cam_stream_flush<DC>(acc, cur, D, out, lane);
}

template <int DC>
static void ba_launch_spmv_dc(const BaDev& D, const BaPath& P, cudaStream_t s) {
  if (D.nblocks_warp) {
    const size_t smem = sizeof(double) * (size_t)D.nc;
    if (P.spmv_smem) {
      const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(5, (size_t)(216 * 1024) / (smem + 1024)));
      const int grid = std::min(D.nblocks_warp, P.sms * per_sm);
      ba_schur_spmv_warp_smem_kernel<DC><<<grid, BA_BLOCK, smem, s>>>(D, D.p);
    } else {
      ba_schur_spmv_warp_kernel<DC><<<D.nblocks_warp, BA_BLOCK, 0, s>>>(D, D.p);
    }
  }
  if (D.nblocks > D.nblocks_warp) ba_schur_spmv_kernel<DC><<<D.nblocks - D.nblocks_warp, BA_BLOCK, 0, s>>>(D, D.p, D.q);
  if (D.nblocks_giant1 > D.nblocks_giant0) {
    cudaMemsetAsync(D.zg, 0, sizeof(double) * 3 * (size_t)D.nvpt, s);
    ba_giant_accumulate_kernel<0><<<D.nblocks_giant1 - D.nblocks_giant0, BA_BLOCK, 0, s>>>(D, D.p);
    ba_giant_finish_kernel<0><<<D.nblocks_giant1 - D.nblocks_giant0, BA_BLOCK, 0, s>>>(D, D.p);
  }
  if (D.nobs_c) {
    const long long ntiles = (D.nobs_c + 31) / 32;
    const long long warps = (long long)P.sms * 2 * (BA_BLOCK / 32) * 2;   // two waves of two resident CTAs per SM
    const int tpw = (int)std::max<long long>(4, (ntiles + warps - 1) / warps);
    const unsigned grid = (unsigned)((ntiles + (long long)tpw * (BA_BLOCK / 32) - 1) / ((long long)tpw * (BA_BLOCK / 32)));
    ba_cam_stream_loop_kernel<DC><<<grid, BA_BLOCK, 0, s>>>(D, D.q, 1, tpw);
  }
}
void ba_launch_spmv(const BaDev& D, const BaPath& P, cudaStream_t s) { BA_DISPATCH_DC(ba_launch_spmv_dc, D, P, s); }
template <int DC> static void ba_allow_spmv_smem_dc(const BaLayout&, cudaError_t* e) {
  *e = cudaFuncSetAttribute(ba_schur_spmv_warp_smem_kernel<DC>, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_SPMV_SMEM_MAX);
}
cudaError_t ba_allow_spmv_smem(const BaLayout& L) { cudaError_t e = cudaSuccess; BA_DISPATCH_DC(ba_allow_spmv_smem_dc, L, &e); return e; }
