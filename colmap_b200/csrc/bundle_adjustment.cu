// bundle_adjustment.cu — CUDA (sm_90a, H100) bundle-adjustment LM solver behind include/b200_bundle_adjustment.h.
//
// Reference behaviour: DefaultBundleAdjuster + ceres::Solve (src/colmap/estimators/bundle_adjustment_ceres.cc),
// residual/Jacobian arithmetic of cost_functions/reprojection_error.h, quaternion_utils.h, sensor/models_jacobian.h.
// Design (DESIGN.md §3): everything of an LM iteration runs on the GPU, fp64 arithmetic over fp32-stored Jacobians —
//   set-up         the host decides which observation sits in which slot (whole tracks per warp / block); the per-slot
//                  arrays, the (camera, pose) order (radix sort), runs and packed index words are built on the device;
//   linearize      residual + analytic Jacobians in the tangent space, evaluated once per storage order (slot order
//                  = track order, and (camera, pose) order), tiles of 32 observations x components;
//   build          H_pp (3x3 per point), g_p, g_c, diag(J'J), diagonal blocks of H_cc (chunk reductions in camera order);
//   damp           (H_pp + D_p^2)^-1, exact SCHUR_JACOBI blocks and the reduced right-hand side (camera order, no
//                  per-observation scratch);
//   PCG            implicit Schur complement product S p in two streaming passes ("SpMV", the roofline kernels) +
//                  one single-CTA launch for all vector work of an iteration; alpha/beta/termination live on the device;
//   backsub/update point step, model cost change, candidate evaluation, manifold retraction.
// The other units (ba_common.cuh lists them): linearisation, SpMV, dense solve and back-substitution, covariance,
// multi-GPU collectives, problem assembly.
#include <chrono>

#include "ba_common.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

// cost of the candidate parameters + per-residual cost change (accurate near convergence)
template <bool WIDE>
__global__ void __launch_bounds__(BA_BLOCK) ba_cost_kernel(const BaDev D, const double* __restrict__ poses,
                                                           const double* __restrict__ cams,
                                                           const double* __restrict__ pts, const double* __restrict__ sensors,
                                                           double* cost_out) {
  __shared__ double sm[8];
  const long long s = (long long)blockIdx.x * BA_BLOCK + threadIdx.x;
  double cost = 0.0, delta = 0.0;
  const int pi = D.s_pose[s];
  if (pi >= 0) {
    const int ci = D.s_cam[s], ti = D.s_pt[s];
    const int id = D.cam_model[ci];
    double pose[7], pt[3], res[2];
    for (int k = 0; k < 7; ++k) pose[k] = poses[7 * (long long)pi + k];
    for (int k = 0; k < 3; ++k) pt[k] = pts[3 * (long long)ti + k];
    const int P = ba_model_num_params(id);
    if (!WIDE) {   // (separate instantiations: the wide path's local arrays and calls would otherwise size the narrow one)
      double prm[5];
      for (int k = 0; k < P; ++k) prm[k] = cams[D.cam_poff[ci] + k];
      ba_reproj(id, pt, pose, prm, D.s_xy[s], D.s_xy[D.nslots + s], res, nullptr, nullptr, nullptr);
    } else {
      double prm[BA_MAXP], sens[7];
      for (int k = 0; k < P; ++k) prm[k] = cams[D.cam_poff[ci] + k];
      const int si = D.cam_sensor[ci];
      if (si >= 0) for (int k = 0; k < 7; ++k) sens[k] = sensors[7 * (long long)si + k];
      ba_residual_any(id, pt, pose, si >= 0 ? sens : nullptr, prm, D.s_xy[s], D.s_xy[D.nslots + s], res);
    }
    double rho[3];
    ba_loss(D.loss_type, D.loss_scale, res[0] * res[0] + res[1] * res[1], rho);
    cost = 0.5 * rho[0];
    delta = cost - D.cost_slot[s];
  }
  const double t = ba_block_sum(cost, sm);
  if (threadIdx.x == 0) atomicAdd(cost_out, t);
  const double t2 = ba_block_sum(delta, sm);
  if (threadIdx.x == 0) atomicAdd(&D.ctl->cost_delta, t2);
}

// squared column norms of the unscaled Jacobian (iteration 0) -> scale_c / scale_p hold the sums
__global__ void __launch_bounds__(BA_BLOCK) ba_colnorm_kernel(const BaDev D) {
  const long long s = (long long)blockIdx.x * BA_BLOCK + threadIdx.x;
  const int pi = D.s_pose[s];
  if (pi < 0) return;
  const int ci = D.s_cam[s], DC = D.DC;
  const int po = D.pose_off[pi], co = D.cam_off[ci], nv = D.cam_width[ci], lp = D.s_lpt[s];
  if (po >= 0) for (int c = 0; c < 6; ++c) { const double a = D.Jc[BA_JC(c, s)], b = D.Jc[BA_JC((DC + c), s)]; atomicAdd(&D.scale_c[po + c], a * a + b * b); }
  if (co >= 0) for (int c = 0; c < nv; ++c) { const double a = D.Jc[BA_JC((6 + c), s)], b = D.Jc[BA_JC((DC + 6 + c), s)]; atomicAdd(&D.scale_c[co + c], a * a + b * b); }
  if (lp >= 0) for (int c = 0; c < 3; ++c) { const double a = D.Jp[BA_JP(c, s)], b = D.Jp[BA_JP((3 + c), s)]; atomicAdd(&D.scale_p[3 * (long long)lp + c], a * a + b * b); }
}
__global__ void ba_make_scale_kernel(double* v, long long n, int enable) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) v[i] = enable ? 1.0 / (1.0 + sqrt(v[i])) : 1.0;
}
__global__ void ba_diag_from_blocks_kernel(const BaDev D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.nc) return;
  const int b = D.off2blk[i], n = D.blk_start[b + 1] - D.blk_start[b], l = i - D.blk_start[b];
  D.diag_c[i] = D.Hbb[D.blk_pack[b] + l * n + l];
}
// point-side: H_pp (sym 6), g_p, diag_p; one thread per variable point
__global__ void ba_build_pt_kernel(const BaDev D) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= D.nvpt) return;
  double H[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
  for (int s = D.vpt_s0[k]; s < D.vpt_s1[k]; ++s) {
    double a[3], b[3];
    for (int c = 0; c < 3; ++c) { a[c] = D.Jp[BA_JP(c, s)]; b[c] = D.Jp[BA_JP((3 + c), s)]; }
    const double r0 = D.r[s], r1 = D.r[D.nslots + s];
    H[0] += a[0] * a[0] + b[0] * b[0]; H[1] += a[0] * a[1] + b[0] * b[1]; H[2] += a[0] * a[2] + b[0] * b[2];
    H[3] += a[1] * a[1] + b[1] * b[1]; H[4] += a[1] * a[2] + b[1] * b[2]; H[5] += a[2] * a[2] + b[2] * b[2];
    for (int c = 0; c < 3; ++c) g[c] += a[c] * r0 + b[c] * r1;
  }
  for (int c = 0; c < 6; ++c) D.Hpp[6 * (long long)k + c] = H[c];
  for (int c = 0; c < 3; ++c) D.gp[3 * (long long)k + c] = g[c];
  D.diag_p[3 * (long long)k] = H[0]; D.diag_p[3 * (long long)k + 1] = H[3]; D.diag_p[3 * (long long)k + 2] = H[5];
}
// || x - Plus(x, -g) ||_inf with the unscaled gradient g = g_scaled / scale
__global__ void ba_gradmax_kernel(const BaDev D) {
  // The three kinds of blocks (poses, cameras, points) occupy thread ranges padded to whole warps: every warp runs ONE of
  // the branches.  (With the three branches inside one warp, ptxas 12.9 has shared uniform registers between the
  // divergent paths and the point lanes compute their address from a clobbered value: illegal address, seen on rigs.)
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long np32 = ((long long)D.nposes + 31) & ~31LL, nc32 = ((long long)D.ncams + 31) & ~31LL;
  double m = 0.0;
  if (i < np32) {
    if (i < D.nposes) {
      const int off = D.pose_off[i];
      if (off >= 0) {
        double d[3], qn[4];
        for (int k = 0; k < 3; ++k) d[k] = -D.gc[off + k] / D.scale_c[off + k];
        ba_quat_plus(D.poses + 7 * i, d, qn);
        for (int k = 0; k < 4; ++k) m = fmax(m, fabs(qn[k] - D.poses[7 * i + k]));
        for (int k = 3; k < 6; ++k) m = fmax(m, fabs(D.gc[off + k] / D.scale_c[off + k]));
      }
    }
  } else if (i < np32 + nc32) {
    const int c = (int)(i - np32);
    const int off = c < D.ncams ? D.cam_off[c] : -1;
    if (off >= 0) {
      int k0 = 0;
      if (D.wide && D.cam_ns[c] == 6) {   // sensor_from_rig tangent: the quaternion part through Plus, like a pose
        double d[3], qn[4];
        const double* q = D.sensors + 7 * (long long)D.cam_sensor[c];
        for (int k = 0; k < 3; ++k) d[k] = -D.gc[off + k] / D.scale_c[off + k];
        ba_quat_plus(q, d, qn);
        for (int k = 0; k < 4; ++k) m = fmax(m, fabs(qn[k] - q[k]));
        k0 = 3;
      }
      for (int k = k0; k < D.cam_width[c]; ++k) m = fmax(m, fabs(D.gc[off + k] / D.scale_c[off + k]));
    }
  } else {
    const long long k = i - np32 - nc32;
    if (k < 3LL * D.nvpt) m = fabs(D.gp[k] / D.scale_p[k]);
  }
  __shared__ double s_m[32];
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {   // one atomic per CTA (tens of thousands of per-warp atomics on one address serialise)
    m = threadIdx.x < ((blockDim.x + 31) >> 5) ? s_m[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    // atomic max on non-negative doubles through their integer representation
    if (threadIdx.x == 0 && m > 0.0) atomicMax(reinterpret_cast<unsigned long long*>(&D.ctl->gmax), (unsigned long long)__double_as_longlong(m));
  }
}

// camera-side accumulations without per-observation atomics: one warp per chunk of a block's observations in
// camera order: g_c and the diagonal block of H_cc (both triangles), reduced with shuffles, one red.add per entry
#define BA_SC_BLOCK 128
__global__ void __launch_bounds__(BA_SC_BLOCK) ba_build_cam_sorted_kernel(const BaDev D) {
  const int chunk = blockIdx.x * (BA_SC_BLOCK / 32) + (threadIdx.x >> 5);
  if (chunk >= D.nchunks) return;
  const int lane = threadIdx.x & 31;
  const int4 ch = D.chunks[chunk];   // w = first column | width << 8 | first row inside the block << 16 | block width << 24
  const int comp0 = ch.w & 0xff, n = (ch.w >> 8) & 0xff, lr0 = (ch.w >> 16) & 0xff, bw = (ch.w >> 24) & 0xff;
  double g[6] = {0, 0, 0, 0, 0, 0}, H[21];
#pragma unroll
  for (int i = 0; i < 21; ++i) H[i] = 0.0;
  // register double buffer: the next step's loads are issued before this step's 27 accumulations
  float an[6], bn[6];
  double r0n = 0.0, r1n = 0.0;
  auto fetch = [&](int kk) {
    if (kk < ch.y) {
      r0n = D.rC[BA_U(0, kk)]; r1n = D.rC[BA_U(1, kk)];
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        an[c] = (c < n) ? D.JcC[BA_JC(comp0 + c, kk)] : 0.f;
        bn[c] = (c < n) ? D.JcC[BA_JC(D.DC + comp0 + c, kk)] : 0.f;
      }
    } else {
      r0n = 0.0; r1n = 0.0;
#pragma unroll
      for (int c = 0; c < 6; ++c) { an[c] = 0.f; bn[c] = 0.f; }
    }
  };
  int k = ch.x + lane;
  fetch(k);
  for (; k < ch.y; k += 32) {
    const double r0 = r0n, r1 = r1n;
    double a[6], b[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) { a[c] = (double)an[c]; b[c] = (double)bn[c]; }
    fetch(k + 32);
#pragma unroll
    for (int c = 0; c < 6; ++c) g[c] += a[c] * r0 + b[c] * r1;
    int idx = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
      for (int c = r; c < 6; ++c) H[idx++] += a[r] * a[c] + b[r] * b[c];
  }
  double* Hb = D.Hbb + D.blk_pack[D.off2blk[ch.z]];
#pragma unroll
  for (int c = 0; c < 6; ++c) {
    double t = g[c];
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0 && c < n) atomicAdd(&D.gc[ch.z + c], t);
  }
  int idx = 0;
#pragma unroll
  for (int r = 0; r < 6; ++r)
#pragma unroll
    for (int c = r; c < 6; ++c) {
      double t = H[idx++];
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if (lane == 0 && r < n && c < n) { atomicAdd(&Hb[(lr0 + r) * bw + lr0 + c], t); if (c != r) atomicAdd(&Hb[(lr0 + c) * bw + lr0 + r], t); }
    }
}

// Camera blocks wider than six columns (wide intrinsics, sensor + intrinsics): the diagonal 6-ranges go through the
// chunk kernels above / below, the pairs (A, B) of different 6-ranges through this one.  SCHUR = false: H_cc block
// += J_A^T J_B; SCHUR = true: SCHUR_JACOBI block -= V_A^T Hinv V_B with V = J_p^T J_c.  One warp per pair chunk.
template <bool SCHUR>
__global__ void __launch_bounds__(BA_SC_BLOCK) ba_cam_offdiag_kernel(const BaDev D) {
  const int chunk = blockIdx.x * (BA_SC_BLOCK / 32) + (threadIdx.x >> 5);
  if (chunk >= D.nchunks_off) return;
  const int lane = threadIdx.x & 31;
  const int4 ch = D.chunks_off[chunk];   // {first obs, end obs, block offset, compA | nA << 8 | compB << 16 | nB << 24}
  const int cA = ch.w & 0xff, nA = (ch.w >> 8) & 0xff, cB = (ch.w >> 16) & 0xff, nB = (ch.w >> 24) & 0xff;
  const int blk = D.off2blk[ch.z], bw = D.blk_start[blk + 1] - D.blk_start[blk];
  double G[36];
#pragma unroll
  for (int i = 0; i < 36; ++i) G[i] = 0.0;
  for (int k = ch.x + lane; k < ch.y; k += 32) {
    double a0[6], a1[6], b0[6], b1[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      a0[c] = (c < nA) ? (double)D.JcC[BA_JC(cA + c, k)] : 0.0; a1[c] = (c < nA) ? (double)D.JcC[BA_JC(D.DC + cA + c, k)] : 0.0;
      b0[c] = (c < nB) ? (double)D.JcC[BA_JC(cB + c, k)] : 0.0; b1[c] = (c < nB) ? (double)D.JcC[BA_JC(D.DC + cB + c, k)] : 0.0;
    }
    if (!SCHUR) {
#pragma unroll
      for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int c = 0; c < 6; ++c) G[6 * r + c] += a0[r] * b0[c] + a1[r] * b1[c];
    } else {
      const int lp = D.c_pack[k].y;
      if (lp < 0) continue;
      const double* I = D.Hpp_inv + 6 * (long long)lp;
      const double Hi[9] = {I[0], I[1], I[2], I[1], I[3], I[4], I[2], I[4], I[5]};
      double p0[3], p1[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) { p0[c] = D.JpC[BA_JP(c, k)]; p1[c] = D.JpC[BA_JP(3 + c, k)]; }
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        // row r of V_A^T Hinv (V_A(t, r) = p0[t] a0[r] + p1[t] a1[r])
        const double v0 = p0[0] * a0[r] + p1[0] * a1[r], v1 = p0[1] * a0[r] + p1[1] * a1[r], v2 = p0[2] * a0[r] + p1[2] * a1[r];
        const double g0 = v0 * Hi[0] + v1 * Hi[3] + v2 * Hi[6], g1 = v0 * Hi[1] + v1 * Hi[4] + v2 * Hi[7], g2 = v0 * Hi[2] + v1 * Hi[5] + v2 * Hi[8];
#pragma unroll
        for (int c = 0; c < 6; ++c) G[6 * r + c] += g0 * (p0[0] * b0[c] + p1[0] * b1[c]) + g1 * (p0[1] * b0[c] + p1[1] * b1[c]) + g2 * (p0[2] * b0[c] + p1[2] * b1[c]);
      }
    }
  }
  double* Mb = (SCHUR ? D.Mbb : D.Hbb) + D.blk_pack[blk];
  const int lrA = cA - 6, lrB = cB - 6;
#pragma unroll
  for (int r = 0; r < 6; ++r)
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      double t = G[6 * r + c];
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if (lane == 0 && r < nA && c < nB) {
        const double v = SCHUR ? -t : t;
        atomicAdd(&Mb[(lrA + r) * bw + lrB + c], v);
        atomicAdd(&Mb[(lrB + c) * bw + lrA + r], v);
      }
    }
}

// Point terms of the reduced system, one warp per chunk of a camera-side block's observations (camera order, so
// every operand streams): for each observation u = J_p Hinv g_p and V = J_p^T J_c,block; accumulated per chunk are
//   rhs(block)  += J_c,block^T u                       (reduced right-hand side  -g_c + H_cp Hinv g_p)
//   Mbb(block)  -= V^T Hinv V                          (point term of the block's SCHUR_JACOBI diagonal block)
// reduced with shuffles, one red.add per entry per chunk.  Nothing per observation is written.  When a track sees the
// same variable-intrinsics camera twice (shared cameras) the intrinsics blocks also need the cross terms between
// different observations of the point: those problems set D.intr_by_pt and the intrinsics blocks come from
// ba_schur_pt_kernel instead.  So do the pose blocks when a track sees a rig frame through two sensors (D.pose_by_pt).
__global__ void __launch_bounds__(BA_SC_BLOCK) ba_schur_cam_kernel(const BaDev D) {
  const int chunk = blockIdx.x * (BA_SC_BLOCK / 32) + (threadIdx.x >> 5);
  if (chunk >= D.nchunks) return;
  const int lane = threadIdx.x & 31;
  const int4 ch = D.chunks[chunk];
  const int comp0 = ch.w & 0xff, n = (ch.w >> 8) & 0xff, lr0 = (ch.w >> 16) & 0xff, bw = (ch.w >> 24) & 0xff;
  const bool want_T = (comp0 == 0) ? !D.pose_by_pt : !D.intr_by_pt;
  double g[6] = {0, 0, 0, 0, 0, 0}, T[21];
#pragma unroll
  for (int i = 0; i < 21; ++i) T[i] = 0.0;
  // Software pipeline: a warp walks its chunk 32 observations at a time and every step has a dependent gather
  // (observation -> point -> Hinv, g_p).  The point index is fetched two steps ahead, the point data and the Jacobian
  // rows one step ahead, so no step waits for a memory round trip.
  int k = ch.x + lane;
  int lp_n = (k < ch.y) ? D.c_pack[k].y : -1;                 // point of step 0
  int lp_nn = (k + 32 < ch.y) ? D.c_pack[k + 32].y : -1;      // point of step 1
  double Hn[6], gn[3];
  float an[3], bn[3], j0n[6], j1n[6];
  auto fetch = [&](int kk, int lp) {
    if (lp >= 0) {
      const double* I = D.Hpp_inv + 6 * (long long)lp;
#pragma unroll
      for (int c = 0; c < 6; ++c) Hn[c] = I[c];
#pragma unroll
      for (int c = 0; c < 3; ++c) gn[c] = D.gp[3 * (long long)lp + c];
#pragma unroll
      for (int c = 0; c < 3; ++c) { an[c] = D.JpC[BA_JP(c, kk)]; bn[c] = D.JpC[BA_JP(3 + c, kk)]; }
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        j0n[c] = (c < n) ? D.JcC[BA_JC(comp0 + c, kk)] : 0.f;
        j1n[c] = (c < n) ? D.JcC[BA_JC(D.DC + comp0 + c, kk)] : 0.f;
      }
    }
  };
  fetch(k, lp_n);
  for (; k < ch.y; k += 32) {
    const int lp = lp_n;
    double I[6], gq[3], a[3], b[3], j0[6], j1[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) { I[c] = Hn[c]; j0[c] = (double)j0n[c]; j1[c] = (double)j1n[c]; }
#pragma unroll
    for (int c = 0; c < 3; ++c) { gq[c] = gn[c]; a[c] = (double)an[c]; b[c] = (double)bn[c]; }
    // next steps' loads go out before this step's arithmetic
    lp_n = lp_nn;
    lp_nn = (k + 64 < ch.y) ? D.c_pack[k + 64].y : -1;
    fetch(k + 32, lp_n);
    if (lp < 0) continue;
    const double Hi[9] = {I[0], I[1], I[2], I[1], I[3], I[4], I[2], I[4], I[5]};
    const double w0 = Hi[0] * gq[0] + Hi[1] * gq[1] + Hi[2] * gq[2], w1 = Hi[3] * gq[0] + Hi[4] * gq[1] + Hi[5] * gq[2],
                 w2 = Hi[6] * gq[0] + Hi[7] * gq[1] + Hi[8] * gq[2];
    const double u0 = a[0] * w0 + a[1] * w1 + a[2] * w2;
    const double u1 = b[0] * w0 + b[1] * w1 + b[2] * w2;
#pragma unroll
    for (int c = 0; c < 6; ++c) g[c] += j0[c] * u0 + j1[c] * u1;
    if (want_T) {
      double V[18];
#pragma unroll
      for (int c = 0; c < 6; ++c)
#pragma unroll
        for (int t = 0; t < 3; ++t) V[t * 6 + c] = a[t] * j0[c] + b[t] * j1[c];
      int idx = 0;
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        // row r of V^T Hinv, then its products with the columns c >= r of V
        const double G0 = V[r] * Hi[0] + V[6 + r] * Hi[3] + V[12 + r] * Hi[6];
        const double G1 = V[r] * Hi[1] + V[6 + r] * Hi[4] + V[12 + r] * Hi[7];
        const double G2 = V[r] * Hi[2] + V[6 + r] * Hi[5] + V[12 + r] * Hi[8];
#pragma unroll
        for (int c = r; c < 6; ++c) T[idx++] += G0 * V[c] + G1 * V[6 + c] + G2 * V[12 + c];
      }
    }
  }
#pragma unroll
  for (int c = 0; c < 6; ++c) {
    double t = g[c];
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0 && c < n) atomicAdd(&D.rhs[ch.z + c], t);
  }
  if (want_T) {
    double* M = D.Mbb + D.blk_pack[D.off2blk[ch.z]];
    int idx = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
      for (int c = r; c < 6; ++c) {
        double t = T[idx++];
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == 0 && r < n && c < n) { atomicAdd(&M[(lr0 + r) * bw + lr0 + c], -t); if (c != r) atomicAdd(&M[(lr0 + c) * bw + lr0 + r], -t); }
      }
  }
}

// (H_pp + D_p^2)^-1 per point
__global__ void ba_damp_pt_kernel(const BaDev D, double inv_radius, double dmin, double dmax, int* fail) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= D.nvpt) return;
  double d[3];
  for (int c = 0; c < 3; ++c) { d[c] = fmin(fmax(D.diag_p[3 * (long long)k + c], dmin), dmax) * inv_radius; D.Dp2[3 * (long long)k + c] = d[c]; }
  const double* H = D.Hpp + 6 * (long long)k;
  const double a = H[0] + d[0], b = H[1], c = H[2], dd = H[3] + d[1], e = H[4], f = H[5] + d[2];
  const double c00 = dd * f - e * e, c01 = c * e - b * f, c02 = b * e - c * dd;
  const double det = a * c00 + b * c01 + c * c02;
  if (!(det > 0)) { atomicExch(fail, 1); return; }
  const double id = 1.0 / det;
  double* I = D.Hpp_inv + 6 * (long long)k;
  I[0] = c00 * id; I[1] = c01 * id; I[2] = c02 * id; I[3] = (a * f - c * c) * id; I[4] = (b * c - a * e) * id; I[5] = (a * dd - b * b) * id;
}
__global__ void ba_damp_cam_kernel(const BaDev D, double inv_radius, double dmin, double dmax) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.nc) return;
  const double d = fmin(fmax(D.diag_c[i], dmin), dmax) * inv_radius;
  D.Dc2[i] = d;
  D.rhs[i] = -D.gc[i];
  const int b = D.off2blk[i], n = D.blk_start[b + 1] - D.blk_start[b], l = i - D.blk_start[b];
  for (int c = 0; c < n; ++c) D.Mbb[D.blk_pack[b] + l * n + c] = D.Hbb[D.blk_pack[b] + l * n + c] + (c == l ? d : 0.0);
}
// per point: the point term of the INTRINSICS blocks of SCHUR_JACOBI, -= V^T Hinv V with V summed over every
// observation of the track made with the same camera (exact cross terms for shared intrinsics).  Only launched when
// some track sees a variable-intrinsics camera more than once (D.intr_by_pt); otherwise ba_schur_cam_kernel has them.
// When a track sees a frame through several rig sensors (D.pose_by_pt) the POSE blocks get the same treatment:
// ceres' block of that frame holds the cross terms between those observations.
__global__ void ba_schur_pt_kernel(const BaDev D) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= D.nvpt) return;
  const double* I = D.Hpp_inv + 6 * (long long)k;
  const double Hi[9] = {I[0], I[1], I[2], I[1], I[3], I[4], I[2], I[4], I[5]};
  const int s0 = D.vpt_s0[k], s1 = D.vpt_s1[k];
  if (D.pose_by_pt) for (int s = s0; s < s1; ++s) {
    const int pi = D.s_pose[s], po = D.pose_off[pi];
    if (po < 0) continue;
    bool first = true;
    for (int s2 = s0; s2 < s && first; ++s2) if (D.s_pose[s2] == pi) first = false;
    if (!first) continue;
    double V[18];
    for (int t = 0; t < 18; ++t) V[t] = 0.0;
    for (int s2 = s; s2 < s1; ++s2) {
      if (D.s_pose[s2] != pi) continue;
      double a2[3], b2[3];
      for (int c = 0; c < 3; ++c) { a2[c] = D.Jp[BA_JP(c, s2)]; b2[c] = D.Jp[BA_JP(3 + c, s2)]; }
      for (int c = 0; c < 6; ++c) {
        const double j0 = D.Jc[BA_JC(c, s2)], j1 = D.Jc[BA_JC(D.DC + c, s2)];
        for (int t = 0; t < 3; ++t) V[t * 6 + c] += a2[t] * j0 + b2[t] * j1;
      }
    }
    double* M = D.Mbb + D.blk_pack[D.off2blk[po]];
    for (int r = 0; r < 6; ++r) {
      const double t0 = V[r] * Hi[0] + V[6 + r] * Hi[3] + V[12 + r] * Hi[6];
      const double t1 = V[r] * Hi[1] + V[6 + r] * Hi[4] + V[12 + r] * Hi[7];
      const double t2 = V[r] * Hi[2] + V[6 + r] * Hi[5] + V[12 + r] * Hi[8];
      for (int c = 0; c < 6; ++c) atomicAdd(&M[r * 6 + c], -(t0 * V[c] + t1 * V[6 + c] + t2 * V[12 + c]));
    }
  }
  if (D.intr_by_pt) for (int s = s0; s < s1; ++s) {
    const int ci = D.s_cam[s];
    const int co = D.cam_off[ci], nv = D.cam_width[ci];
    if (co < 0) continue;
    bool first = true;
    for (int s2 = s0; s2 < s && first; ++s2) if (D.s_cam[s2] == ci) first = false;
    if (!first) continue;
    double V[3 * BA_MAXCB];
    for (int t = 0; t < 3 * nv; ++t) V[t] = 0.0;
    for (int s2 = s; s2 < s1; ++s2) {
      if (D.s_cam[s2] != ci) continue;
      double a2[3], b2[3];
      for (int c = 0; c < 3; ++c) { a2[c] = D.Jp[BA_JP(c, s2)]; b2[c] = D.Jp[BA_JP(3 + c, s2)]; }
      for (int c = 0; c < nv; ++c) {
        const double j0 = D.Jc[BA_JC(6 + c, s2)], j1 = D.Jc[BA_JC(D.DC + 6 + c, s2)];
        for (int t = 0; t < 3; ++t) V[t * nv + c] += a2[t] * j0 + b2[t] * j1;
      }
    }
    double* M = D.Mbb + D.blk_pack[D.off2blk[co]];
    for (int r = 0; r < nv; ++r) {
      const double t0 = V[r] * Hi[0] + V[nv + r] * Hi[3] + V[2 * nv + r] * Hi[6];
      const double t1 = V[r] * Hi[1] + V[nv + r] * Hi[4] + V[2 * nv + r] * Hi[7];
      const double t2 = V[r] * Hi[2] + V[nv + r] * Hi[5] + V[2 * nv + r] * Hi[8];
      for (int c = 0; c < nv; ++c) atomicAdd(&M[r * nv + c], -(t0 * V[c] + t1 * V[nv + c] + t2 * V[2 * nv + c]));
    }
  }
}
// invert the preconditioner blocks (Cholesky); one thread per block.  MAXN = 6: the narrow layout (pose blocks and <= 5
// intrinsics); MAXN = BA_MAXCB: wide camera blocks.  A camera block that holds a sensor_from_rig part AND an intrinsics
// part is two parameter blocks for ceres' SCHUR_JACOBI: blk_split keeps their diagonal sub-blocks and drops the cross terms.
// One thread per COLUMN of a diagonal block (nc threads, not nblk): the thread factorises the (sub-)block its column
// belongs to - a few dozen flops, done redundantly by the block's columns - and back-substitutes its own unit vector.
// Same operations in the same order as a block-serial inversion, a sixth of its latency.
template <int MAXN>
__global__ void ba_invert_blocks_kernel(const BaDev D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.nc) return;
  const int b = D.off2blk[i], r0 = D.blk_start[b], n = D.blk_start[b + 1] - r0, cc = i - r0;
  const double* M = D.Mbb + D.blk_pack[b];
  double* O = D.Minv + D.blk_pack[b];
  const int split = (MAXN > 6 && D.blk_split) ? D.blk_split[b] : 0;   // [pose | intrinsics] blocks are inverted separately
  const int s0 = (split && cc >= split) ? split : 0, s1 = split ? (cc >= split ? n : split) : n;
  const int m = s1 - s0, c = cc - s0;
  double L[MAXN * MAXN];
  bool ok = true;
  for (int j = 0; j < m && ok; ++j) {
    double d = M[(s0 + j) * n + s0 + j];
    for (int k = 0; k < j; ++k) d -= L[j * m + k] * L[j * m + k];
    if (!(d > 0)) { ok = false; break; }
    d = sqrt(d); L[j * m + j] = d;
    for (int r = j + 1; r < m; ++r) {
      double t = M[(s0 + r) * n + s0 + j];
      for (int k = 0; k < j; ++k) t -= L[r * m + k] * L[j * m + k];
      L[r * m + j] = t / d;
    }
  }
  double col[MAXN];
  for (int r = 0; r < m; ++r) col[r] = r == c ? 1.0 : 0.0;
  if (ok) {
    for (int r = 0; r < m; ++r) { double t = col[r]; for (int k = 0; k < r; ++k) t -= L[r * m + k] * col[k]; col[r] = t / L[r * m + r]; }
    for (int r = m - 1; r >= 0; --r) { double t = col[r]; for (int k = r + 1; k < m; ++k) t -= L[k * m + r] * col[k]; col[r] = t / L[r * m + r]; }
  }
  for (int r = 0; r < n; ++r) O[r * n + cc] = (r >= s0 && r < s1) ? col[r - s0] : 0.0;
}

// ------------------------------------------------------------------------------------------------
// PCG on the reduced camera system; all scalars live in D.ctl, kernels are no-ops once ctl->done is set.
// ------------------------------------------------------------------------------------------------
// z_i = (M^-1)_i . r over the block of row i (ri = D.row_info[i], rblock = r + ri.x).  The row of M^-1 is fetched with
// one batch of predicated loads instead of a dependent load per column; the columns past 11 of a wide block follow.
__device__ __forceinline__ double ba_precond_row(int4 ri, const double* __restrict__ Minv, const double* rblock) {
  const double* __restrict__ M = Minv + ri.y;
  double m[11];
#pragma unroll
  for (int k = 0; k < 11; ++k) m[k] = k < ri.z ? M[k] : 0.0;
  double t = 0;
#pragma unroll
  for (int k = 0; k < 11; ++k) if (k < ri.z) t += m[k] * rblock[k];
  for (int k = 11; k < ri.z; ++k) t += M[k] * rblock[k];
  return t;
}
// The end of a PCG iteration, after `it` completed ones: scalar bookkeeping and termination, in one thread.  Returns
// done.  Inexact mode: ceres ConjugateGradientsSolver's Q-tolerance, zeta = it (Q1 - Q0) / Q1 below eta.  Exact mode
// (DENSE_/SPARSE_SCHUR requested): relative residual |r| <= r_tolerance |b|.
__device__ __forceinline__ int ba_pcg_end_iteration(BaCtl* c, int it, double rho, double Q0, double Q1, double rnorm2,
                                                    double norm_b, double q_tolerance, double r_tolerance, int max_iters) {
  it += 1;
  const bool converged = r_tolerance > 0.0 ? rnorm2 <= r_tolerance * r_tolerance * norm_b : it * (Q1 - Q0) / Q1 < q_tolerance;
  const int done = converged || it >= max_iters;
  c->it = it; c->iters_total += 1;
  c->Q0 = Q1; c->Q1 = 0.0; c->rnorm2 = 0.0;
  c->last_rho = rho; c->rho = 0.0; c->pq = 0.0;
  c->done = done;
  return done;
}

__global__ void ba_pcg_init_kernel(const BaDev D) {  // x = 0, r = b, norm_b
  __shared__ double sm[8];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0;
  if (i < D.nc) { D.x[i] = 0.0; D.rr[i] = D.rhs[i]; v = D.rhs[i] * D.rhs[i]; }
  const double t = ba_block_sum(v, sm);
  if (threadIdx.x == 0) atomicAdd(&D.ctl->norm_b, t);
}
// z = M^-1 r ; rho = r.z
__global__ void ba_pcg_precond_kernel(const BaDev D) {
  __shared__ double sm[8];
  if (D.ctl->done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0;
  if (i < D.nc) {
    const int4 ri = D.row_info[i];
    const double t = ba_precond_row(ri, D.Minv, D.rr + ri.x);
    D.z[i] = t;
    v = t * D.rr[i];
  }
  const double t = ba_block_sum(v, sm);
  if (threadIdx.x == 0) atomicAdd(&D.ctl->rho, t);
}
// p = z + beta p ; q = D_c^2 p (the SpMV adds the rest)
__global__ void ba_pcg_direction_kernel(const BaDev D) {
  if (D.ctl->done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.nc) return;
  // first iteration: p = z (never reads the uninitialised / recycled p buffer)
  const double p = (D.ctl->it == 0) ? D.z[i] : D.z[i] + (D.ctl->rho / D.ctl->last_rho) * D.p[i];
  D.p[i] = p;
  D.q[i] = D.Dc2[i] * p;
}

// ---- PCG vector work between two SpMVs in one single-CTA kernel (camera-side dimension is small: a few thousand) ----
#define BA_PCG_T 1024
#define BA_PCG_FUSED_MAX 65536   // tests/test_ba_paths_gpu.py mirrors this threshold
// Two sums in one pass through the barriers, for a CTA of BA_PCG_T threads (32 warps); the totals are valid in thread 0.
__device__ __forceinline__ void ba_cta_sum2(double& a, double& w, double (*sm2)[33]) {
  for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); w += __shfl_xor_sync(0xffffffffu, w, o); }
  const int wid = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { sm2[0][wid] = a; sm2[1][wid] = w; }
  __syncthreads();
  if (threadIdx.x < 32) {
    a = sm2[0][threadIdx.x]; w = sm2[1][threadIdx.x];
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); w += __shfl_xor_sync(0xffffffffu, w, o); }
  }
}
// One launch between two SpMVs: the tail of PCG iteration i (pq = p.q ; x += alpha p ; r -= alpha q ; Q1 = -x.(b + r) ;
// |r|^2 ; termination, see ba_pcg_end_iteration) followed by the head of iteration i + 1 (z = M^-1 r ; rho = r.z ;
// p = z + beta p ; q = D_c^2 p — the SpMV adds the rest).  do_post = 0 for the very first call of a solve.
__global__ void __launch_bounds__(BA_PCG_T) ba_pcg_mid_kernel(const BaDev D, double q_tolerance, double r_tolerance,
                                                              int max_iters, int zero_q, int do_post, int r_in_smem) {
  extern __shared__ double s_r[];   // [nc] when r_in_smem
  __shared__ double sm[33];
  __shared__ double sm2[2][33];
  __shared__ int s_done;
  BaCtl* c = D.ctl;
  if (c->done) return;
  // independent restrict views: the vectors never alias, which lets the loads of all elements go out together
  double* __restrict__ X = D.x; double* __restrict__ R = D.rr; double* __restrict__ P = D.p; double* __restrict__ Q = D.q;
  double* __restrict__ Z = D.z;
  const double* __restrict__ RHS = D.rhs; const double* __restrict__ DC2 = D.Dc2; const double* __restrict__ MI = D.Minv;
  const int nc = D.nc;
  int it = c->it;
  double last_rho = c->last_rho;
  const double rho_in = c->rho, norm_b = c->norm_b, Q0 = c->Q0;
  if (do_post) {
    double v = 0.0;
    for (int i = threadIdx.x; i < nc; i += BA_PCG_T) v += P[i] * Q[i];
    const double pq = ba_cta_allsum(v, sm);
    if (!(pq > 0.0)) { if (threadIdx.x == 0) c->done = 1; return; }
    const double alpha = rho_in / pq;
    double a = 0.0, w = 0.0;
    for (int i = threadIdx.x; i < nc; i += BA_PCG_T) {
      const double x = X[i] + alpha * P[i];
      const double r = R[i] - alpha * Q[i];
      X[i] = x; R[i] = r;
      if (r_in_smem) s_r[i] = r;
      a += -x * (RHS[i] + r);
      w += r * r;
    }
    ba_cta_sum2(a, w, sm2);
    if (threadIdx.x == 0) s_done = ba_pcg_end_iteration(c, it, rho_in, Q0, a, w, norm_b, q_tolerance, r_tolerance, max_iters);
    __syncthreads();   // also orders the R stores above before the preconditioner reads below
    if (s_done) return;
    it += 1;
    last_rho = rho_in;
  }
  // z = M^-1 r, block row by block row.  The residual of the whole camera side sits in shared memory when it fits (the
  // rows of a block belong to different threads): this kernel is a chain of latencies, not of bytes.
  if (r_in_smem && !do_post) {
    for (int i = threadIdx.x; i < nc; i += BA_PCG_T) s_r[i] = R[i];
    __syncthreads();
  }
  const double* __restrict__ RV = r_in_smem ? s_r : R;
  double v = 0.0;
  for (int i = threadIdx.x; i < nc; i += BA_PCG_T) {
    const int4 ri = D.row_info[i];
    const double t = ba_precond_row(ri, MI, RV + ri.x);
    Z[i] = t;
    v += t * RV[i];
  }
  const double rho = ba_cta_allsum(v, sm);
  const bool first = (it == 0);   // first iteration: p = z (never reads the uninitialised / recycled p buffer)
  const double beta = first ? 0.0 : rho / last_rho;
  for (int i = threadIdx.x; i < nc; i += BA_PCG_T) {
    const double p = first ? Z[i] : Z[i] + beta * P[i];
    P[i] = p;
    Q[i] = zero_q ? 0.0 : DC2[i] * p;
  }
  if (threadIdx.x == 0) c->rho = rho;
}

// Latency-tuned form of ba_pcg_mid_kernel for camera sides of up to BA_PCG_T * BA_MID_EPT unknowns (B3: 3994).  The
// single CTA is a chain of dependent memory round trips, so everything a thread will need is requested up front:
// r, x, b and the block-row descriptors stream into shared memory with cp.async while p, q arrive in registers and the
// first reduction runs; the rows of M^-1 are fetched with batched predicated loads.  Same arithmetic, in the same
// order, as ba_pcg_mid_kernel (bit-identical results).
#define BA_MID_EPT 5   // tests/test_ba_paths_gpu.py mirrors the threshold BA_PCG_T * BA_MID_EPT
#define BA_MID_STAGE_BYTES_PER_ROW 40   // r, x, b (doubles) + row_info (int4)
__global__ void __launch_bounds__(BA_PCG_T) ba_pcg_mid_staged_kernel(const BaDev D, double q_tolerance, double r_tolerance,
                                                                     int max_iters, int zero_q, int do_post) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  __shared__ double sm[33];
  __shared__ double sm2[2][33];
  __shared__ int s_done;
  BaCtl* c = D.ctl;
  if (c->done) return;
  const int nc = D.nc;
  int4* s_ri = (int4*)s_raw;                      // [nc]
  double* s_r = (double*)(s_ri + nc);             // [nc]
  double* s_x = s_r + nc;                         // [nc]
  double* s_b = s_x + nc;                         // [nc]
  double* __restrict__ X = D.x; double* __restrict__ R = D.rr; double* __restrict__ P = D.p; double* __restrict__ Q = D.q;
  double* __restrict__ Z = D.z;
  const double* __restrict__ RHS = D.rhs; const double* __restrict__ DC2 = D.Dc2; const double* __restrict__ MI = D.Minv;
#pragma unroll
  for (int e = 0; e < BA_MID_EPT; ++e) {
    const int i = threadIdx.x + e * BA_PCG_T;
    if (i < nc) {
      asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" :: "r"((unsigned)__cvta_generic_to_shared(s_ri + i)), "l"(D.row_info + i) : "memory");
      asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" :: "r"((unsigned)__cvta_generic_to_shared(s_r + i)), "l"(R + i) : "memory");
      if (do_post) {
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" :: "r"((unsigned)__cvta_generic_to_shared(s_x + i)), "l"(X + i) : "memory");
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" :: "r"((unsigned)__cvta_generic_to_shared(s_b + i)), "l"(RHS + i) : "memory");
      }
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  int it = c->it;
  double last_rho = c->last_rho;
  const double rho_in = c->rho, norm_b = c->norm_b, Q0 = c->Q0;
  double pv[BA_MID_EPT];
#pragma unroll
  for (int e = 0; e < BA_MID_EPT; ++e) pv[e] = 0.0;
  if (do_post) {
    double qv[BA_MID_EPT], v = 0.0;
#pragma unroll
    for (int e = 0; e < BA_MID_EPT; ++e) { const int i = threadIdx.x + e * BA_PCG_T; pv[e] = i < nc ? P[i] : 0.0; qv[e] = i < nc ? Q[i] : 0.0; }
#pragma unroll
    for (int e = 0; e < BA_MID_EPT; ++e) { const int i = threadIdx.x + e * BA_PCG_T; if (i < nc) v += pv[e] * qv[e]; }
    const double pq = ba_cta_allsum(v, sm);
    if (!(pq > 0.0)) { if (threadIdx.x == 0) c->done = 1; asm volatile("cp.async.wait_all;" ::: "memory"); return; }
    const double alpha = rho_in / pq;
    asm volatile("cp.async.wait_all;" ::: "memory");   // own elements only: no barrier needed yet
    double a = 0.0, w = 0.0;
#pragma unroll
    for (int e = 0; e < BA_MID_EPT; ++e) {
      const int i = threadIdx.x + e * BA_PCG_T;
      if (i < nc) {
        const double x = s_x[i] + alpha * pv[e], r = s_r[i] - alpha * qv[e];
        X[i] = x; R[i] = r; s_r[i] = r;
        a += -x * (s_b[i] + r); w += r * r;
      }
    }
    ba_cta_sum2(a, w, sm2);
    if (threadIdx.x == 0) s_done = ba_pcg_end_iteration(c, it, rho_in, Q0, a, w, norm_b, q_tolerance, r_tolerance, max_iters);
    __syncthreads();   // publishes s_r (the rows of a block belong to different threads)
    if (s_done) return;
    it += 1;
    last_rho = rho_in;
  } else {
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
  }
  double dv[BA_MID_EPT], zv[BA_MID_EPT], v = 0.0;
#pragma unroll
  for (int e = 0; e < BA_MID_EPT; ++e) { const int i = threadIdx.x + e * BA_PCG_T; dv[e] = (i < nc && !zero_q) ? DC2[i] : 0.0; }
#pragma unroll
  for (int e = 0; e < BA_MID_EPT; ++e) {
    const int i = threadIdx.x + e * BA_PCG_T;
    zv[e] = 0.0;
    if (i < nc) {
      const int4 ri = s_ri[i];
      const double t = ba_precond_row(ri, MI, s_r + ri.x);
      Z[i] = t; zv[e] = t;
      v += t * s_r[i];
    }
  }
  const double rho = ba_cta_allsum(v, sm);
  const bool first = (it == 0);   // first iteration: p = z (never reads the uninitialised / recycled p buffer)
  const double beta = first ? 0.0 : rho / last_rho;
#pragma unroll
  for (int e = 0; e < BA_MID_EPT; ++e) {
    const int i = threadIdx.x + e * BA_PCG_T;
    if (i < nc) {
      const double p = first ? zv[e] : zv[e] + beta * pv[e];
      P[i] = p;
      Q[i] = zero_q ? 0.0 : dv[e] * p;
    }
  }
  if (threadIdx.x == 0) c->rho = rho;
}

__global__ void ba_pcg_dot_pq_kernel(const BaDev D) {
  __shared__ double sm[8];
  if (D.ctl->done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const double v = (i < D.nc) ? D.p[i] * D.q[i] : 0.0;
  const double t = ba_block_sum(v, sm);
  if (threadIdx.x == 0) atomicAdd(&D.ctl->pq, t);
}
// x += alpha p ; r -= alpha q ; Q1 = -x.(b + r) ; |r|^2
__global__ void ba_pcg_update_kernel(const BaDev D) {
  __shared__ double sm[8];
  if (D.ctl->done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v = 0, w = 0;
  const double pq = D.ctl->pq;
  if (pq > 0.0 && i < D.nc) {
    const double alpha = D.ctl->rho / pq;
    const double x = D.x[i] + alpha * D.p[i];
    const double r = D.rr[i] - alpha * D.q[i];
    D.x[i] = x; D.rr[i] = r;
    v = -x * (D.rhs[i] + r);
    w = r * r;
  }
  const double t = ba_block_sum(v, sm);
  const double t2 = ba_block_sum(w, sm);
  if (threadIdx.x == 0) { atomicAdd(&D.ctl->Q1, t); atomicAdd(&D.ctl->rnorm2, t2); }
}
__global__ void ba_pcg_step_kernel(const BaDev D, double q_tolerance, double r_tolerance, int max_iters) {
  BaCtl* c = D.ctl;
  if (c->done) return;
  if (!(c->pq > 0.0)) { c->done = 1; return; }
  ba_pcg_end_iteration(c, c->it, c->rho, c->Q0, c->Q1, c->rnorm2, c->norm_b, q_tolerance, r_tolerance, max_iters);
}

// candidate parameters = Plus(current, scale * step)
__global__ void ba_update_kernel(const BaDev D) {
  // thread ranges padded to whole warps, one kind of block per warp (see ba_gradmax_kernel)
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long np32 = ((long long)D.nposes + 31) & ~31LL, nc32 = ((long long)D.ncams + 31) & ~31LL;
  if (i < np32) {
    if (i >= D.nposes) return;
    const int off = D.pose_off[i];
    for (int k = 0; k < 7; ++k) D.nposes_[7 * i + k] = D.poses[7 * i + k];
    if (off >= 0) {
      const unsigned m = D.pose_mask[i];
      double d[6];
      for (int k = 0; k < 6; ++k) d[k] = ((m >> k) & 1u) ? D.x[off + k] * D.scale_c[off + k] : 0.0;
      ba_quat_plus(D.poses + 7 * i, d, D.nposes_ + 7 * i);
      for (int k = 0; k < 3; ++k) D.nposes_[7 * i + 4 + k] = D.poses[7 * i + 4 + k] + d[3 + k];
    }
  } else if (i < np32 + nc32) {
    const int c = (int)(i - np32);
    if (c >= D.ncams) return;
    const int P = ba_model_num_params(D.cam_model[c]);
    for (int k = 0; k < P; ++k) D.ncams_[D.cam_poff[c] + k] = D.cams[D.cam_poff[c] + k];
    const int off = D.cam_off[c];
    const int ns = D.wide ? D.cam_ns[c] : 0;
    if (off >= 0) for (int k = 0; k < D.cam_nvar[c]; ++k) D.ncams_[D.cam_poff[c] + D.cam_var[BA_MAXP * c + k]] += D.x[off + ns + k] * D.scale_c[off + ns + k];
    if (D.wide && D.cam_sensor[c] >= 0) {   // the camera's sensor_from_rig: Plus(current, scaled step) or a copy
      const long long si = D.cam_sensor[c];
      for (int k = 0; k < 7; ++k) D.nsensors_[7 * si + k] = D.sensors[7 * si + k];
      if (off >= 0 && ns == 6) {
        double d[6];
        for (int k = 0; k < 6; ++k) d[k] = D.x[off + k] * D.scale_c[off + k];
        ba_quat_plus(D.sensors + 7 * si, d, D.nsensors_ + 7 * si);
        for (int k = 0; k < 3; ++k) D.nsensors_[7 * si + 4 + k] = D.sensors[7 * si + 4 + k] + d[3 + k];
      }
    }
  } else {
    const long long p = i - np32 - nc32;
    if (p >= D.npts) return;
    const int v = D.pt_var[p];
    for (int k = 0; k < 3; ++k) D.npts_[3 * p + k] = D.pts[3 * p + k] + (v >= 0 ? D.dp[3 * (long long)v + k] * D.scale_p[3 * (long long)v + k] : 0.0);
  }
}

// ------------------------------------------------------------------------------------------------
// problem set-up on the device: the host decides only which observation sits in which slot (s_obs); the per-slot
// arrays, the (camera, pose) order and everything indexed by it are produced here from the caller's raw arrays.
// ------------------------------------------------------------------------------------------------
__global__ void ba_setup_slot_kernel(long long nslots, const int* __restrict__ s_obs, const int* __restrict__ obs_pose,
                                     const int* __restrict__ obs_cam, const int* __restrict__ obs_pt,
                                     const double* __restrict__ obs_xy, int* __restrict__ s_pose, int* __restrict__ s_cam,
                                     int* __restrict__ s_pt, double* __restrict__ s_xy, unsigned long long* __restrict__ key,
                                     int* __restrict__ val) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nslots) return;
  const int obs = s_obs[s];
  val[s] = (int)s;
  if (obs < 0) {
    s_pose[s] = -1; s_cam[s] = -1; s_pt[s] = -1; s_xy[s] = 0.0; s_xy[nslots + s] = 0.0;
    key[s] = ~0ull;   // padding sorts behind every observation
    return;
  }
  const int pose = obs_pose[obs], cam = obs_cam[obs];
  s_pose[s] = pose; s_cam[s] = cam; s_pt[s] = obs_pt[obs];
  const double2 xy = reinterpret_cast<const double2*>(obs_xy)[obs];
  s_xy[s] = xy.x; s_xy[nslots + s] = xy.y;
  key[s] = ((unsigned long long)(unsigned)cam << 32) | (unsigned)pose;   // (camera, pose) lexicographic
}
// k = position in (camera, pose) order; c2s / keys are the sorted (stable) slot indices and keys
__global__ void ba_setup_cam_kernel(long long nobs_c, long long nobs_c_pad, long long nslots, const unsigned long long* __restrict__ keys,
                                    const int* __restrict__ c2s, const int* __restrict__ s_pt, const int* __restrict__ s_lpt,
                                    const double* __restrict__ s_xy, int* __restrict__ s2c, int2* __restrict__ c_pack,
                                    double* __restrict__ xyC, int* __restrict__ head) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nobs_c_pad) return;
  if (k >= nobs_c) { c_pack[k] = make_int2(0, -1); xyC[BA_U(0, k)] = 0.0; xyC[BA_U(1, k)] = 0.0; return; }
  const int sl = c2s[k];
  s2c[sl] = (int)k;
  c_pack[k] = make_int2(s_pt[sl], s_lpt[sl]);
  xyC[BA_U(0, k)] = s_xy[sl]; xyC[BA_U(1, k)] = s_xy[nslots + sl];
  head[k] = (k == 0 || keys[k] != keys[k - 1]) ? 1 : 0;
}
__global__ void ba_setup_run_kernel(long long nobs_c, const int* __restrict__ run_incl, int* __restrict__ c_run,
                                    const int* __restrict__ head, const unsigned long long* __restrict__ keys,
                                    int* __restrict__ run_start, unsigned long long* __restrict__ run_key) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nobs_c) return;
  const int r = run_incl[k] - 1;
  c_run[k] = r;
  if (head[k]) { run_start[r] = (int)k; run_key[r] = keys[k]; }
}
__global__ void ba_setup_pack_kernel(long long nslots, const int* __restrict__ s_pose, const int* __restrict__ s_cam,
                                     const int* __restrict__ s_lpt, const int* __restrict__ s_seg, const int* __restrict__ s2c,
                                     const int* __restrict__ pose_off, const int* __restrict__ cam_off,
                                     const int* __restrict__ cam_width, int wide, int4* __restrict__ s_pack) {
  const long long sl = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (sl >= nslots) return;
  const int pose = s_pose[sl];
  if (pose < 0) { s_pack[sl] = make_int4(-1, 0, -1, -1); return; }
  const int cam = s_cam[sl];
  const unsigned seg = (unsigned)s_seg[sl];
  const unsigned y = (unsigned)(cam_off[cam] + 1) | ((unsigned)cam_width[cam] << (wide ? 17 : 19)) | ((seg & 0xffu) << 22) | ((seg >> 8) << 27);
  s_pack[sl] = make_int4(pose_off[pose], (int)y, s_lpt[sl], s2c[sl]);
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
thread_local std::string g_ba_error;

// makes o->gpu_index (< 0: the current device) the calling thread's device
int ba_use_device(const b200ba_options* o) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return ba_fail(-101, "no CUDA device: colmap_b200 has no CPU fallback");
  if (o->gpu_index >= 0) {
    if (o->gpu_index >= ndev) return ba_fail(-101, "gpu_index out of range");
    BA_CUDA(cudaSetDevice(o->gpu_index));
  }
  return 0;
}
static int ba_sm_count() { int dev = 0, n = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); return n; }

// Validation, the "used" flags and the variable blocks: pose and camera offsets and masks, camera blocks, variable points.
// neff_cam: effective camera-side parameters.
static int ba_flatten_blocks(const b200ba_options* o, const b200ba_problem* p, BaReducer* red, BaLayout& L,
                             std::vector<int>& used, int& neff_cam) {
  const int NP = p->num_poses, NCAM = p->num_cameras, NS = p->num_sensors;
  const long long NPT = p->num_points, NOBS = p->num_observations;
  for (int c = 0; c < NCAM; ++c) if (ba_model_num_params(p->camera_model_id[c]) < 0) return ba_fail(-2, "unknown camera model id");
  L.wide = NS > 0;
  for (int c = 0; c < NCAM; ++c) {
    if (!ba_model_is_narrow(p->camera_model_id[c])) L.wide = true;
    if (p->camera_sensor_idx && p->camera_sensor_idx[c] >= NS) return ba_fail(-2, "camera_sensor_idx out of range");
  }
  if (NS > 0 && (!p->sensor_from_rig || !p->camera_sensor_idx)) return ba_fail(-2, "rig sensors need sensor_from_rig and camera_sensor_idx");
  used.assign(NP + NCAM, 0);   // [poses | cameras]
  std::vector<unsigned char> pt_used(NPT, 0);
  for (long long i = 0; i < NOBS; ++i) {   // range check and "block appears in an observation" in one pass
    const int a = p->obs_pose_idx[i], b = p->obs_camera_idx[i], c = p->obs_point_idx[i];
    if ((unsigned)a >= (unsigned)NP || (unsigned)b >= (unsigned)NCAM || c < 0 || c >= NPT) return ba_fail(-2, "observation index out of range");
    used[a] = 1; used[NP + b] = 1; pt_used[c] = 1;
  }
  // sharded: a block is "used" if any rank observes it, which keeps the camera-side layout identical on every rank
  if (red) BA_TRY(red->agree(used, ncclInt32, ncclMax));
  const int* cam_used = used.data() + NP;
  L.pose_off.assign(NP, -1); L.pose_mask.assign(NP, 0); L.cam_off.assign(NCAM, -1); L.cam_nvar.assign(NCAM, 0);
  L.cam_poff.resize(NCAM); L.cam_model.resize(NCAM); L.pt_var.assign(NPT, -1); L.cam_var.assign(BA_MAXP * (size_t)NCAM, 0);
  int off = 0, pack = 0;
  neff_cam = 0;
  for (int i = 0; i < NP; ++i) {
    const bool cst = !o->refine_rig_from_world || (p->pose_constant && p->pose_constant[i]) || !used[i];
    if (cst) continue;
    unsigned m = 0x3f;
    if (o->constant_rig_from_world_rotation) m &= ~0x07u;
    if (p->pose_fixed_translation_dim && p->pose_fixed_translation_dim[i] >= 0) m &= ~(1u << (3 + p->pose_fixed_translation_dim[i]));
    L.pose_off[i] = off; L.pose_mask[i] = (unsigned char)m; L.blk_start.push_back(off); L.blk_pack.push_back(pack); off += 6; pack += 36;
    neff_cam += __builtin_popcount(m);
  }
  L.cam_sensor.assign(NCAM, -1); L.cam_ns.assign(NCAM, 0); L.cam_width.assign(NCAM, 0); L.sens_cam.assign(NS, -1);
  L.blk_split.assign(L.blk_start.size(), 0);
  for (int c = 0; c < NCAM; ++c) {
    const int id = p->camera_model_id[c], P = ba_model_num_params(id);
    L.cam_model[c] = id; L.cam_poff[c] = p->camera_param_offset[c];
    L.ncamparams = std::max<long long>(L.ncamparams, L.cam_poff[c] + P);
    int nv = 0;
    if (!(p->camera_constant && p->camera_constant[c]) && cam_used[c])
      for (int k = 0; k < P; ++k) {
        const int g = ba_param_group(id, k);
        const int refine = g == 0 ? o->refine_focal_length : (g == 1 ? o->refine_principal_point : (g == 2 ? o->refine_extra_params : 0));
        if (refine) L.cam_var[BA_MAXP * (size_t)c + nv++] = (signed char)k;
      }
    L.cam_nvar[c] = nv;
    // the camera's sensor_from_rig (non-reference rig sensor): variable iff refined, not constant and observed
    // (ParameterizeRigsAndFrames, bundle_adjustment_ceres.cc:478-539)
    const int si = (NS > 0) ? p->camera_sensor_idx[c] : -1;
    L.cam_sensor[c] = si;
    if (si >= 0) {
      if (L.sens_cam[si] >= 0) return ba_fail(-2, "a sensor_from_rig pose must belong to exactly one camera");
      L.sens_cam[si] = c;
      if (o->refine_sensor_from_rig && !(p->sensor_constant && p->sensor_constant[si]) && cam_used[c]) L.cam_ns[c] = 6;
    }
    const int w = L.cam_ns[c] + nv;
    L.cam_width[c] = w;
    if (w) {
      L.cam_off[c] = off; L.blk_start.push_back(off); L.blk_pack.push_back(pack); L.blk_split.push_back((L.cam_ns[c] && nv) ? 6 : 0);
      off += w; pack += w * w; neff_cam += w; L.dkmax = std::max(L.dkmax, w);
    }
  }
  L.nc = off; L.nblk = (int)L.blk_start.size(); L.pack = pack;
  L.blk_start.push_back(L.nc); L.blk_pack.push_back(pack);
  L.off2blk.resize(L.nc);
  for (int b = 0; b < L.nblk; ++b) for (int i = L.blk_start[b]; i < L.blk_start[b + 1]; ++i) L.off2blk[i] = b;
  for (long long i = 0; i < NPT; ++i) {
    const bool cst = !o->refine_points3D || (p->point_constant && p->point_constant[i]) || !pt_used[i];
    if (!cst) L.pt_var[i] = L.nvpt++;
  }
  return 0;
}
// Packs the tracks (observations vobs[vcount[k] .. vcount[k + 1]) of variable point k) into slots.  Variable points are
// renumbered: tracks of <= 32 observations first (packed so that none crosses a warp), then the longer ones (packed so
// that none crosses a block), then those longer than a block; the observations of constant points follow.
static void ba_pack_tracks(const std::vector<long long>& vcount, const std::vector<long long>& vobs,
                           const std::vector<long long>& const_obs, BaLayout& L) {
  const int nvpt = L.nvpt;
  const size_t cap = (size_t)(L.nobs_eff + L.nobs_eff / 8 + 4 * BA_BLOCK);
  L.s_obs.reserve(cap); L.s_lpt.reserve(cap); L.s_seg.reserve(cap);
  L.vpt_s0.resize(nvpt); L.vpt_s1.resize(nvpt); L.vpt_point.resize(nvpt);
  std::vector<int> order_pts; order_pts.reserve(nvpt);
  std::vector<long long> olen(nvpt), ostart(nvpt);
  for (int k = 0; k < nvpt; ++k) { olen[k] = vcount[k + 1] - vcount[k]; ostart[k] = vcount[k]; }
  {  // short tracks: fill every 32-slot warp greedily with the longest track that still fits (length buckets), so that
     // almost no slot is padding (a first-come packing wastes ~11% at an average track length of 6-7)
    std::vector<std::vector<int>> bucket(33);
    for (int k = nvpt - 1; k >= 0; --k) if (olen[k] <= 32) bucket[olen[k]].push_back(k);   // pop_back yields ascending k
    size_t remaining = 0;
    for (int l = 1; l <= 32; ++l) remaining += bucket[l].size();
    while (remaining) {
      int cap = 32;
      while (cap > 0) {
        int l = std::min(cap, 32);
        while (l > 0 && bucket[l].empty()) --l;
        if (l == 0) break;
        order_pts.push_back(bucket[l].back()); bucket[l].pop_back(); --remaining;
        cap -= l;
      }
    }
  }
  const int nshort = (int)order_pts.size();
  for (int k = 0; k < nvpt; ++k) if (olen[k] > 32 && olen[k] <= BA_BLOCK) order_pts.push_back(k);
  const int nmid = (int)order_pts.size();
  for (int k = 0; k < nvpt; ++k) if (olen[k] > BA_BLOCK) order_pts.push_back(k);
  // renumber: new variable index = position in order_pts
  std::vector<int> newidx(nvpt);
  for (int n = 0; n < nvpt; ++n) newidx[order_pts[n]] = n;
  for (int& v : L.pt_var) if (v >= 0) v = newidx[v];
  for (size_t i = 0; i < L.pt_var.size(); ++i) if (L.pt_var[i] >= 0) L.vpt_point[L.pt_var[i]] = (int)i;
  auto pad_to = [&](size_t mult) {
    const size_t r = L.s_obs.size() % mult;
    if (r) { const size_t add = mult - r; L.s_obs.insert(L.s_obs.end(), add, -1); L.s_lpt.insert(L.s_lpt.end(), add, -1); L.s_seg.insert(L.s_seg.end(), add, 0); }
  };
  auto append_track = [&](int n, int seg) {   // variable point n: its observations vobs[ostart .. ostart + olen)
    const int k = order_pts[n];
    const size_t at = L.s_obs.size(), len = (size_t)olen[k];
    L.vpt_s0[n] = (int)at;
    L.s_obs.resize(at + len); L.s_lpt.insert(L.s_lpt.end(), len, n); L.s_seg.insert(L.s_seg.end(), len, seg);
    for (size_t j = 0; j < len; ++j) L.s_obs[at + j] = (int)vobs[ostart[k] + (long long)j];
    L.vpt_s1[n] = (int)L.s_obs.size();
  };
  auto note_block = [&](int n) {
    const int b = (int)(L.s_obs.size() / BA_BLOCK);
    while ((int)L.blk_pt0.size() <= b) { L.blk_pt0.push_back(n); L.blk_npt.push_back(0); }
    L.blk_npt[b]++;
  };
  for (int n = 0; n < nshort; ++n) {
    const int len = (int)olen[order_pts[n]];
    if ((int)(L.s_obs.size() % 32) + len > 32) pad_to(32);
    note_block(n);
    const int head = (int)(L.s_obs.size() % 32), last = head + len - 1;
    append_track(n, head | (last << 8));
  }
  pad_to(BA_BLOCK);
  L.nblocks_warp = (int)(L.s_obs.size() / BA_BLOCK);
  for (int n = nshort; n < nmid; ++n) {
    if ((int)(L.s_obs.size() % BA_BLOCK) + (int)olen[order_pts[n]] > BA_BLOCK) pad_to(BA_BLOCK);
    note_block(n);
    append_track(n, 0);
  }
  pad_to(BA_BLOCK);
  L.nblocks_giant0 = (int)(L.s_obs.size() / BA_BLOCK);
  for (int n = nmid; n < nvpt; ++n) append_track(n, 0);   // tracks longer than a block: back to back, generic kernels
  pad_to(BA_BLOCK);
  L.nblocks_giant1 = (int)(L.s_obs.size() / BA_BLOCK);
  for (long long i : const_obs) { L.s_obs.push_back((int)i); L.s_lpt.push_back(-1); L.s_seg.push_back(0); }
  pad_to(BA_BLOCK);
  L.nblocks = (int)(L.s_obs.size() / BA_BLOCK);
  L.blk_pt0.resize(L.nblocks, nvpt); L.blk_npt.resize(L.nblocks, 0);
}
// The host flattening of a solve.  red: the reducer of a sharded solve (the ranks agree on the used blocks and on the
// counts), null for a single-GPU solve, which then touches no CUDA API.  Fills the sizes and the solver type of *sum.
int ba_flatten(const b200ba_options* o, const b200ba_problem* p, BaReducer* red, BaLayout& L, b200ba_summary* sum) {
  const int NP = p->num_poses;
  const long long NOBS = p->num_observations;
  std::vector<int> used;   // poses, cameras
  int neff = 0;
  BA_TRY(ba_flatten_blocks(o, p, red, L, used, neff));
  const int nvpt = L.nvpt;
  // effective observations grouped by variable point
  std::vector<long long> vcount(nvpt + 1, 0), const_obs;
  for (long long i = 0; i < NOBS; ++i) {
    const int pv = L.pt_var[p->obs_point_idx[i]];
    if (pv >= 0) { vcount[pv + 1]++; L.nobs_eff++; }
    else if (L.pose_off[p->obs_pose_idx[i]] >= 0 || L.cam_off[p->obs_camera_idx[i]] >= 0) { const_obs.push_back(i); L.nobs_eff++; }
  }
  std::vector<long long> cnt = {L.nobs_eff, 3LL * nvpt};   // over all ranks: effective observations, point parameters
  if (red) BA_TRY(red->agree(cnt, ncclInt64, ncclSum));
  neff += (int)cnt[1];
  sum->num_residuals = (int)(2 * cnt[0]);
  sum->num_effective_parameters = neff;
  L.lst = o->linear_solver_type;
  if (L.lst == B200BA_AUTO) {
    // config.NumImages() decides (bundle_adjustment_ceres.cc:131,204-210), not the number of poses of the whole model:
    // a local BA of six images inside a large reconstruction is a DENSE_SCHUR problem.  Flat callers that do not say
    // get the number of poses that appear in observations.
    int nimg = p->num_config_images;
    if (nimg <= 0) for (int i = 0; i < NP; ++i) nimg += used[i] ? 1 : 0;
    L.lst = nimg <= 50 ? B200BA_DENSE_SCHUR : (nimg <= 1000 ? B200BA_SPARSE_SCHUR : B200BA_ITERATIVE_SCHUR);
  }
  sum->linear_solver_type_used = L.lst;
  if (cnt[0] == 0 || neff == 0) { L.nothing_to_solve = true; return 0; }
  for (int k = 0; k < nvpt; ++k) vcount[k + 1] += vcount[k];
  std::vector<long long> vobs(vcount[nvpt]);
  {
    std::vector<long long> cur(vcount.begin(), vcount.end() - 1);
    for (long long i = 0; i < NOBS; ++i) { const int pv = L.pt_var[p->obs_point_idx[i]]; if (pv >= 0) vobs[cur[pv]++] = i; }
  }
  // rig sensors: a track that sees one variable frame twice (through two of its sensors) needs the cross terms between
  // those observations in the frame's SCHUR_JACOBI block, which ba_schur_pt_kernel forms
  if (p->num_sensors > 0) {
    for (int k = 0; k < nvpt && !L.pose_by_pt; ++k)
      for (long long a = vcount[k]; a < vcount[k + 1] && !L.pose_by_pt; ++a) {
        const int pa = p->obs_pose_idx[vobs[a]];
        if (L.pose_off[pa] < 0) continue;
        for (long long b = a + 1; b < vcount[k + 1]; ++b) if (p->obs_pose_idx[vobs[b]] == pa) { L.pose_by_pt = 1; break; }
      }
  }
  if (NOBS >= (1LL << 31)) return ba_fail(-3, "problem too large for 32-bit observation indices");
  ba_pack_tracks(vcount, vobs, const_obs, L);
  if ((long long)L.s_obs.size() >= (1LL << 31)) return ba_fail(-3, "problem too large for 32-bit slot indices");
  if (L.nc >= (1 << (L.wide ? 17 : 19)) - 1) return ba_fail(-3, L.wide ? "camera-side dimension above 2^17 is not supported with wide camera blocks" : "camera-side dimension above 2^19 is not supported");
  L.DC = 6 + L.dkmax;
  if (L.wide) L.DC = L.dkmax <= 8 ? 14 : (L.dkmax <= 12 ? 18 : (L.dkmax <= 16 ? 22 : 28));
  else if (L.dkmax > BA_MAXDK) return ba_fail(-3, "internal: narrow layout with a camera block wider than five");
  return 0;
}
// ---- device setup ----
static int ba_select_path(const b200ba_options* o, const BaLayout& L, bool sharded, int sms, BaPath& P) {
  const int nc = L.nc;
  const bool exact = L.lst != B200BA_ITERATIVE_SCHUR;
  // exact reduced solves: dense Cholesky of the explicit reduced camera matrix when it is small (camera-side dimension
  // <= BA_DENSE_MAX: the local bundle adjustments of the mapper); larger exact requests run the PCG to a 1e-12 relative
  // residual instead
  P.dense = exact && nc > 0 && nc <= BA_DENSE_MAX && !sharded && getenv("B200BA_NO_DENSE") == nullptr;
  P.r_tol = exact ? 1e-12 : -1.0;
  P.max_cg = exact ? std::max(10 * nc + 100, o->max_linear_solver_iterations) : o->max_linear_solver_iterations;
  P.fused_pcg = nc <= BA_PCG_FUSED_MAX && getenv("B200BA_PCG_MULTI") == nullptr;
  // r of ba_pcg_mid_kernel in (at most 160 KB of) shared memory; tests/test_ba_paths_gpu.py mirrors this threshold
  P.mid_smem = (P.fused_pcg && (size_t)nc * sizeof(double) <= 160 * 1024 && getenv("B200BA_MID_GLOBAL") == nullptr) ? (size_t)nc * sizeof(double) : 0;
  P.mid_staged = (P.fused_pcg && nc <= BA_PCG_T * BA_MID_EPT && getenv("B200BA_MID_PLAIN") == nullptr) ? (size_t)nc * BA_MID_STAGE_BYTES_PER_ROW : 0;
  const char* e = getenv("B200BA_SPMV_SMEM");
  P.spmv_smem = L.nblocks_warp && (!e || atoi(e) != 0) && sizeof(double) * (size_t)nc <= BA_SPMV_SMEM_MAX;
  P.sms = sms;
  // function attributes are per device: set by every solve that needs them (a process may drive several GPUs)
  if (P.mid_smem) BA_CUDA(cudaFuncSetAttribute(ba_pcg_mid_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
  if (P.mid_staged) BA_CUDA(cudaFuncSetAttribute(ba_pcg_mid_staged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_PCG_T * BA_MID_EPT * BA_MID_STAGE_BYTES_PER_ROW));
  if (P.spmv_smem && sizeof(double) * (size_t)nc > 48 * 1024) BA_CUDA(ba_allow_spmv_smem(L));
  return 0;
}
static void ba_normalize_quat(double* q) { const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]); for (int k = 0; k < 4; ++k) q[k] /= n; }
// The per-slot arrays and the camera order, built on the device from the caller's arrays: a stable radix sort of the
// slots by (camera, pose), then runs of equal (camera, pose) and the chunks of the camera-block builds on the host.
static int ba_setup_order(const BaLayout& L, const b200ba_problem* p, long long nobs_c_pad, BaPool& pool, cudaStream_t st, BaDev& D) {
  const long long NOBS = p->num_observations, nslots = D.nslots;
  const long long nobs_c = L.nobs_eff;   // every non-padding slot is an observation connected to a variable block
  std::vector<int4> runs, chunks, chunks_off;
  std::vector<int2> runs_pc;
  int *d_sobs, *d_opose, *d_ocam, *d_opt, *d_val, *d_c2s, *d_head, *d_incl, *d_run_start;
  double* d_oxy;
  unsigned long long *d_key, *d_key_sorted, *d_run_key;
  BA_CUDA(pool.upload(&d_sobs, L.s_obs, st));
  BA_CUDA(pool.alloc(&d_opose, (size_t)NOBS)); BA_CUDA(pool.alloc(&d_ocam, (size_t)NOBS)); BA_CUDA(pool.alloc(&d_opt, (size_t)NOBS)); BA_CUDA(pool.alloc(&d_oxy, 2 * (size_t)NOBS));
  BA_CUDA(cudaMemcpyAsync(d_opose, p->obs_pose_idx, sizeof(int) * (size_t)NOBS, cudaMemcpyHostToDevice, st));
  BA_CUDA(cudaMemcpyAsync(d_ocam, p->obs_camera_idx, sizeof(int) * (size_t)NOBS, cudaMemcpyHostToDevice, st));
  BA_CUDA(cudaMemcpyAsync(d_opt, p->obs_point_idx, sizeof(int) * (size_t)NOBS, cudaMemcpyHostToDevice, st));
  BA_CUDA(cudaMemcpyAsync(d_oxy, p->obs_xy, sizeof(double) * 2 * (size_t)NOBS, cudaMemcpyHostToDevice, st));
  int *t_pose, *t_cam, *t_pt, *t_s2c, *t_crun; double *t_xy, *t_xyC; int2* t_cpack; int4* t_spack;
  BA_CUDA(pool.alloc(&t_pose, (size_t)nslots)); BA_CUDA(pool.alloc(&t_cam, (size_t)nslots)); BA_CUDA(pool.alloc(&t_pt, (size_t)nslots));
  BA_CUDA(pool.alloc(&t_xy, 2 * (size_t)nslots)); BA_CUDA(pool.alloc(&t_s2c, (size_t)nslots)); BA_CUDA(pool.alloc(&t_spack, (size_t)nslots));
  BA_CUDA(pool.alloc(&t_crun, (size_t)nobs_c_pad)); BA_CUDA(pool.alloc(&t_xyC, 2 * (size_t)nobs_c_pad)); BA_CUDA(pool.alloc(&t_cpack, (size_t)nobs_c_pad));
  BA_CUDA(pool.alloc(&d_key, (size_t)nslots)); BA_CUDA(pool.alloc(&d_key_sorted, (size_t)nslots)); BA_CUDA(pool.alloc(&d_val, (size_t)nslots)); BA_CUDA(pool.alloc(&d_c2s, (size_t)nslots));
  BA_CUDA(pool.alloc(&d_head, (size_t)nobs_c_pad)); BA_CUDA(pool.alloc(&d_incl, (size_t)nobs_c_pad));
  const unsigned sb = (unsigned)((nslots + 255) / 256), cb = (unsigned)((nobs_c_pad + 255) / 256);
  ba_setup_slot_kernel<<<sb, 256, 0, st>>>(nslots, d_sobs, d_opose, d_ocam, d_opt, d_oxy, t_pose, t_cam, t_pt, t_xy, d_key, d_val);
  // stable radix sort by (camera, pose): ties keep slot order, padding (key = ~0) ends up behind the nobs_c observations
  size_t tmp_bytes = 0, tmp2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d_key, d_key_sorted, d_val, d_c2s, (int)nslots, 0, 64, st);
  cub::DeviceScan::InclusiveSum(nullptr, tmp2, d_head, d_incl, (int)nobs_c_pad, st);
  tmp_bytes = std::max(tmp_bytes, tmp2);
  unsigned char* d_tmp; BA_CUDA(pool.alloc(&d_tmp, tmp_bytes));
  BA_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_key, d_key_sorted, d_val, d_c2s, (int)nslots, 0, 64, st));
  BA_CUDA(cudaMemsetAsync(t_s2c, 0xff, sizeof(int) * (size_t)nslots, st));
  BA_CUDA(cudaMemsetAsync(d_head, 0, sizeof(int) * (size_t)nobs_c_pad, st));
  BA_CUDA(cudaMemsetAsync(t_crun, 0xff, sizeof(int) * (size_t)nobs_c_pad, st));
  if (nobs_c_pad) ba_setup_cam_kernel<<<cb, 256, 0, st>>>(nobs_c, nobs_c_pad, nslots, d_key_sorted, d_c2s, t_pt, D.s_lpt, t_xy, t_s2c, t_cpack, t_xyC, d_head);
  if (nobs_c) BA_CUDA(cub::DeviceScan::InclusiveSum(d_tmp, tmp_bytes, d_head, d_incl, (int)nobs_c, st));
  int nruns = 0;
  if (nobs_c) {
    BA_CUDA(cudaMemcpyAsync(&nruns, d_incl + (nobs_c - 1), sizeof(int), cudaMemcpyDeviceToHost, st));
    BA_CUDA(cudaStreamSynchronize(st));
  }
  BA_CUDA(pool.alloc(&d_run_start, (size_t)nruns + 1)); BA_CUDA(pool.alloc(&d_run_key, (size_t)nruns + 1));
  if (nobs_c) ba_setup_run_kernel<<<cb, 256, 0, st>>>(nobs_c, d_incl, t_crun, d_head, d_key_sorted, d_run_start, d_run_key);
  ba_setup_pack_kernel<<<sb, 256, 0, st>>>(nslots, t_pose, t_cam, D.s_lpt, D.s_seg, t_s2c, D.pose_off, D.cam_off, D.cam_width, D.wide, t_spack);
  std::vector<int> run_start((size_t)nruns + 1);
  std::vector<unsigned long long> run_key((size_t)nruns + 1);
  if (nruns) {
    BA_CUDA(cudaMemcpyAsync(run_start.data(), d_run_start, sizeof(int) * (size_t)nruns, cudaMemcpyDeviceToHost, st));
    BA_CUDA(cudaMemcpyAsync(run_key.data(), d_run_key, sizeof(unsigned long long) * (size_t)nruns, cudaMemcpyDeviceToHost, st));
    BA_CUDA(cudaStreamSynchronize(st));
  }
  run_start[nruns] = (int)nobs_c;
  // runs of equal (camera, pose); chunks (<= BA_CHUNK observations of one pose block / one intrinsics block)
  // chunk word: first column | width << 8 | first row inside the block << 16 | block width << 24
  auto add_chunks = [&](long long k0, long long k1, int out, int comp0, int ncomp, int lr0, int bw) {
    for (long long c0 = k0; c0 < k1; c0 += BA_CHUNK) chunks.push_back(make_int4((int)c0, (int)std::min<long long>(c0 + BA_CHUNK, k1), out, comp0 | (ncomp << 8) | (lr0 << 16) | (bw << 24)));
  };
  auto add_pair_chunks = [&](long long k0, long long k1, int blk_off, int cA, int nA, int cB, int nB) {
    for (long long c0 = k0; c0 < k1; c0 += BA_CHUNK) chunks_off.push_back(make_int4((int)c0, (int)std::min<long long>(c0 + BA_CHUNK, k1), blk_off, cA | (nA << 8) | (cB << 16) | (nB << 24)));
  };
  long long cam_start = 0;
  for (int r = 0; r < nruns; ++r) {
    const int pose = (int)(run_key[r] & 0xffffffffu), cam = (int)(run_key[r] >> 32);
    const long long k = run_start[r], e = run_start[r + 1];
    runs.push_back(make_int4(L.pose_off[pose], L.cam_off[cam], L.cam_width[cam], 0));
    runs_pc.push_back(make_int2(pose, cam));
    if (L.pose_off[pose] >= 0) add_chunks(k, e, L.pose_off[pose], 0, 6, 0, 6);
    const bool cam_ends = (r + 1 == nruns) || (int)(run_key[r + 1] >> 32) != cam;
    // a variable camera block seen from several poses: some track may see it twice -> the camera blocks of
    // the preconditioner need the cross terms between observations of one point (ba_schur_pt_kernel)
    if (!cam_ends && L.cam_off[cam] >= 0) D.intr_by_pt = 1;
    if (cam_ends) {
      if (L.cam_off[cam] >= 0) {
        const int w = L.cam_width[cam];
        for (int a = 0; a < w; a += 6) {   // 6-column ranges of the block: diagonal ranges here, pairs of ranges separately
          add_chunks(cam_start, e, L.cam_off[cam] + a, 6 + a, std::min(6, w - a), a, w);
          for (int b = a + 6; b < w; b += 6) add_pair_chunks(cam_start, e, L.cam_off[cam], 6 + a, std::min(6, w - a), 6 + b, std::min(6, w - b));
        }
      }
      cam_start = e;
    }
  }
  D.s_pose = t_pose; D.s_cam = t_cam; D.s_pt = t_pt; D.s_xy = t_xy; D.s2c = t_s2c; D.s_pack = t_spack;
  D.c_run = t_crun; D.xyC = t_xyC; D.c_pack = t_cpack;
  BA_CUDA(pool.upload(&D.runs_pc, runs_pc, st));
  BA_CUDA(pool.upload(&D.chunks, chunks, st));
  BA_CUDA(pool.upload(&D.chunks_off, chunks_off, st));
  BA_CUDA(pool.upload(&D.runs, runs, st));
  D.nchunks = (int)chunks.size(); D.nchunks_off = (int)chunks_off.size(); D.nobs_c = nobs_c;
  return 0;
}
// Everything the device holds for one solve: the parameters (current and candidate), the maps of the layout, the slot
// and camera-order arrays and the scratch of the LM and PCG loops.  comm: set for a sharded solve.
int ba_upload(const BaLayout& L, const b200ba_options* o, const b200ba_problem* p, const BaPath& path,
                     b200ba_comm* comm, BaPool& pool, cudaStream_t st, BaDev& D) {
  const int NP = p->num_poses, NS = p->num_sensors, nc = L.nc, nvpt = L.nvpt, pack = L.pack;
  const long long NPT = p->num_points, nslots = (long long)L.s_obs.size();
  memset(&D, 0, sizeof(D));
  D.nposes = NP; D.ncams = p->num_cameras; D.npts = (int)NPT; D.nvpt = nvpt; D.nc = nc; D.DC = L.DC; D.nblocks = L.nblocks;
  D.wide = L.wide ? 1 : 0; D.nsensors = NS;
  D.nblocks_var = L.nblocks_giant0;   // blocks whose tracks are eliminated in shared memory / by shuffles
  D.nslots = nslots; D.loss_type = o->loss_function_type; D.loss_scale = o->loss_function_scale;
  D.nblk = L.nblk;
  std::vector<double> h_poses(p->poses, p->poses + 7 * (size_t)NP), h_cams(p->camera_params, p->camera_params + L.ncamparams),
      h_pts(p->points, p->points + 3 * (size_t)NPT), h_sens(p->sensor_from_rig, p->sensor_from_rig + 7 * (size_t)NS);
  // ParameterizeRigsAndFrames normalises the quaternions of parameterised frames and sensors (bundle_adjustment_ceres.cc:514)
  for (int i = 0; i < NP; ++i) if (L.pose_off[i] >= 0) ba_normalize_quat(h_poses.data() + 7 * (size_t)i);
  for (int k = 0; k < NS; ++k) if (L.sens_cam[k] >= 0 && L.cam_ns[L.sens_cam[k]]) ba_normalize_quat(h_sens.data() + 7 * (size_t)k);
  BA_CUDA(pool.upload(&D.poses, h_poses, st)); BA_CUDA(pool.upload(&D.cams, h_cams, st)); BA_CUDA(pool.upload(&D.pts, h_pts, st));
  BA_CUDA(pool.alloc(&D.nposes_, h_poses.size())); BA_CUDA(pool.alloc(&D.ncams_, h_cams.size())); BA_CUDA(pool.alloc(&D.npts_, h_pts.size()));
  BA_CUDA(pool.upload(&D.pose_off, L.pose_off, st));
  BA_CUDA(pool.upload(&D.pose_mask, L.pose_mask, st));
  BA_CUDA(pool.upload(&D.cam_model, L.cam_model, st));
  BA_CUDA(pool.upload(&D.cam_poff, L.cam_poff, st));
  BA_CUDA(pool.upload(&D.cam_off, L.cam_off, st));
  BA_CUDA(pool.upload(&D.cam_nvar, L.cam_nvar, st));
  BA_CUDA(pool.upload(&D.cam_var, L.cam_var, st));
  BA_CUDA(pool.upload(&D.cam_width, L.cam_width, st));
  BA_CUDA(pool.upload(&D.cam_sensor, L.cam_sensor, st));
  BA_CUDA(pool.upload(&D.cam_ns, L.cam_ns, st));
  BA_CUDA(pool.upload(&D.sens_cam, L.sens_cam, st));
  BA_CUDA(pool.upload(&D.blk_split, L.blk_split, st));
  BA_CUDA(pool.upload(&D.sensors, h_sens, st)); BA_CUDA(pool.alloc(&D.nsensors_, h_sens.size()));
  if (NS) BA_CUDA(cudaMemcpyAsync(D.nsensors_, D.sensors, sizeof(double) * h_sens.size(), cudaMemcpyDeviceToDevice, st));
  BA_CUDA(pool.upload(&D.pt_var, L.pt_var, st));
  BA_CUDA(pool.upload(&D.vpt_point, L.vpt_point, st));
  BA_CUDA(pool.upload(&D.s_lpt, L.s_lpt, st));
  BA_CUDA(pool.upload(&D.s_seg, L.s_seg, st));
  const long long nobs_c_pad = (L.nobs_eff + BA_BLOCK - 1) / BA_BLOCK * BA_BLOCK;
  BA_TRY(ba_setup_order(L, p, nobs_c_pad, pool, st, D));
  BA_CUDA(pool.upload(&D.blk_pt0, L.blk_pt0, st));
  BA_CUDA(pool.upload(&D.blk_npt, L.blk_npt, st));
  BA_CUDA(pool.upload(&D.vpt_s0, L.vpt_s0, st));
  BA_CUDA(pool.upload(&D.vpt_s1, L.vpt_s1, st));
  BA_CUDA(pool.upload(&D.blk_start, L.blk_start, st));
  BA_CUDA(pool.upload(&D.blk_pack, L.blk_pack, st));
  BA_CUDA(pool.upload(&D.off2blk, L.off2blk, st));
  std::vector<int4> row_info((size_t)nc);
  for (int i = 0; i < nc; ++i) {
    const int b = L.off2blk[i], n = L.blk_start[b + 1] - L.blk_start[b], l = i - L.blk_start[b];
    row_info[i] = make_int4(L.blk_start[b], L.blk_pack[b] + l * n, n, 0);
  }
  BA_CUDA(pool.upload(&D.row_info, row_info, st));
  BA_CUDA(pool.alloc(&D.Jc, (size_t)2 * D.DC * nslots)); BA_CUDA(pool.alloc(&D.Jp, (size_t)6 * nslots));
  BA_CUDA(pool.alloc(&D.JcC, (size_t)2 * D.DC * nobs_c_pad)); BA_CUDA(pool.alloc(&D.u, (size_t)nobs_c_pad)); BA_CUDA(pool.alloc(&D.rC, (size_t)2 * nobs_c_pad)); BA_CUDA(pool.alloc(&D.JpC, (size_t)6 * nobs_c_pad));
  D.pose_by_pt = L.pose_by_pt;
  D.nblocks_warp = L.nblocks_warp; D.nblocks_giant0 = L.nblocks_giant0; D.nblocks_giant1 = L.nblocks_giant1;
  BA_CUDA(pool.alloc(&D.zg, (size_t)3 * nvpt));
  BA_CUDA(pool.alloc(&D.r, (size_t)2 * nslots)); BA_CUDA(pool.alloc(&D.cost_slot, (size_t)nslots));
  BA_CUDA(pool.alloc(&D.scale_c, (size_t)nc)); BA_CUDA(pool.alloc(&D.scale_p, (size_t)3 * nvpt));
  BA_CUDA(pool.alloc(&D.Hpp, (size_t)6 * nvpt)); BA_CUDA(pool.alloc(&D.Hpp_inv, (size_t)6 * nvpt)); BA_CUDA(pool.alloc(&D.gp, (size_t)3 * nvpt));
  BA_CUDA(pool.alloc(&D.diag_p, (size_t)3 * nvpt)); BA_CUDA(pool.alloc(&D.Dp2, (size_t)3 * nvpt)); BA_CUDA(pool.alloc(&D.dp, (size_t)3 * nvpt));
  BA_CUDA(pool.alloc(&D.gc, (size_t)nc)); BA_CUDA(pool.alloc(&D.diag_c, (size_t)nc)); BA_CUDA(pool.alloc(&D.Dc2, (size_t)nc)); BA_CUDA(pool.alloc(&D.rhs, (size_t)nc));
  if (comm) {   // symmetric peer buffers for the latency-bound collectives of the LM / PCG loops (kept by the communicator)
    const size_t grouped = (size_t)nc + (size_t)pack + 1;
    ba_p2p_ensure(comm, grouped * sizeof(double) <= BA_P2P_MAX_BYTES ? grouped : ((size_t)nc * sizeof(double) <= BA_P2P_MAX_BYTES ? (size_t)nc : 4), st);
    if (getenv("B200BA_VERBOSE") && comm->rank == 0) fprintf(stderr, "[b200ba] peer-memory all-reduce: %s (cap %zu doubles)\n", comm->p2p.ok ? "on" : "off (NCCL)", comm->p2p.cap);
  }
  BA_CUDA(pool.alloc(&D.Hbb, (size_t)pack)); BA_CUDA(pool.alloc(&D.Mbb, (size_t)pack)); BA_CUDA(pool.alloc(&D.Minv, (size_t)pack));
  BA_CUDA(pool.alloc(&D.x, (size_t)nc)); BA_CUDA(pool.alloc(&D.rr, (size_t)nc)); BA_CUDA(pool.alloc(&D.z, (size_t)nc)); BA_CUDA(pool.alloc(&D.p, (size_t)nc)); BA_CUDA(pool.alloc(&D.q, (size_t)nc));
  if (path.dense) BA_CUDA(pool.alloc(&D.Sd, (size_t)nc * nc));
  BA_CUDA(pool.alloc(&D.ctl, 1));
  BA_CUDA(cudaMemsetAsync(D.ctl, 0, sizeof(BaCtl), st));
  BA_CUDA(cudaMemsetAsync(D.x, 0, sizeof(double) * (nc ? nc : 1), st));
  BA_CUDA(cudaMemsetAsync(D.dp, 0, sizeof(double) * (nvpt ? 3 * (size_t)nvpt : 1), st));
  BA_CUDA(cudaStreamSynchronize(st));
  return 0;
}
// weight chol(cov^-1)^T (CovarianceWeightedCostFunctor::LeftSqrtInformation) of a symmetric positive definite 3x3
// covariance; false when it is not finite, not symmetric or not positive definite
static bool ba_prior_weight(const double* C, double* W) {
  double scale = 0.0;
  for (int k = 0; k < 9; ++k) { if (!std::isfinite(C[k])) return false; scale = std::max(scale, fabs(C[k])); }
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < a; ++b) if (fabs(C[3 * a + b] - C[3 * b + a]) > 1e-12 * scale) return false;
  // positive definite: the leading minors
  const double m1 = C[0], m2 = C[0] * C[4] - C[1] * C[3];
  const double c00 = C[4] * C[8] - C[5] * C[7], c01 = C[5] * C[6] - C[3] * C[8], c02 = C[3] * C[7] - C[4] * C[6];
  const double det = C[0] * c00 + C[1] * c01 + C[2] * c02;
  if (!(m1 > 0.0) || !(m2 > 0.0) || !(det > 0.0)) return false;
  const double id = 1.0 / det;
  const double I[9] = {c00 * id, (C[2] * C[7] - C[1] * C[8]) * id, (C[1] * C[5] - C[2] * C[4]) * id,
                       c01 * id, (C[0] * C[8] - C[2] * C[6]) * id, (C[2] * C[3] - C[0] * C[5]) * id,
                       c02 * id, (C[1] * C[6] - C[0] * C[7]) * id, (C[0] * C[4] - C[1] * C[3]) * id};
  double L[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};   // lower Cholesky factor of the information matrix (its lower triangle)
  for (int j = 0; j < 3; ++j) {
    double d = I[4 * j];
    for (int k = 0; k < j; ++k) d -= L[3 * j + k] * L[3 * j + k];
    if (!(d > 0.0)) return false;
    L[4 * j] = sqrt(d);
    for (int r = j + 1; r < 3; ++r) {
      double t = I[3 * r + j];
      for (int k = 0; k < j; ++k) t -= L[3 * r + k] * L[3 * j + k];
      L[3 * r + j] = t / L[4 * j];
    }
  }
  for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) W[3 * a + b] = L[3 * b + a];
  return std::isfinite(W[0]) && std::isfinite(W[4]) && std::isfinite(W[8]);
}
// linearisation: residual, Jacobian (ceres Corrector with the priors' loss, Jacobi scaling when apply_scale), cost
__global__ void __launch_bounds__(BA_BLOCK) ba_prior_linearize_kernel(const BaDev D, const BaPrior P, int apply_scale) {
  __shared__ double sm[8];
  const int k = blockIdx.x * BA_BLOCK + threadIdx.x;
  double cost = 0.0;
  if (k < P.n) {
    double rw[3], J[36], rho[3];
    ba_prior_eval(D, P, k, D.poses, D.sensors, rw, J);
    const double sq = rw[0] * rw[0] + rw[1] * rw[1] + rw[2] * rw[2];
    ba_loss(P.loss_type, P.loss_scale, sq, rho);
    cost = 0.5 * rho[0];
    const double rs = ba_prior_correct(P, rw, sq, rho, J);
    const int4 ix = P.idx[k];
    for (int j = 0; j < 12; ++j) {
      const int col = ba_prior_col(ix, j);
      const double sc = (apply_scale && col >= 0) ? D.scale_c[col] : 1.0;
      for (int a = 0; a < 3; ++a) P.J[36 * (long long)k + 12 * a + j] = J[12 * a + j] * sc;
    }
    for (int a = 0; a < 3; ++a) P.r[3 * (long long)k + a] = rs * rw[a];
    P.cost[k] = cost;
  }
  const double t = ba_block_sum(cost, sm);
  if (threadIdx.x == 0) atomicAdd(&D.ctl->cost, t);
}
// iteration 0: squared column norms of the unscaled prior rows into scale_c (before ba_make_scale_kernel)
__global__ void ba_prior_colnorm_kernel(const BaDev D, const BaPrior P) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= P.n) return;
  const int4 ix = P.idx[k];
  const double* J = P.J + 36 * (long long)k;
  for (int j = 0; j < 12; ++j) {
    const int col = ba_prior_col(ix, j);
    if (col >= 0) atomicAdd(&D.scale_c[col], J[j] * J[j] + J[12 + j] * J[12 + j] + J[24 + j] * J[24 + j]);
  }
}
// build: J^T J into the diagonal blocks H_bb (the pose block; the sensor part of the camera block) and J^T r into g_c
__global__ void ba_prior_build_kernel(const BaDev D, const BaPrior P) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= P.n) return;
  const int4 ix = P.idx[k];
  const double* J = P.J + 36 * (long long)k;
  const double* r = P.r + 3 * (long long)k;
  for (int blk = 0; blk < 2; ++blk) {
    const int off = blk == 0 ? ix.z : ix.w, j0 = 6 * blk;
    if (off < 0) continue;
    const int b = D.off2blk[off], n = D.blk_start[b + 1] - D.blk_start[b], l0 = off - D.blk_start[b];
    double* H = D.Hbb + D.blk_pack[b];
    for (int i = 0; i < 6; ++i) {
      atomicAdd(&D.gc[off + i], J[j0 + i] * r[0] + J[12 + j0 + i] * r[1] + J[24 + j0 + i] * r[2]);
      for (int j = 0; j < 6; ++j)
        atomicAdd(&H[(l0 + i) * n + l0 + j], J[j0 + i] * J[j0 + j] + J[12 + j0 + i] * J[12 + j0 + j] + J[24 + j0 + i] * J[24 + j0 + j]);
    }
  }
}
// PCG: q += J^T (J p) after the observations' SpMV
__global__ void ba_prior_spmv_kernel(const BaDev D, const BaPrior P) {
  if (D.ctl->done) return;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= P.n) return;
  const int4 ix = P.idx[k];
  const double* J = P.J + 36 * (long long)k;
  double y[3] = {0.0, 0.0, 0.0};
  for (int j = 0; j < 12; ++j) {
    const int col = ba_prior_col(ix, j);
    if (col < 0) continue;
    const double v = D.p[col];
    for (int a = 0; a < 3; ++a) y[a] += J[12 * a + j] * v;
  }
  for (int j = 0; j < 12; ++j) {
    const int col = ba_prior_col(ix, j);
    if (col >= 0) atomicAdd(&D.q[col], J[j] * y[0] + J[12 + j] * y[1] + J[24 + j] * y[2]);
  }
}
// the candidate: model decrease -(J d)^T (r + J d / 2) of the prior rows, their cost at the candidate parameters and
// rho(new) - rho(old) prior by prior
__global__ void __launch_bounds__(BA_BLOCK) ba_prior_step_kernel(const BaDev D, const BaPrior P) {
  __shared__ double sm[8];
  const int k = blockIdx.x * BA_BLOCK + threadIdx.x;
  double model = 0.0, cost = 0.0, delta = 0.0;
  if (k < P.n) {
    const int4 ix = P.idx[k];
    const double* J = P.J + 36 * (long long)k;
    const double* r = P.r + 3 * (long long)k;
    double y[3] = {0.0, 0.0, 0.0};
    for (int j = 0; j < 12; ++j) {
      const int col = ba_prior_col(ix, j);
      if (col < 0) continue;
      const double v = D.x[col];
      for (int a = 0; a < 3; ++a) y[a] += J[12 * a + j] * v;
    }
    model = -(y[0] * (r[0] + 0.5 * y[0]) + y[1] * (r[1] + 0.5 * y[1]) + y[2] * (r[2] + 0.5 * y[2]));
    double rw[3], rho[3];
    ba_prior_eval(D, P, k, D.nposes_, D.nsensors_, rw, nullptr);
    ba_loss(P.loss_type, P.loss_scale, rw[0] * rw[0] + rw[1] * rw[1] + rw[2] * rw[2], rho);
    cost = 0.5 * rho[0];
    delta = cost - P.cost[k];
  }
  double t = ba_block_sum(model, sm);
  if (threadIdx.x == 0) atomicAdd(&D.ctl->model, t);
  t = ba_block_sum(cost, sm);
  if (threadIdx.x == 0) atomicAdd(&D.ctl->new_cost, t);
  t = ba_block_sum(delta, sm);
  if (threadIdx.x == 0) atomicAdd(&D.ctl->cost_delta, t);
}
// Host checks of the caller's priors, before any device work: indices, finite values, SPD covariances.  W receives the
// weights of all priors.
int ba_prior_check(const b200ba_problem* p, const b200ba_position_priors* pr, std::vector<double>& W) {
  if (pr->num_priors < 0) return ba_fail(-2, "num_priors < 0");
  if (pr->num_priors && (!pr->pose_idx || !pr->position || !pr->covariance)) return ba_fail(-1, "null prior array");
  const int t = pr->loss_function_type;
  if (t != B200BA_LOSS_TRIVIAL && t != B200BA_LOSS_SOFT_L1 && t != B200BA_LOSS_CAUCHY && t != B200BA_LOSS_HUBER)
    return ba_fail(-2, "unknown prior loss function type");
  if (t != B200BA_LOSS_TRIVIAL && !(pr->loss_function_scale > 0.0 && std::isfinite(pr->loss_function_scale)))
    return ba_fail(-2, "prior loss function scale must be positive and finite");
  W.assign(9 * (size_t)pr->num_priors, 0.0);
  for (int k = 0; k < pr->num_priors; ++k) {
    const std::string at = "prior " + std::to_string(k) + ": ";
    if (pr->pose_idx[k] < 0 || pr->pose_idx[k] >= p->num_poses) return ba_fail(-2, at + "pose_idx out of range");
    const int s = pr->sensor_idx ? pr->sensor_idx[k] : -1;
    if (s < -1 || s >= p->num_sensors) return ba_fail(-2, at + "sensor_idx out of range");
    for (int a = 0; a < 3; ++a) if (!std::isfinite(pr->position[3 * (size_t)k + a])) return ba_fail(-2, at + "position is not finite");
    for (int a = 0; a < 9; ++a) if (!std::isfinite(pr->covariance[9 * (size_t)k + a])) return ba_fail(-2, at + "covariance is not finite");
    if (!ba_prior_weight(pr->covariance + 9 * (size_t)k, W.data() + 9 * (size_t)k)) return ba_fail(-2, at + "covariance is not symmetric positive definite");
  }
  return 0;
}
// The priors the solve keeps (a pose or sensor block of theirs is variable), uploaded; returns their number in P.n.
int ba_prior_setup(const b200ba_position_priors* pr, const std::vector<double>& W, const BaLayout& L, BaPool& pool,
                          cudaStream_t st, BaPrior& P) {
  std::vector<int4> idx;
  std::vector<double> c, w;
  for (int k = 0; k < pr->num_priors; ++k) {
    const int pi = pr->pose_idx[k], si = pr->sensor_idx ? pr->sensor_idx[k] : -1;
    const int cam = si >= 0 ? L.sens_cam[si] : -1;
    const int po = L.pose_off[pi], so = (cam >= 0 && L.cam_ns[cam] == 6) ? L.cam_off[cam] : -1;
    if (po < 0 && so < 0) continue;   // all its blocks constant (bundle_adjustment_ceres.cc:992-1000)
    idx.push_back(make_int4(pi, si, po, so));
    c.insert(c.end(), pr->position + 3 * (size_t)k, pr->position + 3 * (size_t)k + 3);
    w.insert(w.end(), W.begin() + 9 * (size_t)k, W.begin() + 9 * (size_t)k + 9);
  }
  P.n = (int)idx.size();
  P.loss_type = pr->loss_function_type; P.loss_scale = pr->loss_function_scale;
  if (!P.n) return 0;
  BA_CUDA(pool.upload(&P.idx, idx, st)); BA_CUDA(pool.upload(&P.c, c, st)); BA_CUDA(pool.upload(&P.W, w, st));
  BA_CUDA(pool.alloc(&P.J, 36 * (size_t)P.n)); BA_CUDA(pool.alloc(&P.r, 3 * (size_t)P.n)); BA_CUDA(pool.alloc(&P.cost, (size_t)P.n));
  return 0;
}

// ---- the LM loop ----
// B200BA_PROFILE=1: device-timeline breakdown of the solve by phase (events between the launches; the interval that
// ends at a "host" mark is GPU idle time spent waiting for the host round trip).  Diagnostic only.
enum { PF_LIN, PF_BUILD, PF_AR_BUILD, PF_DIAG, PF_DAMP_SCHUR, PF_AR_SCHUR, PF_INVERT, PF_PCG_INIT, PF_SPMV, PF_AR_Q, PF_MID,
       PF_HOST, PF_BACKSUB, PF_UPDATE_COST, PF_AR_COST, PF_N };
// The phases of one solve on the device and the state they share.  Each returns 0 or a b200ba error code.  The stream
// and events are destroyed on every return path (declared after the pool, so before its release).
struct BaSolve {
  const b200ba_options* o = nullptr;
  cudaStream_t st = nullptr;
  cudaEvent_t ev[4] = {};   // solve start and end; around the first SpMV of every PCG batch
  BaReducer red;
  BaPath path;
  BaDev D;
  BaPrior P;                 // position priors (P.n = 0: none)
  int pack = 0, dkmax = 0;   // packed size of the camera-side blocks, widest camera block
  const bool check = getenv("B200BA_CHECK") != nullptr;   // synchronise and test for asynchronous errors after every group of launches
  const bool profile = getenv("B200BA_PROFILE") != nullptr;
  std::vector<cudaEvent_t> pf_ev;
  std::vector<int> pf_tag;   // phase of the interval that ends at pf_ev[k]
  int launches = 0, spmv_launches = 0;
  double spmv_ms = 0.0;
  BaCtl* h = nullptr;                           // host copy of the control block (pinned when possible)
  BaCtl h_pageable;
  ~BaSolve() {
    for (cudaEvent_t e : pf_ev) cudaEventDestroy(e);
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    if (st) { cudaStreamSynchronize(st); cudaStreamDestroy(st); }
  }
  void mark(int tag) { if (!profile) return; cudaEvent_t e; if (cudaEventCreate(&e) != cudaSuccess) return; cudaEventRecord(e, st); pf_ev.push_back(e); pf_tag.push_back(tag); }
  void report(int world, int lm, float solve_ms) const {
    static const char* const names[PF_N] = {"linearize", "build (cam blocks, gradient)", "all-reduce gc+Hbb", "diag/build_pt/gradmax(+AR)",
        "damp + schur_cam", "all-reduce rhs+Mbb", "invert blocks", "pcg init", "spmv (both passes)", "all-reduce q", "pcg mid",
        "host round trip (GPU idle)", "backsub", "update + cost", "all-reduce cost"};
    double acc[PF_N] = {0}; int cnt[PF_N] = {0};
    for (size_t k = 1; k < pf_ev.size(); ++k) { float ms = 0; if (cudaEventElapsedTime(&ms, pf_ev[k - 1], pf_ev[k]) == cudaSuccess) { acc[pf_tag[k]] += ms; cnt[pf_tag[k]]++; } }
    fprintf(stderr, "[b200ba profile] world %d, %d LM iterations, %.1f ms on the device\n", world, lm, solve_ms);
    for (int t = 0; t < PF_N; ++t) if (cnt[t]) fprintf(stderr, "[b200ba profile] %-30s %8.2f ms %5.1f %%  n=%6d  %7.1f us each  %7.1f us / LM it\n", names[t], acc[t], 100.0 * acc[t] / solve_ms, cnt[t], 1e3 * acc[t] / cnt[t], 1e3 * acc[t] / std::max(lm, 1));
  }
  unsigned gc_blocks() const { return (unsigned)((D.nc + 255) / 256); }
  unsigned gp_blocks() const { return (unsigned)((D.nvpt + 255) / 256); }
  unsigned prior_blocks() const { return (unsigned)((P.n + 255) / 256); }
  bool replica() const { return red.comm && red.comm->rank != 0; }   // sharded, not rank 0: replicated terms come from rank 0
  cudaError_t zero(void* field, size_t bytes = sizeof(double)) { return cudaMemsetAsync(field, 0, bytes, st); }
  cudaError_t read_ctl() { cudaError_t e = cudaMemcpyAsync(h, D.ctl, sizeof(BaCtl), cudaMemcpyDeviceToHost, st); if (e != cudaSuccess) return e; return cudaStreamSynchronize(st); }
  int checkpoint(const char* label) {
    if (!check) return 0;
    cudaError_t e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? 0 : ba_fail(-100, std::string("checkpoint ") + label + ": " + cudaGetErrorString(e));
  }
  int linearize(int apply_scale) {
    BA_CUDA(zero(&D.ctl->cost));
    ba_launch_linearize(D, apply_scale, st);
    if (P.n) { ba_prior_linearize_kernel<<<prior_blocks(), BA_BLOCK, 0, st>>>(D, P, apply_scale); ++launches; }
    mark(PF_LIN);
    BA_CUDA(red(&D.ctl->cost, 1, ncclDouble, ncclSum));
    mark(PF_AR_COST);
    launches += 2;
    return 0;
  }
  // iteration 0: Jacobian and jacobi scaling, then the scaled Jacobian (fp32) in both orders
  int linearize_scaled() {
    BA_TRY(linearize(0));
    BA_TRY(checkpoint("linearize(0)"));
    BA_CUDA(zero(D.scale_c, sizeof(double) * (D.nc ? D.nc : 1)));
    BA_CUDA(zero(D.scale_p, sizeof(double) * (D.nvpt ? 3 * (size_t)D.nvpt : 1)));
    ba_colnorm_kernel<<<D.nblocks, BA_BLOCK, 0, st>>>(D);
    if (P.n) { ba_prior_colnorm_kernel<<<prior_blocks(), 256, 0, st>>>(D, P); ++launches; }   // ceres scales over every residual row
    BA_CUDA(red(D.scale_c, D.nc, ncclDouble, ncclSum));
    if (D.nc) ba_make_scale_kernel<<<gc_blocks(), 256, 0, st>>>(D.scale_c, D.nc, o->jacobi_scaling);
    if (D.nvpt) ba_make_scale_kernel<<<(3 * D.nvpt + 255) / 256, 256, 0, st>>>(D.scale_p, 3LL * D.nvpt, o->jacobi_scaling);
    launches += 3;
    BA_TRY(checkpoint("colnorm"));
    BA_TRY(linearize(1));
    return checkpoint("linearize(1)");
  }
  // normal equations from the current (scaled) Jacobian: camera blocks and gradient, point blocks, gradient max-norm
  int build() {
    BA_CUDA(zero(D.gc, sizeof(double) * (D.nc ? D.nc : 1)));
    BA_CUDA(zero(D.Hbb, sizeof(double) * (pack ? pack : 1)));
    BA_CUDA(zero(&D.ctl->gmax));
    if (D.nchunks) ba_build_cam_sorted_kernel<<<(D.nchunks + BA_SC_BLOCK / 32 - 1) / (BA_SC_BLOCK / 32), BA_SC_BLOCK, 0, st>>>(D);
    BA_TRY(checkpoint("build_cam_sorted"));
    if (D.nchunks_off) ba_cam_offdiag_kernel<false><<<(D.nchunks_off + BA_SC_BLOCK / 32 - 1) / (BA_SC_BLOCK / 32), BA_SC_BLOCK, 0, st>>>(D);
    BA_TRY(checkpoint("cam_offdiag<false>"));
    if (P.n) { ba_prior_build_kernel<<<prior_blocks(), 256, 0, st>>>(D, P); ++launches; }   // before the LM diagonal and gmax read them
    mark(PF_BUILD);
    red.begin();
    BA_CUDA(red(D.gc, D.nc, ncclDouble, ncclSum));
    BA_CUDA(red(D.Hbb, pack, ncclDouble, ncclSum));
    BA_CUDA(red.end());
    mark(PF_AR_BUILD);
    if (D.nc) ba_diag_from_blocks_kernel<<<gc_blocks(), 256, 0, st>>>(D);
    if (D.nvpt) ba_build_pt_kernel<<<gp_blocks(), 256, 0, st>>>(D);
    BA_TRY(checkpoint("diag + build_pt"));
    { const long long n = (((long long)D.nposes + 31) & ~31LL) + (((long long)D.ncams + 31) & ~31LL) + 3LL * D.nvpt; ba_gradmax_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(D); }
    BA_TRY(checkpoint("gradmax"));
    launches += 4;
    BA_CUDA(red(&D.ctl->gmax, 1, ncclDouble, ncclMax));
    mark(PF_DIAG);
    return 0;
  }
  // LM damping, the reduced camera system (rhs and camera blocks) and the inverses of its diagonal blocks
  int damp(double radius) {
    int* d_fail = &D.ctl->fail;   // part of the control block: travels with the per-iteration read
    BA_CUDA(zero(d_fail, sizeof(int)));
    if (D.nvpt) ba_damp_pt_kernel<<<gp_blocks(), 256, 0, st>>>(D, 1.0 / radius, o->min_lm_diagonal, o->max_lm_diagonal, d_fail);
    if (D.nc) ba_damp_cam_kernel<<<gc_blocks(), 256, 0, st>>>(D, 1.0 / radius, o->min_lm_diagonal, o->max_lm_diagonal);
    if (replica()) {  // the replicated terms (-g_c, H_bb + D) are contributed by rank 0 only
      BA_CUDA(zero(D.rhs, sizeof(double) * (D.nc ? D.nc : 1)));
      BA_CUDA(zero(D.Mbb, sizeof(double) * (pack ? pack : 1)));
    }
    if (D.nvpt && D.nc) {
      if (D.nchunks) ba_schur_cam_kernel<<<(D.nchunks + BA_SC_BLOCK / 32 - 1) / (BA_SC_BLOCK / 32), BA_SC_BLOCK, 0, st>>>(D);
      if (D.nchunks_off && !D.intr_by_pt) ba_cam_offdiag_kernel<true><<<(D.nchunks_off + BA_SC_BLOCK / 32 - 1) / (BA_SC_BLOCK / 32), BA_SC_BLOCK, 0, st>>>(D);
      const bool schur_pt = (dkmax > 0 && D.intr_by_pt) || D.pose_by_pt;
      if (schur_pt) ba_schur_pt_kernel<<<gp_blocks(), 256, 0, st>>>(D);
      launches += 1 + (schur_pt ? 1 : 0);
    }
    mark(PF_DAMP_SCHUR);
    red.begin();
    BA_CUDA(red(D.rhs, D.nc, ncclDouble, ncclSum));
    BA_CUDA(red(D.Mbb, pack, ncclDouble, ncclSum));
    BA_CUDA(red(d_fail, 1, ncclInt32, ncclMax));
    BA_CUDA(red.end());
    mark(PF_AR_SCHUR);
    BA_TRY(checkpoint("damp + schur_cam / schur_pt"));
    if (D.nblk && D.nc) { if (D.wide) ba_invert_blocks_kernel<BA_MAXCB><<<(D.nc + 127) / 128, 128, 0, st>>>(D); else ba_invert_blocks_kernel<6><<<(D.nc + 127) / 128, 128, 0, st>>>(D); }
    launches += 4;
    mark(PF_INVERT);
    return checkpoint("invert_blocks");
  }
  // The reduced camera system: dense Cholesky, or PCG in batches of 8 iterations with one host round trip per batch.
  // *h is current afterwards when read is set (the PCG always reads it back).
  int linear_solve(const double& cost, bool read) {
    BA_CUDA(zero(D.ctl, offsetof(BaCtl, iters_total)));  // keeps iters_total
    BA_CUDA(cudaMemcpyAsync(&D.ctl->cost, &cost, sizeof(double), cudaMemcpyHostToDevice, st));
    if (!D.nc || path.dense) {
      if (D.nc) { ba_launch_dense(D, P, st); launches += 3 + (P.n ? 1 : 0); }
      if (read) BA_CUDA(read_ctl());
      return 0;
    }
    ba_pcg_init_kernel<<<gc_blocks(), 256, 0, st>>>(D);
    ++launches;
    mark(PF_PCG_INIT);
    const int zero_q = replica() ? 1 : 0;   // D_c^2 p is contributed by rank 0 only
    auto mid = [&](int do_post) {
      if (path.mid_staged) ba_pcg_mid_staged_kernel<<<1, BA_PCG_T, path.mid_staged, st>>>(D, o->eta, path.r_tol, path.max_cg, zero_q, do_post);
      else ba_pcg_mid_kernel<<<1, BA_PCG_T, path.mid_smem, st>>>(D, o->eta, path.r_tol, path.max_cg, zero_q, do_post, path.mid_smem ? 1 : 0);
    };
    if (path.fused_pcg) { mid(0); ++launches; }
    for (int issued = 0;;) {
      const int batch = std::min(8, path.max_cg - issued);
      for (int b = 0; b < batch; ++b) {
        if (!path.fused_pcg) {
          ba_pcg_precond_kernel<<<gc_blocks(), 256, 0, st>>>(D);
          ba_pcg_direction_kernel<<<gc_blocks(), 256, 0, st>>>(D);
          if (zero_q) BA_CUDA(zero(D.q, sizeof(double) * D.nc));
        }
        if (b == 0) BA_CUDA(cudaEventRecord(ev[2], st));  // first SpMV of a batch always does real work
        ba_launch_spmv(D, path, st);
        if (b == 0) BA_CUDA(cudaEventRecord(ev[3], st));
        if (P.n) { ba_prior_spmv_kernel<<<prior_blocks(), 256, 0, st>>>(D, P); ++launches; }   // q += J^T J p of the prior rows
        mark(PF_SPMV);
        BA_CUDA(red(D.q, D.nc, ncclDouble, ncclSum, &D.ctl->done));  // the one data-path collective of a PCG iteration
        mark(PF_AR_Q);
        if (path.fused_pcg) {
          mid(1);
          launches += 3;
          mark(PF_MID);
        } else {
          ba_pcg_dot_pq_kernel<<<gc_blocks(), 256, 0, st>>>(D);
          ba_pcg_update_kernel<<<gc_blocks(), 256, 0, st>>>(D);
          ba_pcg_step_kernel<<<1, 1, 0, st>>>(D, o->eta, path.r_tol, path.max_cg);
          launches += 7;
        }
      }
      issued += batch;
      BA_CUDA(read_ctl());
      mark(PF_HOST);
      if (batch > 0) { float ms = 0; cudaEventElapsedTime(&ms, ev[2], ev[3]); spmv_ms += ms; spmv_launches += 1; }
      if (h->done || issued >= path.max_cg) return 0;
    }
  }
  // the candidate: point steps by back-substitution, the parameter update, its cost and the model decrease, read back
  int evaluate_step() {
    BA_CUDA(zero(&D.ctl->model));
    ba_launch_backsub(D, st);
    mark(PF_BACKSUB);
    BA_TRY(checkpoint("backsub"));
    { const long long n = (((long long)D.nposes + 31) & ~31LL) + (((long long)D.ncams + 31) & ~31LL) + D.npts; ba_update_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(D); }
    BA_CUDA(zero(&D.ctl->new_cost));
    BA_CUDA(zero(&D.ctl->cost_delta));
    if (D.wide) ba_cost_kernel<true><<<D.nblocks, BA_BLOCK, 0, st>>>(D, D.nposes_, D.ncams_, D.npts_, D.nsensors_, &D.ctl->new_cost);
    else ba_cost_kernel<false><<<D.nblocks, BA_BLOCK, 0, st>>>(D, D.nposes_, D.ncams_, D.npts_, D.nsensors_, &D.ctl->new_cost);
    if (P.n) { ba_prior_step_kernel<<<prior_blocks(), BA_BLOCK, 0, st>>>(D, P); ++launches; }
    BA_TRY(checkpoint("update + cost"));
    mark(PF_UPDATE_COST);
    BA_CUDA(red(&D.ctl->new_cost, 3, ncclDouble, ncclSum));   // new_cost, model, cost_delta are adjacent in BaCtl
    mark(PF_AR_COST);
    launches += 3;
    BA_CUDA(read_ctl());
    mark(PF_HOST);
    return 0;
  }
};
// Copies the variable blocks back into the caller's arrays (constants stay bit-identical).
static int ba_write_back(const BaLayout& L, const BaDev& D, b200ba_problem* p) {
  const int NP = p->num_poses, NCAM = p->num_cameras, NS = p->num_sensors;
  const long long NPT = p->num_points;
  std::vector<double> h_poses(7 * (size_t)NP), h_cams(L.ncamparams), h_pts(3 * (size_t)NPT), h_sens(7 * (size_t)NS);
  BA_CUDA(cudaMemcpy(h_poses.data(), D.poses, sizeof(double) * h_poses.size(), cudaMemcpyDeviceToHost));
  BA_CUDA(cudaMemcpy(h_cams.data(), D.cams, sizeof(double) * h_cams.size(), cudaMemcpyDeviceToHost));
  BA_CUDA(cudaMemcpy(h_pts.data(), D.pts, sizeof(double) * h_pts.size(), cudaMemcpyDeviceToHost));
  for (int i = 0; i < NP; ++i) if (L.pose_off[i] >= 0) memcpy(p->poses + 7 * (size_t)i, h_poses.data() + 7 * (size_t)i, 56);
  for (int c = 0; c < NCAM; ++c) for (int k = 0; k < L.cam_nvar[c]; ++k) { const int idx = L.cam_poff[c] + L.cam_var[BA_MAXP * (size_t)c + k]; p->camera_params[idx] = h_cams[idx]; }
  if (NS) {
    BA_CUDA(cudaMemcpy(h_sens.data(), D.sensors, sizeof(double) * h_sens.size(), cudaMemcpyDeviceToHost));
    for (int k = 0; k < NS; ++k) if (L.sens_cam[k] >= 0 && L.cam_ns[L.sens_cam[k]]) memcpy(p->sensor_from_rig + 7 * (size_t)k, h_sens.data() + 7 * (size_t)k, 56);
  }
  for (long long i = 0; i < NPT; ++i) if (L.pt_var[i] >= 0) memcpy(p->points + 3 * i, h_pts.data() + 3 * i, 24);
  return 0;
}
static int ba_solve_impl(const b200ba_options* o, b200ba_problem* p, b200ba_summary* sum, b200ba_comm* comm,
                         const b200ba_position_priors* priors = nullptr) {
  if (!o || !p || !sum) return ba_fail(-1, "null argument");
  memset(sum, 0, sizeof(*sum));
  sum->termination_type = B200BA_FAILURE;
  if (priors && priors->num_priors == 0) priors = nullptr;
  std::vector<double> prior_w;   // checked before any device work
  if (priors) BA_TRY(ba_prior_check(p, priors, prior_w));
  BaPool pool;
  const auto t_setup0 = std::chrono::steady_clock::now();
  BA_TRY(ba_use_device(o));
  BaSolve S;
  BA_CUDA(cudaStreamCreateWithFlags(&S.st, cudaStreamNonBlocking));
  S.o = o;
  BaReducer& red = S.red;
  red.comm = comm && comm->world > 1 ? comm : nullptr; red.st = S.st; red.pool = &pool; red.sms = ba_sm_count();
  BaLayout L;
  BA_TRY(ba_flatten(o, p, red.comm ? &red : nullptr, L, sum));
  if (L.nothing_to_solve) { sum->termination_type = B200BA_CONVERGENCE; return 0; }
  S.pack = L.pack; S.dkmax = L.dkmax;
  BA_TRY(ba_select_path(o, L, red.comm != nullptr, red.sms, S.path));
  BA_TRY(ba_upload(L, o, p, S.path, red.comm, pool, S.st, S.D));
  if (priors) {
    BA_TRY(ba_prior_setup(priors, prior_w, L, pool, S.st, S.P));
    sum->num_residuals += 3 * S.P.n;
  }
  sum->setup_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_setup0).count();

  for (int i = 0; i < 4; ++i) BA_CUDA(cudaEventCreate(&S.ev[i]));
  // the control block is read back into pinned memory (a pageable destination makes the copy a staged, slower one)
  static thread_local BaCtl* h_pinned = nullptr;
  if (!h_pinned && cudaHostAlloc((void**)&h_pinned, sizeof(BaCtl), cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); h_pinned = nullptr; }
  S.h = h_pinned ? h_pinned : &S.h_pageable;
  const BaCtl& h = *S.h;
  BA_CUDA(cudaEventRecord(S.ev[0], S.st));
  BA_TRY(S.linearize_scaled());
  BA_CUDA(S.read_ctl());
  double cost = h.cost;
  sum->initial_cost = cost;
  double radius = o->initial_trust_region_radius, decrease_factor = 2.0, last_gmax = 0.0;
  int iter = 0, discarded_pcg = 0;
  sum->termination_type = B200BA_NO_CONVERGENCE;
  bool finished = false;
  const bool verbose = getenv("B200BA_VERBOSE") != nullptr;
  while (!finished) {
    BA_TRY(S.build());
    // The gradient-norm test of this iteration is read back together with the first linear-solve batch (one host
    // round trip less per LM iteration); if it says "converged" the enqueued solve is discarded.
    bool check_gmax = true, accepted = false;
    while (!accepted) {
      if (iter >= o->max_num_iterations) {
        if (check_gmax) { BA_CUDA(S.read_ctl()); last_gmax = h.gmax; if (h.gmax <= o->gradient_tolerance) sum->termination_type = B200BA_CONVERGENCE; }
        finished = true; break;
      }
      ++iter;
      BA_TRY(S.damp(radius));
      BA_TRY(S.linear_solve(cost, check_gmax));
      if (check_gmax) {
        check_gmax = false;
        last_gmax = h.gmax;
        if (h.gmax <= o->gradient_tolerance) {
          --iter; discarded_pcg = L.nc ? h.it : 0;
          sum->termination_type = B200BA_CONVERGENCE; finished = true; break;
        }
      }
      BA_TRY(S.checkpoint("linear solve"));
      BA_TRY(S.evaluate_step());
      const int failed = h.fail;
      const double model = h.model, new_cost = h.new_cost;
      // cost change summed residual by residual (same quantity as cost - new_cost, without the cancellation)
      const double cost_change = -h.cost_delta;
      const double rho_q = (!failed && model > 0) ? cost_change / model : 0.0;
      if (verbose) fprintf(stderr, "[b200ba] it %d cost %.12g new %.12g model %.6g rho %.6g radius %.4g pcg_it %d (total %d) gmax %.4g failed %d\n",
                           iter, cost, new_cost, model, rho_q, radius, h.it, h.iters_total, last_gmax, failed);
      if (!failed && model > 0 && rho_q > o->min_relative_decrease) {
        accepted = true;
        sum->num_successful_steps++;
        std::swap(S.D.poses, S.D.nposes_); std::swap(S.D.cams, S.D.ncams_); std::swap(S.D.pts, S.D.npts_); std::swap(S.D.sensors, S.D.nsensors_);
        BA_TRY(S.linearize(1));
        // the cost at the accepted point is the candidate cost just evaluated: no third host round trip per LM iteration
        // (the re-linearisation sums the same per-observation values; it only differs in the order of the block sums)
        cost = new_cost;
        const double t = 2.0 * rho_q - 1.0;
        radius = radius / std::max(1.0 / 3.0, 1.0 - t * t * t);
        radius = std::min(o->max_trust_region_radius, radius);
        decrease_factor = 2.0;
        if (fabs(cost_change) <= o->function_tolerance * cost) { sum->termination_type = B200BA_CONVERGENCE; finished = true; }
      } else {
        sum->num_unsuccessful_steps++;
        radius = radius / decrease_factor;
        decrease_factor *= 2.0;
        if (radius < o->min_trust_region_radius) { sum->termination_type = B200BA_CONVERGENCE; finished = true; break; }
      }
    }
  }
  BA_CUDA(cudaEventRecord(S.ev[1], S.st));
  BA_CUDA(S.read_ctl());
  float solve_ms = 0;
  BA_CUDA(cudaEventElapsedTime(&solve_ms, S.ev[0], S.ev[1]));
  sum->solve_ms = solve_ms;
  if (S.profile && !S.replica()) S.report(red.comm ? red.comm->world : 1, sum->num_successful_steps + sum->num_unsuccessful_steps, solve_ms);
  if (red.comm && red.comm->p2p.ok) {
    unsigned long long timed_out = 0;
    BA_CUDA(cudaMemcpy(&timed_out, red.comm->p2p.state + 2, sizeof(timed_out), cudaMemcpyDeviceToHost));
    if (timed_out) return ba_fail(-111, "peer-memory all-reduce timed out waiting for a rank");
  }
  sum->final_cost = cost;
  sum->num_linear_solver_iterations = h.iters_total - discarded_pcg;
  sum->kernel_launches = S.launches + red.launches;
  sum->spmv_launches = S.spmv_launches;
  sum->spmv_ms_total = S.spmv_ms;
  return ba_write_back(L, S.D, p);   // pool, stream and events are released by their guards
}

extern "C" {

const char* b200ba_last_error(void) { return g_ba_error.c_str(); }

void b200ba_options_init(b200ba_options* o) {
  o->refine_focal_length = 1; o->refine_principal_point = 0; o->refine_extra_params = 1; o->refine_rig_from_world = 1;
  o->refine_points3D = 1; o->constant_rig_from_world_rotation = 0; o->loss_function_type = B200BA_LOSS_TRIVIAL;
  o->loss_function_scale = 1.0; o->linear_solver_type = B200BA_AUTO; o->max_num_iterations = 100;
  o->max_linear_solver_iterations = 200; o->function_tolerance = 0.0; o->gradient_tolerance = 1e-4;
  o->parameter_tolerance = 0.0; o->initial_trust_region_radius = 1e4; o->max_trust_region_radius = 1e16;
  o->min_trust_region_radius = 1e-32; o->min_relative_decrease = 1e-3; o->min_lm_diagonal = 1e-6;
  o->max_lm_diagonal = 1e32; o->eta = 0.1; o->jacobi_scaling = 1; o->gpu_index = -1; o->refine_sensor_from_rig = 1;
}

int b200ba_solve(const b200ba_options* o, b200ba_problem* p, b200ba_summary* sum) { return ba_solve_impl(o, p, sum, nullptr); }

// Point-sharded solve: every rank passes the SAME poses / cameras and its own shard of points with all their
// observations (SURVEY.md §8e).  Collectives: one all-reduce of the camera-side vector per PCG iteration, a handful
// of small ones per LM iteration.  poses / camera_params come back identical on every rank.
int b200ba_solve_sharded(const b200ba_options* o, b200ba_problem* p, b200ba_comm_t comm, b200ba_summary* sum) {
  if (!comm) return ba_fail(-1, "null communicator");
  return ba_solve_impl(o, p, sum, comm);
}

// ---- host-side hooks for the CPU test tier ----
int b200ba_test_reproj(int model_id, const double* point, const double* pose, const double* params, const double* xy,
                       double* res, double* J_point, double* J_pose, double* J_params) {
  return ba_reproj(model_id, point, pose, params, xy[0], xy[1], res, J_point, J_pose, J_params) ? 1 : 0;
}
void b200ba_test_quat_plus(const double* q, const double* d, double* out) { ba_quat_plus(q, d, out); }
// RigReprojErrorCostFunctor with analytic derivatives, any of the eighteen models (host evaluation of the device code):
// sensor == NULL -> trivial frame.  J_params is [2 x P] row-major.  Returns 1 / 0 (behind the camera) / -1 (unknown model).
int b200ba_test_reproj_rig(int model_id, const double* point, const double* rig, const double* sensor, const double* params,
                           const double* xy, double* res, double* J_point, double* J_rig, double* J_sensor, double* J_params) {
  const int P = ba_model_num_params(model_id);
  if (P < 0) return -1;
  double Jp[2 * BA_MAXP];
  const bool ok = ba_reproj_rig(model_id, point, rig, sensor, params, xy[0], xy[1], res, J_point, J_rig, J_sensor, Jp);
  for (int k = 0; k < P; ++k) { J_params[k] = Jp[k]; J_params[P + k] = Jp[BA_MAXP + k]; }
  return ok ? 1 : 0;
}

// The twelve camera models outside the radial pinhole family (ba_models.cuh: formulas + dual numbers), host evaluation for the CPU
// test tier: xy[2], J_uvw[2x3], J_params[2xP].  Returns 1 / 0 (depth guard) / -1 (unknown model).
int b200ba_test_project_wide(int model_id, const double* params, const double* uvw, double* xy, double* J_uvw, double* J_params) {
  switch (ba_wide_model_num_params(model_id)) {
    case 2: return ba_project_wide_with_jac<2>(model_id, params, uvw[0], uvw[1], uvw[2], xy, J_uvw, J_params) ? 1 : 0;
    case 3: return ba_project_wide_with_jac<3>(model_id, params, uvw[0], uvw[1], uvw[2], xy, J_uvw, J_params) ? 1 : 0;
    case 4: return ba_project_wide_with_jac<4>(model_id, params, uvw[0], uvw[1], uvw[2], xy, J_uvw, J_params) ? 1 : 0;
    case 6: return ba_project_wide_with_jac<6>(model_id, params, uvw[0], uvw[1], uvw[2], xy, J_uvw, J_params) ? 1 : 0;
    case 16: return ba_project_wide_with_jac<16>(model_id, params, uvw[0], uvw[1], uvw[2], xy, J_uvw, J_params) ? 1 : 0;
    case 5: return ba_project_wide_with_jac<5>(model_id, params, uvw[0], uvw[1], uvw[2], xy, J_uvw, J_params) ? 1 : 0;
    case 8: return ba_project_wide_with_jac<8>(model_id, params, uvw[0], uvw[1], uvw[2], xy, J_uvw, J_params) ? 1 : 0;
    case 12: return ba_project_wide_with_jac<12>(model_id, params, uvw[0], uvw[1], uvw[2], xy, J_uvw, J_params) ? 1 : 0;
    default: return -1;
  }
}

// The host flattening of b200ba_solve without a GPU: which observation sits in which slot.  Two-call pattern: with
// capacity 0 only the sizes come back.  info[10] = {nslots, nvpt, nblocks_warp, nblocks_var, nblocks_giant0,
// nblocks_giant1, camera-side dimension, max variable intrinsics, num_residuals, num_effective_parameters}.  A problem
// with nothing to solve returns 0 and leaves info as it is.
int b200ba_test_pack(const b200ba_options* o, b200ba_problem* p, int64_t capacity, int32_t* s_obs, int32_t* s_lpt,
                     int32_t* s_seg, int32_t* vpt_s0, int32_t* vpt_s1, int32_t* vpt_point, int64_t* info) {
  if (!o || !p) return ba_fail(-1, "null argument");
  BaLayout L;
  b200ba_summary sum = {};
  const int rc = ba_flatten(o, p, nullptr, L, &sum);
  if (rc || L.nothing_to_solve) return rc;
  info[0] = (int64_t)L.s_obs.size(); info[1] = L.nvpt; info[2] = L.nblocks_warp; info[3] = L.nblocks_giant0;
  info[4] = L.nblocks_giant0; info[5] = L.nblocks_giant1; info[6] = L.nc; info[7] = L.dkmax;
  info[8] = sum.num_residuals; info[9] = sum.num_effective_parameters;
  if (capacity == 0) return 0;
  if (capacity < (int64_t)L.s_obs.size()) return -12;
  memcpy(s_obs, L.s_obs.data(), sizeof(int) * L.s_obs.size());
  memcpy(s_lpt, L.s_lpt.data(), sizeof(int) * L.s_lpt.size());
  memcpy(s_seg, L.s_seg.data(), sizeof(int) * L.s_seg.size());
  memcpy(vpt_s0, L.vpt_s0.data(), sizeof(int) * L.vpt_s0.size());
  memcpy(vpt_s1, L.vpt_s1.data(), sizeof(int) * L.vpt_s1.size());
  memcpy(vpt_point, L.vpt_point.data(), sizeof(int) * L.vpt_point.size());
  return 0;
}

// ---- position priors (include/b200_ba_pose_prior.h) ----
void b200ba_position_priors_init(b200ba_position_priors* p) {
  memset(p, 0, sizeof(*p));
  p->loss_function_type = B200BA_LOSS_TRIVIAL;
  p->loss_function_scale = 2.7954834829151074;   // sqrt(7.814727903251179), the chi-square 95 % quantile of 3 DoF
}
int b200ba_solve_with_position_priors(const b200ba_options* o, b200ba_problem* p, const b200ba_position_priors* priors,
                                      b200ba_summary* out) {
  return ba_solve_impl(o, p, out, nullptr, priors);
}
void b200ba_test_prior_position(const double* rig, const double* sensor, const double* position, double* res,
                                double* J_rig, double* J_sensor) {
  ba_prior_position(rig, sensor, position, res, J_rig, J_sensor);
}
int b200ba_test_prior_weight(const double* covariance, double* weight) {
  return ba_prior_weight(covariance, weight) ? 0 : ba_fail(-2, "covariance is not symmetric positive definite");
}

}  // extern "C"
