// ba_linearize.cu — linearisation of the observations: residual and scaled Jacobian rows in both storage orders.
#include "ba_common.cuh"

// Linearisation, pass 1 (slot order = track order): scaled Jacobians Jc / Jp (fp32), residual, per-slot cost.
// (two CTAs per SM: the register cap of 128 matters - at 130 the occupancy halves)
template <int DC, bool WIDE>
__global__ void __launch_bounds__(BA_BLOCK, WIDE ? 1 : 2) ba_linearize_slot_kernel(const BaDev D, int apply_scale, double* cost_out) {
  __shared__ double sm[8];
  const long long s = (long long)blockIdx.x * BA_BLOCK + threadIdx.x;
  double cost = 0.0;
  const int pi = D.s_pose[s];
  double Jc[2 * DC], Jpt[6], rr[2] = {0.0, 0.0};
  if (pi >= 0) {
    cost = ba_obs_linearize<DC, WIDE>(D, D.poses, D.cams, D.pts, pi, D.s_cam[s], D.s_pt[s], D.s_lpt[s], D.s_xy[s],
                                D.s_xy[D.nslots + s], apply_scale, Jc, Jpt, rr);
  } else {
#pragma unroll
    for (int k = 0; k < 2 * DC; ++k) Jc[k] = 0.0;
#pragma unroll
    for (int k = 0; k < 6; ++k) Jpt[k] = 0.0;
  }
#pragma unroll
  for (int k = 0; k < 2 * DC; ++k) D.Jc[BA_JC(k, s)] = (float)Jc[k];
#pragma unroll
  for (int k = 0; k < 6; ++k) D.Jp[BA_JP(k, s)] = (float)Jpt[k];
  D.r[s] = rr[0];
  D.r[D.nslots + s] = rr[1];
  D.cost_slot[s] = cost;
  const double t = ba_block_sum(cost, sm);
  if (threadIdx.x == 0) atomicAdd(cost_out, t);
}
// Linearisation, pass 2 (camera order): the same rows again, written as JcC / JpC / rC for the passes that reduce per
// camera-side block.  Recomputing (one 24-byte point gather per observation) replaces 2*DC + 2 scattered stores.
template <int DC, bool WIDE>
__global__ void __launch_bounds__(BA_BLOCK, WIDE ? 1 : 2) ba_linearize_cam_kernel(const BaDev D, int apply_scale) {
  const long long k = (long long)blockIdx.x * BA_BLOCK + threadIdx.x;
  const int run = D.c_run[k];
  if (run < 0) return;
  const int2 pc = D.runs_pc[run];
  const int2 tl = D.c_pack[k];
  double Jc[2 * DC], Jpt[6], rr[2];
  ba_obs_linearize<DC, WIDE>(D, D.poses, D.cams, D.pts, pc.x, pc.y, tl.x, tl.y, D.xyC[BA_U(0, k)], D.xyC[BA_U(1, k)], apply_scale,
                       Jc, Jpt, rr);
#pragma unroll
  for (int c = 0; c < 2 * DC; ++c) D.JcC[BA_JC(c, k)] = (float)Jc[c];
#pragma unroll
  for (int c = 0; c < 6; ++c) D.JpC[BA_JP(c, k)] = (float)Jpt[c];
  D.rC[BA_U(0, k)] = rr[0];
  D.rC[BA_U(1, k)] = rr[1];
}
template <int DC>
static void ba_launch_linearize_dc(const BaDev& D, int apply_scale, cudaStream_t s) {
  constexpr bool WIDE = DC >= 14;
  ba_linearize_slot_kernel<DC, WIDE><<<D.nblocks, BA_BLOCK, 0, s>>>(D, apply_scale, &D.ctl->cost);
  if (D.nobs_c) ba_linearize_cam_kernel<DC, WIDE><<<(unsigned)((D.nobs_c + BA_BLOCK - 1) / BA_BLOCK), BA_BLOCK, 0, s>>>(D, apply_scale);
}
void ba_launch_linearize(const BaDev& D, int apply_scale, cudaStream_t s) { BA_DISPATCH_DC(ba_launch_linearize_dc, D, apply_scale, s); }
