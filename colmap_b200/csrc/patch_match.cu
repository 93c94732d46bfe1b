// patch_match.cu — CUDA (sm_90a, H100) PatchMatch MVS sweep behind the C-ABI of include/b200_patch_match.h.
//
// Reference behaviour: src/colmap/mvs/patch_match_cuda.cu (PatchMatchCuda).  Design (DESIGN.md §2):
//   * no physical Rotate() between sweeps (patch_match_cuda.cu:1859-1939): the four sweep
//     directions are index maps (frames) over buffers that stay in the original orientation;
//   * each sweep runs as four passes: R draws every row's random hypothesis and Monte-Carlo uniforms
//     from the column's PRNG stream, M (beside R) computes the column's HMM messages over the
//     sweep-start costs, P evaluates pixel-parallel everything that does not depend on the row above,
//     and S, one CTA of WPC warps per column, carries the column's sequential state (propagated plane,
//     forward messages, sampling, argmin, filter);
//   * each NCC is evaluated by an 8-lane group, so a warp runs four (hypothesis, image) pairs at once;
//   * bilateral weights are computed once per pixel (they only depend on the reference patch) instead
//     of once per NCC evaluation, and each (hypothesis, source image) pair is evaluated once per pixel
//     instead of once per Monte-Carlo sample (NCC is a pure function of the pair);
//   * source images are stored as 2x2-footprint words so a bilinear tap is one 32-bit load;
//   * XORWOW state is kept only for the border pixels the sweeps actually consume
//     (the reference keeps and rotates a 48 B/pixel state map, :1811,1872-1878).
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/b200_patch_match.h"
#include "device_cache.h"
#include "pm_device.cuh"

// ------------------------------------------------------------------------------------------------
// parameter blocks
// ------------------------------------------------------------------------------------------------
struct PmSrcDesc {
  int w, h, pitch, pad;
  long long quad_off;   // in 32-bit words
  long long depth_off;  // in floats
};

struct PmParams {
  int W0, H0, N;
  int radius, step, nside, ntaps, ntaps_pad, num_samples;
  int geom, filter_min_num_consistent;
  float depth_min, depth_max, spatial_norm, color_norm;
  PmLikelihood L;
  float geom_reg, geom_max_cost, filter_geom_max_cost, min_ncc_prob, cos_filter_tri;
  const uint8_t* ref_raw;
  uint8_t* ref_img;
  float* ref_sum;
  float* ref_sqsum;
  float4* hyp;     // {depth, nx, ny, nz} per pixel, original orientation
  float* cost;     // [pixel][N]
  uint8_t* mask;   // [pixel][N]
  const uint32_t* quads;
  const float* src_depth;
  const PmSrcDesc* src;
  const float* poses;  // [4][N][43]
  const float* init_depth;   // geom mode
  const float* init_normal;  // geom mode, 3 planes
  uint32_t* rng;       // [perimeter][6]
  float2* patch_store; // [pixel][ntaps_st] {w, w * ref} of every tap in the original orientation (pm_patch_kernel);
                       // nullptr: every consumer builds the reference patch inline (pm_build_patch)
  float* patch_inv;    // [pixel][4] 1 / sum(w), summed in the tap order of sweep frame 0..3
  int ntaps_st;        // taps per pixel block of patch_store: ntaps rounded up to even (16-byte aligned blocks)
  float K[4][4], invK[4][4];
};

struct PmSweepArgs {
  int rot;
  float perturbation, perturbation_pi, prev_w;
  int last_filter;
  float* sel_cur;
  const float* sel_prev;
  // split pipeline scratch (per pixel, original-orientation pixel index)
  float4* rand_hyp;        // random hypothesis of the pixel in the sweep frame {depth, n}
  float* usamp;            // [pixel][num_samples] Monte-Carlo uniforms (already minus FLT_EPSILON, :1129)
  float* prior3;           // [pixel][3][N] triangulation / incident / resolution priors of the current hypothesis
  float* tab3;             // [pixel][3][N] NCC of hypotheses 2,3,4 for every source image
  float* gtab2;            // [pixel][2][N] geometric cost at cur / rand depth (geom mode)
  float* fwd_pred;         // [pixel][N] forward messages of the column over the sweep-START costs (pass M): the pixel pass
                           // predicts which images the serial pass will sample from them
  int prune;               // 0: the pixel pass evaluates every (hypothesis, image) pair; 1: prediction + exact early-out;
                           // 2: (tests) the pixel pass evaluates nothing, the serial pass fills every entry itself
  int col0;                // always 0; pm_serial_kernel reads its column as col0 + blockIdx.x because with blockIdx.x
                           // alone the compiler schedules the row loop differently and the serial pass measured ~0.7 ms
                           // per C2 sweep slower (H100 80GB HBM3 SXM, 400 W power limit)
};
#define PM_NOT_EVALUATED (-1.0f)   // tab3 sentinel (an NCC cost is always in [0, 2])

// ------------------------------------------------------------------------------------------------
// frame maps: frame k = the reference's buffers after k Rotate() calls (cuda_rotate.h:57-75):
//   (r_{k+1}, c_{k+1}) = (w_k - 1 - c_k, r_k)
// ------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ void pm_frame_to_orig(int W0, int H0, int rot, int r, int c, int* r0, int* c0) {
  switch (rot) {
    case 0: *r0 = r; *c0 = c; break;
    case 1: *r0 = c; *c0 = W0 - 1 - r; break;
    case 2: *r0 = H0 - 1 - r; *c0 = W0 - 1 - c; break;
    default: *r0 = H0 - 1 - c; *c0 = r; break;
  }
}
// The four frame maps are affine in (r, c): pixel index = base + r * stride_r + c * stride_c (two IMADs, no branch)
__host__ __device__ __forceinline__ size_t pm_pix0(int W0, int H0, int rot, int r, int c) {
  const int sr = (rot == 0) ? W0 : ((rot == 1) ? -1 : ((rot == 2) ? -W0 : 1));
  const int sc = (rot == 0) ? 1 : ((rot == 1) ? W0 : ((rot == 2) ? -1 : -W0));
  const int base = (rot == 0) ? 0 : ((rot == 1) ? (W0 - 1) : ((rot == 2) ? (H0 * W0 - 1) : ((H0 - 1) * W0)));
  return (size_t)(base + r * sr + c * sc);
}
// RotateNormalMap applied k times / undone (patch_match_cuda.cu:849-861)
__host__ __device__ __forceinline__ void pm_normal_to_frame(int rot, float& nx, float& ny) {
  const float x = nx, y = ny;
  switch (rot) {
    case 0: break;
    case 1: nx = y; ny = -x; break;
    case 2: nx = -x; ny = -y; break;
    default: nx = -y; ny = x; break;
  }
}
__device__ __forceinline__ void pm_normal_to_orig(int rot, float& nx, float& ny) {
  const float x = nx, y = ny;
  switch (rot) {
    case 0: break;
    case 1: nx = -y; ny = x; break;
    case 2: nx = -x; ny = -y; break;
    default: nx = y; ny = -x; break;
  }
}
// index of a border pixel in the compact PRNG state array
__host__ __device__ __forceinline__ int pm_border_index(int W0, int H0, int r0, int c0) {
  if (r0 == 0) return c0;
  if (r0 == H0 - 1) return W0 + c0;
  if (c0 == 0) return 2 * W0 + (r0 - 1);
  return 2 * W0 + (H0 - 2) + (r0 - 1);
}
// (float)v / 255.0f for v = 0..255, IEEE division done once on the host: the same bits as the division it replaces.
// Every kernel that reads reference colours copies it into shared memory first (pm_load_lut): the lanes of a warp
// index it with different bytes, which __constant__ memory would serialise.
__device__ float pm_lut255[256];
static void pm_upload_lut() {
  static thread_local int done_dev = -1;
  int dev = 0; cudaGetDevice(&dev);
  if (done_dev == dev) return;
  float h[256];
  for (int i = 0; i < 256; ++i) { volatile float a = (float)i, b = 255.0f; h[i] = a / b; }
  cudaMemcpyToSymbol(pm_lut255, h, sizeof(h));
  done_dev = dev;
}
__device__ __forceinline__ void pm_load_lut(float* lut, int tid, int nthreads) {
  for (int i = tid; i < 256; i += nthreads) lut[i] = pm_lut255[i];
}
__device__ __forceinline__ float pm_ref_color(const PmParams& P, const float* lut, int rot, int fw, int fh, int r, int c) {
  if (r < 0 || c < 0 || r >= fh || c >= fw) return 0.0f;
  return lut[P.ref_img[pm_pix0(P.W0, P.H0, rot, r, c)]];
}
// Tap t = (tr, tc) of sweep frame `rot` (offset (dr, dc) = (-radius + step * tr, -radius + step * tc)) is the tap of
// the original orientation at the offset the frame map rotates (dr, dc) to: (dc, -dr), (-dr, -dc), (-dc, dr) for
// frames 1, 2, 3.  The window is symmetric, so that offset is a tap too; this returns its index.
__device__ __forceinline__ int pm_orig_tap(int rot, int nside, int t) {
  const int tr = t / nside, tc = t - tr * nside, m = nside - 1;
  switch (rot) {
    case 0: return t;
    case 1: return tc * nside + (m - tr);
    case 2: return (m - tr) * nside + (m - tc);
    default: return (m - tc) * nside + tr;
  }
}

// ------------------------------------------------------------------------------------------------
// one-off kernels
// ------------------------------------------------------------------------------------------------
// GpuMatRefImage::Filter / FilterKernel (gpu_mat_ref_image.cu:39-82)
__global__ void pm_prefilter_kernel(const PmParams P) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = blockIdx.y * blockDim.y + threadIdx.y;
  if (col >= P.W0 || row >= P.H0) return;
  const int w = P.W0, h = P.H0, r = P.radius, s = P.step;
  const float center = (float)P.ref_raw[(size_t)row * w + col] / 255.0f;
  float cs = 0.0f, cq = 0.0f, ws = 0.0f;
  for (int dr = -r; dr <= r; dr += s) {
    for (int dc = -r; dc <= r; dc += s) {
      const int rr = row + dr, cc = col + dc;
      const float color = (rr < 0 || cc < 0 || rr >= h || cc >= w) ? 0.0f : (float)P.ref_raw[(size_t)rr * w + cc] / 255.0f;
      const float bw = pm_bilateral_weight(P.spatial_norm, P.color_norm, dr, dc, center, color);
      const float wc = bw * color;
      cs += wc;
      cq = fmaf(wc, color, cq);
      ws += bw;
    }
  }
  P.ref_sum[(size_t)row * w + col] = cs / ws;
  P.ref_sqsum[(size_t)row * w + col] = cq / ws;
  P.ref_img[(size_t)row * w + col] = (uint8_t)(255.0f * center);
}

// 2x2 footprint packing of one source image with a 2-pixel zero apron.
__global__ void pm_pack_quads_kernel(const uint8_t* __restrict__ img, int w, int h, int pitch, uint32_t* __restrict__ out) {
  const int X = blockIdx.x * blockDim.x + threadIdx.x;  // 0 .. w+3
  const int Y = blockIdx.y * blockDim.y + threadIdx.y;  // 0 .. h+3
  if (X >= w + 4 || Y >= h + 4) return;
  const int x = X - 2, y = Y - 2;
  auto T = [&](int xx, int yy) -> uint32_t {
    return (xx < 0 || yy < 0 || xx >= w || yy >= h) ? 0u : (uint32_t)img[(size_t)yy * w + xx];
  };
  out[(size_t)Y * pitch + X] = T(x, y) | (T(x + 1, y) << 8) | (T(x, y + 1) << 16) | (T(x + 1, y + 1) << 24);
}

// GpuMatPRNG ctor + FillWithRandomNumbers + InitNormalMap (gpu_mat_prng.cu:36-48, gpu_mat.h:371-387,
// patch_match_cuda.cu:835-846), or the geometric-mode copy (:1814-1852); prev_sel_prob = 0.5 (:1835).
__global__ void pm_init_kernel(const PmParams P, float* sel_prev) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = blockIdx.y * blockDim.y + threadIdx.y;
  if (col >= P.W0 || row >= P.H0) return;
  const size_t p = (size_t)row * P.W0 + col;
  const int gx = (P.W0 - 1) / 32 + 1;
  const unsigned long long id =
      (unsigned long long)((row / 16) * gx + (col / 32)) * 512ull + (unsigned long long)((row % 16) * 32 + (col % 32));
  PmRng rs;
  pm_rng_init(rs, id);
  float4 hy;
  if (P.geom) {
    const size_t n = (size_t)P.W0 * P.H0;
    hy = make_float4(P.init_depth[p], P.init_normal[p], P.init_normal[n + p], P.init_normal[2 * n + p]);
  } else {
    const float depth = fmaf(pm_rng_uniform(rs), P.depth_max - P.depth_min, P.depth_min);
    float nv[3];
    pm_random_normal(P.invK[0], (float)row, (float)col, rs, nv);
    hy = make_float4(depth, nv[0], nv[1], nv[2]);
  }
  P.hyp[p] = hy;
  if (row == 0 || col == 0 || row == P.H0 - 1 || col == P.W0 - 1) {
    uint32_t* st = P.rng + 6 * (size_t)pm_border_index(P.W0, P.H0, row, col);
    st[0] = rs.v0; st[1] = rs.v1; st[2] = rs.v2; st[3] = rs.v3; st[4] = rs.v4; st[5] = rs.d;
  }
  for (int i = 0; i < P.N; ++i) sel_prev[p * P.N + i] = 0.5f;
}

// ------------------------------------------------------------------------------------------------
// NCC of one (hypothesis, source image) pair by an 8-lane group
// (PhotoConsistencyCostComputer::Compute, patch_match_cuda.cu:489-593)
// ------------------------------------------------------------------------------------------------
// Phases of the pixel pass.  A build with -DPM_PIXEL_PHASES (tools/pm_pixel_phases.py; never the library build())
// adds the clock() cycles lane 0 of every pixel-pass warp spends in each phase to pm_phase_cycles[pruned][phase]; in
// every other build the phase marks are PmNoPhase and compile to nothing.
enum { PM_PH_WAIT, PM_PH_SETUP, PM_PH_SELECT, PM_PH_TAPS, PM_PH_FINAL, PM_PH_BOUND, PM_PH_OTHER, PM_PH_COUNT };
struct PmNoPhase {
  __device__ __forceinline__ void operator()(int) const {}
};
#ifdef PM_PIXEL_PHASES
__device__ unsigned long long pm_phase_cycles[2][PM_PH_COUNT];
// mark(k): the cycles since the previous mark belong to phase k.  State in shared memory, one row per warp.
struct PmPhaseClock {
  unsigned long long* acc;
  unsigned* last;
  __device__ __forceinline__ void operator()(int k) const {
    if ((threadIdx.x & 31) == 0) {
      const unsigned now = (unsigned)clock();
      acc[k] += now - *last;
      *last = now;
    }
  }
};
// pm_pool_counts[pruned][k], the same build only: k = 0 NCCs pm_pixel4_kernel evaluated, 1 its rounds (four group slots
// each), 2 NCCs the serial pass evaluated itself (entries the pixel pass left out)
enum { PM_CNT_P_NCC, PM_CNT_P_ROUNDS, PM_CNT_S_NCC, PM_CNT_COUNT };
__device__ unsigned long long pm_pool_counts[2][PM_CNT_COUNT];
#define PM_POOL_COUNT(var, v) ((var) += (v))
#else
#define PM_POOL_COUNT(var, v) ((void)0)
#endif
// Lane `sub` adds taps sub, sub + 8, ... in ascending order.  The loop is a software pipeline of depth D: the quad words
// of the lane's next D - 1 taps are in flight while a tap is blended, so a warp waits on one gather latency per D taps
// instead of one per tap.  The look-ahead index is clamped to the lane's last tap (the extra loads of the last
// iterations re-read that word and are dropped); a lane without taps fetches slot `sub` of the padded patch, whose
// offsets are finite, and adds nothing.  Depth and unroll per caller, by C2 run time on an H100 80GB HBM3 at 700 W
// (DESIGN.md §2 has the grid): the pixel pass <3, 3> (P 12.65 ms per sweep against 13.43 with the loop it replaced;
// every U = 1 point and D = 4 lost, as did 7 and 6 resident CTAs); the serial pass and the initial cost <1, 5>, where
// ptxas already overlaps the loads of the unrolled copies (S at D = 2 or 3 took 13.4-17.2 ms per sweep against 12.2).
// The patch is read as two float2 arrays, tap t at wr[PS * t] ({w, w * ref}) and off[PS * t] ({dx, dy}): PS = 2 for the
// interleaved float4 patch {w, w * ref, dx, dy} (off = wr + 1), PS = 1 for a split patch with a per-CTA offset table.
template <int D, int UNROLL, int PS, class Phase = PmNoPhase>
__device__ __forceinline__ float pm_ncc_group(const float2* __restrict__ wrp, const float2* __restrict__ offp, int ntaps,
                                              const float* __restrict__ pose,
                                              const float iK[4], const uint32_t* __restrict__ quads, int pitch, int W,
                                              int H, float rowf, float colf, float d, float n0, float n1, float n2,
                                              float inv_wsum, float rsum, float rsq, int sub, unsigned gmask,
                                              Phase phase = Phase()) {
  float Hm[9];
  pm_compose_homography(pose, iK, rowf, colf, d, n0, n1, n2, Hm);
  const uint32_t* quads0 = quads + (2 * pitch + 2);
  asm("" : "+l"(quads0));  // keep the image base as one opaque 64-bit value: the tap address is a single IMAD.WIDE
  const float hi_x = (float)(W + 1), hi_y = (float)(H + 1);
  float s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
  // H (x, y, 1) with (x, y) = (col + dx, row + dy): the pixel part is folded into the constant term once per NCC
  const float cx = fmaf(Hm[0], colf, fmaf(Hm[1], rowf, Hm[2]));
  const float cy = fmaf(Hm[3], colf, fmaf(Hm[4], rowf, Hm[5]));
  const float cz = fmaf(Hm[6], colf, fmaf(Hm[7], rowf, Hm[8]));
  auto fetch = [&](int t) {
    const float2 off = offp[PS * t];
    const float zx = fmaf(Hm[0], off.x, fmaf(Hm[1], off.y, cx));
    const float zy = fmaf(Hm[3], off.x, fmaf(Hm[4], off.y, cy));
    const float zz = fmaf(Hm[6], off.x, fmaf(Hm[7], off.y, cz));
    const float inv_z = pm_rcp_clamped(zz);
    return pm_quad_fetch(quads0, pitch, hi_x, hi_y, inv_z * zx, inv_z * zy);
  };
  auto consume = [&](int t, const PmQuadTap& q) {
    const float color = pm_quad_blend(q);
    const float2 wr = wrp[PS * t];
    const float ws = wr.x * color;
    s1 += ws;
    s2 = fmaf(ws, color, s2);
    s3 = fmaf(wr.y, color, s3);
  };
  phase(PM_PH_FINAL);   // the homography counts with the finalize: both are paid once per NCC
  const int cnt = (ntaps >> 3) + ((sub < (ntaps & 7)) ? 1 : 0);
  const int last = sub + 8 * (cnt > 0 ? cnt - 1 : 0);
  PmQuadTap st[D];
#pragma unroll
  for (int k = 0; k < D - 1; ++k) st[k] = fetch(min(sub + 8 * k, last));
#pragma unroll UNROLL
  for (int j = 0; j < cnt; ++j) {
    const int t = sub + 8 * j;
    st[D - 1] = fetch(min(t + 8 * (D - 1), last));
    consume(t, st[0]);
#pragma unroll
    for (int k = 0; k < D - 1; ++k) st[k] = st[k + 1];
  }
  phase(PM_PH_TAPS);
#pragma unroll
  for (int o = 1; o < 8; o <<= 1) {
    s1 = s1 + __shfl_xor_sync(gmask, s1, o);
    s2 = s2 + __shfl_xor_sync(gmask, s2, o);
    s3 = s3 + __shfl_xor_sync(gmask, s3, o);
  }
  const float ncc = pm_ncc_finalize(s1, s2, s3, inv_wsum, rsum, rsq);
  phase(PM_PH_FINAL);
  return ncc;
}


// TransformPDFToCDF (:683-696) over the per-image lanes: sum in image order, then the running sum of prob / sum.
// For N <= 8 the N values are fetched once and both passes run on registers (lanes >= N hold prob = 0: adding +0.0
// changes nothing, so the loops can run over all 8 slots); same operations in the same order as the plain loops.
// width 8 (N <= 8 only): each 8-lane segment is one pixel, `lane` is the lane within the segment.
__device__ __forceinline__ float pm_cdf_lanes(float prob, int N, int lane, int width = 32) {
  const unsigned full = 0xffffffffu;
  float cdf = 0.0f;
  if (N <= 8) {
    float pv[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) pv[i] = __shfl_sync(full, prob, i, width);
    float sum = 0.0f;
#pragma unroll
    for (int i = 0; i < 8; ++i) sum += pv[i];
    const float inv = 1.0f / sum;
    float cum = 0.0f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i < N) { cum += pv[i] * inv; if (lane == i) cdf = cum; }
    }
  } else {
    float sum = 0.0f;
    for (int i = 0; i < N; ++i) sum += __shfl_sync(full, prob, i);
    const float inv = 1.0f / sum;
    float cum = 0.0f;
    for (int i = 0; i < N; ++i) {
      cum += __shfl_sync(full, prob, i) * inv;
      if (lane == i) cdf = cum;
    }
  }
  return cdf;
}
// index of the first image whose CDF value exceeds u (-1: none), per lane; width as in pm_cdf_lanes
__device__ __forceinline__ int pm_sample_image(float cdf, float u, int N, int width = 32) {
  const unsigned full = 0xffffffffu;
  int img = -1;
  if (N <= 8) {
#pragma unroll
    for (int i = 7; i >= 0; --i) {
      const float ci = __shfl_sync(full, cdf, i, width);
      if (i < N && ci > u) img = i;     // descending i: the smallest qualifying index wins
    }
  } else {
    for (int i = 0; i < N; ++i) {
      const float ci = __shfl_sync(full, cdf, i);
      if (img < 0 && ci > u) img = i;
    }
  }
  return img;
}

// reference patch of one pixel: bilateral weights + weighted colours + 1/sum(w); executed by one warp.  Patch layout as in
// pm_ncc_group.
template <int PS>
__device__ __forceinline__ void pm_build_patch(const PmParams& P, const float* lut, int rot, int fw, int fh, int row, int col,
                                               const float2* off, float2* wr, int lane, float* inv_wsum_out) {
  const float center = pm_ref_color(P, lut, rot, fw, fh, row, col);
  float partial = 0.0f;
  for (int t = lane; t < P.ntaps; t += 32) {
    const float2 o = off[PS * t];
    const int dc = (int)o.x, dr = (int)o.y;
    const float c = pm_ref_color(P, lut, rot, fw, fh, row + dr, col + dc);
    const float bw = pm_bilateral_weight(P.spatial_norm, P.color_norm, dr, dc, center, c);
    wr[PS * t] = make_float2(bw, bw * c);
    partial += bw;
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) partial = partial + __shfl_xor_sync(0xffffffffu, partial, o);
  *inv_wsum_out = 1.0f / partial;
}

__device__ __forceinline__ void pm_fill_tap_offsets(const PmParams& P, float4* patch, int tid, int nthreads) {
  for (int t = tid; t < P.ntaps_pad; t += nthreads) {
    const int tr = t / P.nside, tc = t - tr * P.nside;
    patch[t] = make_float4(0.0f, 0.0f, (float)(-P.radius + P.step * tc), (float)(-P.radius + P.step * tr));
  }
}
// per CTA: tsrc[t] = index in a stored pixel block of the tap in slot t of frame `rot`'s patch
__device__ __forceinline__ void pm_fill_tap_src(const PmParams& P, int rot, int* tsrc, int tid, int nthreads) {
  for (int t = tid; t < P.ntaps; t += nthreads) tsrc[t] = pm_orig_tap(rot, P.nside, t);
}

// Reference patches of every pixel, once per run, for the patch store: the {w, w * ref} pairs of all taps in the
// original orientation, and 1 / sum(w) for each of the four sweep frames.  Frame k's tap (dr, dc) reads the original tap
// at the rotated offset (pm_orig_tap), whose weight and colour have the same bits (the weight depends on dr^2 + dc^2 and
// the colour difference only).  The weight sum is a rounded fp32 sum, so it is formed per frame in that frame's tap order
// with pm_build_patch's lane split and shfl.xor tree: every consumer gets exactly what its inline build would compute.
__global__ void __launch_bounds__(128) pm_patch_kernel(const PmParams P) {
  extern __shared__ float smemf[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* lut = smemf;
  int2* toff = reinterpret_cast<int2*>(smemf + 256);                  // (dr, dc) of original tap t
  int* tmap = reinterpret_cast<int*>(toff + P.ntaps_pad);              // [3][ntaps_pad] pm_orig_tap of frames 1..3
  float* wt = reinterpret_cast<float*>(tmap + 3 * P.ntaps_pad) + warp * P.ntaps_pad;   // this warp's pixel: tap weights
  pm_load_lut(lut, threadIdx.x, blockDim.x);
  for (int t = threadIdx.x; t < P.ntaps; t += blockDim.x) {
    const int tr = t / P.nside, tc = t - tr * P.nside;
    toff[t] = make_int2(-P.radius + P.step * tr, -P.radius + P.step * tc);
    for (int k = 1; k < 4; ++k) tmap[(k - 1) * P.ntaps_pad + t] = pm_orig_tap(k, P.nside, t);
  }
  __syncthreads();
  const int npix = P.W0 * P.H0;
  for (int p = blockIdx.x * 4 + warp; p < npix; p += gridDim.x * 4) {
    const int row = p / P.W0, col = p - row * P.W0;
    const float center = pm_ref_color(P, lut, 0, P.W0, P.H0, row, col);
    float2* blk = P.patch_store + (size_t)p * P.ntaps_st;
    float partial0 = 0.0f;
    for (int t = lane; t < P.ntaps; t += 32) {
      const int2 o = toff[t];
      const float c = pm_ref_color(P, lut, 0, P.W0, P.H0, row + o.x, col + o.y);
      const float bw = pm_bilateral_weight(P.spatial_norm, P.color_norm, o.x, o.y, center, c);
      blk[t] = make_float2(bw, bw * c);
      wt[t] = bw;
      partial0 += bw;   // frame 0: the stored order is its tap order
    }
    __syncwarp();
    float partial1 = 0.0f, partial2 = 0.0f, partial3 = 0.0f;
    for (int t = lane; t < P.ntaps; t += 32) {
      partial1 += wt[tmap[t]];
      partial2 += wt[tmap[P.ntaps_pad + t]];
      partial3 += wt[tmap[2 * P.ntaps_pad + t]];
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      partial0 = partial0 + __shfl_xor_sync(0xffffffffu, partial0, o);
      partial1 = partial1 + __shfl_xor_sync(0xffffffffu, partial1, o);
      partial2 = partial2 + __shfl_xor_sync(0xffffffffu, partial2, o);
      partial3 = partial3 + __shfl_xor_sync(0xffffffffu, partial3, o);
    }
    const float inv[4] = {1.0f / partial0, 1.0f / partial1, 1.0f / partial2, 1.0f / partial3};
    if (lane < 4) P.patch_inv[(size_t)p * 4 + lane] = (lane == 0) ? inv[0] : ((lane == 1) ? inv[1] : ((lane == 2) ? inv[2] : inv[3]));
    __syncwarp();
  }
}

// Copy of pixel p's stored block into patch[t].xy in frame order (tsrc from pm_fill_tap_src): one 8-byte cp.async per
// tap, so the copy is in flight while the issuing warp does other work.  The taps of a frame are a permutation of the
// stored order, so every lane writes its own slot; the 121 x 8 B a warp reads are one contiguous block.
// the two halves of an interleaved patch entry {w, w * ref, dx, dy}
__device__ __forceinline__ float2* pm_wr(float4* patch) { return reinterpret_cast<float2*>(patch); }
__device__ __forceinline__ const float2* pm_off(const float4* patch) { return reinterpret_cast<const float2*>(patch) + 1; }
template <int PS>
__device__ __forceinline__ void pm_copy_patch(const PmParams& P, const int* tsrc, size_t p, float2* wr, int lane) {
  const float2* blk = P.patch_store + p * P.ntaps_st;
  for (int t = lane; t < P.ntaps; t += 32) {
    const unsigned dst = (unsigned)__cvta_generic_to_shared(&wr[PS * t]);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(dst), "l"(blk + tsrc[t]) : "memory");
  }
}
__device__ __forceinline__ void pm_copy_scalar(float* dst_smem, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst_smem)), "l"(src)
               : "memory");
}
// this thread's copies have landed (other threads see them after the next barrier)
__device__ __forceinline__ void pm_copy_wait() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

// ComputeInitialCost (patch_match_cuda.cu:863-912), pixel-parallel: one warp per pixel.
__global__ void __launch_bounds__(128) pm_initial_cost_kernel(const PmParams P) {
  extern __shared__ float4 smem4[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int N = P.N;
  float* poses = reinterpret_cast<float*>(smem4 + 4 * P.ntaps_pad);
  int* tsrc = reinterpret_cast<int*>(poses + N * PM_POSE_STRIDE);
  float* lut = reinterpret_cast<float*>(tsrc + P.ntaps_pad);
  float4* patch = smem4 + warp * P.ntaps_pad;
  for (int i = threadIdx.x; i < N * PM_POSE_STRIDE; i += blockDim.x) poses[i] = P.poses[i];
  pm_fill_tap_offsets(P, patch, lane, 32);
  pm_fill_tap_src(P, 0, tsrc, threadIdx.x, blockDim.x);
  pm_load_lut(lut, threadIdx.x, blockDim.x);
  __syncthreads();
  const size_t npix = (size_t)P.W0 * P.H0;
  const int g = lane >> 3, sub = lane & 7;
  const unsigned gmask = 0xffu << (8 * g);
  for (size_t p = (size_t)blockIdx.x * 4 + warp; p < npix; p += (size_t)gridDim.x * 4) {
    const int row = (int)(p / P.W0), col = (int)(p - (size_t)row * P.W0);
    float inv_wsum;
    if (P.patch_store) {
      pm_copy_patch<2>(P, tsrc, p, pm_wr(patch), lane);
      inv_wsum = P.patch_inv[p * 4];
      pm_copy_wait();
    } else {
      pm_build_patch<2>(P, lut, 0, P.W0, P.H0, row, col, pm_off(patch), pm_wr(patch), lane, &inv_wsum);
    }
    __syncwarp();
    const float4 hy = P.hyp[p];
    const float rsum = P.ref_sum[p], rsq = P.ref_sqsum[p];
    for (int base = 0; base < N; base += 4) {
      const int img = base + g;
      if (img < N) {
        const PmSrcDesc sd = P.src[img];
        const float c = pm_ncc_group<1, 5, 2>(pm_wr(patch), pm_off(patch), P.ntaps, poses + img * PM_POSE_STRIDE, P.invK[0], P.quads + sd.quad_off,
                                     sd.pitch, sd.w, sd.h, (float)row, (float)col, hy.x, hy.y, hy.z, hy.w, inv_wsum,
                                     rsum, rsq, sub, gmask);
        if (sub == 0) P.cost[p * N + img] = c;
      }
    }
    __syncwarp();
  }
}

// ================================================================================================
// Sweep: SweepFromTopToBottom (patch_match_cuda.cu:933-1288) in four passes.
//   R  pm_rand_kernel    one warp per column: consumes the column's XORWOW stream to produce every row's
//                        random hypothesis and Monte-Carlo uniforms (the stream position of a row does not
//                        depend on the sweep's results, only on the hypotheses of the previous sweep);
//   M  pm_msg_kernel     one thread per (column, image), beside R: the column's HMM messages over the
//                        costs the sweep starts with;
//   P  pm_pixel_kernel   pixel-parallel, one warp per pixel (pm_pixel4_kernel for N <= 8: four pixels per warp,
//                        their NCC rounds pooled): everything that does not depend on the row
//                        above — the NCC of hypotheses 2..4 (rand/rand, cur/rand-normal, rand-depth/cur)
//                        against every source image, the per-image priors, geometric costs;
//   S  pm_serial_kernel  one CTA per column: propagation, HMM messages, Monte-Carlo sampling, the NCC
//                        of the propagated hypothesis, argmin, filter.
// ================================================================================================
// pixel-index step from row r to row r + 1 of frame `rot` (the row stride of pm_pix0)
__device__ __forceinline__ int pm_row_stride(int W0, int rot) {
  return (rot == 0) ? W0 : ((rot == 1) ? -1 : ((rot == 2) ? -W0 : 1));
}

// R  pm_rand_kernel: one warp per PM_RAND_CPW columns.  A row takes 1 + 3 * rounds + num_samples draws from the
// column's stream, and only `rounds` (PerturbNormal's trials) depends on anything but the stream; that is the only
// serial part of the pass.  Per block of 32 rows, lane j < PM_RAND_CPW walks column j's stream alone and leaves every
// row's start state in a shared ring; then lane k restarts from row k's state, column by column, and computes that row
// with the same functions and draws as a column-serial loop (pm_rand_column_host).  On the tall frames the rows of a
// column are adjacent pixels, so the 32 lanes' stores are one contiguous run.
// The walk keeps no results.  A trial's draws are the same whether it is accepted or not, so the walk advances a copy
// of the stream past the row's sample draws while the trial's acceptance test is computed, and keeps that copy when the
// trial ends the row; with NS = num_samples known at compile time the two are one straight block the scheduler
// interleaves (NS = 0: num_samples read at run time, for the configurations other than the default 15).
#define PM_RAND_WARPS 2   // warps per CTA
#define PM_RAND_CPW 4     // columns per warp
template <int NS>
__global__ void __launch_bounds__(32 * PM_RAND_WARPS) pm_rand_kernel(const PmParams P, const PmSweepArgs A) {
  constexpr int CPW = PM_RAND_CPW;
  __shared__ uint32_t ring[PM_RAND_WARPS][CPW][6][32];   // [column][state word][row of the block]
  __shared__ float4 hyr[PM_RAND_WARPS][CPW][32];         // the block's current hypotheses, for the walks' trials
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rot = A.rot;
  const int fw = (rot & 1) ? P.H0 : P.W0, fh = (rot & 1) ? P.W0 : P.H0;
  const int col0 = (blockIdx.x * PM_RAND_WARPS + warp) * CPW;
  if (col0 >= fw) return;
  const int ncols = min(CPW, fw - col0);
  const float iK[4] = {P.invK[rot][0], P.invK[rot][1], P.invK[rot][2], P.invK[rot][3]};
  const int ns = NS ? NS : P.num_samples;
  const bool walker = lane < ncols;
  const int wcol = col0 + (walker ? lane : 0);   // the column lane `lane` walks
  int r0, c0;
  pm_frame_to_orig(P.W0, P.H0, rot, 0, wcol, &r0, &c0);
  uint32_t* slot = P.rng + 6 * (size_t)pm_border_index(P.W0, P.H0, r0, c0);
  PmRng rs;
  if (walker) { rs.v0 = slot[0]; rs.v1 = slot[1]; rs.v2 = slot[2]; rs.v3 = slot[3]; rs.v4 = slot[4]; rs.d = slot[5]; }
  const long long rstep = pm_row_stride(P.W0, rot);
  const long long cstep = (long long)pm_pix0(P.W0, P.H0, rot, 0, 1) - (long long)pm_pix0(P.W0, P.H0, rot, 0, 0);
  const size_t p_top = pm_pix0(P.W0, P.H0, rot, 0, col0);   // column col0 + j, row r: p_top + j * cstep + r * rstep
  float4 nx[CPW];
#pragma unroll
  for (int j = 0; j < CPW; ++j)
    nx[j] = (j < ncols && lane < fh) ? P.hyp[p_top + j * cstep + lane * rstep] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  for (int base = 0; base < fh; base += 32) {
    const int row = base + lane;
    float4 cur[CPW];
#pragma unroll
    for (int j = 0; j < CPW; ++j) {
      cur[j] = nx[j];
      if (j < ncols && row + 32 < fh) nx[j] = P.hyp[p_top + j * cstep + (row + 32) * rstep];   // next block's, in flight
      hyr[warp][j][lane] = cur[j];
    }
    __syncwarp();
    if (walker) {
      const int nrows = min(32, fh - base);
      const float colf = (float)wcol;
      const float rx = fmaf(iK[0], colf, iK[1]);   // pm_perturb_normal's viewing ray
      for (int k = 0; k < nrows; ++k) {
        ring[warp][lane][0][k] = rs.v0; ring[warp][lane][1][k] = rs.v1; ring[warp][lane][2][k] = rs.v2;
        ring[warp][lane][3][k] = rs.v3; ring[warp][lane][4][k] = rs.v4; ring[warp][lane][5][k] = rs.d;
        const float4 h = hyr[warp][lane][k];
        float n0 = h.y, n1 = h.z;
        pm_normal_to_frame(rot, n0, n1);
        const float ry = fmaf(iK[2], (float)(base + k), iK[3]);
        pm_rng_next(rs);   // the random depth
        float perturbation = A.perturbation_pi;
        for (int trial = 0;; ++trial) {
          const float u1 = pm_rng_uniform(rs);
          const float u2 = pm_rng_uniform(rs);
          const float u3 = pm_rng_uniform(rs);
          PmRng after = rs;   // the stream past the row's sample draws, if this trial ends the row
          if (NS) {
#pragma unroll
            for (int s = 0; s < NS; ++s) pm_rng_next(after);
          } else {
            for (int s = 0; s < ns; ++s) pm_rng_next(after);
          }
          float out[3];
          if (pm_perturb_trial(rx, ry, perturbation, u1, u2, u3, n0, n1, h.w, out) || trial == 3) { rs = after; break; }
          perturbation = 0.5f * perturbation;
        }
      }
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < CPW; ++j) {
      if (j < ncols && row < fh) {
        PmRng rk;
        rk.v0 = ring[warp][j][0][lane]; rk.v1 = ring[warp][j][1][lane]; rk.v2 = ring[warp][j][2][lane];
        rk.v3 = ring[warp][j][3][lane]; rk.v4 = ring[warp][j][4][lane]; rk.d = ring[warp][j][5][lane];
        const float4 c4 = cur[j];
        float n0 = c4.y, n1 = c4.z;
        pm_normal_to_frame(rot, n0, n1);
        const float dmin = (1.0f - A.perturbation) * c4.x;
        const float dmax = (1.0f + A.perturbation) * c4.x;
        const float rand_d = fmaf(pm_rng_uniform(rk), dmax - dmin, dmin);
        float rn[3];
        pm_perturb_normal(iK, (float)row, (float)(col0 + j), A.perturbation_pi, n0, n1, c4.w, rk, rn);
        const size_t p = p_top + j * cstep + row * rstep;
        A.rand_hyp[p] = make_float4(rand_d, rn[0], rn[1], rn[2]);
        for (int s = 0; s < ns; ++s) A.usamp[p * ns + s] = pm_rng_uniform(rk) - FLT_EPSILON;
      }
    }
    // (the next block's first __syncwarp orders this block's ring and hyr reads before their next writes)
  }
  if (walker) { slot[0] = rs.v0; slot[1] = rs.v1; slot[2] = rs.v2; slot[3] = rs.v3; slot[4] = rs.v4; slot[5] = rs.d; }
}

// M  pm_msg_kernel: one thread per (column, image).  Backward messages of the whole column (:976-989) - the same
// recurrence pm_serial_kernel used to run at its start, now available BEFORE the pixel pass - and the forward
// messages over the sweep-start costs ("nothing above this row changes"), which is what the serial pass will see
// wherever no new hypothesis won above.  From them the pixel pass predicts the Monte-Carlo samples of every pixel.
// The two recurrences are independent and run interleaved, step k of both together (backward at row fh - 1 - k,
// forward at row k).  A step's likelihood pm_ncc_prob(cost) does not depend on the message, so it is computed off the
// chains, and the costs are read a chunk of PM_MSG_CHUNK rows ahead: the next chunk's loads are in flight while a chunk
// is consumed.  Per step the messages are the same operations in the same order as pm_msg_column_host.
#define PM_MSG_CHUNK 16
#define PM_MSG_THREADS 64
__global__ void __launch_bounds__(PM_MSG_THREADS) pm_msg_kernel(const PmParams P, const PmSweepArgs A) {
  const int rot = A.rot, N = P.N;
  const int fw = (rot & 1) ? P.H0 : P.W0, fh = (rot & 1) ? P.W0 : P.H0;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int col = t / N, img = t - col * N;
  if (col >= fw) return;
  const bool fwd = A.fwd_pred != nullptr;
  // value (row, img) of a [pixel][N] map is at top + row * rstep
  const size_t top = pm_pix0(P.W0, P.H0, rot, 0, col) * N + img;
  const long long rstep = (long long)pm_row_stride(P.W0, rot) * N;
  const float* cost = P.cost + top;
  constexpr int C = PM_MSG_CHUNK;
  float cb[C], cf[C];   // the chunk's costs: backward rows fh - 1 - k, forward rows k
  auto load = [&](int k0, float* b, float* f) {
#pragma unroll
    for (int j = 0; j < C; ++j) {
      const int k = k0 + j;
      b[j] = (k < fh) ? cost[(fh - 1 - k) * rstep] : 0.0f;
      f[j] = (fwd && k < fh) ? cost[k * rstep] : 0.0f;
    }
  };
  load(0, cb, cf);
  float beta = 0.5f, f = 0.5f;
  for (int k0 = 0; k0 < fh; k0 += C) {
    float eb[C], ef[C];
#pragma unroll
    for (int j = 0; j < C; ++j) { eb[j] = pm_ncc_prob(P.L, cb[j]); ef[j] = pm_ncc_prob(P.L, cf[j]); }
    load(k0 + C, cb, cf);
#pragma unroll
    for (int j = 0; j < C; ++j) {
      const int k = k0 + j;
      if (k >= fh) break;
      beta = pm_backward_message_e(eb[j], beta);
      A.sel_cur[top + (fh - 1 - k) * rstep] = beta;
      if (fwd) {
        f = pm_forward_message_e(ef[j], f);
        A.fwd_pred[top + k * rstep] = f;
      }
    }
  }
}

// P  pm_pixel_kernel.  With A.prune == 1 the pass does not evaluate all 3N (hypothesis, image) pairs of a pixel:
//   * it PREDICTS the Monte-Carlo samples of the pixel (the uniforms are known from pass R, the CDF from the
//     sweep-start messages of pass M) and from them how often every image will be sampled;
//   * per hypothesis it evaluates the sampled images in order of multiplicity and stops as soon as the partial cost
//     sum exceeds the (predicted) cost sum of the current hypothesis: a sum of non-negative terms only grows, so
//     that hypothesis can no longer win the argmin (:1175-1182);
//   * entries it did not evaluate stay PM_NOT_EVALUATED.
// Exactness does not depend on the prediction: pm_serial_kernel re-checks "partial sum > cost sum of hypothesis 0"
// with the true samples in the true summation order and evaluates any entry it really needs itself.
template <bool GEOM, bool PRUNE>
__global__ void __launch_bounds__(128, 8) pm_pixel_kernel(const PmParams P, const PmSweepArgs A) {
  extern __shared__ float4 smem4[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rot = A.rot, N = P.N;
  const int fw = (rot & 1) ? P.H0 : P.W0, fh = (rot & 1) ? P.W0 : P.H0;
  float* poses = reinterpret_cast<float*>(smem4 + 4 * P.ntaps_pad);
  int* tsrc = reinterpret_cast<int*>(poses + N * PM_POSE_STRIDE);
  float* lut = reinterpret_cast<float*>(tsrc + P.ntaps_pad);
  float4* patch = smem4 + warp * P.ntaps_pad;
  for (int i = threadIdx.x; i < N * PM_POSE_STRIDE; i += blockDim.x) poses[i] = P.poses[(size_t)rot * N * PM_POSE_STRIDE + i];
  pm_fill_tap_offsets(P, patch, lane, 32);
  pm_fill_tap_src(P, rot, tsrc, threadIdx.x, blockDim.x);
  pm_load_lut(lut, threadIdx.x, blockDim.x);
  const float iK[4] = {P.invK[rot][0], P.invK[rot][1], P.invK[rot][2], P.invK[rot][3]};
  const float Kr[4] = {P.K[rot][0], P.K[rot][1], P.K[rot][2], P.K[rot][3]};
  __syncthreads();
  const size_t npix = (size_t)fw * fh;
  const int g = lane >> 3, sub = lane & 7;
  const unsigned gmask = 0xffu << (8 * g);
  const unsigned full = 0xffffffffu;
  const unsigned nmask = (N >= 32) ? 0xffffffffu : ((1u << N) - 1u);
  const int ns = P.num_samples, nsl = ns < 32 ? ns : 32;
  const int mode = PRUNE ? A.prune : 0;
  (void)fw; (void)nsl; (void)full; (void)nmask;
#ifdef PM_PIXEL_PHASES
  __shared__ unsigned long long ph_acc[4][PM_PH_COUNT];
  __shared__ unsigned ph_last[4];
  if (lane == 0) {
    for (int k = 0; k < PM_PH_COUNT; ++k) ph_acc[warp][k] = 0ull;
    ph_last[warp] = (unsigned)clock();
  }
  __syncwarp();
  const PmPhaseClock ph{ph_acc[warp], &ph_last[warp]};
#else
  const PmNoPhase ph;
#endif
  // (an SM-local tiling of the pixel order was measured: L1 hit rate 67% -> 55%, slower; plain grid stride kept)
  for (size_t q = (size_t)blockIdx.x * 4 + warp; q < npix; q += (size_t)gridDim.x * 4) {
    const int row = (int)(q / fw), col = (int)(q - (size_t)row * fw);  // sweep-frame pixel
    const size_t p = pm_pix0(P.W0, P.H0, rot, row, col);
    const float rowf = (float)row, colf = (float)col;
    float inv_wsum;
    if (P.patch_store) {   // in flight while the pixel's inputs load and its priors are computed
      pm_copy_patch<2>(P, tsrc, p, pm_wr(patch), lane);
      inv_wsum = P.patch_inv[p * 4 + rot];
    } else {
      pm_build_patch<2>(P, lut, rot, fw, fh, row, col, pm_off(patch), pm_wr(patch), lane, &inv_wsum);
    }
    ph(PM_PH_OTHER);
    const float4 cur4 = P.hyp[p];
    float cn0 = cur4.y, cn1 = cur4.z;
    pm_normal_to_frame(rot, cn0, cn1);
    const float cur_d = cur4.x, cn2 = cur4.w;
    const float4 r4 = A.rand_hyp[p];
    const float rsum = P.ref_sum[p], rsq = P.ref_sqsum[p];
    float prob = 0.0f, cost_i = 0.0f, gcur = 0.0f, grand = 0.0f;
    if (lane < N) {  // per-image priors of the current hypothesis (:1079-1103)
      const float* pose = poses + lane * PM_POSE_STRIDE;
      const float rx = fmaf(iK[0], colf, iK[1]), ry = fmaf(iK[2], rowf, iK[3]);
      float ct, ci;
      pm_viewing_angles(pose, cur_d * rx, cur_d * ry, cur_d, cn0, cn1, cn2, &ct, &ci);
      float Hm[9];
      pm_compose_homography(pose, iK, rowf, colf, cur_d, cn0, cn1, cn2, Hm);
      // kept as three factors: the serial pass evaluates sel_prob * tri * inc * res left to right (:1103)
      const float pt = pm_tri_prob(P.L, ct), pi = pm_inc_prob(P.L, ci), pr = pm_res_prob(Hm, rowf, colf, P.radius);
      A.prior3[(p * 3 + 0) * N + lane] = pt;
      A.prior3[(p * 3 + 1) * N + lane] = pi;
      A.prior3[(p * 3 + 2) * N + lane] = pr;
      if (GEOM) {
        const PmSrcDesc sd = P.src[lane];
        const float* dm = P.src_depth + sd.depth_off;
        gcur = pm_geom_cost(pose, Kr, iK, dm, sd.w, sd.h, rowf, colf, cur_d, P.geom_max_cost);
        grand = pm_geom_cost(pose, Kr, iK, dm, sd.w, sd.h, rowf, colf, r4.x, P.geom_max_cost);
        A.gtab2[(p * 2 + 0) * N + lane] = gcur;
        A.gtab2[(p * 2 + 1) * N + lane] = grand;
      }
      if (mode == 1) {
        cost_i = P.cost[p * N + lane];
        const float sp = pm_sel_prob(A.fwd_pred[p * N + lane], A.sel_cur[p * N + lane], A.sel_prev[p * N + lane], A.prev_w);
        prob = sp * pt * pi * pr;
      }
    }
    ph(PM_PH_SETUP);
    pm_copy_wait();
    ph(PM_PH_WAIT);
    if (!PRUNE) {   // every (hypothesis, image) pair, four per round
      __syncwarp();
      const int npairs = 3 * N;
      for (int base = 0; base < npairs; base += 4) {
        const int pair = base + g;
        if (pair < npairs) {
          const int hsel = pair / N, img = pair - hsel * N;
          const float hd = (hsel == 1) ? cur_d : r4.x;
          const float hn0 = (hsel == 2) ? cn0 : r4.y, hn1 = (hsel == 2) ? cn1 : r4.z, hn2 = (hsel == 2) ? cn2 : r4.w;
          const PmSrcDesc sd = P.src[img];
          ph(PM_PH_SELECT);
          const float c = pm_ncc_group<3, 3, 2>(pm_wr(patch), pm_off(patch), P.ntaps, poses + img * PM_POSE_STRIDE, iK, P.quads + sd.quad_off, sd.pitch,
                                       sd.w, sd.h, rowf, colf, hd, hn0, hn1, hn2, inv_wsum, rsum, rsq, sub, gmask, ph);
          if (sub == 0) A.tab3[(p * 3 + hsel) * N + img] = c;
          ph(PM_PH_FINAL);
        }
      }
      __syncwarp();
      continue;
    }
    for (int e = lane; e < 3 * N; e += 32) A.tab3[p * 3 * N + e] = PM_NOT_EVALUATED;
    __syncwarp();   // patch complete; sentinel stores ordered before the result stores of other lanes
    // ---- which images will be sampled, and how often (prediction; mode 0: every image once)
    int mult = (lane < N) ? 1 : 0;
    unsigned rem0 = nmask, rem1 = nmask, rem2 = nmask, ev0 = 0u, ev1 = 0u, ev2 = 0u;
    bool act0 = true, act1 = true, act2 = true, ext0 = true, ext1 = true, ext2 = true;
    float thr = 3.0e38f;
    if (mode == 1) {
      const float cdf = pm_cdf_lanes(prob, N, lane);
      const float u = (lane < nsl) ? A.usamp[p * ns + lane] : 2.0f;
      const int img = pm_sample_image(cdf, u, N);
      mult = 0;
      for (int s2 = 0; s2 < nsl; ++s2) mult += (__shfl_sync(full, img, s2) == lane) ? 1 : 0;
      if (lane >= N) mult = 0;
      const unsigned needed = __ballot_sync(full, mult > 0);
      float t = (float)mult * (GEOM ? fmaf(P.geom_reg, gcur, cost_i) : cost_i);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(full, t, o);
      thr = fmaf(t, 1.001f, 1e-3f);   // predicted cost sum of the current hypothesis, with a margin for the true order of summation
      rem0 = rem1 = rem2 = needed;
      ext0 = ext1 = ext2 = false;
      act0 = act1 = act2 = needed != 0u;
    } else if (mode != 0) {
      act0 = act1 = act2 = false;
    }
    ph(PM_PH_SETUP);
    float L0 = 0.0f, L1 = 0.0f, L2 = 0.0f;
    while (act0 || act1 || act2) {
      // up to four (hypothesis, image) pairs per round, hypotheses taking turns, images by multiplicity
      int my_k = -1, my_img = 0, slot = 0;
#pragma unroll
      for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const bool a = (k == 0) ? act0 : ((k == 1) ? act1 : act2);
          const unsigned rem = (k == 0) ? rem0 : ((k == 1) ? rem1 : rem2);
          if (slot < 4 && a && rem) {
            const unsigned key = ((rem >> lane) & 1u) ? ((((unsigned)mult) << 5) | (unsigned)(31 - lane)) + 1u : 0u;
            const unsigned best = __reduce_max_sync(full, key);
            const int im = 31 - (int)((best - 1u) & 31u);
            const unsigned bit = 1u << im;
            if (k == 0) { rem0 &= ~bit; ev0 |= bit; } else if (k == 1) { rem1 &= ~bit; ev1 |= bit; } else { rem2 &= ~bit; ev2 |= bit; }
            if (slot == g) { my_k = k; my_img = im; }
            ++slot;
          }
        }
      }
      ph(PM_PH_SELECT);
      if (slot == 0) break;
      float c = 0.0f;
      if (my_k >= 0) {   // hsel 0: rand/rand, 1: cur depth + rand normal, 2: rand depth + cur normal
        const float hd = (my_k == 1) ? cur_d : r4.x;
        const float hn0 = (my_k == 2) ? cn0 : r4.y, hn1 = (my_k == 2) ? cn1 : r4.z, hn2 = (my_k == 2) ? cn2 : r4.w;
        const PmSrcDesc sd = P.src[my_img];
        c = pm_ncc_group<3, 3, 2>(pm_wr(patch), pm_off(patch), P.ntaps, poses + my_img * PM_POSE_STRIDE, iK, P.quads + sd.quad_off, sd.pitch, sd.w, sd.h,
                         rowf, colf, hd, hn0, hn1, hn2, inv_wsum, rsum, rsq, sub, gmask, ph);
        if (sub == 0) A.tab3[(p * 3 + my_k) * N + my_img] = c;
        ph(PM_PH_FINAL);
      }
      if (mode == 1) {
#pragma unroll
        for (int s2 = 0; s2 < 4; ++s2) {
          const int ks = __shfl_sync(full, my_k, 8 * s2), is = __shfl_sync(full, my_img, 8 * s2);
          float v = __shfl_sync(full, c, 8 * s2);
          const float w = (float)__shfl_sync(full, mult, is & 31);
          if (GEOM) v = fmaf(P.geom_reg, __shfl_sync(full, (ks == 1) ? gcur : grand, is & 31), v);
          if (ks == 0) L0 = fmaf(w, v, L0); else if (ks == 1) L1 = fmaf(w, v, L1); else if (ks == 2) L2 = fmaf(w, v, L2);
        }
        // a hypothesis whose partial sum already exceeds the current hypothesis' sum is out; one that survives all its
        // sampled images is a likely winner: the images nobody sampled are then needed for the cost map (:1184-1196)
        if (act0) { if (L0 > thr) act0 = false; else if (!rem0) { if (!ext0) { ext0 = true; rem0 = nmask & ~ev0; } if (!rem0) act0 = false; } }
        if (act1) { if (L1 > thr) act1 = false; else if (!rem1) { if (!ext1) { ext1 = true; rem1 = nmask & ~ev1; } if (!rem1) act1 = false; } }
        if (act2) { if (L2 > thr) act2 = false; else if (!rem2) { if (!ext2) { ext2 = true; rem2 = nmask & ~ev2; } if (!rem2) act2 = false; } }
      } else {
        act0 = rem0 != 0u; act1 = rem1 != 0u; act2 = rem2 != 0u;
      }
      ph(PM_PH_BOUND);
    }
    __syncwarp();
  }
#ifdef PM_PIXEL_PHASES
  if (lane == 0)
    for (int k = 0; k < PM_PH_COUNT; ++k) atomicAdd(&pm_phase_cycles[PRUNE ? 1 : 0][k], ph_acc[warp][k]);
#endif
}

// P for N <= 8: a warp takes a batch of four consecutive pixels (by index in the sweep frame, so a batch may run over
// a row end) and lane (g, sub) = (lane >> 3, lane & 7) does the set-up of pixel g against image sub: the priors,
// the geometric costs, the selection probability, the CDF and the sample prediction of all four pixels at once (the
// kernel above runs them on N of 32 lanes, once per pixel).  The same functions on the same values, so prior3 / gtab2
// hold the same bits.  The NCC rounds are pooled over the batch: a round's four group slots take pairs of any of the
// four pixels, one per pixel and pass, and after each round every pixel applies the early-out rules of the kernel above
// to its own results.  Which entries the pass fills changes, never their values.  Shared memory: the four reference
// patches of a warp as {w, w * ref} (8 B per tap and pixel) and one {dx, dy} table per CTA:
// 8 * 17 * ntaps_pad + 4 * (43 N + ntaps_pad + 256) bytes, 20.3 KB at C2 (window 11, N = 8), so 8 CTAs still fit an SM.
template <bool GEOM, bool PRUNE>
__global__ void __launch_bounds__(128, 8) pm_pixel4_kernel(const PmParams P, const PmSweepArgs A) {
  extern __shared__ float4 smem4[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rot = A.rot, N = P.N, tp = P.ntaps_pad;
  const int fw = (rot & 1) ? P.H0 : P.W0, fh = (rot & 1) ? P.W0 : P.H0;
  float2* wr_warp = reinterpret_cast<float2*>(smem4) + (size_t)warp * 4 * tp;   // [4 pixels][ntaps_pad] {w, w * ref}
  float2* off = reinterpret_cast<float2*>(smem4) + 16 * tp;                     // [ntaps_pad] {dx, dy}
  float* poses = reinterpret_cast<float*>(off + tp);
  int* tsrc = reinterpret_cast<int*>(poses + N * PM_POSE_STRIDE);
  float* lut = reinterpret_cast<float*>(tsrc + tp);
  for (int i = threadIdx.x; i < N * PM_POSE_STRIDE; i += blockDim.x) poses[i] = P.poses[(size_t)rot * N * PM_POSE_STRIDE + i];
  for (int t = threadIdx.x; t < tp; t += blockDim.x) {   // pm_fill_tap_offsets' {dx, dy}
    const int tr = t / P.nside, tc = t - tr * P.nside;
    off[t] = make_float2((float)(-P.radius + P.step * tc), (float)(-P.radius + P.step * tr));
  }
  pm_fill_tap_src(P, rot, tsrc, threadIdx.x, blockDim.x);
  pm_load_lut(lut, threadIdx.x, blockDim.x);
  const float iK[4] = {P.invK[rot][0], P.invK[rot][1], P.invK[rot][2], P.invK[rot][3]};
  const float Kr[4] = {P.K[rot][0], P.K[rot][1], P.K[rot][2], P.K[rot][3]};
  __syncthreads();
  const size_t npix = (size_t)fw * fh;
  const int g = lane >> 3, sub = lane & 7;
  const unsigned gmask = 0xffu << (8 * g);
  const unsigned full = 0xffffffffu;
  const unsigned nmask = (1u << N) - 1u;
  const int ns = P.num_samples, nsl = ns < 32 ? ns : 32;
  const int mode = PRUNE ? A.prune : 0;
  const bool img_lane = sub < N;
  (void)nsl;
#ifdef PM_PIXEL_PHASES
  __shared__ unsigned long long ph_acc[4][PM_PH_COUNT];
  __shared__ unsigned ph_last[4];
  if (lane == 0) {
    for (int k = 0; k < PM_PH_COUNT; ++k) ph_acc[warp][k] = 0ull;
    ph_last[warp] = (unsigned)clock();
  }
  __syncwarp();
  const PmPhaseClock ph{ph_acc[warp], &ph_last[warp]};
  unsigned long long n_ncc = 0ull, n_rounds = 0ull;
#else
  const PmNoPhase ph;
#endif
  for (size_t q0 = ((size_t)blockIdx.x * 4 + warp) * 4; q0 < npix; q0 += (size_t)gridDim.x * 16) {
    const int npx = (int)min((size_t)4, npix - q0);   // pixels of the batch inside the frame
    const bool live = g < npx;
    const size_t q = live ? q0 + g : q0;              // a group past the frame's end repeats pixel q0 and stores nothing
    const int row = (int)(q / fw), col = (int)(q - (size_t)row * fw);
    const size_t p = pm_pix0(P.W0, P.H0, rot, row, col);
    const float rowf = (float)row, colf = (float)col;
    float inv_wsum = 0.0f;
    for (int k = 0; k < npx; ++k) {   // the batch's patches: copies in flight while the set-up below runs
      const int rk = __shfl_sync(full, row, 8 * k), ck = __shfl_sync(full, col, 8 * k);
      if (P.patch_store) {
        pm_copy_patch<1>(P, tsrc, pm_pix0(P.W0, P.H0, rot, rk, ck), wr_warp + k * tp, lane);
      } else {
        float iw;
        pm_build_patch<1>(P, lut, rot, fw, fh, rk, ck, off, wr_warp + k * tp, lane, &iw);
        if (g == k) inv_wsum = iw;
      }
    }
    if (P.patch_store) inv_wsum = P.patch_inv[p * 4 + rot];
    ph(PM_PH_OTHER);
    const float4 cur4 = P.hyp[p];
    float cn0 = cur4.y, cn1 = cur4.z;
    pm_normal_to_frame(rot, cn0, cn1);
    const float cur_d = cur4.x, cn2 = cur4.w;
    const float4 r4 = A.rand_hyp[p];
    const float rsum = P.ref_sum[p], rsq = P.ref_sqsum[p];
    float prob = 0.0f, cost_i = 0.0f, gcur = 0.0f, grand = 0.0f;
    if (img_lane) {  // per-image priors of the current hypothesis (:1079-1103)
      const float* pose = poses + sub * PM_POSE_STRIDE;
      const float rx = fmaf(iK[0], colf, iK[1]), ry = fmaf(iK[2], rowf, iK[3]);
      float ct, ci;
      pm_viewing_angles(pose, cur_d * rx, cur_d * ry, cur_d, cn0, cn1, cn2, &ct, &ci);
      float Hm[9];
      pm_compose_homography(pose, iK, rowf, colf, cur_d, cn0, cn1, cn2, Hm);
      // kept as three factors: the serial pass evaluates sel_prob * tri * inc * res left to right (:1103)
      const float pt = pm_tri_prob(P.L, ct), pi = pm_inc_prob(P.L, ci), pr = pm_res_prob(Hm, rowf, colf, P.radius);
      if (live) {
        A.prior3[(p * 3 + 0) * N + sub] = pt;
        A.prior3[(p * 3 + 1) * N + sub] = pi;
        A.prior3[(p * 3 + 2) * N + sub] = pr;
      }
      if (GEOM) {
        const PmSrcDesc sd = P.src[sub];
        const float* dm = P.src_depth + sd.depth_off;
        gcur = pm_geom_cost(pose, Kr, iK, dm, sd.w, sd.h, rowf, colf, cur_d, P.geom_max_cost);
        grand = pm_geom_cost(pose, Kr, iK, dm, sd.w, sd.h, rowf, colf, r4.x, P.geom_max_cost);
        if (live) {
          A.gtab2[(p * 2 + 0) * N + sub] = gcur;
          A.gtab2[(p * 2 + 1) * N + sub] = grand;
        }
      }
      if (mode == 1) {
        cost_i = P.cost[p * N + sub];
        const float sp = pm_sel_prob(A.fwd_pred[p * N + sub], A.sel_cur[p * N + sub], A.sel_prev[p * N + sub], A.prev_w);
        prob = sp * pt * pi * pr;
      }
    }
    // ---- which images will be sampled, and how often (prediction; mode 0: every image once), per 8-lane segment
    int mult = img_lane ? 1 : 0;
    unsigned needed4 = 0u;   // bits 8k..8k+7: images pixel k samples
    float thr = 3.0e38f;
    if (PRUNE) {
      if (live)
        for (int e = sub; e < 3 * N; e += 8) A.tab3[p * 3 * N + e] = PM_NOT_EVALUATED;
      if (mode == 1) {
        const float cdf = pm_cdf_lanes(prob, N, sub, 8);
        mult = 0;
        for (int s0 = 0; s0 < nsl; s0 += 8) {   // lane sub predicts sample s0 + sub of its pixel
          const float u = (s0 + sub < nsl) ? A.usamp[p * ns + s0 + sub] : 2.0f;
          const int img = pm_sample_image(cdf, u, N, 8);
#pragma unroll
          for (int j = 0; j < 8; ++j) mult += (__shfl_sync(full, img, j, 8) == sub) ? 1 : 0;
        }
        if (!img_lane) mult = 0;
        needed4 = __ballot_sync(full, live && mult > 0);
        float t = (float)mult * (GEOM ? fmaf(P.geom_reg, gcur, cost_i) : cost_i);
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) t += __shfl_xor_sync(full, t, o);
        thr = fmaf(t, 1.001f, 1e-3f);   // predicted cost sum of the current hypothesis, with a margin for the true order of summation
      }
    }
    ph(PM_PH_SETUP);
    pm_copy_wait();
    __syncwarp();   // patches complete; sentinel stores ordered before the result stores of other lanes
    ph(PM_PH_WAIT);
    // ---- pooled rounds.  Segment k (lanes 8k..8k+7) carries pixel k's round state, warp-uniform within the segment:
    // per hypothesis h (0: rand/rand, 1: cur depth + rand normal, 2: rand depth + cur normal) the images left (rem) and
    // the images evaluated (ev), byte h of each, a bit per image RANK: rank r is image (ord >> 4r) & 15, the images
    // sorted by multiplicity, then by index (the order in which a hypothesis takes its images; the images nobody
    // sampled come last, and lanes >= N after them).  Unpruned (mode 0), every image of every hypothesis is left and
    // nothing is ever dropped.
    const unsigned key = (((unsigned)mult << 5) | (unsigned)(31 - sub)) + 1u;
    int rank = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) rank += (__shfl_sync(full, key, j, 8) > key) ? 1 : 0;
    unsigned ord = (unsigned)sub << (4 * rank);
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) ord |= __shfl_xor_sync(full, ord, o, 8);
    unsigned rem = nmask * 0x10101u, ev = 0u, act = live ? 7u : 0u, ext = 7u;   // act / ext: bit h
    if (PRUNE) {
      const unsigned need = (1u << __popc((needed4 >> (8 * g)) & 0xffu)) - 1u;   // the sampled images: the first ranks
      rem = need * 0x10101u;
      ext = 0u;
      act = (mode == 1 && need) ? 7u : 0u;
    }
    float L0 = 0.0f, L1 = 0.0f, L2 = 0.0f;
    unsigned hp = 0u;   // the hypothesis whose turn is next
    for (;;) {
      // Fill the four group slots in passes: in each pass every pixel with a pair left proposes one, its next
      // hypothesis in turn and that hypothesis' first image left, and pixel by pixel the proposals take the free slots.
      // A pixel left alone takes all four slots in four passes.  Group g evaluates the pair of slot g.
      int my_code = -1, slot = 0;   // my_code: pixel << 8 | h << 4 | image
      for (int pass = 0; pass < 4 && slot < 4; ++pass) {
        const unsigned avail = act & (((rem & 0xffu) ? 1u : 0u) | ((rem & 0xff00u) ? 2u : 0u) | ((rem & 0xff0000u) ? 4u : 0u));
        const unsigned turn = ((avail | (avail << 3)) >> hp) & 7u;
        unsigned h = hp + (unsigned)__ffs(turn) - 1u;
        if (h >= 3u) h -= 3u;
        const unsigned rbit = ((rem >> (8 * h)) & 0xffu) & (0u - ((rem >> (8 * h)) & 0xffu));   // lowest rank left
        const int img = (int)((ord >> (4 * (__ffs(rbit) - 1))) & 15u);
        const unsigned b = __ballot_sync(full, turn != 0u);
        const unsigned pm = (b & 1u) | ((b >> 7) & 2u) | ((b >> 14) & 4u) | ((b >> 21) & 8u);   // pixels proposing
        if (!pm) break;
        if (turn && slot + __popc(pm & ((1u << g) - 1u)) < 4) {   // this pixel's proposal got a slot
          rem &= ~(rbit << (8 * h));
          ev |= rbit << (8 * h);
          hp = (h == 2u) ? 0u : h + 1u;
        }
        const int j = g - slot;   // this group's slot takes the proposal of the j-th proposing pixel, if there is one
        int src = g;
#pragma unroll
        for (int kk = 3; kk >= 0; --kk)
          if (((pm >> kk) & 1u) && __popc(pm & ((1u << kk) - 1u)) == j) src = kk;
        const int code = (g << 8) | (int)(h << 4) | img;
        const int got = __shfl_sync(full, code, 8 * src);
        if (j >= 0 && j < __popc(pm)) my_code = got;
        slot = min(4, slot + __popc(pm));
      }
      ph(PM_PH_SELECT);
      if (slot == 0) break;
      PM_POOL_COUNT(n_rounds, 1);
      PM_POOL_COUNT(n_ncc, slot);
      // pixel kk's values, from the lanes of segment kk
      const int kk = my_code < 0 ? g : (my_code >> 8), my_h = (my_code >> 4) & 15, my_img = my_code & 15;
      const float krow = __shfl_sync(full, rowf, 8 * kk), kcol = __shfl_sync(full, colf, 8 * kk);
      const float kd = __shfl_sync(full, cur_d, 8 * kk), kn0 = __shfl_sync(full, cn0, 8 * kk), kn1 = __shfl_sync(full, cn1, 8 * kk),
                  kn2 = __shfl_sync(full, cn2, 8 * kk);
      const float rd = __shfl_sync(full, r4.x, 8 * kk), rn0 = __shfl_sync(full, r4.y, 8 * kk), rn1 = __shfl_sync(full, r4.z, 8 * kk),
                  rn2 = __shfl_sync(full, r4.w, 8 * kk);
      const float kiw = __shfl_sync(full, inv_wsum, 8 * kk), krs = __shfl_sync(full, rsum, 8 * kk), krq = __shfl_sync(full, rsq, 8 * kk);
      float c = 0.0f;
      if (my_code >= 0) {
        const float hd = (my_h == 1) ? kd : rd;
        const float hn0 = (my_h == 2) ? kn0 : rn0, hn1 = (my_h == 2) ? kn1 : rn1, hn2 = (my_h == 2) ? kn2 : rn2;
        const PmSrcDesc sd = P.src[my_img];
        ph(PM_PH_SELECT);
        c = pm_ncc_group<3, 3, 1>(wr_warp + kk * tp, off, P.ntaps, poses + my_img * PM_POSE_STRIDE, iK, P.quads + sd.quad_off,
                                  sd.pitch, sd.w, sd.h, krow, kcol, hd, hn0, hn1, hn2, kiw, krs, krq, sub, gmask, ph);
        const size_t kp = pm_pix0(P.W0, P.H0, rot, (int)krow, (int)kcol);
        if (sub == 0) A.tab3[(kp * 3 + my_h) * N + my_img] = c;
        ph(PM_PH_FINAL);
      }
      if (PRUNE) {
        // each segment adds its pixel's results of the round, in slot order
#pragma unroll
        for (int s2 = 0; s2 < 4; ++s2) {
          const int cs = __shfl_sync(full, my_code, 8 * s2);
          float v = __shfl_sync(full, c, 8 * s2);
          const int hs = (cs >> 4) & 15, is = cs & 7;
          const float w = (float)__shfl_sync(full, mult, 8 * g + is);
          if (GEOM) v = fmaf(P.geom_reg, __shfl_sync(full, (hs == 1) ? gcur : grand, 8 * g + is), v);
          if (cs >= 0 && (cs >> 8) == g) {
            if (hs == 0) L0 = fmaf(w, v, L0); else if (hs == 1) L1 = fmaf(w, v, L1); else L2 = fmaf(w, v, L2);
          }
        }
      }
      // a hypothesis whose partial sum already exceeds the current hypothesis' sum is out; one that survives all its
      // sampled images is a likely winner: the images nobody sampled are then needed for the cost map (:1184-1196)
#pragma unroll
      for (int h = 0; h < 3; ++h) {
        const float Lh = (h == 0) ? L0 : ((h == 1) ? L1 : L2);
        if ((act >> h) & 1u) {
          if (Lh > thr) {
            act &= ~(1u << h);
          } else if (!((rem >> (8 * h)) & 0xffu)) {
            if (!((ext >> h) & 1u)) { ext |= 1u << h; rem |= (nmask & ~(ev >> (8 * h))) << (8 * h); }
            if (!((rem >> (8 * h)) & 0xffu)) act &= ~(1u << h);
          }
        }
      }
      ph(PM_PH_BOUND);
    }
    __syncwarp();   // every group is done with the batch's patches before the next batch's copies overwrite them
  }
#ifdef PM_PIXEL_PHASES
  if (lane == 0) {
    for (int k = 0; k < PM_PH_COUNT; ++k) atomicAdd(&pm_phase_cycles[PRUNE ? 1 : 0][k], ph_acc[warp][k]);
    atomicAdd(&pm_pool_counts[PRUNE ? 1 : 0][PM_CNT_P_NCC], n_ncc);
    atomicAdd(&pm_pool_counts[PRUNE ? 1 : 0][PM_CNT_P_ROUNDS], n_rounds);
  }
#endif
}

// STORE: the patch comes from the patch store (P.patch_store set).  A template parameter, not a runtime branch, so that
// neither variant of this register-bound (128 of 128) kernel carries the other's code.
template <int WPC, bool GEOM, bool STORE>
__global__ void __launch_bounds__(32 * WPC, 16 / WPC) pm_serial_kernel(const PmParams P, const PmSweepArgs A) {
  extern __shared__ float4 smem4[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col = A.col0 + blockIdx.x;
  const int rot = A.rot, N = P.N;
  const int fw = (rot & 1) ? P.H0 : P.W0, fh = (rot & 1) ? P.W0 : P.H0;
  // the reference patch and its scalars are double-buffered by row parity: the last warp builds row + 1 while warp 0
  // may still evaluate NCCs of row (the rare entries the pixel pass left out)
  float4* patch2 = smem4;
  float* poses = reinterpret_cast<float*>(patch2 + 2 * P.ntaps_pad);
  float* tab1 = poses + N * PM_POSE_STRIDE;  // [32] NCC of the propagated hypothesis per image
  float* hyp1 = tab1 + 32;                   // depth, normal of the propagated hypothesis
  float* fctl2 = hyp1 + 4;                   // [2][4] inv_wsum, ref_sum, ref_sqsum
  float* accb = fctl2 + 8;                   // [8][33] per-sample costs of the five hypotheses (+ three geometric costs)
  int* tsrc = reinterpret_cast<int*>(accb + 272);
  float* lut = reinterpret_cast<float*>(tsrc + P.ntaps_pad);
  for (int i = threadIdx.x; i < N * PM_POSE_STRIDE; i += blockDim.x) poses[i] = P.poses[(size_t)rot * N * PM_POSE_STRIDE + i];
  pm_fill_tap_offsets(P, patch2, threadIdx.x, blockDim.x);
  pm_fill_tap_offsets(P, patch2 + P.ntaps_pad, threadIdx.x, blockDim.x);
  pm_fill_tap_src(P, rot, tsrc, threadIdx.x, blockDim.x);
  pm_load_lut(lut, threadIdx.x, blockDim.x);
  // with the patch store, the last warp copies row + 1's patch and scalars into the other half of the double buffer
  // while row is processed, so nothing of the patch is left on the per-row chain
  const bool store = STORE;
  auto copy_row = [&](int row) {
    const size_t p = pm_pix0(P.W0, P.H0, rot, row, col);
    float* fc = fctl2 + 4 * (row & 1);
    pm_copy_patch<2>(P, tsrc, p, pm_wr(patch2 + (row & 1) * P.ntaps_pad), lane);
    if (lane == 0) { pm_copy_scalar(fc, P.patch_inv + p * 4 + rot); pm_copy_scalar(fc + 1, P.ref_sum + p); pm_copy_scalar(fc + 2, P.ref_sqsum + p); }
  };
  const float iK[4] = {P.invK[rot][0], P.invK[rot][1], P.invK[rot][2], P.invK[rot][3]};
  const float Kr[4] = {P.K[rot][0], P.K[rot][1], P.K[rot][2], P.K[rot][3]};
  const float colf = (float)col;
  const int g = lane >> 3, sub = lane & 7;
  const unsigned gmask = 0xffu << (8 * g);
  const unsigned full = 0xffffffffu;
  const bool img_lane = lane < N;
  __syncthreads();   // tap offsets and tap map complete
  if (store && warp == WPC - 1) copy_row(0);

  float fwd = 0.5f;
  float prev_d = 0.0f, prev_n0 = 0.0f, prev_n1 = 0.0f, prev_n2 = 0.0f;
  const int ns = P.num_samples;
  if (warp == 0) {   // (the backward messages of the column, :976-989, were written to sel_cur by pm_msg_kernel)
    int r0, c0;
    pm_frame_to_orig(P.W0, P.H0, rot, 0, col, &r0, &c0);
    const float4 h0 = P.hyp[(size_t)r0 * P.W0 + c0];
    prev_d = h0.x; prev_n0 = h0.y; prev_n1 = h0.z; prev_n2 = h0.w;
    pm_normal_to_frame(rot, prev_n0, prev_n1);
  }

  // software pipeline: the per-row inputs do not depend on the sweep state, so warp 0 fetches row + 1 while
  // row is being processed (takes two L2 round trips off the per-row critical path)
  float4 nx_cur4 = make_float4(0.f, 0.f, 0.f, 0.f), nx_r4 = nx_cur4;
  float nx_u = 2.0f;
  float nx_cost = 0.f, nx_beta = 0.f, nx_prevp = 0.f, nx_t = 0.f, nx_i = 0.f, nx_r = 0.f, nx_c2 = 0.f, nx_c3 = 0.f, nx_c4 = 0.f,
        nx_gc = 0.f, nx_gr = 0.f;
  auto fetch_row = [&](int row) {
    const size_t p = pm_pix0(P.W0, P.H0, rot, row, col);
    nx_cur4 = P.hyp[p];
    nx_r4 = A.rand_hyp[p];
    nx_u = (lane < ns) ? A.usamp[p * ns + lane] : 2.0f;   // first 32 Monte-Carlo uniforms, one per lane
    if (img_lane) {
      nx_cost = P.cost[p * N + lane];
      nx_beta = A.sel_cur[p * N + lane];
      nx_prevp = A.sel_prev[p * N + lane];
      nx_t = A.prior3[(p * 3 + 0) * N + lane]; nx_i = A.prior3[(p * 3 + 1) * N + lane]; nx_r = A.prior3[(p * 3 + 2) * N + lane];
      nx_c2 = A.tab3[(p * 3 + 0) * N + lane]; nx_c3 = A.tab3[(p * 3 + 1) * N + lane]; nx_c4 = A.tab3[(p * 3 + 2) * N + lane];
      if (GEOM) { nx_gc = A.gtab2[(p * 2 + 0) * N + lane]; nx_gr = A.gtab2[(p * 2 + 1) * N + lane]; }
    }
  };
  if (warp == 0) fetch_row(0);

  for (int row = 0; row < fh; ++row) {
    const size_t p = pm_pix0(P.W0, P.H0, rot, row, col);
    const float rowf = (float)row;
    float4* patch = patch2 + (row & 1) * P.ntaps_pad;
    float* fctl = fctl2 + 4 * (row & 1);
    if (warp == WPC - 1) {
      if (store) {
        pm_copy_wait();
      } else {
        float inv_wsum;
        pm_build_patch<2>(P, lut, rot, fw, fh, row, col, pm_off(patch), pm_wr(patch), lane, &inv_wsum);
        if (lane == 0) { fctl[0] = inv_wsum; fctl[1] = P.ref_sum[p]; fctl[2] = P.ref_sqsum[p]; }
      }
    }
    // ---- phase A (warp 0): propagated hypothesis, sampling distribution, samples
    float cost_i = 0.0f, beta_i = 0.0f, prevp_i = 0.0f, cdf = 0.0f;
    float c2 = 0.0f, c3 = 0.0f, c4 = 0.0f, g_cur = 0.0f, g_rand = 0.0f;
    float cur_d = 0.0f, cur_n0 = 0.0f, cur_n1 = 0.0f, cur_n2 = 0.0f;
    float4 r4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float u_first = 2.0f;
    if (warp == 0) {
      prev_d = pm_propagate_depth(iK, prev_d, prev_n1, prev_n2, (float)(row - 1), rowf);
      const float4 cur4 = nx_cur4;
      cur_d = cur4.x; cur_n0 = cur4.y; cur_n1 = cur4.z; cur_n2 = cur4.w;
      pm_normal_to_frame(rot, cur_n0, cur_n1);
      r4 = nx_r4;
      u_first = nx_u;
      float prob = 0.0f;
      if (img_lane) {
        cost_i = nx_cost; beta_i = nx_beta; prevp_i = nx_prevp;
        const float alpha = pm_forward_message(P.L, cost_i, fwd);
        const float sp = pm_sel_prob(alpha, beta_i, prevp_i, A.prev_w);
        prob = sp * nx_t * nx_i * nx_r;
        c2 = nx_c2; c3 = nx_c3; c4 = nx_c4;
        if (GEOM) { g_cur = nx_gc; g_rand = nx_gr; }
      }
      cdf = pm_cdf_lanes(prob, N, lane);
      if (lane == 0) { hyp1[0] = prev_d; hyp1[1] = prev_n0; hyp1[2] = prev_n1; hyp1[3] = prev_n2; }
    }
    __syncthreads();  // #1: patch + propagated hypothesis visible; every warp is done with row - 1's half of the buffer
    if (store && warp == WPC - 1 && row + 1 < fh) copy_row(row + 1);
    if (warp == 0 && row + 1 < fh) fetch_row(row + 1);

    // ---- phase B (all warps): NCC of the propagated hypothesis against every source image
    const float inv_wsum = fctl[0], rsum = fctl[1], rsq = fctl[2];
    {
      const float hd = hyp1[0], hn0 = hyp1[1], hn1 = hyp1[2], hn2 = hyp1[3];
      for (int img = warp * 4 + g; img < N; img += 4 * WPC) {
        const PmSrcDesc sd = P.src[img];
        const float c = pm_ncc_group<1, 5, 2>(pm_wr(patch), pm_off(patch), P.ntaps, poses + img * PM_POSE_STRIDE, iK, P.quads + sd.quad_off, sd.pitch,
                                     sd.w, sd.h, rowf, colf, hd, hn0, hn1, hn2, inv_wsum, rsum, rsq, sub, gmask);
        if (sub == 0) tab1[img] = c;
      }
    }
    __syncthreads();  // #2: tab1 complete

    // ---- phase C+E (warp 0): sampled costs, argmin, messages, filter, carry state
    if (warp == 0) {
      const float c1 = img_lane ? tab1[lane] : 0.0f;
      float g_prev = 0.0f;
      if (GEOM && img_lane) {
        const PmSrcDesc sd = P.src[lane];
        g_prev = pm_geom_cost(poses + lane * PM_POSE_STRIDE, Kr, iK, P.src_depth + sd.depth_off, sd.w, sd.h, rowf, colf,
                              prev_d, P.geom_max_cost);
      }
      // NCC of hypothesis k (2: rand/rand, 3: cur depth + rand normal, 4: rand depth + cur normal) for the images in
      // `todo`, by this warp's four groups; the results land in lane == image of c2 / c3 / c4
      auto evaluate = [&](int k, unsigned todo) {
        const float hd = (k == 3) ? cur_d : r4.x;
        const float hn0 = (k == 4) ? cur_n0 : r4.y, hn1 = (k == 4) ? cur_n1 : r4.z, hn2 = (k == 4) ? cur_n2 : r4.w;
#ifdef PM_PIXEL_PHASES
        if (lane == 0) atomicAdd(&pm_pool_counts[A.prune ? 1 : 0][PM_CNT_S_NCC], (unsigned long long)__popc(todo));
#endif
        while (todo) {
          int my_img = -1;
#pragma unroll
          for (int s2 = 0; s2 < 4; ++s2)
            if (todo) { const int im = __ffs(todo) - 1; todo &= todo - 1; if (s2 == g) my_img = im; }
          float c = 0.0f;
          if (my_img >= 0) {
            const PmSrcDesc sd = P.src[my_img];
            c = pm_ncc_group<1, 5, 2>(pm_wr(patch), pm_off(patch), P.ntaps, poses + my_img * PM_POSE_STRIDE, iK, P.quads + sd.quad_off, sd.pitch, sd.w, sd.h,
                             rowf, colf, hd, hn0, hn1, hn2, inv_wsum, rsum, rsq, sub, gmask);
          }
#pragma unroll
          for (int s2 = 0; s2 < 4; ++s2) {
            const int is = __shfl_sync(full, my_img, 8 * s2);
            const float cs = __shfl_sync(full, c, 8 * s2);
            if (is == lane) { if (k == 2) c2 = cs; else if (k == 3) c3 = cs; else c4 = cs; }
          }
        }
      };
      // Monte-Carlo accumulation (:1128-1173).  The uniforms were drawn by pass R; lanes pick the sampled image of
      // one sample each, then the five cost sums are accumulated in sample order (a skipped sample adds +0, exact).
      // Entries the pixel pass did not evaluate count as 0: the sums of hypotheses 2..4 are then LOWER bounds
      // (non-negative terms, monotone rounding), which is enough to rule a hypothesis out when the bound already
      // exceeds the sum of hypothesis 0; otherwise the missing entries are evaluated here and the sums redone.
      float a0, a1, a2, a3, a4;
      unsigned out_mask = 0u;   // bit k: hypothesis k is excluded (lower bound > a0)
      for (int attempt = 0;; ++attempt) {
        float acc = 0.0f;
        unsigned sampled = 0u;
        for (int base = 0; base < ns; base += 32) {
          const int sidx = base + lane;
          const float u = (base == 0) ? u_first : ((sidx < ns) ? A.usamp[p * ns + sidx] : 2.0f);
          const int img = pm_sample_image(cdf, u, N);
          const int src = img < 0 ? 0 : img;
          float v0 = __shfl_sync(full, cost_i, src), v1 = __shfl_sync(full, c1, src),
                v2 = __shfl_sync(full, c2, src), v3 = __shfl_sync(full, c3, src),
                v4 = __shfl_sync(full, c4, src);
          float gcv = 0.0f, gpv = 0.0f, grv = 0.0f;
          if (GEOM) { gcv = __shfl_sync(full, g_cur, src); gpv = __shfl_sync(full, g_prev, src); grv = __shfl_sync(full, g_rand, src); }
          if (img < 0) { v0 = v1 = v2 = v3 = v4 = 0.0f; gcv = gpv = grv = 0.0f; }
          v2 = fmaxf(v2, 0.0f); v3 = fmaxf(v3, 0.0f); v4 = fmaxf(v4, 0.0f);   // PM_NOT_EVALUATED -> 0
          if (attempt == 0) sampled |= __reduce_or_sync(full, img < 0 ? 0u : (1u << img));
          // transpose through shared memory: lane k (k = 0..4) then adds the samples of hypothesis k in sample order
          // (15 LDS + 15 FADD on five lanes at once instead of 75 shuffles + 75 adds on the whole warp)
          accb[0 * 33 + lane] = v0; accb[1 * 33 + lane] = v1; accb[2 * 33 + lane] = v2; accb[3 * 33 + lane] = v3; accb[4 * 33 + lane] = v4;
          if (GEOM) { accb[5 * 33 + lane] = gcv; accb[6 * 33 + lane] = gpv; accb[7 * 33 + lane] = grv; }
          __syncwarp();
          const int cnt = min(32, ns - base);
          if (lane < 5) {
            const float* vk = accb + lane * 33;
            const float* gk = accb + ((lane == 1) ? 6 : ((lane == 2 || lane == 4) ? 7 : 5)) * 33;   // cur, prev, rand, cur, rand (:1117-1126)
            for (int j = 0; j < cnt; ++j) {
              acc += vk[j];
              if (GEOM) acc = fmaf(P.geom_reg, gk[j], acc);
            }
          }
          __syncwarp();
        }
        a0 = __shfl_sync(full, acc, 0); a1 = __shfl_sync(full, acc, 1); a2 = __shfl_sync(full, acc, 2);
        a3 = __shfl_sync(full, acc, 3); a4 = __shfl_sync(full, acc, 4);
        if (attempt != 0) break;
        // which sampled entries are missing?
        const unsigned in_s = img_lane && ((sampled >> lane) & 1u);
        const unsigned m2 = __ballot_sync(full, in_s && c2 < 0.0f), m3 = __ballot_sync(full, in_s && c3 < 0.0f),
                       m4 = __ballot_sync(full, in_s && c4 < 0.0f);
        if (!(m2 | m3 | m4)) break;
        unsigned t2 = 0u, t3 = 0u, t4 = 0u;
        if (m2) { if (a2 > a0) out_mask |= 4u; else t2 = m2; }
        if (m3) { if (a3 > a0) out_mask |= 8u; else t3 = m3; }
        if (m4) { if (a4 > a0) out_mask |= 16u; else t4 = m4; }
        if (!(t2 | t3 | t4)) break;
        if (t2) evaluate(2, t2);
        if (t3) evaluate(3, t3);
        if (t4) evaluate(4, t4);
      }
      int best = 0;
      float mn = a0;
      if (a1 <= mn) { mn = a1; best = 1; }
      if (!(out_mask & 4u) && a2 <= mn) { mn = a2; best = 2; }
      if (!(out_mask & 8u) && a3 <= mn) { mn = a3; best = 3; }
      if (!(out_mask & 16u) && a4 <= mn) { mn = a4; best = 4; }
      if (best >= 2) {   // the winner's cost for EVERY image goes to the cost map (:1184-1196)
        const float cb = (best == 2) ? c2 : ((best == 3) ? c3 : c4);
        const unsigned miss = __ballot_sync(full, img_lane && cb < 0.0f);
        if (miss) evaluate(best, miss);
      }
      float best_d, bn0, bn1, bn2;
      switch (best) {
        case 0: best_d = cur_d; bn0 = cur_n0; bn1 = cur_n1; bn2 = cur_n2; break;
        case 1: best_d = prev_d; bn0 = prev_n0; bn1 = prev_n1; bn2 = prev_n2; break;
        case 2: best_d = r4.x; bn0 = r4.y; bn1 = r4.z; bn2 = r4.w; break;
        case 3: best_d = cur_d; bn0 = r4.y; bn1 = r4.z; bn2 = r4.w; break;
        default: best_d = r4.x; bn0 = cur_n0; bn1 = cur_n1; bn2 = cur_n2; break;
      }
      float sp = 0.0f;
      if (img_lane) {
        float c = cost_i;
        if (best != 0) {
          c = (best == 1) ? c1 : ((best == 2) ? c2 : ((best == 3) ? c3 : c4));
          P.cost[p * N + lane] = c;
        }
        const float alpha = pm_forward_message(P.L, c, fwd);
        sp = pm_sel_prob(alpha, beta_i, prevp_i, A.prev_w);
        A.sel_cur[p * N + lane] = sp;
        fwd = alpha;
      }
      bool zero = false;
      if (A.last_filter) {
        bool ok = false;
        if (img_lane) {
          const float* pose = poses + lane * PM_POSE_STRIDE;
          const float rx = fmaf(iK[0], colf, iK[1]), ry = fmaf(iK[2], rowf, iK[3]);
          float ct, ci;
          pm_viewing_angles(pose, best_d * rx, best_d * ry, best_d, bn0, bn1, bn2, &ct, &ci);
          if (!(ct > P.cos_filter_tri || ci <= 0.0f)) {
            ok = sp >= P.min_ncc_prob;
            if (GEOM && ok) {
              const PmSrcDesc sd = P.src[lane];
              ok = pm_geom_cost(pose, Kr, iK, P.src_depth + sd.depth_off, sd.w, sd.h, rowf, colf, best_d,
                                P.geom_max_cost) <= P.filter_geom_max_cost;
            }
          }
        }
        const int cnt = __popc(__ballot_sync(full, ok));
        zero = cnt < P.filter_min_num_consistent;
        if (img_lane) P.mask[p * N + lane] = (ok && !zero) ? 1 : 0;
      }
      if (lane == 0) {
        float o0 = bn0, o1 = bn1;
        pm_normal_to_orig(rot, o0, o1);
        if (zero) {
          float z0 = 0.0f, z1 = 0.0f;
          pm_normal_to_orig(rot, z0, z1);
          P.hyp[p] = make_float4(0.0f, z0, z1, 0.0f);
        } else {
          P.hyp[p] = make_float4(best_d, o0, o1, bn2);
        }
      }
      prev_d = best_d; prev_n0 = bn0; prev_n1 = bn1; prev_n2 = bn2;
    }
  }
}

// exhaustive check of pm_rcp_clamped against the IEEE division over all float bit patterns
__global__ void pm_rcp_check_kernel(unsigned long long* mismatches) {
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  unsigned long long bad = 0;
  for (unsigned long long b = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; b < (1ull << 32); b += stride) {
    const float z = __uint_as_float((unsigned)b);
    const float want = 1.0f / pm_clamp_z(z);
    const float got = pm_rcp_clamped(z);
    if (__float_as_uint(want) != __float_as_uint(got)) ++bad;
  }
  if (bad) atomicAdd(mismatches, bad);
}

// outputs in mvs::Mat<float> layout (slice-major)
__global__ void pm_export_kernel(const PmParams P, const float* sel, float* depth, float* normal, float* sel_out,
                                 uint8_t* mask_out) {
  const size_t n = (size_t)P.W0 * P.H0;
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const float4 h = P.hyp[p];
  if (depth) depth[p] = h.x;
  if (normal) { normal[p] = h.y; normal[n + p] = h.z; normal[2 * n + p] = h.w; }
  if (sel_out) for (int i = 0; i < P.N; ++i) sel_out[(size_t)i * n + p] = sel[p * P.N + i];
  if (mask_out) for (int i = 0; i < P.N; ++i) mask_out[(size_t)i * n + p] = P.mask ? P.mask[p * P.N + i] : 0;
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_pm_error;
static int pm_fail(int code, const std::string& msg) { g_pm_error = msg; return code; }
#define PM_CUDA(call)                                                                              \
  do {                                                                                             \
    cudaError_t e__ = (call);                                                                      \
    if (e__ != cudaSuccess)                                                                        \
      return pm_fail(-100, std::string(#call) + ": " + cudaGetErrorString(e__));                  \
  } while (0)

#define PM_NUM_PASS_TIMES 5   // b200pm_last_pass_ms indices: R|M, P, S, R alone, M alone

struct b200pm_context {
  b200pm_options opt;
  PmParams P;
  int device = 0;
  int wpc = 2;
  bool wpc_auto = true;   // B200PM_WPC unset: the serial pass picks its schedule per sweep (one wave of columns)
  int num_sms = 132;
  cudaStream_t stream = nullptr;
  cudaStream_t stream2 = nullptr;     // pass M runs here, next to pass R on the main stream
  cudaEvent_t fork_ev = nullptr, join_ev = nullptr;   // main stream -> pass M on stream2 -> main stream
  int prune = 1, prune_from = 1;      // exact early-out in the pixel pass (B200PM_PRUNE), from this sweep on (B200PM_PRUNE_FROM)
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  std::vector<std::pair<void*, size_t>> allocs;
  float* sel[2] = {nullptr, nullptr};
  int final_sel = 0;
  bool dirty = false, ran = false;
  float last_ms = 0.0f, last_sweep_ms = 0.0f;
  // rand(+msg) / pixel / serial passes of the last run, then rand and msg alone (b200pm_last_pass_ms)
  float last_kernel_ms[PM_NUM_PASS_TIMES] = {};
  std::vector<float> last_sweep_pass_ms;          // the same per sweep: [sweep][PM_NUM_PASS_TIMES]
  std::vector<cudaEvent_t> sweep_ev;              // [sweep][4] on the main stream: start, R|M done, P done, S done
  std::vector<cudaEvent_t> rm_ev;                 // [sweep][3]: R done (main stream), M start and M done (stream2)
  int last_launches = 0;
  std::vector<int> src_image_idxs;
  size_t smem_init = 0, smem_serial = 0, smem_patch = 0;
  size_t smem_pixel4 = 0;   // 0: the pixel pass runs pm_pixel_kernel (N > 8, or four split patches do not fit a CTA)
  size_t patch_store_bytes = 0;   // 0: the reference patches are built inline by every consumer
  int last_sweeps = 0;      // sweeps the last run did (B200PM_MAX_SWEEPS can stop it early)
  float4* rand_hyp = nullptr; float* usamp = nullptr; float* prior3 = nullptr; float* tab3 = nullptr; float* gtab2 = nullptr;
  float* fwd_pred = nullptr;
};
// pixels a pixel-pass warp handles before its CTA retires (4 measured fastest on the H100; 8 was ~7 ms per C2 run slower)
#define PM_PIXELS_PER_WARP 4
// Device memory the patch store may take (DESIGN.md §2): 2.06 GB at 1920x1080 with window 11; 4K frames (8.2 GB) and
// large windows (13.5 KB per pixel at radius 20) stay on the inline patch build.
#define PM_PATCH_STORE_BUDGET (3ull << 30)

template <typename T>
static cudaError_t pm_alloc(b200pm_context* c, T** p, size_t count) {
  const size_t bytes = sizeof(T) * (count ? count : 1);
  cudaError_t e = B200DeviceCache::get().alloc((void**)p, bytes);
  if (e == cudaSuccess) c->allocs.push_back({(void*)*p, bytes});
  return e;
}

// image.cc:97-150 composed in double and rounded once (ComputeRelativePose, ComputeProjectionCenter,
// ComposeProjectionMatrix, ComposeInverseProjectionMatrix)
static void pm_compose_pose_row(const double refR[9], const double refT[3], const float K[9], const float R2f[9],
                                const float T2f[3], float out[PM_POSE_STRIDE]) {
  double R2[9], T2[3], R[9], T[3], C[3], Pm[12], iP[12];
  for (int i = 0; i < 9; ++i) R2[i] = R2f[i];
  for (int i = 0; i < 3; ++i) T2[i] = T2f[i];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      R[3 * r + c] = R2[3 * r] * refR[3 * c] + R2[3 * r + 1] * refR[3 * c + 1] + R2[3 * r + 2] * refR[3 * c + 2];
  for (int r = 0; r < 3; ++r) T[r] = T2[r] - (R[3 * r] * refT[0] + R[3 * r + 1] * refT[1] + R[3 * r + 2] * refT[2]);
  for (int c = 0; c < 3; ++c) C[c] = -(R[c] * T[0] + R[3 + c] * T[1] + R[6 + c] * T[2]);
  const double fx = K[0], cx = K[2], fy = K[4], cy = K[5];
  for (int c = 0; c < 3; ++c) {
    Pm[c] = fx * R[c] + cx * R[6 + c];
    Pm[4 + c] = fy * R[3 + c] + cy * R[6 + c];
    Pm[8 + c] = R[6 + c];
  }
  Pm[3] = fx * T[0] + cx * T[2];
  Pm[7] = fy * T[1] + cy * T[2];
  Pm[11] = T[2];
  for (int r = 0; r < 3; ++r) {
    iP[4 * r + 0] = R[r] / fx;
    iP[4 * r + 1] = R[3 + r] / fy;
    iP[4 * r + 2] = R[6 + r] - R[r] * cx / fx - R[3 + r] * cy / fy;
    iP[4 * r + 3] = C[r];
  }
  out[0] = K[0]; out[1] = K[2]; out[2] = K[4]; out[3] = K[5];
  for (int i = 0; i < 9; ++i) out[4 + i] = (float)R[i];
  for (int i = 0; i < 3; ++i) out[13 + i] = (float)T[i];
  for (int i = 0; i < 3; ++i) out[16 + i] = (float)C[i];
  for (int i = 0; i < 12; ++i) out[19 + i] = (float)Pm[i];
  for (int i = 0; i < 12; ++i) out[31 + i] = (float)iP[i];
}

// PatchMatchCuda::InitTransforms (patch_match_cuda.cu:1694-1808)
static void pm_init_transforms(const b200pm_problem* p, float K4[4][4], float iK4[4][4], std::vector<float>& poses) {
  const float fx = p->ref_K[0], cx = p->ref_K[2], fy = p->ref_K[4], cy = p->ref_K[5];
  const float Wm1 = (float)(p->ref_width - 1), Hm1 = (float)(p->ref_height - 1);
  const float Kt[4][4] = {{fx, cx, fy, cy}, {fy, cy, fx, Wm1 - cx}, {fx, Wm1 - cx, fy, Hm1 - cy}, {fy, Hm1 - cy, fx, cx}};
  for (int k = 0; k < 4; ++k) {
    for (int i = 0; i < 4; ++i) K4[k][i] = Kt[k][i];
    iK4[k][0] = 1.0f / Kt[k][0];
    iK4[k][1] = -Kt[k][1] / Kt[k][0];
    iK4[k][2] = 1.0f / Kt[k][2];
    iK4[k][3] = -Kt[k][3] / Kt[k][2];
  }
  const int N = p->num_src;
  poses.resize((size_t)4 * N * PM_POSE_STRIDE);
  double R[9], T[3];
  for (int i = 0; i < 9; ++i) R[i] = p->ref_R[i];
  for (int i = 0; i < 3; ++i) T[i] = p->ref_T[i];
  for (int k = 0; k < 4; ++k) {
    for (int i = 0; i < N; ++i)
      pm_compose_pose_row(R, T, p->src_K + 9 * i, p->src_R + 9 * i, p->src_T + 3 * i,
                          poses.data() + ((size_t)k * N + i) * PM_POSE_STRIDE);
    double nR[9], nT[3];
    for (int c = 0; c < 3; ++c) { nR[c] = R[3 + c]; nR[3 + c] = -R[c]; nR[6 + c] = R[6 + c]; }
    nT[0] = T[1]; nT[1] = -T[0]; nT[2] = T[2];
    memcpy(R, nR, sizeof(R)); memcpy(T, nT, sizeof(T));
  }
}

extern "C" {

void b200pm_options_init(b200pm_options* o) {
  o->depth_min = -1.0; o->depth_max = -1.0; o->sigma_spatial = -1.0; o->sigma_color = 0.2f;
  o->ncc_sigma = 0.6f; o->min_triangulation_angle = 1.0f; o->incident_angle_sigma = 0.9f;
  o->geom_consistency_regularizer = 0.3f; o->geom_consistency_max_cost = 3.0f; o->filter_min_ncc = 0.1f;
  o->filter_min_triangulation_angle = 3.0f; o->filter_geom_consistency_max_cost = 1.0f;
  o->window_radius = 5; o->window_step = 1; o->num_samples = 15; o->num_iterations = 5;
  o->filter_min_num_consistent = 2; o->geom_consistency = 1; o->filter = 1; o->gpu_index = -1;
}

const char* b200pm_last_error(void) { return g_pm_error.c_str(); }
void b200pm_internal_set_error(const char* msg) { g_pm_error = msg ? msg : ""; }   // pm_workspace.cu reports through the same channel

int b200pm_check(const b200pm_options* o, const b200pm_problem* p) {
  if (!o || !p) return pm_fail(-1, "null options/problem");
  // PatchMatchOptions::Check (patch_match_options.cc:72-99)
  if (!(o->depth_min >= 0.0 && o->depth_min <= o->depth_max)) return pm_fail(-2, "depth range must be resolved: 0 <= depth_min <= depth_max");
  if (o->window_radius <= 0 || o->window_radius > 20) return pm_fail(-2, "window_radius must be in 1..20");
  if (o->window_step <= 0 || o->window_step > 2) return pm_fail(-2, "window_step must be 1 or 2");
  if (!(o->sigma_color > 0.0)) return pm_fail(-2, "sigma_color must be > 0");
  if (o->num_samples <= 0 || o->num_samples > 1024) return pm_fail(-2, "num_samples must be in 1..1024");
  if (!(o->ncc_sigma > 0.0)) return pm_fail(-2, "ncc_sigma must be > 0");
  if (!(o->min_triangulation_angle >= 0.0 && o->min_triangulation_angle < 180.0)) return pm_fail(-2, "min_triangulation_angle out of range");
  if (!(o->incident_angle_sigma > 0.0)) return pm_fail(-2, "incident_angle_sigma must be > 0");
  if (o->num_iterations <= 0) return pm_fail(-2, "num_iterations must be > 0");
  if (!(o->geom_consistency_regularizer >= 0.0) || !(o->geom_consistency_max_cost >= 0.0)) return pm_fail(-2, "geom_consistency_* must be >= 0");
  if (!(o->filter_min_ncc >= -1.0 && o->filter_min_ncc <= 1.0)) return pm_fail(-2, "filter_min_ncc out of range");
  if (!(o->filter_min_triangulation_angle >= 0.0 && o->filter_min_triangulation_angle <= 180.0)) return pm_fail(-2, "filter_min_triangulation_angle out of range");
  if (o->filter_min_num_consistent < 0) return pm_fail(-2, "filter_min_num_consistent must be >= 0");
  if (!(o->filter_geom_consistency_max_cost >= 0.0)) return pm_fail(-2, "filter_geom_consistency_max_cost must be >= 0");
  // PatchMatch::Check (patch_match.cc:67-126)
  if (p->ref_width <= 0 || p->ref_height <= 0 || !p->ref_gray) return pm_fail(-3, "reference image missing");
  if (p->num_src < 1) return pm_fail(-3, "at least one source image is required");
  if (p->num_src > PM_MAX_SRC) return pm_fail(-3, "more than 32 source images are not supported");
  if (!p->src_width || !p->src_height || !p->src_gray || !p->src_K || !p->src_R || !p->src_T) return pm_fail(-3, "source image arrays missing");
  auto checkK = [](const float* K) { return K[1] == 0.0f && K[3] == 0.0f && K[6] == 0.0f && K[7] == 0.0f && K[8] == 1.0f; };
  if (!checkK(p->ref_K)) return pm_fail(-3, "reference K must have zero skew and K[8] == 1");
  for (int i = 0; i < p->num_src; ++i) {
    if (p->src_width[i] <= 0 || p->src_height[i] <= 0 || !p->src_gray[i]) return pm_fail(-3, "source bitmap missing");
    if (!checkK(p->src_K + 9 * i)) return pm_fail(-3, "source K must have zero skew and K[8] == 1");
    if (p->src_image_idxs)
      for (int j = 0; j < i; ++j)
        if (p->src_image_idxs[i] == p->src_image_idxs[j]) return pm_fail(-3, "duplicate source image index");
  }
  if (o->geom_consistency) {
    if (!p->src_depth || !p->ref_depth_init || !p->ref_normal_init) return pm_fail(-3, "geom_consistency requires depth and normal maps");
    for (int i = 0; i < p->num_src; ++i)
      if (!p->src_depth[i]) return pm_fail(-3, "geom_consistency requires every source depth map");
  }
  return 0;
}

int b200pm_create(const b200pm_options* o, const b200pm_problem* p, b200pm_handle* out) {
  if (!out) return pm_fail(-1, "null handle pointer");
  *out = nullptr;
  const int rc = b200pm_check(o, p);
  if (rc != 0) return rc;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return pm_fail(-101, "no CUDA device: colmap_b200 has no CPU fallback");
  b200pm_context* c = new b200pm_context();
  c->opt = *o;
  if (o->gpu_index >= 0) {
    if (o->gpu_index >= ndev) { delete c; return pm_fail(-101, "gpu_index out of range"); }
    c->device = o->gpu_index;
  } else {
    cudaGetDevice(&c->device);
  }
  PM_CUDA(cudaSetDevice(c->device));
  pm_upload_lut();
  PM_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  for (int i = 0; i < 4; ++i) PM_CUDA(cudaEventCreate(&c->ev[i]));
  PM_CUDA(cudaStreamCreateWithFlags(&c->stream2, cudaStreamNonBlocking));
  PM_CUDA(cudaEventCreateWithFlags(&c->fork_ev, cudaEventDisableTiming));
  PM_CUDA(cudaEventCreateWithFlags(&c->join_ev, cudaEventDisableTiming));
  // Test and diagnostic seams; none changes the result.  B200PM_WPC forces the serial pass's warps per column (the
  // automatic choice depends on the column count against the SM count, so small problems never reach WPC = 1 without
  // it); B200PM_PRUNE / B200PM_PRUNE_FROM select the pixel pass's early-out schedule (PRUNE=2 evaluates nothing there,
  // which shows the serial pass does not depend on the prediction); B200PM_MAX_SWEEPS (read per run by b200pm_run)
  // stops a run after that many sweeps, for sweep-by-sweep comparison with the oracle.  B200PM_PATCH_STORE=0 keeps the
  // inline reference-patch build even where the patch store fits its budget.
  bool patch_store = true;
  if (const char* e = getenv("B200PM_PATCH_STORE")) patch_store = atoi(e) != 0;
  if (const char* e = getenv("B200PM_PRUNE")) c->prune = atoi(e);
  if (const char* e = getenv("B200PM_PRUNE_FROM")) c->prune_from = atoi(e);
  if (const char* e = getenv("B200PM_WPC")) { c->wpc = atoi(e); c->wpc_auto = false; }
  if (c->wpc != 1 && c->wpc != 2 && c->wpc != 4) c->wpc = 2;
  cudaDeviceGetAttribute(&c->num_sms, cudaDevAttrMultiProcessorCount, c->device);

  PmParams& P = c->P;
  memset(&P, 0, sizeof(P));
  P.W0 = p->ref_width; P.H0 = p->ref_height; P.N = p->num_src;
  P.radius = o->window_radius; P.step = o->window_step;
  P.nside = (2 * P.radius) / P.step + 1;
  P.ntaps = P.nside * P.nside;
  P.ntaps_pad = (P.ntaps + 7) & ~7;
  P.ntaps_st = (P.ntaps + 1) & ~1;
  P.num_samples = o->num_samples;
  P.geom = o->geom_consistency ? 1 : 0;
  P.filter_min_num_consistent = o->filter_min_num_consistent;
  P.depth_min = (float)o->depth_min; P.depth_max = (float)o->depth_max;
  const float sigma_spatial = (float)(o->sigma_spatial <= 0 ? (double)o->window_radius : o->sigma_spatial);
  const float sigma_color = (float)o->sigma_color, ncc_sigma = (float)o->ncc_sigma;
  const float inc_sigma = (float)o->incident_angle_sigma;
  P.spatial_norm = 1.0f / (2.0f * sigma_spatial * sigma_spatial);
  P.color_norm = 1.0f / (2.0f * sigma_color * sigma_color);
  P.L.cos_min_tri = cosf((float)(o->min_triangulation_angle * 0.0174532925199432));
  P.L.inv_inc_sigma_sq = -0.5f / (inc_sigma * inc_sigma);
  P.L.inv_ncc_sigma_sq = -0.5f / (ncc_sigma * ncc_sigma);
  P.L.ncc_norm = 2.0f / (sqrtf(2.0f * (float)M_PI) * ncc_sigma * erff(2.0f / (ncc_sigma * 1.414213562f)));
  P.geom_reg = (float)o->geom_consistency_regularizer;
  P.geom_max_cost = (float)o->geom_consistency_max_cost;
  P.filter_geom_max_cost = (float)o->filter_geom_consistency_max_cost;
  P.min_ncc_prob = pm_ncc_prob(P.L, 1.0f - (float)o->filter_min_ncc);
  P.cos_filter_tri = cosf((float)(o->filter_min_triangulation_angle * 0.0174532925199432));

  const size_t n = (size_t)P.W0 * P.H0;
  const int N = P.N;
  c->src_image_idxs.resize(N);
  for (int i = 0; i < N; ++i) c->src_image_idxs[i] = p->src_image_idxs ? p->src_image_idxs[i] : i;

  std::vector<float> poses;
  pm_init_transforms(p, P.K, P.invK, poses);

  uint8_t* d_ref_raw; float* d_poses; PmSrcDesc* d_src; uint32_t* d_quads; float* d_src_depth = nullptr;
  float *d_init_depth = nullptr, *d_init_normal = nullptr;
  PM_CUDA(pm_alloc(c, &d_ref_raw, n));
  PM_CUDA(pm_alloc(c, &P.ref_img, n));
  PM_CUDA(pm_alloc(c, &P.ref_sum, n));
  PM_CUDA(pm_alloc(c, &P.ref_sqsum, n));
  PM_CUDA(pm_alloc(c, &P.hyp, n));
  PM_CUDA(pm_alloc(c, &P.cost, n * N));
  PM_CUDA(pm_alloc(c, &c->sel[0], n * N));
  PM_CUDA(pm_alloc(c, &c->sel[1], n * N));
  if (o->filter) PM_CUDA(pm_alloc(c, &P.mask, n * N));
  PM_CUDA(pm_alloc(c, &d_poses, poses.size()));
  PM_CUDA(pm_alloc(c, &d_src, (size_t)N));
  PM_CUDA(pm_alloc(c, &P.rng, (size_t)6 * (2 * (size_t)P.W0 + 2 * (size_t)P.H0)));
  std::vector<PmSrcDesc> descs(N);
  size_t quad_words = 0, depth_floats = 0, raw_bytes = 0;
  for (int i = 0; i < N; ++i) {
    descs[i].w = p->src_width[i]; descs[i].h = p->src_height[i];
    descs[i].pitch = (p->src_width[i] + 4 + 7) & ~7;
    descs[i].pad = 0;
    descs[i].quad_off = (long long)quad_words;
    descs[i].depth_off = (long long)depth_floats;
    quad_words += (size_t)descs[i].pitch * (descs[i].h + 4);
    depth_floats += (size_t)descs[i].w * descs[i].h;
    raw_bytes = std::max(raw_bytes, (size_t)descs[i].w * descs[i].h);
  }
  PM_CUDA(pm_alloc(c, &d_quads, quad_words));
  uint8_t* d_raw;
  PM_CUDA(pm_alloc(c, &d_raw, raw_bytes));
  if (P.geom) {
    PM_CUDA(pm_alloc(c, &d_src_depth, depth_floats));
    PM_CUDA(pm_alloc(c, &d_init_depth, n));
    PM_CUDA(pm_alloc(c, &d_init_normal, 3 * n));
  }
  P.ref_raw = d_ref_raw; P.poses = d_poses; P.src = d_src; P.quads = d_quads; P.src_depth = d_src_depth;
  P.init_depth = d_init_depth; P.init_normal = d_init_normal;

  cudaStream_t s = c->stream;
  const cudaMemcpyKind map_kind = p->maps_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  PM_CUDA(cudaMemcpyAsync(d_ref_raw, p->ref_gray, n, cudaMemcpyHostToDevice, s));
  PM_CUDA(cudaMemcpyAsync(d_poses, poses.data(), poses.size() * sizeof(float), cudaMemcpyHostToDevice, s));
  PM_CUDA(cudaMemcpyAsync(d_src, descs.data(), sizeof(PmSrcDesc) * N, cudaMemcpyHostToDevice, s));
  for (int i = 0; i < N; ++i) {
    const size_t bytes = (size_t)descs[i].w * descs[i].h;
    PM_CUDA(cudaMemcpyAsync(d_raw, p->src_gray[i], bytes, cudaMemcpyHostToDevice, s));
    dim3 blk(32, 8), grd((descs[i].w + 4 + 31) / 32, (descs[i].h + 4 + 7) / 8);
    pm_pack_quads_kernel<<<grd, blk, 0, s>>>(d_raw, descs[i].w, descs[i].h, descs[i].pitch, d_quads + descs[i].quad_off);
    if (P.geom)
      PM_CUDA(cudaMemcpyAsync(d_src_depth + descs[i].depth_off, p->src_depth[i], bytes * sizeof(float), map_kind, s));
  }
  if (P.geom) {
    PM_CUDA(cudaMemcpyAsync(d_init_depth, p->ref_depth_init, n * sizeof(float), map_kind, s));
    PM_CUDA(cudaMemcpyAsync(d_init_normal, p->ref_normal_init, 3 * n * sizeof(float), map_kind, s));
  }
  {
    dim3 blk(32, 8), grd((P.W0 + 31) / 32, (P.H0 + 7) / 8);
    pm_prefilter_kernel<<<grd, blk, 0, s>>>(P);
    pm_init_kernel<<<grd, blk, 0, s>>>(P, c->sel[1]);
  }
  // patches, poses, then the tap map (pm_fill_tap_src) and the /255 table
  c->smem_init = sizeof(float4) * 4 * P.ntaps_pad + sizeof(float) * ((size_t)N * PM_POSE_STRIDE + P.ntaps_pad + 256);
  c->smem_serial = sizeof(float4) * 2 * P.ntaps_pad + sizeof(float) * ((size_t)N * PM_POSE_STRIDE + 32 + 4 + 8 + 272 + P.ntaps_pad + 256);
  c->smem_patch = sizeof(float) * (256 + 9 * (size_t)P.ntaps_pad);   // lut, tap offsets (int2), 3 tap maps, 4 warps' weights
  {   // pm_pixel4_kernel: 16 split patches, the {dx, dy} table, poses, tap map, /255 table
    const size_t bytes = sizeof(float2) * 17 * P.ntaps_pad + sizeof(float) * ((size_t)N * PM_POSE_STRIDE + P.ntaps_pad + 256);
    int optin = 0;
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device);
    if (N <= 8 && bytes <= (size_t)optin) c->smem_pixel4 = bytes;
  }
  const size_t store_bytes = n * ((size_t)P.ntaps_st * sizeof(float2) + 4 * sizeof(float));
  if (patch_store && store_bytes <= PM_PATCH_STORE_BUDGET) {
    PM_CUDA(pm_alloc(c, &P.patch_store, n * P.ntaps_st));
    PM_CUDA(pm_alloc(c, &P.patch_inv, 4 * n));
    c->patch_store_bytes = store_bytes;
  }
  PM_CUDA(pm_alloc(c, &c->rand_hyp, n));
  PM_CUDA(pm_alloc(c, &c->usamp, n * (size_t)o->num_samples));
  PM_CUDA(pm_alloc(c, &c->prior3, 3 * n * N));
  PM_CUDA(pm_alloc(c, &c->tab3, 3 * n * N));
  if (P.geom) PM_CUDA(pm_alloc(c, &c->gtab2, 2 * n * N));
  PM_CUDA(pm_alloc(c, &c->fwd_pred, n * N));
  PM_CUDA(cudaStreamSynchronize(s));
  PM_CUDA(cudaGetLastError());
  *out = c;
  return 0;
}

}  // extern "C"

template <int WPC, bool STORE>
static void pm_launch_serial_store(b200pm_context* c, const PmSweepArgs& A, int fw) {
  if (c->smem_serial > 48 * 1024) {
    cudaFuncSetAttribute(pm_serial_kernel<WPC, true, STORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_serial);
    cudaFuncSetAttribute(pm_serial_kernel<WPC, false, STORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_serial);
  }
  if (c->P.geom)
    pm_serial_kernel<WPC, true, STORE><<<fw, 32 * WPC, c->smem_serial, c->stream>>>(c->P, A);
  else
    pm_serial_kernel<WPC, false, STORE><<<fw, 32 * WPC, c->smem_serial, c->stream>>>(c->P, A);
}
template <int WPC>
static void pm_launch_serial(b200pm_context* c, const PmSweepArgs& A, int fw) {
  if (c->P.patch_store) pm_launch_serial_store<WPC, true>(c, A, fw);
  else pm_launch_serial_store<WPC, false>(c, A, fw);
}

// The arguments of sweep t (iteration t / 4, frame t % 4) of a run
static PmSweepArgs pm_sweep_args(const b200pm_context* c, int t) {
  const int iters = c->opt.num_iterations, iter = t / 4, sweep = t % 4;
  const float total_steps = (float)(iters * 4);
  PmSweepArgs A;
  memset(&A, 0, sizeof(A));
  A.rot = sweep;
  A.perturbation = 1.0f / powf(2.0f, (float)iter + (float)sweep / 4.0f);
  A.perturbation_pi = (float)((double)A.perturbation * M_PI);
  A.prev_w = (float)(iter * 4 + sweep) / total_steps;
  A.last_filter = (iter == iters - 1 && sweep == 3 && c->opt.filter) ? 1 : 0;
  A.sel_cur = c->sel[t & 1];
  A.sel_prev = c->sel[(t + 1) & 1];
  A.rand_hyp = c->rand_hyp; A.usamp = c->usamp; A.prior3 = c->prior3; A.tab3 = c->tab3; A.gtab2 = c->gtab2;
  A.fwd_pred = c->fwd_pred;
  A.prune = (c->prune == 1) ? ((t >= c->prune_from) ? 1 : 0) : c->prune;
  return A;
}

// Pass M (messages) on stream2 beside pass R (random hypotheses) on the main stream: both only read the state the last
// sweep left.  The main stream goes on when both are done.  ev: nullptr, or the sweep's timing events {R done, M start,
// M done}.
static void pm_launch_rand_msg(b200pm_context* c, const PmSweepArgs& A, const cudaEvent_t* ev) {
  const int fw = (A.rot & 1) ? c->P.H0 : c->P.W0;
  cudaEventRecord(c->fork_ev, c->stream);
  cudaStreamWaitEvent(c->stream2, c->fork_ev, 0);
  if (ev) cudaEventRecord(ev[1], c->stream2);
  pm_msg_kernel<<<(fw * c->P.N + PM_MSG_THREADS - 1) / PM_MSG_THREADS, PM_MSG_THREADS, 0, c->stream2>>>(c->P, A);
  if (ev) cudaEventRecord(ev[2], c->stream2);
  cudaEventRecord(c->join_ev, c->stream2);
  const int rgrid = (fw + PM_RAND_WARPS * PM_RAND_CPW - 1) / (PM_RAND_WARPS * PM_RAND_CPW);
  if (c->P.num_samples == 15) pm_rand_kernel<15><<<rgrid, 32 * PM_RAND_WARPS, 0, c->stream>>>(c->P, A);
  else pm_rand_kernel<0><<<rgrid, 32 * PM_RAND_WARPS, 0, c->stream>>>(c->P, A);
  if (ev) cudaEventRecord(ev[0], c->stream);
  cudaStreamWaitEvent(c->stream, c->join_ev, 0);
}

extern "C" {

// PatchMatchCuda::RunWithWindowSizeAndStep (patch_match_cuda.cu:1393-1546)
int b200pm_run(b200pm_handle c) {
  if (!c) return pm_fail(-1, "null handle");
  PM_CUDA(cudaSetDevice(c->device));
  const PmParams& P = c->P;
  cudaStream_t s = c->stream;
  if (c->smem_patch > 48 * 1024)
    PM_CUDA(cudaFuncSetAttribute(pm_patch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_patch));
  if (c->smem_init > 48 * 1024) {
    PM_CUDA(cudaFuncSetAttribute(pm_initial_cost_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_init));
    PM_CUDA(cudaFuncSetAttribute(pm_pixel_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_init));
    PM_CUDA(cudaFuncSetAttribute(pm_pixel_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_init));
    PM_CUDA(cudaFuncSetAttribute(pm_pixel_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_init));
    PM_CUDA(cudaFuncSetAttribute(pm_pixel_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_init));
  }
  if (c->smem_pixel4 > 48 * 1024) {
    PM_CUDA(cudaFuncSetAttribute(pm_pixel4_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_pixel4));
    PM_CUDA(cudaFuncSetAttribute(pm_pixel4_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_pixel4));
    PM_CUDA(cudaFuncSetAttribute(pm_pixel4_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_pixel4));
    PM_CUDA(cudaFuncSetAttribute(pm_pixel4_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_pixel4));
  }
  int launches = 0;
  PM_CUDA(cudaEventRecord(c->ev[0], s));
  if (c->dirty) {  // a previous run consumed the initial state: rebuild it (same as the constructor)
    dim3 blk(32, 8), grd((P.W0 + 31) / 32, (P.H0 + 7) / 8);
    pm_init_kernel<<<grd, blk, 0, s>>>(P, c->sel[1]);
    ++launches;
  }
  c->dirty = true;
  {
    const size_t n = (size_t)P.W0 * P.H0;
    const int grid = (int)std::min<size_t>((n + 3) / 4, (size_t)c->num_sms * 64);
    if (P.patch_store) {
      pm_patch_kernel<<<grid, 128, c->smem_patch, s>>>(P);
      ++launches;
    }
    pm_initial_cost_kernel<<<grid, 128, c->smem_init, s>>>(P);
    ++launches;
  }
  PM_CUDA(cudaEventRecord(c->ev[1], s));
  const int iters = c->opt.num_iterations;
  int t = 0;
  const int max_sweeps = getenv("B200PM_MAX_SWEEPS") ? atoi(getenv("B200PM_MAX_SWEEPS")) : -1;
  c->final_sel = 1;   // until a sweep runs, the selection probability is the 0.5 that pm_init_kernel wrote to sel[1]
  for (int iter = 0; iter < iters; ++iter) {
    for (int sweep = 0; sweep < 4; ++sweep, ++t) {
      if (max_sweeps >= 0 && t >= max_sweeps) break;
      const PmSweepArgs A = pm_sweep_args(c, t);
      const int fw = (sweep & 1) ? P.H0 : P.W0;
      auto event = [&](std::vector<cudaEvent_t>& evs, size_t id) {
        while (evs.size() <= id) { cudaEvent_t e; cudaEventCreate(&e); evs.push_back(e); }
        return evs[id];
      };
      auto mark = [&](int idx) { cudaEventRecord(event(c->sweep_ev, (size_t)t * 4 + idx), s); };
      mark(0);
      event(c->rm_ev, (size_t)t * 3 + 2);   // creates the sweep's three R and M events
      pm_launch_rand_msg(c, A, &c->rm_ev[(size_t)t * 3]);
      mark(1);
      const size_t npx = (size_t)fw * ((sweep & 1) ? P.W0 : P.H0);
      const int pgrid = (int)((npx + 4 * PM_PIXELS_PER_WARP - 1) / (4 * PM_PIXELS_PER_WARP));
      const size_t s4 = c->smem_pixel4;
      if (s4 && P.geom) {
        if (A.prune) pm_pixel4_kernel<true, true><<<pgrid, 128, s4, s>>>(P, A);
        else pm_pixel4_kernel<true, false><<<pgrid, 128, s4, s>>>(P, A);
      } else if (s4) {
        if (A.prune) pm_pixel4_kernel<false, true><<<pgrid, 128, s4, s>>>(P, A);
        else pm_pixel4_kernel<false, false><<<pgrid, 128, s4, s>>>(P, A);
      } else if (P.geom) {
        if (A.prune) pm_pixel_kernel<true, true><<<pgrid, 128, c->smem_init, s>>>(P, A);
        else pm_pixel_kernel<true, false><<<pgrid, 128, c->smem_init, s>>>(P, A);
      } else {
        if (A.prune) pm_pixel_kernel<false, true><<<pgrid, 128, c->smem_init, s>>>(P, A);
        else pm_pixel_kernel<false, false><<<pgrid, 128, c->smem_init, s>>>(P, A);
      }
      mark(2);
      // The serial pass is one CTA per column marching down all rows: a second wave of CTAs lengthens its critical
      // path.  Pick the widest schedule whose resident capacity covers all fw columns in ONE wave (register-file
      // bound: 128 registers x 32*WPC threads per CTA).  On the H100 (132 SMs) every C2 sweep, 1920 or 1080 columns,
      // runs WPC = 1 (a fixed WPC = 2 is ~18 ms per run slower).
      int wpc = c->wpc;
      if (c->wpc_auto) wpc = (fw <= c->num_sms * 4) ? 4 : ((fw <= c->num_sms * 8) ? 2 : 1);
      if (wpc == 1) pm_launch_serial<1>(c, A, fw);
      else if (wpc == 2) pm_launch_serial<2>(c, A, fw);
      else pm_launch_serial<4>(c, A, fw);
      launches += 4;
      mark(3);
      c->final_sel = t & 1;
    }
  }
  PM_CUDA(cudaEventRecord(c->ev[2], s));
  PM_CUDA(cudaStreamSynchronize(s));
  PM_CUDA(cudaGetLastError());
  PM_CUDA(cudaEventElapsedTime(&c->last_ms, c->ev[0], c->ev[2]));
  PM_CUDA(cudaEventElapsedTime(&c->last_sweep_ms, c->ev[1], c->ev[2]));
  c->last_sweeps = t;
  for (float& ms : c->last_kernel_ms) ms = 0.0f;
  c->last_sweep_pass_ms.assign((size_t)t * PM_NUM_PASS_TIMES, 0.0f);
  for (int i = 0; i < t; ++i) {
    const cudaEvent_t* sw = &c->sweep_ev[(size_t)i * 4];
    const cudaEvent_t* rm = &c->rm_ev[(size_t)i * 3];
    const cudaEvent_t from[PM_NUM_PASS_TIMES] = {sw[0], sw[1], sw[2], sw[0], rm[1]};
    const cudaEvent_t to[PM_NUM_PASS_TIMES] = {sw[1], sw[2], sw[3], rm[0], rm[2]};
    for (int kk = 0; kk < PM_NUM_PASS_TIMES; ++kk) {
      float ms = 0.0f;
      if (cudaEventElapsedTime(&ms, from[kk], to[kk]) == cudaSuccess) {
        c->last_kernel_ms[kk] += ms;
        c->last_sweep_pass_ms[(size_t)i * PM_NUM_PASS_TIMES + kk] = ms;
      }
    }
  }
  c->last_launches = launches;
  c->ran = true;
  return 0;
}

float b200pm_last_run_ms(b200pm_handle c) { return c ? c->last_ms : -1.0f; }
float b200pm_last_sweep_ms(b200pm_handle c) { return c ? c->last_sweep_ms : -1.0f; }
int b200pm_last_num_launches(b200pm_handle c) { return c ? c->last_launches : -1; }
float b200pm_last_pass_ms(b200pm_handle c, int which) {
  return (c && which >= 0 && which < PM_NUM_PASS_TIMES) ? c->last_kernel_ms[which] : -1.0f;
}
float b200pm_last_sweep_pass_ms(b200pm_handle c, int sweep, int which) {
  if (!c || which < 0 || which >= PM_NUM_PASS_TIMES || sweep < 0 ||
      (size_t)sweep * PM_NUM_PASS_TIMES >= c->last_sweep_pass_ms.size())
    return -1.0f;
  return c->last_sweep_pass_ms[(size_t)sweep * PM_NUM_PASS_TIMES + which];
}
size_t b200pm_patch_store_bytes(b200pm_handle c) { return c ? c->patch_store_bytes : 0; }

static int pm_export(b200pm_handle c, float* depth, float* normal, float* sel, uint8_t* mask) {
  if (!c) return pm_fail(-1, "null handle");
  PM_CUDA(cudaSetDevice(c->device));
  const PmParams& P = c->P;
  const size_t n = (size_t)P.W0 * P.H0;
  float *d_depth = nullptr, *d_normal = nullptr, *d_sel = nullptr;
  uint8_t* d_mask = nullptr;
  B200DeviceCache& cache = B200DeviceCache::get();
  if (depth) PM_CUDA(cache.alloc((void**)&d_depth, n * sizeof(float)));
  if (normal) PM_CUDA(cache.alloc((void**)&d_normal, 3 * n * sizeof(float)));
  if (sel) PM_CUDA(cache.alloc((void**)&d_sel, n * P.N * sizeof(float)));
  if (mask) PM_CUDA(cache.alloc((void**)&d_mask, n * P.N));
  pm_export_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c->stream>>>(P, c->sel[c->ran ? c->final_sel : 1], d_depth, d_normal, d_sel, d_mask);
  if (depth) PM_CUDA(cudaMemcpyAsync(depth, d_depth, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  if (normal) PM_CUDA(cudaMemcpyAsync(normal, d_normal, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  if (sel) PM_CUDA(cudaMemcpyAsync(sel, d_sel, n * P.N * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  if (mask) PM_CUDA(cudaMemcpyAsync(mask, d_mask, n * P.N, cudaMemcpyDeviceToHost, c->stream));
  PM_CUDA(cudaStreamSynchronize(c->stream));
  cache.free(d_depth, n * sizeof(float)); cache.free(d_normal, 3 * n * sizeof(float)); cache.free(d_sel, n * P.N * sizeof(float)); cache.free(d_mask, n * P.N);
  PM_CUDA(cudaGetLastError());
  return 0;
}

// device-to-device export: the maps never leave HBM (geometric phase of a workspace run)
static int pm_export_device(b200pm_handle c, float* d_depth, float* d_normal) {
  if (!c) return pm_fail(-1, "null handle");
  if (!d_depth && !d_normal) return pm_fail(-1, "null device buffer");
  PM_CUDA(cudaSetDevice(c->device));
  const size_t n = (size_t)c->P.W0 * c->P.H0;
  pm_export_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c->stream>>>(c->P, c->sel[c->ran ? c->final_sel : 1], d_depth, d_normal, nullptr, nullptr);
  PM_CUDA(cudaStreamSynchronize(c->stream));
  PM_CUDA(cudaGetLastError());
  return 0;
}
int b200pm_get_depth_device(b200pm_handle c, float* d_depth) { return pm_export_device(c, d_depth, nullptr); }
int b200pm_get_normal_device(b200pm_handle c, float* d_normal) { return pm_export_device(c, nullptr, d_normal); }
int b200pm_get_depth(b200pm_handle c, float* depth) { return pm_export(c, depth, nullptr, nullptr, nullptr); }
int b200pm_get_normal(b200pm_handle c, float* normal) { return pm_export(c, nullptr, normal, nullptr, nullptr); }
int b200pm_get_sel_prob(b200pm_handle c, float* sel) { return pm_export(c, nullptr, nullptr, sel, nullptr); }
int b200pm_get_consistency_mask(b200pm_handle c, uint8_t* mask) { return pm_export(c, nullptr, nullptr, nullptr, mask); }

// PatchMatchCuda::GetConsistentImageIdxs (patch_match_cuda.cu:1367-1391)
int b200pm_get_consistency(b200pm_handle c, int** data, size_t* count) {
  if (!c || !data || !count) return pm_fail(-1, "null argument");
  const PmParams& P = c->P;
  const size_t n = (size_t)P.W0 * P.H0;
  std::vector<uint8_t> mask(n * P.N);
  const int rc = pm_export(c, nullptr, nullptr, nullptr, mask.data());
  if (rc != 0) return rc;
  std::vector<int> list;
  std::vector<int> px;
  for (int r = 0; r < P.H0; ++r)
    for (int col = 0; col < P.W0; ++col) {
      px.clear();
      const size_t p = (size_t)r * P.W0 + col;
      for (int d = 0; d < P.N; ++d)
        if (mask[(size_t)d * n + p]) px.push_back(c->src_image_idxs[d]);
      if (!px.empty()) {
        list.push_back(col); list.push_back(r); list.push_back((int)px.size());
        list.insert(list.end(), px.begin(), px.end());
      }
    }
  *count = list.size();
  *data = (int*)malloc(sizeof(int) * (list.size() ? list.size() : 1));
  memcpy(*data, list.data(), sizeof(int) * list.size());
  return 0;
}

void b200pm_free(void* p) { free(p); }

// Drops the device blocks kept for reuse by destroyed handles / finished solves (both paths share the cache).
void b200_release_cached_memory(void) { B200DeviceCache::get().release(); }

void b200pm_destroy(b200pm_handle c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  for (auto& a : c->allocs) B200DeviceCache::get().free(a.first, a.second);
  for (int i = 0; i < 4; ++i) if (c->ev[i]) cudaEventDestroy(c->ev[i]);
  for (cudaEvent_t e : c->sweep_ev) cudaEventDestroy(e);
  for (cudaEvent_t e : c->rm_ev) cudaEventDestroy(e);
  if (c->fork_ev) cudaEventDestroy(c->fork_ev);
  if (c->join_ev) cudaEventDestroy(c->join_ev);
  if (c->stream2) { cudaStreamSynchronize(c->stream2); cudaStreamDestroy(c->stream2); }
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
}

// debug: cost map in slice-major layout (N*H*W)
int b200pm_debug_get_cost(b200pm_handle c, float* cost) {
  if (!c) return pm_fail(-1, "null handle");
  const PmParams& P = c->P;
  const size_t n = (size_t)P.W0 * P.H0;
  std::vector<float> tmp(n * P.N);
  PM_CUDA(cudaMemcpy(tmp.data(), P.cost, sizeof(float) * n * P.N, cudaMemcpyDeviceToHost));
  for (size_t p = 0; p < n; ++p)
    for (int i = 0; i < P.N; ++i) cost[(size_t)i * n + p] = tmp[p * P.N + i];
  return 0;
}

// debug: the last sweep's tab3 ([pixel][3][N], pixel in the original orientation), PM_NOT_EVALUATED where the pixel
// pass left an entry out
int b200pm_debug_get_tab3(b200pm_handle c, float* out) {
  if (!c) return pm_fail(-1, "null handle");
  PM_CUDA(cudaSetDevice(c->device));
  const size_t n = (size_t)c->P.W0 * c->P.H0;
  PM_CUDA(cudaMemcpy(out, c->tab3, sizeof(float) * 3 * n * c->P.N, cudaMemcpyDeviceToHost));
  return 0;
}

// debug: passes R and M of the sweep that follows the last run (sweep t = the run's sweep count, which B200PM_MAX_SWEEPS
// sets), on the state that run left.  Out, pixels in the original orientation: rand_hyp [pixel][4], usamp
// [pixel][num_samples], the backward messages sel [pixel][N] (pass S overwrites them with the selection probabilities,
// so they are read here, before any pass S), fwd [pixel][N], and the RNG border slots [2 W + 2 H][6] after pass R.  The
// handle's maps are unchanged; its RNG slots advance as that sweep's pass R advances them.
int b200pm_debug_rand_msg(b200pm_handle c, float* rand_hyp, float* usamp, float* sel, float* fwd, uint32_t* rng) {
  if (!c) return pm_fail(-1, "null handle");
  if (!c->ran || c->last_sweeps >= 4 * c->opt.num_iterations) return pm_fail(-1, "no sweep follows the last run");
  PM_CUDA(cudaSetDevice(c->device));
  const PmParams& P = c->P;
  const size_t n = (size_t)P.W0 * P.H0, nN = n * P.N;
  const PmSweepArgs A = pm_sweep_args(c, c->last_sweeps);
  pm_launch_rand_msg(c, A, nullptr);
  PM_CUDA(cudaStreamSynchronize(c->stream));
  PM_CUDA(cudaGetLastError());
  PM_CUDA(cudaMemcpy(rand_hyp, A.rand_hyp, sizeof(float4) * n, cudaMemcpyDeviceToHost));
  PM_CUDA(cudaMemcpy(usamp, A.usamp, sizeof(float) * n * P.num_samples, cudaMemcpyDeviceToHost));
  PM_CUDA(cudaMemcpy(sel, A.sel_cur, sizeof(float) * nN, cudaMemcpyDeviceToHost));
  PM_CUDA(cudaMemcpy(fwd, A.fwd_pred, sizeof(float) * nN, cudaMemcpyDeviceToHost));
  PM_CUDA(cudaMemcpy(rng, P.rng, sizeof(uint32_t) * 6 * (2 * (size_t)P.W0 + 2 * (size_t)P.H0), cudaMemcpyDeviceToHost));
  return 0;
}

// The column-serial statement of pass R: one column's rows in order, each from where the previous one left the stream.
static void pm_rand_column_host(const PmParams& P, const PmSweepArgs& A, const float4* hyp, uint32_t* rng, int col,
                                float4* rand_hyp, float* usamp, uint8_t* rounds) {
  const int rot = A.rot;
  const int fh = (rot & 1) ? P.W0 : P.H0;
  const float iK[4] = {P.invK[rot][0], P.invK[rot][1], P.invK[rot][2], P.invK[rot][3]};
  int r0, c0;
  pm_frame_to_orig(P.W0, P.H0, rot, 0, col, &r0, &c0);
  uint32_t* slot = rng + 6 * (size_t)pm_border_index(P.W0, P.H0, r0, c0);
  PmRng rs;
  rs.v0 = slot[0]; rs.v1 = slot[1]; rs.v2 = slot[2]; rs.v3 = slot[3]; rs.v4 = slot[4]; rs.d = slot[5];
  const float colf = (float)col;
  for (int row = 0; row < fh; ++row) {
    const size_t p = pm_pix0(P.W0, P.H0, rot, row, col);
    const float4 cur4 = hyp[p];
    float n0 = cur4.y, n1 = cur4.z;
    pm_normal_to_frame(rot, n0, n1);
    const float dmin = (1.0f - A.perturbation) * cur4.x;
    const float dmax = (1.0f + A.perturbation) * cur4.x;
    const float rand_d = fmaf(pm_rng_uniform(rs), dmax - dmin, dmin);
    float rn[3];
    rounds[p] = (uint8_t)pm_perturb_normal(iK, (float)row, colf, A.perturbation_pi, n0, n1, cur4.w, rs, rn);
    rand_hyp[p] = make_float4(rand_d, rn[0], rn[1], rn[2]);
    for (int s = 0; s < P.num_samples; ++s) usamp[p * P.num_samples + s] = pm_rng_uniform(rs) - FLT_EPSILON;
  }
  slot[0] = rs.v0; slot[1] = rs.v1; slot[2] = rs.v2; slot[3] = rs.v3; slot[4] = rs.v4; slot[5] = rs.d;
}
// The column-serial statement of pass M for one (column, image): the backward recurrence, then the forward one.
static void pm_msg_column_host(const PmParams& P, const PmSweepArgs& A, const float* cost, int col, int img, float* sel,
                               float* fwd) {
  const int rot = A.rot, N = P.N;
  const int fh = (rot & 1) ? P.W0 : P.H0;
  float beta = 0.5f;
  for (int row = fh - 1; row >= 0; --row) {
    const size_t p = pm_pix0(P.W0, P.H0, rot, row, col);
    beta = pm_backward_message(P.L, cost[p * N + img], beta);
    sel[p * N + img] = beta;
  }
  float f = 0.5f;
  for (int row = 0; row < fh; ++row) {
    const size_t p = pm_pix0(P.W0, P.H0, rot, row, col);
    f = pm_forward_message(P.L, cost[p * N + img], f);
    fwd[p * N + img] = f;
  }
}

// test: what b200pm_debug_rand_msg returns, computed on the host by pm_rand_column_host and pm_msg_column_host from the
// device state the last run left, plus the PerturbNormal rounds of every pixel (rounds [pixel]).  Changes nothing.
int b200pm_test_rand_msg(b200pm_handle c, float* rand_hyp, float* usamp, float* sel, float* fwd, uint32_t* rng,
                         uint8_t* rounds) {
  if (!c) return pm_fail(-1, "null handle");
  if (!c->ran || c->last_sweeps >= 4 * c->opt.num_iterations) return pm_fail(-1, "no sweep follows the last run");
  PM_CUDA(cudaSetDevice(c->device));
  const PmParams& P = c->P;
  const size_t n = (size_t)P.W0 * P.H0;
  const PmSweepArgs A = pm_sweep_args(c, c->last_sweeps);
  std::vector<float4> hyp(n);
  std::vector<float> cost(n * P.N);
  PM_CUDA(cudaMemcpy(hyp.data(), P.hyp, sizeof(float4) * n, cudaMemcpyDeviceToHost));
  PM_CUDA(cudaMemcpy(cost.data(), P.cost, sizeof(float) * n * P.N, cudaMemcpyDeviceToHost));
  PM_CUDA(cudaMemcpy(rng, P.rng, sizeof(uint32_t) * 6 * (2 * (size_t)P.W0 + 2 * (size_t)P.H0), cudaMemcpyDeviceToHost));
  const int fw = (A.rot & 1) ? P.H0 : P.W0;
  for (int col = 0; col < fw; ++col) {
    pm_rand_column_host(P, A, hyp.data(), rng, col, reinterpret_cast<float4*>(rand_hyp), usamp, rounds);
    for (int img = 0; img < P.N; ++img) pm_msg_column_host(P, A, cost.data(), col, img, sel, fwd);
  }
  return 0;
}

// ---- host-side hooks for the CPU test tier (bit-level comparison with the oracle; no GPU needed) ----
float b200pm_test_expf(float x) { return pm_expf(x); }
void b200pm_test_sincosf(float a, float* s, float* c) { pm_sincosf(a, s, c); }
void b200pm_test_rng_stream(unsigned long long seed, int count, float* out) {
  PmRng r; pm_rng_init(r, seed);
  for (int i = 0; i < count; ++i) out[i] = pm_rng_uniform(r);
}
int b200pm_test_poses(const b200pm_problem* p, int k, float* poses_out, float* K_out, float* invK_out) {
  float K4[4][4], iK4[4][4];
  std::vector<float> poses;
  pm_init_transforms(p, K4, iK4, poses);
  memcpy(poses_out, poses.data() + (size_t)k * p->num_src * PM_POSE_STRIDE, sizeof(float) * p->num_src * PM_POSE_STRIDE);
  memcpy(K_out, K4[k], 16); memcpy(invK_out, iK4[k], 16);
  return 0;
}
float b200pm_test_rcp_clamped(float z) { return pm_rcp_clamped(z); }
// GPU: number of float bit patterns for which the fast reciprocal differs from IEEE 1/clamp(z) (must be 0)
long long b200pm_test_rcp_exhaustive(void) {
  unsigned long long* d = nullptr;
  unsigned long long h = 0;
  if (cudaMalloc(&d, 8) != cudaSuccess) return -1;
  cudaMemset(d, 0, 8);
  pm_rcp_check_kernel<<<132 * 8, 256>>>(d);
  if (cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost) != cudaSuccess) { cudaFree(d); return -1; }
  cudaFree(d);
  return (long long)h;
}
void b200pm_test_homography(const float* pose, const float* iK, float row, float col, float depth, const float* n, float* H) {
  pm_compose_homography(pose, iK, row, col, depth, n[0], n[1], n[2], H);
}
int b200pm_test_border_index(int W0, int H0, int r0, int c0) { return pm_border_index(W0, H0, r0, c0); }

#ifdef PM_PIXEL_PHASES
// diagnostic build: out[pruned * PM_PH_COUNT + phase] = pixel-pass cycles since the last call, then reset
int b200pm_debug_pixel_phases(unsigned long long* out) {
  PM_CUDA(cudaDeviceSynchronize());
  PM_CUDA(cudaMemcpyFromSymbol(out, pm_phase_cycles, sizeof(pm_phase_cycles)));
  const unsigned long long zero[2][PM_PH_COUNT] = {};
  PM_CUDA(cudaMemcpyToSymbol(pm_phase_cycles, zero, sizeof(zero)));
  return PM_PH_COUNT;
}
// diagnostic build: out[pruned * PM_CNT_COUNT + k] = pm_pool_counts since the last call, then reset
int b200pm_debug_pool_counts(unsigned long long* out) {
  PM_CUDA(cudaDeviceSynchronize());
  PM_CUDA(cudaMemcpyFromSymbol(out, pm_pool_counts, sizeof(pm_pool_counts)));
  const unsigned long long zero[2][PM_CNT_COUNT] = {};
  PM_CUDA(cudaMemcpyToSymbol(pm_pool_counts, zero, sizeof(zero)));
  return PM_CNT_COUNT;
}
#endif

}  // extern "C"
