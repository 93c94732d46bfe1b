// sift_matching.cu — SIFT feature matching behind include/b200_sift_matching.h: FindBestMatchesBruteForce
// (src/colmap/feature/sift.cc:772-864) on the tensor cores, for a list of image pairs per call.
//
// Schedule (DESIGN.md, "SIFT feature matching"):
//   1. sm_scan_kernel: one CTA per (pair, direction, 128-row strip of the query image).  Four warps, 32 query rows
//      each, hold their rows' descriptors in registers; 128-column tiles of the other image stream through a
//      three-stage cp.async ring in shared memory.  u8 x u8 -> s32 mma.sync (m16n8k32, four k-steps per 128-byte
//      descriptor) gives exact dot products, which go straight into a per-row top-2 (best, index, second) in
//      registers; the dot matrix never leaves the SM.  After the last tile the four lanes of a row merge their top-2,
//      and the row's one-way decision (distance and ratio test through the acosf table) is written.  With
//      cross_check the pair is scanned a second time with the images swapped, which is the transposed matrix.
//   2. sm_compact_kernel: one CTA per pair; the cross-check and an ordered compaction (ascending point2D_idx1).
//   3. sm_offsets_kernel / sm_gather_kernel: the pairs' match counts become offsets, the matches one packed list.
// Guided matching (b200sm_match_guided_pairs, DESIGN.md "Guided matching") replaces step 1 with sm_guided_kernel: the
// same strips, tiles and products, exact L2 distances, a per-candidate E/F/H filter and a min top-2.
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/b200_sift_matching.h"

static thread_local std::string g_sm_err;

namespace {

constexpr int kDim = B200SM_DESCRIPTOR_DIM;
constexpr int kStrip = 128;          // query rows per CTA: 4 warps x 32 rows
constexpr int kTile = 128;           // columns per shared-memory tile; slots are zero-padded to a multiple of this
constexpr int kStages = 3;
constexpr int kThreads = 128;
constexpr int kAcosN = 262145;       // acosf(k * 2^-18), k = 0..2^18
constexpr size_t kTileBytes = (size_t)kTile * kDim;
constexpr size_t kScanSmem = kStages * kTileBytes;
static_assert(kTile % kStrip == 0, "slots are padded to whole tiles, which must hold whole strips");

int fail(int code, const std::string& msg) { g_sm_err = msg; return code; }

#define SM_CHECK(x)                                                                          \
  do {                                                                                       \
    cudaError_t e_ = (x);                                                                    \
    if (e_ != cudaSuccess) return fail(B200SM_ERR_CUDA, std::string(#x ": ") + cudaGetErrorString(e_)); \
  } while (0)

struct ScanItem {
  const uint8_t* a;   // first row of the strip (zero-padded rows up to the strip's end)
  const uint8_t* b;   // the other image, zero-padded to num_tiles * kTile rows
  int64_t out;        // the strip's first row in the one-way match list (each row: its match, or -1)
  int rows;           // valid rows of the strip
  int num_tiles;
};

struct PairItem {
  int64_t m12, m21;    // first row of the pair's one-way lists (image 1 -> 2, 2 -> 1; m21 < 0 without cross_check)
  int n1, n2;
  int64_t base;        // start of the pair's region in the scratch list
};

// The top-2 of the reference's sequential scan (sift.cc:787-797) over the columns seen so far: best and second are
// the largest and second-largest dot product counted with multiplicity, floored at 0, and idx is the smallest column
// holding best (-1 while best == 0).  Two such summaries of disjoint column sets merge exactly and associatively.
__device__ __forceinline__ void top2_merge(int& b, int& s, int& i, int ob, int os, int oi) {
  const int ns = max(max(s, os), min(b, ob));
  i = ob > b ? oi : (ob == b ? min(i, oi) : i);
  b = max(b, ob);
  s = ns;
}

// One column, visited in ascending order within the thread: the reference's update rule itself.
__device__ __forceinline__ void top2_push(int& b, int& s, int& i, int v, int j) {
  const bool gt = v > b;
  s = gt ? b : max(s, v);
  i = gt ? j : i;
  b = gt ? v : b;
}

__device__ __forceinline__ void mma_u8(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                       uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// A tile is 128 columns x 8 chunks of 16 bytes; chunk ch of column c is stored at c * 8 + (ch ^ (c & 7)) so that the
// fragment loads below (column g of an 8-column group, chunks 2t and 2t+1) fall on distinct banks.
__device__ __forceinline__ void load_tile(uint4* stage, const uint8_t* b, int tile) {
  const uint8_t* src = b + (size_t)tile * kTileBytes;
  for (int c = threadIdx.x; c < kTile * 8; c += kThreads) {
    const int col = c >> 3, ch = c & 7;
    cp_async16(stage + col * 8 + (ch ^ (col & 7)), src + (size_t)col * kDim + ch * 16);
  }
}

// The k order inside the MMAs is permuted identically for both operands (a sum does not depend on its order): at
// k-step s, lane quad position t supplies descriptor bytes [32t + 8s, 32t + 8s + 8) as its two 4-byte k-words, so each
// lane's operands for all four k-steps are one 32-byte run of the descriptor, loaded as two 16-byte vectors.
__global__ void __launch_bounds__(kThreads) sm_scan_kernel(const ScanItem* __restrict__ items,
                                                           const float* __restrict__ acos_tab, float max_ratio,
                                                           float max_distance, int32_t* __restrict__ m) {
  extern __shared__ __align__(128) uint4 smem[];
  const ScanItem it = items[blockIdx.x];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;

  uint32_t a[2][2][8];   // [m-tile][row g, row g + 8][k-word]
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint4* p = reinterpret_cast<const uint4*>(it.a + (size_t)(warp * 32 + mt * 16 + h * 8 + g) * kDim + 32 * t);
      const uint4 lo = __ldg(p), hi = __ldg(p + 1);
      a[mt][h][0] = lo.x; a[mt][h][1] = lo.y; a[mt][h][2] = lo.z; a[mt][h][3] = lo.w;
      a[mt][h][4] = hi.x; a[mt][h][5] = hi.y; a[mt][h][6] = hi.z; a[mt][h][7] = hi.w;
    }

  int best[2][2], sec[2][2], idx[2][2];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) { best[mt][h] = 0; sec[mt][h] = 0; idx[mt][h] = -1; }

  const int nt = it.num_tiles;
#pragma unroll
  for (int s = 0; s < kStages - 1; ++s) {
    if (s < nt) load_tile(smem + s * (kTileBytes / 16), it.b, s);
    cp_async_commit();
  }
  for (int tile = 0; tile < nt; ++tile) {
    cp_async_wait<kStages - 2>();
    __syncthreads();   // tile `tile` is visible to all, and every warp is done with the stage refilled next
    const int next = tile + kStages - 1;
    if (next < nt) load_tile(smem + (next % kStages) * (kTileBytes / 16), it.b, next);
    cp_async_commit();
    const uint4* S = smem + (tile % kStages) * (kTileBytes / 16);
#pragma unroll 4
    for (int n8 = 0; n8 < kTile / 8; ++n8) {
      const int col = n8 * 8 + g;
      const uint4 lo = S[col * 8 + ((2 * t) ^ (col & 7))], hi = S[col * 8 + ((2 * t + 1) ^ (col & 7))];
      const uint32_t bw[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
      const int j = tile * kTile + n8 * 8 + 2 * t;
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        int c[4] = {0, 0, 0, 0};
#pragma unroll
        for (int s = 0; s < 4; ++s)
          mma_u8(c, a[mt][0][2 * s], a[mt][1][2 * s], a[mt][0][2 * s + 1], a[mt][1][2 * s + 1], bw[2 * s], bw[2 * s + 1]);
        top2_push(best[mt][0], sec[mt][0], idx[mt][0], c[0], j);
        top2_push(best[mt][0], sec[mt][0], idx[mt][0], c[1], j + 1);
        top2_push(best[mt][1], sec[mt][1], idx[mt][1], c[2], j);
        top2_push(best[mt][1], sec[mt][1], idx[mt][1], c[3], j + 1);
      }
    }
  }
  cp_async_wait<0>();

#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int b = best[mt][h], s = sec[mt][h], i = idx[mt][h];
#pragma unroll
      for (int x = 1; x <= 2; x <<= 1) {
        const int ob = __shfl_xor_sync(0xffffffffu, b, x), os = __shfl_xor_sync(0xffffffffu, s, x),
                  oi = __shfl_xor_sync(0xffffffffu, i, x);
        top2_merge(b, s, i, ob, os, oi);
      }
      const int row = warp * 32 + mt * 16 + h * 8 + g;
      if (t == 0 && row < it.rows) {
        int match = -1;
        if (i >= 0) {
          // std::acos(std::min(dot * 2^-18, 1.0f)); dot * 2^-18 is exact, so the table index is min(dot, 2^18)
          const float d1 = __ldg(acos_tab + min(b, kAcosN - 1));
          if (!(d1 > max_distance)) {
            const float d2 = __ldg(acos_tab + min(s, kAcosN - 1));
            if (!(d1 >= __fmul_rn(max_ratio, d2))) match = i;
          }
        }
        m[it.out + row] = match;
      }
    }
}

// ---------------------------------------------------------------------------------------------- guided matching
// One pair's geometric filter (sift.cc:1226-1262), with everything it reads.  geo rows: the unit ray, the row-major
// 3 x 2 pixel Jacobian, then 1 for a valid ray and 0 for an invalid one.
constexpr int kGeo = 10;
constexpr float kSqNorm = 262144.0f;   // kSqSiftDescriptorNorm: the distance of a rejected candidate
struct GuidedPair {
  const float2* xy1;
  const float2* xy2;
  const double* geo1;
  const double* geo2;
  double Md[9];        // E (fp64)
  float Mf[9];         // F or H rounded to float
  double thr_d;        // max_error^2
  float thr_f;         // (float)(max_error^2)
  int type;
};

struct GuidedItem {
  ScanItem s;
  const int32_t* na;   // squared norms of the strip's rows
  const int32_t* nb;   // squared norms of the other image's rows (padding rows: 0)
  int pair, dir;       // dir 1: the strip's rows are image 2's (the cross-check scan)
  int r0, n2;          // the strip's first row in its image; the other image's valid rows
};

// The scan's state mirrored for minima (FindBestMatchesOneWayIndex, sift.cc:876-890): best and second are the smallest
// and second-smallest distance counted with multiplicity (FLT_MAX while unseen), idx the smallest column holding best.
__device__ __forceinline__ void min2_merge(float& b, float& s, int& i, float ob, float os, int oi) {
  const float ns = fminf(fminf(s, os), fmaxf(b, ob));
  i = ob < b ? oi : (ob == b ? min(i, oi) : i);
  b = fminf(b, ob);
  s = ns;
}
__device__ __forceinline__ void min2_push(float& b, float& s, int& i, float v, int j) {
  const bool lt = v < b;
  s = lt ? b : fminf(s, v);
  i = lt ? j : i;
  b = lt ? v : b;
}

__device__ __forceinline__ float f3(const float* m, float x, float y) {   // (m0 x + m1 y) + m2, no contraction
  return __fadd_rn(__fadd_rn(__fmul_rn(m[0], x), __fmul_rn(m[1], y)), m[2]);
}
__device__ __forceinline__ double d3(double a0, double b0, double a1, double b1, double a2, double b2) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2));
}
// SquaredPixelGradientNorm (essential_matrix.h:189-194) of a row-major 3 x 2 J
__device__ __forceinline__ double pixel_grad_sq(const double* J, double g0, double g1, double g2) {
  const double gx = d3(J[0], g0, J[2], g1, J[4], g2), gy = d3(J[1], g0, J[3], g1, J[5], g2);
  return __dadd_rn(__dmul_rn(gx, gx), __dmul_rn(gy, gy));
}

// Whether the pair's geometry rejects the candidate (i1, i2).  A comparison with a NaN operand does not reject.  Not
// inlined: the scan calls it only for candidates that could enter a row's top-2, and one copy keeps the scan's
// registers for the products.
__device__ __noinline__ bool guided_reject(const GuidedPair* __restrict__ P, int i1, int i2) {
  const int type = P->type;
  if (type == B200SM_GUIDED_E) {
    const double* g1 = P->geo1 + (size_t)i1 * kGeo;
    const double* g2 = P->geo2 + (size_t)i2 * kGeo;
    if (g1[9] == 0.0 || g2[9] == 0.0) return true;
    const double* E = P->Md;
    const double r10 = g1[0], r11 = g1[1], r12 = g1[2], r20 = g2[0], r21 = g2[1], r22 = g2[2];
    const double e0 = d3(E[0], r10, E[1], r11, E[2], r12), e1 = d3(E[3], r10, E[4], r11, E[5], r12),
                 e2 = d3(E[6], r10, E[7], r11, E[8], r12);                       // E ray1
    const double t0 = d3(E[0], r20, E[3], r21, E[6], r22), t1 = d3(E[1], r20, E[4], r21, E[7], r22),
                 t2 = d3(E[2], r20, E[5], r21, E[8], r22);                       // E^T ray2
    const double num = d3(r20, e0, r21, e1, r22, e2);
    const double den = __dadd_rn(pixel_grad_sq(g1 + 3, t0, t1, t2), pixel_grad_sq(g2 + 3, e0, e1, e2));
    const double err = den == 0.0 ? DBL_MAX : __ddiv_rn(__dmul_rn(num, num), den);
    return err > P->thr_d;
  }
  const float2 p1 = P->xy1[i1], p2 = P->xy2[i2];
  const float* M = P->Mf;
  if (type == B200SM_GUIDED_F) {
    const float e0 = f3(M, p1.x, p1.y), e1 = f3(M + 3, p1.x, p1.y), e2 = f3(M + 6, p1.x, p1.y);   // F p1
    const float t0 = __fadd_rn(__fadd_rn(__fmul_rn(M[0], p2.x), __fmul_rn(M[3], p2.y)), M[6]);     // F^T p2
    const float t1 = __fadd_rn(__fadd_rn(__fmul_rn(M[1], p2.x), __fmul_rn(M[4], p2.y)), M[7]);
    const float nom = __fadd_rn(__fadd_rn(__fmul_rn(p2.x, e0), __fmul_rn(p2.y, e1)), e2);
    const float den = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(e0, e0), __fmul_rn(e1, e1)), __fmul_rn(t0, t0)),
                                __fmul_rn(t1, t1));
    return __fmul_rn(nom, nom) > __fmul_rn(P->thr_f, den);
  }
  const float hx = f3(M, p1.x, p1.y), hy = f3(M + 3, p1.x, p1.y), hz = f3(M + 6, p1.x, p1.y);     // H p1
  const float dx = __fsub_rn(__fdiv_rn(hx, hz), p2.x), dy = __fsub_rn(__fdiv_rn(hy, hz), p2.y);
  return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) > P->thr_f;
}

// The guided scan: sm_scan_kernel's strips, tile ring and u8 products; the epilogue turns each dot into the exact L2
// |a|^2 + |b|^2 - 2 dot (below 2^24, so exact in fp32) and keeps a min top-2 per row.  A candidate is pushed with
// distance 512^2 when the filter rejects it.  The filter runs only where it can matter: a candidate whose real
// distance and 512^2 are both >= the row's current second changes nothing whatever the filter says.  Padding columns
// (j >= n2) are skipped; unlike a zero dot, a padding row's L2 is real and would win.
__global__ void __launch_bounds__(kThreads) sm_guided_kernel(const GuidedItem* __restrict__ items,
                                                             const GuidedPair* __restrict__ pairs, float max_ratio,
                                                             float max_l2, int32_t* __restrict__ m) {
  extern __shared__ __align__(128) uint4 smem[];
  const GuidedItem it = items[blockIdx.x];
  const GuidedPair* P = pairs + it.pair;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;

  uint32_t a[2][2][8];
  int na[2][2];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = warp * 32 + mt * 16 + h * 8 + g;
      const uint4* p = reinterpret_cast<const uint4*>(it.s.a + (size_t)row * kDim + 32 * t);
      const uint4 lo = __ldg(p), hi = __ldg(p + 1);
      a[mt][h][0] = lo.x; a[mt][h][1] = lo.y; a[mt][h][2] = lo.z; a[mt][h][3] = lo.w;
      a[mt][h][4] = hi.x; a[mt][h][5] = hi.y; a[mt][h][6] = hi.z; a[mt][h][7] = hi.w;
      na[mt][h] = __ldg(it.na + row);
    }

  float best[2][2], sec[2][2];
  int idx[2][2];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) { best[mt][h] = FLT_MAX; sec[mt][h] = FLT_MAX; idx[mt][h] = -1; }

  const int nt = it.s.num_tiles, n2 = it.n2, rows = it.s.rows, r0 = it.r0, dir = it.dir;
#pragma unroll
  for (int s = 0; s < kStages - 1; ++s) {
    if (s < nt) load_tile(smem + s * (kTileBytes / 16), it.s.b, s);
    cp_async_commit();
  }
  for (int tile = 0; tile < nt; ++tile) {
    cp_async_wait<kStages - 2>();
    __syncthreads();
    const int next = tile + kStages - 1;
    if (next < nt) load_tile(smem + (next % kStages) * (kTileBytes / 16), it.s.b, next);
    cp_async_commit();
    const uint4* S = smem + (tile % kStages) * (kTileBytes / 16);
#pragma unroll 2
    for (int n8 = 0; n8 < kTile / 8; ++n8) {
      const int col = n8 * 8 + g;
      const uint4 lo = S[col * 8 + ((2 * t) ^ (col & 7))], hi = S[col * 8 + ((2 * t + 1) ^ (col & 7))];
      const uint32_t bw[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
      const int j = tile * kTile + n8 * 8 + 2 * t;
      const int2 nb = __ldg(reinterpret_cast<const int2*>(it.nb + j));
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        int c[4] = {0, 0, 0, 0};
#pragma unroll
        for (int s = 0; s < 4; ++s)
          mma_u8(c, a[mt][0][2 * s], a[mt][1][2 * s], a[mt][0][2 * s + 1], a[mt][1][2 * s + 1], bw[2 * s], bw[2 * s + 1]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int h = k >> 1, q = k & 1, jj = j + q;
          const float v = (float)(na[mt][h] + (q ? nb.y : nb.x) - 2 * c[k]);
          const int row = warp * 32 + mt * 16 + h * 8 + g;
          if (jj < n2 && row < rows && fminf(v, kSqNorm) < sec[mt][h]) {
            const int qr = r0 + row;
            const bool rej = guided_reject(P, dir ? jj : qr, dir ? qr : jj);
            min2_push(best[mt][h], sec[mt][h], idx[mt][h], rej ? kSqNorm : v, jj);
          }
        }
      }
    }
  }
  cp_async_wait<0>();

#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float b = best[mt][h], s = sec[mt][h];
      int i = idx[mt][h];
#pragma unroll
      for (int x = 1; x <= 2; x <<= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, b, x), os = __shfl_xor_sync(0xffffffffu, s, x);
        const int oi = __shfl_xor_sync(0xffffffffu, i, x);
        min2_merge(b, s, i, ob, os, oi);
      }
      const int row = warp * 32 + mt * 16 + h * 8 + g;
      if (t == 0 && row < rows) {
        int match = -1;
        // sift.cc:893-906: sqrtf is correctly rounded, as std::sqrt(float) is
        if (i >= 0 && !(b > max_l2) && !(__fsqrt_rn(b) >= __fmul_rn(max_ratio, __fsqrt_rn(s)))) match = i;
        m[it.s.out + row] = match;
      }
    }
}

__global__ void sm_norms_kernel(const uint8_t* __restrict__ d, int64_t rows, int32_t* __restrict__ out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const uint4* p = reinterpret_cast<const uint4*>(d + (size_t)r * kDim);
  uint32_t s = 0;
#pragma unroll
  for (int k = 0; k < kDim / 16; ++k) {
    const uint4 v = __ldg(p + k);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int b = 0; b < 4; ++b) s = __dp4a(w[b], w[b], s);
  }
  out[r] = (int32_t)s;
}

// Exclusive prefix of a per-thread count over a 1024-thread block; returns the block total in *total.
__device__ __forceinline__ int block_exclusive_scan(int v, int* warp_sums, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = lane < nw ? warp_sums[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w += y;
    }
    if (lane < nw) warp_sums[lane] = w;
  }
  __syncthreads();
  const int r = (warp > 0 ? warp_sums[warp - 1] : 0) + x - v;
  *total = warp_sums[nw - 1];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(1024) sm_compact_kernel(const PairItem* __restrict__ pairs,
                                                          const int32_t* __restrict__ m, uint2* __restrict__ scratch,
                                                          uint32_t* __restrict__ counts) {
  __shared__ int warp_sums[32];
  const PairItem p = pairs[blockIdx.x];
  int running = 0;
  if (p.n1 > 0 && p.n2 > 0) {
    for (int base = 0; base < p.n1; base += blockDim.x) {
      const int i1 = base + threadIdx.x;
      int j = -1;
      if (i1 < p.n1) {
        j = m[p.m12 + i1];
        if (j >= 0 && p.m21 >= 0 && m[p.m21 + j] != i1) j = -1;
      }
      int total;
      const int pos = block_exclusive_scan(j >= 0 ? 1 : 0, warp_sums, &total);
      if (j >= 0) scratch[p.base + running + pos] = make_uint2((uint32_t)i1, (uint32_t)j);
      running += total;
    }
  }
  if (threadIdx.x == 0) counts[blockIdx.x] = (uint32_t)running;
}

// offsets[0..P] = exclusive prefix of counts, in one 1024-thread block (each thread sums a contiguous run).
__global__ void __launch_bounds__(1024) sm_offsets_kernel(const uint32_t* __restrict__ counts, int P,
                                                          unsigned long long* __restrict__ offsets) {
  __shared__ unsigned long long part[1024];
  const int per = (P + blockDim.x - 1) / blockDim.x;
  const int lo = min(P, (int)threadIdx.x * per), hi = min(P, lo + per);
  unsigned long long s = 0;
  for (int k = lo; k < hi; ++k) s += counts[k];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int d = 1; d < (int)blockDim.x; d <<= 1) {
    const unsigned long long y = threadIdx.x >= (unsigned)d ? part[threadIdx.x - d] : 0ull;
    __syncthreads();
    part[threadIdx.x] += y;
    __syncthreads();
  }
  unsigned long long run = part[threadIdx.x] - s;
  for (int k = lo; k < hi; ++k) { offsets[k] = run; run += counts[k]; }
  if (threadIdx.x == blockDim.x - 1) offsets[P] = part[threadIdx.x];
}

__global__ void sm_gather_kernel(const PairItem* __restrict__ pairs, const uint2* __restrict__ scratch,
                                 const uint32_t* __restrict__ counts, const unsigned long long* __restrict__ offsets,
                                 uint2* __restrict__ out) {
  const int64_t base = pairs[blockIdx.x].base;
  const unsigned long long o = offsets[blockIdx.x];
  for (uint32_t k = threadIdx.x; k < counts[blockIdx.x]; k += blockDim.x) out[o + k] = scratch[base + k];
}


// Device buffer that only grows.
template <typename T>
struct Buf {
  T* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    const cudaError_t e = cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T));
    if (e == cudaSuccess) cap = n;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

struct Slot {
  uint8_t* d = nullptr;
  int64_t n = 0;
  int64_t cap_rows = 0;
  // guided matching
  int64_t n_desc = 0;          // descriptor rows as given, before the max_num_matches clamp
  int64_t n_kp = -1;           // keypoints as given (-1: none)
  std::vector<float> kp;       // the first n keypoints (x, y), on the host for the rays
  Buf<float2> xy;              // the first n keypoints
  Buf<double> geo;             // kGeo doubles per row: ray, Jacobian, validity
  Buf<int32_t> norms;          // squared descriptor norms, padded rows included
  bool has_camera = false, norms_ok = false;
  void release() { if (d) cudaFree(d); d = nullptr; xy.release(); geo.release(); norms.release(); }
};

}  // namespace

struct b200sm_matcher {
  b200sm_options o;
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
  float* acos_tab = nullptr;
  std::vector<Slot> slots;
  Buf<ScanItem> items;
  Buf<PairItem> pairs;
  Buf<GuidedItem> gitems;
  Buf<GuidedPair> gpairs;
  Buf<int32_t> m;
  Buf<uint2> scratch, out;
  Buf<uint32_t> counts;
  Buf<unsigned long long> offsets;
  double scan_ms = -1, total_ms = -1;
};

static int use_device(b200sm_handle h) {
  SM_CHECK(cudaSetDevice(h->device));
  return 0;
}

static int finish_pairs(b200sm_handle h, int num_pairs, int64_t bound, uint64_t* offsets, uint32_t* matches);
bool sm_cam_ray_with_jac(int id, const double* params, double x, double y, double* out9);   // sift_rays.cu

extern "C" {

const char* b200sm_last_error(void) { return g_sm_err.c_str(); }

void b200sm_options_init(b200sm_options* o) {
  if (!o) return;
  o->max_ratio = 0.8; o->max_distance = 0.7; o->cross_check = 1; o->max_num_matches = 32768; o->gpu_index = -1;
}

int b200sm_create(const b200sm_options* o, int num_slots, b200sm_handle* out) {
  if (!o || !out) return fail(B200SM_ERR_INPUT, "null options or output handle");
  *out = nullptr;
  if (!(o->max_ratio > 0)) return fail(B200SM_ERR_INPUT, "max_ratio must be > 0");
  if (!(o->max_distance > 0)) return fail(B200SM_ERR_INPUT, "max_distance must be > 0");
  if (o->max_num_matches < 0) return fail(B200SM_ERR_INPUT, "max_num_matches must be >= 0");
  if (num_slots < 1) return fail(B200SM_ERR_INPUT, "num_slots must be >= 1");
  if (o->gpu_index < -1) return fail(B200SM_ERR_INPUT, "gpu_index must be >= -1");
  if (o->max_num_matches > B200SM_MAX_NUM_FEATURES)
    return fail(B200SM_ERR_TOO_LARGE, "max_num_matches exceeds B200SM_MAX_NUM_FEATURES");
  if (num_slots > B200SM_MAX_NUM_SLOTS) return fail(B200SM_ERR_TOO_LARGE, "num_slots exceeds B200SM_MAX_NUM_SLOTS");

  int ndev = 0;
  SM_CHECK(cudaGetDeviceCount(&ndev));
  if (o->gpu_index >= ndev) return fail(B200SM_ERR_INPUT, "gpu_index out of range");
  int device = o->gpu_index;
  if (device < 0) SM_CHECK(cudaGetDevice(&device));
  SM_CHECK(cudaSetDevice(device));

  // std::acos(float) is the C library's acosf; its argument dot * 2^-18 takes only these values
  std::vector<float> tab(kAcosN);
  for (int k = 0; k < kAcosN; ++k) tab[k] = acosf((float)k * (1.0f / 262144.0f));

  b200sm_matcher* h = new b200sm_matcher();
  h->o = *o;
  h->device = device;
  h->slots.resize(num_slots);
  auto cleanup = [&](int rc) { b200sm_destroy(h); return rc; };
  cudaError_t e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  for (int k = 0; k < 3 && e == cudaSuccess; ++k) e = cudaEventCreate(&h->ev[k]);
  if (e == cudaSuccess) e = cudaMalloc(&h->acos_tab, sizeof(float) * kAcosN);
  if (e == cudaSuccess) e = cudaMemcpy(h->acos_tab, tab.data(), sizeof(float) * kAcosN, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(sm_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kScanSmem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(sm_guided_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kScanSmem);
  if (e != cudaSuccess) return cleanup(fail(B200SM_ERR_CUDA, std::string("b200sm_create: ") + cudaGetErrorString(e)));
  *out = h;
  return 0;
}

int b200sm_set_descriptors(b200sm_handle h, int slot, int64_t n, const uint8_t* desc) {
  if (!h) return fail(B200SM_ERR_INPUT, "null handle");
  if (slot < 0 || slot >= (int)h->slots.size()) return fail(B200SM_ERR_INPUT, "slot out of range");
  if (n < 0) return fail(B200SM_ERR_INPUT, "negative number of descriptors");
  if (n > 0 && !desc) return fail(B200SM_ERR_INPUT, "null descriptors");
  const int64_t rows = std::min<int64_t>(n, h->o.max_num_matches);
  Slot& s = h->slots[slot];
  if (use_device(h)) return B200SM_ERR_CUDA;
  s.n = 0;
  s.n_desc = n; s.n_kp = -1; s.kp.clear(); s.has_camera = false; s.norms_ok = false;
  if (rows == 0) return 0;
  const int64_t padded = (rows + kTile - 1) / kTile * kTile;
  if (padded > s.cap_rows) {
    if (s.d) SM_CHECK(cudaFree(s.d));
    s.d = nullptr; s.cap_rows = 0;
    SM_CHECK(cudaMalloc(&s.d, (size_t)padded * kDim));
    s.cap_rows = padded;
  }
  SM_CHECK(cudaMemcpyAsync(s.d, desc, (size_t)rows * kDim, cudaMemcpyHostToDevice, h->stream));
  // zero rows have dot 0 with everything, which the top-2 scan never takes as best or second: no masking needed
  SM_CHECK(cudaMemsetAsync(s.d + (size_t)rows * kDim, 0, (size_t)(padded - rows) * kDim, h->stream));
  SM_CHECK(cudaStreamSynchronize(h->stream));
  s.n = rows;
  return 0;
}

int64_t b200sm_match_capacity(b200sm_handle h, int num_pairs, const int* slot1, const int* slot2) {
  if (!h) return fail(B200SM_ERR_INPUT, "null handle");
  if (num_pairs < 0) return fail(B200SM_ERR_INPUT, "negative number of pairs");
  if (num_pairs > 0 && (!slot1 || !slot2)) return fail(B200SM_ERR_INPUT, "null slot list");
  const int ns = (int)h->slots.size();
  int64_t bound = 0;
  for (int p = 0; p < num_pairs; ++p) {
    if (slot1[p] < 0 || slot1[p] >= ns || slot2[p] < 0 || slot2[p] >= ns)
      return fail(B200SM_ERR_INPUT, "slot out of range in pair " + std::to_string(p));
    const int64_t n1 = h->slots[slot1[p]].n, n2 = h->slots[slot2[p]].n;
    bound += h->o.cross_check ? std::min(n1, n2) : n1;
  }
  return bound;
}

int b200sm_match_pairs(b200sm_handle h, int num_pairs, const int* slot1, const int* slot2, uint64_t* offsets,
                       uint32_t* matches, size_t capacity) {
  if (!h) return fail(B200SM_ERR_INPUT, "null handle");
  if (num_pairs < 0) return fail(B200SM_ERR_INPUT, "negative number of pairs");
  if (!offsets) return fail(B200SM_ERR_INPUT, "null offsets");
  const int64_t bound = b200sm_match_capacity(h, num_pairs, slot1, slot2);
  if (bound < 0) return (int)bound;
  if (bound > 0 && !matches) return fail(B200SM_ERR_INPUT, "null matches");
  if ((uint64_t)capacity < (uint64_t)bound)
    return fail(B200SM_ERR_INPUT, "capacity " + std::to_string(capacity) + " is below the bound " + std::to_string(bound));
  const bool cc = h->o.cross_check != 0;

  // the work lists, on the host
  std::vector<ScanItem> items;
  std::vector<PairItem> pairs(num_pairs);
  int64_t rows = 0, base = 0;
  for (int p = 0; p < num_pairs; ++p) {
    const Slot &s1 = h->slots[slot1[p]], &s2 = h->slots[slot2[p]];
    PairItem& q = pairs[p];
    q.n1 = (int)s1.n; q.n2 = (int)s2.n; q.base = base;
    q.m12 = q.m21 = -1;
    if (s1.n == 0 || s2.n == 0) continue;
    base += cc ? std::min(s1.n, s2.n) : s1.n;
    for (int dir = 0; dir < (cc ? 2 : 1); ++dir) {
      const Slot& qa = dir ? s2 : s1;
      const Slot& qb = dir ? s1 : s2;
      (dir ? q.m21 : q.m12) = rows;
      for (int64_t r0 = 0; r0 < qa.n; r0 += kStrip)
        items.push_back({qa.d + (size_t)r0 * kDim, qb.d, rows + r0,
                         (int)std::min<int64_t>(kStrip, qa.n - r0), (int)((qb.n + kTile - 1) / kTile)});
      rows += qa.n;
    }
  }
  if (rows > B200SM_MAX_ROWS_PER_CALL)
    return fail(B200SM_ERR_TOO_LARGE, "the pairs of one call hold more than B200SM_MAX_ROWS_PER_CALL rows");
  offsets[0] = 0;
  if (num_pairs == 0) return 0;

  if (use_device(h)) return B200SM_ERR_CUDA;
  SM_CHECK(h->m.reserve((size_t)rows));
  SM_CHECK(h->items.reserve(items.size()));
  SM_CHECK(h->pairs.reserve((size_t)num_pairs));
  SM_CHECK(h->scratch.reserve((size_t)bound));
  SM_CHECK(h->out.reserve((size_t)bound));
  SM_CHECK(h->counts.reserve((size_t)num_pairs));
  SM_CHECK(h->offsets.reserve((size_t)num_pairs + 1));

  cudaStream_t st = h->stream;
  SM_CHECK(cudaMemcpyAsync(h->items.p, items.data(), sizeof(ScanItem) * items.size(), cudaMemcpyHostToDevice, st));
  SM_CHECK(cudaMemcpyAsync(h->pairs.p, pairs.data(), sizeof(PairItem) * pairs.size(), cudaMemcpyHostToDevice, st));
  SM_CHECK(cudaEventRecord(h->ev[0], st));
  if (!items.empty()) {
    sm_scan_kernel<<<(unsigned)items.size(), kThreads, kScanSmem, st>>>(h->items.p, h->acos_tab, (float)h->o.max_ratio,
                                                                       (float)h->o.max_distance, h->m.p);
    SM_CHECK(cudaGetLastError());
  }
  SM_CHECK(cudaEventRecord(h->ev[1], st));
  return finish_pairs(h, num_pairs, bound, offsets, matches);
}

}  // extern "C"

// After the scan: the cross-check and compaction, the offsets and the gather, the copies back and the timings.
static int finish_pairs(b200sm_handle h, int num_pairs, int64_t bound, uint64_t* offsets, uint32_t* matches) {
  cudaStream_t st = h->stream;
  sm_compact_kernel<<<num_pairs, 1024, 0, st>>>(h->pairs.p, h->m.p, h->scratch.p, h->counts.p);
  SM_CHECK(cudaGetLastError());
  sm_offsets_kernel<<<1, 1024, 0, st>>>(h->counts.p, num_pairs, h->offsets.p);
  SM_CHECK(cudaGetLastError());
  sm_gather_kernel<<<num_pairs, 256, 0, st>>>(h->pairs.p, h->scratch.p, h->counts.p, h->offsets.p, h->out.p);
  SM_CHECK(cudaGetLastError());
  static_assert(sizeof(unsigned long long) == sizeof(uint64_t), "offsets are 64-bit");
  SM_CHECK(cudaMemcpyAsync(offsets, h->offsets.p, sizeof(uint64_t) * ((size_t)num_pairs + 1), cudaMemcpyDeviceToHost, st));
  SM_CHECK(cudaStreamSynchronize(st));
  const uint64_t total = offsets[num_pairs];
  if (total > (uint64_t)bound) return fail(B200SM_ERR_CUDA, "internal: more matches than the bound");
  if (total > 0) SM_CHECK(cudaMemcpyAsync(matches, h->out.p, sizeof(uint2) * total, cudaMemcpyDeviceToHost, st));
  SM_CHECK(cudaEventRecord(h->ev[2], st));
  SM_CHECK(cudaStreamSynchronize(st));
  float a = 0, b = 0;
  SM_CHECK(cudaEventElapsedTime(&a, h->ev[0], h->ev[1]));
  SM_CHECK(cudaEventElapsedTime(&b, h->ev[0], h->ev[2]));
  h->scan_ms = a; h->total_ms = b;
  return 0;
}

extern "C" {

int b200sm_last_timing(b200sm_handle h, double* scan_ms, double* total_ms) {
  if (!h) return fail(B200SM_ERR_INPUT, "null handle");
  if (scan_ms) *scan_ms = h->scan_ms;
  if (total_ms) *total_ms = h->total_ms;
  return 0;
}

// ---------------------------------------------------------------------------------------------- guided matching
static const int kModelParams[18] = {3, 4, 4, 5, 8, 8, 12, 5, 4, 5, 12, 16, 4, 5, 3, 4, 6, 2};

int b200sm_cam_ray_from_img_with_jac(int model_id, const double* params, const double* xy, double* out9) {
  if (model_id < 0 || model_id > 17) return fail(B200SM_ERR_INPUT, "unknown camera model " + std::to_string(model_id));
  if (!params || !xy || !out9) return fail(B200SM_ERR_INPUT, "null argument");
  return sm_cam_ray_with_jac(model_id, params, xy[0], xy[1], out9) ? 1 : 0;
}

int b200sm_set_keypoints(b200sm_handle h, int slot, int64_t n, const float* xy) {
  if (!h) return fail(B200SM_ERR_INPUT, "null handle");
  if (slot < 0 || slot >= (int)h->slots.size()) return fail(B200SM_ERR_INPUT, "slot out of range");
  if (n < 0) return fail(B200SM_ERR_INPUT, "negative number of keypoints");
  if (n > 0 && !xy) return fail(B200SM_ERR_INPUT, "null keypoints");
  Slot& s = h->slots[slot];
  if (use_device(h)) return B200SM_ERR_CUDA;
  s.n_kp = -1; s.has_camera = false;
  const int64_t rows = std::min<int64_t>(n, h->o.max_num_matches);
  s.kp.assign(xy, xy + 2 * rows);
  SM_CHECK(s.xy.reserve((size_t)std::max<int64_t>(rows, 1)));
  if (rows > 0) SM_CHECK(cudaMemcpy(s.xy.p, xy, sizeof(float2) * (size_t)rows, cudaMemcpyHostToDevice));
  s.n_kp = n;
  return 0;
}

int b200sm_set_camera(b200sm_handle h, int slot, int model_id, const double* params) {
  if (!h) return fail(B200SM_ERR_INPUT, "null handle");
  if (slot < 0 || slot >= (int)h->slots.size()) return fail(B200SM_ERR_INPUT, "slot out of range");
  if (model_id < 0 || model_id > 17) return fail(B200SM_ERR_INPUT, "unknown camera model " + std::to_string(model_id));
  if (!params) return fail(B200SM_ERR_INPUT, "null camera parameters");
  Slot& s = h->slots[slot];
  if (s.n_kp < 0) return fail(B200SM_ERR_INPUT, "the slot has no keypoints");
  if (use_device(h)) return B200SM_ERR_CUDA;
  s.has_camera = false;
  double p[16] = {};
  memcpy(p, params, sizeof(double) * kModelParams[model_id]);
  const int64_t rows = (int64_t)s.kp.size() / 2;
  std::vector<double> geo((size_t)std::max<int64_t>(rows, 1) * kGeo, 0.0);
  for (int64_t r = 0; r < rows; ++r)
    geo[r * kGeo + 9] = sm_cam_ray_with_jac(model_id, p, (double)s.kp[2 * r], (double)s.kp[2 * r + 1], &geo[r * kGeo]) ? 1.0 : 0.0;
  SM_CHECK(s.geo.reserve(geo.size()));
  SM_CHECK(cudaMemcpy(s.geo.p, geo.data(), sizeof(double) * geo.size(), cudaMemcpyHostToDevice));
  s.has_camera = true;
  return 0;
}

int b200sm_match_guided_pairs(b200sm_handle h, int num_pairs, const int* slot1, const int* slot2,
                              const b200sm_guided_geometry* g, uint64_t* offsets, uint32_t* matches, size_t capacity) {
  if (!h) return fail(B200SM_ERR_INPUT, "null handle");
  if (num_pairs < 0) return fail(B200SM_ERR_INPUT, "negative number of pairs");
  if (!offsets) return fail(B200SM_ERR_INPUT, "null offsets");
  if (num_pairs > 0 && !g) return fail(B200SM_ERR_INPUT, "null geometry list");
  const int64_t bound = b200sm_match_capacity(h, num_pairs, slot1, slot2);
  if (bound < 0) return (int)bound;
  if (bound > 0 && !matches) return fail(B200SM_ERR_INPUT, "null matches");
  if ((uint64_t)capacity < (uint64_t)bound)
    return fail(B200SM_ERR_INPUT, "capacity " + std::to_string(capacity) + " is below the bound " + std::to_string(bound));
  for (int p = 0; p < num_pairs; ++p) {
    const std::string at = " in pair " + std::to_string(p);
    const int type = g[p].type;
    if (type < B200SM_GUIDED_NONE || type > B200SM_GUIDED_H) return fail(B200SM_ERR_INPUT, "unknown geometry type" + at);
    if (type == B200SM_GUIDED_NONE) continue;
    if (!std::isfinite(g[p].max_error) || g[p].max_error < 0)
      return fail(B200SM_ERR_INPUT, "max_error must be finite and >= 0" + at);
    for (const int sl : {slot1[p], slot2[p]}) {
      const Slot& s = h->slots[sl];
      if (s.n_kp < 0) return fail(B200SM_ERR_INPUT, "slot " + std::to_string(sl) + " has no keypoints" + at);
      if (type == B200SM_GUIDED_E && !s.has_camera)
        return fail(B200SM_ERR_INPUT, "slot " + std::to_string(sl) + " has no camera" + at);
      if (s.n_kp != s.n_desc)
        return fail(B200SM_ERR_INPUT, "slot " + std::to_string(sl) + " has " + std::to_string(s.n_kp) +
                                          " keypoints and " + std::to_string(s.n_desc) + " descriptors" + at);
    }
  }
  const bool cc = h->o.cross_check != 0;
  auto scanned = [&](int p) {
    return g[p].type != B200SM_GUIDED_NONE && h->slots[slot1[p]].n > 0 && h->slots[slot2[p]].n > 0;
  };
  int64_t total_rows = 0;
  for (int p = 0; p < num_pairs; ++p)
    if (scanned(p)) total_rows += h->slots[slot1[p]].n + (cc ? h->slots[slot2[p]].n : 0);
  if (total_rows > B200SM_MAX_ROWS_PER_CALL)
    return fail(B200SM_ERR_TOO_LARGE, "the pairs of one call hold more than B200SM_MAX_ROWS_PER_CALL rows");

  // the work lists, on the host.  A slot is marked as holding its norms only once their kernel is launched, so that
  // no refusal or failure below leaves a slot marked without them.
  std::vector<GuidedItem> items;
  std::vector<GuidedPair> gp(num_pairs);
  std::vector<PairItem> pairs(num_pairs);
  std::vector<int> need_norms;
  std::vector<char> queued(h->slots.size(), 0);
  int64_t rows = 0, base = 0;
  for (int p = 0; p < num_pairs; ++p) {
    Slot &s1 = h->slots[slot1[p]], &s2 = h->slots[slot2[p]];
    PairItem& q = pairs[p];
    q.n1 = q.n2 = 0; q.base = base;
    q.m12 = q.m21 = -1;
    if (!scanned(p)) continue;
    q.n1 = (int)s1.n; q.n2 = (int)s2.n;
    GuidedPair& G = gp[p];
    G.type = g[p].type;
    G.xy1 = s1.xy.p; G.xy2 = s2.xy.p; G.geo1 = s1.geo.p; G.geo2 = s2.geo.p;
    for (int k = 0; k < 9; ++k) { G.Md[k] = g[p].M[k]; G.Mf[k] = (float)g[p].M[k]; }
    const double thr = g[p].max_error * g[p].max_error;
    G.thr_d = thr; G.thr_f = (float)thr;
    for (const int sl : {slot1[p], slot2[p]})
      if (!h->slots[sl].norms_ok && !queued[sl]) { need_norms.push_back(sl); queued[sl] = 1; }
    base += cc ? std::min(s1.n, s2.n) : s1.n;
    for (int dir = 0; dir < (cc ? 2 : 1); ++dir) {
      const Slot& qa = dir ? s2 : s1;
      const Slot& qb = dir ? s1 : s2;
      (dir ? q.m21 : q.m12) = rows;
      for (int64_t r0 = 0; r0 < qa.n; r0 += kStrip) {
        GuidedItem it;
        it.s = {qa.d + (size_t)r0 * kDim, qb.d, rows + r0, (int)std::min<int64_t>(kStrip, qa.n - r0),
                (int)((qb.n + kTile - 1) / kTile)};
        it.na = nullptr; it.nb = nullptr;   // set below, once the norm buffers exist
        it.pair = p; it.dir = dir; it.r0 = (int)r0; it.n2 = (int)qb.n;
        items.push_back(it);
      }
      rows += qa.n;
    }
  }
  offsets[0] = 0;
  if (num_pairs == 0) return 0;

  if (use_device(h)) return B200SM_ERR_CUDA;
  cudaStream_t st = h->stream;
  for (const int sl : need_norms) {
    Slot& s = h->slots[sl];
    const int64_t padded = (s.n + kTile - 1) / kTile * kTile;
    SM_CHECK(s.norms.reserve((size_t)padded));
    sm_norms_kernel<<<(unsigned)((padded + 255) / 256), 256, 0, st>>>(s.d, padded, s.norms.p);
    SM_CHECK(cudaGetLastError());
    s.norms_ok = true;
  }
  for (GuidedItem& it : items) {
    const int p = it.pair;
    const Slot &s1 = h->slots[slot1[p]], &s2 = h->slots[slot2[p]];
    it.na = (it.dir ? s2 : s1).norms.p + it.r0;
    it.nb = (it.dir ? s1 : s2).norms.p;
  }
  SM_CHECK(h->m.reserve((size_t)rows));
  SM_CHECK(h->gitems.reserve(items.size()));
  SM_CHECK(h->gpairs.reserve((size_t)num_pairs));
  SM_CHECK(h->pairs.reserve((size_t)num_pairs));
  SM_CHECK(h->scratch.reserve((size_t)bound));
  SM_CHECK(h->out.reserve((size_t)bound));
  SM_CHECK(h->counts.reserve((size_t)num_pairs));
  SM_CHECK(h->offsets.reserve((size_t)num_pairs + 1));

  SM_CHECK(cudaMemcpyAsync(h->gitems.p, items.data(), sizeof(GuidedItem) * items.size(), cudaMemcpyHostToDevice, st));
  SM_CHECK(cudaMemcpyAsync(h->gpairs.p, gp.data(), sizeof(GuidedPair) * gp.size(), cudaMemcpyHostToDevice, st));
  SM_CHECK(cudaMemcpyAsync(h->pairs.p, pairs.data(), sizeof(PairItem) * pairs.size(), cudaMemcpyHostToDevice, st));
  SM_CHECK(cudaEventRecord(h->ev[0], st));
  if (!items.empty()) {
    // FindBestMatchesOneWayIndex's threshold, kSqSiftDescriptorNorm * max_distance * max_distance in fp32
    const float md = (float)h->o.max_distance, max_l2 = (kSqNorm * md) * md;
    sm_guided_kernel<<<(unsigned)items.size(), kThreads, kScanSmem, st>>>(h->gitems.p, h->gpairs.p,
                                                                         (float)h->o.max_ratio, max_l2, h->m.p);
    SM_CHECK(cudaGetLastError());
  }
  SM_CHECK(cudaEventRecord(h->ev[1], st));
  return finish_pairs(h, num_pairs, bound, offsets, matches);
}

void b200sm_destroy(b200sm_handle h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (Slot& s : h->slots) s.release();
  h->items.release(); h->pairs.release(); h->gitems.release(); h->gpairs.release(); h->m.release(); h->scratch.release(); h->out.release();
  h->counts.release(); h->offsets.release();
  if (h->acos_tab) cudaFree(h->acos_tab);
  for (cudaEvent_t e : h->ev) if (e) cudaEventDestroy(e);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

}  // extern "C"
