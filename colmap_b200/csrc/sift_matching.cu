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
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
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

struct Slot {
  uint8_t* d = nullptr;
  int64_t n = 0;
  int64_t cap_rows = 0;
};

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

int b200sm_last_timing(b200sm_handle h, double* scan_ms, double* total_ms) {
  if (!h) return fail(B200SM_ERR_INPUT, "null handle");
  if (scan_ms) *scan_ms = h->scan_ms;
  if (total_ms) *total_ms = h->total_ms;
  return 0;
}

void b200sm_destroy(b200sm_handle h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (Slot& s : h->slots) if (s.d) cudaFree(s.d);
  h->items.release(); h->pairs.release(); h->m.release(); h->scratch.release(); h->out.release();
  h->counts.release(); h->offsets.release();
  if (h->acos_tab) cudaFree(h->acos_tab);
  for (cudaEvent_t e : h->ev) if (e) cudaEventDestroy(e);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

}  // extern "C"
