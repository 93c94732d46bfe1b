// solver_host.cuh — host scaffolding shared by the global positioning and rotation averaging solves: the error
// message, grid sizes, the finite check, the owner of a solve's device buffers and events, and the deterministic sum.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <string>
#include <vector>

// Formats the message into err (the module's thread-local last-error string) and returns code.
static inline int solver_fail(std::string& err, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  err = buf;
  return code;
}

// Returns code with the failed call's text and CUDA's message in err.
#define SOLVER_CUDA(err, code, call)                                                                          \
  do {                                                                                                        \
    const cudaError_t e_ = (call);                                                                            \
    if (e_ != cudaSuccess) return solver_fail(err, code, "%s: %s", #call, cudaGetErrorString(e_));          \
  } while (0)
// Propagates a non-zero return code.
#define SOLVER_TRY(call) do { if (const int rc_ = (call)) return rc_; } while (0)

static inline unsigned grid_blocks(int64_t n, int t) { return (unsigned)std::max<int64_t>(1, (n + t - 1) / t); }

static inline bool all_finite(const double* a, int64_t n) {
  for (int64_t i = 0; i < n; ++i) if (!std::isfinite(a[i])) return false;
  return true;
}

// The device buffers and events of one solve.  Plain cudaMalloc, not B200DeviceCache: the dense reduced matrices reach
// several GB at the size limits, and a cache would keep them after the solve.  Everything is freed on every return.
struct SolverBuffers {
  std::vector<void*> ptrs;
  std::vector<cudaEvent_t> events;
  template <typename T> cudaError_t alloc(T** p, size_t n) {
    const cudaError_t e = cudaMalloc((void**)p, std::max<size_t>(sizeof(T) * n, 8));
    if (e == cudaSuccess) ptrs.push_back((void*)*p);
    return e;
  }
  template <typename T> cudaError_t upload(T** p, const std::vector<T>& v) {
    const cudaError_t e = alloc(p, v.size());
    if (e != cudaSuccess || v.empty()) return e;
    return cudaMemcpy(*p, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice);
  }
  template <typename T> cudaError_t upload(const T** p, const std::vector<T>& v) {   // read-only device-struct fields
    return upload(const_cast<T**>(p), v);
  }
  cudaError_t event(cudaEvent_t* ev) {
    const cudaError_t e = cudaEventCreate(ev);
    if (e == cudaSuccess) events.push_back(*ev);
    return e;
  }
  ~SolverBuffers() {
    for (void* q : ptrs) cudaFree(q);
    for (cudaEvent_t ev : events) cudaEventDestroy(ev);
  }
};

// Deterministic sums: a fixed grid of G CTAs, a fixed per-thread order and a fixed tree, so that a sum is bit-identical
// from run to run.  Pass 1 leaves G partial sums in part[0..G), pass 2 adds them into *out.
#define SOLVER_RB 256
enum { SOLVER_SUM = 0,        // sum of a
       SOLVER_SUM_SQDIFF = 1, // sum of (a - b)^2 over the masked terms
       SOLVER_SUM_SQ = 2 };   // sum of a^2 over the masked terms
// mask (may be null): term i counts when mask[i / mstride] is set
template <int G>
__global__ void k_solver_sum1(const double* a, const double* b, const uint8_t* mask, int mstride, int64_t n, int mode,
                              double* part) {
  __shared__ double sh[SOLVER_RB];
  double s = 0;
  for (int64_t i = blockIdx.x * (int64_t)SOLVER_RB + threadIdx.x; i < n; i += (int64_t)G * SOLVER_RB) {
    if (mode && mask && !mask[i / mstride]) continue;
    const double v = mode == SOLVER_SUM_SQDIFF ? a[i] - b[i] : a[i];
    s += mode ? v * v : v;
  }
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = SOLVER_RB / 2; o; o >>= 1) { if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (!threadIdx.x) part[blockIdx.x] = sh[0];
}
template <int G>
__global__ void k_solver_sum2(const double* part, double* out) {
  __shared__ double sh[G];
  for (int i = threadIdx.x; i < G; i += SOLVER_RB) sh[i] = part[i];
  __syncthreads();
  for (int o = G / 2; o; o >>= 1) { for (int i = threadIdx.x; i < o; i += SOLVER_RB) sh[i] += sh[i + o]; __syncthreads(); }
  if (!threadIdx.x) *out = sh[0];
}
// Launches both passes on the legacy default stream; part holds G doubles.
template <int G>
static void solver_sum(int mode, const double* a, const double* b, const uint8_t* mask, int mstride, int64_t n, double* part,
                       double* out) {
  k_solver_sum1<G><<<G, SOLVER_RB>>>(a, b, mask, mstride, n, mode, part);
  k_solver_sum2<G><<<1, SOLVER_RB>>>(part, out);
}
