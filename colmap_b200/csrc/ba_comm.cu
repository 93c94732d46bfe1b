// ba_comm.cu — the collectives of the point-sharded multi-GPU solve and the b200ba_comm_* C ABI.
// NCCL binding: libnccl is resolved at run time with dlopen so that the library also loads where NCCL is absent;
// whichever libnccl.so.2 the process already holds (e.g. torch's) is reused.
#include <dlfcn.h>

#include "ba_common.cuh"

struct BaNccl {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
static BaNccl& ba_nccl() {
  static BaNccl n;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (h) {
      n.GetUniqueId = (decltype(n.GetUniqueId))dlsym(h, "ncclGetUniqueId");
      n.CommInitRank = (decltype(n.CommInitRank))dlsym(h, "ncclCommInitRank");
      n.AllReduce = (decltype(n.AllReduce))dlsym(h, "ncclAllReduce");
      n.CommDestroy = (decltype(n.CommDestroy))dlsym(h, "ncclCommDestroy");
      n.GroupStart = (decltype(n.GroupStart))dlsym(h, "ncclGroupStart");
      n.GroupEnd = (decltype(n.GroupEnd))dlsym(h, "ncclGroupEnd");
      n.GetErrorString = (decltype(n.GetErrorString))dlsym(h, "ncclGetErrorString");
      n.ok = n.GetUniqueId && n.CommInitRank && n.AllReduce && n.CommDestroy && n.GroupStart && n.GroupEnd;
    }
  }
  return n;
}
// ---- one-shot all-reduce over NVLink peer memory -------------------------------------------------------------------------
// The collectives of a sharded solve are tiny (the camera-side vector of a PCG iteration is a few thousand doubles) and
// latency-bound.  Every rank owns a symmetric buffer (cudaMalloc + cudaIpc*MemHandle, mapped by every peer once per
// communicator) of 16-byte cells  cell[2 parities][world][cap] = {lo32, seq, hi32, seq}:  a double travels as two 8-byte
// words that each carry the sequence number of the collective, so the data is its own arrival flag (the "LL" idea: no
// fence, no separate flag, one NVLink one-way latency).  One kernel launch per collective: every thread PUSHES its
// elements of the local partial into cell[parity][rank][i] of every peer (posted 16-byte stores; 8-byte halves are
// delivered whole), then spins on the world cells of the same elements in its own buffer and combines them in rank order
// - all ranks produce bit-identical results, like ncclAllReduce.  The sequence number lives in device memory and only
// advances when the kernel really ran (the PCG launches behind a converged solve return early on every rank alike).
// Two parities suffice: a rank can be at most one collective ahead of a peer, because finishing collective s+1 needs
// that peer's cells of s+1, which it only sends after it has consumed collective s.
enum { BA_RED_F64_SUM = 0, BA_RED_F64_MAX = 1, BA_RED_I32_MAX = 2 };
struct BaP2PSeg { void* ptr; int count; int kind; };
struct BaP2PArgs {
  BaP2PSeg seg[3];
  int nseg, total, rank, world;
  unsigned long long cap;                 // cells per (parity, rank)
  char* peer[BA_P2P_MAX_WORLD];           // base of every rank's symmetric buffer as mapped here (peer[rank] = own)
  unsigned long long* state;              // local: [0] sequence, [1] finished-CTA counter, [2] time-out flag
  const int* done;                        // optional: skip when *done (identical on all ranks)
};
__device__ __forceinline__ uint4* ba_p2p_cell(char* base, int world, unsigned long long cap, int parity, int r) {
  return (uint4*)base + ((size_t)parity * world + r) * cap;
}
__global__ void __launch_bounds__(256) ba_p2p_allreduce_kernel(const BaP2PArgs A) {
  if (A.done && *A.done) return;
  if (*(volatile unsigned long long*)&A.state[2]) return;   // an earlier collective timed out: the solve is lost, do not wait again
  const unsigned long long seq64 = *(volatile unsigned long long*)&A.state[0] + 1;
  const unsigned seq = (unsigned)seq64;
  const int parity = (int)(seq64 & 1);
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < A.total; i += stride) {
    int s = 0, j = i;
    while (s + 1 < A.nseg && j >= A.seg[s].count) { j -= A.seg[s].count; ++s; }
    const int kind = A.seg[s].kind;
    const double v = kind == BA_RED_I32_MAX ? (double)((const int*)A.seg[s].ptr)[j] : ((const double*)A.seg[s].ptr)[j];
    const unsigned lo = (unsigned)__double2loint(v), hi = (unsigned)__double2hiint(v);
    for (int r = 0; r < A.world; ++r) {
      uint4* c = ba_p2p_cell(A.peer[r], A.world, A.cap, parity, A.rank) + i;
      asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" :: "l"(c), "r"(lo), "r"(seq), "r"(hi), "r"(seq) : "memory");
    }
    double acc = 0.0;
    const long long t0 = clock64();
    for (int r = 0; r < A.world; ++r) {
      const uint4* c = ba_p2p_cell(A.peer[A.rank], A.world, A.cap, parity, r) + i;
      unsigned a, fa, b, fb;
      for (;;) {
        asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(fa), "=r"(b), "=r"(fb) : "l"(c) : "memory");
        if (fa == seq && fb == seq) break;
        if (clock64() - t0 > 120000000000LL) { A.state[2] = 1; break; }   // ~60 s: a peer died; the host reports it
      }
      const double w = __hiloint2double((int)b, (int)a);
      acc = r == 0 ? w : (kind == BA_RED_F64_SUM ? acc + w : fmax(acc, w));
    }
    if (kind == BA_RED_I32_MAX) ((int*)A.seg[s].ptr)[j] = (int)acc; else ((double*)A.seg[s].ptr)[j] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&A.state[1], 1ULL) == gridDim.x - 1) { A.state[1] = 0; __threadfence(); *(volatile unsigned long long*)&A.state[0] = seq64; }
  }
}

static void ba_p2p_teardown(b200ba_comm* c) {
  BaP2P& P = c->p2p;
  for (int r = 0; r < BA_P2P_MAX_WORLD; ++r) if (P.peer[r] && r != c->rank) cudaIpcCloseMemHandle(P.peer[r]);
  if (P.local) cudaFree(P.local);
  if (P.state) cudaFree(P.state);
  P = BaP2P();
}
// Collective (every rank calls it with the same `need`): maps the symmetric buffers.  Any failure leaves ok = false and
// the solve keeps using NCCL for its collectives.
void ba_p2p_ensure(b200ba_comm* c, size_t need_doubles, cudaStream_t st) {
  BaP2P& P = c->p2p;
  if (P.tried && (!P.ok || need_doubles <= P.cap)) return;
  if (P.tried) { cudaStreamSynchronize(st); ba_p2p_teardown(c); }
  P.tried = true;
  if (c->world > BA_P2P_MAX_WORLD || getenv("B200BA_NO_P2P")) return;
  const size_t cap = std::max<size_t>((need_doubles + 1023) & ~(size_t)1023, 64 * 1024);
  const size_t bytes = sizeof(uint4) * 2 * c->world * cap;
  int good = 1;
  cudaIpcMemHandle_t mine;
  memset(&mine, 0, sizeof(mine));
  if (cudaMalloc(&P.local, bytes) != cudaSuccess) { P.local = nullptr; good = 0; }
  if (good && cudaMalloc(&P.state, 4 * sizeof(unsigned long long)) != cudaSuccess) { P.state = nullptr; good = 0; }
  if (good && (cudaMemsetAsync(P.local, 0, bytes, st) != cudaSuccess || cudaMemsetAsync(P.state, 0, 4 * sizeof(unsigned long long), st) != cudaSuccess)) good = 0;
  if (good && cudaIpcGetMemHandle(&mine, P.local) != cudaSuccess) good = 0;
  cudaGetLastError();
  // handles (and the "good so far" votes) travel as an all-reduce(sum) of a buffer in which every rank fills its own row
  const int row = (int)(sizeof(cudaIpcMemHandle_t) / sizeof(int)) + 1;
  std::vector<int> h((size_t)row * c->world, 0);
  memcpy(&h[(size_t)row * c->rank], &mine, sizeof(mine));
  h[(size_t)row * c->rank + row - 1] = good;
  int* d = nullptr;
  if (cudaMalloc(&d, sizeof(int) * h.size()) != cudaSuccess) { cudaGetLastError(); return; }   // cannot even vote: peers time out in NCCL, as they would anyway
  cudaMemcpyAsync(d, h.data(), sizeof(int) * h.size(), cudaMemcpyHostToDevice, st);
  ba_nccl().AllReduce(d, d, h.size(), ncclInt32, ncclSum, c->comm, st);
  cudaMemcpyAsync(h.data(), d, sizeof(int) * h.size(), cudaMemcpyDeviceToHost, st);
  cudaStreamSynchronize(st);
  for (int r = 0; r < c->world; ++r) good &= h[(size_t)row * r + row - 1];
  int opened = good;
  if (good) {
    for (int r = 0; r < c->world && opened; ++r) {
      if (r == c->rank) { P.peer[r] = P.local; continue; }
      cudaIpcMemHandle_t hd;
      memcpy(&hd, &h[(size_t)row * r], sizeof(hd));
      void* q = nullptr;
      if (cudaIpcOpenMemHandle(&q, hd, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); opened = 0; }
      else P.peer[r] = (char*)q;
    }
  }
  // second vote: everybody mapped everybody (also the barrier that orders the memsets before the first push)
  cudaMemcpyAsync(d, &opened, sizeof(int), cudaMemcpyHostToDevice, st);
  ba_nccl().AllReduce(d, d, 1, ncclInt32, ncclMin, c->comm, st);
  cudaMemcpyAsync(&opened, d, sizeof(int), cudaMemcpyDeviceToHost, st);
  cudaStreamSynchronize(st);
  cudaFree(d);
  if (!opened) { ba_p2p_teardown(c); P.tried = true; return; }
  P.cap = cap; P.bytes = bytes; P.ok = true;
}

cudaError_t BaReducer::flush() {
  if (pending.empty()) return cudaSuccess;
  size_t total = 0;
  bool p2p = comm->p2p.ok && pending.size() <= 3;
  for (const Red& r : pending) {
    total += r.count;
    const bool f64 = r.dt == ncclDouble && (r.op == ncclSum || r.op == ncclMax), i32 = r.dt == ncclInt32 && r.op == ncclMax;
    if (!f64 && !i32) p2p = false;
  }
  if (p2p && (total > comm->p2p.cap || total * sizeof(double) > BA_P2P_MAX_BYTES)) p2p = false;
  if (p2p) {
    BaP2PArgs A;
    memset(&A, 0, sizeof(A));
    for (size_t i = 0; i < pending.size(); ++i) {
      const Red& r = pending[i];
      A.seg[i].ptr = r.buf; A.seg[i].count = (int)r.count;
      A.seg[i].kind = r.dt == ncclInt32 ? BA_RED_I32_MAX : (r.op == ncclSum ? BA_RED_F64_SUM : BA_RED_F64_MAX);
    }
    A.nseg = (int)pending.size(); A.total = (int)total; A.rank = comm->rank; A.world = comm->world; A.cap = comm->p2p.cap;
    for (int r = 0; r < comm->world; ++r) A.peer[r] = comm->p2p.peer[r];
    A.state = comm->p2p.state; A.done = pending[0].done;
    const int ctas = (int)std::min<size_t>(2 * (size_t)sms, std::max<size_t>(1, (total + 255) / 256));   // all CTAs resident: they wait for each other's peers
    ba_p2p_allreduce_kernel<<<ctas, 256, 0, st>>>(A);
    ++launches;
    pending.clear();
    return cudaGetLastError();
  }
  ncclResult_t res = ncclSuccess;
  if (pending.size() > 1) ba_nccl().GroupStart();
  for (const Red& r : pending) { const ncclResult_t q = ba_nccl().AllReduce(r.buf, r.buf, r.count, r.dt, r.op, comm->comm, st); if (q != ncclSuccess) res = q; }
  if (pending.size() > 1) ba_nccl().GroupEnd();
  pending.clear();
  return res == ncclSuccess ? cudaSuccess : cudaErrorUnknown;
}

extern "C" {

int b200ba_comm_unique_id(void* id128) {
  if (!ba_nccl().ok) return ba_fail(-110, "libnccl not available");
  ncclUniqueId id;
  if (ba_nccl().GetUniqueId(&id) != ncclSuccess) return ba_fail(-110, "ncclGetUniqueId failed");
  memcpy(id128, &id, sizeof(id));
  return 0;
}
int b200ba_comm_init(const void* id128, int rank, int world, b200ba_comm_t* out) {
  if (!ba_nccl().ok) return ba_fail(-110, "libnccl not available");
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  b200ba_comm* c = new b200ba_comm();
  c->rank = rank; c->world = world;
  const ncclResult_t r = ba_nccl().CommInitRank(&c->comm, world, id, rank);
  if (r != ncclSuccess) { delete c; return ba_fail(-110, std::string("ncclCommInitRank: ") + (ba_nccl().GetErrorString ? ba_nccl().GetErrorString(r) : "error")); }
  *out = c;
  return 0;
}
int b200ba_comm_peer_memory(b200ba_comm_t c) { return c && c->p2p.ok ? 1 : 0; }
void b200ba_comm_destroy(b200ba_comm_t c) {
  if (!c) return;
  ba_p2p_teardown(c);
  if (c->comm) ba_nccl().CommDestroy(c->comm);
  delete c;
}

}  // extern "C"
