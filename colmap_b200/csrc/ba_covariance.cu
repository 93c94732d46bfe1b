// ba_covariance.cu — covariance of a solved problem (include/b200_ba_covariance.h; EstimateBACovariance,
// src/colmap/estimators/covariance.cc; DESIGN.md §3).  The solve's flattening and device set-up are reused as they
// are; the Jacobian is re-evaluated in fp64 (no Jacobi scaling) and never stored in fp32.  S = H_cc - H_cp
// (H_pp + damping I)^-1 H_pc over the camera-side rows that the reference keeps, ordered [others (sensor_from_rig, intrinsics) | poses], then one dense Cholesky and S^-1 in place (ba_dense_f64.cu).
// With the others first, the pivots of the pose rows are those of S_cc - S_co S_oo^-1 S_oc, so damping the others'
// diagonal and factorising once is SchurEliminateOtherParams followed by the reference's rank test on the pose matrix,
// provided the rank test starts at the first pose row: the others' rows fail only on a pivot <= 0, as the reference's
// LLT of S_oo + damping I does (a weakly determined intrinsic is eliminated, not reported).
#include <chrono>
#include <memory>

#include "ba_common.cuh"
#include "ba_dense_f64.h"

#define BA_COV_MAX_N 32768
struct BaCov {
  double* J;          // [2*DC + 6][nslots]: fp64 rows of every slot, camera side (2 x DC) then point side (2 x 3)
  const int* colmap;  // [nc] camera-side column -> row of S, or -1 (masked dimension, or not estimated)
  double* S; long long N;   // padded dense matrix, lower triangle: element (i, j), i >= j, at S[j * N + i]
  double* pcov;       // [9 * nvpt] (H_pp + damping I)^-1 of every variable point, or null
  double damping;
  int want_S;
};
template <int DC, bool WIDE>
__global__ void __launch_bounds__(BA_BLOCK) ba_cov_linearize_kernel(const BaDev D, const BaCov C) {
  const long long s = (long long)blockIdx.x * BA_BLOCK + threadIdx.x;
  if (s >= D.nslots) return;
  const int pi = D.s_pose[s];
  double Jc[2 * DC], Jpt[6], rr[2];
  if (pi >= 0) {
    ba_obs_linearize<DC, WIDE>(D, D.poses, D.cams, D.pts, pi, D.s_cam[s], D.s_pt[s], D.s_lpt[s], D.s_xy[s], D.s_xy[D.nslots + s], 0,
                               Jc, Jpt, rr);
  } else {
    for (int k = 0; k < 2 * DC; ++k) Jc[k] = 0.0;
    for (int k = 0; k < 6; ++k) Jpt[k] = 0.0;
  }
  for (int k = 0; k < 2 * DC; ++k) C.J[k * D.nslots + s] = Jc[k];
  for (int k = 0; k < 6; ++k) C.J[(2 * DC + k) * D.nslots + s] = Jpt[k];
}
// the rows of S that the DC camera-side columns of slot s map to (-1: none)
template <int DC>
__device__ __forceinline__ void ba_cov_slot_rows(const BaDev& D, const BaCov& C, long long s, double* J0, double* J1, int* idx) {
  const int pi = D.s_pose[s];
  const int po = pi >= 0 ? D.pose_off[pi] : -1, ci = pi >= 0 ? D.s_cam[s] : 0;
  const int co = pi >= 0 ? D.cam_off[ci] : -1, w = pi >= 0 ? D.cam_width[ci] : 0;
  for (int c = 0; c < DC; ++c) {
    J0[c] = C.J[c * D.nslots + s]; J1[c] = C.J[(DC + c) * D.nslots + s];
    const int col = c < 6 ? (po >= 0 ? po + c : -1) : ((co >= 0 && c - 6 < w) ? co + c - 6 : -1);
    idx[c] = col >= 0 ? C.colmap[col] : -1;
  }
}
// S += J_c^T J_c, one thread per slot (observations of variable and of constant points)
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_cov_gram_kernel(const BaDev D, const BaCov C) {
  const long long s = (long long)blockIdx.x * BA_BLOCK + threadIdx.x;
  if (s >= D.nslots) return;
  double J0[DC], J1[DC];
  int idx[DC];
  ba_cov_slot_rows<DC>(D, C, s, J0, J1, idx);
  for (int r = 0; r < DC; ++r) {
    if (idx[r] < 0) continue;
    for (int c = 0; c < DC; ++c)
      if (idx[c] >= 0 && idx[r] >= idx[c]) atomicAdd(&C.S[(long long)idx[c] * C.N + idx[r]], J0[r] * J0[c] + J1[r] * J1[c]);
  }
}
// One warp per variable point: H_pp + damping I over its track, its inverse (the point block), and
// S -= W_i^T (H_pp + damping I)^-1 W_j over the ordered observation pairs (i, j) of the track, W_o = J_p(o)^T J_c(o)
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_cov_point_kernel(const BaDev D, const BaCov C) {
  const int k = blockIdx.x * (BA_BLOCK / 32) + (threadIdx.x >> 5);
  if (k >= D.nvpt) return;
  const int lane = threadIdx.x & 31;
  const int s0 = D.vpt_s0[k], L = D.vpt_s1[k] - s0;
  const long long ns = D.nslots;
  const double* Jp = C.J + 2 * DC * ns;
  double h[6] = {0, 0, 0, 0, 0, 0};   // xx xy xz yy yz zz
  for (int i = lane; i < L; i += 32) {
    double p[6];
    for (int c = 0; c < 6; ++c) p[c] = Jp[c * ns + s0 + i];
    h[0] += p[0] * p[0] + p[3] * p[3]; h[1] += p[0] * p[1] + p[3] * p[4]; h[2] += p[0] * p[2] + p[3] * p[5];
    h[3] += p[1] * p[1] + p[4] * p[4]; h[4] += p[1] * p[2] + p[4] * p[5]; h[5] += p[2] * p[2] + p[5] * p[5];
  }
  for (int c = 0; c < 6; ++c)
    for (int o = 16; o > 0; o >>= 1) h[c] += __shfl_xor_sync(0xffffffffu, h[c], o);
  h[0] += C.damping; h[3] += C.damping; h[5] += C.damping;
  // symmetric 3x3 inverse by cofactors
  const double c00 = h[3] * h[5] - h[4] * h[4], c01 = h[2] * h[4] - h[1] * h[5], c02 = h[1] * h[4] - h[2] * h[3];
  const double c11 = h[0] * h[5] - h[2] * h[2], c12 = h[1] * h[2] - h[0] * h[4], c22 = h[0] * h[3] - h[1] * h[1];
  const double id = 1.0 / (h[0] * c00 + h[1] * c01 + h[2] * c02);
  const double Hi[9] = {c00 * id, c01 * id, c02 * id, c01 * id, c11 * id, c12 * id, c02 * id, c12 * id, c22 * id};
  if (C.pcov && lane < 9) C.pcov[9 * (long long)k + lane] = Hi[lane];
  if (!C.want_S) return;
  for (long long t = lane; t < (long long)L * L; t += 32) {
    const int i = (int)(t / L), j = (int)(t - (long long)i * L);
    double A0[DC], A1[DC], B0[DC], B1[DC];
    int ia[DC], ib[DC];
    ba_cov_slot_rows<DC>(D, C, s0 + i, A0, A1, ia);
    ba_cov_slot_rows<DC>(D, C, s0 + j, B0, B1, ib);
    double pa[6], pb[6];
    for (int c = 0; c < 6; ++c) { pa[c] = Jp[c * ns + s0 + i]; pb[c] = Jp[c * ns + s0 + j]; }
    double G[3][DC];   // Hinv W_j
    for (int c = 0; c < DC; ++c) {
      const double w0 = pb[0] * B0[c] + pb[3] * B1[c], w1 = pb[1] * B0[c] + pb[4] * B1[c], w2 = pb[2] * B0[c] + pb[5] * B1[c];
      G[0][c] = Hi[0] * w0 + Hi[1] * w1 + Hi[2] * w2;
      G[1][c] = Hi[3] * w0 + Hi[4] * w1 + Hi[5] * w2;
      G[2][c] = Hi[6] * w0 + Hi[7] * w1 + Hi[8] * w2;
    }
    for (int r = 0; r < DC; ++r) {
      if (ia[r] < 0) continue;
      const double v0 = pa[0] * A0[r] + pa[3] * A1[r], v1 = pa[1] * A0[r] + pa[4] * A1[r], v2 = pa[2] * A0[r] + pa[5] * A1[r];
      for (int c = 0; c < DC; ++c)
        if (ib[c] >= 0 && ia[r] >= ib[c]) atomicAdd(&C.S[(long long)ib[c] * C.N + ia[r]], -(v0 * G[0][c] + v1 * G[1][c] + v2 * G[2][c]));
    }
  }
}
// Position priors (b200ba_estimate_covariance_with_position_priors): S += J^T J of each kept prior's weighted,
// loss-corrected, unscaled 3 x 12 rows [pose | sensor], fp64, one thread per prior.  The rows touch camera-side blocks
// only (pose, pose-sensor cross terms, sensor), so the point elimination above is unaffected.  The solve's
// ba_prior_linearize_kernel is not reused: it applies Jacobi scaling and sums the cost into the LM control block.
__global__ void ba_cov_prior_kernel(const BaDev D, const BaPrior P, const BaCov C) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= P.n) return;
  double rw[3], J[36], rho[3];
  ba_prior_eval(D, P, k, D.poses, D.sensors, rw, J);
  const double sq = rw[0] * rw[0] + rw[1] * rw[1] + rw[2] * rw[2];
  ba_loss(P.loss_type, P.loss_scale, sq, rho);
  ba_prior_correct(P, rw, sq, rho, J);
  const int4 ix = P.idx[k];
  int row[12];
  for (int j = 0; j < 12; ++j) {
    const int col = ba_prior_col(ix, j);
    row[j] = col >= 0 ? C.colmap[col] : -1;
  }
  for (int a = 0; a < 12; ++a) {
    if (row[a] < 0) continue;
    for (int b = 0; b < 12; ++b)
      if (row[b] >= 0 && row[a] >= row[b])
        atomicAdd(&C.S[(long long)row[b] * C.N + row[a]], J[a] * J[b] + J[12 + a] * J[12 + b] + J[24 + a] * J[24 + b]);
  }
}
// diagonal: damping on rows [0, n_damp) (the others, eliminated in POSES mode), 1 on the padding rows [n, N)
__global__ void ba_cov_diag_kernel(double* S, long long N, int n, int n_damp, double damping) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_damp) S[i * N + i] += damping;
  else if (i >= n && i < N) S[i * N + i] = 1.0;
}
// blocks {first row, rows, first column, columns} of the symmetric matrix (lower triangle stored) -> out[b * stride], row-major
__global__ void ba_cov_gather_kernel(const double* S, long long N, const int4* blocks, int stride, double* out) {
  const int4 b = blocks[blockIdx.x];
  for (int e = threadIdx.x; e < b.y * b.w; e += blockDim.x) {
    const long long i = b.x + e / b.w, j = b.z + e % b.w;
    out[(long long)blockIdx.x * stride + e] = i >= j ? S[j * N + i] : S[i * N + j];
  }
}
template <int DC>
static void ba_cov_launch_build_dc(const BaDev& D, const BaCov& C, cudaStream_t s) {
  constexpr bool WIDE = DC >= 14;
  ba_cov_linearize_kernel<DC, WIDE><<<D.nblocks, BA_BLOCK, 0, s>>>(D, C);
  if (C.want_S) ba_cov_gram_kernel<DC><<<D.nblocks, BA_BLOCK, 0, s>>>(D, C);
  if (D.nvpt && (C.want_S || C.pcov)) ba_cov_point_kernel<DC><<<(D.nvpt + BA_BLOCK / 32 - 1) / (BA_BLOCK / 32), BA_BLOCK, 0, s>>>(D, C);
}
static void ba_cov_launch_build(const BaDev& D, const BaCov& C, cudaStream_t s) { BA_DISPATCH_DC(ba_cov_launch_build_dc, D, C, s); }

struct b200ba_covariance {
  int dev = 0;
  BaPool pool;                        // S^-1 and the point blocks, until b200ba_covariance_free
  double* S = nullptr; long long N = 0; int n = 0;
  double* pcov = nullptr;
  double* g_out = nullptr; int4* g_blk = nullptr; int g_cap = 0;   // gather scratch of the getters
  std::vector<int> pt_var;            // point -> variable index, or -1
  std::vector<int> pose_row, pose_size, cam_row, cam_size, sens_row, sens_size;   // first row in S and size (0 = none)
  double ms[4] = {0, 0, 0, 0};        // set-up, build, factorisation, inverse
};
struct BaCovStream {                  // destroyed before the work pool releases its blocks
  cudaStream_t st = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  ~BaCovStream() { for (auto e : ev) if (e) cudaEventDestroy(e); if (st) cudaStreamDestroy(st); }
};
// the block of S that row r belongs to, for the "not estimable" message
static std::string ba_cov_row_name(const b200ba_covariance& H, int r) {
  char b[96];
  for (size_t i = 0; i < H.pose_row.size(); ++i)
    if (H.pose_size[i] && r >= H.pose_row[i] && r < H.pose_row[i] + H.pose_size[i]) { snprintf(b, sizeof(b), "pose %zu, tangent row %d", i, r - H.pose_row[i]); return b; }
  for (size_t i = 0; i < H.cam_row.size(); ++i)
    if (H.cam_size[i] && r >= H.cam_row[i] && r < H.cam_row[i] + H.cam_size[i]) { snprintf(b, sizeof(b), "intrinsics of camera %zu, row %d", i, r - H.cam_row[i]); return b; }
  for (size_t i = 0; i < H.sens_row.size(); ++i)
    if (H.sens_size[i] && r >= H.sens_row[i] && r < H.sens_row[i] + H.sens_size[i]) { snprintf(b, sizeof(b), "sensor_from_rig %zu, tangent row %d", i, r - H.sens_row[i]); return b; }
  return "padding";
}
// priors: the position priors the problem was solved with (PosePriorBundleAdjuster), or null
static int ba_cov_impl(const b200ba_options* o, const b200ba_covariance_options* co, const b200ba_problem* p,
                       const b200ba_position_priors* priors, b200ba_covariance_t* out) {
  if (!o || !co || !p || !out) return ba_fail(-1, "null argument");
  *out = nullptr;
  if (co->params < B200BA_COV_POSES || co->params > B200BA_COV_ALL) return ba_fail(-2, "unknown covariance mode");
  if (!(co->damping >= 0.0)) return ba_fail(-2, "damping must be >= 0");
  if (priors && priors->num_priors == 0) priors = nullptr;
  std::vector<double> prior_w;   // checked before any device work
  if (priors) BA_TRY(ba_prior_check(p, priors, prior_w));
  const auto t0 = std::chrono::steady_clock::now();
  BA_TRY(ba_use_device(o));
  const bool want_pts = co->params != B200BA_COV_POSES, want_S = co->params != B200BA_COV_POINTS;
  const bool want_others = co->params == B200BA_COV_ALL;
  BaLayout L;
  b200ba_summary sum = {};
  BA_TRY(ba_flatten(o, p, nullptr, L, &sum));
  std::unique_ptr<b200ba_covariance> H(new b200ba_covariance);
  cudaGetDevice(&H->dev);
  const int NP = p->num_poses, NCAM = p->num_cameras, NS = p->num_sensors;
  H->pose_row.assign(NP, 0); H->pose_size.assign(NP, 0); H->cam_row.assign(NCAM, 0); H->cam_size.assign(NCAM, 0);
  H->sens_row.assign(NS, 0); H->sens_size.assign(NS, 0);
  H->pt_var = L.pt_var;
  if (L.nothing_to_solve) { *out = H.release(); return 0; }
  // rows of S: others first (per camera block: sensor_from_rig, then intrinsics), then the unmasked pose dimensions
  std::vector<int> colmap(L.nc, -1);
  int n = 0, n_others = 0;
  if (want_S) {
    for (int c = 0; c < NCAM; ++c) {
      if (L.cam_off[c] < 0) continue;
      const int ns = L.cam_ns[c], nv = L.cam_nvar[c];
      if (ns) { H->sens_row[L.cam_sensor[c]] = n; H->sens_size[L.cam_sensor[c]] = ns; }
      for (int k = 0; k < ns; ++k) colmap[L.cam_off[c] + k] = n++;
      if (nv) { H->cam_row[c] = n; H->cam_size[c] = nv; }
      for (int k = 0; k < nv; ++k) colmap[L.cam_off[c] + ns + k] = n++;
    }
    n_others = n;
    for (int i = 0; i < NP; ++i) {
      if (L.pose_off[i] < 0) continue;
      H->pose_row[i] = n;
      for (int d = 0; d < 6; ++d) if ((L.pose_mask[i] >> d) & 1) colmap[L.pose_off[i] + d] = n++;
      H->pose_size[i] = n - H->pose_row[i];
    }
  }
  if (n > BA_COV_MAX_N)
    return ba_fail(-3, "covariance: reduced matrix dimension " + std::to_string(n) + " above the dense limit " + std::to_string(BA_COV_MAX_N));
  // the rank test covers the rows the reference tests: all of S in ALL mode, the poses only when the others are eliminated
  const int n_test0 = want_others ? 0 : n_others;
  const long long N = (n + BA_TILE - 1) / BA_TILE * BA_TILE;
  BaPool work;            // the solve's device layout and the scratch of this estimate
  BaCovStream G;
  BA_CUDA(cudaStreamCreateWithFlags(&G.st, cudaStreamNonBlocking));
  for (auto& e : G.ev) BA_CUDA(cudaEventCreate(&e));
  BaPath path = {};       // no reduced-system path: only the layout and the slot arrays are used
  BaDev D;
  BA_TRY(ba_upload(L, o, p, path, nullptr, work, G.st, D));
  BaPrior P;              // the priors only enter S: none are set up when S is not formed (POINTS mode)
  if (priors && n) BA_TRY(ba_prior_setup(priors, prior_w, L, work, G.st, P));
  BaCov C = {};
  C.damping = co->damping; C.want_S = n > 0; C.N = N;
  BA_CUDA(work.alloc(&C.J, (size_t)(2 * L.DC + 6) * (size_t)D.nslots));
  BA_CUDA(work.upload(&C.colmap, colmap, G.st));
  if (want_pts) BA_CUDA(H->pool.alloc(&C.pcov, (size_t)9 * L.nvpt));
  if (n) {
    if (H->pool.alloc(&C.S, (size_t)(N * N)) != cudaSuccess) {
      cudaGetLastError();
      return ba_fail(-3, "covariance: cannot allocate the " + std::to_string(N) + " x " + std::to_string(N) + " fp64 matrix");
    }
    BA_CUDA(cudaMemsetAsync(C.S, 0, sizeof(double) * (size_t)(N * N), G.st));
  }
  BA_CUDA(cudaStreamSynchronize(G.st));
  H->ms[0] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  BA_CUDA(cudaEventRecord(G.ev[0], G.st));
  ba_cov_launch_build(D, C, G.st);
  if (P.n) ba_cov_prior_kernel<<<(P.n + 127) / 128, 128, 0, G.st>>>(D, P, C);
  if (n) ba_cov_diag_kernel<<<(unsigned)((N + 255) / 256), 256, 0, G.st>>>(C.S, N, n, want_others ? 0 : n_others, co->damping);
  BA_CUDA(cudaGetLastError());
  BA_CUDA(cudaEventRecord(G.ev[1], G.st));
  BaDenseFlag flag = {};
  if (n) {
    BaDenseFlag* d_flag; double *dinv, *panel;
    BA_CUDA(work.alloc(&d_flag, 1)); BA_CUDA(work.alloc(&dinv, (size_t)N * BA_TILE)); BA_CUDA(work.alloc(&panel, (size_t)N * BA_TILE));
    BA_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(BaDenseFlag), G.st));
    BA_CUDA(ba_dense_potrf(C.S, (int)N, n_test0, n, 1e-6, dinv, d_flag, G.st));
    BA_CUDA(cudaEventRecord(G.ev[2], G.st));
    BA_CUDA(ba_dense_potri(C.S, (int)N, dinv, panel, d_flag, G.st));
    BA_CUDA(cudaEventRecord(G.ev[3], G.st));
    BA_CUDA(cudaMemcpyAsync(&flag, d_flag, sizeof(flag), cudaMemcpyDeviceToHost, G.st));
  } else {
    BA_CUDA(cudaEventRecord(G.ev[2], G.st)); BA_CUDA(cudaEventRecord(G.ev[3], G.st));
  }
  BA_CUDA(cudaStreamSynchronize(G.st));
  if (flag.bad) {
    char b[160];
    snprintf(b, sizeof(b), "covariance not estimable: pivot %.3g <= %s at row %d of %d of the reduced matrix (", flag.pivot,
             flag.row < n_test0 ? "0" : "1e-6", flag.row, n);
    return ba_fail(1, std::string(b) + ba_cov_row_name(*H, flag.row) + "): the problem has an unfixed gauge or another degeneracy");
  }
  if (!want_others) {   // the others are eliminated: no blocks of their own (the reference's L_inv has no rows for them)
    std::fill(H->cam_size.begin(), H->cam_size.end(), 0); std::fill(H->sens_size.begin(), H->sens_size.end(), 0);
  }
  for (int k = 0; k < 3; ++k) { float ms = 0; BA_CUDA(cudaEventElapsedTime(&ms, G.ev[k], G.ev[k + 1])); H->ms[1 + k] = ms; }
  H->S = C.S; H->N = N; H->n = n; H->pcov = C.pcov;
  H->g_cap = std::max(NP, 1);
  BA_CUDA(H->pool.alloc(&H->g_out, (size_t)36 * H->g_cap + 256)); BA_CUDA(H->pool.alloc(&H->g_blk, (size_t)H->g_cap));
  *out = H.release();
  return 0;
}
// gathers nb blocks (each rows x cols <= stride) of S^-1 into out
static int ba_cov_gather(b200ba_covariance* h, const std::vector<int4>& blocks, int stride, double* out) {
  if (blocks.empty()) return 0;
  BA_CUDA(cudaMemcpy(h->g_blk, blocks.data(), sizeof(int4) * blocks.size(), cudaMemcpyHostToDevice));
  ba_cov_gather_kernel<<<(unsigned)blocks.size(), 256>>>(h->S, h->N, h->g_blk, stride, h->g_out);
  BA_CUDA(cudaGetLastError());
  BA_CUDA(cudaMemcpy(out, h->g_out, sizeof(double) * (size_t)stride * blocks.size(), cudaMemcpyDeviceToHost));
  return 0;
}
// selects the device the estimate lives on; a failure is left in b200ba_last_error
static int ba_cov_use_device(const b200ba_covariance* h) {
  BA_CUDA(cudaSetDevice(h->dev));
  return 0;
}
static int ba_cov_block(b200ba_covariance* h, int r0, int a, int c0, int b, double* out) {
  if (!h || !a || !b || ba_cov_use_device(h)) return 0;
  double tmp[256];
  if (ba_cov_gather(h, {make_int4(r0, a, c0, b)}, 256, tmp)) return 0;
  memcpy(out, tmp, sizeof(double) * a * b);
  return a * b;
}

extern "C" {

// ---- hook for the GPU test tier: the dense kernels alone ----
// ba_dense_potrf and, when invert != 0, ba_dense_potri on the caller's device matrix A (N x N, column-major, lower
// triangle, N a multiple of 64), on the legacy default stream.  Returns 0, 1 after a failed pivot (its row and value in
// bad_row / bad_pivot), or < 0.
int b200ba_test_dense_f64(double* A, int N, int n_test0, int n_check, double pivot_min, int invert, int* bad_row, double* bad_pivot) {
  if (!A || !bad_row || !bad_pivot) return ba_fail(-1, "null argument");
  if (N <= 0 || N % BA_TILE || N > BA_COV_MAX_N) return ba_fail(-2, "N must be a positive multiple of 64 up to 32768");
  BaPool work;
  BaDenseFlag flag = {}, *d_flag;
  double *dinv, *panel;
  BA_CUDA(work.alloc(&d_flag, 1)); BA_CUDA(work.alloc(&dinv, (size_t)N * BA_TILE)); BA_CUDA(work.alloc(&panel, (size_t)N * BA_TILE));
  BA_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(BaDenseFlag), 0));
  BA_CUDA(ba_dense_potrf(A, N, n_test0, n_check, pivot_min, dinv, d_flag, 0));
  if (invert) BA_CUDA(ba_dense_potri(A, N, dinv, panel, d_flag, 0));
  BA_CUDA(cudaMemcpy(&flag, d_flag, sizeof(flag), cudaMemcpyDeviceToHost));
  *bad_row = flag.row; *bad_pivot = flag.pivot;
  return flag.bad ? 1 : 0;
}

// ---- hook for the GPU test tier: the triangular solves alone ----
// ba_dense_potrf (positivity test up to n_check) then ba_dense_potrs on the caller's device matrix A (as above), nrhs
// device columns B (ld N, solved in place) and device scratch W (nrhs * N), on the legacy default stream.  Returns 0,
// 1 after a failed pivot (its row and value in bad_row / bad_pivot; the solve's launches then return at once), or < 0.
int b200ba_test_dense_potrs(double* A, int N, int n_check, int nrhs, double* B, double* W, int* bad_row, double* bad_pivot) {
  if (!A || !B || !W || !bad_row || !bad_pivot) return ba_fail(-1, "null argument");
  if (N <= 0 || N % BA_TILE || N > BA_COV_MAX_N) return ba_fail(-2, "N must be a positive multiple of 64 up to 32768");
  if (nrhs <= 0 || nrhs > 65535) return ba_fail(-3, "nrhs must be in 1..65535");
  BaPool work;
  BaDenseFlag flag = {}, *d_flag;
  double* dinv;
  BA_CUDA(work.alloc(&d_flag, 1)); BA_CUDA(work.alloc(&dinv, (size_t)N * BA_TILE));
  BA_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(BaDenseFlag), 0));
  BA_CUDA(ba_dense_potrf(A, N, n_check, n_check, 0.0, dinv, d_flag, 0));
  BA_CUDA(ba_dense_potrs(A, N, dinv, nrhs, B, W, d_flag, 0));
  BA_CUDA(cudaMemcpy(&flag, d_flag, sizeof(flag), cudaMemcpyDeviceToHost));
  *bad_row = flag.row; *bad_pivot = flag.pivot;
  return flag.bad ? 1 : 0;
}

void b200ba_covariance_options_init(b200ba_covariance_options* c) { c->params = B200BA_COV_ALL; c->damping = 1e-8; }

int b200ba_estimate_covariance(const b200ba_options* o, const b200ba_covariance_options* c, const b200ba_problem* p,
                               b200ba_covariance_t* out) {
  return ba_cov_impl(o, c, p, nullptr, out);
}
int b200ba_estimate_covariance_with_position_priors(const b200ba_options* o, const b200ba_covariance_options* c,
                                                    const b200ba_problem* p, const b200ba_position_priors* priors,
                                                    b200ba_covariance_t* out) {
  return ba_cov_impl(o, c, p, priors, out);
}

int b200ba_covariance_point(b200ba_covariance_t h, int64_t point, double out[9]) {
  if (!h || !h->pcov || point < 0 || point >= (int64_t)h->pt_var.size() || h->pt_var[point] < 0 || ba_cov_use_device(h)) return 0;
  if (cudaMemcpy(out, h->pcov + 9 * (size_t)h->pt_var[point], sizeof(double) * 9, cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
  return 3;
}
int b200ba_covariance_pose(b200ba_covariance_t h, int pose, double out[36]) {
  if (!h || pose < 0 || pose >= (int)h->pose_size.size()) return 0;
  const int s = h->pose_size[pose];
  return ba_cov_block(h, h->pose_row[pose], s, h->pose_row[pose], s, out) ? s : 0;
}
int b200ba_covariance_pose_cross(b200ba_covariance_t h, int pose1, int pose2, double out[36], int* rows, int* cols) {
  if (rows) *rows = 0;
  if (cols) *cols = 0;
  if (!h || pose1 < 0 || pose2 < 0 || pose1 >= (int)h->pose_size.size() || pose2 >= (int)h->pose_size.size()) return 0;
  const int a = h->pose_size[pose1], b = h->pose_size[pose2];
  const int r = ba_cov_block(h, h->pose_row[pose1], a, h->pose_row[pose2], b, out);
  if (r && rows) *rows = a;
  if (r && cols) *cols = b;
  return r;
}
int b200ba_covariance_camera(b200ba_covariance_t h, int camera, double out[256]) {
  if (!h || camera < 0 || camera >= (int)h->cam_size.size()) return 0;
  const int s = h->cam_size[camera];
  return ba_cov_block(h, h->cam_row[camera], s, h->cam_row[camera], s, out) ? s : 0;
}
int b200ba_covariance_sensor(b200ba_covariance_t h, int sensor, double out[36]) {
  if (!h || sensor < 0 || sensor >= (int)h->sens_size.size()) return 0;
  const int s = h->sens_size[sensor];
  return ba_cov_block(h, h->sens_row[sensor], s, h->sens_row[sensor], s, out) ? s : 0;
}
int b200ba_covariance_poses_all(b200ba_covariance_t h, double* out, int8_t* size) {
  if (!h) return ba_fail(-1, "null argument");
  BA_TRY(ba_cov_use_device(h));
  const int NP = (int)h->pose_size.size();
  std::vector<int4> blocks;
  std::vector<int> which;
  for (int i = 0; i < NP; ++i) {
    size[i] = (int8_t)h->pose_size[i];
    if (h->pose_size[i]) { blocks.push_back(make_int4(h->pose_row[i], h->pose_size[i], h->pose_row[i], h->pose_size[i])); which.push_back(i); }
  }
  std::vector<double> g(36 * blocks.size());
  BA_TRY(ba_cov_gather(h, blocks, 36, g.data()));
  memset(out, 0, sizeof(double) * 36 * (size_t)NP);
  for (size_t b = 0; b < which.size(); ++b) memcpy(out + 36 * (size_t)which[b], g.data() + 36 * b, sizeof(double) * 36);
  return 0;
}
int b200ba_covariance_points_all(b200ba_covariance_t h, double* out, uint8_t* valid) {
  if (!h) return ba_fail(-1, "null argument");
  const size_t NPT = h->pt_var.size();
  long long nvpt = 0;
  for (int v : h->pt_var) nvpt = std::max<long long>(nvpt, v + 1);
  std::vector<double> g(9 * (size_t)nvpt);
  if (h->pcov && nvpt) {
    BA_TRY(ba_cov_use_device(h));
    BA_CUDA(cudaMemcpy(g.data(), h->pcov, sizeof(double) * g.size(), cudaMemcpyDeviceToHost));
  }
  for (size_t i = 0; i < NPT; ++i) {
    const int v = h->pcov ? h->pt_var[i] : -1;
    valid[i] = v >= 0 ? 1 : 0;
    if (v >= 0) memcpy(out + 9 * i, g.data() + 9 * (size_t)v, sizeof(double) * 9); else memset(out + 9 * i, 0, sizeof(double) * 9);
  }
  return 0;
}
int b200ba_covariance_info(b200ba_covariance_t h, double* ms4) {
  if (!h) return -1;
  if (ms4) for (int k = 0; k < 4; ++k) ms4[k] = h->ms[k];
  return h->n;
}
void b200ba_covariance_free(b200ba_covariance_t h) {
  if (!h) return;
  ba_cov_use_device(h);   // the device blocks go back to this device's cache
  delete h;
}

}  // extern "C"
