// rotation_averaging.cu — RotationAveragingSolver::Solve (include/b200_rotation_averaging.h) on the H100 in fp64.
//
// The reference factors the sparse normal matrix A^T D A (+ ridge) of size num_params with CHOLMOD.  Every non-zero of
// A links residual component i of a row triple to parameter component i (a 1-DOF frame's single component and a 1-DOF
// pair's single row are y), and D is constant over a pair's rows, so after a permutation the matrix is
// blockdiag(M_x, M_y, M_z) with M_x = M_z over the 3-DOF blocks (frames, then estimated cameras) and M_y over all
// blocks.  Without 1-DOF frames M_y = M_xz, and one factorisation serves three right-hand sides.  Each matrix is built
// densely, one thread per column through a block -> incident-pair CSR, sums in a fixed order, no atomics, lower
// triangle only; ba_dense_potrf factors it (positivity test only) and ba_dense_potrs solves.
//
// Everything else is per pair (residuals, IRLS weights, A x), per parameter block (A^T v, UpdateState, the step size)
// or per estimated camera (the quaternion average of UpdateState, one CTA each), and every norm is a two-pass
// reduction on a fixed grid, so repeated solves are bit-identical.  Not restated: the random jitter the reference adds to
// a 1-DOF residual within 0.01 of +-pi (ComputeGravityAligned1DOFResidual), and CHOLMOD's fallback to LDL^T when the
// Cholesky factorisation fails, which is reported here as B200RA_FACTORIZATION_FAILED (DESIGN.md, "Rotation averaging").
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/b200_rotation_averaging.h"
#include "ba_dense_f64.h"

static thread_local std::string g_ra_err;
static int ra_fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  g_ra_err = buf;
  return code;
}
extern "C" const char* b200ra_last_error(void) { return g_ra_err.c_str(); }

extern "C" void b200ra_options_init(b200ra_options* o) {
  o->max_num_l1_iterations = 5; o->l1_step_convergence_threshold = 1e-3;
  o->max_num_irls_iterations = 100; o->irls_step_convergence_threshold = 1e-3;
  o->irls_loss_parameter_sigma = 5.0; o->ridge_regularization = 1e-9;
  o->weight_type = B200RA_GEMAN_MCCLURE; o->gpu_index = -1;
}

// ------------------------------------------------------------------------------------------------ rotations
// AngleAxisToRotationMatrix (geometry/pose.cc:137-156: Eigen's AngleAxis above 1e-12, I + [w]x below), row-major
__device__ void ra_exp(const double* w, double* R) {
  const double angle = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  if (angle > 1e-12) {
    const double a[3] = {w[0] / angle, w[1] / angle, w[2] / angle};
    const double s = sin(angle), c = cos(angle);
    const double sa[3] = {s * a[0], s * a[1], s * a[2]}, ca[3] = {(1.0 - c) * a[0], (1.0 - c) * a[1], (1.0 - c) * a[2]};
    double t = ca[0] * a[1]; R[1] = t - sa[2]; R[3] = t + sa[2];
    t = ca[0] * a[2]; R[2] = t + sa[1]; R[6] = t - sa[1];
    t = ca[1] * a[2]; R[5] = t - sa[0]; R[7] = t + sa[0];
    R[0] = ca[0] * a[0] + c; R[4] = ca[1] * a[1] + c; R[8] = ca[2] * a[2] + c;
  } else {
    R[0] = 1; R[3] = w[2]; R[6] = -w[1];
    R[1] = -w[2]; R[4] = 1; R[7] = w[0];
    R[2] = w[1]; R[5] = -w[0]; R[8] = 1;
  }
}

// Eigen's Quaternion from a rotation matrix; q = (x, y, z, w)
__device__ void ra_quat(const double* R, double* q) {
  const double t = R[0] + R[4] + R[8];
  if (t > 0.0) {
    double s = sqrt(t + 1.0);
    q[3] = 0.5 * s; s = 0.5 / s;
    q[0] = (R[7] - R[5]) * s; q[1] = (R[2] - R[6]) * s; q[2] = (R[3] - R[1]) * s;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[3 * i + i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double s = sqrt(R[3 * i + i] - R[3 * j + j] - R[3 * k + k] + 1.0);
    q[i] = 0.5 * s; s = 0.5 / s;
    q[3] = (R[3 * k + j] - R[3 * j + k]) * s;
    q[j] = (R[3 * j + i] + R[3 * i + j]) * s;
    q[k] = (R[3 * k + i] + R[3 * i + k]) * s;
  }
}

// RotationMatrixToAngleAxis of a quaternion (Eigen's AngleAxis(Quaternion))
__device__ void ra_log_quat(const double* q, double* w) {
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
  if (n != 0.0) {
    const double angle = 2.0 * atan2(n, fabs(q[3])), f = (q[3] < 0.0 ? -angle : angle) / n;
    w[0] = f * q[0]; w[1] = f * q[1]; w[2] = f * q[2];
  } else {
    w[0] = w[1] = w[2] = 0.0;
  }
}

__device__ void ra_log(const double* R, double* w) { double q[4]; ra_quat(R, q); ra_log_quat(q, w); }

__device__ void ra_mul(const double* A, const double* B, double* C) {   // C = A B
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
__device__ void ra_mul_tn(const double* A, const double* B, double* C) {   // C = A^T B
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
}

// ------------------------------------------------------------------------------------------------ device data
// Parameter blocks b: frames 0..F-1, then cameras.  off[b]: first parameter component, dof[b]: 1 or 3, cx[b]: column
// in the x/z matrix (-1 for a 1-DOF frame); the y column of block b is b.  Pair p owns rows roff[p].. (3 or 1), the gauge
// the last 1 or 3 rows.  The incidence list of block b is bent[bstart[b] .. bstart[b+1]), each entry 4p + slot with
// slot 0: frame1 (-1), 1: frame2 (+1), 2: cam1 (-1), 3: cam2 (+1).
struct RaDev {
  int F, C, nb, P, m, np, gauge, gdof, same_y;
  int n_xz, n_y, Np_xz, Np_y;
  const int *off, *dof, *cx, *xz_blk;
  const int *f1, *f2, *c1, *c2, *roff;
  const uint8_t* pdof;
  const double *R12, *ang, *xz, *rw, *rwrow;
  const int *bstart, *bent;
  const int *cstart, *cfr;
  double g0[3];
  double *rot, *step, *res, *w;
};

__device__ __forceinline__ int ra_slot_block(const RaDev& g, int p, int s) {
  return s == 0 ? g.f1[p] : s == 1 ? g.f2[p] : s == 2 ? g.c1[p] : g.c2[p];
}

// rotation of a frame block (a 1-DOF frame: AngleAxisToRotationMatrix((0, angle, 0)))
__device__ void ra_frame_R(const RaDev& g, int b, double* R) {
  const double* r = g.rot + g.off[b];
  if (g.dof[b] == 3) { ra_exp(r, R); return; }
  const double w[3] = {0.0, r[0], 0.0};
  ra_exp(w, R);
}

// ComputeResiduals (rotation_averaging_impl.cc:499-577); thread P is the gauge
__global__ void k_ra_residuals(RaDev g) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > g.P) return;
  if (p == g.P) {
    const double* r = g.rot + g.off[g.gauge];
    double* o = g.res + g.m - g.gdof;
    if (g.gdof == 1) { o[0] = r[0] - g.g0[1]; return; }
    double R0[9], R[9], D[9];
    ra_exp(g.g0, R0); ra_exp(r, R); ra_mul_tn(R0, R, D);
    ra_log(D, o);
    return;
  }
  double* o = g.res + g.roff[p];
  if (g.pdof[p] == 1) {
    o[0] = remainder((g.rot[g.off[g.f2[p]]] - g.rot[g.off[g.f1[p]]]) - g.ang[p], 2 * M_PI);
    return;
  }
  double R1[9], R2[9], T[9], U[9];
  ra_frame_R(g, g.f1[p], R1); ra_frame_R(g, g.f2[p], R2);
  if (g.c1[p] >= 0) { ra_exp(g.rot + g.off[g.c1[p]], T); ra_mul(T, R1, U); memcpy(R1, U, sizeof U); }
  if (g.c2[p] >= 0) { ra_exp(g.rot + g.off[g.c2[p]], T); ra_mul(T, R2, U); memcpy(R2, U, sizeof U); }
  ra_mul_tn(R2, g.R12 + 9LL * p, T); ra_mul(T, R1, U);
  double w[3];
  ra_log(U, w);
  o[0] = -w[0]; o[1] = -w[1]; o[2] = -w[2];
}

// ComputeIRLSWeights (:772-833) with the reweighting folded in; a NaN weight sets *bad
__global__ void k_ra_irls_weights(RaDev g, double sigma, int half_norm, int* bad) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= g.P) return;
  const double* r = g.res + g.roff[p];
  const double e2 = g.pdof[p] == 1 ? r[0] * r[0] + g.xz[p] : r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
  double w;
  if (half_norm) { w = pow(e2, (0.5 - 2) / 2); }
  else { const double t = e2 + sigma * sigma; w = sigma * sigma / (t * t); }
  if (isnan(w)) *bad = 1;
  g.w[p] = w * g.rw[p];
}

// One thread per column c of an axis matrix (column-major, ld Npad, lower triangle): sum over the column's incident rows
// of w_row * a(row, c) * a(row, c2) into (c2, c) for c2 >= c, then the gauge row (weight 1) and the ridge.
__global__ void k_ra_build(RaDev g, int axis_y, const double* w, double ridge, double* M, int Npad) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = axis_y ? g.n_y : g.n_xz;
  if (c >= n) return;
  const int b = axis_y ? c : g.xz_blk[c];
  double* col = M + (long long)c * Npad;
  for (int e = g.bstart[b]; e < g.bstart[b + 1]; ++e) {
    const int p = g.bent[e] >> 2, s = g.bent[e] & 3;
    if (!axis_y && g.pdof[p] == 1) continue;
    const double ws = (s & 1) ? w[p] : -w[p];
    for (int s2 = 0; s2 < 4; ++s2) {
      const int b2 = ra_slot_block(g, p, s2);
      if (b2 < 0) continue;
      const int c2 = axis_y ? b2 : g.cx[b2];
      if (c2 < c) continue;   // also a 1-DOF frame (-1) on the x/z axis
      col[c2] += (s2 & 1) ? ws : -ws;
    }
  }
  if (b == g.gauge && (axis_y || g.gdof == 3)) col[c] += 1.0;
  if (ridge > 0.0) col[c] += ridge;
}

__global__ void k_ra_pad_identity(double* M, int n, int Npad) {
  const int i = n + blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Npad) M[(long long)i * Npad + i] = 1.0;
}

// out = A^T diag(w) v in parameter order, one thread per block: the incident rows in list order, then the gauge (weight 1)
__global__ void k_ra_atv(RaDev g, const double* w, const double* v, double* out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= g.nb) return;
  const int d = g.dof[b];
  double acc[3] = {0.0, 0.0, 0.0};
  for (int e = g.bstart[b]; e < g.bstart[b + 1]; ++e) {
    const int p = g.bent[e] >> 2, s = g.bent[e] & 3;
    const double ws = (s & 1) ? w[p] : -w[p];
    const double* vr = v + g.roff[p];
    if (d == 3) { for (int i = 0; i < 3; ++i) acc[i] += ws * vr[i]; }
    else acc[0] += ws * (g.pdof[p] == 1 ? vr[0] : vr[1]);
  }
  if (b == g.gauge) { const double* vr = v + g.m - g.gdof; for (int i = 0; i < d; ++i) acc[i] += vr[i]; }
  for (int i = 0; i < d; ++i) out[g.off[b] + i] = acc[i];
}

// ax = diag(rwrow) A x, one thread per pair (thread P: the gauge rows)
__global__ void k_ra_ax(RaDev g, const double* x, double* ax) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > g.P) return;
  if (p == g.P) { for (int i = 0; i < g.gdof; ++i) ax[g.m - g.gdof + i] = x[g.off[g.gauge] + i]; return; }
  const int r = g.roff[p];
  if (g.pdof[p] == 1) { ax[r] = g.rw[p] * (-x[g.off[g.f1[p]]] + x[g.off[g.f2[p]]]); return; }
  double a[3] = {0.0, 0.0, 0.0};
  for (int s = 0; s < 4; ++s) {
    const int b = ra_slot_block(g, p, s);
    if (b < 0) continue;
    const double sg = (s & 1) ? 1.0 : -1.0;
    if (g.dof[b] == 3) { for (int i = 0; i < 3; ++i) a[i] += sg * x[g.off[b] + i]; }
    else a[1] += sg * x[g.off[b]];
  }
  for (int i = 0; i < 3; ++i) ax[r + i] = g.rw[p] * a[i];
}

// parameter order <-> the per-axis right-hand sides: X/Z in columns 0/1 of B_xz (or X/Y/Z in 0/1/2 when M_y = M_xz),
// Y in B_y
__global__ void k_ra_scatter(RaDev g, const double* v, double* Bxz, double* By, int to_axes) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= g.nb) return;
  double* t[3];
  const int o = g.off[b];
  if (g.dof[b] == 1) { t[0] = By + b; }
  else if (g.same_y) { for (int i = 0; i < 3; ++i) t[i] = Bxz + (long long)i * g.Np_xz + b; }
  else { t[0] = Bxz + g.cx[b]; t[1] = By + b; t[2] = Bxz + g.Np_xz + g.cx[b]; }
  for (int i = 0; i < g.dof[b]; ++i) { if (to_axes) *t[i] = v[o + i]; else g.step[o + i] = *t[i]; }
}

// the rows of one ADMM iteration (least_absolute_deviations.cc:170-194) after x and A x
__global__ void k_ra_admm_rows(int m, const double* ax, const double* bv, double* z, double* u, double* dz, double* er) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  const double a = ax[r], b = bv[r], zo = z[r];
  const double ah = B200RA_ADMM_ALPHA * a + (1.0 - B200RA_ADMM_ALPHA) * (zo + b);
  const double q = ah - b + u[r], k = 1.0 / B200RA_ADMM_RHO;
  const double zn = fmin(q + k, 0.0) + fmax(q - k, 0.0);
  u[r] += ah - zn - b;
  z[r] = zn; dz[r] = zn - zo; er[r] = a - zn - b;
}

// v = b + z - u
__global__ void k_ra_admm_rhs(int m, const double* bv, const double* z, const double* u, double* v) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < m) v[r] = bv[r] + z[r] - u[r];
}

__global__ void k_ra_mul(int m, const double* a, const double* b, double* c) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < m) c[r] = a[r] * b[r];
}

// UpdateState, frames (:579-593): R <- R exp(-step) for 3-DOF frames, angle -= step for 1-DOF frames; also writes the
// per-frame term of AverageStepSize (:631-642)
__global__ void k_ra_update_frames(RaDev g, double* stepsz) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= g.F) return;
  double* r = g.rot + g.off[f];
  const double* s = g.step + g.off[f];
  if (g.dof[f] == 1) { r[0] -= s[0]; stepsz[f] = fabs(s[0]); return; }
  const double ms[3] = {-s[0], -s[1], -s[2]};
  double R[9], U[9], T[9];
  ra_exp(r, R); ra_exp(ms, U); ra_mul(R, U, T);
  ra_log(T, r);
  stepsz[f] = sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
}

// UpdateState, estimated cameras (:607-628): one CTA per camera averages quat(R_c R exp(-step_c) R^T) over the camera's
// frames (AverageQuaternions / AverageUnitVectors, geometry/pose.cc:40-75, 182-199): the principal eigenvector of the
// mean of q q^T, a fixed-order sum over the CTA and a cyclic Jacobi eigensolver.  The sign of the average and of each
// q does not change the rotation.
#define RA_CB 128
__global__ void __launch_bounds__(RA_CB) k_ra_update_cameras(RaDev g) {
  const int c = blockIdx.x, b = g.F + c, tid = threadIdx.x;
  __shared__ double sh[10][RA_CB];
  __shared__ double Rc[9], Ru[9];
  if (tid == 0) {
    const double* s = g.step + g.off[b];
    const double ms[3] = {-s[0], -s[1], -s[2]};
    ra_exp(g.rot + g.off[b], Rc); ra_exp(ms, Ru);
  }
  __syncthreads();
  double acc[10];
  for (int i = 0; i < 10; ++i) acc[i] = 0.0;
  const int k0 = g.cstart[c], k1 = g.cstart[c + 1];
  for (int k = k0 + tid; k < k1; k += RA_CB) {
    double R[9], A[9], B[9], q[4];
    ra_frame_R(g, g.cfr[k], R);
    ra_mul(Rc, R, A); ra_mul(A, Ru, B);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) A[3 * i + j] = B[3 * i] * R[3 * j] + B[3 * i + 1] * R[3 * j + 1] + B[3 * i + 2] * R[3 * j + 2];
    ra_quat(A, q);
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    for (int i = 0; i < 4; ++i) q[i] /= n;
    int e = 0;
    for (int i = 0; i < 4; ++i) for (int j = i; j < 4; ++j) acc[e++] += q[i] * q[j];
  }
  for (int i = 0; i < 10; ++i) sh[i][tid] = acc[i];
  __syncthreads();
  for (int o = RA_CB / 2; o; o >>= 1) {
    if (tid < o) for (int i = 0; i < 10; ++i) sh[i][tid] += sh[i][tid + o];
    __syncthreads();
  }
  if (tid) return;
  const double cnt = (double)(k1 - k0);
  double A[4][4], V[4][4];
  int e = 0;
  for (int i = 0; i < 4; ++i) for (int j = i; j < 4; ++j) { A[i][j] = A[j][i] = sh[e++][0] / cnt; }
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) V[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 50; ++sweep) {
    double off = 0.0;
    for (int i = 0; i < 4; ++i) for (int j = i + 1; j < 4; ++j) off += A[i][j] * A[i][j];
    if (off == 0.0) break;
    for (int p = 0; p < 4; ++p)
      for (int q = p + 1; q < 4; ++q) {
        if (A[p][q] == 0.0) continue;
        const double th = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
        const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
        const double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
        for (int k = 0; k < 4; ++k) {   // A <- A J
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = cs * akp - sn * akq; A[k][q] = sn * akp + cs * akq;
        }
        for (int k = 0; k < 4; ++k) {   // A <- J^T A
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = cs * apk - sn * aqk; A[q][k] = sn * apk + cs * aqk;
        }
        for (int k = 0; k < 4; ++k) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = cs * vkp - sn * vkq; V[k][q] = sn * vkp + cs * vkq;
        }
      }
  }
  int best = 0;
  for (int i = 1; i < 4; ++i) if (A[i][i] > A[best][best]) best = i;
  double q[4] = {V[0][best], V[1][best], V[2][best], V[3][best]};   // (x, y, z, w)
  // toRotationMatrix then RotationMatrixToAngleAxis: the log of the unit quaternion
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int i = 0; i < 4; ++i) q[i] /= n;
  double R[9];
  {
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w); R[2] = 2 * (x * z + y * w);
    R[3] = 2 * (x * y + z * w); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
    R[6] = 2 * (x * z - y * w); R[7] = 2 * (y * z + x * w); R[8] = 1 - 2 * (x * x + y * y);
  }
  ra_log(R, g.rot + g.off[b]);
}

// deterministic sums: fixed grid, fixed per-thread order, fixed tree.  mode 0: sum a; 1: sum a^2
#define RA_RB 256
#define RA_RG 256
__global__ void k_ra_reduce1(const double* a, int64_t n, int mode, double* part) {
  __shared__ double sh[RA_RB];
  double s = 0;
  for (int64_t i = blockIdx.x * (int64_t)RA_RB + threadIdx.x; i < n; i += (int64_t)RA_RG * RA_RB) s += mode ? a[i] * a[i] : a[i];
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = RA_RB / 2; o; o >>= 1) { if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (!threadIdx.x) part[blockIdx.x] = sh[0];
}
__global__ void k_ra_reduce2(const double* part, double* out) {
  __shared__ double sh[RA_RG];
  sh[threadIdx.x] = part[threadIdx.x];
  __syncthreads();
  for (int o = RA_RG / 2; o; o >>= 1) { if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (!threadIdx.x) *out = sh[0];
}

// ------------------------------------------------------------------------------------------------ host
static inline unsigned ra_blocks(int64_t n, int t) { return (unsigned)std::max<int64_t>(1, (n + t - 1) / t); }
static bool ra_finite(const double* a, int64_t n) { for (int64_t i = 0; i < n; ++i) if (!std::isfinite(a[i])) return false; return true; }

#define RA_CUDA(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { rc = ra_fail(B200RA_ERR_CUDA, "%s: %s", #x, cudaGetErrorString(e_)); goto cleanup; } } while (0)

extern "C" int b200ra_solve(const b200ra_options* o, b200ra_problem* p, b200ra_summary* out) {
  g_ra_err.clear();
  if (!o || !p || !out) return ra_fail(B200RA_ERR_INPUT, "null argument");
  // ---- options
  if (o->max_num_l1_iterations < 0 || o->max_num_irls_iterations < 0 || !(o->l1_step_convergence_threshold >= 0) ||
      !(o->irls_step_convergence_threshold >= 0) || !(o->irls_loss_parameter_sigma > 0) ||
      !std::isfinite(o->irls_loss_parameter_sigma) || !(o->ridge_regularization >= 0) ||
      !std::isfinite(o->ridge_regularization) || (o->weight_type != B200RA_GEMAN_MCCLURE && o->weight_type != B200RA_HALF_NORM))
    return ra_fail(B200RA_ERR_INPUT, "invalid solver options");
  // ---- problem
  const int F = p->num_frames, C = p->num_cameras, P = p->num_pairs;
  if (F < 1 || C < 0 || P < 0) return ra_fail(B200RA_ERR_INPUT, "need at least one frame and non-negative sizes");
  if (!p->frame_dof || !p->rotations || (P && (!p->pair_frame1 || !p->pair_frame2 || !p->pair_dof)))
    return ra_fail(B200RA_ERR_INPUT, "missing array");
  if (C && (!p->cam_frame_start || !p->cam_frames)) return ra_fail(B200RA_ERR_INPUT, "estimated cameras need the camera -> frames lists");
  const int nb = F + C;
  std::vector<int> off(nb), dof(nb), cx(nb, -1), xz_blk;
  int np = 0;
  for (int b = 0; b < nb; ++b) {
    const int d = b < F ? p->frame_dof[b] : 3;
    if (d != 1 && d != 3) return ra_fail(B200RA_ERR_INPUT, "frame %d: dof %d is neither 1 nor 3", b, d);
    off[b] = np; dof[b] = d; np += d;
    if (d == 3) { cx[b] = (int)xz_blk.size(); xz_blk.push_back(b); }
  }
  if (!ra_finite(p->rotations, np)) return ra_fail(B200RA_ERR_INPUT, "non-finite rotation");
  const int n_xz = (int)xz_blk.size(), n_y = nb;
  std::vector<int> roff(P);
  std::vector<double> rw(P, 1.0);
  int64_t m = 0;
  for (int q = 0; q < P; ++q) {
    const int a = p->pair_frame1[q], b = p->pair_frame2[q];
    const int c1 = p->pair_cam1 ? p->pair_cam1[q] : -1, c2 = p->pair_cam2 ? p->pair_cam2[q] : -1;
    if (a < 0 || a >= F || b < 0 || b >= F) return ra_fail(B200RA_ERR_INPUT, "pair %d: frame out of range", q);
    if (c1 < -1 || c1 >= C || c2 < -1 || c2 >= C) return ra_fail(B200RA_ERR_INPUT, "pair %d: camera out of range", q);
    const int d = p->pair_dof[q];
    if (d == 1) {
      if (dof[a] != 1 || dof[b] != 1) return ra_fail(B200RA_ERR_INPUT, "pair %d: a 1-DOF pair needs two 1-DOF frames", q);
      if (c1 >= 0 || c2 >= 0) return ra_fail(B200RA_ERR_INPUT, "pair %d: a 1-DOF pair cannot have estimated cameras", q);
      if (!p->pair_angle || !p->pair_xz_error) return ra_fail(B200RA_ERR_INPUT, "1-DOF pairs need pair_angle and pair_xz_error");
      if (!std::isfinite(p->pair_angle[q]) || !(p->pair_xz_error[q] >= 0) || !std::isfinite(p->pair_xz_error[q]))
        return ra_fail(B200RA_ERR_INPUT, "pair %d: non-finite angle or xz_error", q);
    } else if (d == 3) {
      if (dof[a] == 1 && dof[b] == 1) return ra_fail(B200RA_ERR_INPUT, "pair %d: a 3-DOF pair between two 1-DOF frames", q);
      if (!p->pair_R || !ra_finite(p->pair_R + 9LL * q, 9)) return ra_fail(B200RA_ERR_INPUT, "pair %d: missing or non-finite R_cam2_from_cam1", q);
    } else {
      return ra_fail(B200RA_ERR_INPUT, "pair %d: dof %d is neither 1 nor 3", q, d);
    }
    if (p->pair_reweighting) {
      rw[q] = p->pair_reweighting[q];
      if (!(rw[q] >= 0) || !std::isfinite(rw[q])) return ra_fail(B200RA_ERR_INPUT, "pair %d: reweighting must be finite and >= 0", q);
    }
    roff[q] = (int)m; m += d;
  }
  const int gauge = p->gauge_frame;
  if (gauge < 0 || gauge >= F) return ra_fail(B200RA_ERR_INPUT, "gauge frame %d out of range", gauge);
  if (!ra_finite(p->gauge_rotation, 3)) return ra_fail(B200RA_ERR_INPUT, "non-finite gauge rotation");
  const int gdof = dof[gauge];
  m += gdof;
  if (m > 0x7fffffff - 16) return ra_fail(B200RA_ERR_INPUT, "too many residual rows");
  std::vector<int> cstart(C + 1, 0), cfr;
  if (C) {
    if (p->cam_frame_start[0] != 0) return ra_fail(B200RA_ERR_INPUT, "cam_frame_start[0] must be 0");
    for (int c = 0; c < C; ++c) {
      cstart[c + 1] = p->cam_frame_start[c + 1];
      if (cstart[c + 1] <= cstart[c]) return ra_fail(B200RA_ERR_INPUT, "camera %d: no frames to average over", c);
    }
    cfr.assign(p->cam_frames, p->cam_frames + cstart[C]);
    for (int f : cfr) if (f < 0 || f >= F) return ra_fail(B200RA_ERR_INPUT, "camera frame list: frame %d out of range", f);
  }
  if (n_xz > B200RA_MAX_AXIS_DIM || n_y > B200RA_MAX_AXIS_DIM)
    return ra_fail(B200RA_ERR_TOO_LARGE, "axis dimensions %d (x/z) and %d (y): the dense limit is %d (a sparse factorisation is not implemented)",
                   n_xz, n_y, B200RA_MAX_AXIS_DIM);
  const int same_y = n_xz == n_y;
  const int Np_xz = (n_xz + BA_TILE - 1) / BA_TILE * BA_TILE, Np_y = same_y ? 0 : (n_y + BA_TILE - 1) / BA_TILE * BA_TILE;
  const int nrhs_xz = same_y ? 3 : 2;
  out->status = B200RA_SUCCESS; out->num_l1_iterations = out->num_irls_iterations = 0;
  out->n_xz = n_xz; out->n_y = n_y; out->num_residuals = (int)m;
  out->l1_ms = out->irls_ms = out->build_ms = out->factor_ms = out->solve_ms = 0;
  if (o->max_num_l1_iterations > 0 && m < np) { out->status = B200RA_UNDERDETERMINED; return 0; }
  if (o->max_num_l1_iterations == 0 && o->max_num_irls_iterations == 0) return 0;

  // block -> incident pair slots, in pair order
  std::vector<int> bstart(nb + 1, 0), bent;
  std::vector<int> h_f1(P), h_f2(P), h_c1(P), h_c2(P);
  std::vector<uint8_t> h_pdof(P);
  for (int q = 0; q < P; ++q) {
    h_f1[q] = p->pair_frame1[q]; h_f2[q] = p->pair_frame2[q];
    h_c1[q] = p->pair_cam1 && p->pair_cam1[q] >= 0 ? F + p->pair_cam1[q] : -1;
    h_c2[q] = p->pair_cam2 && p->pair_cam2[q] >= 0 ? F + p->pair_cam2[q] : -1;
    h_pdof[q] = p->pair_dof[q];
    const int bl[4] = {h_f1[q], h_f2[q], h_c1[q], h_c2[q]};
    for (int s = 0; s < 4; ++s) if (bl[s] >= 0) bstart[bl[s] + 1]++;
  }
  for (int b = 0; b < nb; ++b) bstart[b + 1] += bstart[b];
  bent.resize(std::max(1, bstart[nb]));
  {
    std::vector<int> fill(bstart.begin(), bstart.end() - 1);
    for (int q = 0; q < P; ++q) {
      const int bl[4] = {h_f1[q], h_f2[q], h_c1[q], h_c2[q]};
      for (int s = 0; s < 4; ++s) if (bl[s] >= 0) bent[fill[bl[s]]++] = 4 * q + s;
    }
  }
  std::vector<double> rwrow(m, 1.0), rw2(P), h_R(9LL * std::max(P, 1), 0.0), h_ang(std::max(P, 1), 0.0), h_xz(std::max(P, 1), 0.0);
  for (int q = 0; q < P; ++q) {
    for (int i = 0; i < h_pdof[q]; ++i) rwrow[roff[q] + i] = rw[q];
    rw2[q] = rw[q] * rw[q];
    if (h_pdof[q] == 3) for (int k = 0; k < 9; ++k) h_R[9LL * q + k] = p->pair_R[9LL * q + k];
    else { h_ang[q] = p->pair_angle[q]; h_xz[q] = p->pair_xz_error[q]; }
  }

  int rc = 0;
  if (o->gpu_index >= 0) {
    int ndev = 0; cudaGetDeviceCount(&ndev);
    if (o->gpu_index >= ndev) return ra_fail(B200RA_ERR_INPUT, "gpu_index out of range");
    cudaSetDevice(o->gpu_index);
  }
  RaDev g; memset(&g, 0, sizeof g);
  g.F = F; g.C = C; g.nb = nb; g.P = P; g.m = (int)m; g.np = np; g.gauge = gauge; g.gdof = gdof; g.same_y = same_y;
  g.n_xz = n_xz; g.n_y = n_y; g.Np_xz = Np_xz; g.Np_y = Np_y;
  for (int k = 0; k < 3; ++k) g.g0[k] = p->gauge_rotation[k];
  std::vector<void*> allocs;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  double *Mxz = nullptr, *My = nullptr, *dinv_xz = nullptr, *dinv_y = nullptr, *Bxz = nullptr, *Wxz = nullptr, *By = nullptr, *Wy = nullptr;
  double *d_rw2 = nullptr, *d_rwrow = nullptr, *bv = nullptr, *z = nullptr, *u = nullptr, *dz = nullptr, *er = nullptr, *ax = nullptr, *v = nullptr;
  double *t1 = nullptr, *t2 = nullptr, *stepsz = nullptr, *red = nullptr;
  BaDenseFlag *flag_xz = nullptr, *flag_y = nullptr;
  int* d_bad = nullptr;
  auto dalloc = [&](size_t bytes) -> void* { void* q = nullptr; if (cudaMalloc(&q, std::max<size_t>(bytes, 8)) != cudaSuccess) return nullptr; allocs.push_back(q); return q; };
  auto dput = [&](const void* h, size_t bytes) -> void* { void* q = dalloc(bytes); if (q && bytes) cudaMemcpy(q, h, bytes, cudaMemcpyHostToDevice); return q; };
#define RA_ALLOC(ptr, type, count) do { ptr = (type*)dalloc(sizeof(type) * (size_t)(count)); if (!ptr) { rc = ra_fail(B200RA_ERR_CUDA, "cudaMalloc failed"); goto cleanup; } } while (0)
#define RA_PUT(ptr, type, vec) do { ptr = (type*)dput((vec).data(), sizeof(type) * (vec).size()); if (!ptr) { rc = ra_fail(B200RA_ERR_CUDA, "cudaMalloc failed"); goto cleanup; } } while (0)
  {
    std::vector<double> rot(p->rotations, p->rotations + np);
    std::vector<int> cs(cstart), cf(cfr.empty() ? std::vector<int>(1, 0) : cfr), xb(xz_blk.empty() ? std::vector<int>(1, 0) : xz_blk);
    std::vector<int> ro(roff.empty() ? std::vector<int>(1, 0) : roff);
    std::vector<double> rwp(rw.empty() ? std::vector<double>(1, 1.0) : rw);
    RA_PUT(g.off, const int, off); RA_PUT(g.dof, const int, dof); RA_PUT(g.cx, const int, cx); RA_PUT(g.xz_blk, const int, xb);
    RA_PUT(g.f1, const int, h_f1); RA_PUT(g.f2, const int, h_f2); RA_PUT(g.c1, const int, h_c1); RA_PUT(g.c2, const int, h_c2);
    RA_PUT(g.roff, const int, ro); RA_PUT(g.pdof, const uint8_t, h_pdof);
    RA_PUT(g.R12, const double, h_R); RA_PUT(g.ang, const double, h_ang); RA_PUT(g.xz, const double, h_xz);
    RA_PUT(g.rw, const double, rwp); RA_PUT(g.rwrow, const double, rwrow); RA_PUT(d_rw2, double, rw2);
    RA_PUT(g.bstart, const int, bstart); RA_PUT(g.bent, const int, bent);
    RA_PUT(g.cstart, const int, cs); RA_PUT(g.cfr, const int, cf);
    RA_PUT(g.rot, double, rot);
    d_rwrow = (double*)g.rwrow;
  }
  RA_ALLOC(g.step, double, np); RA_ALLOC(g.res, double, m); RA_ALLOC(g.w, double, std::max(P, 1));
  RA_ALLOC(bv, double, m); RA_ALLOC(z, double, m); RA_ALLOC(u, double, m); RA_ALLOC(dz, double, m); RA_ALLOC(er, double, m);
  RA_ALLOC(ax, double, m); RA_ALLOC(v, double, m); RA_ALLOC(t1, double, np); RA_ALLOC(t2, double, np);
  RA_ALLOC(stepsz, double, F); RA_ALLOC(red, double, RA_RG + 16); RA_ALLOC(d_bad, int, 1);
  RA_ALLOC(flag_xz, BaDenseFlag, 1); RA_ALLOC(flag_y, BaDenseFlag, 1);
  if (n_xz) {
    RA_ALLOC(Mxz, double, (size_t)Np_xz * Np_xz); RA_ALLOC(dinv_xz, double, (size_t)Np_xz * BA_TILE);
    RA_ALLOC(Bxz, double, (size_t)Np_xz * nrhs_xz); RA_ALLOC(Wxz, double, (size_t)Np_xz * nrhs_xz);
    RA_CUDA(cudaMemset(Bxz, 0, sizeof(double) * (size_t)Np_xz * nrhs_xz));
  }
  if (!same_y) {
    RA_ALLOC(My, double, (size_t)Np_y * Np_y); RA_ALLOC(dinv_y, double, (size_t)Np_y * BA_TILE);
    RA_ALLOC(By, double, Np_y); RA_ALLOC(Wy, double, Np_y);
    RA_CUDA(cudaMemset(By, 0, sizeof(double) * Np_y));
  }
  for (int k = 0; k < 4; ++k) RA_CUDA(cudaEventCreate(&ev[k]));
  {
    double sums[8];
    // deterministic sum (mode 0) or sum of squares (mode 1) of n doubles into sums[slot] (read back by fetch())
    auto dsum = [&](const double* x, int64_t n, int mode, int slot) {
      k_ra_reduce1<<<RA_RG, RA_RB>>>(x, n, mode, red);
      k_ra_reduce2<<<1, RA_RG>>>(red, red + RA_RG + slot);
    };
    auto fetch = [&](int k) -> cudaError_t { return cudaMemcpy(sums, red + RA_RG, sizeof(double) * k, cudaMemcpyDeviceToHost); };
    float ms = 0;
    // timed section helpers: ev[2], ev[3] bracket build / factor / solve pieces
    auto tic = [&]() { cudaEventRecord(ev[2]); };
    auto toc = [&](double* acc) { cudaEventRecord(ev[3]); cudaEventSynchronize(ev[3]); float t = 0; cudaEventElapsedTime(&t, ev[2], ev[3]); *acc += t; };
    // build and factor the axis matrices with pair weights w; false on a failed pivot
    auto build_factor = [&](const double* w) -> int {
      tic();
      if (n_xz) {
        cudaMemset(Mxz, 0, sizeof(double) * (size_t)Np_xz * Np_xz);
        k_ra_build<<<ra_blocks(n_xz, 128), 128>>>(g, 0, w, o->ridge_regularization, Mxz, Np_xz);
        if (Np_xz > n_xz) k_ra_pad_identity<<<ra_blocks(Np_xz - n_xz, 64), 64>>>(Mxz, n_xz, Np_xz);
      }
      if (!same_y) {
        cudaMemset(My, 0, sizeof(double) * (size_t)Np_y * Np_y);
        k_ra_build<<<ra_blocks(n_y, 128), 128>>>(g, 1, w, o->ridge_regularization, My, Np_y);
        if (Np_y > n_y) k_ra_pad_identity<<<ra_blocks(Np_y - n_y, 64), 64>>>(My, n_y, Np_y);
      }
      toc(&out->build_ms);
      tic();
      BaDenseFlag fl{0, 0, 0.0};
      cudaMemcpy(flag_xz, &fl, sizeof fl, cudaMemcpyHostToDevice);
      cudaMemcpy(flag_y, &fl, sizeof fl, cudaMemcpyHostToDevice);
      if (n_xz) ba_dense_potrf(Mxz, Np_xz, n_xz, n_xz, 0.0, dinv_xz, flag_xz, 0);
      if (!same_y) ba_dense_potrf(My, Np_y, n_y, n_y, 0.0, dinv_y, flag_y, 0);
      toc(&out->factor_ms);
      BaDenseFlag a{0, 0, 0.0}, b{0, 0, 0.0};
      cudaMemcpy(&a, flag_xz, sizeof a, cudaMemcpyDeviceToHost);
      cudaMemcpy(&b, flag_y, sizeof b, cudaMemcpyDeviceToHost);
      return !a.bad && !b.bad;
    };
    // step (parameter order) = (A^T W A)^-1 rhs (parameter order)
    auto solve = [&](const double* rhs) {
      tic();
      k_ra_scatter<<<ra_blocks(nb, 128), 128>>>(g, rhs, Bxz, By, 1);
      if (n_xz) ba_dense_potrs(Mxz, Np_xz, dinv_xz, nrhs_xz, Bxz, Wxz, flag_xz, 0);
      if (!same_y) ba_dense_potrs(My, Np_y, dinv_y, 1, By, Wy, flag_y, 0);
      k_ra_scatter<<<ra_blocks(nb, 128), 128>>>(g, nullptr, Bxz, By, 0);
      toc(&out->solve_ms);
    };
    // UpdateState and AverageStepSize; returns the average step
    auto update = [&]() -> double {
      k_ra_update_frames<<<ra_blocks(F, 128), 128>>>(g, stepsz);
      if (C) k_ra_update_cameras<<<C, RA_CB>>>(g);
      dsum(stepsz, F, 0, 0);
      fetch(1);
      return sums[0] / F;
    };
    const unsigned pb = ra_blocks((int64_t)P + 1, 128), mb = ra_blocks(m, 256);
    int hist = 0;
    // ---------------- L1 (SolveL1Regression, :704-770)
    if (o->max_num_l1_iterations > 0) {
      RA_CUDA(cudaEventRecord(ev[0]));
      if (!build_factor(d_rw2)) { out->status = B200RA_FACTORIZATION_FAILED; goto done; }
      double prev_norm = 0, curr_norm = 0;
      int max_admm = 10;
      const double eps_pri0 = sqrt((double)m) * B200RA_ADMM_ABS_TOL, eps_dual0 = sqrt((double)np) * B200RA_ADMM_ABS_TOL;
      int it = 0;
      for (; it < o->max_num_l1_iterations; ++it) {
        k_ra_residuals<<<pb, 128>>>(g);
        k_ra_mul<<<mb, 256>>>((int)m, d_rwrow, g.res, bv);
        RA_CUDA(cudaMemset(z, 0, sizeof(double) * m));
        RA_CUDA(cudaMemset(u, 0, sizeof(double) * m));
        dsum(bv, m, 1, 0);
        RA_CUDA(fetch(1));
        const double b_norm = sqrt(sums[0]);
        int i = 0;
        for (; i < max_admm; ++i) {
          k_ra_admm_rhs<<<mb, 256>>>((int)m, bv, z, u, v);
          k_ra_atv<<<ra_blocks(nb, 128), 128>>>(g, g.rw, v, t1);
          solve(t1);
          k_ra_ax<<<pb, 128>>>(g, g.step, ax);
          k_ra_admm_rows<<<mb, 256>>>((int)m, ax, bv, z, u, dz, er);
          k_ra_atv<<<ra_blocks(nb, 128), 128>>>(g, g.rw, dz, t1);
          k_ra_atv<<<ra_blocks(nb, 128), 128>>>(g, g.rw, u, t2);
          dsum(er, m, 1, 0); dsum(ax, m, 1, 1); dsum(z, m, 1, 2); dsum(t1, np, 1, 3); dsum(t2, np, 1, 4);
          RA_CUDA(fetch(5));
          const double r_norm = sqrt(sums[0]);
          const double s_norm = B200RA_ADMM_RHO * sqrt(sums[3]);
          const double eps_pri = eps_pri0 + B200RA_ADMM_REL_TOL * std::max(b_norm, std::max(sqrt(sums[1]), sqrt(sums[2])));
          const double eps_dual = eps_dual0 + B200RA_ADMM_REL_TOL * (B200RA_ADMM_RHO * sqrt(sums[4]));
          if (r_norm < eps_pri && s_norm < eps_dual) { ++i; break; }
        }
        if (out->admm_iterations) out->admm_iterations[it] = i;
        prev_norm = curr_norm;
        dsum(g.step, np, 1, 0);
        RA_CUDA(fetch(1));
        curr_norm = sqrt(sums[0]);
        if (std::isnan(curr_norm)) { out->status = B200RA_NAN_STEP; out->num_l1_iterations = it; goto done; }
        const double avg = update();
        if (out->step_history) out->step_history[hist] = avg;
        ++hist;
        if (avg < o->l1_step_convergence_threshold || fabs(prev_norm - curr_norm) < 1e-12) { ++it; break; }
        max_admm = std::min(max_admm * 2, 100);
      }
      out->num_l1_iterations = it;
      RA_CUDA(cudaEventRecord(ev[1])); RA_CUDA(cudaEventSynchronize(ev[1]));
      cudaEventElapsedTime(&ms, ev[0], ev[1]); out->l1_ms = ms;
    }
    // ---------------- IRLS (SolveIRLS, :835-902)
    if (o->max_num_irls_iterations > 0) {
      RA_CUDA(cudaEventRecord(ev[0]));
      const double sigma = o->irls_loss_parameter_sigma * M_PI / 180.0;
      int it = 0;
      for (; it < o->max_num_irls_iterations; ++it) {
        k_ra_residuals<<<pb, 128>>>(g);
        int zero = 0;
        RA_CUDA(cudaMemcpy(d_bad, &zero, sizeof zero, cudaMemcpyHostToDevice));
        if (P) k_ra_irls_weights<<<ra_blocks(P, 128), 128>>>(g, sigma, o->weight_type == B200RA_HALF_NORM, d_bad);
        int bad = 0;
        RA_CUDA(cudaMemcpy(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost));
        if (bad) { out->status = B200RA_NAN_WEIGHT; out->num_irls_iterations = it; goto done; }
        if (!build_factor(g.w)) { out->status = B200RA_FACTORIZATION_FAILED; out->num_irls_iterations = it; goto done; }
        k_ra_atv<<<ra_blocks(nb, 128), 128>>>(g, g.w, g.res, t1);
        solve(t1);
        dsum(g.step, np, 1, 0);
        RA_CUDA(fetch(1));
        if (std::isnan(sums[0])) { out->status = B200RA_NAN_STEP; out->num_irls_iterations = it; goto done; }
        const double avg = update();
        if (out->step_history) out->step_history[hist] = avg;
        ++hist;
        if (avg < o->irls_step_convergence_threshold) { ++it; break; }
      }
      out->num_irls_iterations = it;
      RA_CUDA(cudaEventRecord(ev[1])); RA_CUDA(cudaEventSynchronize(ev[1]));
      cudaEventElapsedTime(&ms, ev[0], ev[1]); out->irls_ms = ms;
    }
  done:
    RA_CUDA(cudaGetLastError());
    RA_CUDA(cudaDeviceSynchronize());
    if (out->status == B200RA_SUCCESS) RA_CUDA(cudaMemcpy(p->rotations, g.rot, sizeof(double) * np, cudaMemcpyDeviceToHost));
  }
cleanup:
  for (void* q : allocs) cudaFree(q);
  for (int k = 0; k < 4; ++k) if (ev[k]) cudaEventDestroy(ev[k]);
  return rc;
}
