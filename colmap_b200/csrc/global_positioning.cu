// global_positioning.cu — the global positioner's LM solve (include/b200_global_positioning.h) on the H100 in fp64.
//
// Ceres solves GlobalPositioner's problem with SPARSE_SCHUR, eliminating the scales and then the points.  The step here
// is the same exact Newton-LM step with a deeper elimination:
//   1. per observation: linearise, apply the Huber corrector, eliminate the observation's scale (a 1x1 block),
//   2. per point: eliminate the 3x3 point block (observations are sorted by point),
//   3. the reduced matrix over frame centres and camera-in-rig positions (3 columns per block) is built densely, one
//      thread per row and no atomics, so that repeated solves are bit-identical; the LM diagonal is added,
//   4. ba_dense_potrf factors it, ba_dense_potrs (forward / backward solves one tile per launch) gives the step,
//   5. back-substitution to the points, then to the scales.
// Trust-region rules (Jacobi scaling from the first Jacobian, LM diagonal clamp, radius update, tolerances) are those of
// oracle/ba_oracle.c; the scale bound is enforced as ceres::ParameterBlock::Plus does, by clamping the candidate, while
// the model cost change uses the unclamped step.  Not restated: the projected Armijo line search Ceres runs on every step
// of a bounded problem (TrustRegionMinimizer::DoLineSearch), which is every step here since all scales are bounded; it
// shortens any full step that fails the Armijo test, so trajectories differ from Ceres' on such steps (DESIGN.md §3).
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/b200_global_positioning.h"
#include "ba_dense_f64.h"
#include "ba_models.cuh"
#include "solver_host.cuh"

static thread_local std::string g_gp_err;
#define GP_CHECK(call) SOLVER_CUDA(g_gp_err, B200GP_ERR_CUDA, call)
extern "C" const char* b200gp_last_error(void) { return g_gp_err.c_str(); }

extern "C" void b200gp_options_init(b200gp_options* o) {
  o->optimize_positions = 1; o->optimize_points = 1; o->optimize_scales = 1; o->refine_sensor_from_rig = 1;
  o->loss_function_scale = 0.1; o->max_num_iterations = 100; o->function_tolerance = 1e-5;
  o->gradient_tolerance = 1e-10; o->parameter_tolerance = 1e-8; o->initial_trust_region_radius = 1e4;
  o->max_trust_region_radius = 1e16; o->min_trust_region_radius = 1e-32; o->min_relative_decrease = 1e-3;
  o->min_lm_diagonal = 1e-6; o->max_lm_diagonal = 1e32; o->gpu_index = -1;
}

// ------------------------------------------------------------------------------------------------ camera rays (host)
// Distortion(extra_params, u, v) of the models that undistort iteratively (sensor/models.h), in dual numbers so that
// the Newton step of IterativeUndistortion (models.h:1141-1190) gets its Jacobian.
template <typename S>
static bool gp_distortion(int id, const double* e, const S& u, const S& v, S* du, S* dv) {
  const S two(2.0);
  if (id == 2 || id == 8) {            // SIMPLE_RADIAL(_FISHEYE): k
    const S r = S(e[0]) * (u * u + v * v); *du = u * r; *dv = v * r;
  } else if (id == 3 || id == 9) {     // RADIAL(_FISHEYE): k1 k2
    const S r2 = u * u + v * v, r = S(e[0]) * r2 + S(e[1]) * r2 * r2; *du = u * r; *dv = v * r;
  } else if (id == 4) {                // OPENCV: k1 k2 p1 p2
    const S u2 = u * u, uv = u * v, v2 = v * v, r2 = u2 + v2, r = S(e[0]) * r2 + S(e[1]) * r2 * r2;
    *du = u * r + two * S(e[2]) * uv + S(e[3]) * (r2 + two * u2);
    *dv = v * r + two * S(e[3]) * uv + S(e[2]) * (r2 + two * v2);
  } else if (id == 5) {                // OPENCV_FISHEYE: k1..k4 on the fisheye coordinates
    const S t2 = u * u + v * v, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
    const S r = S(e[0]) * t2 + S(e[1]) * t4 + S(e[2]) * t6 + S(e[3]) * t8; *du = u * r; *dv = v * r;
  } else if (id == 6) {                // FULL_OPENCV: k1 k2 p1 p2 k3 k4 k5 k6
    const S u2 = u * u, uv = u * v, v2 = v * v, r2 = u2 + v2, r4 = r2 * r2, r6 = r4 * r2;
    const S r = (S(1.0) + S(e[0]) * r2 + S(e[1]) * r4 + S(e[4]) * r6) / (S(1.0) + S(e[5]) * r2 + S(e[6]) * r4 + S(e[7]) * r6);
    *du = u * r + two * S(e[2]) * uv + S(e[3]) * (r2 + two * u2) - u;
    *dv = v * r + two * S(e[3]) * uv + S(e[2]) * (r2 + two * v2) - v;
  } else if (id == 10) {               // THIN_PRISM_FISHEYE: k1 k2 p1 p2 k3 k4 sx1 sy1
    const S u2 = u * u, uv = u * v, v2 = v * v, r2 = u2 + v2, r4 = r2 * r2, r6 = r4 * r2, r8 = r6 * r2;
    const S r = S(e[0]) * r2 + S(e[1]) * r4 + S(e[4]) * r6 + S(e[5]) * r8;
    *du = u * r + two * S(e[2]) * uv + S(e[3]) * (r2 + two * u2) + S(e[6]) * r2;
    *dv = v * r + two * S(e[3]) * uv + S(e[2]) * (r2 + two * v2) + S(e[7]) * r2;
  } else if (id == 11) {               // RAD_TAN_THIN_PRISM_FISHEYE: k0..k5 p0 p1 s0..s3
    const S t2 = u * u + v * v;
    S radial(1.0), power(1.0);
    for (int i = 0; i < 6; ++i) { power = power * t2; radial = radial + S(e[i]) * power; }
    const S px = radial * u, py = radial * v;
    const S x2 = px * px, y2 = py * py, xy = px * py, r2 = x2 + y2, r4 = r2 * r2;
    *du = px + (two * S(e[7]) * xy + S(e[6]) * (r2 + two * x2)) + (S(e[8]) * r2 + S(e[9]) * r4) - u;
    *dv = py + (two * S(e[6]) * xy + S(e[7]) * (r2 + two * y2)) + (S(e[10]) * r2 + S(e[11]) * r4) - v;
  } else {
    return false;
  }
  return true;
}

static bool gp_iterative_undistortion(int id, const double* e, double* u, double* v) {
  const double x0[2] = {*u, *v};
  double x[2] = {*u, *v};
  for (int it = 0; it < 100; ++it) {
    typedef BaDual<2> D;
    D du, dv;
    gp_distortion<D>(id, e, D::variable(x[0], 0), D::variable(x[1], 1), &du, &dv);
    const double J00 = du.d[0] + 1, J01 = du.d[1], J10 = dv.d[0], J11 = dv.d[1] + 1;
    const double b0 = x[0] + du.v - x0[0], b1 = x[1] + dv.v - x0[1];
    // J.partialPivLu().solve(b) for 2x2: partial pivoting on the first column
    double s0, s1;
    if (fabs(J10) > fabs(J00)) {
      const double l = J00 / J10, u11 = J01 - l * J11;
      s1 = (b0 - l * b1) / u11; s0 = (b1 - J11 * s1) / J10;
    } else {
      const double l = J10 / J00, u11 = J11 - l * J01;
      s1 = (b1 - l * b0) / u11; s0 = (b0 - J01 * s1) / J00;
    }
    const double radius_sqr = std::max((x[0] * x[0] + x[1] * x[1]) * 0.01, 0.01);
    const double n2 = s0 * s0 + s1 * s1;
    if (n2 > radius_sqr) { const double f = sqrt(radius_sqr / n2); s0 *= f; s1 *= f; }
    x[0] -= s0; x[1] -= s1;
    if (s0 * s0 + s1 * s1 < 1e-10) { *u = x[0]; *v = x[1]; return true; }
  }
  *u = x[0]; *v = x[1];
  return false;
}

static void gp_normal_from_fisheye(double uu, double vv, double* u, double* v) {
  *u = uu; *v = vv;
  const double theta = sqrt(uu * uu + vv * vv), tct = theta * cos(theta);
  if (tct > DBL_EPSILON) { const double s = sin(theta) / tct; *u *= s; *v *= s; }
}

// CamFromImg of every model but EQUIRECTANGULAR's ray (models.h:1248-2900)
static bool gp_cam_from_img(int id, const double* p, double x, double y, double* u, double* v) {
  switch (id) {
    case 0: *u = (x - p[1]) / p[0]; *v = (y - p[2]) / p[0]; return true;
    case 1: *u = (x - p[2]) / p[0]; *v = (y - p[3]) / p[1]; return true;
    case 2: case 3: *u = (x - p[1]) / p[0]; *v = (y - p[2]) / p[0]; return gp_iterative_undistortion(id, p + 3, u, v);
    case 4: case 6: *u = (x - p[2]) / p[0]; *v = (y - p[3]) / p[1]; return gp_iterative_undistortion(id, p + 4, u, v);
    case 5: case 10: case 11: case 8: case 9: {
      const bool simple = id == 8 || id == 9;
      double uu = simple ? (x - p[1]) / p[0] : (x - p[2]) / p[0], vv = simple ? (y - p[2]) / p[0] : (y - p[3]) / p[1];
      if (!gp_iterative_undistortion(id, p + (simple ? 3 : 4), &uu, &vv)) return false;
      gp_normal_from_fisheye(uu, vv, u, v);
      return true;
    }
    case 7: {   // FOV: closed-form Undistortion (models.h:1891-1925)
      const double uu = (x - p[2]) / p[0], vv = (y - p[3]) / p[1], omega = p[4];
      const double r2 = uu * uu + vv * vv, o2 = omega * omega;
      double f;
      if (o2 < 1e-4) f = (o2 * r2) / 3.0 - o2 / 12.0 + 1.0;
      else if (r2 < 1e-4) f = (omega * (omega * omega * r2 + 3.0)) / (6.0 * tan(omega / 2.0));
      else { const double r = sqrt(r2); f = tan(r * omega) / (r * 2.0 * tan(omega / 2.0)); }
      *u = uu * f; *v = vv * f;
      return true;
    }
    case 12: case 13: {
      const bool s = id == 12;
      const double x0 = s ? (x - p[1]) / p[0] : (x - p[2]) / p[0], y0 = s ? (y - p[2]) / p[0] : (y - p[3]) / p[1];
      const double den = 1.0 + (s ? p[3] : p[4]) * (x0 * x0 + y0 * y0);
      *u = x0 / den; *v = y0 / den;
      return true;
    }
    case 14: gp_normal_from_fisheye((x - p[1]) / p[0], (y - p[2]) / p[0], u, v); return true;
    case 15: gp_normal_from_fisheye((x - p[2]) / p[0], (y - p[3]) / p[1], u, v); return true;
    case 16: {  // EUCM (models.h:2796-2830)
      *u = (x - p[2]) / p[0]; *v = (y - p[3]) / p[1];
      const double alpha = p[4], beta = p[5], r2 = *u * *u + *v * *v, gamma = 1.0 - alpha;
      const double rad = 1.0 - (alpha - gamma) * beta * r2;
      if (rad < 0) return false;
      const double hden = alpha * sqrt(rad) + gamma;
      if (hden < DBL_EPSILON) return false;
      const double h = (1.0 - alpha * alpha * beta * r2) / hden;
      if (h < DBL_EPSILON) return false;
      *u /= h; *v /= h;
      return true;
    }
    default: return false;
  }
}

extern "C" int b200gp_cam_ray_from_img(int model_id, const double* params, const double* xy, double* ray) {
  if (model_id < 0 || model_id > 17 || !params || !xy || !ray) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "cam_ray_from_img: bad arguments");
  if (model_id == 17) {   // EquirectangularCameraModel::CamRayFromImg (models.h:809-829)
    const double theta = 2.0 * M_PI * (xy[0] / params[0] - 0.5), phi = M_PI * (0.5 - xy[1] / params[1]);
    const double cp = cos(phi);
    ray[0] = cp * sin(theta); ray[1] = -sin(phi); ray[2] = cp * cos(theta);
    return 0;
  }
  double u = 0, v = 0;
  if (!gp_cam_from_img(model_id, params, xy[0], xy[1], &u, &v)) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "cam_ray_from_img: not unprojectable");
  const double n = sqrt(u * u + v * v + 1.0);
  ray[0] = u / n; ray[1] = v / n; ray[2] = 1.0 / n;
  return 0;
}

// ------------------------------------------------------------------------------------------------ device data
// Observations are in point-sorted order j.  Camera-side blocks: variable frames first, then sensors; block b owns
// columns 3b..3b+2 of the reduced system.  slot 0 of an observation is its frame block, slot 1 its sensor block (-1: none
// or constant).
struct GpDev {
  int64_t N, P; int F, S, nb, n, Npad, nvp;
  // static per observation
  const double *ray, *off, *R;        // R: world_from_rig (row-major) for sensor observations
  const double *w;                    // loss weight
  const int *fr, *sen, *blk;          // blk[2N]
  const int64_t *pt;                  // point index
  const uint8_t *svar;                // scale variable
  // per point (variable points with observations): obs range and point index
  const int64_t *vp_start, *vp_pt;    // [2 nvp]: [start, end) of each variable point's observations; [nvp]
  const int64_t *obs_vp;              // [N]: the variable point of an observation, -1 for a constant point
  // camera-side block lists: entries e in [bl_start[b], bl_start[b+1]) are (obs j, slot k) as 2j+k
  const int64_t *bl_start, *bl_ent;
  const int *blk_frame, *blk_sensor;  // block -> frame (or -1) / sensor (or -1)
  // state
  double *c, *X, *q, *s;              // current
  double *c2, *X2, *q2, *s2;          // candidate
  // linearisation
  double *r, *u, *js, *cost;          // r~ [3N], u = sqrt(w)*s [N], js = -sqrt(w) v [3N], cost [N]
  double *Dc, *Dp, *Ds;               // Jacobi scaling [n], [3P], [N]
  double *nc, *np, *ns;               // squared column norms of the unscaled Jacobian
  double *gc, *gp, *gs;               // unscaled gradient
  // elimination
  double *P9, *e, *Hss, *gss;         // per obs
  double *E, *Fm;                     // per obs and slot: 3x3 each, [18N]
  double *Hinv, *h, *gpt;             // per point index [9P], [3P], [3P]
  double *A, *rhs, *dC, *dX, *ds, *model;
  double *dinv; BaDenseFlag* flag;
  int* bad;
  unsigned long long* gmax;
  double* red;                        // reduction scratch
};

__device__ __forceinline__ double gp_clamp(double v, double lo, double hi) { return fmin(fmax(v, lo), hi); }

// residual, Huber corrector, cost of one observation at state (c, X, q, s)
__device__ void gp_residual(const GpDev& g, int64_t j, const double* c, const double* X, const double* q, const double* s,
                            double a, double* v, double* r, double* cost, double* sw) {
  const int f = g.fr[j], sn = g.sen[j]; const int64_t p = g.pt[j];
  double t[3];
  if (sn >= 0) {
    const double* R = g.R + 9 * j;
    for (int m = 0; m < 3; ++m) t[m] = -(R[3 * m] * q[3 * sn] + R[3 * m + 1] * q[3 * sn + 1] + R[3 * m + 2] * q[3 * sn + 2]);
  } else {
    for (int m = 0; m < 3; ++m) t[m] = g.off[3 * j + m];
  }
  const double sc = s[j];
  for (int m = 0; m < 3; ++m) { v[m] = X[3 * p + m] - c[3 * f + m] + t[m]; r[m] = g.ray[3 * j + m] - sc * v[m]; }
  const double s2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
  double rho0, rho1;
  if (s2 > a * a) { const double rr = sqrt(s2); rho0 = 2.0 * a * rr - a * a; rho1 = fmax(DBL_MIN, a / rr); }
  else { rho0 = s2; rho1 = 1.0; }
  const double lam = g.w[j];
  *cost = 0.5 * lam * rho0;
  *sw = sqrt(lam * rho1);   // Corrector: rho'' <= 0 for Huber, so the Jacobian and residual scale by sqrt(rho')
}

__global__ void k_linearize(GpDev g, int candidate, double a) {
  const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= g.N) return;
  double v[3], r[3], cost, sw;
  if (candidate) { gp_residual(g, j, g.c2, g.X2, g.q2, g.s2, a, v, r, &cost, &sw); g.cost[j] = cost; return; }
  gp_residual(g, j, g.c, g.X, g.q, g.s, a, v, r, &cost, &sw);
  g.cost[j] = cost;
  g.u[j] = sw * g.s[j];
  for (int m = 0; m < 3; ++m) { g.r[3 * j + m] = sw * r[m]; g.js[3 * j + m] = -sw * v[m]; }
}

// unscaled Jacobian of slot k of observation j (3x3 row-major), without the column scaling
__device__ __forceinline__ void gp_slot_jac(const GpDev& g, int64_t j, int k, double* J) {
  const double u = g.u[j];
  if (k == 0) { for (int m = 0; m < 9; ++m) J[m] = 0.0; J[0] = J[4] = J[8] = u; }
  else { const double* R = g.R + 9 * j; for (int m = 0; m < 9; ++m) J[m] = u * R[m]; }
}

__device__ __forceinline__ void gp_atomic_max(unsigned long long* m, double v) {
  atomicMax(m, (unsigned long long)__double_as_longlong(fabs(v)));   // non-negative doubles order as their bits
}

// column norms and gradient of the unscaled Jacobian: camera-side rows
__global__ void k_cam_stats(GpDev g) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.n) return;
  const int b = i / 3, a = i % 3;
  double nn = 0, gg = 0, J[9];
  for (int64_t e = g.bl_start[b]; e < g.bl_start[b + 1]; ++e) {
    const int64_t j = g.bl_ent[e] >> 1; const int k = (int)(g.bl_ent[e] & 1);
    gp_slot_jac(g, j, k, J);
    for (int m = 0; m < 3; ++m) { nn += J[3 * m + a] * J[3 * m + a]; gg += J[3 * m + a] * g.r[3 * j + m]; }
  }
  g.nc[i] = nn; g.gc[i] = gg;
  gp_atomic_max(g.gmax, gg);
}

__global__ void k_point_stats(GpDev g) {
  const int64_t vp = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (vp >= g.nvp) return;
  const int64_t p = g.vp_pt[vp];
  double nn = 0, gg[3] = {0, 0, 0};
  for (int64_t j = g.vp_start[2 * vp]; j < g.vp_start[2 * vp + 1]; ++j) {
    const double u = g.u[j];
    nn += u * u;
    for (int m = 0; m < 3; ++m) gg[m] += -u * g.r[3 * j + m];
  }
  for (int m = 0; m < 3; ++m) { g.np[3 * p + m] = nn; g.gp[3 * p + m] = gg[m]; gp_atomic_max(g.gmax, gg[m]); }
}

__global__ void k_scale_stats(GpDev g) {
  const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= g.N || !g.svar[j]) return;
  const double* js = g.js + 3 * j; const double* r = g.r + 3 * j;
  const double gg = js[0] * r[0] + js[1] * r[1] + js[2] * r[2];
  g.ns[j] = js[0] * js[0] + js[1] * js[1] + js[2] * js[2]; g.gs[j] = gg;
  // projected gradient under the lower bound: x - max(x - g, lb)
  const double x = g.s[j];
  gp_atomic_max(g.gmax, x - fmax(x - gg, B200GP_SCALE_LOWER_BOUND));
}

__global__ void k_jacobi(double* D, const double* nrm, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) D[i] = 1.0 / (1.0 + sqrt(nrm[i]));
}

// per observation: eliminate the scale; P = I - j j^T / H_ss, e = r~ - j g_s / H_ss (scaled j)
__global__ void k_obs_elim(GpDev g, double radius, double dmin, double dmax) {
  const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= g.N) return;
  double* P = g.P9 + 9 * j; double* e = g.e + 3 * j; const double* r = g.r + 3 * j;
  for (int m = 0; m < 9; ++m) P[m] = (m % 4 == 0) ? 1.0 : 0.0;
  for (int m = 0; m < 3; ++m) e[m] = r[m];
  if (!g.svar[j]) return;
  const double D = g.Ds[j];
  const double jv[3] = {D * g.js[3 * j], D * g.js[3 * j + 1], D * g.js[3 * j + 2]};
  const double d2 = jv[0] * jv[0] + jv[1] * jv[1] + jv[2] * jv[2];
  const double H = d2 + gp_clamp(d2, dmin, dmax) / radius;
  const double gs = jv[0] * r[0] + jv[1] * r[1] + jv[2] * r[2];
  g.Hss[j] = H; g.gss[j] = gs;
  for (int m = 0; m < 3; ++m) { e[m] -= jv[m] * gs / H; for (int n = 0; n < 3; ++n) P[3 * m + n] -= jv[m] * jv[n] / H; }
}

// scaled slot Jacobian: J * diag(D of the block's columns)
__device__ __forceinline__ void gp_slot_jac_scaled(const GpDev& g, int64_t j, int k, double* J) {
  gp_slot_jac(g, j, k, J);
  const int b = g.blk[2 * j + k];
  for (int m = 0; m < 3; ++m) for (int c = 0; c < 3; ++c) J[3 * m + c] *= g.Dc[3 * b + c];
}

// per variable point: H_pp, its inverse, h = H^-1 g_p, and for every (observation, slot) E = J_X^T P J_k, F = H^-1 E
__global__ void k_point(GpDev g, double radius, double dmin, double dmax) {
  const int64_t vp = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (vp >= g.nvp) return;
  const int64_t p = g.vp_pt[vp];
  const double Dp[3] = {g.Dp[3 * p], g.Dp[3 * p + 1], g.Dp[3 * p + 2]};
  double H[9] = {0}, gv[3] = {0, 0, 0};
  for (int64_t j = g.vp_start[2 * vp]; j < g.vp_start[2 * vp + 1]; ++j) {
    const double u = g.u[j]; const double* P = g.P9 + 9 * j; const double* e = g.e + 3 * j;
    // J_X = -u diag(Dp)
    for (int a = 0; a < 3; ++a) {
      for (int b = 0; b < 3; ++b) H[3 * a + b] += u * u * Dp[a] * Dp[b] * P[3 * a + b];
      gv[a] += -u * Dp[a] * e[a];
    }
  }
  for (int a = 0; a < 3; ++a) H[4 * a] += gp_clamp(Dp[a] * Dp[a] * g.np[3 * p + a], dmin, dmax) / radius;
  // symmetric 3x3 inverse by cofactors
  const double c00 = H[4] * H[8] - H[5] * H[7], c01 = H[5] * H[6] - H[3] * H[8], c02 = H[3] * H[7] - H[4] * H[6];
  const double det = H[0] * c00 + H[1] * c01 + H[2] * c02;
  if (!(det > 0.0) || !(H[0] > 0.0)) { *g.bad = 1; return; }
  double* Hi = g.Hinv + 9 * p;
  const double id = 1.0 / det;
  Hi[0] = c00 * id; Hi[1] = (H[2] * H[7] - H[1] * H[8]) * id; Hi[2] = (H[1] * H[5] - H[2] * H[4]) * id;
  Hi[3] = c01 * id; Hi[4] = (H[0] * H[8] - H[2] * H[6]) * id; Hi[5] = (H[2] * H[3] - H[0] * H[5]) * id;
  Hi[6] = c02 * id; Hi[7] = (H[1] * H[6] - H[0] * H[7]) * id; Hi[8] = (H[0] * H[4] - H[1] * H[3]) * id;
  for (int a = 0; a < 3; ++a) { g.gpt[3 * p + a] = gv[a]; g.h[3 * p + a] = Hi[3 * a] * gv[0] + Hi[3 * a + 1] * gv[1] + Hi[3 * a + 2] * gv[2]; }
  for (int64_t j = g.vp_start[2 * vp]; j < g.vp_start[2 * vp + 1]; ++j) {
    const double u = g.u[j]; const double* P = g.P9 + 9 * j;
    for (int k = 0; k < 2; ++k) {
      if (g.blk[2 * j + k] < 0) continue;
      double J[9], E[9];
      gp_slot_jac_scaled(g, j, k, J);
      for (int a = 0; a < 3; ++a)
        for (int c = 0; c < 3; ++c) {
          double t = 0;
          for (int m = 0; m < 3; ++m) t += P[3 * a + m] * J[3 * m + c];
          E[3 * a + c] = -u * Dp[a] * t;
        }
      double* Eo = g.E + 18 * j + 9 * k; double* Fo = g.Fm + 18 * j + 9 * k;
      for (int m = 0; m < 9; ++m) Eo[m] = E[m];
      for (int a = 0; a < 3; ++a)
        for (int c = 0; c < 3; ++c) Fo[3 * a + c] = Hi[3 * a] * E[c] + Hi[3 * a + 1] * E[3 + c] + Hi[3 * a + 2] * E[6 + c];
    }
  }
}

// one thread per row i of the reduced system: S(i, :) and rhs(i), column-major A[col * Npad + i]
__global__ void k_rows(GpDev g, double radius, double dmin, double dmax, const uint8_t* pvar) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.n) return;
  const int b = i / 3, a = i % 3;
  double* A = g.A; const int64_t N = g.Npad;
  double rhs = 0.0, J[9], J2[9];
  for (int64_t e = g.bl_start[b]; e < g.bl_start[b + 1]; ++e) {
    const int64_t j = g.bl_ent[e] >> 1; const int k = (int)(g.bl_ent[e] & 1);
    const double* P = g.P9 + 9 * j; const double* ev = g.e + 3 * j;
    gp_slot_jac_scaled(g, j, k, J);
    double PJa[3];   // (P J_k)[:, a]... row vector J_k[:, a]^T P
    for (int n = 0; n < 3; ++n) PJa[n] = J[a] * P[n] + J[3 + a] * P[3 + n] + J[6 + a] * P[6 + n];
    rhs -= J[a] * ev[0] + J[3 + a] * ev[1] + J[6 + a] * ev[2];
    for (int k2 = 0; k2 < 2; ++k2) {
      const int b2 = g.blk[2 * j + k2];
      if (b2 < 0) continue;
      gp_slot_jac_scaled(g, j, k2, J2);
      for (int c = 0; c < 3; ++c) A[(int64_t)(3 * b2 + c) * N + i] += PJa[0] * J2[c] + PJa[1] * J2[3 + c] + PJa[2] * J2[6 + c];
    }
    const int64_t p = g.pt[j];
    if (!pvar[p]) continue;
    const double* E = g.E + 18 * j + 9 * k;
    rhs += E[a] * g.h[3 * p] + E[3 + a] * g.h[3 * p + 1] + E[6 + a] * g.h[3 * p + 2];
    const int64_t vp = g.obs_vp[j];
    for (int64_t j2 = g.vp_start[2 * vp]; j2 < g.vp_start[2 * vp + 1]; ++j2)
      for (int k2 = 0; k2 < 2; ++k2) {
        const int b2 = g.blk[2 * j2 + k2];
        if (b2 < 0) continue;
        const double* F = g.Fm + 18 * j2 + 9 * k2;
        for (int c = 0; c < 3; ++c) A[(int64_t)(3 * b2 + c) * N + i] -= E[a] * F[c] + E[3 + a] * F[3 + c] + E[6 + a] * F[6 + c];
      }
  }
  A[(int64_t)i * N + i] += gp_clamp(g.Dc[i] * g.Dc[i] * g.nc[i], dmin, dmax) / radius;
  g.rhs[i] = rhs;
}

// back-substitution to the points: dX = H^-1 (-g_p - sum E dC)
__global__ void k_back_points(GpDev g) {
  const int64_t vp = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (vp >= g.nvp) return;
  const int64_t p = g.vp_pt[vp];
  double t[3] = {-g.gpt[3 * p], -g.gpt[3 * p + 1], -g.gpt[3 * p + 2]};
  for (int64_t j = g.vp_start[2 * vp]; j < g.vp_start[2 * vp + 1]; ++j)
    for (int k = 0; k < 2; ++k) {
      const int b = g.blk[2 * j + k];
      if (b < 0) continue;
      const double* E = g.E + 18 * j + 9 * k; const double* d = g.dC + 3 * b;
      for (int a = 0; a < 3; ++a) t[a] -= E[3 * a] * d[0] + E[3 * a + 1] * d[1] + E[3 * a + 2] * d[2];
    }
  const double* Hi = g.Hinv + 9 * p;
  for (int a = 0; a < 3; ++a) g.dX[3 * p + a] = Hi[3 * a] * t[0] + Hi[3 * a + 1] * t[1] + Hi[3 * a + 2] * t[2];
}

// back-substitution to the scales, the model cost change per observation, and the candidate scale
__global__ void k_back_obs(GpDev g, const uint8_t* pvar) {
  const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= g.N) return;
  double y[3] = {0, 0, 0}, J[9];
  for (int k = 0; k < 2; ++k) {
    const int b = g.blk[2 * j + k];
    if (b < 0) continue;
    gp_slot_jac_scaled(g, j, k, J);
    const double* d = g.dC + 3 * b;
    for (int m = 0; m < 3; ++m) y[m] += J[3 * m] * d[0] + J[3 * m + 1] * d[1] + J[3 * m + 2] * d[2];
  }
  const int64_t p = g.pt[j];
  if (pvar[p]) { const double u = g.u[j]; for (int m = 0; m < 3; ++m) y[m] += -u * g.Dp[3 * p + m] * g.dX[3 * p + m]; }
  const double* r = g.r + 3 * j;
  g.s2[j] = g.s[j];
  if (g.svar[j]) {
    const double D = g.Ds[j];
    const double jv[3] = {D * g.js[3 * j], D * g.js[3 * j + 1], D * g.js[3 * j + 2]};
    const double ds = (-g.gss[j] - (jv[0] * y[0] + jv[1] * y[1] + jv[2] * y[2])) / g.Hss[j];
    for (int m = 0; m < 3; ++m) y[m] += jv[m] * ds;
    g.s2[j] = fmax(g.s[j] + D * ds, B200GP_SCALE_LOWER_BOUND);   // ParameterBlock::Plus clamps to the bound
  }
  g.model[j] = -(y[0] * (r[0] + 0.5 * y[0]) + y[1] * (r[1] + 0.5 * y[1]) + y[2] * (r[2] + 0.5 * y[2]));
}

__global__ void k_update_blocks(GpDev g, const uint8_t* pvar) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < g.n) {
    const int b = (int)(i / 3), a = (int)(i % 3);
    const double d = g.Dc[i] * g.dC[i];
    if (g.blk_frame[b] >= 0) g.c2[3 * g.blk_frame[b] + a] = g.c[3 * g.blk_frame[b] + a] + d;
    else g.q2[3 * g.blk_sensor[b] + a] = g.q[3 * g.blk_sensor[b] + a] + d;
  }
  if (i < 3 * g.P) { const int64_t p = i / 3; g.X2[i] = pvar[p] ? g.X[i] + g.Dp[i] * g.dX[i] : g.X[i]; }
}


// ------------------------------------------------------------------------------------------------ host
#define GP_RG 512   // CTAs of the deterministic sums

// options and problem checks, host only
static int gp_check(const b200gp_options* o, const b200gp_problem* p) {
  if (!(o->loss_function_scale > 0) || !std::isfinite(o->loss_function_scale)) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "loss_function_scale must be positive");
  if (o->max_num_iterations < 0 || !(o->function_tolerance >= 0) || !(o->gradient_tolerance >= 0) || !(o->parameter_tolerance >= 0) ||
      !(o->initial_trust_region_radius > 0) || !(o->max_trust_region_radius >= o->initial_trust_region_radius) ||
      !(o->min_trust_region_radius >= 0) || !(o->min_lm_diagonal > 0) || !(o->max_lm_diagonal >= o->min_lm_diagonal) ||
      !(o->min_relative_decrease >= 0))
    return solver_fail(g_gp_err, B200GP_ERR_INPUT, "invalid solver options");
  const int F = p->num_frames, S = p->num_sensors; const int64_t P = p->num_points, N = p->num_observations;
  if (F < 0 || S < 0 || P < 0 || N < 0) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "negative size");
  if ((F && !p->frame_centers) || (P && !p->points) || (S && !p->cams_in_rig) ||
      (N && (!p->obs_frame || !p->obs_point || !p->obs_ray || !p->obs_scale)))
    return solver_fail(g_gp_err, B200GP_ERR_INPUT, "missing array");
  if (!all_finite(p->frame_centers, 3LL * F)) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "non-finite frame centre");
  if (!all_finite(p->points, 3 * P)) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "non-finite point");
  if (!all_finite(p->cams_in_rig, 3LL * S)) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "non-finite camera-in-rig position");
  if (!all_finite(p->obs_ray, 3 * N)) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "non-finite ray");
  if (p->obs_rig_offset && !all_finite(p->obs_rig_offset, 3 * N)) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "non-finite rig offset");
  for (int64_t j = 0; j < N; ++j) {
    const int f = p->obs_frame[j]; const int64_t q = p->obs_point[j]; const int s = p->obs_sensor ? p->obs_sensor[j] : -1;
    if (f < 0 || f >= F) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "observation %lld: frame %d out of range", (long long)j, f);
    if (q < 0 || q >= P) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "observation %lld: point %lld out of range", (long long)j, (long long)q);
    if (s < -1 || s >= S) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "observation %lld: sensor %d out of range", (long long)j, s);
    if (s >= 0 && !o->refine_sensor_from_rig)
      return solver_fail(g_gp_err, B200GP_ERR_INPUT, "observation %lld: variable camera-in-rig position but refine_sensor_from_rig = 0", (long long)j);
    if (s >= 0 && !p->world_from_rig) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "world_from_rig is needed for sensor observations");
    if (s >= 0 && !all_finite(p->world_from_rig + 9LL * f, 9)) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "non-finite world_from_rig of frame %d", f);
    const double sc = p->obs_scale[j];
    if (!std::isfinite(sc) || sc < B200GP_SCALE_LOWER_BOUND) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "observation %lld: scale %g below the bound 1e-5 or not finite", (long long)j, sc);
    const double w = p->obs_loss_weight ? p->obs_loss_weight[j] : 1.0;
    if (!(w > 0) || !std::isfinite(w)) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "observation %lld: loss weight must be positive", (long long)j);
  }
  return 0;
}

// The device layout of a checked problem: variable blocks, and the observations sorted by point with the per-point
// ranges and the block -> (observation, slot) lists of GpDev.
struct GpLayout {
  int nb, n, Npad;
  int64_t nvp;
  std::vector<int> fblk, sblk, blk_frame, blk_sensor;   // frame / sensor -> block (-1: constant), block -> frame / sensor
  std::vector<uint8_t> pvar, fmask, sensor_used;        // variable points, variable frames, variable sensors
  std::vector<int64_t> perm;                            // sorted position -> caller's observation
  std::vector<double> ray, off, R, w, s;
  std::vector<int> fr, sen, blk;
  std::vector<int64_t> pt, vp_start, vp_pt, obs_vp, bl_start, bl_ent;
  std::vector<uint8_t> svar;
};

static int gp_layout(const b200gp_options* o, const b200gp_problem* p, GpLayout& L) {
  const int F = p->num_frames, S = p->num_sensors; const int64_t P = p->num_points, N = p->num_observations;
  std::vector<uint8_t> frame_used(F, 0), point_used(P, 0);
  L.sensor_used.assign(S, 0);
  for (int64_t j = 0; j < N; ++j) {
    frame_used[p->obs_frame[j]] = 1; point_used[p->obs_point[j]] = 1;
    if (p->obs_sensor && p->obs_sensor[j] >= 0) L.sensor_used[p->obs_sensor[j]] = 1;
  }
  // ---- variable blocks
  L.fblk.assign(F, -1); L.sblk.assign(S, -1);
  for (int f = 0; f < F; ++f)
    if (frame_used[f] && o->optimize_positions && !(p->frame_constant && p->frame_constant[f])) { L.fblk[f] = (int)L.blk_frame.size(); L.blk_frame.push_back(f); L.blk_sensor.push_back(-1); }
  for (int s = 0; s < S; ++s)
    if (L.sensor_used[s]) { L.sblk[s] = (int)L.blk_frame.size(); L.blk_frame.push_back(-1); L.blk_sensor.push_back(s); }
  const int nb = (int)L.blk_frame.size();
  if (3LL * nb > B200GP_MAX_REDUCED_DIM)
    return solver_fail(g_gp_err, B200GP_ERR_TOO_LARGE, "reduced dimension %lld exceeds the dense limit %d (a sparse reduced solve is not implemented)", 3LL * nb, B200GP_MAX_REDUCED_DIM);
  L.nb = nb; L.n = 3 * nb; L.Npad = (L.n + BA_TILE - 1) / BA_TILE * BA_TILE;
  L.pvar.assign(P, 0);
  for (int64_t q = 0; q < P; ++q) L.pvar[q] = point_used[q] && o->optimize_points;
  L.fmask.assign(F, 0);
  for (int f = 0; f < F; ++f) L.fmask[f] = L.fblk[f] >= 0;
  // ---- sort observations by point (stable)
  L.perm.resize(N);
  for (int64_t j = 0; j < N; ++j) L.perm[j] = j;
  std::stable_sort(L.perm.begin(), L.perm.end(), [&](int64_t a, int64_t b) { return p->obs_point[a] < p->obs_point[b]; });
  L.ray.resize(3 * N); L.off.assign(3 * N, 0.0); L.R.assign(9 * N, 0.0); L.w.resize(N); L.s.resize(N);
  L.fr.resize(N); L.sen.resize(N); L.blk.resize(2 * N); L.pt.resize(N); L.svar.resize(N);
  L.bl_start.assign(nb + 1, 0);
  std::vector<int64_t> vp_first;
  for (int64_t j = 0; j < N; ++j) {
    const int64_t o_ = L.perm[j];
    const int f = p->obs_frame[o_], s = p->obs_sensor ? p->obs_sensor[o_] : -1;
    for (int m = 0; m < 3; ++m) { L.ray[3 * j + m] = p->obs_ray[3 * o_ + m]; if (s < 0 && p->obs_rig_offset) L.off[3 * j + m] = p->obs_rig_offset[3 * o_ + m]; }
    if (s >= 0) for (int m = 0; m < 9; ++m) L.R[9 * j + m] = p->world_from_rig[9LL * f + m];
    L.w[j] = p->obs_loss_weight ? p->obs_loss_weight[o_] : 1.0;
    L.s[j] = p->obs_scale[o_];
    L.fr[j] = f; L.sen[j] = s; L.pt[j] = p->obs_point[o_];
    L.blk[2 * j] = L.fblk[f]; L.blk[2 * j + 1] = s >= 0 ? L.sblk[s] : -1;
    L.svar[j] = o->optimize_scales && o_ != 0;
    for (int k = 0; k < 2; ++k) if (L.blk[2 * j + k] >= 0) L.bl_start[L.blk[2 * j + k] + 1]++;
    if (L.pvar[L.pt[j]] && (j == 0 || L.pt[j - 1] != L.pt[j])) { vp_first.push_back(j); L.vp_pt.push_back(L.pt[j]); }
  }
  const int64_t nvp = (int64_t)L.vp_pt.size();
  L.nvp = nvp;
  // [start, end) per variable point: a point's observations are contiguous in the sorted order
  L.vp_start.assign(std::max<int64_t>(1, 2 * nvp), 0);
  for (int64_t k = 0; k < nvp; ++k) {
    int64_t e = vp_first[k];
    while (e < N && L.pt[e] == L.vp_pt[k]) ++e;
    L.vp_start[2 * k] = vp_first[k]; L.vp_start[2 * k + 1] = e;
  }
  L.obs_vp.assign(N, -1);
  for (int64_t k = 0; k < nvp; ++k) for (int64_t j = L.vp_start[2 * k]; j < L.vp_start[2 * k + 1]; ++j) L.obs_vp[j] = k;
  for (int b = 0; b < nb; ++b) L.bl_start[b + 1] += L.bl_start[b];
  L.bl_ent.assign(std::max<int64_t>(1, L.bl_start[nb]), 0);
  std::vector<int64_t> fill(L.bl_start.begin(), L.bl_start.end() - 1);
  for (int64_t j = 0; j < N; ++j) for (int k = 0; k < 2; ++k) { const int b = L.blk[2 * j + k]; if (b >= 0) L.bl_ent[fill[b]++] = 2 * j + k; }
  return 0;
}

// The LM solve (Levenberg-Marquardt with Ceres' trust-region rules) on the device state g.  Every method returns 0 or
// B200GP_ERR_CUDA.
struct GpSolve {
  const b200gp_options* o;
  b200gp_summary* out;
  GpDev g;
  uint8_t *pvar, *fmask, *qmask, *smask;   // variable points, frames, sensors and scales

  // deterministic sum of cnt terms (solver_sum mode) into *r
  int dsum(int mode, const double* x, const double* y, const uint8_t* mask, int stride, int64_t cnt, double* r) {
    *r = 0.0;
    if (cnt <= 0) return 0;
    solver_sum<GP_RG>(mode, x, y, mask, stride, cnt, g.red, g.red + GP_RG);
    GP_CHECK(cudaMemcpy(r, g.red + GP_RG, sizeof(double), cudaMemcpyDeviceToHost));
    return 0;
  }
  // residuals and Jacobian factors at the current state, and its cost
  int linearize(double* cost) {
    k_linearize<<<grid_blocks(g.N, 256), 256>>>(g, 0, o->loss_function_scale);
    return dsum(SOLVER_SUM, g.cost, nullptr, nullptr, 1, g.N, cost);
  }
  // column norms and gradient of the unscaled Jacobian, and the max norm of the projected gradient
  int stats(double* gnorm) {
    GP_CHECK(cudaMemset(g.gmax, 0, sizeof(unsigned long long)));
    if (g.n) k_cam_stats<<<grid_blocks(g.n, 128), 128>>>(g);
    if (g.nvp) k_point_stats<<<grid_blocks(g.nvp, 128), 128>>>(g);
    k_scale_stats<<<grid_blocks(g.N, 256), 256>>>(g);
    unsigned long long m = 0;
    GP_CHECK(cudaMemcpy(&m, g.gmax, sizeof m, cudaMemcpyDeviceToHost));
    memcpy(gnorm, &m, sizeof m);
    return 0;
  }
  // norm of the variable parameters
  int xnorm(double* r) {
    double c, X, q, sc;
    SOLVER_TRY(dsum(SOLVER_SUM_SQ, g.c, nullptr, fmask, 3, 3LL * g.F, &c));
    SOLVER_TRY(dsum(SOLVER_SUM_SQ, g.X, nullptr, pvar, 3, 3 * g.P, &X));
    SOLVER_TRY(dsum(SOLVER_SUM_SQ, g.q, nullptr, qmask, 3, 3LL * g.S, &q));
    SOLVER_TRY(dsum(SOLVER_SUM_SQ, g.s, nullptr, smask, 1, g.N, &sc));
    *r = sqrt(c + X + q + sc);
    return 0;
  }
  // One inner step at this radius: eliminate the scales and points, build, factor and solve the reduced system,
  // back-substitute, and the model cost change (0 unless *ok: no failed elimination or pivot).
  int step(double radius, bool* ok, double* model) {
    const double dmin = o->min_lm_diagonal, dmax = o->max_lm_diagonal;
    const int n = g.n, Npad = g.Npad;
    int zero = 0;
    GP_CHECK(cudaMemcpy(g.bad, &zero, sizeof(int), cudaMemcpyHostToDevice));
    k_obs_elim<<<grid_blocks(g.N, 256), 256>>>(g, radius, dmin, dmax);
    if (g.nvp) k_point<<<grid_blocks(g.nvp, 128), 128>>>(g, radius, dmin, dmax);
    BaDenseFlag fl{0, 0, 0.0};
    GP_CHECK(cudaMemcpy(g.flag, &fl, sizeof fl, cudaMemcpyHostToDevice));
    if (n) {
      GP_CHECK(cudaMemset(g.A, 0, sizeof(double) * (size_t)Npad * Npad));
      GP_CHECK(cudaMemset(g.rhs, 0, sizeof(double) * Npad));
      k_rows<<<grid_blocks(n, 64), 64>>>(g, radius, dmin, dmax, pvar);
      GP_CHECK(ba_dense_pad_identity(g.A, Npad, n, 0));
      GP_CHECK(cudaMemcpy(g.dC, g.rhs, sizeof(double) * Npad, cudaMemcpyDeviceToDevice));
      GP_CHECK(ba_dense_potrf(g.A, Npad, n, n, 0.0, g.dinv, g.flag, 0));
      // b in dC, the solution back into dC; rhs is the scratch
      GP_CHECK(ba_dense_potrs(g.A, Npad, g.dinv, 1, g.dC, g.rhs, g.flag, 0));
    }
    if (g.nvp) k_back_points<<<grid_blocks(g.nvp, 128), 128>>>(g);
    k_back_obs<<<grid_blocks(g.N, 256), 256>>>(g, pvar);
    GP_CHECK(cudaGetLastError());
    int bad = 0;
    GP_CHECK(cudaMemcpy(&bad, g.bad, sizeof(int), cudaMemcpyDeviceToHost));
    GP_CHECK(cudaMemcpy(&fl, g.flag, sizeof fl, cudaMemcpyDeviceToHost));
    *ok = !bad && !fl.bad;
    *model = 0;
    return *ok ? dsum(SOLVER_SUM, g.model, nullptr, nullptr, 1, g.N, model) : 0;
  }
  // The candidate state from the step, its cost and the step norm.
  int candidate(double* new_cost, double* step_norm) {
    k_update_blocks<<<grid_blocks(std::max<int64_t>(g.n, 3 * g.P), 256), 256>>>(g, pvar);
    k_linearize<<<grid_blocks(g.N, 256), 256>>>(g, 1, o->loss_function_scale);
    SOLVER_TRY(dsum(SOLVER_SUM, g.cost, nullptr, nullptr, 1, g.N, new_cost));
    double c, X, q, sc;
    SOLVER_TRY(dsum(SOLVER_SUM_SQDIFF, g.c2, g.c, fmask, 3, 3LL * g.F, &c));
    SOLVER_TRY(dsum(SOLVER_SUM_SQDIFF, g.X2, g.X, pvar, 3, 3 * g.P, &X));
    SOLVER_TRY(dsum(SOLVER_SUM_SQDIFF, g.q2, g.q, qmask, 3, 3LL * g.S, &q));
    SOLVER_TRY(dsum(SOLVER_SUM_SQDIFF, g.s2, g.s, smask, 1, g.N, &sc));
    *step_norm = sqrt(c + X + q + sc);
    return 0;
  }
  // the candidate becomes the current state, and the next candidate starts from it
  int accept() {
    std::swap(g.c, g.c2); std::swap(g.X, g.X2); std::swap(g.q, g.q2); std::swap(g.s, g.s2);
    GP_CHECK(cudaMemcpy(g.c2, g.c, sizeof(double) * 3 * g.F, cudaMemcpyDeviceToDevice));
    GP_CHECK(cudaMemcpy(g.X2, g.X, sizeof(double) * 3 * g.P, cudaMemcpyDeviceToDevice));
    if (g.S) GP_CHECK(cudaMemcpy(g.q2, g.q, sizeof(double) * 3 * g.S, cudaMemcpyDeviceToDevice));
    return 0;
  }
  // The LM iterations from the uploaded state.  Sets the termination type, the step counts and the cost history, and
  // leaves the last accepted state in (c, X, q, s) and its cost in *cost.
  int minimize(double* cost) {
    SOLVER_TRY(linearize(cost));
    out->initial_cost = *cost;
    if (out->cost_history) out->cost_history[0] = *cost;
    double radius = o->initial_trust_region_radius, decrease_factor = 2.0;
    int iter = 0;
    out->termination_type = B200GP_NO_CONVERGENCE;
    double gnorm;
    SOLVER_TRY(stats(&gnorm));
    if (g.n) k_jacobi<<<grid_blocks(g.n, 256), 256>>>(g.Dc, g.nc, g.n);
    if (g.P) k_jacobi<<<grid_blocks(3 * g.P, 256), 256>>>(g.Dp, g.np, 3 * g.P);
    k_jacobi<<<grid_blocks(g.N, 256), 256>>>(g.Ds, g.ns, g.N);
    for (;;) {
      if (gnorm <= o->gradient_tolerance) { out->termination_type = B200GP_CONVERGENCE; return 0; }
      double x_norm;   // constant in the inner loop
      SOLVER_TRY(xnorm(&x_norm));
      bool accepted = false;
      while (!accepted) {
        if (iter >= o->max_num_iterations) return 0;
        ++iter;
        bool ok; double model;
        SOLVER_TRY(step(radius, &ok, &model));
        double new_cost = *cost, rho = 0;
        if (ok && model > 0) {
          double step_norm;
          SOLVER_TRY(candidate(&new_cost, &step_norm));
          rho = (*cost - new_cost) / model;
          // ParameterToleranceReached, then FunctionToleranceReached (checked on every step, as Ceres does); a converged
          // candidate is not taken: Ceres returns with the last accepted parameters
          if (step_norm / (x_norm + o->parameter_tolerance) <= o->parameter_tolerance ||
              fabs(*cost - new_cost) <= o->function_tolerance * *cost) {
            out->termination_type = B200GP_CONVERGENCE;
            if (out->cost_history) out->cost_history[iter] = *cost;
            out->num_iterations = iter;
            return 0;
          }
        }
        if (ok && model > 0 && rho > o->min_relative_decrease) {
          accepted = true;
          out->num_successful_steps++;
          SOLVER_TRY(accept());
          SOLVER_TRY(linearize(cost));
          SOLVER_TRY(stats(&gnorm));
          const double t = 2.0 * rho - 1.0;
          radius = std::min(o->max_trust_region_radius, radius / std::max(1.0 / 3.0, 1.0 - t * t * t));
          decrease_factor = 2.0;
        } else {
          out->num_unsuccessful_steps++;
          radius /= decrease_factor;
          decrease_factor *= 2.0;
        }
        if (out->cost_history) out->cost_history[iter] = *cost;
        out->num_iterations = iter;
        if (!accepted && radius < o->min_trust_region_radius) { out->termination_type = B200GP_CONVERGENCE; return 0; }
      }
    }
  }
};

// GpDev's buffers: the layout and the initial state uploaded (current and candidate), the work arrays allocated
static int gp_upload(const b200gp_problem* p, const GpLayout& L, SolverBuffers& pool, GpSolve& s) {
  const int F = p->num_frames, S = p->num_sensors; const int64_t P = p->num_points, N = p->num_observations;
  const int n = L.n, Npad = L.Npad;
  GpDev& g = s.g;
  memset(&g, 0, sizeof g);
  g.N = N; g.P = P; g.F = F; g.S = S; g.nb = L.nb; g.n = n; g.Npad = Npad; g.nvp = L.nvp;
  const std::vector<double> hc(p->frame_centers, p->frame_centers + 3LL * F), hX(p->points, p->points + 3 * P),
      hq(p->cams_in_rig ? p->cams_in_rig : nullptr, p->cams_in_rig ? p->cams_in_rig + 3LL * S : nullptr);
  GP_CHECK(pool.upload(&g.ray, L.ray)); GP_CHECK(pool.upload(&g.off, L.off)); GP_CHECK(pool.upload(&g.R, L.R));
  GP_CHECK(pool.upload(&g.w, L.w)); GP_CHECK(pool.upload(&g.fr, L.fr)); GP_CHECK(pool.upload(&g.sen, L.sen));
  GP_CHECK(pool.upload(&g.blk, L.blk)); GP_CHECK(pool.upload(&g.pt, L.pt)); GP_CHECK(pool.upload(&g.svar, L.svar));
  GP_CHECK(pool.upload(&g.vp_start, L.vp_start)); GP_CHECK(pool.upload(&g.vp_pt, L.vp_pt));
  GP_CHECK(pool.upload(&g.obs_vp, L.obs_vp));
  GP_CHECK(pool.upload(&g.bl_start, L.bl_start)); GP_CHECK(pool.upload(&g.bl_ent, L.bl_ent));
  GP_CHECK(pool.upload(&g.blk_frame, L.blk_frame)); GP_CHECK(pool.upload(&g.blk_sensor, L.blk_sensor));
  GP_CHECK(pool.upload(&g.c, hc)); GP_CHECK(pool.upload(&g.X, hX)); GP_CHECK(pool.upload(&g.q, hq)); GP_CHECK(pool.upload(&g.s, L.s));
  GP_CHECK(pool.upload(&g.c2, hc)); GP_CHECK(pool.upload(&g.X2, hX)); GP_CHECK(pool.upload(&g.q2, hq)); GP_CHECK(pool.upload(&g.s2, L.s));
  GP_CHECK(pool.upload(&s.pvar, L.pvar)); GP_CHECK(pool.upload(&s.fmask, L.fmask)); GP_CHECK(pool.upload(&s.qmask, L.sensor_used));
  GP_CHECK(pool.upload(&s.smask, L.svar));
  GP_CHECK(pool.alloc(&g.r, 3 * N)); GP_CHECK(pool.alloc(&g.u, N)); GP_CHECK(pool.alloc(&g.js, 3 * N)); GP_CHECK(pool.alloc(&g.cost, N));
  GP_CHECK(pool.alloc(&g.Dc, n)); GP_CHECK(pool.alloc(&g.Dp, 3 * P)); GP_CHECK(pool.alloc(&g.Ds, N));
  GP_CHECK(pool.alloc(&g.nc, n)); GP_CHECK(pool.alloc(&g.np, 3 * P)); GP_CHECK(pool.alloc(&g.ns, N));
  GP_CHECK(pool.alloc(&g.gc, n)); GP_CHECK(pool.alloc(&g.gp, 3 * P)); GP_CHECK(pool.alloc(&g.gs, N));
  GP_CHECK(pool.alloc(&g.P9, 9 * N)); GP_CHECK(pool.alloc(&g.e, 3 * N)); GP_CHECK(pool.alloc(&g.Hss, N)); GP_CHECK(pool.alloc(&g.gss, N));
  GP_CHECK(pool.alloc(&g.E, 18 * N)); GP_CHECK(pool.alloc(&g.Fm, 18 * N));
  GP_CHECK(pool.alloc(&g.Hinv, 9 * P)); GP_CHECK(pool.alloc(&g.h, 3 * P)); GP_CHECK(pool.alloc(&g.gpt, 3 * P));
  GP_CHECK(pool.alloc(&g.A, (size_t)Npad * Npad)); GP_CHECK(pool.alloc(&g.rhs, Npad)); GP_CHECK(pool.alloc(&g.dC, Npad));
  GP_CHECK(pool.alloc(&g.dX, 3 * P)); GP_CHECK(pool.alloc(&g.ds, N)); GP_CHECK(pool.alloc(&g.model, N));
  GP_CHECK(pool.alloc(&g.dinv, (size_t)Npad * BA_TILE)); GP_CHECK(pool.alloc(&g.flag, 1)); GP_CHECK(pool.alloc(&g.bad, 1));
  GP_CHECK(pool.alloc(&g.gmax, 1)); GP_CHECK(pool.alloc(&g.red, GP_RG + 8));
  GP_CHECK(cudaMemset(g.dX, 0, sizeof(double) * 3 * std::max<int64_t>(P, 1)));
  GP_CHECK(cudaMemset(g.ns, 0, sizeof(double) * N));
  GP_CHECK(cudaMemset(g.np, 0, sizeof(double) * 3 * std::max<int64_t>(P, 1)));
  return 0;
}

// the variable blocks back into the caller's arrays (constants stay bit-identical)
static int gp_write_back(const GpLayout& L, const GpDev& g, b200gp_problem* p) {
  const int F = g.F, S = g.S; const int64_t P = g.P, N = g.N;
  std::vector<double> hc(3LL * F), hX(3 * P), hq(3LL * S), hs(N);
  GP_CHECK(cudaMemcpy(hc.data(), g.c, sizeof(double) * 3 * F, cudaMemcpyDeviceToHost));
  GP_CHECK(cudaMemcpy(hX.data(), g.X, sizeof(double) * 3 * P, cudaMemcpyDeviceToHost));
  if (S) GP_CHECK(cudaMemcpy(hq.data(), g.q, sizeof(double) * 3 * S, cudaMemcpyDeviceToHost));
  GP_CHECK(cudaMemcpy(hs.data(), g.s, sizeof(double) * N, cudaMemcpyDeviceToHost));
  for (int f = 0; f < F; ++f) if (L.fblk[f] >= 0) for (int m = 0; m < 3; ++m) p->frame_centers[3 * f + m] = hc[3 * f + m];
  for (int64_t q = 0; q < P; ++q) if (L.pvar[q]) for (int m = 0; m < 3; ++m) p->points[3 * q + m] = hX[3 * q + m];
  for (int s = 0; s < S; ++s) if (L.sblk[s] >= 0) for (int m = 0; m < 3; ++m) p->cams_in_rig[3 * s + m] = hq[3 * s + m];
  for (int64_t j = 0; j < N; ++j) if (L.svar[j]) p->obs_scale[L.perm[j]] = hs[j];
  return 0;
}

extern "C" int b200gp_solve(const b200gp_options* o, b200gp_problem* p, b200gp_summary* out) {
  g_gp_err.clear();
  if (!o || !p || !out) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "null argument");
  SOLVER_TRY(gp_check(o, p));
  GpLayout L;
  SOLVER_TRY(gp_layout(o, p, L));
  const int64_t N = p->num_observations;
  out->num_residuals = (int)(3 * N); out->reduced_dim = L.n; out->num_successful_steps = out->num_unsuccessful_steps = 0;
  out->num_iterations = 0; out->termination_type = B200GP_FAILURE; out->solve_ms = 0; out->initial_cost = out->final_cost = 0;
  if (N == 0) { out->termination_type = B200GP_CONVERGENCE; if (out->cost_history) out->cost_history[0] = 0.0; return 0; }

  if (o->gpu_index >= 0) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess) ndev = 0;   // no usable device: the index is out of range
    if (o->gpu_index >= ndev) return solver_fail(g_gp_err, B200GP_ERR_INPUT, "gpu_index out of range");
    GP_CHECK(cudaSetDevice(o->gpu_index));
  }
  SolverBuffers pool;
  GpSolve s{o, out};
  SOLVER_TRY(gp_upload(p, L, pool, s));
  cudaEvent_t ev0, ev1;
  GP_CHECK(pool.event(&ev0)); GP_CHECK(pool.event(&ev1));
  GP_CHECK(cudaEventRecord(ev0));
  double cost = 0;
  SOLVER_TRY(s.minimize(&cost));
  GP_CHECK(cudaEventRecord(ev1));
  GP_CHECK(cudaEventSynchronize(ev1));
  float ms = 0;
  GP_CHECK(cudaEventElapsedTime(&ms, ev0, ev1));
  out->solve_ms = ms; out->final_cost = cost;
  return gp_write_back(L, s.g, p);
}
