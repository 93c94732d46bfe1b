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
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <memory>
#include <numeric>
#include <string>
#include <vector>

#include "../../include/b200_bundle_adjustment.h"
#include "../../include/b200_ba_covariance.h"
#include "../../include/b200_ba_pose_prior.h"
#include "device_cache.h"
#include "ba_models.cuh"
#include "ba_dense_f64.h"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#define BA_MAXDK 5      // variable intrinsics of the narrow (<= 5-parameter) models: hand-written Jacobians, DC <= 11 kernels
#define BA_MAXP 16      // parameters of one camera (RAD_TAN_THIN_PRISM_FISHEYE)
#define BA_MAXCB 22     // width of a camera-side "camera block": [sensor_from_rig tangent (6, rigs only) | variable intrinsics (<= 16)]
#define BA_BLOCK 256
#define BA_CHUNK 512
#define BA_HD __host__ __device__ __forceinline__
// Jacobian storage: tiles of 32 observations, component-major inside a tile ("AoSoA"): a warp reads a whole tile
// as 2*DC (or 6) consecutive 128-byte lines, which keeps each warp on one DRAM page instead of 2*DC streams.
#define BA_JC(k, s) ((((long long)(s) >> 5) * (2 * D.DC) + (k)) * 32 + ((s) & 31))
#define BA_JP(k, s) ((((long long)(s) >> 5) * 6 + (k)) * 32 + ((s) & 31))
#define BA_U(k, s) ((((long long)(s) >> 5) * 2 + (k)) * 32 + ((s) & 31))

// ------------------------------------------------------------------------------------------------
// camera models + reprojection (host/device so the CPU test tier can check them without a GPU)
// ------------------------------------------------------------------------------------------------
BA_HD bool ba_model_is_narrow(int id) { return id == 0 || id == 1 || id == 2 || id == 3 || id == 8 || id == 9; }
BA_HD int ba_model_num_params(int id) {
  return id == 0 ? 3 : (id == 1 ? 4 : (id == 2 ? 4 : (id == 3 ? 5 : (id == 8 ? 4 : (id == 9 ? 5 : ba_wide_model_num_params(id))))));
}
// 0 focal, 1 principal point, 2 extra, 3 metadata (never refined) - the Initialize*Idxs of sensor/models.h:1206-2740: every
// model is (f, cx, cy, extra...) or (fx, fy, cx, cy, extra...); EQUIRECTANGULAR's (width, height) are sensor metadata
BA_HD int ba_param_group(int id, int k) {
  if (id == 17) return 3;
  const bool single = id == 0 || id == 2 || id == 3 || id == 8 || id == 9 || id == 12 || id == 14;
  if (single) return k == 0 ? 0 : (k < 3 ? 1 : 2);
  return k < 2 ? 0 : (k < 4 ? 1 : 2);
}

// ImgFromCamWithJac (sensor/models_jacobian.h:139-398); depth guard models.h:281-285.  Jp = d(x,y)/d(params) as two
// rows of stride 5 (fixed stride: the callers index it with compile-time constants).
BA_HD bool ba_img_from_cam(int id, const double* q, double u, double v, double w, double* x, double* y, double* Jp,
                           double* Juvw) {
  if (!(w >= 2.220446049250313e-16)) return false;
  const double iw = 1.0 / w, uu = u * iw, vv = v * iw;
  if (id == 0) {
    const double f = q[0];
    *x = f * uu + q[1]; *y = f * vv + q[2];
    const double fi = f * iw;
    Juvw[0] = fi; Juvw[1] = 0; Juvw[2] = -fi * uu; Juvw[3] = 0; Juvw[4] = fi; Juvw[5] = -fi * vv;
    Jp[0] = uu; Jp[1] = 1; Jp[2] = 0; Jp[5] = vv; Jp[6] = 0; Jp[7] = 1;
  } else if (id == 1) {
    *x = q[0] * uu + q[2]; *y = q[1] * vv + q[3];
    Juvw[0] = q[0] * iw; Juvw[1] = 0; Juvw[2] = -q[0] * iw * uu; Juvw[3] = 0; Juvw[4] = q[1] * iw; Juvw[5] = -q[1] * iw * vv;
    Jp[0] = uu; Jp[1] = 0; Jp[2] = 1; Jp[3] = 0; Jp[5] = 0; Jp[6] = vv; Jp[7] = 0; Jp[8] = 1;
  } else if (id == 2) {
    const double f = q[0], k = q[3];
    const double uu2 = uu * uu, vv2 = vv * vv, r2 = uu2 + vv2, kr2 = k * r2, alpha = 1.0 + kr2;
    const double xd = alpha * uu, yd = alpha * vv;
    *x = f * xd + q[1]; *y = f * yd + q[2];
    const double two_k = 2.0 * k, fi = f * iw, beta = 1.0 + 3.0 * kr2, cross = two_k * uu * vv;
    Juvw[0] = fi * (alpha + two_k * uu2); Juvw[1] = fi * cross; Juvw[2] = -fi * uu * beta;
    Juvw[3] = fi * cross; Juvw[4] = fi * (alpha + two_k * vv2); Juvw[5] = -fi * vv * beta;
    Jp[0] = xd; Jp[1] = 1; Jp[2] = 0; Jp[3] = f * uu * r2; Jp[5] = yd; Jp[6] = 0; Jp[7] = 1; Jp[8] = f * vv * r2;
  } else if (id == 8 || id == 9) {
    // SIMPLE_RADIAL_FISHEYE {f, cx, cy, k} / RADIAL_FISHEYE {f, cx, cy, k1, k2} (models_jacobian.h:44-83, 725-851):
    // equidistant mapping (a, b) -> (theta / r)(a, b) with theta = atan r, then radial distortion in fisheye coordinates
    const double f = q[0], k1 = q[3], k2 = (id == 9) ? q[4] : 0.0;
    const double r2 = uu * uu + vv * vv, r = sqrt(r2);
    double s = 1.0, g = 0.0;   // s = theta / r, g = (ds/dr) / r; identity in the limit r -> 0
    if (r >= 2.220446049250313e-16) { const double th = atan(r); s = th / r; g = (r / (1.0 + r2) - th) / (r2 * r); }
    const double fu = s * uu, fv = s * vv;
    const double F00 = s + uu * uu * g, F01 = uu * vv * g, F11 = s + vv * vv * g;          // d(fu, fv) / d(a, b)
    const double fu2 = fu * fu, fv2 = fv * fv, t2 = fu2 + fv2, t4 = t2 * t2, radial = k1 * t2 + k2 * t4;
    const double xd = fu + fu * radial, yd = fv + fv * radial;
    *x = f * xd + q[1]; *y = f * yd + q[2];
    const double dr = k1 + 2.0 * k2 * t2, cross = 2.0 * fu * fv * dr;
    const double D00 = 1.0 + radial + 2.0 * fu2 * dr, D11 = 1.0 + radial + 2.0 * fv2 * dr;   // I + d(distortion) / d(fu, fv)
    const double a00 = f * (D00 * F00 + cross * F01), a01 = f * (D00 * F01 + cross * F11);
    const double a10 = f * (cross * F00 + D11 * F01), a11 = f * (cross * F01 + D11 * F11);
    Juvw[0] = a00 * iw; Juvw[1] = a01 * iw; Juvw[2] = -(a00 * uu + a01 * vv) * iw;
    Juvw[3] = a10 * iw; Juvw[4] = a11 * iw; Juvw[5] = -(a10 * uu + a11 * vv) * iw;
    Jp[0] = xd; Jp[1] = 1; Jp[2] = 0; Jp[3] = f * fu * t2; Jp[4] = f * fu * t4;
    Jp[5] = yd; Jp[6] = 0; Jp[7] = 1; Jp[8] = f * fv * t2; Jp[9] = f * fv * t4;
  } else {
    const double f = q[0], k1 = q[3], k2 = q[4];
    const double uu2 = uu * uu, vv2 = vv * vv, r2 = uu2 + vv2, r4 = r2 * r2, radial = k1 * r2 + k2 * r4;
    const double xd = uu * (1.0 + radial), yd = vv * (1.0 + radial);
    *x = f * xd + q[1]; *y = f * yd + q[2];
    const double dr = k1 + 2.0 * k2 * r2, cross = 2.0 * uu * vv * dr;
    const double a00 = f * (1.0 + radial + 2.0 * uu2 * dr), a01 = f * cross, a11 = f * (1.0 + radial + 2.0 * vv2 * dr);
    Juvw[0] = a00 * iw; Juvw[1] = a01 * iw; Juvw[2] = -(a00 * uu + a01 * vv) * iw;
    Juvw[3] = a01 * iw; Juvw[4] = a11 * iw; Juvw[5] = -(a01 * uu + a11 * vv) * iw;
    Jp[0] = xd; Jp[1] = 1; Jp[2] = 0; Jp[3] = f * uu * r2; Jp[4] = f * uu * r4;
    Jp[5] = yd; Jp[6] = 0; Jp[7] = 1; Jp[8] = f * vv * r2; Jp[9] = f * vv * r4;
  }
  return true;
}

// QuaternionRotatePointWithJac (cost_functions/quaternion_utils.h:105-153), q = (x,y,z,w)
BA_HD void ba_quat_rotate_jac(const double* q, const double* p, double out[3], double J[12]) {
  const double qx = q[0], qy = q[1], qz = q[2], qw = q[3], px = p[0], py = p[1], pz = p[2];
  const double qx_py = qx * py, qx_pz = qx * pz, qy_px = qy * px, qy_pz = qy * pz, qz_px = qz * px, qz_py = qz * py;
  const double c0 = qy_pz - qz_py, c1 = qz_px - qx_pz, c2 = qx_py - qy_px;
  const double d0 = qy * c2 - qz * c1, d1 = qz * c0 - qx * c2, d2 = qx * c1 - qy * c0;
  out[0] = px + 2.0 * (qw * c0 + d0); out[1] = py + 2.0 * (qw * c1 + d1); out[2] = pz + 2.0 * (qw * c2 + d2);
  if (J) {
    const double qx_px = qx * px, qy_py = qy * py, qz_pz = qz * pz, qw_px = qw * px, qw_py = qw * py, qw_pz = qw * pz;
    J[0] = 2.0 * (qy_py + qz_pz); J[1] = 2.0 * (-2.0 * qy_px + qx_py + qw_pz); J[2] = 2.0 * (-2.0 * qz_px - qw_py + qx_pz); J[3] = 2.0 * (-qz_py + qy_pz);
    J[4] = 2.0 * (qy_px - 2.0 * qx_py - qw_pz); J[5] = 2.0 * (qx_px + qz_pz); J[6] = 2.0 * (qw_px - 2.0 * qz_py + qy_pz); J[7] = 2.0 * (qz_px - qx_pz);
    J[8] = 2.0 * (qz_px + qw_py - 2.0 * qx_pz); J[9] = 2.0 * (-qw_px + qz_py - 2.0 * qy_pz); J[10] = 2.0 * (qx_px + qy_py); J[11] = 2.0 * (-qy_px + qx_py);
  }
}
BA_HD void ba_quat_to_R(const double* q, double R[9]) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z, twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x,
               txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}
// EigenQuaternionManifold::Plus: [sin|d| d/|d|, cos|d|] * q
BA_HD void ba_quat_plus(const double* q, const double* d, double* out) {
  const double n = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  if (n == 0.0) { out[0] = q[0]; out[1] = q[1]; out[2] = q[2]; out[3] = q[3]; return; }
  const double s = sin(n) / n, dw = cos(n), dx = s * d[0], dy = s * d[1], dz = s * d[2];
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  out[0] = dw * x + dx * w + dy * z - dz * y;
  out[1] = dw * y - dx * z + dy * w + dz * x;
  out[2] = dw * z + dx * y - dy * x + dz * w;
  out[3] = dw * w - dx * x - dy * y - dz * z;
}
// AnalyticalReprojErrorCostFunction::Evaluate (reprojection_error.h:69-135)
// J_params: [2][P] when params_stride == 0, else two rows of `params_stride` (>= P) entries.
BA_HD bool ba_reproj(int id, const double* point, const double* pose, const double* params, double ox, double oy,
                     double* res, double* J_point, double* J_pose, double* J_params, int params_stride = 0) {
  double pc[3], Jq[12], Juvw[6];
  ba_quat_rotate_jac(pose, point, pc, J_pose ? Jq : nullptr);
  pc[0] += pose[4]; pc[1] += pose[5]; pc[2] += pose[6];
  double x, y, Jp[10];
  const int P = ba_model_num_params(id);
  if (!ba_img_from_cam(id, params, pc[0], pc[1], pc[2], &x, &y, Jp, Juvw)) {
    res[0] = res[1] = 0;
    if (J_point) for (int i = 0; i < 6; ++i) J_point[i] = 0;
    if (J_pose) for (int i = 0; i < 14; ++i) J_pose[i] = 0;
    if (J_params) {
      const int st = params_stride ? params_stride : P;
#pragma unroll
      for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int j = 0; j < 5; ++j) if (j < P) J_params[st * r + j] = 0;
    }
    return false;
  }
  res[0] = x - ox; res[1] = y - oy;
  if (J_point) {
    double R[9]; ba_quat_to_R(pose, R);
    for (int r = 0; r < 2; ++r)
      for (int c = 0; c < 3; ++c) J_point[3 * r + c] = Juvw[3 * r] * R[c] + Juvw[3 * r + 1] * R[3 + c] + Juvw[3 * r + 2] * R[6 + c];
  }
  if (J_pose) {
    for (int r = 0; r < 2; ++r) {
      for (int c = 0; c < 4; ++c) J_pose[7 * r + c] = Juvw[3 * r] * Jq[c] + Juvw[3 * r + 1] * Jq[4 + c] + Juvw[3 * r + 2] * Jq[8 + c];
      for (int c = 0; c < 3; ++c) J_pose[7 * r + 4 + c] = Juvw[3 * r + c];
    }
  }
  if (J_params) {
    const int st = params_stride ? params_stride : P;
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int j = 0; j < 5; ++j) if (j < P) J_params[st * r + j] = Jp[5 * r + j];
  }
  return true;
}
// Ceres loss functions (SoftLOneLoss, CauchyLoss, HuberLoss): rho, rho', rho''
BA_HD void ba_loss(int type, double a, double s, double rho[3]) {
  const double b = a * a, c = 1.0 / b;
  if (type == B200BA_LOSS_SOFT_L1) {
    const double sum = 1.0 + s * c, tmp = sqrt(sum);
    rho[0] = 2.0 * b * (tmp - 1.0); rho[1] = fmax(2.2250738585072014e-308, 1.0 / tmp); rho[2] = -(c * rho[1]) / (2.0 * sum);
  } else if (type == B200BA_LOSS_CAUCHY) {
    const double sum = 1.0 + s * c, inv = 1.0 / sum;
    rho[0] = b * log(sum); rho[1] = fmax(2.2250738585072014e-308, inv); rho[2] = -c * (inv * inv);
  } else if (type == B200BA_LOSS_HUBER) {
    if (s > b) { const double r = sqrt(s); rho[0] = 2.0 * a * r - b; rho[1] = fmax(2.2250738585072014e-308, a / r); rho[2] = -rho[1] / (2.0 * s); }
    else { rho[0] = s; rho[1] = 1.0; rho[2] = 0.0; }
  } else { rho[0] = s; rho[1] = 1.0; rho[2] = 0.0; }
}

// ------------------------------------------------------------------------------------------------
// device problem
// ------------------------------------------------------------------------------------------------
struct BaCtl {          // device-resident scalars of the LM / PCG loops
  double cost, new_cost, model, cost_delta;
  double rho, last_rho, pq, Q0, Q1, norm_b, rnorm2;
  int it, done;
  // everything above is cleared before each linear solve; the fields below persist
  int iters_total, fail;
  double gmax;
};

struct BaDev {
  // sizes
  int nposes, ncams, npts, nvpt, nc, DC, nblocks, nblocks_var;  // nc = camera-side dimension, DC = 6 + max dk
  long long nslots;
  int loss_type; double loss_scale;
  // parameters (current / candidate)
  double *poses, *cams, *pts, *nposes_, *ncams_, *npts_;
  // rigs + wide models: cam_from_world = sensor_from_rig * rig_from_world; a camera-side "camera block" is
  // [sensor_from_rig tangent (cam_ns = 6 when variable) | variable intrinsics (cam_nvar)], one block per camera
  int wide;                     // any camera model beyond the <= 5-parameter family, or any rig sensor: wide kernels + s_pack layout
  int nsensors;
  double *sensors, *nsensors_;  // [7*nsensors] current / candidate sensor_from_rig
  const int *cam_sensor, *cam_ns, *sens_cam;   // [ncams] sensor index or -1; [ncams] 0 | 6; [nsensors] camera of the sensor
  const int* cam_width;         // [ncams] cam_ns + cam_nvar: width of the camera block
  const int* blk_split;         // [nblk] 6 where a camera block holds both a sensor and an intrinsics part (block-Jacobi keeps them apart)
  const int4* chunks_off; int nchunks_off;   // sub-block pairs of camera blocks wider than 6 (see ba_build_cam_offdiag_kernel)
  // static per-block-variable maps
  const int *pose_off; const unsigned char* pose_mask;                 // [nposes]
  const int *cam_model, *cam_poff, *cam_off, *cam_nvar; const signed char* cam_var;  // [ncams], cam_var [ncams*BA_MAXP]
  const int* pt_var;                                                    // [npts] -> variable index or -1
  const int* vpt_point;                                                 // [nvpt] -> global point index
  // slots (block-packed observations)
  const int *s_pose, *s_cam, *s_pt;   // global indices, -1 for padding
  const int* s_lpt;                   // variable point index (global var idx) or -1
  const double* s_xy;                 // [2][nslots]
  const int *blk_pt0, *blk_npt;       // [nblocks] first variable point index / count
  const int *vpt_s0, *vpt_s1;         // [nvpt] slot range
  // linearisation (scaled) SoA
  float *Jc, *Jp;                     // Jc [2*DC][nslots], Jp [6][nslots]: scaled Jacobians, fp32 storage (the PCG operator)
  float* JcC;                         // [2*DC][nobs_c] the camera-side Jacobian again, in camera-sorted order
  double* r;                          // r [2][nslots]
  const int* s2c;                     // [nslots] slot -> position in camera order (-1 padding)
  const int4* s_pack;                 // [nslots] {pose offset, (cam offset + 1) | nv << 19 | head << 22 | last << 27, variable point, camera-order position}: one 16-byte load per slot in the SpMV
  const int* s_seg;                   // [nslots] head lane | last lane << 8 of the slot's track inside its warp (warp-packed region)
  int nblocks_warp;                   // leading blocks whose tracks never cross a warp (tracks <= 32 observations)
  int nblocks_giant0, nblocks_giant1; // block range of the tracks longer than a block (> 256 observations): generic two-kernel path
  double* zg;                         // [3*nvpt] scratch of the generic path (sum J_p^T y per point)
  float2* u;                          // [nobs_c] per-observation 2-vector exchanged between the two SpMV passes (fp32 like the operator)
  double* rC;                         // [2][nobs_c] residuals in camera order
  float* JpC;                         // [6][nobs_c] point-side Jacobian in camera order
  const double* xyC;                  // [2][nobs_c] observed image points in camera order
  const int2* c_pack;                 // [nobs_c] {point index, variable point index or -1} in camera order
  const int2* runs_pc;                // per run {pose index, camera index}
  int intr_by_pt;                     // some track sees one variable-intrinsics camera twice: intrinsics blocks via ba_schur_pt_kernel
  int pose_by_pt;                     // some track sees one variable frame twice (rig sensors): pose blocks via ba_schur_pt_kernel too
  const int* c_run;                   // [nobs_c padded] run id of the observation in camera order: one run = one (camera, pose) pair
  const int4* runs;                   // per run {pose offset or -1, camera offset or -1, #variable intrinsics, 0}
  const int4* chunks;                 // {c0, c1, out offset, comp0 | ncomp << 8}: <= BA_CHUNK observations of one block
  int nchunks; long long nobs_c;
  double* cost_slot;                  // [nslots] 1/2 rho(|r|^2) at the linearisation point
  double *scale_c, *scale_p;          // [nc], [3*nvpt]
  // normal equations
  double *Hpp, *Hpp_inv, *gp, *diag_p, *Dp2;      // [6*nvpt] sym, [6*nvpt] sym, [3*nvpt]...
  double *gc, *diag_c, *Dc2, *rhs;                // [nc]
  double *Hbb, *Mbb, *Minv;                       // packed camera-side blocks
  const int *blk_start, *blk_pack, *off2blk;      // [nblk+1], [nblk+1], [nc]
  const int4* row_info;                           // [nc] {first row of the row's block, offset of the row in the packed blocks, block size, 0}
  int nblk;
  // PCG vectors
  double *x, *rr, *z, *p, *q, *dp;
  double* Sd;   // dense reduced camera matrix [nc*nc] (DENSE_SCHUR path), column-major == row-major (symmetric)
  BaCtl* ctl;
};

struct BaPrior {          // position priors of one solve (n = 0: none, and no prior launch happens; see ba_prior_position)
  int n = 0, loss_type = 0;
  double loss_scale = 1.0;
  const int4* idx = nullptr;   // {pose index, sensor index or -1, pose offset or -1, offset of the sensor tangent or -1}
  const double* c = nullptr;   // [3n] prior positions
  const double* W = nullptr;   // [9n] chol(cov^-1)^T, row-major
  double* J = nullptr;         // [36n] rows of the weighted, loss-corrected (scaled after iteration 0) Jacobian: 3 x [pose 6 | sensor 6]
  double* r = nullptr;         // [3n] loss-corrected weighted residual
  double* cost = nullptr;      // [n] 1/2 rho at the linearisation point
};

__device__ __forceinline__ double ba_block_sum(double v, double* sm) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) sm[w] = v;
  __syncthreads();
  double t = 0;
  if (threadIdx.x < 32) {
    t = (threadIdx.x < (blockDim.x >> 5)) ? sm[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  __syncthreads();
  return t;  // valid in thread 0
}

// ImgFromCamWithJac of ANY of the eighteen models: the hand-written Jacobians of the <= 5-parameter family, forward-mode
// dual numbers (ba_models.cuh) for the twelve others.  Jp: two rows of stride BA_MAXP.
// (not inlined: the dual-number evaluation of eight parameter counts is compiled once, not once per kernel instantiation)
__host__ __device__ __noinline__ bool ba_img_from_cam_any(int id, const double* q, double u, double v, double w, double* x, double* y, double* Jp,
                               double* Juvw) {
  if (ba_model_is_narrow(id)) {
    double J5[10];
    if (!ba_img_from_cam(id, q, u, v, w, x, y, J5, Juvw)) return false;
    const int P = ba_model_num_params(id);
    for (int k = 0; k < 5; ++k) if (k < P) { Jp[k] = J5[k]; Jp[BA_MAXP + k] = J5[5 + k]; }
    return true;
  }
  double xy[2], Jw[2 * BA_MAXP];
  bool ok = false;
  int P = 0;
  switch (ba_wide_model_num_params(id)) {
    case 2: P = 2; ok = ba_project_wide_with_jac<2>(id, q, u, v, w, xy, Juvw, Jw); break;
    case 3: P = 3; ok = ba_project_wide_with_jac<3>(id, q, u, v, w, xy, Juvw, Jw); break;
    case 4: P = 4; ok = ba_project_wide_with_jac<4>(id, q, u, v, w, xy, Juvw, Jw); break;
    case 5: P = 5; ok = ba_project_wide_with_jac<5>(id, q, u, v, w, xy, Juvw, Jw); break;
    case 6: P = 6; ok = ba_project_wide_with_jac<6>(id, q, u, v, w, xy, Juvw, Jw); break;
    case 8: P = 8; ok = ba_project_wide_with_jac<8>(id, q, u, v, w, xy, Juvw, Jw); break;
    case 12: P = 12; ok = ba_project_wide_with_jac<12>(id, q, u, v, w, xy, Juvw, Jw); break;
    case 16: P = 16; ok = ba_project_wide_with_jac<16>(id, q, u, v, w, xy, Juvw, Jw); break;
    default: return false;
  }
  if (!ok) return false;
  *x = xy[0]; *y = xy[1];
  for (int k = 0; k < P; ++k) { Jp[k] = Jw[k]; Jp[BA_MAXP + k] = Jw[P + k]; }
  return true;
}
// residual only, any model, trivial frame or rig sensor (sensor == nullptr: identity): the candidate-cost evaluation
__host__ __device__ __noinline__ bool ba_residual_any(int id, const double* point, const double* rig, const double* sensor, const double* params,
                           double ox, double oy, double* res) {
  double pr[3], pc[3];
  ba_quat_rotate_jac(rig, point, pr, nullptr);
  pr[0] += rig[4]; pr[1] += rig[5]; pr[2] += rig[6];
  if (sensor) { ba_quat_rotate_jac(sensor, pr, pc, nullptr); pc[0] += sensor[4]; pc[1] += sensor[5]; pc[2] += sensor[6]; }
  else { pc[0] = pr[0]; pc[1] = pr[1]; pc[2] = pr[2]; }
  double x = 0, y = 0;
  bool ok;
  if (ba_model_is_narrow(id)) { double J5[10], Juvw[6]; ok = ba_img_from_cam(id, params, pc[0], pc[1], pc[2], &x, &y, J5, Juvw); }
  else { ok = ba_project_wide<double>(id, params, pc[0], pc[1], pc[2], &x, &y); }
  if (!ok) { res[0] = res[1] = 0.0; return false; }
  res[0] = x - ox; res[1] = y - oy;
  return true;
}
// RigReprojErrorCostFunctor / ReprojErrorCostFunctor (reprojection_error.h:217-420) with analytic derivatives:
// p_cam = R(q_s) (R(q_r) X + t_r) + t_s.  J_rig / J_sensor: 2x7 ambient; J_params: two rows of stride BA_MAXP.
__host__ __device__ __noinline__ bool ba_reproj_rig(int id, const double* point, const double* rig, const double* sensor, const double* params, double ox,
                         double oy, double* res, double* J_point, double* J_rig, double* J_sensor, double* J_params) {
  double pr[3], Jqr[12], pc[3], Jqs[12], Rs[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, Rr[9];
  ba_quat_rotate_jac(rig, point, pr, Jqr);
  pr[0] += rig[4]; pr[1] += rig[5]; pr[2] += rig[6];
  if (sensor) {
    ba_quat_rotate_jac(sensor, pr, pc, Jqs);
    pc[0] += sensor[4]; pc[1] += sensor[5]; pc[2] += sensor[6];
    ba_quat_to_R(sensor, Rs);
  } else { pc[0] = pr[0]; pc[1] = pr[1]; pc[2] = pr[2]; }
  double x, y, Juvw[6];
  for (int k = 0; k < 2 * BA_MAXP; ++k) J_params[k] = 0.0;
  if (!ba_img_from_cam_any(id, params, pc[0], pc[1], pc[2], &x, &y, J_params, Juvw)) {
    res[0] = res[1] = 0.0;
    for (int k = 0; k < 6; ++k) J_point[k] = 0.0;
    for (int k = 0; k < 14; ++k) { J_rig[k] = 0.0; J_sensor[k] = 0.0; }
    for (int k = 0; k < 2 * BA_MAXP; ++k) J_params[k] = 0.0;
    return false;
  }
  res[0] = x - ox; res[1] = y - oy;
  double A[6];   // d(x, y) / d(p_rig) = J_uvw R_s
  for (int r = 0; r < 2; ++r) for (int c = 0; c < 3; ++c) A[3 * r + c] = Juvw[3 * r] * Rs[c] + Juvw[3 * r + 1] * Rs[3 + c] + Juvw[3 * r + 2] * Rs[6 + c];
  ba_quat_to_R(rig, Rr);
  for (int r = 0; r < 2; ++r) {
    for (int c = 0; c < 3; ++c) J_point[3 * r + c] = A[3 * r] * Rr[c] + A[3 * r + 1] * Rr[3 + c] + A[3 * r + 2] * Rr[6 + c];
    for (int c = 0; c < 4; ++c) J_rig[7 * r + c] = A[3 * r] * Jqr[c] + A[3 * r + 1] * Jqr[4 + c] + A[3 * r + 2] * Jqr[8 + c];
    for (int c = 0; c < 3; ++c) J_rig[7 * r + 4 + c] = A[3 * r + c];
    for (int c = 0; c < 4; ++c) J_sensor[7 * r + c] = sensor ? Juvw[3 * r] * Jqs[c] + Juvw[3 * r + 1] * Jqs[4 + c] + Juvw[3 * r + 2] * Jqs[8 + c] : 0.0;
    for (int c = 0; c < 3; ++c) J_sensor[7 * r + 4 + c] = sensor ? Juvw[3 * r + c] : 0.0;
  }
  return true;
}

// Robust-loss corrector (ceres Corrector), Jacobi scaling and the scaled residual of ONE observation whose raw rows are
// in registers: the common tail of the narrow and the wide linearisation.  co / nvc: offset and width of the camera block.
template <int DC>
__device__ __forceinline__ void ba_obs_finish(const BaDev& D, const double* res, const double* rho, double sq, int po, int co,
                                              int nvc, int lp, int apply_scale, double* Jc, double* Jpt, double* rr) {
  if (lp < 0) {
#pragma unroll
    for (int k = 0; k < 6; ++k) Jpt[k] = 0.0;
  }
  double rs = 1.0;
  if (D.loss_type != B200BA_LOSS_TRIVIAL) {  // ceres Corrector
    const double sqrt_rho1 = sqrt(rho[1]);
    double alpha_sq_norm = 0.0;
    rs = sqrt_rho1;
    if (sq != 0.0 && rho[2] > 0.0) {
      const double Dd = 1.0 + 2.0 * sq * rho[2] / rho[1];
      const double alpha = 1.0 - sqrt(Dd);
      rs = sqrt_rho1 / (1 - alpha);
      alpha_sq_norm = alpha / sq;
    }
#pragma unroll
    for (int c = 0; c < DC; ++c) {
      const double rj = res[0] * Jc[c] + res[1] * Jc[DC + c];
      Jc[c] = sqrt_rho1 * (Jc[c] - alpha_sq_norm * res[0] * rj);
      Jc[DC + c] = sqrt_rho1 * (Jc[DC + c] - alpha_sq_norm * res[1] * rj);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double rj = res[0] * Jpt[c] + res[1] * Jpt[3 + c];
      Jpt[c] = sqrt_rho1 * (Jpt[c] - alpha_sq_norm * res[0] * rj);
      Jpt[3 + c] = sqrt_rho1 * (Jpt[3 + c] - alpha_sq_norm * res[1] * rj);
    }
  }
  if (apply_scale) {
    if (po >= 0) {
#pragma unroll
      for (int c = 0; c < 6; ++c) { const double sc = D.scale_c[po + c]; Jc[c] *= sc; Jc[DC + c] *= sc; }
    }
    if (co >= 0) {
#pragma unroll
      for (int c = 0; c < DC - 6; ++c) if (c < nvc) { const double sc = D.scale_c[co + c]; Jc[6 + c] *= sc; Jc[DC + 6 + c] *= sc; }
    }
    if (lp >= 0) {
#pragma unroll
      for (int c = 0; c < 3; ++c) { const double sc = D.scale_p[3 * (long long)lp + c]; Jpt[c] *= sc; Jpt[3 + c] *= sc; }
    }
  }
  rr[0] = rs * res[0]; rr[1] = rs * res[1];
}

// Residual, robustified + Jacobi-scaled Jacobian rows of ONE observation, in registers.  Shared by the slot-ordered and
// the camera-ordered linearisation passes: both evaluate the same expression tree on the same inputs, so the two fp32
// copies of the camera-side Jacobian hold identical values (the PCG operator stays symmetric) without any scattered
// store.  Returns 1/2 rho(|r|^2).  WIDE = false: trivial frames and the <= 5-parameter models (the tuned path);
// WIDE = true: any of the eighteen models, rig sensors.
template <int DC, bool WIDE>
__device__ __forceinline__ double ba_obs_linearize(const BaDev& D, const double* __restrict__ poses,
                                                   const double* __restrict__ cams, const double* __restrict__ pts,
                                                   int pi, int ci, int ti, int lp, double ox, double oy, int apply_scale,
                                                   double* Jc, double* Jpt, double* rr) {
  const int id = D.cam_model[ci];
  double pose[7], pt[3];
#pragma unroll
  for (int k = 0; k < 7; ++k) pose[k] = poses[7 * (long long)pi + k];
#pragma unroll
  for (int k = 0; k < 3; ++k) pt[k] = pts[3 * (long long)ti + k];
  const int P = ba_model_num_params(id);
  const int poff = D.cam_poff[ci];
  const int po = D.pose_off[pi], co = D.cam_off[ci], nv = D.cam_nvar[ci];
  double res[2], rho[3], sq;
#pragma unroll
  for (int k = 0; k < 2 * DC; ++k) Jc[k] = 0.0;
  if (!WIDE) {
    double prm[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) prm[k] = (k < P) ? cams[poff + k] : 0.0;
    double Jps[14], Jpr[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) Jpr[k] = 0.0;
    ba_reproj(id, pt, pose, prm, ox, oy, res, Jpt, Jps, Jpr, 5);
    sq = res[0] * res[0] + res[1] * res[1];
    ba_loss(D.loss_type, D.loss_scale, sq, rho);
    if (po >= 0) {
      const unsigned m = D.pose_mask[pi];
      const double PJ[12] = {pose[3], pose[2], -pose[1], -pose[2], pose[3], pose[0], pose[1], -pose[0], pose[3], -pose[0], -pose[1], -pose[2]};
#pragma unroll
      for (int r = 0; r < 2; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          double v = 0;
#pragma unroll
          for (int k = 0; k < 4; ++k) v += Jps[7 * r + k] * PJ[3 * k + c];
          Jc[DC * r + c] = ((m >> c) & 1u) ? v : 0.0;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) Jc[DC * r + 3 + c] = ((m >> (3 + c)) & 1u) ? Jps[7 * r + 4 + c] : 0.0;
      }
    }
    if (co >= 0) {
#pragma unroll
      for (int k = 0; k < DC - 6; ++k) {
        if (k < nv) {
          const int var = D.cam_var[BA_MAXP * ci + k];
          // pick the entry with selects so that the array stays in registers
          double v0 = 0.0, v1 = 0.0;
#pragma unroll
          for (int j = 0; j < 5; ++j) if (j == var) { v0 = Jpr[j]; v1 = Jpr[5 + j]; }
          Jc[6 + k] = v0; Jc[DC + 6 + k] = v1;
        }
      }
    }
    ba_obs_finish<DC>(D, res, rho, sq, po, co, nv, lp, apply_scale, Jc, Jpt, rr);
  } else {
    double prm[BA_MAXP], sens[7];
    for (int k = 0; k < BA_MAXP; ++k) prm[k] = (k < P) ? cams[poff + k] : 0.0;
    const int si = D.cam_sensor[ci], ns = D.cam_ns[ci];
    if (si >= 0) for (int k = 0; k < 7; ++k) sens[k] = D.sensors[7 * (long long)si + k];
    double Jrig[14], Jsen[14], Jprm[2 * BA_MAXP];
    ba_reproj_rig(id, pt, pose, si >= 0 ? sens : nullptr, prm, ox, oy, res, Jpt, Jrig, Jsen, Jprm);
    sq = res[0] * res[0] + res[1] * res[1];
    ba_loss(D.loss_type, D.loss_scale, sq, rho);
    for (int blk = 0; blk < 2; ++blk) {   // rig_from_world, then sensor_from_rig: quaternion (x) R^3 tangent
      const bool on = blk == 0 ? (po >= 0) : (co >= 0 && ns == 6);
      if (!on) continue;
      const double* q = blk == 0 ? pose : sens;
      const double* Ja = blk == 0 ? Jrig : Jsen;
      const unsigned m = blk == 0 ? D.pose_mask[pi] : 0x3fu;
      const int jo = blk == 0 ? 0 : 6;
      const double PJ[12] = {q[3], q[2], -q[1], -q[2], q[3], q[0], q[1], -q[0], q[3], -q[0], -q[1], -q[2]};
      for (int r = 0; r < 2; ++r) {
        for (int c = 0; c < 3; ++c) {
          double v = 0;
          for (int k = 0; k < 4; ++k) v += Ja[7 * r + k] * PJ[3 * k + c];
          Jc[DC * r + jo + c] = ((m >> c) & 1u) ? v : 0.0;
        }
        for (int c = 0; c < 3; ++c) Jc[DC * r + jo + 3 + c] = ((m >> (3 + c)) & 1u) ? Ja[7 * r + 4 + c] : 0.0;
      }
    }
    if (co >= 0)
      for (int k = 0; k < nv; ++k) {
        const int var = D.cam_var[BA_MAXP * ci + k];
        if (6 + ns + k < DC) { Jc[6 + ns + k] = Jprm[var]; Jc[DC + 6 + ns + k] = Jprm[BA_MAXP + var]; }
      }
    ba_obs_finish<DC>(D, res, rho, sq, po, co, ns + nv, lp, apply_scale, Jc, Jpt, rr);
  }
  return 0.5 * rho[0];
}

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

// Warp-packed variant of pass 1 (tracks of <= 32 observations, i.e. almost all of them): the track never crosses
// a warp, so the point-block elimination is a segmented shuffle reduction — no shared memory, no block barrier,
// every lane stays busy.  Same arithmetic as ba_schur_spmv_kernel below.
__device__ __forceinline__ double ba_shfl_down_f64(double v, int off) { return __shfl_down_sync(0xffffffffu, v, off); }
__device__ __forceinline__ double ba_shfl_f64(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }

// s_pack.y = (camera-block offset + 1) | width << (19 | 17) | head lane << 22 | last lane << 27: 19 + 3 bits for the narrow
// layout (width <= 5), 17 + 5 bits when the problem has wide camera blocks
__device__ __forceinline__ void ba_unpack_cam(unsigned pky, int wide, int& co, int& nv) {
  if (wide) { co = (int)(pky & 0x1ffffu) - 1; nv = (int)((pky >> 17) & 31u); }
  else { co = (int)(pky & 0x7ffffu) - 1; nv = (int)((pky >> 19) & 7u); }
}
template <int DC>
__device__ __forceinline__ void ba_spmv_slot(const BaDev& D, const long long s, const int lane, const double* __restrict__ pvec) {
  const int4 pk = __ldg(D.s_pack + s);          // all per-slot indices in one coalesced 16-byte load
  const unsigned pky = (unsigned)pk.y;
  const int po = pk.x;
  int co, nv;
  ba_unpack_cam(pky, DC > 11 ? D.wide : 0, co, nv);
  const int lp = pk.z;
  const long long cp = pk.w;                     // -1 on padding slots
  int head = lane, last = lane;
  double y0 = 0.0, y1 = 0.0;
  // the Jacobian rows are fetched unconditionally (padding slots hold zeros) so that their loads are in flight
  // together with the index load instead of behind it
  float J0[DC], J1[DC], jp[6];
#pragma unroll
  for (int c = 0; c < DC; ++c) { J0[c] = D.Jc[BA_JC(c, s)]; J1[c] = D.Jc[BA_JC(DC + c, s)]; }
#pragma unroll
  for (int c = 0; c < 6; ++c) jp[c] = D.Jp[BA_JP(c, s)];
  if (cp >= 0) {
    head = (int)((pky >> 22) & 31u); last = (int)((pky >> 27) & 31u);
    if (po >= 0) {   // pose blocks are 6 doubles wide: the offset is 16-byte aligned -> three 128-bit loads
      const double2* v2 = reinterpret_cast<const double2*>(pvec + po);
      const double2 va = v2[0], vb = v2[1], vc = v2[2];
      const double v[6] = {va.x, va.y, vb.x, vb.y, vc.x, vc.y};
#pragma unroll
      for (int c = 0; c < 6; ++c) { y0 += (double)J0[c] * v[c]; y1 += (double)J1[c] * v[c]; }
    }
    if (co >= 0) {
#pragma unroll
      for (int c = 0; c < DC - 6; ++c) if (c < nv) { const double v = pvec[co + c]; y0 += (double)J0[6 + c] * v; y1 += (double)J1[6 + c] * v; }
    }
  }
  double z0 = (double)jp[0] * y0 + (double)jp[3] * y1, z1 = (double)jp[1] * y0 + (double)jp[4] * y1, z2 = (double)jp[2] * y0 + (double)jp[5] * y1;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const double t0 = ba_shfl_down_f64(z0, off), t1 = ba_shfl_down_f64(z1, off), t2 = ba_shfl_down_f64(z2, off);
    if (lane + off <= last) { z0 += t0; z1 += t1; z2 += t2; }
  }
  double w0 = 0.0, w1 = 0.0, w2 = 0.0;
  if (lane == head && lp >= 0) {
    const double2* I2 = reinterpret_cast<const double2*>(D.Hpp_inv + 6 * (long long)lp);   // 48-byte records: 16-byte aligned
    const double2 ia = I2[0], ib = I2[1], ic = I2[2];
    w0 = ia.x * z0 + ia.y * z1 + ib.x * z2;
    w1 = ia.y * z0 + ib.y * z1 + ic.x * z2;
    w2 = ib.x * z0 + ic.x * z1 + ic.y * z2;
  }
  w0 = ba_shfl_f64(w0, head); w1 = ba_shfl_f64(w1, head); w2 = ba_shfl_f64(w2, head);
  if (cp >= 0) {
    if (lp >= 0) {
      y0 -= (double)jp[0] * w0 + (double)jp[1] * w1 + (double)jp[2] * w2;
      y1 -= (double)jp[3] * w0 + (double)jp[4] * w1 + (double)jp[5] * w2;
    }
    D.u[cp] = make_float2((float)y0, (float)y1);   // one 8-byte scattered store per observation
  }
}

template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_schur_spmv_warp_kernel(const BaDev D, const double* __restrict__ pvec) {
  if (D.ctl->done) return;
  ba_spmv_slot<DC>(D, (long long)blockIdx.x * BA_BLOCK + threadIdx.x, threadIdx.x & 31, pvec);
}
// Persistent form with the camera-side vector staged in shared memory: the per-lane gathers p[pose], p[camera] (every
// lane of a warp looks at a different camera) cost one L1 wavefront per lane and instruction from global memory, a few
// bank-conflict cycles from shared memory.  Grid = SMs x resident CTAs, each CTA loads p once and walks the slot blocks.
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_schur_spmv_warp_smem_kernel(const BaDev D, const double* __restrict__ pvec) {
  extern __shared__ double2 ba_sp2[];
  double* sp = reinterpret_cast<double*>(ba_sp2);
  if (D.ctl->done) return;
  for (int i = threadIdx.x; i < D.nc; i += BA_BLOCK) sp[i] = pvec[i];
  __syncthreads();
  for (int blk = blockIdx.x; blk < D.nblocks_warp; blk += gridDim.x)
    ba_spmv_slot<DC>(D, (long long)blk * BA_BLOCK + threadIdx.x, threadIdx.x & 31, sp);
}

// THE ROOFLINE KERNEL, pass 1 of 2: u_o = J_c p - J_p (H_pp + D_p^2)^-1 sum_track J_p^T J_c p per observation.
// One thread per observation slot; a block holds whole tracks, so the point-block elimination
// (z_p = sum J_p^T y, w_p = Hinv z_p) is a shared-memory exchange.  u is written in camera-sorted order and
// reduced per camera-side block by ba_cam_stream_loop_kernel.
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_schur_spmv_kernel(const BaDev D, const double* __restrict__ pvec,
                                                                 double* __restrict__ qvec) {
  __shared__ double sy[2][BA_BLOCK];
  __shared__ double sw[3][BA_BLOCK];
  if (D.ctl->done) return;
  const int blk = blockIdx.x + D.nblocks_warp;   // blocks after the warp-packed region
  if (blk >= D.nblocks_giant0 && blk < D.nblocks_giant1) return;   // tracks longer than a block: generic path
  const long long s = (long long)blk * BA_BLOCK + threadIdx.x;
  const int pi = D.s_pose[s];
  int po = -1, co = -1, nv = 0;
  double J0[DC], J1[DC], y0 = 0.0, y1 = 0.0;
  if (pi >= 0) {
    const int ci = D.s_cam[s];
    po = D.pose_off[pi]; co = D.cam_off[ci]; nv = D.cam_width[ci];
#pragma unroll
    for (int c = 0; c < DC; ++c) { J0[c] = D.Jc[BA_JC(c, s)]; J1[c] = D.Jc[BA_JC((DC + c), s)]; }
    if (po >= 0) {
#pragma unroll
      for (int c = 0; c < 6; ++c) { const double v = pvec[po + c]; y0 += J0[c] * v; y1 += J1[c] * v; }
    }
    if (co >= 0) {
#pragma unroll
      for (int c = 0; c < DC - 6; ++c) if (c < nv) { const double v = pvec[co + c]; y0 += J0[6 + c] * v; y1 += J1[6 + c] * v; }
    }
  }
  const bool var_block = blk < D.nblocks_var;
  if (var_block) {
    sy[0][threadIdx.x] = y0; sy[1][threadIdx.x] = y1;
    __syncthreads();
    // one thread per track of this block
    if (threadIdx.x < D.blk_npt[blk]) {
      const int k = D.blk_pt0[blk] + threadIdx.x;
      const int s0 = D.vpt_s0[k], s1 = D.vpt_s1[k];
      double z0 = 0, z1 = 0, z2 = 0;
      for (int t = s0; t < s1; ++t) {
        const int l = t - blk * BA_BLOCK;
        const double a0 = sy[0][l], a1 = sy[1][l];
        z0 += D.Jp[BA_JP(0, t)] * a0 + D.Jp[BA_JP(3, t)] * a1;
        z1 += D.Jp[BA_JP(1, t)] * a0 + D.Jp[BA_JP(4, t)] * a1;
        z2 += D.Jp[BA_JP(2, t)] * a0 + D.Jp[BA_JP(5, t)] * a1;
      }
      const double* I = D.Hpp_inv + 6 * (long long)k;
      sw[0][threadIdx.x] = I[0] * z0 + I[1] * z1 + I[2] * z2;
      sw[1][threadIdx.x] = I[1] * z0 + I[3] * z1 + I[4] * z2;
      sw[2][threadIdx.x] = I[2] * z0 + I[4] * z1 + I[5] * z2;
    }
    __syncthreads();
    const int lp = (pi >= 0) ? D.s_lpt[s] : -1;
    if (lp >= 0) {
      const int lt = lp - D.blk_pt0[blk];
      const double w0 = sw[0][lt], w1 = sw[1][lt], w2 = sw[2][lt];
      y0 -= D.Jp[BA_JP(0, s)] * w0 + D.Jp[BA_JP(1, s)] * w1 + D.Jp[BA_JP(2, s)] * w2;
      y1 -= D.Jp[BA_JP(3, s)] * w0 + D.Jp[BA_JP(4, s)] * w1 + D.Jp[BA_JP(5, s)] * w2;
    }
  }
  if (pi >= 0) {
    const long long cp = D.s2c[s];
    D.u[cp] = make_float2((float)y0, (float)y1);   // one 8-byte scattered store per observation
  }
}

// Warp-reduces the per-lane sums of one (camera, pose) run and adds them to the run's pose / camera blocks of out.
template <int DC>
__device__ __forceinline__ void ba_cam_stream_flush(double* acc, int run, const BaDev& D, double* __restrict__ out, int lane) {
  if (run < 0) return;
  const int4 rd = D.runs[run];
  double mine = 0.0;
#pragma unroll
  for (int c = 0; c < DC; ++c) {
    double t = acc[c];
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == c) mine = t;
    acc[c] = 0.0;
  }
  if (lane < 6) { if (rd.x >= 0) atomicAdd(&out[rd.x + lane], mine); }
  else if (lane < 6 + rd.z) { if (rd.y >= 0) atomicAdd(&out[rd.y + lane - 6], mine); }
}
// Second SpMV pass (streaming): out[block] += sum over the block's observations of J_c^T u, observations in camera
// order.  A warp walks a contiguous range of 32-observation tiles (fully coalesced tile lines); the next tile's loads
// are issued before the current tile is accumulated (register double buffer).  The products are accumulated per lane
// while the tiles stay inside one (camera, pose) run — runs are thousands of observations long — and reduced with
// shuffles only when the run changes or the range ends: 6 + nv red.adds per run a warp touches.  No shared memory, no barrier.
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_cam_stream_loop_kernel(const BaDev D, double* __restrict__ out, int respect_done,
                                                                      int tiles_per_warp) {
  if (respect_done && D.ctl->done) return;
  const int lane = threadIdx.x & 31;
  const long long ntiles = (D.nobs_c + 31) >> 5;
  long long t = ((long long)blockIdx.x * (BA_BLOCK / 32) + (threadIdx.x >> 5)) * tiles_per_warp;
  const long long t1 = (t + tiles_per_warp < ntiles) ? t + tiles_per_warp : ntiles;
  if (t >= t1) return;
  int run_c;
  float j0c[DC], j1c[DC], u0c, u1c;
  {
    const long long k = t * 32 + lane;
    run_c = D.c_run[k];
#pragma unroll
    for (int c = 0; c < DC; ++c) { j0c[c] = D.JcC[BA_JC(c, k)]; j1c[c] = D.JcC[BA_JC(DC + c, k)]; }
    { const float2 uu = D.u[k]; u0c = uu.x; u1c = uu.y; }
  }
  double acc[DC];
#pragma unroll
  for (int c = 0; c < DC; ++c) acc[c] = 0.0;
  int cur = -1;
  for (; t < t1; ++t) {
    int run_n = -1;
    float j0n[DC], j1n[DC], u0n = 0.f, u1n = 0.f;
    if (t + 1 < t1) {
      const long long k = (t + 1) * 32 + lane;
      run_n = D.c_run[k];
#pragma unroll
      for (int c = 0; c < DC; ++c) { j0n[c] = D.JcC[BA_JC(c, k)]; j1n[c] = D.JcC[BA_JC(DC + c, k)]; }
      { const float2 uu = D.u[k]; u0n = uu.x; u1n = uu.y; }
    } else {
#pragma unroll
      for (int c = 0; c < DC; ++c) { j0n[c] = 0.f; j1n[c] = 0.f; }
    }
    const int r0 = __shfl_sync(0xffffffffu, run_c, 0);
    const bool uniform = __all_sync(0xffffffffu, run_c == r0);
    if (uniform) {
      if (r0 != cur) { ba_cam_stream_flush<DC>(acc, cur, D, out, lane); cur = r0; }
      if (r0 >= 0) {
#pragma unroll
        for (int c = 0; c < DC; ++c) acc[c] += (double)j0c[c] * (double)u0c + (double)j1c[c] * (double)u1c;
      }
    } else {  // the tile straddles a run boundary (or is the ragged tail): per-observation adds (rare)
      ba_cam_stream_flush<DC>(acc, cur, D, out, lane); cur = -1;
      if (run_c >= 0) {
        const int4 rd = D.runs[run_c];
#pragma unroll
        for (int c = 0; c < DC; ++c) {
          const double v = (double)j0c[c] * (double)u0c + (double)j1c[c] * (double)u1c;
          if (c < 6) { if (rd.x >= 0) atomicAdd(&out[rd.x + c], v); }
          else if (c < 6 + rd.z) { if (rd.y >= 0) atomicAdd(&out[rd.y + c - 6], v); }
        }
      }
    }
    run_c = run_n; u0c = u0n; u1c = u1n;
#pragma unroll
    for (int c = 0; c < DC; ++c) { j0c[c] = j0n[c]; j1c[c] = j1n[c]; }
  }
  ba_cam_stream_flush<DC>(acc, cur, D, out, lane);
}

// ---- PCG vector work between two SpMVs in one single-CTA kernel (camera-side dimension is small: a few thousand) ----
#define BA_PCG_T 1024
#define BA_PCG_FUSED_MAX 65536   // tests/test_ba_paths_gpu.py mirrors this threshold
__device__ __forceinline__ double ba_cta_allsum(double v, double* sm /* [33] */) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) sm[w] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    double t = (threadIdx.x < (blockDim.x >> 5)) ? sm[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) sm[32] = t;
  }
  __syncthreads();
  const double t = sm[32];
  __syncthreads();
  return t;  // valid in every thread
}
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

// Generic path for tracks longer than a block (> 256 observations; rare): the per-point sum goes through global
// atomics.  MODE 0: SpMV (vec = p, writes u); MODE 1: back-substitution / model cost (vec = x, writes d_p, model).
template <int MODE>
__global__ void __launch_bounds__(BA_BLOCK) ba_giant_accumulate_kernel(const BaDev D, const double* __restrict__ vec) {
  if (MODE == 0 && D.ctl->done) return;
  const long long s = (long long)(blockIdx.x + D.nblocks_giant0) * BA_BLOCK + threadIdx.x;
  const int pi = D.s_pose[s];
  if (pi < 0) return;
  const int ci = D.s_cam[s], DC = D.DC;
  const int po = D.pose_off[pi], co = D.cam_off[ci], nv = D.cam_width[ci], lp = D.s_lpt[s];
  double y0 = 0.0, y1 = 0.0;
  if (po >= 0) for (int c = 0; c < 6; ++c) { const double v = vec[po + c]; y0 += D.Jc[BA_JC(c, s)] * v; y1 += D.Jc[BA_JC((DC + c), s)] * v; }
  if (co >= 0) for (int c = 0; c < nv; ++c) { const double v = vec[co + c]; y0 += D.Jc[BA_JC((6 + c), s)] * v; y1 += D.Jc[BA_JC((DC + 6 + c), s)] * v; }
  for (int c = 0; c < 3; ++c) atomicAdd(&D.zg[3 * (long long)lp + c], D.Jp[BA_JP(c, s)] * y0 + D.Jp[BA_JP(3 + c, s)] * y1);
}
template <int MODE>
__global__ void __launch_bounds__(BA_BLOCK) ba_giant_finish_kernel(const BaDev D, const double* __restrict__ vec) {
  __shared__ double sm[8];
  if (MODE == 0 && D.ctl->done) return;
  const long long s = (long long)(blockIdx.x + D.nblocks_giant0) * BA_BLOCK + threadIdx.x;
  const int pi = D.s_pose[s];
  double m = 0.0;
  if (pi >= 0) {
    const int ci = D.s_cam[s], DC = D.DC;
    const int po = D.pose_off[pi], co = D.cam_off[ci], nv = D.cam_width[ci], lp = D.s_lpt[s];
    double y0 = 0.0, y1 = 0.0;
    if (po >= 0) for (int c = 0; c < 6; ++c) { const double v = vec[po + c]; y0 += D.Jc[BA_JC(c, s)] * v; y1 += D.Jc[BA_JC((DC + c), s)] * v; }
    if (co >= 0) for (int c = 0; c < nv; ++c) { const double v = vec[co + c]; y0 += D.Jc[BA_JC((6 + c), s)] * v; y1 += D.Jc[BA_JC((DC + 6 + c), s)] * v; }
    const double* I = D.Hpp_inv + 6 * (long long)lp;
    double z0 = D.zg[3 * (long long)lp], z1 = D.zg[3 * (long long)lp + 1], z2 = D.zg[3 * (long long)lp + 2];
    if (MODE == 1) { z0 = -D.gp[3 * (long long)lp] - z0; z1 = -D.gp[3 * (long long)lp + 1] - z1; z2 = -D.gp[3 * (long long)lp + 2] - z2; }
    const double w0 = I[0] * z0 + I[1] * z1 + I[2] * z2, w1 = I[1] * z0 + I[3] * z1 + I[4] * z2, w2 = I[2] * z0 + I[4] * z1 + I[5] * z2;
    const double j0 = D.Jp[BA_JP(0, s)] * w0 + D.Jp[BA_JP(1, s)] * w1 + D.Jp[BA_JP(2, s)] * w2;
    const double j1 = D.Jp[BA_JP(3, s)] * w0 + D.Jp[BA_JP(4, s)] * w1 + D.Jp[BA_JP(5, s)] * w2;
    if (MODE == 0) {
      const long long cp = D.s2c[s];
      D.u[cp] = make_float2((float)(y0 - j0), (float)(y1 - j1));
    } else {
      if ((int)s == D.vpt_s0[lp]) { D.dp[3 * (long long)lp] = w0; D.dp[3 * (long long)lp + 1] = w1; D.dp[3 * (long long)lp + 2] = w2; }
      y0 += j0; y1 += j1;
      m = -(y0 * (D.r[s] + 0.5 * y0) + y1 * (D.r[D.nslots + s] + 0.5 * y1));
    }
  }
  if (MODE == 1) {
    const double t = ba_block_sum(m, sm);
    if (threadIdx.x == 0) atomicAdd(&D.ctl->model, t);
  }
}


// ------------------------------------------------------------------------------------------------
// DENSE_SCHUR: the reduced camera matrix S = H_cc + D_c^2 - H_cp (H_pp + D_p^2)^-1 H_pc formed explicitly and factorised
// (ceres DENSE_SCHUR = SchurEliminator + dense Cholesky; COLMAP picks it for <= 50 images, bundle_adjustment_ceres.cc:
// 202-206).  Built from the same fp32-stored scaled Jacobians the implicit operator of the PCG path reads.
// ------------------------------------------------------------------------------------------------
template <int DC>
__device__ __forceinline__ void ba_slot_rows(const BaDev& D, long long s, float* J0, float* J1, int* idx) {
  const int4 pk = __ldg(D.s_pack + s);
  const unsigned pky = (unsigned)pk.y;
  const int po = pk.x;
  int co, nv;
  ba_unpack_cam(pky, DC > 11 ? D.wide : 0, co, nv);
#pragma unroll
  for (int c = 0; c < DC; ++c) { J0[c] = D.Jc[BA_JC(c, s)]; J1[c] = D.Jc[BA_JC(DC + c, s)]; }
#pragma unroll
  for (int c = 0; c < DC; ++c) idx[c] = (c < 6) ? (po >= 0 ? po + c : -1) : ((co >= 0 && c - 6 < nv) ? co + c - 6 : -1);
  if (pk.w < 0) {
#pragma unroll
    for (int c = 0; c < DC; ++c) idx[c] = -1;
  }
}
// S += J_c^T J_c, one thread per observation slot (pose block, intrinsics block and their coupling)
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_dense_gram_kernel(const BaDev D) {
  const long long s = (long long)blockIdx.x * BA_BLOCK + threadIdx.x;
  float J0[DC], J1[DC];
  int idx[DC];
  ba_slot_rows<DC>(D, s, J0, J1, idx);
#pragma unroll
  for (int r = 0; r < DC; ++r) {
    if (idx[r] < 0) continue;
#pragma unroll
    for (int c = 0; c < DC; ++c)
      if (idx[c] >= 0 && idx[r] >= idx[c])   // lower triangle only: element (i, j), i >= j, lives at Sd[j * nc + i]
        atomicAdd(&D.Sd[(long long)idx[c] * D.nc + idx[r]], (double)J0[r] * (double)J0[c] + (double)J1[r] * (double)J1[c]);
  }
}
// S -= sum over the pairs (i, j) of a track of W_i^T Hinv W_j with W_o = J_p(o)^T J_c(o); one warp per variable point
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_dense_schur_kernel(const BaDev D) {
  const int k = blockIdx.x * (BA_BLOCK / 32) + (threadIdx.x >> 5);
  if (k >= D.nvpt) return;
  const int lane = threadIdx.x & 31;
  const int s0 = D.vpt_s0[k], L = D.vpt_s1[k] - s0;
  const double* I = D.Hpp_inv + 6 * (long long)k;
  const double Hi[9] = {I[0], I[1], I[2], I[1], I[3], I[4], I[2], I[4], I[5]};
  for (long long t = lane; t < (long long)L * L; t += 32) {
    const int i = (int)(t / L), j = (int)(t - (long long)i * L);
    float A0[DC], A1[DC], B0[DC], B1[DC];
    int ia[DC], ib[DC];
    ba_slot_rows<DC>(D, s0 + i, A0, A1, ia);
    ba_slot_rows<DC>(D, s0 + j, B0, B1, ib);
    double pa[6], pb[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) { pa[c] = D.Jp[BA_JP(c, s0 + i)]; pb[c] = D.Jp[BA_JP(c, s0 + j)]; }
    // G = Hinv W_j (3 x DC)
    double G[3][DC];
#pragma unroll
    for (int c = 0; c < DC; ++c) {
      const double w0 = pb[0] * B0[c] + pb[3] * B1[c], w1 = pb[1] * B0[c] + pb[4] * B1[c], w2 = pb[2] * B0[c] + pb[5] * B1[c];
      G[0][c] = Hi[0] * w0 + Hi[1] * w1 + Hi[2] * w2;
      G[1][c] = Hi[3] * w0 + Hi[4] * w1 + Hi[5] * w2;
      G[2][c] = Hi[6] * w0 + Hi[7] * w1 + Hi[8] * w2;
    }
#pragma unroll
    for (int r = 0; r < DC; ++r) {
      if (ia[r] < 0) continue;
      const double v0 = pa[0] * A0[r] + pa[3] * A1[r], v1 = pa[1] * A0[r] + pa[4] * A1[r], v2 = pa[2] * A0[r] + pa[5] * A1[r];
#pragma unroll
      for (int c = 0; c < DC; ++c)
        if (ib[c] >= 0 && ia[r] >= ib[c]) atomicAdd(&D.Sd[(long long)ib[c] * D.nc + ia[r]], -(v0 * G[0][c] + v1 * G[1][c] + v2 * G[2][c]));
    }
  }
}
// S += D_c^2 on the diagonal, Cholesky S = L L^T in place (lower triangle, left-looking, one CTA), then L L^T x = rhs.
// The matrix is symmetric, so "row i" is read as column i: consecutive threads touch consecutive addresses.
#define BA_DENSE_T 1024
// tools/ba_small.py compares the two: the mapper's small reduced systems (nc = 64-80) are faster dense than by PCG to
// 1e-12, while at nc = 450 (50 images, 80k observations) the dense build's 41M fp64 atomics per LM iteration lose - so
// dense only below 256
#define BA_DENSE_MAX 256   // tests/test_ba_paths_gpu.py mirrors this threshold
__global__ void __launch_bounds__(BA_DENSE_T) ba_dense_solve_kernel(const BaDev D) {
  __shared__ double s_d;
  __shared__ int s_bad;
  const int n = D.nc, tid = threadIdx.x;
  double* S = D.Sd;
  // element (i, j), i >= j, of the lower triangle lives at S[j * n + i]
  if (tid == 0) s_bad = 0;
  for (int i = tid; i < n; i += BA_DENSE_T) S[(long long)i * n + i] += D.Dc2[i];
  __syncthreads();
  for (int j = 0; j < n; ++j) {
    // column j: L(i, j) = (S(i, j) - sum_{k < j} L(i, k) L(j, k)) / L(j, j), i = j .. n - 1
    for (int i = j + tid; i < n; i += BA_DENSE_T) {
      double acc = S[(long long)j * n + i];
      for (int k = 0; k < j; ++k) acc -= S[(long long)k * n + i] * S[(long long)k * n + j];
      S[(long long)j * n + i] = acc;
    }
    __syncthreads();
    if (tid == 0) { const double d = S[(long long)j * n + j]; if (!(d > 0.0)) { s_bad = 1; s_d = 1.0; } else s_d = sqrt(d); }
    __syncthreads();
    const double inv = 1.0 / s_d;
    for (int i = j + tid; i < n; i += BA_DENSE_T) S[(long long)j * n + i] = (i == j) ? s_d : S[(long long)j * n + i] * inv;
    __syncthreads();
  }
  if (s_bad) { if (tid == 0) D.ctl->fail = 1; return; }
  // forward: L y = b (column-oriented), then backward: L^T x = y
  double* x = D.x;
  for (int i = tid; i < n; i += BA_DENSE_T) x[i] = D.rhs[i];
  __syncthreads();
  for (int j = 0; j < n; ++j) {
    if (tid == 0) x[j] = x[j] / S[(long long)j * n + j];
    __syncthreads();
    const double xj = x[j];
    for (int i = j + 1 + tid; i < n; i += BA_DENSE_T) x[i] -= S[(long long)j * n + i] * xj;
    __syncthreads();
  }
  for (int j = n - 1; j >= 0; --j) {
    // x_j = (y_j - sum_{i > j} L(i, j) x_i) / L(j, j): a dot product over column j
    double acc = 0.0;
    for (int i = j + 1 + tid; i < n; i += BA_DENSE_T) acc += S[(long long)j * n + i] * x[i];
    __shared__ double red[33];
    const double tot = ba_cta_allsum(acc, red);
    if (tid == 0) x[j] = (x[j] - tot) / S[(long long)j * n + j];
    __syncthreads();
  }
}

// d_p = Hinv (-g_p - H_pc d_c); also the model cost change -(Jd)^T (r + Jd/2), one thread per slot block-wise
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_backsub_model_kernel(const BaDev D, int blk0) {
  __shared__ double sy[2][BA_BLOCK];
  __shared__ double sw[3][BA_BLOCK];
  __shared__ double sm[8];
  const int blk = blockIdx.x + blk0;
  if (blk >= D.nblocks_giant0 && blk < D.nblocks_giant1) return;
  const long long s = (long long)blk * BA_BLOCK + threadIdx.x;
  const int pi = D.s_pose[s];
  double y0 = 0.0, y1 = 0.0;
  if (pi >= 0) {
    const int ci = D.s_cam[s];
    const int po = D.pose_off[pi], co = D.cam_off[ci], nv = D.cam_width[ci];
    if (po >= 0) for (int c = 0; c < 6; ++c) { const double v = D.x[po + c]; y0 += D.Jc[BA_JC(c, s)] * v; y1 += D.Jc[BA_JC((DC + c), s)] * v; }
    if (co >= 0) for (int c = 0; c < nv; ++c) { const double v = D.x[co + c]; y0 += D.Jc[BA_JC((6 + c), s)] * v; y1 += D.Jc[BA_JC((DC + 6 + c), s)] * v; }
  }
  if (blk < D.nblocks_var) {
    sy[0][threadIdx.x] = y0; sy[1][threadIdx.x] = y1;
    __syncthreads();
    if (threadIdx.x < D.blk_npt[blk]) {
      const int k = D.blk_pt0[blk] + threadIdx.x;
      double t0 = -D.gp[3 * (long long)k], t1 = -D.gp[3 * (long long)k + 1], t2 = -D.gp[3 * (long long)k + 2];
      for (int t = D.vpt_s0[k]; t < D.vpt_s1[k]; ++t) {
        const int l = t - blk * BA_BLOCK;
        const double a0 = sy[0][l], a1 = sy[1][l];
        t0 -= D.Jp[BA_JP(0, t)] * a0 + D.Jp[BA_JP(3, t)] * a1;
        t1 -= D.Jp[BA_JP(1, t)] * a0 + D.Jp[BA_JP(4, t)] * a1;
        t2 -= D.Jp[BA_JP(2, t)] * a0 + D.Jp[BA_JP(5, t)] * a1;
      }
      const double* I = D.Hpp_inv + 6 * (long long)k;
      const double d0 = I[0] * t0 + I[1] * t1 + I[2] * t2, d1 = I[1] * t0 + I[3] * t1 + I[4] * t2, d2 = I[2] * t0 + I[4] * t1 + I[5] * t2;
      D.dp[3 * (long long)k] = d0; D.dp[3 * (long long)k + 1] = d1; D.dp[3 * (long long)k + 2] = d2;
      sw[0][threadIdx.x] = d0; sw[1][threadIdx.x] = d1; sw[2][threadIdx.x] = d2;
    }
    __syncthreads();
    const int lp = (pi >= 0) ? D.s_lpt[s] : -1;
    if (lp >= 0) {
      const int lt = lp - D.blk_pt0[blk];
      const double w0 = sw[0][lt], w1 = sw[1][lt], w2 = sw[2][lt];
      y0 += D.Jp[BA_JP(0, s)] * w0 + D.Jp[BA_JP(1, s)] * w1 + D.Jp[BA_JP(2, s)] * w2;
      y1 += D.Jp[BA_JP(3, s)] * w0 + D.Jp[BA_JP(4, s)] * w1 + D.Jp[BA_JP(5, s)] * w2;
    }
  }
  double m = 0.0;
  if (pi >= 0) m = -(y0 * (D.r[s] + 0.5 * y0) + y1 * (D.r[D.nslots + s] + 0.5 * y1));
  const double t = ba_block_sum(m, sm);
  if (threadIdx.x == 0) atomicAdd(&D.ctl->model, t);
}

// Warp-packed blocks (tracks of <= 32 observations): the same step with the per-track sums as segmented shuffle
// reductions (cf. ba_spmv_slot) — no shared-memory exchange, no per-track serial loop.
template <int DC>
__global__ void __launch_bounds__(BA_BLOCK) ba_backsub_warp_kernel(const BaDev D) {
  __shared__ double sm[8];
  const long long s = (long long)blockIdx.x * BA_BLOCK + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const int4 pk = __ldg(D.s_pack + s);
  const unsigned pky = (unsigned)pk.y;
  const int po = pk.x;
  int co, nv;
  ba_unpack_cam(pky, DC > 11 ? D.wide : 0, co, nv);
  const int lp = pk.z;
  const long long cp = pk.w;
  float J0[DC], J1[DC], jp[6];
#pragma unroll
  for (int c = 0; c < DC; ++c) { J0[c] = D.Jc[BA_JC(c, s)]; J1[c] = D.Jc[BA_JC(DC + c, s)]; }
#pragma unroll
  for (int c = 0; c < 6; ++c) jp[c] = D.Jp[BA_JP(c, s)];
  const double r0 = D.r[s], r1 = D.r[D.nslots + s];
  int head = lane, last = lane;
  double y0 = 0.0, y1 = 0.0;
  if (cp >= 0) {
    head = (int)((pky >> 22) & 31u); last = (int)((pky >> 27) & 31u);
    if (po >= 0) {
#pragma unroll
      for (int c = 0; c < 6; ++c) { const double v = D.x[po + c]; y0 += (double)J0[c] * v; y1 += (double)J1[c] * v; }
    }
    if (co >= 0) {
#pragma unroll
      for (int c = 0; c < DC - 6; ++c) if (c < nv) { const double v = D.x[co + c]; y0 += (double)J0[6 + c] * v; y1 += (double)J1[6 + c] * v; }
    }
  }
  double z0 = (double)jp[0] * y0 + (double)jp[3] * y1, z1 = (double)jp[1] * y0 + (double)jp[4] * y1, z2 = (double)jp[2] * y0 + (double)jp[5] * y1;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const double t0 = ba_shfl_down_f64(z0, off), t1 = ba_shfl_down_f64(z1, off), t2 = ba_shfl_down_f64(z2, off);
    if (lane + off <= last) { z0 += t0; z1 += t1; z2 += t2; }
  }
  double d0 = 0.0, d1 = 0.0, d2 = 0.0;
  if (lane == head && lp >= 0 && cp >= 0) {
    const double t0 = -D.gp[3 * (long long)lp] - z0, t1 = -D.gp[3 * (long long)lp + 1] - z1, t2 = -D.gp[3 * (long long)lp + 2] - z2;
    const double* I = D.Hpp_inv + 6 * (long long)lp;
    d0 = I[0] * t0 + I[1] * t1 + I[2] * t2; d1 = I[1] * t0 + I[3] * t1 + I[4] * t2; d2 = I[2] * t0 + I[4] * t1 + I[5] * t2;
    D.dp[3 * (long long)lp] = d0; D.dp[3 * (long long)lp + 1] = d1; D.dp[3 * (long long)lp + 2] = d2;
  }
  d0 = ba_shfl_f64(d0, head); d1 = ba_shfl_f64(d1, head); d2 = ba_shfl_f64(d2, head);
  double m = 0.0;
  if (cp >= 0) {
    if (lp >= 0) {
      y0 += (double)jp[0] * d0 + (double)jp[1] * d1 + (double)jp[2] * d2;
      y1 += (double)jp[3] * d0 + (double)jp[4] * d1 + (double)jp[5] * d2;
    }
    m = -(y0 * (r0 + 0.5 * y0) + y1 * (r1 + 0.5 * y1));
  }
  const double t = ba_block_sum(m, sm);
  if (threadIdx.x == 0) atomicAdd(&D.ctl->model, t);
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
static thread_local std::string g_ba_error;
static int ba_fail(int code, const std::string& msg) { g_ba_error = msg; return code; }
#define BA_CUDA(call)                                                                               \
  do {                                                                                              \
    cudaError_t e__ = (call);                                                                       \
    if (e__ != cudaSuccess) return ba_fail(-100, std::string(#call) + ": " + cudaGetErrorString(e__)); \
  } while (0)
#define BA_TRY(call) do { const int rc__ = (call); if (rc__) return rc__; } while (0)   // propagates a b200ba error code

struct BaPool {
  std::vector<std::pair<void*, size_t>> ptrs;
  template <typename T> cudaError_t alloc(T** p, size_t n) {
    const size_t bytes = sizeof(T) * (n ? n : 1);
    cudaError_t e = B200DeviceCache::get().alloc((void**)p, bytes);
    if (e == cudaSuccess) ptrs.push_back({(void*)*p, bytes});
    return e;
  }
  template <typename T> cudaError_t upload(T** p, const std::vector<T>& v, cudaStream_t s) {
    cudaError_t e = alloc(p, v.size());
    if (e != cudaSuccess) return e;
    return cudaMemcpyAsync(*p, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice, s);
  }
  template <typename T> cudaError_t upload(const T** p, const std::vector<T>& v, cudaStream_t s) {   // read-only BaDev fields
    return upload(const_cast<T**>(p), v, s);
  }
  void release() { if (ptrs.empty()) return; cudaDeviceSynchronize(); for (auto& a : ptrs) B200DeviceCache::get().free(a.first, a.second); ptrs.clear(); }
  ~BaPool() { release(); }   // every return path of a solve gives its blocks back
};

static int ba_sm_count() { int dev = 0, n = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); return n; }
// The reduced-system kernels of one solve, chosen once per solve by ba_select_path from nc and the solver type.
// B200BA_NO_DENSE, B200BA_PCG_MULTI, B200BA_MID_GLOBAL, B200BA_MID_PLAIN and B200BA_SPMV_SMEM=0 turn a path off (test
// seams).  B200BA_MID_PLAIN runs small problems through ba_pcg_mid_kernel, the loop that larger ones (B5) take.
struct BaPath {
  bool dense;          // dense Cholesky of the explicit reduced camera matrix
  bool fused_pcg;      // single-CTA PCG vector step between the SpMVs (else five kernels per iteration)
  bool spmv_smem;      // SpMV pass 1 of the warp-packed blocks with p staged in shared memory
  size_t mid_smem;     // dynamic shared memory of ba_pcg_mid_kernel (> 0: r in shared memory)
  size_t mid_staged;   // dynamic shared memory of ba_pcg_mid_staged_kernel (> 0: it runs instead of ba_pcg_mid_kernel)
  int max_cg, sms;
  double r_tol;        // relative residual that ends an exact PCG solve; -1 for ITERATIVE_SCHUR
};
#define BA_SPMV_SMEM_MAX (72 * 1024)   // tests/test_ba_paths_gpu.py mirrors this threshold
template <int DC>
static void ba_launch_spmv(const BaDev& D, const BaPath& P, cudaStream_t s) {
  if (D.nblocks_warp) {
    const size_t smem = sizeof(double) * (size_t)D.nc;
    if (P.spmv_smem) {
      const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(5, (size_t)(216 * 1024) / (smem + 1024)));
      const int grid = std::min(D.nblocks_warp, P.sms * per_sm);
      ba_schur_spmv_warp_smem_kernel<DC><<<grid, BA_BLOCK, smem, s>>>(D, D.p);
    } else {
      ba_schur_spmv_warp_kernel<DC><<<D.nblocks_warp, BA_BLOCK, 0, s>>>(D, D.p);
    }
  }
  if (D.nblocks > D.nblocks_warp) ba_schur_spmv_kernel<DC><<<D.nblocks - D.nblocks_warp, BA_BLOCK, 0, s>>>(D, D.p, D.q);
  if (D.nblocks_giant1 > D.nblocks_giant0) {
    cudaMemsetAsync(D.zg, 0, sizeof(double) * 3 * (size_t)D.nvpt, s);
    ba_giant_accumulate_kernel<0><<<D.nblocks_giant1 - D.nblocks_giant0, BA_BLOCK, 0, s>>>(D, D.p);
    ba_giant_finish_kernel<0><<<D.nblocks_giant1 - D.nblocks_giant0, BA_BLOCK, 0, s>>>(D, D.p);
  }
  if (D.nobs_c) {
    const long long ntiles = (D.nobs_c + 31) / 32;
    const long long warps = (long long)P.sms * 2 * (BA_BLOCK / 32) * 2;   // two waves of two resident CTAs per SM
    const int tpw = (int)std::max<long long>(4, (ntiles + warps - 1) / warps);
    const unsigned grid = (unsigned)((ntiles + (long long)tpw * (BA_BLOCK / 32) - 1) / ((long long)tpw * (BA_BLOCK / 32)));
    ba_cam_stream_loop_kernel<DC><<<grid, BA_BLOCK, 0, s>>>(D, D.q, 1, tpw);
  }
}
__global__ void ba_prior_dense_kernel(const BaDev D, const BaPrior P);
template <int DC>
static void ba_launch_dense(const BaDev& D, const BaPrior& P, cudaStream_t s) {
  cudaMemsetAsync(D.Sd, 0, sizeof(double) * (size_t)D.nc * D.nc, s);
  ba_dense_gram_kernel<DC><<<D.nblocks, BA_BLOCK, 0, s>>>(D);
  if (D.nvpt) ba_dense_schur_kernel<DC><<<(D.nvpt + BA_BLOCK / 32 - 1) / (BA_BLOCK / 32), BA_BLOCK, 0, s>>>(D);
  if (P.n) ba_prior_dense_kernel<<<(P.n + 255) / 256, 256, 0, s>>>(D, P);
  ba_dense_solve_kernel<<<1, BA_DENSE_T, 0, s>>>(D);
}
template <int DC>
static void ba_launch_backsub(const BaDev& D, cudaStream_t s) {
  if (D.nblocks_warp) ba_backsub_warp_kernel<DC><<<D.nblocks_warp, BA_BLOCK, 0, s>>>(D);
  if (D.nblocks > D.nblocks_warp) ba_backsub_model_kernel<DC><<<D.nblocks - D.nblocks_warp, BA_BLOCK, 0, s>>>(D, D.nblocks_warp);
  if (D.nblocks_giant1 > D.nblocks_giant0) {
    cudaMemsetAsync(D.zg, 0, sizeof(double) * 3 * (size_t)D.nvpt, s);
    ba_giant_accumulate_kernel<1><<<D.nblocks_giant1 - D.nblocks_giant0, BA_BLOCK, 0, s>>>(D, D.x);
    ba_giant_finish_kernel<1><<<D.nblocks_giant1 - D.nblocks_giant0, BA_BLOCK, 0, s>>>(D, D.x);
  }
}
// DC = 6 + widest camera block.  6..11: the narrow layout (trivial frames, <= 5-parameter models); 14 / 18 / 22 / 28: the wide
// instantiations (any model, rig sensors), DC rounded up to the next of them.
template <int DC>
static void ba_launch_linearize(const BaDev& D, int apply_scale, cudaStream_t s) {
  constexpr bool WIDE = DC >= 14;
  ba_linearize_slot_kernel<DC, WIDE><<<D.nblocks, BA_BLOCK, 0, s>>>(D, apply_scale, &D.ctl->cost);
  if (D.nobs_c) ba_linearize_cam_kernel<DC, WIDE><<<(unsigned)((D.nobs_c + BA_BLOCK - 1) / BA_BLOCK), BA_BLOCK, 0, s>>>(D, apply_scale);
}
#define BA_DISPATCH_DC(FN, D, ...)               \
  switch ((D).DC) {                              \
    case 6: FN<6>(D, __VA_ARGS__); break;        \
    case 7: FN<7>(D, __VA_ARGS__); break;        \
    case 8: FN<8>(D, __VA_ARGS__); break;        \
    case 9: FN<9>(D, __VA_ARGS__); break;        \
    case 10: FN<10>(D, __VA_ARGS__); break;      \
    case 11: FN<11>(D, __VA_ARGS__); break;      \
    case 14: FN<14>(D, __VA_ARGS__); break;      \
    case 18: FN<18>(D, __VA_ARGS__); break;      \
    case 22: FN<22>(D, __VA_ARGS__); break;      \
    default: FN<28>(D, __VA_ARGS__); break;      \
  }


// ------------------------------------------------------------------------------------------------
// NCCL binding (point-sharded multi-GPU solve).  libnccl is resolved at run time with dlopen so that the library
// also loads where NCCL is absent; whichever libnccl.so.2 the process already holds (e.g. torch's) is reused.
// ------------------------------------------------------------------------------------------------
#include <dlfcn.h>
#include <nccl.h>
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
#define BA_P2P_MAX_WORLD 8
#define BA_P2P_MAX_BYTES (2u << 20)     // larger payloads (bandwidth-bound) go through NCCL
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

struct BaP2P {
  bool tried = false, ok = false;
  size_t cap = 0, bytes = 0;
  char* local = nullptr;
  char* peer[BA_P2P_MAX_WORLD] = {};
  unsigned long long* state = nullptr;
};
struct b200ba_comm {
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1;
  BaP2P p2p;
};
static void ba_p2p_teardown(b200ba_comm* c) {
  BaP2P& P = c->p2p;
  for (int r = 0; r < BA_P2P_MAX_WORLD; ++r) if (P.peer[r] && r != c->rank) cudaIpcCloseMemHandle(P.peer[r]);
  if (P.local) cudaFree(P.local);
  if (P.state) cudaFree(P.state);
  P = BaP2P();
}
// Collective (every rank calls it with the same `need`): maps the symmetric buffers.  Any failure leaves ok = false and
// the solve keeps using NCCL for its collectives.
static void ba_p2p_ensure(b200ba_comm* c, size_t need_doubles, cudaStream_t st) {
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

// All-reduce of device buffers over the ranks of a sharded solve (no-op without a communicator).  Calls between begin()
// and end() travel together: as ONE launch of the peer-memory kernel when the communicator has its symmetric buffers
// mapped (ba_p2p_ensure) and the payload is latency-sized, else as one NCCL group.
struct BaReducer {
  struct Red { void* buf; size_t count; ncclDataType_t dt; ncclRedOp_t op; const int* done; };
  b200ba_comm* comm = nullptr;   // set only for a sharded solve (world > 1)
  cudaStream_t st = nullptr;
  BaPool* pool = nullptr;        // holds the device copies of agree()
  int sms = 0, launches = 0;     // launches of ba_p2p_allreduce_kernel
  bool grouped = false;
  std::vector<Red> pending;
  cudaError_t operator()(void* buf, size_t count, ncclDataType_t dt, ncclRedOp_t op, const int* done = nullptr) {
    if (!comm || count == 0) return cudaSuccess;
    pending.push_back({buf, count, dt, op, done});
    return grouped ? cudaSuccess : flush();
  }
  void begin() { grouped = true; }
  cudaError_t end() { grouped = false; return flush(); }
  // the host vector v becomes the reduction of every rank's v
  template <typename T> int agree(std::vector<T>& v, ncclDataType_t dt, ncclRedOp_t op) {
    T* d;
    BA_CUDA(pool->upload(&d, v, st));
    BA_CUDA((*this)(d, v.size(), dt, op));
    BA_CUDA(cudaMemcpyAsync(v.data(), d, sizeof(T) * v.size(), cudaMemcpyDeviceToHost, st));
    BA_CUDA(cudaStreamSynchronize(st));
    return 0;
  }
  cudaError_t flush() {
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
};

static int ba_solve_impl(const b200ba_options* o, b200ba_problem* p, b200ba_summary* sum, b200ba_comm* comm,
                         const b200ba_position_priors* priors = nullptr);

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

// FixGaugeWithTwoCamsFromWorld (bundle_adjustment_ceres.cc:308-417), trivial frames, poses in ascending image id.
int b200ba_fix_gauge_two_cams_from_world(const b200ba_problem* p, const b200ba_options* o, uint8_t* pose_constant_out,
                                         int8_t* fixed_dim_out) {
  for (int i = 0; i < p->num_poses; ++i) {
    pose_constant_out[i] = p->pose_constant ? p->pose_constant[i] : 0;
    fixed_dim_out[i] = p->pose_fixed_translation_dim ? p->pose_fixed_translation_dim[i] : -1;
  }
  if (!o->refine_rig_from_world) return 0;
  int image1 = -1, image2 = -1, dim2 = 0;
  for (int i = 0; i < p->num_poses; ++i)
    if (pose_constant_out[i]) {
      if (image1 < 0) image1 = i;
      else return 0;  // two frames already fixed
    }
  for (int i = 0; i < p->num_poses; ++i) {
    if (image1 < 0) { image1 = i; continue; }
    if (i == image1) continue;
    // baseline = (frame1_from_world * inverse(frame_i_from_world)).translation = t1 - R1 R_i^T t_i
    const double* a = p->poses + 7 * image1;
    const double* b = p->poses + 7 * i;
    double Ra[9], Rb[9];
    ba_quat_to_R(a, Ra); ba_quat_to_R(b, Rb);
    double ci[3];  // -R_i^T t_i
    for (int r = 0; r < 3; ++r) ci[r] = -(Rb[r] * b[4] + Rb[3 + r] * b[5] + Rb[6 + r] * b[6]);
    double base[3];
    for (int r = 0; r < 3; ++r) base[r] = Ra[3 * r] * ci[0] + Ra[3 * r + 1] * ci[1] + Ra[3 * r + 2] * ci[2] + a[4 + r];
    int mi = 0;
    for (int r = 1; r < 3; ++r) if (fabs(base[r]) > fabs(base[mi])) mi = r;
    if (fabs(base[mi]) > 1e-9) { image2 = i; dim2 = mi; break; }
  }
  if (image1 < 0 || image2 < 0) return 1;
  pose_constant_out[image1] = 1;
  if (!pose_constant_out[image2]) fixed_dim_out[image2] = (int8_t)dim2;
  return 0;
}

// ---- problem assembly (see the header): DefaultBundleAdjuster's constructor on flat views ----
}  // extern "C"
struct b200ba_assembly {
  std::vector<double> poses, cam_params, points, obs_xy;
  std::vector<uint8_t> pose_constant, cam_constant, point_constant;
  std::vector<int8_t> pose_fixed_dim;
  std::vector<int32_t> cam_model, cam_off, obs_pose, obs_cam, obs_point;
  std::vector<double> sensors;              // rigs: sensor_from_rig of the non-reference cameras
  std::vector<uint8_t> sensor_constant;
  std::vector<int32_t> cam_sensor;
  b200ba_problem problem;
};
extern "C" {

int b200ba_assemble(const b200ba_options* o, const b200ba_scene* sc, const b200ba_config* cfg, b200ba_assembly_t* out) {
  if (!o || !sc || !cfg || !out) return ba_fail(-1, "null argument");
  const int NI = sc->num_images, NC = sc->num_cameras;
  const int64_t NPT = sc->num_points3D;
  auto flag = [](const uint8_t* f, int64_t i) { return f && f[i]; };
  for (int i = 0; i < NI; ++i) if (sc->image_camera[i] < 0 || sc->image_camera[i] >= NC) return ba_fail(-2, "image references a camera outside the scene");
  for (int c = 0; c < NC; ++c) if (ba_model_num_params(sc->camera_model_id[c]) < 0) return ba_fail(-2, "unsupported camera model");
  const int NF = sc->num_frames;
  const bool rigs = NF > 0;
  if (rigs) {
    if (!sc->image_frame || !sc->rig_from_world || !sc->frame_rig || !sc->rig_ref_camera || !sc->camera_rig || !sc->camera_sensor_from_rig)
      return ba_fail(-2, "frames need image_frame, rig_from_world, frame_rig, rig_ref_camera, camera_rig and camera_sensor_from_rig");
    for (int i = 0; i < NI; ++i) if (sc->image_frame[i] < 0 || sc->image_frame[i] >= NF) return ba_fail(-2, "image references a frame outside the scene");
    for (int f = 0; f < NF; ++f) if (sc->frame_rig[f] < 0 || sc->frame_rig[f] >= sc->num_rigs) return ba_fail(-2, "frame references a rig outside the scene");
    for (int c = 0; c < NC; ++c) if (sc->camera_rig[c] < 0 || sc->camera_rig[c] >= sc->num_rigs) return ba_fail(-2, "camera references a rig outside the scene");
    for (int r = 0; r < sc->num_rigs; ++r) if (sc->rig_ref_camera[r] < 0 || sc->rig_ref_camera[r] >= NC) return ba_fail(-2, "rig references a camera outside the scene");
  }
  b200ba_assembly* A = new b200ba_assembly();
  std::vector<int64_t> point_num_obs((size_t)NPT, 0);
  auto track_len = [&](int64_t pid) { return sc->track_offset[pid + 1] - sc->track_offset[pid]; };
  std::vector<int> extra_pose_of_image;     // rigs: constant pose entry of an image outside the config (-1 = none yet)
  if (rigs) { extra_pose_of_image.assign(NI, -1); A->poses.assign(sc->rig_from_world, sc->rig_from_world + 7 * (size_t)NF); }
  auto push = [&](int img, int64_t pid, const double* xy) {
    int pose = img;
    if (rigs) {
      if (flag(cfg->image_in_config, img)) pose = sc->image_frame[img];
      else {
        if (extra_pose_of_image[img] < 0) {
          extra_pose_of_image[img] = (int)(A->poses.size() / 7);
          const double* f = sc->rig_from_world + 7 * (size_t)sc->image_frame[img];
          A->poses.insert(A->poses.end(), f, f + 7);
        }
        pose = extra_pose_of_image[img];
      }
    }
    A->obs_pose.push_back(pose); A->obs_cam.push_back(sc->image_camera[img]); A->obs_point.push_back((int32_t)pid);
    A->obs_xy.push_back(xy[0]); A->obs_xy.push_back(xy[1]);
    point_num_obs[pid] += 1;
  };
  // AddImageToProblem: every observation of the config's images (:688-751); an image (and its camera) counts as
  // parameterized only if it contributed at least one observation (:745-748)
  std::vector<uint8_t> image_parameterized(NI, 0);
  for (int i = 0; i < NI; ++i) {
    if (!flag(cfg->image_in_config, i)) continue;
    const size_t before = A->obs_pose.size();
    for (int64_t k = sc->point2D_offset[i]; k < sc->point2D_offset[i + 1]; ++k) {
      const int64_t pid = sc->point2D_point3D[k];
      if (pid < 0) continue;
      if (pid >= NPT) { delete A; return ba_fail(-2, "point2D references a point outside the scene"); }
      if (flag(cfg->point_ignored, pid)) continue;
      if (track_len(pid) < cfg->min_track_length) continue;
      push(i, pid, sc->point2D_xy + 2 * k);
    }
    if (A->obs_pose.size() > before) image_parameterized[i] = 1;
  }
  // AddPointToProblem: explicit config points bring the observations made by images outside the config (:829-888)
  for (int64_t pid = 0; pid < NPT; ++pid) {
    if (!flag(cfg->point_variable, pid) && !flag(cfg->point_constant, pid)) continue;
    if (cfg->min_track_length > 0 && track_len(pid) < cfg->min_track_length) continue;   // :835-838
    if (point_num_obs[pid] == track_len(pid)) continue;
    for (int64_t t = sc->track_offset[pid]; t < sc->track_offset[pid + 1]; ++t) {
      const int img = sc->track_image[t];
      if (img < 0 || img >= NI) { delete A; return ba_fail(-2, "track references an image outside the scene"); }
      if (flag(cfg->image_in_config, img)) continue;
      const int64_t k = sc->point2D_offset[img] + sc->track_point2D[t];
      if (k < sc->point2D_offset[img] || k >= sc->point2D_offset[img + 1]) { delete A; return ba_fail(-2, "track references a point2D outside its image"); }
      push(img, pid, sc->point2D_xy + 2 * k);
    }
  }
  if (!rigs) A->poses.assign(sc->cam_from_world, sc->cam_from_world + 7 * (size_t)NI);
  const int NPOSE = (int)(A->poses.size() / 7);
  A->pose_constant.assign(NPOSE, 1);
  A->pose_fixed_dim.assign(NPOSE, -1);
  std::vector<uint8_t> cam_in_cfg(NC, 0);
  for (int i = 0; i < NI; ++i)
    if (flag(cfg->image_in_config, i)) {
      if (image_parameterized[i]) cam_in_cfg[sc->image_camera[i]] = 1;
      if (rigs) { if (!flag(cfg->frame_constant_pose, sc->image_frame[i])) A->pose_constant[sc->image_frame[i]] = 0; }
      else if (!flag(cfg->image_constant_pose, i)) A->pose_constant[i] = 0;
    }
  // cameras seen only through constant-pose factors of outside images stay constant (:863-878)
  A->cam_constant.resize(NC);
  for (int c = 0; c < NC; ++c) A->cam_constant[c] = (!cam_in_cfg[c] || flag(cfg->camera_constant, c)) ? 1 : 0;
  A->cam_model.assign(sc->camera_model_id, sc->camera_model_id + NC);
  A->cam_off.assign(sc->camera_param_offset, sc->camera_param_offset + NC);
  int64_t nparams = 0;
  for (int c = 0; c < NC; ++c) nparams = std::max<int64_t>(nparams, sc->camera_param_offset[c] + ba_model_num_params(sc->camera_model_id[c]));
  A->cam_params.assign(sc->camera_params, sc->camera_params + nparams);
  // ParameterizePoints (:540-565): variable iff refined and fully observed inside the problem; explicit constants win
  A->points.assign(sc->xyz, sc->xyz + 3 * (size_t)NPT);
  A->point_constant.assign((size_t)NPT, 1);
  for (int64_t pid = 0; pid < NPT; ++pid) {
    if (point_num_obs[pid] > 0 && o->refine_points3D && track_len(pid) <= point_num_obs[pid]) A->point_constant[pid] = 0;
    if (flag(cfg->point_constant, pid)) A->point_constant[pid] = 1;
  }
  b200ba_problem& P = A->problem;
  memset(&P, 0, sizeof(P));
  P.num_poses = NPOSE; P.poses = A->poses.data(); P.pose_constant = A->pose_constant.data(); P.pose_fixed_translation_dim = A->pose_fixed_dim.data();
  P.num_cameras = NC; P.camera_model_id = A->cam_model.data(); P.camera_param_offset = A->cam_off.data(); P.camera_params = A->cam_params.data();
  P.camera_constant = A->cam_constant.data();
  P.num_points = NPT; P.points = A->points.data(); P.point_constant = A->point_constant.data();
  P.num_observations = (int64_t)A->obs_pose.size();
  P.obs_pose_idx = A->obs_pose.data(); P.obs_camera_idx = A->obs_cam.data(); P.obs_point_idx = A->obs_point.data(); P.obs_xy = A->obs_xy.data();
  P.num_config_images = 0;
  for (int i = 0; i < NI; ++i) if (flag(cfg->image_in_config, i)) P.num_config_images += 1;   // config.NumImages() (:131)
  bool three_points = cfg->fixed_gauge == 2;
  if (rigs) {
    // ParameterizeRigsAndFrames (:470-538): sensor_from_rig is constant when not refined, constant in the config, or when
    // the reference sensor of its rig is not part of the problem.  Sensors = non-reference cameras, ascending camera index.
    A->cam_sensor.assign(NC, -1);
    for (int c = 0; c < NC; ++c)
      if (sc->rig_ref_camera[sc->camera_rig[c]] != c) {
        A->cam_sensor[c] = (int32_t)A->sensor_constant.size();
        A->sensors.insert(A->sensors.end(), sc->camera_sensor_from_rig + 7 * (size_t)c, sc->camera_sensor_from_rig + 7 * (size_t)c + 7);
        // (a parameter block only through a parameterized image of the config on that camera; outside images are baked)
        A->sensor_constant.push_back((!o->refine_sensor_from_rig || flag(cfg->camera_constant_sensor_from_rig, c) || !cam_in_cfg[c]) ? 1 : 0);
      }
    std::vector<uint8_t> rig_param(sc->num_rigs, 0);
    for (int i = 0; i < NI; ++i) if (flag(cfg->image_in_config, i) && image_parameterized[i]) rig_param[sc->frame_rig[sc->image_frame[i]]] = 1;
    for (int c = 0; c < NC; ++c) {
      const int r = sc->camera_rig[c];
      if (A->cam_sensor[c] >= 0 && rig_param[r] && !cam_in_cfg[sc->rig_ref_camera[r]]) A->sensor_constant[A->cam_sensor[c]] = 1;
    }
    P.num_sensors = (int)A->sensor_constant.size();
    P.sensor_from_rig = A->sensors.data(); P.sensor_constant = A->sensor_constant.data(); P.camera_sensor_idx = A->cam_sensor.data();
    // FixGaugeWithTwoCamsFromWorld with rigs (:308-417), over the parameterized images in ascending image id
    if (cfg->fixed_gauge == 1 && o->refine_rig_from_world) {
      auto const_sensor = [&](int img) { const int sidx = A->cam_sensor[sc->image_camera[img]]; return sidx < 0 || A->sensor_constant[sidx]; };   // IsParameterizedConstSensor
      int image1 = -1, image2 = -1, dim2 = 0;
      bool done = false;
      for (int i = 0; i < NI && !done; ++i) {
        if (!flag(cfg->image_in_config, i) || !image_parameterized[i]) continue;
        if (flag(cfg->frame_constant_pose, sc->image_frame[i]) && const_sensor(i)) {
          if (image1 < 0) image1 = i;
          else if (sc->image_frame[image1] != sc->image_frame[i]) done = true;   // two frames are already fixed
        }
      }
      if (!done) {
        for (int i = 0; i < NI; ++i) {
          if (!flag(cfg->image_in_config, i) || !image_parameterized[i]) continue;
          const int f = sc->image_frame[i];
          if (image1 < 0 && const_sensor(i)) { image1 = i; continue; }
          if (image1 >= 0 && sc->image_frame[image1] != f && const_sensor(i) && !flag(cfg->frame_constant_pose, f)) {
            // baseline = (frame1_from_world * inverse(frame_from_world)).translation = t1 - R1 R^T t
            const double* a = sc->rig_from_world + 7 * (size_t)sc->image_frame[image1];
            const double* b = sc->rig_from_world + 7 * (size_t)f;
            double Ra[9], Rb[9], ci[3], base[3];
            ba_quat_to_R(a, Ra); ba_quat_to_R(b, Rb);
            for (int r = 0; r < 3; ++r) ci[r] = -(Rb[r] * b[4] + Rb[3 + r] * b[5] + Rb[6 + r] * b[6]);
            for (int r = 0; r < 3; ++r) base[r] = Ra[3 * r] * ci[0] + Ra[3 * r + 1] * ci[1] + Ra[3 * r + 2] * ci[2] + a[4 + r];
            int mi = 0;
            for (int r = 1; r < 3; ++r) if (fabs(base[r]) > fabs(base[mi])) mi = r;
            if (fabs(base[mi]) > 1e-9) { image2 = i; dim2 = mi; break; }
          }
        }
        if (image1 < 0 || image2 < 0) three_points = true;   // "Falling back to fixing Gauge with three points" (:390-394)
        else {
          A->pose_constant[sc->image_frame[image1]] = 1;
          if (!flag(cfg->frame_constant_pose, sc->image_frame[image2])) A->pose_fixed_dim[sc->image_frame[image2]] = (int8_t)dim2;
        }
      }
    }
  }
  // FixGauge (:270-417), TWO_CAMS_FROM_WORLD, trivial frames: the search runs over the config's images in ascending image id
  if (!rigs && cfg->fixed_gauge == 1 && o->refine_rig_from_world) {
    std::vector<int> idx;
    for (int i = 0; i < NI; ++i) if (flag(cfg->image_in_config, i) && image_parameterized[i]) idx.push_back(i);   // parameterized_image_ids_
    std::vector<double> sp(7 * idx.size());
    std::vector<uint8_t> sc_in(idx.size()), sc_out(idx.size());
    std::vector<int8_t> sd_in(idx.size(), -1), sd_out(idx.size());
    for (size_t k = 0; k < idx.size(); ++k) { memcpy(sp.data() + 7 * k, A->poses.data() + 7 * (size_t)idx[k], 56); sc_in[k] = A->pose_constant[idx[k]]; }
    b200ba_problem sub;
    memset(&sub, 0, sizeof(sub));
    sub.num_poses = (int)idx.size(); sub.poses = sp.data(); sub.pose_constant = sc_in.data(); sub.pose_fixed_translation_dim = sd_in.data();
    if (b200ba_fix_gauge_two_cams_from_world(&sub, o, sc_out.data(), sd_out.data()) == 1) {
      three_points = true;   // "Failed to fix Gauge with two cameras. Falling back to fixing Gauge with three points." (:390-394)
    } else {
      for (size_t k = 0; k < idx.size(); ++k) { A->pose_constant[idx[k]] = sc_out[k]; A->pose_fixed_dim[idx[k]] = sd_out[k]; }
    }
  }
  // FixGaugeWithThreePoints (:270-306): three points whose coordinate vectors are linearly independent stay fixed; points
  // that are already constant count first.  The reference walks a hash map (unspecified order); here ascending point id.
  if (three_points) {
    double basis[9];
    int nfixed = 0;
    double max_pivot = 0.0;
    auto maybe_add = [&](const double* X) {   // rank test of [fixed points | X] by Gram-Schmidt, Eigen's default threshold
      if (nfixed >= 3) return false;
      double r[3] = {X[0], X[1], X[2]};
      for (int b = 0; b < nfixed; ++b) {
        const double* q = basis + 3 * b;
        const double d = r[0] * q[0] + r[1] * q[1] + r[2] * q[2];
        for (int c = 0; c < 3; ++c) r[c] -= d * q[c];
      }
      const double nr = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
      const double nx = sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]);
      if (!(nr > 3.0 * 2.220446049250313e-16 * std::max(max_pivot, nx))) return false;
      for (int c = 0; c < 3; ++c) basis[3 * nfixed + c] = r[c] / nr;
      max_pivot = std::max(max_pivot, nx);
      ++nfixed;
      return true;
    };
    for (int64_t pid = 0; pid < NPT && nfixed < 3; ++pid)
      if (point_num_obs[pid] > 0 && A->point_constant[pid]) maybe_add(A->points.data() + 3 * pid);
    for (int64_t pid = 0; pid < NPT && nfixed < 3; ++pid)
      if (point_num_obs[pid] > 0 && !A->point_constant[pid] && maybe_add(A->points.data() + 3 * pid)) A->point_constant[pid] = 1;
    if (nfixed < 3) g_ba_error = "Failed to fix Gauge due to insufficient number of fixed points";   // warning, like the reference
  }
  *out = A;
  return 0;
}
b200ba_problem* b200ba_assembly_problem(b200ba_assembly_t a) { return a ? &a->problem : nullptr; }
void b200ba_assembly_free(b200ba_assembly_t a) { delete a; }

int b200ba_solve(const b200ba_options* o, b200ba_problem* p, b200ba_summary* sum) { return ba_solve_impl(o, p, sum, nullptr); }

// Point-sharded solve: every rank passes the SAME poses / cameras and its own shard of points with all their
// observations (SURVEY.md §8e).  Collectives: one all-reduce of the camera-side vector per PCG iteration, a handful
// of small ones per LM iteration.  poses / camera_params come back identical on every rank.
int b200ba_solve_sharded(const b200ba_options* o, b200ba_problem* p, b200ba_comm_t comm, b200ba_summary* sum) {
  if (!comm) return ba_fail(-1, "null communicator");
  return ba_solve_impl(o, p, sum, comm);
}
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

// ---- host flattening: everything a solve decides before the device is involved ----
// The slot layout packs whole tracks into blocks of BA_BLOCK slots.  The host only decides WHICH observation sits in
// which slot (s_obs); every per-slot / per-camera-order array is built on the device from the caller's arrays.
struct BaLayout {
  bool wide = false;                 // any camera model beyond the <= 5-parameter family, or any rig sensor
  bool nothing_to_solve = false;     // no effective observation or no effective parameter
  int lst = 0;                       // linear solver type, AUTO resolved
  std::vector<int> pose_off, cam_off, cam_nvar, cam_poff, cam_model, pt_var, cam_sensor, cam_ns, cam_width, sens_cam;
  std::vector<unsigned char> pose_mask;
  std::vector<signed char> cam_var;  // [ncams * BA_MAXP] indices of the variable intrinsics
  std::vector<int> blk_start, blk_pack, blk_split, off2blk;                        // camera-side blocks
  std::vector<int> s_obs, s_lpt, s_seg, blk_pt0, blk_npt, vpt_s0, vpt_s1, vpt_point;  // slots, variable points
  int nc = 0, nblk = 0, pack = 0, dkmax = 0, DC = 6, nvpt = 0, pose_by_pt = 0;
  int nblocks = 0, nblocks_warp = 0, nblocks_giant0 = 0, nblocks_giant1 = 0;
  long long ncamparams = 0, nobs_eff = 0;   // nobs_eff: observations of this rank connected to a variable block
};

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
static int ba_flatten(const b200ba_options* o, const b200ba_problem* p, BaReducer* red, BaLayout& L, b200ba_summary* sum) {
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
template <int DC> static void ba_allow_spmv_smem(const BaLayout&, cudaError_t* e) {
  *e = cudaFuncSetAttribute(ba_schur_spmv_warp_smem_kernel<DC>, cudaFuncAttributeMaxDynamicSharedMemorySize, BA_SPMV_SMEM_MAX);
}
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
  cudaError_t spmv_attr = cudaSuccess;
  if (P.spmv_smem && sizeof(double) * (size_t)nc > 48 * 1024) BA_DISPATCH_DC(ba_allow_spmv_smem, L, &spmv_attr);
  BA_CUDA(spmv_attr);
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
static int ba_upload(const BaLayout& L, const b200ba_options* o, const b200ba_problem* p, const BaPath& path,
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
// ---- position priors (PosePriorBundleAdjuster, bundle_adjustment_ceres.cc:987-1039; DESIGN.md §3) ----
// One covariance-weighted 3-vector residual per prior on camera-side blocks only (a frame's rig_from_world and, for a
// non-reference sensor, its sensor_from_rig), so the priors add to the reduced camera matrix directly and never enter the
// point elimination.  Everything per prior is fp64 and one thread per prior; each LM phase gets one extra launch, and
// only when the solve has priors.
// AbsolutePosePositionPriorCostFunctor / AbsoluteRigPosePositionPriorCostFunctor (cost_functions/pose_prior.h:75-126):
// r = c + R^T t of cam_from_world = sensor_from_rig * rig_from_world (sensor == nullptr: identity), and its Jacobians in the
// tangent space of ba_quat_plus, [rotation | translation], 3x6 row-major.  Plus multiplies by [sin|d| d/|d|, cos|d|] on
// the left, i.e. R' = (I + 2 [d]x) R to first order, so d(R^T u)/dd = 2 R^T [u]x.
BA_HD void ba_prior_position(const double* rig, const double* sensor, const double* c, double* res, double* Jr, double* Js) {
  double Rr[9], Rs[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, ts[3] = {0, 0, 0};
  ba_quat_to_R(rig, Rr);
  if (sensor) { ba_quat_to_R(sensor, Rs); ts[0] = sensor[4]; ts[1] = sensor[5]; ts[2] = sensor[6]; }
  double v[3], u[3];   // v = R_s^T t_s, u = v + t_r
  for (int a = 0; a < 3; ++a) { v[a] = Rs[a] * ts[0] + Rs[3 + a] * ts[1] + Rs[6 + a] * ts[2]; u[a] = v[a] + rig[4 + a]; }
  double A[9];         // A = R_r^T R_s^T
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) A[3 * a + b] = Rr[a] * Rs[3 * b] + Rr[3 + a] * Rs[3 * b + 1] + Rr[6 + a] * Rs[3 * b + 2];
  for (int a = 0; a < 3; ++a) res[a] = c[a] + Rr[a] * u[0] + Rr[3 + a] * u[1] + Rr[6 + a] * u[2];
  const double ux[9] = {0, -u[2], u[1], u[2], 0, -u[0], -u[1], u[0], 0};
  const double tx[9] = {0, -ts[2], ts[1], ts[2], 0, -ts[0], -ts[1], ts[0], 0};
  for (int a = 0; a < 3; ++a)
    for (int j = 0; j < 3; ++j) {
      Jr[6 * a + j] = 2.0 * (Rr[a] * ux[j] + Rr[3 + a] * ux[3 + j] + Rr[6 + a] * ux[6 + j]);
      Jr[6 * a + 3 + j] = Rr[3 * j + a];
      Js[6 * a + j] = sensor ? 2.0 * (A[3 * a] * tx[j] + A[3 * a + 1] * tx[3 + j] + A[3 * a + 2] * tx[6 + j]) : 0.0;
      Js[6 * a + 3 + j] = sensor ? A[3 * a + j] : 0.0;
    }
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
// weighted residual (and, when Jw is set, its weighted tangent Jacobian 3 x 12 [pose | sensor] with the columns of constant
// blocks and of masked pose dimensions zero) of prior k at (poses, sensors)
__device__ __forceinline__ void ba_prior_eval(const BaDev& D, const BaPrior& P, int k, const double* poses, const double* sensors,
                                              double* rw, double* Jw) {
  const int4 ix = P.idx[k];
  double pose[7], sens[7], c[3], res[3], Jr[18], Js[18];
  for (int j = 0; j < 7; ++j) pose[j] = poses[7 * (long long)ix.x + j];
  if (ix.y >= 0) for (int j = 0; j < 7; ++j) sens[j] = sensors[7 * (long long)ix.y + j];
  for (int j = 0; j < 3; ++j) c[j] = P.c[3 * (long long)k + j];
  ba_prior_position(pose, ix.y >= 0 ? sens : nullptr, c, res, Jr, Js);
  const double* W = P.W + 9 * (long long)k;
  for (int a = 0; a < 3; ++a) rw[a] = W[3 * a] * res[0] + W[3 * a + 1] * res[1] + W[3 * a + 2] * res[2];
  if (!Jw) return;
  const unsigned m = ix.z >= 0 ? D.pose_mask[ix.x] : 0u;
  for (int a = 0; a < 3; ++a)
    for (int j = 0; j < 6; ++j) {
      const double jr = W[3 * a] * Jr[j] + W[3 * a + 1] * Jr[6 + j] + W[3 * a + 2] * Jr[12 + j];
      const double js = W[3 * a] * Js[j] + W[3 * a + 1] * Js[6 + j] + W[3 * a + 2] * Js[12 + j];
      Jw[12 * a + j] = ((m >> j) & 1u) ? jr : 0.0;
      Jw[12 * a + 6 + j] = ix.w >= 0 ? js : 0.0;
    }
}
// camera-side offset of column j of a prior's Jacobian, or -1
__device__ __forceinline__ int ba_prior_col(const int4& ix, int j) { return j < 6 ? (ix.z >= 0 ? ix.z + j : -1) : (ix.w >= 0 ? ix.w + j - 6 : -1); }
// ceres Corrector of the priors' loss (rho at sq = |rw|^2) applied to the weighted 3 x 12 Jacobian J in place; returns
// the factor of the corrected residual
__device__ __forceinline__ double ba_prior_correct(const BaPrior& P, const double* rw, double sq, const double* rho, double* J) {
  double rs = 1.0;
  if (P.loss_type != B200BA_LOSS_TRIVIAL) {
    const double sqrt_rho1 = sqrt(rho[1]);
    double alpha_sq_norm = 0.0;
    rs = sqrt_rho1;
    if (sq != 0.0 && rho[2] > 0.0) {
      const double alpha = 1.0 - sqrt(1.0 + 2.0 * sq * rho[2] / rho[1]);
      rs = sqrt_rho1 / (1 - alpha);
      alpha_sq_norm = alpha / sq;
    }
    for (int j = 0; j < 12; ++j) {
      const double rj = rw[0] * J[j] + rw[1] * J[12 + j] + rw[2] * J[24 + j];
      for (int a = 0; a < 3; ++a) J[12 * a + j] = sqrt_rho1 * (J[12 * a + j] - alpha_sq_norm * rw[a] * rj);
    }
  }
  return rs;
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
// dense path: the full J^T J (pose-sensor cross block included) into the lower triangle of S (element (i, j), i >= j, at
// Sd[j * nc + i])
__global__ void ba_prior_dense_kernel(const BaDev D, const BaPrior P) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= P.n) return;
  const int4 ix = P.idx[k];
  const double* J = P.J + 36 * (long long)k;
  for (int a = 0; a < 12; ++a) {
    const int ia = ba_prior_col(ix, a);
    if (ia < 0) continue;
    for (int b = 0; b < 12; ++b) {
      const int ib = ba_prior_col(ix, b);
      if (ib >= 0 && ia >= ib) atomicAdd(&D.Sd[(long long)ib * D.nc + ia], J[a] * J[b] + J[12 + a] * J[12 + b] + J[24 + a] * J[24 + b]);
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
static int ba_prior_check(const b200ba_problem* p, const b200ba_position_priors* pr, std::vector<double>& W) {
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
static int ba_prior_setup(const b200ba_position_priors* pr, const std::vector<double>& W, const BaLayout& L, BaPool& pool,
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
    BA_DISPATCH_DC(ba_launch_linearize, D, apply_scale, st);
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
      if (D.nc) { BA_DISPATCH_DC(ba_launch_dense, D, P, st); launches += 3 + (P.n ? 1 : 0); }
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
        BA_DISPATCH_DC(ba_launch_spmv, D, path, st);
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
    BA_DISPATCH_DC(ba_launch_backsub, D, st);
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
                         const b200ba_position_priors* priors) {
  if (!o || !p || !sum) return ba_fail(-1, "null argument");
  memset(sum, 0, sizeof(*sum));
  sum->termination_type = B200BA_FAILURE;
  if (priors && priors->num_priors == 0) priors = nullptr;
  std::vector<double> prior_w;   // checked before any device work
  if (priors) BA_TRY(ba_prior_check(p, priors, prior_w));
  BaPool pool;
  const auto t_setup0 = std::chrono::steady_clock::now();
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return ba_fail(-101, "no CUDA device: colmap_b200 has no CPU fallback");
  if (o->gpu_index >= 0) {
    if (o->gpu_index >= ndev) return ba_fail(-101, "gpu_index out of range");
    cudaSetDevice(o->gpu_index);
  }
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

// ------------------------------------------------------------------------------------------------
// Covariance of a solved problem (EstimateBACovariance, src/colmap/estimators/covariance.cc; DESIGN.md §3).  The solve's
// flattening and device set-up are reused as they are; the Jacobian is re-evaluated in fp64 (no Jacobi scaling) and
// never stored in fp32.  S = H_cc - H_cp (H_pp + damping I)^-1 H_pc over the camera-side rows that the reference keeps,
// ordered [others (sensor_from_rig, intrinsics) | poses], then one dense Cholesky and S^-1 in place (ba_dense_f64.cu).
// With the others first, the pivots of the pose rows are those of S_cc - S_co S_oo^-1 S_oc, so damping the others'
// diagonal and factorising once is SchurEliminateOtherParams followed by the reference's rank test on the pose matrix,
// provided the rank test starts at the first pose row: the others' rows fail only on a pivot <= 0, as the reference's
// LLT of S_oo + damping I does (a weakly determined intrinsic is eliminated, not reported).
// ------------------------------------------------------------------------------------------------
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
static void ba_cov_launch_build(const BaDev& D, const BaCov& C, cudaStream_t s) {
  constexpr bool WIDE = DC >= 14;
  ba_cov_linearize_kernel<DC, WIDE><<<D.nblocks, BA_BLOCK, 0, s>>>(D, C);
  if (C.want_S) ba_cov_gram_kernel<DC><<<D.nblocks, BA_BLOCK, 0, s>>>(D, C);
  if (D.nvpt && (C.want_S || C.pcov)) ba_cov_point_kernel<DC><<<(D.nvpt + BA_BLOCK / 32 - 1) / (BA_BLOCK / 32), BA_BLOCK, 0, s>>>(D, C);
}

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
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return ba_fail(-101, "no CUDA device: colmap_b200 has no CPU fallback");
  if (o->gpu_index >= 0) {
    if (o->gpu_index >= ndev) return ba_fail(-101, "gpu_index out of range");
    cudaSetDevice(o->gpu_index);
  }
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
  BA_DISPATCH_DC(ba_cov_launch_build, D, C, G.st);
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
static int ba_cov_block(b200ba_covariance* h, int r0, int a, int c0, int b, double* out) {
  if (!h || !a || !b) return 0;
  cudaSetDevice(h->dev);
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
  if (!h || !h->pcov || point < 0 || point >= (int64_t)h->pt_var.size() || h->pt_var[point] < 0) return 0;
  cudaSetDevice(h->dev);
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
  cudaSetDevice(h->dev);
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
    cudaSetDevice(h->dev);
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
  cudaSetDevice(h->dev);
  delete h;
}

}  // extern "C"
