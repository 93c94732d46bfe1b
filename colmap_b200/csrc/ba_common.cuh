// ba_common.cuh — what the bundle-adjustment translation units share (internal; the C ABI is include/b200_ba*.h).
//   bundle_adjustment.cu  LM and PCG kernels, layout and upload, the solve and its entry points, the CPU test hooks
//   ba_linearize.cu       per-observation linearisation kernels          ba_spmv.cu            implicit Schur product
//   ba_dense_backsub.cu   dense reduced matrix and back-substitution     ba_covariance.cu      covariance estimate
//   ba_comm.cu            multi-GPU all-reduce (NCCL, peer memory)       ba_assembly.cu        problem assembly, gauge
// Each kernel family templated on the camera-block width DC is instantiated in one unit only and launched through
// that unit's run-time dispatching launcher, so the units compile side by side.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/b200_bundle_adjustment.h"
#include "../../include/b200_ba_covariance.h"
#include "../../include/b200_ba_pose_prior.h"
#include "device_cache.h"
#include "ba_models.cuh"

#include <nccl.h>

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
static __host__ __device__ __noinline__ bool ba_img_from_cam_any(int id, const double* q, double u, double v, double w, double* x, double* y, double* Jp,
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
static __host__ __device__ __noinline__ bool ba_residual_any(int id, const double* point, const double* rig, const double* sensor, const double* params,
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
static __host__ __device__ __noinline__ bool ba_reproj_rig(int id, const double* point, const double* rig, const double* sensor, const double* params, double ox,
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

__device__ __forceinline__ double ba_shfl_down_f64(double v, int off) { return __shfl_down_sync(0xffffffffu, v, off); }
__device__ __forceinline__ double ba_shfl_f64(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }

// s_pack.y = (camera-block offset + 1) | width << (19 | 17) | head lane << 22 | last lane << 27: 19 + 3 bits for the narrow
// layout (width <= 5), 17 + 5 bits when the problem has wide camera blocks
__device__ __forceinline__ void ba_unpack_cam(unsigned pky, int wide, int& co, int& nv) {
  if (wide) { co = (int)(pky & 0x1ffffu) - 1; nv = (int)((pky >> 17) & 31u); }
  else { co = (int)(pky & 0x7ffffu) - 1; nv = (int)((pky >> 19) & 7u); }
}
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
// host
// ------------------------------------------------------------------------------------------------
extern thread_local std::string g_ba_error;   // defined once, in bundle_adjustment.cu: b200ba_last_error reports every unit
inline int ba_fail(int code, const std::string& msg) { g_ba_error = msg; return code; }
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
// tools/ba_small.py compares the two: the mapper's small reduced systems (nc = 64-80) are faster dense than by PCG to
// 1e-12, while at nc = 450 (50 images, 80k observations) the dense build's 41M fp64 atomics per LM iteration lose - so
// dense only below 256
#define BA_DENSE_MAX 256   // tests/test_ba_paths_gpu.py mirrors this threshold

// DC = 6 + widest camera block.  6..11: the narrow layout (trivial frames, <= 5-parameter models); 14 / 18 / 22 / 28: the wide
// instantiations (any model, rig sensors), DC rounded up to the next of them.
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

// the communicator of a sharded solve; ba_p2p_ensure (ba_comm.cu) maps its peer-memory buffers
#define BA_P2P_MAX_WORLD 8
#define BA_P2P_MAX_BYTES (2u << 20)     // larger payloads (bandwidth-bound) go through NCCL
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
  cudaError_t flush();
};

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

// ---- host functions shared by the units ----
int ba_use_device(const b200ba_options* o);
int ba_flatten(const b200ba_options* o, const b200ba_problem* p, BaReducer* red, BaLayout& L, b200ba_summary* sum);
int ba_upload(const BaLayout& L, const b200ba_options* o, const b200ba_problem* p, const BaPath& path, b200ba_comm* comm,
              BaPool& pool, cudaStream_t st, BaDev& D);
int ba_prior_check(const b200ba_problem* p, const b200ba_position_priors* pr, std::vector<double>& W);
int ba_prior_setup(const b200ba_position_priors* pr, const std::vector<double>& W, const BaLayout& L, BaPool& pool,
                   cudaStream_t st, BaPrior& P);
void ba_p2p_ensure(b200ba_comm* c, size_t need_doubles, cudaStream_t st);
// launchers: DC = D.DC, dispatched inside the unit that defines the kernels
void ba_launch_linearize(const BaDev& D, int apply_scale, cudaStream_t s);
void ba_launch_spmv(const BaDev& D, const BaPath& P, cudaStream_t s);
cudaError_t ba_allow_spmv_smem(const BaLayout& L);
void ba_launch_dense(const BaDev& D, const BaPrior& P, cudaStream_t s);
void ba_launch_backsub(const BaDev& D, cudaStream_t s);
