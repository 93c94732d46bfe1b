/*
 * pm_oracle.c — CPU restatement of COLMAP's PatchMatch MVS sweep.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product (colmap_b200/, include/)
 * may call, link or import this file; only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs do.
 *
 * It follows the reference algorithm step by step, including the physical 90
 * degree rotation of every buffer between sweeps (the CUDA product instead
 * sweeps in four directions by index arithmetic, so the two are independent
 * statements of the same schedule):
 *   src/colmap/mvs/patch_match_cuda.cu      (everything; cited per function)
 *   src/colmap/mvs/gpu_mat_ref_image.{h,cu} (bilateral prefilter)
 *   src/colmap/mvs/gpu_mat_prng.cu, gpu_mat.h:371-387 (per-pixel XORWOW states)
 *   src/colmap/mvs/cuda_rotate.h:57-75      (rotation convention)
 *   src/colmap/mvs/image.cc:97-150          (pose helpers)
 *   curand_kernel.h (CUDA toolkit)          (XORWOW, curand_uniform)
 *
 * PARITY STATUS: the reference holds no numerical test of PatchMatchCuda (SURVEY.md §4/§8c) and has no bit-level
 * definition, so bit-level parity with it is undefined.  Pinned instead:
 *   - by the reference's own tests, checked in tests/test_pm_cpu.py + tests/test_golden_cpu.py against
 *     tests/golden/reference_known_answers.json: the rotation convention (gpu_mat_test.cu:188-206), the pose
 *     helpers' known answers (image_test.cc:149-212), the .bin map format;
 *   - by OUTPUTS OF THE REFERENCE ITSELF: the unmodified PatchMatchCuda is compiled in place (oracle/build_ref.sh ->
 *     oracle/_ref/libpm_ref.so) and run on the GPU; depth / normal maps agree statistically (completeness,
 *     accuracy against analytic ground truth, per-pixel agreement: tests/test_pm_gpu.py, fixtures
 *     tests/golden/pm_reference_cuda_160x120.npz and reference_samples.npz).
 * The depth/normal output of THIS file is frozen in tests/golden/pm_case_96x64.npz.
 *
 * Floating-point contract ("the spec"): fp32 throughout, IEEE add/mul/div/sqrt,
 * fused multiply-add ONLY where fmaf() is written, no re-association, and
 * exp/sin/cos are the polynomial routines below (so that the CUDA kernels can
 * match this file bit for bit; the reference itself is built with
 * --use_fast_math and hardware texture filtering and therefore has no
 * bit-level definition).  Documented deviations from the reference, all at the
 * level of fp32 rounding: (1) homography applied per tap directly (as
 * H*(dx,dy,0) + H*(col,row,1)) instead of incrementally (patch_match_cuda.cu:503-569); (2) software bilinear
 * interpolation on raw 8-bit values instead of the 9-bit-weight texture unit;
 * (3) the NCC sums are accumulated in 8 interleaved partial sums joined by a
 * fixed tree; (4) pose matrices are composed in double and rounded once;
 * (5) the magnitude of the per-tap projective depth is clamped to [1e-30, 1e30]
 * before the reciprocal, its sign kept; z = 0 and NaN sample the zero border
 * (where the reference divides by zero).  tests/pm_fp64.py restates the
 * reference in float64 without these deviations; tests/test_pm_fp64_cpu.py
 * holds this file to it within fp32 error bounds.
 *
 * Build: gcc -O2 -ffp-contract=off -mfma -fopenmp -shared -fPIC (see Makefile).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/b200_patch_match.h"

#define PM_MAX_SRC 32
#define PM_POSE_STRIDE 43 /* K(4) R(9) T(3) C(3) P(12) invP(12): patch_match_cuda.cu:1762 */

/* ------------------------------------------------------------------------- */
/* math spec                                                                  */
/* ------------------------------------------------------------------------- */
static inline int32_t f2i_bits(float f) { int32_t i; memcpy(&i, &f, 4); return i; }
static inline float i2f_bits(int32_t i) { float f; memcpy(&f, &i, 4); return f; }

/* exp(x) for x in [-87, 88] (clamped), ~2 ulp. */
static inline float pm_expf(float x) {
  if (!(x > -87.0f)) x = -87.0f;
  if (x > 88.0f) x = 88.0f;
  const float t = fmaf(x, 1.44269504f, 12582912.0f);
  const float n = t - 12582912.0f;
  const int32_t ni = f2i_bits(t) - 0x4B400000;
  float r = fmaf(n, -0.693145752f, x);
  r = fmaf(n, -1.42860677e-6f, r);
  float p = 1.98412698e-4f;       /* 1/5040 */
  p = fmaf(p, r, 1.38888889e-3f); /* 1/720 */
  p = fmaf(p, r, 8.33333333e-3f); /* 1/120 */
  p = fmaf(p, r, 4.16666667e-2f); /* 1/24 */
  p = fmaf(p, r, 1.66666667e-1f); /* 1/6 */
  p = fmaf(p, r, 0.5f);
  p = fmaf(p, r, 1.0f);
  p = fmaf(p, r, 1.0f);
  return i2f_bits(f2i_bits(p) + (ni << 23));
}

/* sin/cos for |a| <= pi/2 (the only range PerturbNormal needs). */
static inline void pm_sincosf(float a, float* s, float* c) {
  const float q = a * a;
  float ps = -2.50521084e-8f;      /* -1/11! */
  ps = fmaf(ps, q, 2.75573192e-6f);  /* 1/9! */
  ps = fmaf(ps, q, -1.98412698e-4f); /* -1/7! */
  ps = fmaf(ps, q, 8.33333333e-3f);  /* 1/5! */
  ps = fmaf(ps, q, -1.66666667e-1f); /* -1/3! */
  ps = ps * q;
  *s = fmaf(ps, a, a);
  float pc = 2.08767570e-9f;       /* 1/12! */
  pc = fmaf(pc, q, -2.75573192e-7f); /* -1/10! */
  pc = fmaf(pc, q, 2.48015873e-5f);  /* 1/8! */
  pc = fmaf(pc, q, -1.38888889e-3f); /* -1/6! */
  pc = fmaf(pc, q, 4.16666667e-2f);  /* 1/4! */
  pc = fmaf(pc, q, -0.5f);
  *c = fmaf(pc, q, 1.0f);
}

static inline float dot3(const float a[3], const float b[3]) {
  return fmaf(a[2], b[2], fmaf(a[1], b[1], a[0] * b[0]));
}

/* ------------------------------------------------------------------------- */
/* XORWOW (curand_kernel.h: _curand_init_inplace, curand(), _curand_uniform)  */
/* ------------------------------------------------------------------------- */
typedef struct { uint32_t v[5]; uint32_t d; } pm_rng;

static inline void rng_init(pm_rng* s, uint64_t seed) {
  const uint32_t s0 = ((uint32_t)seed) ^ 0xaad26b49u;
  const uint32_t s1 = ((uint32_t)(seed >> 32)) ^ 0xf7dcefddu;
  const uint32_t t0 = 1099087573u * s0;
  const uint32_t t1 = 2591861531u * s1;
  s->d = 6615241u + t1 + t0;
  s->v[0] = 123456789u + t0;
  s->v[1] = 362436069u ^ t0;
  s->v[2] = 521288629u + t1;
  s->v[3] = 88675123u ^ t1;
  s->v[4] = 5783321u + t0;
}
static inline uint32_t rng_next(pm_rng* s) {
  const uint32_t t = s->v[0] ^ (s->v[0] >> 2);
  s->v[0] = s->v[1]; s->v[1] = s->v[2]; s->v[2] = s->v[3]; s->v[3] = s->v[4];
  s->v[4] = (s->v[4] ^ (s->v[4] << 4)) ^ (t ^ (t << 1));
  s->d += 362437u;
  return s->v[4] + s->d;
}
static inline float rng_uniform(pm_rng* s) {
  const float x = (float)rng_next(s);
  return x * 2.3283064365386963e-10f + 1.1641532182693481e-10f;
}

/* ------------------------------------------------------------------------- */
/* state of one run                                                           */
/* ------------------------------------------------------------------------- */
typedef struct {
  /* options resolved to floats (patch_match_cuda.cu:1420-1438) */
  int radius, step, nside, ntaps, num_samples, num_iterations;
  int geom, filter, filter_min_num_consistent;
  float depth_min, depth_max, sigma_spatial, sigma_color, ncc_sigma;
  float min_tri_angle_rad, incident_angle_sigma;
  float geom_reg, geom_max_cost, filter_min_ncc, filter_min_tri_rad, filter_geom_max_cost;
  float spatial_norm, color_norm;
  /* likelihood constants (LikelihoodComputer ctor, :700-707) */
  float cos_min_tri, inv_inc_sigma_sq, inv_ncc_sigma_sq, ncc_norm;
  /* geometry */
  int W0, H0;          /* original reference size */
  int w, h;            /* current (rotated) frame size */
  int rot;             /* rotation_in_half_pi_ */
  int N;               /* number of source images */
  float refK[4][4], refinvK[4][4];
  float* poses[4];     /* [N * 43] per rotation */
  /* source images (never rotated) */
  int src_w[PM_MAX_SRC], src_h[PM_MAX_SRC];
  const uint8_t* src_img[PM_MAX_SRC];
  const float* src_depth[PM_MAX_SRC];
  /* rotating buffers, all (h x w) row-major, multi-slice = slice-major */
  uint8_t* ref_img;
  float *ref_sum, *ref_sqsum;
  float *depth, *normal, *cost, *sel_prob, *prev_sel_prob;
  uint8_t* mask; /* allocated for the last sweep if filter */
  pm_rng* rand_state;
  float lut255[256];
} pm_state;

/* ------------------------------------------------------------------------- */
/* pose helpers: image.cc:97-150, composed in double, rounded once            */
/* ------------------------------------------------------------------------- */
static void compose_pose_row(const double refR[9], const double refT[3], const float K[9],
                             const float R2f[9], const float T2f[3], float out[PM_POSE_STRIDE]) {
  double R2[9], T2[3], R[9], T[3], C[3], P[12], invP[12];
  for (int i = 0; i < 9; ++i) R2[i] = R2f[i];
  for (int i = 0; i < 3; ++i) T2[i] = T2f[i];
  /* ComputeRelativePose: R = R2 * R1^T ; T = T2 - R * T1 */
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      R[3 * r + c] = R2[3 * r] * refR[3 * c] + R2[3 * r + 1] * refR[3 * c + 1] + R2[3 * r + 2] * refR[3 * c + 2];
  for (int r = 0; r < 3; ++r)
    T[r] = T2[r] - (R[3 * r] * refT[0] + R[3 * r + 1] * refT[1] + R[3 * r + 2] * refT[2]);
  /* ComputeProjectionCenter: C = -R^T T */
  for (int c = 0; c < 3; ++c) C[c] = -(R[c] * T[0] + R[3 + c] * T[1] + R[6 + c] * T[2]);
  /* ComposeProjectionMatrix: P = K [R | T] */
  const double fx = K[0], cx = K[2], fy = K[4], cy = K[5];
  for (int c = 0; c < 3; ++c) {
    P[c] = fx * R[c] + cx * R[6 + c];
    P[4 + c] = fy * R[3 + c] + cy * R[6 + c];
    P[8 + c] = R[6 + c];
  }
  P[3] = fx * T[0] + cx * T[2];
  P[7] = fy * T[1] + cy * T[2];
  P[11] = T[2];
  /* ComposeInverseProjectionMatrix: top three rows of [P;0 0 0 1]^-1 = [R^T K^-1 | -R^T T] */
  for (int r = 0; r < 3; ++r) {
    invP[4 * r + 0] = R[r] / fx;
    invP[4 * r + 1] = R[3 + r] / fy;
    invP[4 * r + 2] = R[6 + r] - R[r] * cx / fx - R[3 + r] * cy / fy;
    invP[4 * r + 3] = C[r];
  }
  out[0] = K[0]; out[1] = K[2]; out[2] = K[4]; out[3] = K[5];
  for (int i = 0; i < 9; ++i) out[4 + i] = (float)R[i];
  for (int i = 0; i < 3; ++i) out[13 + i] = (float)T[i];
  for (int i = 0; i < 3; ++i) out[16 + i] = (float)C[i];
  for (int i = 0; i < 12; ++i) out[19 + i] = (float)P[i];
  for (int i = 0; i < 12; ++i) out[31 + i] = (float)invP[i];
}

/* InitTransforms: patch_match_cuda.cu:1694-1808 */
static void init_transforms(pm_state* st, const b200pm_problem* p) {
  const float fx = p->ref_K[0], cx = p->ref_K[2], fy = p->ref_K[4], cy = p->ref_K[5];
  const float Wm1 = (float)(st->W0 - 1), Hm1 = (float)(st->H0 - 1);
  const float K4[4][4] = {{fx, cx, fy, cy}, {fy, cy, fx, Wm1 - cx}, {fx, Wm1 - cx, fy, Hm1 - cy}, {fy, Hm1 - cy, fx, cx}};
  for (int k = 0; k < 4; ++k) {
    for (int i = 0; i < 4; ++i) st->refK[k][i] = K4[k][i];
    st->refinvK[k][0] = 1.0f / K4[k][0];
    st->refinvK[k][1] = -K4[k][1] / K4[k][0];
    st->refinvK[k][2] = 1.0f / K4[k][2];
    st->refinvK[k][3] = -K4[k][3] / K4[k][2];
  }
  double R[9], T[3];
  for (int i = 0; i < 9; ++i) R[i] = p->ref_R[i];
  for (int i = 0; i < 3; ++i) T[i] = p->ref_T[i];
  for (int k = 0; k < 4; ++k) {
    st->poses[k] = (float*)malloc(sizeof(float) * PM_POSE_STRIDE * st->N);
    for (int i = 0; i < st->N; ++i)
      compose_pose_row(R, T, p->src_K + 9 * i, p->src_R + 9 * i, p->src_T + 3 * i, st->poses[k] + PM_POSE_STRIDE * i);
    /* RotatePose with R_z90 = [0 1 0; -1 0 0; 0 0 1] (image.cc:144-150) */
    double nR[9], nT[3];
    for (int c = 0; c < 3; ++c) { nR[c] = R[3 + c]; nR[3 + c] = -R[c]; nR[6 + c] = R[6 + c]; }
    nT[0] = T[1]; nT[1] = -T[0]; nT[2] = T[2];
    memcpy(R, nR, sizeof(R)); memcpy(T, nT, sizeof(T));
  }
}

/* ------------------------------------------------------------------------- */
/* rotation: cuda_rotate.h:57-75  out(row = W-1-x, col = y) = in(row = y, col = x) */
/* ------------------------------------------------------------------------- */
#define DEFINE_ROTATE(NAME, T)                                                      \
  static T* NAME(T* in, int w, int h, int slices) {                                \
    T* out = (T*)malloc(sizeof(T) * (size_t)w * h * slices);                        \
    for (int s = 0; s < slices; ++s)                                                \
      for (int y = 0; y < h; ++y)                                                   \
        for (int x = 0; x < w; ++x)                                                 \
          out[(size_t)s * w * h + (size_t)(w - 1 - x) * h + y] = in[(size_t)s * w * h + (size_t)y * w + x]; \
    free(in);                                                                       \
    return out;                                                                     \
  }
DEFINE_ROTATE(rotate_f32, float)
DEFINE_ROTATE(rotate_u8, uint8_t)
DEFINE_ROTATE(rotate_rng, pm_rng)

/* exported for the rotate-convention test (gpu_mat_test.cu:188-206) */
void pm_oracle_rotate_f32(const float* in, int w, int h, int slices, float* out) {
  float* tmp = (float*)malloc(sizeof(float) * (size_t)w * h * slices);
  memcpy(tmp, in, sizeof(float) * (size_t)w * h * slices);
  tmp = rotate_f32(tmp, w, h, slices);
  memcpy(out, tmp, sizeof(float) * (size_t)w * h * slices);
  free(tmp);
}

/* PatchMatchCuda::Rotate: patch_match_cuda.cu:1859-1939 */
static void rotate_all(pm_state* st, int after_sweep) {
  const int w = st->w, h = st->h;
  const size_t n = (size_t)w * h;
  st->rand_state = rotate_rng(st->rand_state, w, h, 1);
  st->depth = rotate_f32(st->depth, w, h, 1);
  /* RotateNormalMap (:849-861): (nx,ny,nz) -> (ny,-nx,nz), then rotate */
  for (size_t i = 0; i < n; ++i) {
    const float nx = st->normal[i], ny = st->normal[n + i];
    st->normal[i] = ny;
    st->normal[n + i] = -nx;
  }
  st->normal = rotate_f32(st->normal, w, h, 3);
  st->ref_img = rotate_u8(st->ref_img, w, h, 1);
  st->ref_sum = rotate_f32(st->ref_sum, w, h, 1);
  st->ref_sqsum = rotate_f32(st->ref_sqsum, w, h, 1);
  if (after_sweep) {
    free(st->prev_sel_prob);
    st->prev_sel_prob = rotate_f32(st->sel_prob, w, h, st->N);
    st->sel_prob = (float*)malloc(sizeof(float) * n * st->N);
  } else { /* only used to bring a partial run back to the original orientation */
    st->prev_sel_prob = rotate_f32(st->prev_sel_prob, w, h, st->N);
  }
  st->cost = rotate_f32(st->cost, w, h, st->N);
  st->w = h; st->h = w;
  st->rot = (st->rot + 1) % 4;
}

/* ------------------------------------------------------------------------- */
/* reference image access + bilateral weights                                 */
/* ------------------------------------------------------------------------- */
/* point-sampled, border -> 0 (BindRefImageTexture :1565-1576) */
static inline float ref_color(const pm_state* st, int row, int col) {
  if (row < 0 || col < 0 || row >= st->h || col >= st->w) return 0.0f;
  return st->lut255[st->ref_img[(size_t)row * st->w + col]];
}

/* BilateralWeightComputer::Compute: gpu_mat_ref_image.h:70-90 */
static inline float bilateral_weight(const pm_state* st, int dr, int dc, float c1, float c2) {
  const float sd = (float)(dr * dr + dc * dc);
  const float a1 = sd * st->spatial_norm;
  const float cd = c1 - c2;
  const float a2 = cd * cd;
  return pm_expf(fmaf(-a2, st->color_norm, -a1));
}

/* GpuMatRefImage::Filter / FilterKernel: gpu_mat_ref_image.cu:39-82 */
static void filter_ref_image(pm_state* st, const uint8_t* gray) {
  const int w = st->w, h = st->h, r = st->radius, s = st->step;
  uint8_t* out = (uint8_t*)malloc((size_t)w * h);
#pragma omp parallel for schedule(static)
  for (int row = 0; row < h; ++row) {
    for (int col = 0; col < w; ++col) {
      const float center = st->lut255[gray[(size_t)row * w + col]];
      float cs = 0.0f, cq = 0.0f, ws = 0.0f;
      for (int dr = -r; dr <= r; dr += s) {
        for (int dc = -r; dc <= r; dc += s) {
          const int rr = row + dr, cc = col + dc;
          const float color = (rr < 0 || cc < 0 || rr >= h || cc >= w) ? 0.0f : st->lut255[gray[(size_t)rr * w + cc]];
          const float bw = bilateral_weight(st, dr, dc, center, color);
          const float wc = bw * color;
          cs += wc;
          cq = fmaf(wc, color, cq);
          ws += bw;
        }
      }
      st->ref_sum[(size_t)row * w + col] = cs / ws;
      st->ref_sqsum[(size_t)row * w + col] = cq / ws;
      out[(size_t)row * w + col] = (uint8_t)(255.0f * center);
    }
  }
  st->ref_img = out;
}

/* ------------------------------------------------------------------------- */
/* geometry helpers                                                           */
/* ------------------------------------------------------------------------- */
/* ComposeHomography: patch_match_cuda.cu:271-332 */
static inline void compose_homography(const pm_state* st, const float* pose, int row, int col, float depth,
                                      const float normal[3], float H[9]) {
  const float* iK = st->refinvK[st->rot];
  const float* K = pose;
  const float* R = pose + 4;
  const float* T = pose + 13;
  const float rx = fmaf(iK[0], (float)col, iK[1]);
  const float ry = fmaf(iK[2], (float)row, iK[3]);
  const float dist = depth * fmaf(normal[0], rx, fmaf(normal[1], ry, normal[2]));
  const float inv_dist = 1.0f / dist;
  const float a0 = inv_dist * normal[0], a1 = inv_dist * normal[1], a2 = inv_dist * normal[2];
  const float m00 = fmaf(a0, T[0], R[0]), m01 = fmaf(a1, T[0], R[1]), m02 = fmaf(a2, T[0], R[2]);
  const float m10 = fmaf(a0, T[1], R[3]), m11 = fmaf(a1, T[1], R[4]), m12 = fmaf(a2, T[1], R[5]);
  const float m20 = fmaf(a0, T[2], R[6]), m21 = fmaf(a1, T[2], R[7]), m22 = fmaf(a2, T[2], R[8]);
  const float g00 = fmaf(K[0], m00, K[1] * m20), g01 = fmaf(K[0], m01, K[1] * m21), g02 = fmaf(K[0], m02, K[1] * m22);
  const float g10 = fmaf(K[2], m10, K[3] * m20), g11 = fmaf(K[2], m11, K[3] * m21), g12 = fmaf(K[2], m12, K[3] * m22);
  H[0] = iK[0] * g00; H[1] = iK[2] * g01; H[2] = fmaf(iK[3], g01, fmaf(iK[1], g00, g02));
  H[3] = iK[0] * g10; H[4] = iK[2] * g11; H[5] = fmaf(iK[3], g11, fmaf(iK[1], g10, g12));
  H[6] = iK[0] * m20; H[7] = iK[2] * m21; H[8] = fmaf(iK[3], m21, fmaf(iK[1], m20, m22));
}

/* bilinear sample of source image i at pixel-index position (px,py); texel centre = integer;
 * border -> 0 (InitSourceImages :1625-1653, tex2DLayered at +0.5 :527-535) */
static inline float sample_src(const pm_state* st, int i, float px, float py) {
  const int W = st->src_w[i], H = st->src_h[i];
  const uint8_t* img = st->src_img[i];
  float pxc = (px > -2.0f) ? px : -2.0f;
  pxc = (pxc < (float)(W + 1)) ? pxc : (float)(W + 1);
  float pyc = (py > -2.0f) ? py : -2.0f;
  pyc = (pyc < (float)(H + 1)) ? pyc : (float)(H + 1);
  const float fx = floorf(pxc), fy = floorf(pyc);
  const int ix = (int)fx, iy = (int)fy;
  const float wx = pxc - fx, wy = pyc - fy;
#define TEXEL(X, Y) (((X) < 0 || (Y) < 0 || (X) >= W || (Y) >= H) ? 0.0f : (float)img[(size_t)(Y) * W + (X)])
  const float a = TEXEL(ix, iy), b = TEXEL(ix + 1, iy), c = TEXEL(ix, iy + 1), d = TEXEL(ix + 1, iy + 1);
#undef TEXEL
  const float top = fmaf(wx, b - a, a);
  const float bot = fmaf(wx, d - c, c);
  const float v = fmaf(wy, bot - top, top);
  return v * 0.00392156886f; /* 1/255 */
}

static inline float tree8(const float p[8]) {
  return ((p[0] + p[1]) + (p[2] + p[3])) + ((p[4] + p[5]) + (p[6] + p[7]));
}

/* per-pixel reference patch: colours, bilateral weights, weight sum (hypothesis independent part of
 * PhotoConsistencyCostComputer::Compute, :510-546) */
typedef struct {
  float w[1681];   /* up to radius 20 */
  float wref[1681];
  float wsum;
} pm_patch;

static void build_patch(const pm_state* st, int row, int col, pm_patch* pt) {
  const int r = st->radius, s = st->step, ns = st->nside;
  const float center = ref_color(st, row, col);
  float part[32];
  for (int i = 0; i < 32; ++i) part[i] = 0.0f;
  for (int t = 0; t < st->ntaps; ++t) {
    const int dr = -r + s * (t / ns), dc = -r + s * (t % ns);
    const float c = ref_color(st, row + dr, col + dc);
    const float bw = bilateral_weight(st, dr, dc, center, c);
    pt->w[t] = bw;
    pt->wref[t] = bw * c;
    part[t & 31] += bw;
  }
  /* 32 interleaved partial sums joined by a butterfly tree */
  for (int stride = 1; stride < 32; stride <<= 1)
    for (int i = 0; i < 32; i += 2 * stride) part[i] = part[i] + part[i + stride];
  pt->wsum = part[0];
}

/* PhotoConsistencyCostComputer::Compute: patch_match_cuda.cu:489-593 */
static float ncc_cost(const pm_state* st, const pm_patch* pt, int row, int col, int image_idx, float depth,
                      const float normal[3], float ref_sum, float ref_sqsum) {
  float H[9];
  compose_homography(st, st->poses[st->rot] + PM_POSE_STRIDE * image_idx, row, col, depth, normal, H);
  const int r = st->radius, s = st->step, ns = st->nside;
  float s1[8] = {0}, s2[8] = {0}, s3[8] = {0};
  /* H (col + dx, row + dy, 1): the pixel part is folded into the constant term once per evaluation */
  const float cx = fmaf(H[0], (float)col, fmaf(H[1], (float)row, H[2]));
  const float cy = fmaf(H[3], (float)col, fmaf(H[4], (float)row, H[5]));
  const float cz = fmaf(H[6], (float)col, fmaf(H[7], (float)row, H[8]));
  for (int t = 0; t < st->ntaps; ++t) {
    const float dx = (float)(-r + s * (t % ns));
    const float dy = (float)(-r + s * (t / ns));
    const float zx = fmaf(H[0], dx, fmaf(H[1], dy, cx));
    const float zy = fmaf(H[3], dx, fmaf(H[4], dy, cy));
    const float zz = fmaf(H[6], dx, fmaf(H[7], dy, cz));
    /* |z| is clamped to [1e-30, 1e30] with its sign kept (keeps the reciprocal in the range where the GPU's
     * MUFU.RCP + one Newton step is correctly rounded).  A point behind the source camera samples its mirror
     * image through the camera centre, as the reference's 1 / z does (:526-535); z < 0 decides the sign, so
     * -0 and NaN give +1e-30, which samples the zero border (pm_device.cuh:pm_clamp_z states the same rule). */
    float za = (zz < 0.0f) ? -zz : zz;
    za = (za > 1e-30f) ? za : 1e-30f;
    za = (za < 1e30f) ? za : 1e30f;
    const float inv_z = 1.0f / ((zz < 0.0f) ? -za : za);
    const float color = sample_src(st, image_idx, inv_z * zx, inv_z * zy);
    const float ws = pt->w[t] * color;
    const int q = t & 7;
    s1[q] += ws;
    s2[q] = fmaf(ws, color, s2[q]);
    s3[q] = fmaf(pt->wref[t], color, s3[q]);
  }
  const float inv_wsum = 1.0f / pt->wsum;
  const float src_sum = tree8(s1) * inv_wsum;
  const float src_sqsum = tree8(s2) * inv_wsum;
  const float src_ref_sum = tree8(s3) * inv_wsum;
  const float ref_var = fmaf(-ref_sum, ref_sum, ref_sqsum);
  const float src_var = fmaf(-src_sum, src_sum, src_sqsum);
  const float kMinVar = 1e-5f;
  if (ref_var < kMinVar || src_var < kMinVar) return 2.0f;
  const float covar = fmaf(-ref_sum, src_sum, src_ref_sum);
  const float denom = sqrtf(ref_var * src_var);
  float c = 1.0f - covar / denom;
  c = (c < 2.0f) ? c : 2.0f;
  c = (c > 0.0f) ? c : 0.0f;
  return c;
}

/* ComputeGeomConsistencyCost: patch_match_cuda.cu:601-667 */
static float geom_cost(const pm_state* st, int row, int col, float depth, int image_idx, float max_cost) {
  const float* pose = st->poses[st->rot] + PM_POSE_STRIDE * image_idx;
  const float* P = pose + 19;
  const float* iP = pose + 31;
  const float* iK = st->refinvK[st->rot];
  const float* K = st->refK[st->rot];
  const float X = depth * fmaf(iK[0], (float)col, iK[1]);
  const float Y = depth * fmaf(iK[2], (float)row, iK[3]);
  const float Z = depth;
  const float fz = fmaf(P[8], X, fmaf(P[9], Y, fmaf(P[10], Z, P[11])));
  const float inv_fz = 1.0f / fz;
  float src_col = inv_fz * fmaf(P[0], X, fmaf(P[1], Y, fmaf(P[2], Z, P[3])));
  float src_row = inv_fz * fmaf(P[4], X, fmaf(P[5], Y, fmaf(P[6], Z, P[7])));
  /* point-sampled depth texel at (src_col + 0.5, src_row + 0.5), border -> 0 */
  float src_depth = 0.0f;
  {
    const int W = st->src_w[image_idx], Hh = st->src_h[image_idx];
    const float cx = src_col + 0.5f, cy = src_row + 0.5f;
    if (cx >= 0.0f && cy >= 0.0f && cx < (float)W && cy < (float)Hh) {
      const int ix = (int)floorf(cx), iy = (int)floorf(cy);
      src_depth = st->src_depth[image_idx][(size_t)iy * W + ix];
    }
  }
  if (src_depth == 0.0f) return max_cost;
  src_col = src_col * src_depth;
  src_row = src_row * src_depth;
  const float bx = fmaf(iP[0], src_col, fmaf(iP[1], src_row, fmaf(iP[2], src_depth, iP[3])));
  const float by = fmaf(iP[4], src_col, fmaf(iP[5], src_row, fmaf(iP[6], src_depth, iP[7])));
  const float bz = fmaf(iP[8], src_col, fmaf(iP[9], src_row, fmaf(iP[10], src_depth, iP[11])));
  const float inv_bz = 1.0f / bz;
  const float bcol = inv_bz * fmaf(K[0], bx, K[1] * bz);
  const float brow = inv_bz * fmaf(K[2], by, K[3] * bz);
  const float dc = (float)col - bcol, dr = (float)row - brow;
  const float e = sqrtf(fmaf(dc, dc, dr * dr));
  return (e < max_cost) ? e : max_cost;
}

/* PropagateDepth: patch_match_cuda.cu:210-236 */
static inline float propagate_depth(const pm_state* st, float depth1, const float normal1[3], float row1, float row2) {
  const float* iK = st->refinvK[st->rot];
  const float x1 = depth1 * fmaf(iK[2], row1, iK[3]);
  const float y1 = depth1;
  const float x2 = x1 + normal1[2];
  const float y2 = y1 - normal1[1];
  const float x4 = fmaf(iK[2], row2, iK[3]);
  const float denom = fmaf(x4, y1 - y2, x2 - x1);
  if (fabsf(denom) < 1e-5f) return depth1;
  const float nom = fmaf(y1, x2, -(x1 * y2));
  return nom / denom;
}

/* GenerateRandomNormal: patch_match_cuda.cu:94-123 */
static void random_normal(const pm_state* st, int row, int col, pm_rng* rs, float n[3]) {
  float v1 = 0.0f, v2 = 0.0f, s = 2.0f;
  while (s >= 1.0f) {
    v1 = fmaf(2.0f, rng_uniform(rs), -1.0f);
    v2 = fmaf(2.0f, rng_uniform(rs), -1.0f);
    s = fmaf(v1, v1, v2 * v2);
  }
  const float s_norm = sqrtf(1.0f - s);
  n[0] = 2.0f * v1 * s_norm;
  n[1] = 2.0f * v2 * s_norm;
  n[2] = fmaf(-2.0f, s, 1.0f);
  const float* iK = st->refinvK[st->rot];
  const float ray[3] = {fmaf(iK[0], (float)col, iK[1]), fmaf(iK[2], (float)row, iK[3]), 1.0f};
  if (dot3(n, ray) > 0.0f) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }
}

/* PerturbNormal: patch_match_cuda.cu:133-196 (recursion unrolled into a loop) */
static void perturb_normal(const pm_state* st, int row, int col, float perturbation, const float normal[3],
                           pm_rng* rs, float out[3]) {
  const float* iK = st->refinvK[st->rot];
  const float ray[3] = {fmaf(iK[0], (float)col, iK[1]), fmaf(iK[2], (float)row, iK[3]), 1.0f};
  for (int trial = 0;; ++trial) {
    const float a1 = (rng_uniform(rs) - 0.5f) * perturbation;
    const float a2 = (rng_uniform(rs) - 0.5f) * perturbation;
    const float a3 = (rng_uniform(rs) - 0.5f) * perturbation;
    float s1, c1, s2, c2, s3, c3;
    pm_sincosf(a1, &s1, &c1);
    pm_sincosf(a2, &s2, &c2);
    pm_sincosf(a3, &s3, &c3);
    float R[9];
    R[0] = c2 * c3;
    R[1] = -(c2 * s3);
    R[2] = s2;
    R[3] = fmaf(c1, s3, c3 * s1 * s2);
    R[4] = fmaf(c1, c3, -(s1 * s2 * s3));
    R[5] = -(c2 * s1);
    R[6] = fmaf(s1, s3, -(c1 * c3 * s2));
    R[7] = fmaf(c3, s1, c1 * s2 * s3);
    R[8] = c1 * c2;
    out[0] = dot3(R, normal);
    out[1] = dot3(R + 3, normal);
    out[2] = dot3(R + 6, normal);
    if (dot3(out, ray) >= 0.0f) {
      if (trial < 3) { perturbation = 0.5f * perturbation; continue; }
      out[0] = normal[0]; out[1] = normal[1]; out[2] = normal[2];
      return;
    }
    const float inv_norm = 1.0f / sqrtf(dot3(out, out));
    out[0] *= inv_norm; out[1] *= inv_norm; out[2] *= inv_norm;
    return;
  }
}

/* ComputeViewingAngles: patch_match_cuda.cu:241-269 */
static inline void viewing_angles(const float* pose, const float point[3], const float normal[3], float* cos_tri,
                                  float* cos_inc) {
  const float* C = pose + 16;
  const float SX[3] = {C[0] - point[0], C[1] - point[1], C[2] - point[2]};
  const float RX_inv = 1.0f / sqrtf(dot3(point, point));
  const float SX_inv = 1.0f / sqrtf(dot3(SX, SX));
  *cos_inc = dot3(SX, normal) * SX_inv;
  *cos_tri = (-dot3(SX, point)) * RX_inv * SX_inv;
}

/* LikelihoodComputer: patch_match_cuda.cu:698-832 */
static inline float ncc_prob(const pm_state* st, float cost) { return pm_expf(cost * cost * st->inv_ncc_sigma_sq) * st->ncc_norm; }
#define K_NOCHANGE 0.99999f
#define K_CHANGE (1.0f - 0.99999f)
static inline float forward_message(const pm_state* st, float cost, float prev) {
  const float e = ncc_prob(st, cost);
  const float om = 1.0f - prev;
  const float zn0 = fmaf(prev, K_CHANGE, om * K_NOCHANGE) * 0.5f;
  const float zn1 = fmaf(prev, K_NOCHANGE, om * K_CHANGE) * e;
  return zn1 / (zn0 + zn1);
}
static inline float backward_message(const pm_state* st, float cost, float prev) {
  const float e = ncc_prob(st, cost);
  const float pe = prev * e;
  const float om = (1.0f - prev) * 0.5f;
  const float zn0 = fmaf(pe, K_CHANGE, om * K_NOCHANGE);
  const float zn1 = fmaf(pe, K_NOCHANGE, om * K_CHANGE);
  return zn1 / (zn0 + zn1);
}
static inline float sel_prob_of(float alpha, float beta, float prev, float prev_weight) {
  const float zn0 = (1.0f - alpha) * (1.0f - beta);
  const float zn1 = alpha * beta;
  const float curr = zn1 / (zn0 + zn1);
  return fmaf(prev_weight, prev, (1.0f - prev_weight) * curr);
}
static inline float tri_prob(const pm_state* st, float cos_tri) {
  if (cos_tri > st->cos_min_tri) {
    const float scaled = 1.0f - (1.0f - cos_tri) / (1.0f - st->cos_min_tri);
    float l = fmaf(-scaled, scaled, 1.0f);
    l = (l > 0.0f) ? l : 0.0f;
    l = (l < 1.0f) ? l : 1.0f;
    return l;
  }
  return 1.0f;
}
static inline float inc_prob(const pm_state* st, float cos_inc) {
  const float x = 1.0f - ((cos_inc > 0.0f) ? cos_inc : 0.0f);
  return pm_expf(x * x * st->inv_inc_sigma_sq);
}
static inline void warp_pt(const float H[9], float x, float y, float out[2]) {
  const float inv_z = 1.0f / fmaf(H[6], x, fmaf(H[7], y, H[8]));
  out[0] = inv_z * fmaf(H[0], x, fmaf(H[1], y, H[2]));
  out[1] = inv_z * fmaf(H[3], x, fmaf(H[4], y, H[5]));
}
/* ComputeResolutionProb: :759-791 */
static inline float res_prob(const pm_state* st, const float H[9], float row, float col) {
  const float r = (float)st->radius;
  float s1[2], s2[2], s3[2], s4[2];
  warp_pt(H, col - r, row - r, s1);
  warp_pt(H, col - r, row + r, s2);
  warp_pt(H, col + r, row + r, s3);
  warp_pt(H, col + r, row - r, s4);
  const float ws = (float)(2 * st->radius + 1);
  const float ref_area = ws * ws;
  float acc = s1[0] * s2[1];
  acc = fmaf(-s2[0], s1[1], acc);
  acc = fmaf(-s1[0], s4[1], acc);
  acc = fmaf(s2[0], s3[1], acc);
  acc = fmaf(-s3[0], s2[1], acc);
  acc = fmaf(s4[0], s1[1], acc);
  acc = fmaf(s3[0], s4[1], acc);
  acc = fmaf(-s4[0], s3[1], acc);
  const float src_area = fabsf(0.5f * acc);
  if (ref_area > src_area) return src_area / ref_area;
  return ref_area / src_area;
}

/* ------------------------------------------------------------------------- */
/* ComputeInitialCost: patch_match_cuda.cu:863-912                            */
/* ------------------------------------------------------------------------- */
static void compute_initial_cost(pm_state* st) {
  const int w = st->w, h = st->h;
  const size_t n = (size_t)w * h;
#pragma omp parallel for schedule(dynamic, 1)
  for (int col = 0; col < w; ++col) {
    pm_patch* pt = (pm_patch*)malloc(sizeof(pm_patch));
    for (int row = 0; row < h; ++row) {
      build_patch(st, row, col, pt);
      const size_t p = (size_t)row * w + col;
      const float nrm[3] = {st->normal[p], st->normal[n + p], st->normal[2 * n + p]};
      for (int i = 0; i < st->N; ++i)
        st->cost[i * n + p] = ncc_cost(st, pt, row, col, i, st->depth[p], nrm, st->ref_sum[p], st->ref_sqsum[p]);
    }
    free(pt);
  }
}

/* ------------------------------------------------------------------------- */
/* SweepFromTopToBottom: patch_match_cuda.cu:933-1288 (one column)            */
/* ------------------------------------------------------------------------- */
static void sweep_column(pm_state* st, int col, float perturbation, float perturbation_pi, float prev_w,
                         int last_filter) {
  const int w = st->w, h = st->h, N = st->N;
  const size_t n = (size_t)w * h;
  float fwd[PM_MAX_SRC], probs[PM_MAX_SRC];
  pm_patch* pt = (pm_patch*)malloc(sizeof(pm_patch));

  /* backward messages (:976-989) */
  for (int i = 0; i < N; ++i) {
    float beta = 0.5f;
    for (int row = h - 1; row >= 0; --row) {
      const size_t p = (size_t)row * w + col;
      beta = backward_message(st, st->cost[i * n + p], beta);
      st->sel_prob[i * n + p] = beta;
    }
    fwd[i] = 0.5f;
  }

  pm_rng rs = st->rand_state[col]; /* row 0 */
  float prev_depth = st->depth[col];
  float prev_normal[3] = {st->normal[col], st->normal[n + col], st->normal[2 * n + col]};
  const float min_ncc_prob = ncc_prob(st, 1.0f - st->filter_min_ncc);
  const float cos_filter_tri = cosf(st->filter_min_tri_rad);
  const float* iK = st->refinvK[st->rot];

  for (int row = 0; row < h; ++row) {
    const size_t p = (size_t)row * w + col;
    build_patch(st, row, col, pt);
    const float rsum = st->ref_sum[p], rsq = st->ref_sqsum[p];

    prev_depth = propagate_depth(st, prev_depth, prev_normal, (float)(row - 1), (float)row);
    const float cur_depth = st->depth[p];
    const float cur_normal[3] = {st->normal[p], st->normal[n + p], st->normal[2 * n + p]};

    /* PerturbDepth (:125-131) */
    float rand_depth, rand_normal[3];
    {
      const float dmin = (1.0f - perturbation) * cur_depth;
      const float dmax = (1.0f + perturbation) * cur_depth;
      rand_depth = fmaf(rng_uniform(&rs), dmax - dmin, dmin);
    }
    perturb_normal(st, row, col, perturbation_pi, cur_normal, &rs, rand_normal);

    const float rx = fmaf(iK[0], (float)col, iK[1]);
    const float ry = fmaf(iK[2], (float)row, iK[3]);
    const float point[3] = {cur_depth * rx, cur_depth * ry, cur_depth};

    /* per-image sampling probabilities (:1070-1104) */
    for (int i = 0; i < N; ++i) {
      const float* pose = st->poses[st->rot] + PM_POSE_STRIDE * i;
      const float alpha = forward_message(st, st->cost[i * n + p], fwd[i]);
      const float beta = st->sel_prob[i * n + p];
      const float sp = sel_prob_of(alpha, beta, st->prev_sel_prob[i * n + p], prev_w);
      float ct, ci;
      viewing_angles(pose, point, cur_normal, &ct, &ci);
      float H[9];
      compose_homography(st, pose, row, col, cur_depth, cur_normal, H);
      probs[i] = sp * tri_prob(st, ct) * inc_prob(st, ci) * res_prob(st, H, (float)row, (float)col);
    }
    /* TransformPDFToCDF (:683-696) */
    {
      float sum = 0.0f;
      for (int i = 0; i < N; ++i) sum += probs[i];
      const float inv = 1.0f / sum;
      float cum = 0.0f;
      for (int i = 0; i < N; ++i) { cum += probs[i] * inv; probs[i] = cum; }
    }

    /* Monte Carlo sampling (:1115-1173); NCC is a pure function of (hypothesis, image), memoised */
    const float depths[5] = {cur_depth, prev_depth, rand_depth, cur_depth, rand_depth};
    const float* normals[5] = {cur_normal, prev_normal, rand_normal, rand_normal, cur_normal};
    float costs[5] = {0, 0, 0, 0, 0};
    float memo[5][PM_MAX_SRC], gmemo[5][PM_MAX_SRC];
    uint8_t have[5][PM_MAX_SRC];
    memset(have, 0, sizeof(have));
    for (int s = 0; s < st->num_samples; ++s) {
      const float u = rng_uniform(&rs) - FLT_EPSILON;
      int img = -1;
      for (int i = 0; i < N; ++i) if (probs[i] > u) { img = i; break; }
      if (img < 0) continue;
      for (int k = 0; k < 5; ++k) {
        if (!have[k][img]) {
          memo[k][img] = (k == 0) ? st->cost[img * n + p]
                                  : ncc_cost(st, pt, row, col, img, depths[k], normals[k], rsum, rsq);
          if (st->geom) gmemo[k][img] = geom_cost(st, row, col, depths[k], img, st->geom_max_cost);
          have[k][img] = 1;
        }
        costs[k] += memo[k][img];
        if (st->geom) costs[k] = fmaf(st->geom_reg, gmemo[k][img], costs[k]);
      }
    }
    /* FindMinCost (:670-681): ties -> last */
    int best = 0;
    {
      float m = costs[0];
      for (int k = 1; k < 5; ++k) if (costs[k] <= m) { m = costs[k]; best = k; }
    }
    const float best_depth = depths[best];
    const float best_normal[3] = {normals[best][0], normals[best][1], normals[best][2]};
    st->depth[p] = best_depth;
    st->normal[p] = best_normal[0]; st->normal[n + p] = best_normal[1]; st->normal[2 * n + p] = best_normal[2];

    /* forward messages and selection probabilities with the new cost (:1184-1207) */
    for (int i = 0; i < N; ++i) {
      float c;
      if (best == 0) {
        c = st->cost[i * n + p];
      } else {
        c = have[best][i] ? memo[best][i] : ncc_cost(st, pt, row, col, i, best_depth, best_normal, rsum, rsq);
        st->cost[i * n + p] = c;
      }
      const float alpha = forward_message(st, c, fwd[i]);
      const float beta = st->sel_prob[i * n + p];
      st->sel_prob[i * n + p] = sel_prob_of(alpha, beta, st->prev_sel_prob[i * n + p], prev_w);
      fwd[i] = alpha;
    }

    /* filtering on the last sweep (:1209-1276) */
    if (last_filter) {
      int num_consistent = 0;
      const float bp[3] = {best_depth * rx, best_depth * ry, best_depth};
      for (int i = 0; i < N; ++i) {
        const float* pose = st->poses[st->rot] + PM_POSE_STRIDE * i;
        float ct, ci;
        viewing_angles(pose, bp, best_normal, &ct, &ci);
        if (ct > cos_filter_tri || ci <= 0.0f) continue;
        int ok = st->sel_prob[i * n + p] >= min_ncc_prob;
        if (ok && st->geom)
          ok = geom_cost(st, row, col, best_depth, i, st->geom_max_cost) <= st->filter_geom_max_cost;
        if (ok) { st->mask[i * n + p] = 1; num_consistent += 1; }
      }
      if (num_consistent < st->filter_min_num_consistent) {
        st->depth[p] = 0.0f;
        st->normal[p] = 0.0f; st->normal[n + p] = 0.0f; st->normal[2 * n + p] = 0.0f;
        for (int i = 0; i < N; ++i) st->mask[i * n + p] = 0;
      }
    }

    prev_depth = best_depth;
    prev_normal[0] = best_normal[0]; prev_normal[1] = best_normal[1]; prev_normal[2] = best_normal[2];
  }
  st->rand_state[col] = rs;
  free(pt);
}

/* ------------------------------------------------------------------------- */
/* driver: PatchMatchCuda ctor + RunWithWindowSizeAndStep (:1290-1302,1393-1546) */
/* ------------------------------------------------------------------------- */
static float ncc_norm_factor(float ncc_sigma) {
  /* ComputeNCCCostNormFactor (:796-802) */
  return 2.0f / (sqrtf(2.0f * (float)M_PI) * ncc_sigma * erff(2.0f / (ncc_sigma * 1.414213562f)));
}

/* stop_after_sweeps < 0: full run; otherwise stop after that many sweeps (the buffers are then rotated
 * back to the original orientation for output so partial runs can be compared too). */
int pm_oracle_run_partial(const b200pm_options* o, const b200pm_problem* p, int stop_after_sweeps, float* depth_out,
                          float* normal_out, float* sel_prob_out, uint8_t* mask_out, float* cost_out) {
  if (p->num_src < 1 || p->num_src > PM_MAX_SRC) return -1;
  if (o->window_radius < 1 || o->window_radius > 20 || o->window_step < 1 || o->window_step > 2) return -2;
  pm_state* st = (pm_state*)calloc(1, sizeof(pm_state));
  st->radius = o->window_radius; st->step = o->window_step;
  st->nside = (2 * st->radius) / st->step + 1;
  st->ntaps = st->nside * st->nside;
  st->num_samples = o->num_samples; st->num_iterations = o->num_iterations;
  st->geom = o->geom_consistency; st->filter = o->filter; st->filter_min_num_consistent = o->filter_min_num_consistent;
  st->depth_min = (float)o->depth_min; st->depth_max = (float)o->depth_max;
  st->sigma_spatial = (float)(o->sigma_spatial <= 0 ? (double)o->window_radius : o->sigma_spatial);
  st->sigma_color = (float)o->sigma_color; st->ncc_sigma = (float)o->ncc_sigma;
  st->min_tri_angle_rad = (float)(o->min_triangulation_angle * 0.0174532925199432);
  st->incident_angle_sigma = (float)o->incident_angle_sigma;
  st->geom_reg = (float)o->geom_consistency_regularizer; st->geom_max_cost = (float)o->geom_consistency_max_cost;
  st->filter_min_ncc = (float)o->filter_min_ncc;
  st->filter_min_tri_rad = (float)(o->filter_min_triangulation_angle * 0.0174532925199432);
  st->filter_geom_max_cost = (float)o->filter_geom_consistency_max_cost;
  st->spatial_norm = 1.0f / (2.0f * st->sigma_spatial * st->sigma_spatial);
  st->color_norm = 1.0f / (2.0f * st->sigma_color * st->sigma_color);
  st->cos_min_tri = cosf(st->min_tri_angle_rad);
  st->inv_inc_sigma_sq = -0.5f / (st->incident_angle_sigma * st->incident_angle_sigma);
  st->inv_ncc_sigma_sq = -0.5f / (st->ncc_sigma * st->ncc_sigma);
  st->ncc_norm = ncc_norm_factor(st->ncc_sigma);
  for (int v = 0; v < 256; ++v) st->lut255[v] = (float)v / 255.0f;

  st->W0 = st->w = p->ref_width; st->H0 = st->h = p->ref_height; st->rot = 0; st->N = p->num_src;
  const int w = st->w, h = st->h, N = st->N;
  const size_t n = (size_t)w * h;
  for (int i = 0; i < N; ++i) {
    st->src_w[i] = p->src_width[i]; st->src_h[i] = p->src_height[i]; st->src_img[i] = p->src_gray[i];
    st->src_depth[i] = (st->geom && p->src_depth) ? p->src_depth[i] : NULL;
  }
  if (st->geom && (!p->src_depth || !p->ref_depth_init || !p->ref_normal_init)) { free(st); return -3; }

  st->ref_sum = (float*)malloc(sizeof(float) * n);
  st->ref_sqsum = (float*)malloc(sizeof(float) * n);
  filter_ref_image(st, p->ref_gray);  /* InitRefImage */
  init_transforms(st, p);             /* InitTransforms */

  /* InitWorkspaceMemory (:1810-1857) */
  st->rand_state = (pm_rng*)malloc(sizeof(pm_rng) * n);
  st->depth = (float*)malloc(sizeof(float) * n);
  st->normal = (float*)malloc(sizeof(float) * 3 * n);
  st->cost = (float*)malloc(sizeof(float) * N * n);
  st->sel_prob = (float*)malloc(sizeof(float) * N * n);
  st->prev_sel_prob = (float*)malloc(sizeof(float) * N * n);
  for (size_t i = 0; i < N * n; ++i) st->prev_sel_prob[i] = 0.5f;
  {
    /* InitRandomStateKernel (gpu_mat_prng.cu:36-48), 32x16 blocks (gpu_mat.h:159-160) */
    const int gx = (w - 1) / 32 + 1;
    for (int row = 0; row < h; ++row)
      for (int col = 0; col < w; ++col) {
        const uint64_t id = (uint64_t)((row / 16) * gx + (col / 32)) * 512u + (uint64_t)((row % 16) * 32 + (col % 32));
        rng_init(&st->rand_state[(size_t)row * w + col], id);
      }
  }
  if (st->geom) {
    memcpy(st->depth, p->ref_depth_init, sizeof(float) * n);
    memcpy(st->normal, p->ref_normal_init, sizeof(float) * 3 * n);
  } else {
    /* FillWithRandomNumbersKernel (gpu_mat.h:371-387) then InitNormalMap (:835-846) */
    for (int row = 0; row < h; ++row)
      for (int col = 0; col < w; ++col) {
        const size_t q = (size_t)row * w + col;
        pm_rng* rs = &st->rand_state[q];
        st->depth[q] = fmaf(rng_uniform(rs), st->depth_max - st->depth_min, st->depth_min);
      }
    for (int row = 0; row < h; ++row)
      for (int col = 0; col < w; ++col) {
        const size_t q = (size_t)row * w + col;
        float nv[3];
        random_normal(st, row, col, &st->rand_state[q], nv);
        st->normal[q] = nv[0]; st->normal[n + q] = nv[1]; st->normal[2 * n + q] = nv[2];
      }
  }

  compute_initial_cost(st);
  if (cost_out && stop_after_sweeps == 0) memcpy(cost_out, st->cost, sizeof(float) * N * n);

  const float total_steps = (float)(st->num_iterations * 4);
  int done = 0;
  for (int iter = 0; iter < st->num_iterations && (stop_after_sweeps < 0 || done < stop_after_sweeps); ++iter) {
    for (int sweep = 0; sweep < 4 && (stop_after_sweeps < 0 || done < stop_after_sweeps); ++sweep, ++done) {
      const float perturbation = 1.0f / powf(2.0f, (float)iter + (float)sweep / 4.0f);
      /* options.perturbation * M_PI is evaluated in double (:1059) */
      const float perturbation_pi = (float)((double)perturbation * M_PI);
      const float prev_w = (float)(iter * 4 + sweep) / total_steps;
      const int last = (iter == st->num_iterations - 1 && sweep == 3);
      const int last_filter = last && st->filter;
      if (last_filter) st->mask = (uint8_t*)calloc((size_t)N * n, 1);
      const int cw = st->w;
#pragma omp parallel for schedule(dynamic, 1)
      for (int col = 0; col < cw; ++col) sweep_column(st, col, perturbation, perturbation_pi, prev_w, last_filter);
      {
        const int mw = st->w, mh = st->h;
        rotate_all(st, 1);
        if (last_filter) st->mask = rotate_u8(st->mask, mw, mh, N);
      }
    }
  }
  /* bring partial runs back to the original orientation */
  while (st->rot != 0) rotate_all(st, 0);

  if (depth_out) memcpy(depth_out, st->depth, sizeof(float) * n);
  if (normal_out) memcpy(normal_out, st->normal, sizeof(float) * 3 * n);
  if (sel_prob_out) memcpy(sel_prob_out, st->prev_sel_prob, sizeof(float) * N * n);
  if (cost_out && stop_after_sweeps != 0) memcpy(cost_out, st->cost, sizeof(float) * N * n);
  if (mask_out) {
    if (st->mask) memcpy(mask_out, st->mask, (size_t)N * n);
    else memset(mask_out, 0, (size_t)N * n);
  }
  for (int k = 0; k < 4; ++k) free(st->poses[k]);
  free(st->rand_state); free(st->depth); free(st->normal); free(st->cost); free(st->sel_prob);
  free(st->prev_sel_prob); free(st->ref_img); free(st->ref_sum); free(st->ref_sqsum); free(st->mask);
  free(st);
  return 0;
}

int pm_oracle_run(const b200pm_options* o, const b200pm_problem* p, float* depth_out, float* normal_out,
                  float* sel_prob_out, uint8_t* mask_out) {
  return pm_oracle_run_partial(o, p, -1, depth_out, normal_out, sel_prob_out, mask_out, NULL);
}

/* ------------------------------------------------------------------------- */
/* test hooks (bit-level comparison of the building blocks with the product)  */
/* ------------------------------------------------------------------------- */
float pm_oracle_expf(float x) { return pm_expf(x); }
void pm_oracle_sincosf(float a, float* s, float* c) { pm_sincosf(a, s, c); }
void pm_oracle_rng_stream(uint64_t seed, int count, float* out) {
  pm_rng r; rng_init(&r, seed);
  for (int i = 0; i < count; ++i) out[i] = rng_uniform(&r);
}
/* poses for rotation k, [N*43] floats, plus rotated K / K^-1 */
int pm_oracle_poses(const b200pm_problem* p, int k, float* poses_out, float* K_out, float* invK_out) {
  pm_state st; memset(&st, 0, sizeof(st));
  st.W0 = p->ref_width; st.H0 = p->ref_height; st.N = p->num_src;
  init_transforms(&st, p);
  memcpy(poses_out, st.poses[k], sizeof(float) * PM_POSE_STRIDE * st.N);
  memcpy(K_out, st.refK[k], 16); memcpy(invK_out, st.refinvK[k], 16);
  for (int i = 0; i < 4; ++i) free(st.poses[i]);
  return 0;
}
/* image.cc known-answer hooks (image_test.cc:149-212) */
void pm_oracle_compose_projection_matrix(const float K[9], const float R[9], const float T[3], float P[12]) {
  const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, Z3[3] = {0, 0, 0};
  float row[PM_POSE_STRIDE];
  compose_pose_row(I3, Z3, K, R, T, row);
  memcpy(P, row + 19, 48);
}
void pm_oracle_compose_inverse_projection_matrix(const float K[9], const float R[9], const float T[3], float iP[12]) {
  const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, Z3[3] = {0, 0, 0};
  float row[PM_POSE_STRIDE];
  compose_pose_row(I3, Z3, K, R, T, row);
  memcpy(iP, row + 31, 48);
}
/* RotatePose (mvs/image.cc:144-150): R <- RR R, T <- RR T, fp32 */
void pm_oracle_rotate_pose(const float RR[9], float R[9], float T[3]) {
  float nR[9], nT[3];
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) nR[3 * r + c] = RR[3 * r] * R[c] + RR[3 * r + 1] * R[3 + c] + RR[3 * r + 2] * R[6 + c];
    nT[r] = RR[3 * r] * T[0] + RR[3 * r + 1] * T[1] + RR[3 * r + 2] * T[2];
  }
  memcpy(R, nR, sizeof(nR)); memcpy(T, nT, sizeof(nT));
}
void pm_oracle_projection_center(const float R[9], const float T[3], float C[3]) {
  const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, Z3[3] = {0, 0, 0};
  const float K[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  float row[PM_POSE_STRIDE];
  compose_pose_row(I3, Z3, K, R, T, row);
  memcpy(C, row + 16, 12);
}
