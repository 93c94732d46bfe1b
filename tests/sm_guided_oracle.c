/* sm_guided_oracle.c — CPU restatement of guided SIFT matching (the reference's SiftCPUFeatureMatcher::MatchGuided
 * with FindBestMatchesIndex), written from the specification in DESIGN.md ("Guided matching"): the first
 * max_num_matches rows of each image, exact integer L2 distances, 512^2 for a candidate the geometric filter rejects,
 * a sequential min top-2 per row in fp32, the distance and ratio tests, and the cross-check.  The F and H filters run
 * in fp32 and the E filter in fp64, in the pinned order (left-to-right sums; compiled with -ffp-contract=off).  Rays
 * and their Jacobians come in as inputs.  OpenMP over rows.  Test infrastructure (tests/oracle_smg.py compiles it on
 * demand). */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

enum { NONE = 0, ESSENTIAL = 1, FUNDAMENTAL = 2, HOMOGRAPHY = 3 };

typedef struct {
  int type;
  const float* xy1;     /* n1 x 2 */
  const float* xy2;     /* n2 x 2 */
  const double* geo1;   /* n1 x 10: ray (3), row-major 3 x 2 Jacobian (6), valid (1 or 0) */
  const double* geo2;
  double E[9];
  float M[9];           /* F or H, rounded to float */
  double thr_d;
  float thr_f;
} Filter;

static double grad_sq(const double* J, double g0, double g1, double g2) {
  const double gx = J[0] * g0 + J[2] * g1 + J[4] * g2, gy = J[1] * g0 + J[3] * g1 + J[5] * g2;
  return gx * gx + gy * gy;
}

/* Whether the filter rejects the candidate (i1, i2); a comparison with a NaN operand does not reject. */
static int reject(const Filter* f, int64_t i1, int64_t i2) {
  if (f->type == ESSENTIAL) {
    const double* g1 = f->geo1 + i1 * 10;
    const double* g2 = f->geo2 + i2 * 10;
    if (g1[9] == 0.0 || g2[9] == 0.0) return 1;
    const double* E = f->E;
    double e[3], t[3];
    for (int r = 0; r < 3; ++r) e[r] = E[3 * r] * g1[0] + E[3 * r + 1] * g1[1] + E[3 * r + 2] * g1[2];
    for (int c = 0; c < 3; ++c) t[c] = E[c] * g2[0] + E[3 + c] * g2[1] + E[6 + c] * g2[2];
    const double num = g2[0] * e[0] + g2[1] * e[1] + g2[2] * e[2];
    const double den = grad_sq(g1 + 3, t[0], t[1], t[2]) + grad_sq(g2 + 3, e[0], e[1], e[2]);
    const double err = den == 0 ? DBL_MAX : num * num / den;
    return err > f->thr_d;
  }
  const float x1 = f->xy1[2 * i1], y1 = f->xy1[2 * i1 + 1], x2 = f->xy2[2 * i2], y2 = f->xy2[2 * i2 + 1];
  const float* M = f->M;
  const float a0 = M[0] * x1 + M[1] * y1 + M[2], a1 = M[3] * x1 + M[4] * y1 + M[5], a2 = M[6] * x1 + M[7] * y1 + M[8];
  if (f->type == FUNDAMENTAL) {
    const float b0 = M[0] * x2 + M[3] * y2 + M[6], b1 = M[1] * x2 + M[4] * y2 + M[7];
    const float nom = x2 * a0 + y2 * a1 + a2;
    const float den = a0 * a0 + a1 * a1 + b0 * b0 + b1 * b1;
    return nom * nom > f->thr_f * den;
  }
  const float dx = a0 / a2 - x2, dy = a1 / a2 - y2;
  return dx * dx + dy * dy > f->thr_f;
}

/* One way: for each row i of a (na rows), its match in b (nb rows), or -1.  swap: a is image 2. */
static void one_way(const uint8_t* a, int64_t na, const uint8_t* b, int64_t nb, const Filter* f, int swap,
                    float max_ratio, float max_distance, int32_t* match) {
  const float max_l2 = 262144.0f * max_distance * max_distance;
#pragma omp parallel for schedule(dynamic, 16)
  for (int64_t i = 0; i < na; ++i) {
    const uint8_t* x = a + i * 128;
    int32_t best_idx = -1;
    float best = FLT_MAX, second = FLT_MAX;
    for (int64_t j = 0; j < nb; ++j) {
      float l2;
      if (reject(f, swap ? j : i, swap ? i : j)) {
        l2 = 262144.0f;
      } else {
        const uint8_t* y = b + j * 128;
        int32_t s = 0;
        for (int k = 0; k < 128; ++k) {
          const int32_t d = (int32_t)x[k] - (int32_t)y[k];
          s += d * d;
        }
        l2 = (float)s;
      }
      if (l2 < best) {
        best_idx = (int32_t)j;
        second = best;
        best = l2;
      } else if (l2 < second) {
        second = l2;
      }
    }
    match[i] = -1;
    if (best_idx == -1) continue;
    if (best > max_l2) continue;
    if (sqrtf(best) >= max_ratio * sqrtf(second)) continue;
    match[i] = best_idx;
  }
}

/* Guided matches of (n1 x 128) against (n2 x 128) uint8 descriptors under the filter `type` with matrix M (row-major,
 * image 1 to image 2).  out receives (idx1, idx2) pairs in ascending idx1 and must hold min(n1, n2) pairs with
 * cross_check, n1 without.  Returns the number of matches, or -1 on allocation failure. */
int64_t smg_oracle_match(const uint8_t* d1, int64_t n1, const uint8_t* d2, int64_t n2, const float* xy1,
                         const float* xy2, const double* geo1, const double* geo2, int type, const double* M,
                         double max_error, double max_ratio, double max_distance, int cross_check,
                         int64_t max_num_matches, uint32_t* out) {
  if (n1 > max_num_matches) n1 = max_num_matches;
  if (n2 > max_num_matches) n2 = max_num_matches;
  if (type == NONE || n1 <= 0 || n2 <= 0) return 0;
  Filter f;
  f.type = type; f.xy1 = xy1; f.xy2 = xy2; f.geo1 = geo1; f.geo2 = geo2;
  for (int k = 0; k < 9; ++k) { f.E[k] = M[k]; f.M[k] = (float)M[k]; }
  f.thr_d = max_error * max_error;
  f.thr_f = (float)f.thr_d;
  const float r = (float)max_ratio, dmax = (float)max_distance;
  int32_t* m12 = (int32_t*)malloc(sizeof(int32_t) * (size_t)n1);
  int32_t* m21 = cross_check ? (int32_t*)malloc(sizeof(int32_t) * (size_t)n2) : NULL;
  if (!m12 || (cross_check && !m21)) {
    free(m12);
    free(m21);
    return -1;
  }
  one_way(d1, n1, d2, n2, &f, 0, r, dmax, m12);
  if (cross_check) one_way(d2, n2, d1, n1, &f, 1, r, dmax, m21);
  int64_t k = 0;
  for (int64_t i = 0; i < n1; ++i) {
    const int32_t j = m12[i];
    if (j == -1) continue;
    if (cross_check && m21[j] != (int32_t)i) continue;
    out[2 * k] = (uint32_t)i;
    out[2 * k + 1] = (uint32_t)j;
    ++k;
  }
  free(m12);
  free(m21);
  return k;
}
