/* sm_oracle.c — CPU restatement of brute-force SIFT matching (FindBestMatchesBruteForce, the reference's
 * SiftCPUFeatureMatcher with cpu_brute_force_matcher), written from the specification in DESIGN.md ("SIFT feature
 * matching"): the first max_num_matches rows of each image, exact dot products, a sequential top-2 scan per row in
 * fp32 with the C library's acosf, the distance and ratio tests, and the cross-check.  OpenMP over rows.  Test
 * infrastructure (tests/oracle_sm.py compiles it on demand). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

/* One way: for each row i of a (na rows), its match in b (nb rows), or -1. */
static void one_way(const uint8_t* a, int64_t na, const uint8_t* b, int64_t nb, float max_ratio, float max_distance,
                    int32_t* match) {
#pragma omp parallel for schedule(dynamic, 16)
  for (int64_t i = 0; i < na; ++i) {
    const uint8_t* x = a + i * 128;
    int32_t best_idx = -1;
    float best = 0.0f, second = 0.0f;
    for (int64_t j = 0; j < nb; ++j) {
      const uint8_t* y = b + j * 128;
      int32_t s = 0;
      for (int k = 0; k < 128; ++k) s += (int32_t)x[k] * (int32_t)y[k];
      const float dot = (float)s;
      if (dot > best) {
        best_idx = (int32_t)j;
        second = best;
        best = dot;
      } else if (dot > second) {
        second = dot;
      }
    }
    match[i] = -1;
    if (best_idx == -1) continue;
    const float inv_sq_norm = (float)(1.0 / (512.0 * 512.0));
    const float d1 = acosf(fminf(inv_sq_norm * best, 1.0f));
    if (d1 > max_distance) continue;
    const float d2 = acosf(fminf(inv_sq_norm * second, 1.0f));
    if (d1 >= max_ratio * d2) continue;
    match[i] = best_idx;
  }
}

/* Matches (n1 x 128) against (n2 x 128) uint8 descriptors.  out receives (idx1, idx2) pairs in ascending idx1 and
 * must hold min(n1, n2) pairs with cross_check, n1 without.  Returns the number of matches, or -1 on allocation
 * failure. */
int64_t sm_oracle_match(const uint8_t* d1, int64_t n1, const uint8_t* d2, int64_t n2, double max_ratio,
                        double max_distance, int cross_check, int64_t max_num_matches, uint32_t* out) {
  if (n1 > max_num_matches) n1 = max_num_matches;
  if (n2 > max_num_matches) n2 = max_num_matches;
  if (n1 <= 0 || n2 <= 0) return 0;
  const float r = (float)max_ratio, dmax = (float)max_distance;
  int32_t* m12 = (int32_t*)malloc(sizeof(int32_t) * (size_t)n1);
  int32_t* m21 = cross_check ? (int32_t*)malloc(sizeof(int32_t) * (size_t)n2) : NULL;
  if (!m12 || (cross_check && !m21)) {
    free(m12);
    free(m21);
    return -1;
  }
  one_way(d1, n1, d2, n2, r, dmax, m12);
  if (cross_check) one_way(d2, n2, d1, n1, r, dmax, m21);
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
