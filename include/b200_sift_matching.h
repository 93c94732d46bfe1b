/*
 * b200_sift_matching.h — C-ABI of SIFT feature matching (CUDA, sm_90a, H100): the brute-force descriptor matcher the
 * exhaustive, sequential and vocabulary-tree matchers run on every image pair (reference: src/colmap/feature/sift.cc,
 * FindBestMatchesBruteForce and SiftGPUFeatureMatcher::Match).  Exact integer dot products of uint8 descriptors on the
 * tensor cores, a two-way top-2 scan fused behind them, the ratio and distance tests, the cross-check and a per-pair
 * compaction, for a whole list of image pairs in one call.
 *
 * The decisions are those of the reference's CPU brute-force matcher, bit for bit: the arc-cosine of the normalised
 * dot product is the C library's acosf, tabulated once per handle on the host over the 2^18 + 1 values its argument
 * can take (see DESIGN.md, "SIFT feature matching").
 *
 * Conventions: 0 == success, negative == error with b200sm_last_error() set, no exceptions; every input is checked on
 * the host before any device work.  A handle is used by one host thread at a time.
 */
#ifndef B200_SIFT_MATCHING_H_
#define B200_SIFT_MATCHING_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { B200SM_OK = 0, B200SM_ERR_INPUT = -1, B200SM_ERR_TOO_LARGE = -2, B200SM_ERR_CUDA = -3 };

/* Bytes of one SIFT descriptor row. */
#define B200SM_DESCRIPTOR_DIM 128
/* Largest max_num_matches, i.e. the most descriptor rows of one image that take part in matching. */
#define B200SM_MAX_NUM_FEATURES (1 << 22)
/* Largest number of image slots of one handle. */
#define B200SM_MAX_NUM_SLOTS (1 << 20)
/* Largest sum over the pairs of one b200sm_match_pairs call of the rows of both images. */
#define B200SM_MAX_ROWS_PER_CALL ((int64_t)1 << 31)

/* SiftMatchingOptions (feature/sift.h:114-123) and FeatureMatchingOptions (feature/matcher.h:81), the fields the
 * matcher reads. */
typedef struct b200sm_options {
  double max_ratio;     /* 0.8; > 0: reject a match whose best distance >= max_ratio * second-best distance */
  double max_distance;  /* 0.7; > 0: reject a match whose best distance > max_distance */
  int cross_check;      /* 1: keep (i1, i2) only when i2's best match in image 1 is i1 */
  int max_num_matches;  /* 32768; only the first max_num_matches descriptor rows of an image take part */
  int gpu_index;        /* -1: current device */
} b200sm_options;
void b200sm_options_init(b200sm_options* o);

typedef struct b200sm_matcher* b200sm_handle;

/* A matcher with num_slots image slots (each starts empty) and the acos table, on the device of o->gpu_index.
 * Refuses max_ratio <= 0, max_distance <= 0, max_num_matches < 0 (SiftMatchingOptions::Check), num_slots < 1;
 * B200SM_ERR_TOO_LARGE for max_num_matches > B200SM_MAX_NUM_FEATURES or num_slots > B200SM_MAX_NUM_SLOTS. */
int b200sm_create(const b200sm_options* o, int num_slots, b200sm_handle* out);

/* Uploads an image's descriptors (n x 128 bytes, row-major) into `slot`, replacing what it held (and clearing its
 * keypoints and camera).  Only the first min(n, max_num_matches) rows are kept.  n == 0 (desc may be NULL) leaves the
 * slot empty: every pair it is in has no matches. */
int b200sm_set_descriptors(b200sm_handle h, int slot, int64_t n, const uint8_t* desc);

/* Upper bound on the matches of b200sm_match_pairs over these pairs: the sum of min(n1, n2) per pair with
 * cross_check, of n1 without.  Negative on an invalid argument. */
int64_t b200sm_match_capacity(b200sm_handle h, int num_pairs, const int* slot1, const int* slot2);

/* Matches every pair p of (slot1[p], slot2[p]).  Pair p's matches are the uint32 pairs
 * matches[2 * offsets[p] .. 2 * offsets[p + 1]), (point2D_idx1, point2D_idx2) in ascending point2D_idx1;
 * offsets[0] == 0.  `capacity` counts matches (pairs of uint32); a capacity below b200sm_match_capacity is refused
 * before any device work.  offsets and matches are host memory. */
int b200sm_match_pairs(b200sm_handle h, int num_pairs, const int* slot1, const int* slot2, uint64_t* offsets,
                       uint32_t* matches, size_t capacity);

/* Device time (CUDA events, ms) of the last b200sm_match_pairs or b200sm_match_guided_pairs: the product and top-2
 * scan, and the whole call's device work (scan, test, cross-check, compaction, copies).  Negative before the first
 * call. */
int b200sm_last_timing(b200sm_handle h, double* scan_ms, double* total_ms);

/* ---- Guided matching (FeatureMatcher::MatchGuided, feature/matcher.h:129), the decisions of the reference's CPU
 * guided matcher (SiftCPUFeatureMatcher::MatchGuided, sift.cc:1148-1300) bit for bit: exact L2 distances of the
 * descriptors, a candidate the pair's geometry rejects takes the distance 512^2, then FindBestMatchesIndex's min-L2
 * top-2, its distance and ratio tests and the cross-check (see DESIGN.md, "Guided matching"). */

/* The filter of one pair.  E: the squared tangent Sampson error of the two slots' camera rays (fp64), F: the squared
 * Sampson distance of the keypoints (fp32), H: the squared transfer error of the keypoints (fp32); a candidate is
 * rejected when its error exceeds max_error^2.  NONE: the pair has no matches. */
enum { B200SM_GUIDED_NONE = 0, B200SM_GUIDED_E = 1, B200SM_GUIDED_F = 2, B200SM_GUIDED_H = 3 };
typedef struct b200sm_guided_geometry {
  int type;           /* B200SM_GUIDED_* */
  double max_error;   /* pixels, finite and >= 0 */
  double M[9];        /* E, F or H, row-major, mapping image 1 to image 2 */
} b200sm_guided_geometry;

/* Uploads an image's keypoints (n x 2 floats: x, y) into `slot`; rows pair with the descriptor rows, so n must equal the
 * slot's descriptor count when a guided pair uses it.  Clears the slot's camera rays.  b200sm_set_descriptors clears
 * the keypoints. */
int b200sm_set_keypoints(b200sm_handle h, int slot, int64_t n, const float* xy);

/* Gives `slot` a camera (model_id 0..17 as in sensor/models.h, its params in the reference's order): computes every
 * keypoint's ray and Jacobian (b200sm_cam_ray_from_img_with_jac) and validity on the host and uploads them.  Needs the
 * slot's keypoints. */
int b200sm_set_camera(b200sm_handle h, int slot, int model_id, const double* params);

/* Camera::CamRayFromImgWithJac (scene/camera.h:355-371) of the pixel xy[2]: out9 = the unit ray, then d(ray)/d(pixel)
 * as a row-major 3 x 2 matrix.  Returns 1, or 0 where the reference returns nullopt (out9 untouched), or negative on
 * an invalid argument. */
int b200sm_cam_ray_from_img_with_jac(int model_id, const double* params, const double* xy, double* out9);

/* Guided matching of every pair p of (slot1[p], slot2[p]) under geometry g[p]; output as b200sm_match_pairs, and
 * capacity bounded by b200sm_match_capacity.  Refused before any device work: an E pair whose slot has no camera, an
 * F or H pair whose slot has no keypoints, keypoint counts that differ from descriptor counts, an unknown type, and a
 * max_error that is non-finite or negative. */
int b200sm_match_guided_pairs(b200sm_handle h, int num_pairs, const int* slot1, const int* slot2,
                              const b200sm_guided_geometry* g, uint64_t* offsets, uint32_t* matches, size_t capacity);

void b200sm_destroy(b200sm_handle h);

const char* b200sm_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_SIFT_MATCHING_H_ */
