/*
 * b200_ba_covariance.h — C-ABI of the bundle-adjustment covariance estimate (CUDA, sm_90a, H100), next to the solver
 * of b200_bundle_adjustment.h: the reference's EstimateBACovariance (src/colmap/estimators/covariance.{h,cc}) on the
 * flat problem a caller solved with b200ba_solve.  Errors are reported through b200ba_last_error().
 */
#ifndef B200_BA_COVARIANCE_H_
#define B200_BA_COVARIANCE_H_

#include "b200_bundle_adjustment.h"
#include "b200_ba_pose_prior.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- covariance of a solved problem: EstimateBACovariance (src/colmap/estimators/covariance.{h,cc}) ----
 * J = the loss-corrected, unscaled tangent-space Jacobian at the current parameters.  Point blocks: (H_pp + damping I)^-1,
 * conditioned on everything else.  Pose / sensor / intrinsics blocks: blocks of S^-1, S = the reduced camera-side matrix
 * (points Schur-eliminated); in POSES and POSES_AND_POINTS mode the intrinsics and sensor blocks are eliminated from S as
 * well, with damping on their diagonal.  Dimensions held constant are omitted from every block (a two-cams gauge pose has
 * 5 dimensions, a pose under constant_rig_from_world_rotation 3); pose blocks are in [rotation, translation] order.  The
 * reduced matrix is factorised densely on the GPU: its dimension is limited to 32768. */
enum { B200BA_COV_POSES = 0, B200BA_COV_POINTS = 1, B200BA_COV_POSES_AND_POINTS = 2, B200BA_COV_ALL = 3 };
typedef struct b200ba_covariance_options {
  int params;       /* B200BA_COV_ALL */
  double damping;   /* 1e-8 */
} b200ba_covariance_options;
void b200ba_covariance_options_init(b200ba_covariance_options* c);
typedef struct b200ba_covariance* b200ba_covariance_t;
/* The same options and problem the caller solved (refine flags, loss, gauge masks, rigs); parameters are read, never
 * written.  0 = ok, 1 = not estimable (a pivot of S <= 1e-6: an unfixed gauge or another degeneracy; b200ba_last_error
 * names the block and the pivot, *out stays NULL), < 0 = error. */
int b200ba_estimate_covariance(const b200ba_options* o, const b200ba_covariance_options* c, const b200ba_problem* p,
                               b200ba_covariance_t* out);
/* The same for a problem solved with b200ba_solve_with_position_priors (the reference's EstimateBACovariance on a
 * PosePriorBundleAdjuster): J also holds the covariance-weighted prior rows, corrected by the priors' own loss, so the
 * priors can make S invertible where no gauge is fixed.  The priors are read at the parameters of p and must be in the
 * same frame.  Priors whose blocks are all constant are skipped; they never touch the point blocks.  Bad priors (index
 * out of range, non-finite values, a covariance that is not SPD) return < 0 with a message before any device work.
 * priors == NULL or num_priors == 0 is b200ba_estimate_covariance.  Return codes and the handle as above. */
int b200ba_estimate_covariance_with_position_priors(const b200ba_options* o, const b200ba_covariance_options* c,
                                                    const b200ba_problem* p, const b200ba_position_priors* priors,
                                                    b200ba_covariance_t* out);
/* Each getter returns the block's tangent size and writes size x size doubles (row-major), or returns 0 when the block is
 * not variable or was not estimated in this mode (the reference's nullopt). */
int b200ba_covariance_point(b200ba_covariance_t h, int64_t point, double out[9]);
int b200ba_covariance_pose(b200ba_covariance_t h, int pose, double out[36]);
/* rows x cols block between two poses; returns rows * cols (0 = either pose not estimated) */
int b200ba_covariance_pose_cross(b200ba_covariance_t h, int pose1, int pose2, double out[36], int* rows, int* cols);
int b200ba_covariance_camera(b200ba_covariance_t h, int camera, double out[256]);   /* variable intrinsics, index order */
int b200ba_covariance_sensor(b200ba_covariance_t h, int sensor, double out[36]);    /* sensor_from_rig, [rotation, translation] */
/* bulk read-back: out[num_poses][36] (each block row-major in its first size*size entries) and size[num_poses] (0 = none);
 * out[num_points][9] and valid[num_points].  Returns 0, or < 0 on error. */
int b200ba_covariance_poses_all(b200ba_covariance_t h, double* out, int8_t* size);
int b200ba_covariance_points_all(b200ba_covariance_t h, double* out, uint8_t* valid);
/* dimension of the factorised matrix and device times (ms) of the phases: set-up, build, factorisation, inverse */
int b200ba_covariance_info(b200ba_covariance_t h, double* ms4);
void b200ba_covariance_free(b200ba_covariance_t h);

#ifdef __cplusplus
}
#endif
#endif /* B200_BA_COVARIANCE_H_ */
