/*
 * b200_ba_pose_prior.h — C-ABI of the pose-prior bundle adjustment (CUDA, sm_90a, H100), next to the solver of
 * b200_bundle_adjustment.h: the residuals the reference's PosePriorBundleAdjuster adds to the problem
 * (src/colmap/estimators/bundle_adjustment_ceres.cc:987-1039), solved by the same GPU LM loop.  The alignment of the
 * reconstruction to the priors and its normalisation stay with the caller; the positions and covariances passed here are
 * already in the problem's frame.  Errors are reported through b200ba_last_error().
 */
#ifndef B200_BA_POSE_PRIOR_H_
#define B200_BA_POSE_PRIOR_H_

#include "b200_bundle_adjustment.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One covariance-weighted position residual per prior (CovarianceWeightedCostFunctor, estimators/cost_functions/utils.h):
 *   reference sensor      r = L^T (c_prior + R(rig_from_world)^T t(rig_from_world))
 *   non-reference sensor  the same on cam_from_world = sensor_from_rig * rig_from_world, with Jacobians for both blocks
 * with L = chol(cov^-1) (the library forms it).  The priors share one robust loss, separate from the observations'. */
typedef struct b200ba_position_priors {
  int num_priors;
  const int32_t* pose_idx;       /* flat pose (rig_from_world / image pose) the prior constrains */
  const int32_t* sensor_idx;     /* -1: reference sensor; else index into problem->sensor_from_rig (NULL: all -1) */
  const double* position;        /* [3*num_priors], already in the problem's (normalized) frame */
  const double* covariance;      /* [9*num_priors] row-major, same frame, symmetric positive definite */
  int loss_function_type;        /* B200BA_LOSS_* ; default TRIVIAL */
  double loss_function_scale;    /* default sqrt(7.814727903251179) */
} b200ba_position_priors;
void b200ba_position_priors_init(b200ba_position_priors* p);
/* b200ba_solve with the prior residuals added.  A prior whose blocks are all constant in the solve (constant or unobserved
 * pose, reference or constant sensor) is skipped; summary->num_residuals counts 3 per prior kept.  Returns < 0, with a
 * message, on an index out of range, a non-finite position or covariance, or a covariance that is not symmetric positive
 * definite.  num_priors == 0 (or priors == NULL) is b200ba_solve. */
int b200ba_solve_with_position_priors(const b200ba_options* o, b200ba_problem* p, const b200ba_position_priors* priors,
                                      b200ba_summary* out);

/* test hook: the unweighted residual c + R^T t of cam_from_world = sensor * rig (sensor NULL: identity) and its Jacobians
 * in the solve's tangent space [rotation (Plus of the quaternion), translation], 3x6 row-major each */
void b200ba_test_prior_position(const double* rig, const double* sensor, const double* position, double* res,
                                double* J_rig, double* J_sensor);
/* test hook: the weight chol(cov^-1)^T (upper triangular, row-major) the solve applies; 0 = ok, < 0 = not SPD / not finite */
int b200ba_test_prior_weight(const double* covariance, double* weight);

#ifdef __cplusplus
}
#endif
#endif /* B200_BA_POSE_PRIOR_H_ */
