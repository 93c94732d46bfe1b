/*
 * b200_rotation_averaging.h — C-ABI of rotation averaging (CUDA, sm_90a, H100): the L1 + IRLS solve the global mapper
 * runs before global positioning (reference: src/colmap/estimators/rotation_averaging_impl.{h,cc},
 * RotationAveragingProblem / RotationAveragingSolver, and optim/least_absolute_deviations.cc).  The caller builds the
 * flat problem (parameter blocks, pair constraints, gauge) as RotationAveragingProblem's constructor does; the library
 * runs RotationAveragingSolver::Solve on it on the GPU in fp64.
 *
 * Parameters: the frame blocks in order (3 components for a 3-DOF angle-axis frame, 1 for a gravity-aligned frame's
 * y-angle), then the estimated camera blocks (3 components each, an angle-axis cam_from_rig).  Residual rows: every
 * pair in order (3 rows for a 3-DOF pair, 1 for a 1-DOF pair), then the gauge rows (1 or 3).  Every non-zero of the
 * constraint matrix links residual component i of a row triple to parameter component i, so the normal matrix splits
 * into one matrix for the x and z components of the 3-DOF blocks and one for the y components of all blocks; each is
 * factored densely (see DESIGN.md, "Rotation averaging").
 *
 * Conventions: 0 == the solve ran (its outcome is summary.status), negative == error with b200ra_last_error() set, no
 * exceptions; every input is checked on the host before any device work.
 */
#ifndef B200_ROTATION_AVERAGING_H_
#define B200_ROTATION_AVERAGING_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { B200RA_OK = 0, B200RA_ERR_INPUT = -1, B200RA_ERR_TOO_LARGE = -2, B200RA_ERR_CUDA = -3 };
/* summary.status: the outcome of a solve that ran; on anything but SUCCESS the caller's rotations are untouched */
enum {
  B200RA_SUCCESS = 0,
  B200RA_FACTORIZATION_FAILED = 1,  /* a non-positive pivot in the L1 or an IRLS factorisation */
  B200RA_NAN_STEP = 2,              /* a step with a NaN component */
  B200RA_NAN_WEIGHT = 3,            /* an IRLS weight is NaN */
  B200RA_UNDERDETERMINED = 4        /* fewer residual rows than parameters with an L1 phase (the reference throws) */
};
enum { B200RA_GEMAN_MCCLURE = 0, B200RA_HALF_NORM = 1 };

/* Largest dimension of either per-axis matrix the dense fp64 factorisation takes. */
#define B200RA_MAX_AXIS_DIM 32768

/* RotationEstimatorOptions (estimators/rotation_averaging.h:25-96), the part the solver reads. */
typedef struct b200ra_options {
  int max_num_l1_iterations;             /* 5; 0 skips the L1 phase */
  double l1_step_convergence_threshold;  /* 1e-3 */
  int max_num_irls_iterations;           /* 100; 0 skips the IRLS phase */
  double irls_step_convergence_threshold;/* 1e-3 */
  double irls_loss_parameter_sigma;      /* 5 (degrees) */
  double ridge_regularization;           /* 1e-9; added to every diagonal entry when > 0 */
  int weight_type;                       /* B200RA_GEMAN_MCCLURE */
  int gpu_index;                         /* -1: current device */
} b200ra_options;
void b200ra_options_init(b200ra_options* o);

/* The ADMM constants of LeastAbsoluteDeviationSolver::Options, fixed: rho, alpha, absolute and relative tolerance.  The
 * ADMM iteration limit starts at 10 and doubles after every L1 outer iteration up to 100. */
#define B200RA_ADMM_RHO 1.0
#define B200RA_ADMM_ALPHA 1.0
#define B200RA_ADMM_ABS_TOL 1e-4
#define B200RA_ADMM_REL_TOL 1e-2

typedef struct b200ra_problem {
  int num_frames;
  const uint8_t* frame_dof;        /* [F] 3 (angle-axis rig_from_world) or 1 (gravity-aligned y-angle) */
  int num_cameras;                 /* estimated cam_from_rig blocks, 3 components each */
  double* rotations;               /* [num_params] in/out: frame blocks, then camera blocks */
  int num_pairs;
  const int32_t* pair_frame1;      /* [P] frame block of image 1 */
  const int32_t* pair_frame2;      /* [P] */
  const int32_t* pair_cam1;        /* [P] or NULL: camera block of image 1, -1 when its cam_from_rig is not estimated */
  const int32_t* pair_cam2;        /* [P] or NULL */
  const uint8_t* pair_dof;         /* [P] 3: R_cam2_from_cam1 is used; 1: angle and xz_error (both frames 1-DOF) */
  const double* pair_R;            /* [9P] row-major R_cam2_from_cam1 (rows of 1-DOF pairs are not read) */
  const double* pair_angle;        /* [P] or NULL if no 1-DOF pair: the y-angle of the gravity-aligned relative rotation */
  const double* pair_xz_error;     /* [P] or NULL if no 1-DOF pair */
  const double* pair_reweighting;  /* [P] or NULL (UNIFORM): the residual-space reweighting in (0, 1] */
  int gauge_frame;                 /* the fixed frame block */
  double gauge_rotation[3];        /* its fixed angle-axis rotation; a 1-DOF gauge reads [1] */
  const int32_t* cam_frame_start;  /* [C + 1] CSR: the frames UpdateState averages each camera's rotation over */
  const int32_t* cam_frames;       /* [cam_frame_start[C]] frame blocks */
} b200ra_problem;

typedef struct b200ra_summary {
  int status;                      /* B200RA_SUCCESS, ... */
  int num_l1_iterations;           /* L1 outer iterations run */
  int num_irls_iterations;
  int* admm_iterations;            /* optional, caller-owned [max_num_l1_iterations]: ADMM iterations per L1 iteration */
  double* step_history;            /* optional, caller-owned [max_num_l1 + max_num_irls]: AverageStepSize of every
                                      iteration, the L1 iterations first, then the IRLS iterations */
  int n_xz;                        /* dimension of the x/z matrix: 3-DOF frames + estimated cameras */
  int n_y;                         /* dimension of the y matrix: all frames + estimated cameras */
  int num_residuals;
  double l1_ms, irls_ms;           /* device time of each phase (CUDA events) */
  double build_ms, factor_ms, solve_ms;  /* of which: matrix builds, factorisations, triangular solves */
} b200ra_summary;

/* RotationAveragingSolver::Solve: the L1 phase, then the IRLS phase (either one is skipped when its iteration count is
 * 0).  On SUCCESS the rotations are updated in place; otherwise they stay bit-identical.  Returns
 * B200RA_ERR_TOO_LARGE, before any device work, when n_xz or n_y exceeds B200RA_MAX_AXIS_DIM. */
int b200ra_solve(const b200ra_options* o, b200ra_problem* p, b200ra_summary* out);

const char* b200ra_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_ROTATION_AVERAGING_H_ */
