/*
 * b200_global_positioning.h — C-ABI of the global positioner (CUDA, sm_90a, H100): the BATA point-to-camera problem the
 * global mapper solves before its bundle adjustment (reference: src/colmap/estimators/global_positioning.{h,cc},
 * GlobalPositioner::AddPoint3DToProblem / ParameterizeVariables, cost functors estimators/cost_functions/
 * motion_averaging.h).  The caller builds the flat problem (frame centres, points, rays, scales) as GlobalPositioner's
 * setup does; the library runs Ceres' trust-region Levenberg-Marquardt on it on the GPU in fp64.
 *
 * Residual per observation, r = d - s (X - c + t), with d the unit ray in the world frame, s the observation's scale,
 * X the point, c the frame centre and
 *   sensor == -1:  t = rig_offset          (trivial frame: zero; constant rig: R(cam_from_world)^T t(cam_from_rig))
 *   sensor >= 0:   t = -R(world_from_rig) cams_in_rig[sensor]   (a camera-in-rig position that is estimated)
 * under Huber(loss_function_scale), times the observation's loss weight (0.5: the reference's ScaledLoss for a camera
 * without a prior focal length).  Conventions: 0 == success, negative == error with b200gp_last_error() set, no
 * exceptions; every input is checked on the host before any device work.
 */
#ifndef B200_GLOBAL_POSITIONING_H_
#define B200_GLOBAL_POSITIONING_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { B200GP_OK = 0, B200GP_ERR_INPUT = -1, B200GP_ERR_TOO_LARGE = -2, B200GP_ERR_CUDA = -3 };
/* termination types, as BundleAdjustmentTerminationType / ceres::TerminationType */
enum { B200GP_CONVERGENCE = 0, B200GP_NO_CONVERGENCE = 1, B200GP_FAILURE = 2 };

/* Largest reduced (frame centre + camera-in-rig) dimension the dense fp64 reduced solve takes: 3 per variable block. */
#define B200GP_MAX_REDUCED_DIM 32768
/* lower bound of every scale (SetParameterLowerBound(&scale, 0, 1e-5)) */
#define B200GP_SCALE_LOWER_BOUND 1e-5

/* GlobalPositionerOptions (global_positioning.h:13-60) and the Ceres solver options it keeps or sets. */
typedef struct b200gp_options {
  int optimize_positions;               /* 1: frame centres variable */
  int optimize_points;                  /* 1: points variable */
  int optimize_scales;                  /* 1: scales variable (the first observation's scale is always constant) */
  int refine_sensor_from_rig;           /* 1; 0 refuses observations with sensor >= 0 */
  double loss_function_scale;           /* 0.1 (Huber) */
  int max_num_iterations;               /* 100 */
  double function_tolerance;            /* 1e-5 */
  double gradient_tolerance;            /* 1e-10 */
  double parameter_tolerance;           /* 1e-8 */
  double initial_trust_region_radius;   /* 1e4 */
  double max_trust_region_radius;       /* 1e16 */
  double min_trust_region_radius;       /* 1e-32 */
  double min_relative_decrease;         /* 1e-3 */
  double min_lm_diagonal;               /* 1e-6 */
  double max_lm_diagonal;               /* 1e32 */
  int gpu_index;                        /* -1: current device */
} b200gp_options;
void b200gp_options_init(b200gp_options* o);

typedef struct b200gp_problem {
  int num_frames;
  double* frame_centers;            /* [3F] in/out: rig centre in the world */
  const uint8_t* frame_constant;    /* [F] or NULL: 1 = held constant */
  const double* world_from_rig;     /* [9F] row-major rotations; read only for observations with sensor >= 0 (NULL if none) */
  int64_t num_points;
  double* points;                   /* [3P] in/out */
  int num_sensors;
  double* cams_in_rig;              /* [3S] in/out: camera centres in their rig's frame, estimated */
  int64_t num_observations;
  const int32_t* obs_frame;         /* [N] */
  const int32_t* obs_point;         /* [N] */
  const int32_t* obs_sensor;        /* [N] or NULL: -1 = none */
  const double* obs_ray;            /* [3N] world-frame direction d */
  const double* obs_rig_offset;     /* [3N] or NULL (zero); used where sensor == -1 */
  double* obs_scale;                /* [N] in/out, >= B200GP_SCALE_LOWER_BOUND; observation 0's scale is the gauge */
  const double* obs_loss_weight;    /* [N] or NULL (1.0): 1.0 or 0.5 */
} b200gp_problem;

typedef struct b200gp_summary {
  int termination_type;
  int num_successful_steps;
  int num_unsuccessful_steps;
  int num_residuals;                /* 3 per observation */
  int reduced_dim;                  /* n of the dense reduced system */
  double initial_cost;
  double final_cost;
  double solve_ms;                  /* device time of the LM loop (CUDA events) */
  double* cost_history;             /* optional, caller-owned [max_num_iterations + 1]: the cost of the current
                                       parameters before iteration 0 and after every iteration */
  int num_iterations;               /* entries written to cost_history minus one */
} b200gp_summary;

/* Solve in place: frame_centers, points, cams_in_rig and obs_scale of variable blocks are updated; constant blocks stay
 * bit-identical.  Returns B200GP_ERR_TOO_LARGE, before any device work, when the reduced dimension exceeds
 * B200GP_MAX_REDUCED_DIM (a sparse reduced factorisation is not implemented). */
int b200gp_solve(const b200gp_options* o, b200gp_problem* p, b200gp_summary* out);

/* CameraModelCamRayFromImg (sensor/models.h:353-370, 3029-3047) on the host, all eighteen models: CamFromImg with the
 * models' iterative undistortion, then normalisation; EQUIRECTANGULAR computes the ray directly.  Returns 0 with the unit
 * ray in ray_out[3], or B200GP_ERR_INPUT where the reference returns nullopt (or the model id is unknown). */
int b200gp_cam_ray_from_img(int model_id, const double* params, const double* xy, double* ray_out);

const char* b200gp_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_GLOBAL_POSITIONING_H_ */
