/*
 * b200_patch_match.h — C-ABI of the CUDA (sm_90a, H100) PatchMatch MVS sweep.
 *
 * This is the drop-in boundary for COLMAP's `mvs::PatchMatchCuda`
 * (reference: src/colmap/mvs/patch_match_cuda.h:49-59, the only caller being
 * src/colmap/mvs/patch_match.cc:128-154).  Every entry point below replaces
 * one member of that class; INTEGRATION.md shows the ~60-line C++ adapter a
 * COLMAP maintainer would add.
 *
 * Conventions: plain pointers and sizes only, no exceptions cross the ABI,
 * 0 == success, negative == error (text via b200pm_last_error()).  A handle
 * is owned by one host thread at a time (same contract as the reference: one
 * PatchMatchCuda instance per host thread per GPU).
 */
#ifndef B200_PATCH_MATCH_H_
#define B200_PATCH_MATCH_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Mirrors mvs::PatchMatchOptions (src/colmap/mvs/patch_match_options.h:37-126);
 * same names, same defaults (b200pm_options_init).  Only the fields that reach
 * PatchMatchCuda are present; cache_size / num_threads / max_image_size /
 * allow_missing_files / write_consistency_graph belong to the controller. */
typedef struct b200pm_options {
  double depth_min;                        /* must be >= 0 here: the controller resolves -1 (patch_match.cc:423-432) */
  double depth_max;
  double sigma_spatial;                    /* <= 0 -> window_radius (patch_match.cc:436-438) */
  double sigma_color;                      /* 0.2 */
  double ncc_sigma;                        /* 0.6 */
  double min_triangulation_angle;          /* degrees, 1.0 */
  double incident_angle_sigma;             /* 0.9 */
  double geom_consistency_regularizer;     /* 0.3 */
  double geom_consistency_max_cost;        /* 3.0 */
  double filter_min_ncc;                   /* 0.1 */
  double filter_min_triangulation_angle;   /* degrees, 3.0 */
  double filter_geom_consistency_max_cost; /* 1.0 */
  int window_radius;                       /* 5 */
  int window_step;                         /* 1 (1 or 2) */
  int num_samples;                         /* 15 */
  int num_iterations;                      /* 5 */
  int filter_min_num_consistent;           /* 2 */
  int geom_consistency;                    /* bool, default 1 */
  int filter;                              /* bool, default 1 */
  int gpu_index;                           /* CUDA device ordinal; -1 = current device */
} b200pm_options;

/* Mirrors mvs::PatchMatch::Problem + the mvs::Image fields PatchMatchCuda reads
 * (patch_match.h:57-75, image.h:39-104): 8-bit grey bitmaps, float K (3x3
 * row-major, zero skew, K[8]==1), R (3x3 row-major), T (3).  All pointers are
 * host memory and only need to stay valid for the duration of b200pm_create. */
typedef struct b200pm_problem {
  int ref_width, ref_height;
  const uint8_t* ref_gray;        /* ref_height * ref_width, row-major */
  float ref_K[9], ref_R[9], ref_T[3];
  int num_src;                    /* 1..32 */
  const int* src_width;           /* [num_src] */
  const int* src_height;          /* [num_src] */
  const uint8_t* const* src_gray; /* [num_src] row-major bitmaps */
  const float* src_K;             /* [num_src*9] */
  const float* src_R;             /* [num_src*9] */
  const float* src_T;             /* [num_src*3] */
  /* geom_consistency only (PatchMatchCuda::InitSourceImages / InitWorkspaceMemory,
   * patch_match_cuda.cu:1657-1691,1814-1852): photometric depth maps of the
   * source images (src_height*src_width each) and the photometric depth /
   * normal map of the reference image (normal: 3 slices of H*W). */
  const float* const* src_depth;  /* [num_src] or NULL */
  const float* ref_depth_init;    /* H*W or NULL */
  const float* ref_normal_init;   /* 3*H*W slice-major or NULL */
  const int* src_image_idxs;      /* [num_src] global image ids reported by get_consistency; NULL -> 0..num_src-1 */
  int maps_on_device;             /* 0: src_depth / ref_depth_init / ref_normal_init are host pointers (the reference's
                                   * contract); 1: they are DEVICE pointers on the handle's GPU - the photometric maps
                                   * stay in HBM between the two phases of a workspace run (b200pm_get_*_device on the
                                   * producing handle, an NCCL all-gather between ranks) instead of the reference's
                                   * round trip through `.photometric.bin` files (patch_match.cc:182-197) */
} b200pm_problem;

typedef struct b200pm_context* b200pm_handle;

/* Defaults of PatchMatchOptions (patch_match_options.h:37-126). */
void b200pm_options_init(b200pm_options* o);

/* PatchMatch::Check (patch_match.cc:67-126) + PatchMatchOptions::Check
 * (patch_match_options.cc:72-99).  Returns 0 or a negative code. */
int b200pm_check(const b200pm_options* o, const b200pm_problem* p);

/* PatchMatchCuda::PatchMatchCuda (patch_match_cuda.cu:1290-1302): selects the
 * device, uploads images/poses, prefilters the reference image, initialises
 * depth / normal / PRNG state.  Host -> device copies happen here. */
int b200pm_create(const b200pm_options* o, const b200pm_problem* p, b200pm_handle* out);

/* PatchMatchCuda::Run (patch_match_cuda.cu:1304-1352,1393-1546): initial cost +
 * num_iterations x 4 sweeps.  Asynchronous work is complete on return. */
int b200pm_run(b200pm_handle h);

/* Device time of the last b200pm_run in milliseconds (CUDA events), the
 * analogue of the reference's "Total" CudaTimer (patch_match_cuda.cu:1398,1545). */
float b200pm_last_run_ms(b200pm_handle h);
/* Device time spent in the sweep kernels only during the last run, and their launch count. */
float b200pm_last_sweep_ms(b200pm_handle h);
int b200pm_last_num_launches(b200pm_handle h);
/* Device time summed over the sweeps of the last run for one pass of the split sweep: 0 = pm_rand_kernel and
 * pm_msg_kernel, which run side by side (from the sweep's start until both are done), 1 = pm_pixel_kernel
 * (pixel-parallel NCC pass, the dominant kernel), 2 = pm_serial_kernel, 3 = pm_rand_kernel alone, 4 = pm_msg_kernel
 * alone (its own stream).  0, 1 and 2 add up to the sweep; 3 and 4 overlap inside 0. */
float b200pm_last_pass_ms(b200pm_handle h, int which);
/* The same for one sweep of the last run (sweep t runs in frame t % 4; -1 for a sweep that did not run). */
float b200pm_last_sweep_pass_ms(b200pm_handle h, int sweep, int which);
/* Device bytes of the handle's patch store (every pixel's bilateral reference patch, built once per run); 0 when the
 * store does not fit its budget (DESIGN.md §2) or B200PM_PATCH_STORE=0, and every pass builds the patch inline. */
size_t b200pm_patch_store_bytes(b200pm_handle h);

/* PatchMatchCuda::GetDepthMap / GetNormalMap / GetSelProbMap
 * (patch_match_cuda.cu:1354-1365).  Layouts match mvs::Mat<float>: slice-major,
 * then row-major: depth H*W, normal 3*H*W, sel_prob num_src*H*W. */
int b200pm_get_depth(b200pm_handle h, float* depth);
int b200pm_get_normal(b200pm_handle h, float* normal);
int b200pm_get_sel_prob(b200pm_handle h, float* sel_prob);
/* The same depth / normal maps written into DEVICE buffers of the caller (same layouts, the handle's GPU); no host copy. */
int b200pm_get_depth_device(b200pm_handle h, float* d_depth);
int b200pm_get_normal_device(b200pm_handle h, float* d_normal);

/* PatchMatchCuda::GetConsistentImageIdxs (patch_match_cuda.cu:1367-1391): flat
 * int list [col,row,n,idx_1..idx_n]... ; *data is malloc'ed, release with
 * b200pm_free.  Only valid when options.filter was set. */
int b200pm_get_consistency(b200pm_handle h, int** data, size_t* count);
/* Raw mask num_src*H*W (slice-major) behind the list above. */
int b200pm_get_consistency_mask(b200pm_handle h, uint8_t* mask);
void b200pm_free(void* p);

void b200pm_destroy(b200pm_handle h);
/* Destroyed handles (and finished BA solves) keep their device blocks in a per-device cache for the next equally sized
 * problem (a workspace run creates hundreds of them); this returns the cached blocks to the driver. */
void b200_release_cached_memory(void);
const char* b200pm_last_error(void);

/* ---- workspace-level entry: PatchMatchController::Run (src/colmap/mvs/patch_match.cc:170-207,385-535) ------------------
 * Reads <workspace>/sparse/{cameras,images,points3D}.bin (mvs::Model::ReadFromCOLMAP, model.cc:56-100), the problem list
 * <workspace>/<stereo>/patch-match.cfg (ReadProblems :240-372), resolves depth ranges from the sparse points (:419-431),
 * and for every problem writes <stereo>/{depth_maps,normal_maps,consistency_graphs}/<image>.<photometric|geometric>.bin.
 * Outputs that already exist are skipped (:410-414).  With options.geom_consistency the photometric pass (no filter) runs
 * for every problem first, then the geometric pass reads those maps back (:176-204).  One worker thread per entry of
 * gpu_indices (list a device twice to keep two problems in flight on it, :375-384).
 * Image decoding is the caller's (COLMAP's Bitmap::Read): load_gray returns a malloc'ed 8-bit grey bitmap; NULL selects
 * the built-in binary PGM (P5) reader.  A bitmap whose size differs from the camera's rescales K (Image::Rescale,
 * mvs/image.cc:66-95).  Multi-process runs (one process per GPU) pass rank / world_size - problems are dealt largest
 * first - and run phase 1, a barrier of their own, then phase 2. */
typedef int (*b200pm_load_gray_fn)(void* user, const char* path, int* width, int* height, uint8_t** data);
typedef struct b200pm_workspace {
  const char* workspace_path;
  const char* stereo_folder;      /* NULL -> "stereo" */
  const char* config_path;        /* NULL -> <workspace>/<stereo>/patch-match.cfg */
  const int* gpu_indices;         /* NULL -> {options.gpu_index} */
  int num_gpu_indices;
  int write_consistency_graph;
  b200pm_load_gray_fn load_gray;
  void* load_gray_user;
  int rank, world_size;           /* 0, 1 for a single process */
  int phase;                      /* 0: everything; 1: photometric pass of a geometric run only; 2: final pass only */
} b200pm_workspace;
int b200pm_run_workspace(const b200pm_options* options, const b200pm_workspace* w, int* num_processed);

#ifdef __cplusplus
}
#endif
#endif /* B200_PATCH_MATCH_H_ */
