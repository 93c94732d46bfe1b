// ba_dense_f64.h — tiled fp64 Cholesky and SPD inverse on the H100's fp64 tensor cores (mma.sync m16n8k4 .f64).
// Used by the bundle-adjustment covariance estimate (b200ba_estimate_covariance) on the reduced camera-side matrix, and
// by the global positioning and rotation averaging solves.
//
// Layout: an N x N column-major matrix, N a multiple of BA_TILE; element (i, j), i >= j, lives at A[j * N + i] (the
// layout of the solve's dense reduced matrix).  Only the lower triangle is input and output.  Outside the 64 x 64
// diagonal tiles the strict upper triangle is neither read nor written; inside them it is scratch (the kernels write
// whole diagonal tiles) and holds no defined value afterwards.  Callers pad the matrix to N with an identity block,
// whose factor and inverse are again the identity.
#pragma once
#include <cuda_runtime.h>

#define BA_TILE 64

// Device-side status of a factorisation.  bad != 0 after a failed pivot d (d before the square root, i.e. the LDL^T
// pivot); later launches of the same factorisation and of ba_dense_potri then return at once.
struct BaDenseFlag {
  int bad;
  int row;        // first row whose pivot failed
  double pivot;   // its value
};

// A = L L^T in place (lower triangle).  The pivot of row r fails when !(d > pivot_min) for n_test0 <= r < n_check
// (the rank test), when !(d > 0) for r < n_test0 (positive definiteness only), and is not tested for r >= n_check
// (padding).  dinv: [N * BA_TILE] scratch that receives the inverse of every diagonal tile of L (read again by
// ba_dense_potri).
cudaError_t ba_dense_potrf(double* A, int N, int n_test0, int n_check, double pivot_min, double* dinv, BaDenseFlag* flag,
                           cudaStream_t st);
// A (holding L from ba_dense_potrf) <- (L L^T)^-1 = L^-T L^-1, lower triangle: TRTRI then LAUUM.  panel: [N * BA_TILE] scratch.
cudaError_t ba_dense_potri(double* A, int N, const double* dinv, double* panel, const BaDenseFlag* flag, cudaStream_t st);
// Solve L L^T X = B for nrhs right-hand sides with L and dinv from ba_dense_potrf.  B: [nrhs * N] column-major (ld N),
// the right-hand sides in, the solutions out; W: [nrhs * N] scratch.  Each right-hand side sees the same arithmetic in
// the same order whatever nrhs is.  Returns at once on every launch when flag->bad is set.
cudaError_t ba_dense_potrs(const double* A, int N, const double* dinv, int nrhs, double* B, double* W, const BaDenseFlag* flag,
                           cudaStream_t st);
