/*
 * ba_prior_oracle.c — CPU restatement (fp64) of the pose-prior bundle adjustment: the LM solve of oracle/ba_oracle.c with
 * the covariance-weighted position-prior residuals of the reference's PosePriorBundleAdjuster added
 * (src/colmap/estimators/bundle_adjustment_ceres.cc:987-1039, cost_functions/pose_prior.h:75-126, utils.h:124-163).
 *
 * TEST INFRASTRUCTURE ONLY: tests/oracle_prior.py compiles it (gcc -O2 -fopenmp) into a temporary directory.  It includes
 * the observation oracle's source unchanged and reuses its building blocks (linearize, schur_apply, the loss, the
 * manifold); the LM loop below is ba_oracle_solve with the prior rows added wherever Ceres sees residual rows: the cost,
 * the Jacobi column norms, the gradient and the LM diagonal, the reduced camera matrix (dense and matrix-free), the
 * SCHUR_JACOBI blocks, the model decrease and the candidate cost.
 *
 * The prior Jacobians take a route independent of the product's analytic formulas: the residual is evaluated over
 * complex numbers, the ambient (quaternion, translation) Jacobian comes from the complex step, and the tangent Jacobian is
 * that times EigenQuaternionManifold's PlusJacobian, as ceres' autodiff cost function with a manifold computes it.
 */
#include "../oracle/ba_oracle.c"
#include "../include/b200_ba_pose_prior.h"

/* ------------------------------------------------------------------------- residual */
static void c_qmul(const cplx* a, const cplx* b, cplx* o) { /* Eigen Hamilton product, storage (x, y, z, w) */
  o[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  o[1] = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0];
  o[2] = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3];
  o[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
}
static void c_rotate(const cplx* q, const cplx* v, cplx* o) { /* Eigen _transformVector: v + w uv + q.vec x uv, uv = 2 q.vec x v */
  const cplx uv[3] = {2.0 * (q[1] * v[2] - q[2] * v[1]), 2.0 * (q[2] * v[0] - q[0] * v[2]), 2.0 * (q[0] * v[1] - q[1] * v[0])};
  o[0] = v[0] + q[3] * uv[0] + (q[1] * uv[2] - q[2] * uv[1]);
  o[1] = v[1] + q[3] * uv[1] + (q[2] * uv[0] - q[0] * uv[2]);
  o[2] = v[2] + q[3] * uv[2] + (q[0] * uv[1] - q[1] * uv[0]);
}
/* AbsolutePosePositionPriorCostFunctor (sensor == NULL) / AbsoluteRigPosePositionPriorCostFunctor */
static void c_prior_residual(const cplx* rig, const cplx* sensor, const double* c, cplx* r) {
  cplx q[4], t[3];
  if (sensor) {
    c_qmul(sensor, rig, q);
    c_rotate(sensor, rig + 4, t);
    for (int a = 0; a < 3; ++a) t[a] += sensor[4 + a];
  } else {
    for (int a = 0; a < 4; ++a) q[a] = rig[a];
    for (int a = 0; a < 3; ++a) t[a] = rig[4 + a];
  }
  const cplx qi[4] = {-q[0], -q[1], -q[2], q[3]};
  cplx v[3];
  c_rotate(qi, t, v);
  for (int a = 0; a < 3; ++a) r[a] = c[a] + v[a];
}
/* residual and tangent Jacobians (3x6 row-major, [rotation | translation]) of both blocks; J_sensor is zero without a
 * sensor */
void ba_oracle_prior_position(const double* rig, const double* sensor, const double* c, double* res, double* J_rig,
                              double* J_sensor) {
  const double h = 1e-40;
  cplx in[14], r[3];
  for (int k = 0; k < 7; ++k) { in[k] = rig[k]; in[7 + k] = sensor ? sensor[k] : 0.0; }
  c_prior_residual(in, sensor ? in + 7 : NULL, c, r);
  for (int a = 0; a < 3; ++a) res[a] = creal(r[a]);
  double Ja[2][21];   /* ambient 3x7 per block */
  for (int blk = 0; blk < 2; ++blk)
    for (int k = 0; k < 7; ++k) {
      if (blk == 1 && !sensor) { for (int a = 0; a < 3; ++a) Ja[1][7 * a + k] = 0.0; continue; }
      const cplx keep = in[7 * blk + k];
      in[7 * blk + k] = keep + h * I;
      c_prior_residual(in, sensor ? in + 7 : NULL, c, r);
      in[7 * blk + k] = keep;
      for (int a = 0; a < 3; ++a) Ja[blk][7 * a + k] = cimag(r[a]) / h;
    }
  for (int blk = 0; blk < 2; ++blk) {
    const double* q = blk == 0 ? rig : (sensor ? sensor : rig);
    const double PJ[12] = {q[3], q[2], -q[1], -q[2], q[3], q[0], q[1], -q[0], q[3], -q[0], -q[1], -q[2]};
    double* J = blk == 0 ? J_rig : J_sensor;
    for (int a = 0; a < 3; ++a) {
      for (int j = 0; j < 3; ++j) {
        double v = 0;
        for (int k = 0; k < 4; ++k) v += Ja[blk][7 * a + k] * PJ[3 * k + j];
        J[6 * a + j] = v;
      }
      for (int j = 0; j < 3; ++j) J[6 * a + 3 + j] = Ja[blk][7 * a + 4 + j];
    }
  }
}

/* ------------------------------------------------------------------------- the priors of one solve */
typedef struct {
  int n, loss;
  double scale;
  int *pi, *si, *po, *so;        /* pose, sensor, camera-side offsets of the pose and sensor blocks (-1: constant) */
  double *c, *W;                 /* [3n], [9n] chol(cov^-1)^T */
  double *J, *r, *cost;          /* [36n] weighted, loss-corrected, unscaled 3 x [pose 6 | sensor 6]; [3n]; [n] */
} prior_set;

static int weight_of(const double* C, double* W) {   /* chol(inv(C))^T via numpy-like dense steps */
  double inv[9];
  if (!chol3_inv(C, inv)) return 0;
  double L[9] = {0};
  for (int j = 0; j < 3; ++j) {
    double d = inv[4 * j];
    for (int k = 0; k < j; ++k) d -= L[3 * j + k] * L[3 * j + k];
    if (!(d > 0)) return 0;
    L[4 * j] = sqrt(d);
    for (int r = j + 1; r < 3; ++r) { double t = inv[3 * r + j]; for (int k = 0; k < j; ++k) t -= L[3 * r + k] * L[3 * j + k]; L[3 * r + j] = t / L[4 * j]; }
  }
  for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) W[3 * a + b] = L[3 * b + a];
  return 1;
}

/* weighted residual rw and (want_jac) its loss-corrected weighted Jacobian and residual at (poses, sens); returns 1/2 rho */
static double prior_eval(const ba_flat* F, prior_set* S, int k, const double* poses, const double* sens, int want_jac) {
  double res[3], Jr[18], Js[18], rw[3], J[36], rho[3];
  ba_oracle_prior_position(poses + 7 * S->pi[k], S->si[k] >= 0 ? sens + 7 * S->si[k] : NULL, S->c + 3 * k, res, Jr, Js);
  const double* W = S->W + 9 * k;
  for (int a = 0; a < 3; ++a) rw[a] = W[3 * a] * res[0] + W[3 * a + 1] * res[1] + W[3 * a + 2] * res[2];
  const double s = rw[0] * rw[0] + rw[1] * rw[1] + rw[2] * rw[2];
  loss_eval(S->loss, S->scale, s, rho);
  if (!want_jac) return 0.5 * rho[0];
  const uint8_t m = S->po[k] >= 0 ? F->pose_mask[S->pi[k]] : 0;
  for (int a = 0; a < 3; ++a)
    for (int j = 0; j < 6; ++j) {
      const double jr = W[3 * a] * Jr[j] + W[3 * a + 1] * Jr[6 + j] + W[3 * a + 2] * Jr[12 + j];
      const double js = W[3 * a] * Js[j] + W[3 * a + 1] * Js[6 + j] + W[3 * a + 2] * Js[12 + j];
      J[12 * a + j] = ((m >> j) & 1) ? jr : 0.0;
      J[12 * a + 6 + j] = S->so[k] >= 0 ? js : 0.0;
    }
  double rs = 1.0;
  if (S->loss != B200BA_LOSS_TRIVIAL) {   /* ceres Corrector */
    const double sqrt_rho1 = sqrt(rho[1]);
    double alpha_sq_norm = 0.0;
    rs = sqrt_rho1;
    if (s != 0.0 && rho[2] > 0.0) {
      const double alpha = 1.0 - sqrt(1.0 + 2.0 * s * rho[2] / rho[1]);
      rs = sqrt_rho1 / (1 - alpha);
      alpha_sq_norm = alpha / s;
    }
    for (int j = 0; j < 12; ++j) {
      const double rj = rw[0] * J[j] + rw[1] * J[12 + j] + rw[2] * J[24 + j];
      for (int a = 0; a < 3; ++a) J[12 * a + j] = sqrt_rho1 * (J[12 * a + j] - alpha_sq_norm * rw[a] * rj);
    }
  }
  memcpy(S->J + 36 * k, J, sizeof(J));
  for (int a = 0; a < 3; ++a) S->r[3 * k + a] = rs * rw[a];
  S->cost[k] = 0.5 * rho[0];
  return 0.5 * rho[0];
}
static inline int col_of(const prior_set* S, int k, int j) { return j < 6 ? (S->po[k] >= 0 ? S->po[k] + j : -1) : (S->so[k] >= 0 ? S->so[k] + j - 6 : -1); }
/* linearize() plus the prior rows: cost, and with want_jac = 0 the per-residual cost change added to F->cost_delta */
static double linearize_all(ba_flat* F, prior_set* S, const double* poses, const double* sens, const double* cams, const double* pts, int want_jac) {
  double cost = linearize(F, poses, sens, cams, pts, want_jac);
  for (int k = 0; k < S->n; ++k) {
    const double c = prior_eval(F, S, k, poses, sens, want_jac);
    cost += c;
    if (!want_jac) F->cost_delta += c - S->cost[k];
  }
  return cost;
}
/* y (3) = J_scaled(k) x */
static void prior_times(const ba_flat* F, const prior_set* S, int k, const double* x, double y[3]) {
  y[0] = y[1] = y[2] = 0;
  for (int j = 0; j < 12; ++j) {
    const int col = col_of(S, k, j);
    if (col < 0) continue;
    const double v = F->scale_c[col] * x[col];
    for (int a = 0; a < 3; ++a) y[a] += S->J[36 * k + 12 * a + j] * v;
  }
}
static void prior_t_times_add(const ba_flat* F, const prior_set* S, int k, const double u[3], double* out) {
  for (int j = 0; j < 12; ++j) {
    const int col = col_of(S, k, j);
    if (col >= 0) out[col] += F->scale_c[col] * (S->J[36 * k + j] * u[0] + S->J[36 * k + 12 + j] * u[1] + S->J[36 * k + 24 + j] * u[2]);
  }
}
static void schur_apply_all(const ba_flat* F, const prior_set* S, const ba_lin* L, const double* x, double* out) {
  schur_apply(F, L, x, out);
  for (int k = 0; k < S->n; ++k) { double y[3]; prior_times(F, S, k, x, y); prior_t_times_add(F, S, k, y, out); }
}
/* schur_jacobi() with the prior rows' J_b^T J_b added to the pose and sensor blocks before the inversion */
static void schur_jacobi_all(const ba_flat* F, const prior_set* S, const ba_lin* L, const int* blk_start, int nblk, double* Minv, const int* blk_pack) {
  /* schur_jacobi() inverts the blocks it forms, so its block formula is restated here (serially) and the prior rows are
   * added before the inversion */
  const size_t msize = (size_t)blk_pack[nblk] + 1;
  double* M = (double*)calloc(msize, sizeof(double));
  for (int64_t j = 0; j < F->nobs; ++j) {
    obs_blk B; obs_blocks(F, j, &B);
    const double* Jc = F->Jc + 2 * JC * j;
    for (int which = 0; which < 3; ++which) {
      const int off = B.off[which], n = B.n[which], jo = B.jo[which];
      if (off < 0) continue;
      int b; { int lo = 0, hi = nblk - 1; while (lo < hi) { const int mid = (lo + hi + 1) / 2; if (blk_start[mid] <= off) lo = mid; else hi = mid - 1; } b = lo; }
      double* Mb = M + blk_pack[b];
      for (int r = 0; r < n; ++r)
        for (int c = 0; c < n; ++c)
          Mb[r * n + c] += F->scale_c[off + r] * F->scale_c[off + c] * (Jc[jo + r] * Jc[jo + c] + Jc[JC + jo + r] * Jc[JC + jo + c]);
    }
  }
  for (int64_t k = 0; k < F->nvpt; ++k) {
    const int64_t s = F->pt_start[k], e2 = F->pt_start[k + 1];
    const double* Hi = L->Hpp_inv + 9 * k;
    for (int64_t j = s; j < e2; ++j)
      for (int which = 0; which < 3; ++which) {
        obs_blk B; obs_blocks(F, j, &B);
        const int off = B.off[which], n = B.n[which];
        if (off < 0) continue;
        int first = 1;
        for (int64_t j2 = s; j2 < j && first; ++j2) { obs_blk B2; obs_blocks(F, j2, &B2); if (B2.off[which] == off) first = 0; }
        if (!first) continue;
        double V[3 * MAXDK];
        memset(V, 0, sizeof(V));
        for (int64_t j2 = j; j2 < e2; ++j2) {
          obs_blk B2; obs_blocks(F, j2, &B2);
          if (B2.off[which] != off) continue;
          const double* Jc = F->Jc + 2 * JC * j2; const double* Jp = F->Jp + 6 * j2; const int jo = B2.jo[which];
          for (int a = 0; a < 3; ++a)
            for (int c = 0; c < n; ++c)
              V[a * n + c] += F->scale_p[3 * k + a] * F->scale_c[off + c] * (Jp[a] * Jc[jo + c] + Jp[3 + a] * Jc[JC + jo + c]);
        }
        int b; { int lo = 0, hi = nblk - 1; while (lo < hi) { const int mid = (lo + hi + 1) / 2; if (blk_start[mid] <= off) lo = mid; else hi = mid - 1; } b = lo; }
        double* Mb = M + blk_pack[b];
        for (int r = 0; r < n; ++r)
          for (int c = 0; c < n; ++c) {
            double t = 0;
            for (int a = 0; a < 3; ++a) for (int a2 = 0; a2 < 3; ++a2) t += V[a * n + r] * Hi[3 * a + a2] * V[a2 * n + c];
            Mb[r * n + c] -= t;
          }
      }
  }
  for (int k = 0; k < S->n; ++k)   /* prior rows: the pose block and the sensor block, no cross term (block diagonal) */
    for (int blk = 0; blk < 2; ++blk) {
      const int off = blk == 0 ? S->po[k] : S->so[k], j0 = 6 * blk;
      if (off < 0) continue;
      int b; { int lo = 0, hi = nblk - 1; while (lo < hi) { const int mid = (lo + hi + 1) / 2; if (blk_start[mid] <= off) lo = mid; else hi = mid - 1; } b = lo; }
      double* Mb = M + blk_pack[b];
      const double* J = S->J + 36 * k;
      for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c)
          Mb[r * 6 + c] += F->scale_c[off + r] * F->scale_c[off + c] * (J[j0 + r] * J[j0 + c] + J[12 + j0 + r] * J[12 + j0 + c] + J[24 + j0 + r] * J[24 + j0 + c]);
    }
  for (int b = 0; b < nblk; ++b) { const int n = blk_start[b + 1] - blk_start[b]; for (int r = 0; r < n; ++r) M[blk_pack[b] + r * n + r] += L->Dc2[blk_start[b] + r]; }
  for (int b = 0; b < nblk; ++b) {
    const int n = blk_start[b + 1] - blk_start[b];
    double A[MAXDK * MAXDK], col[MAXDK];
    for (int c = 0; c < n; ++c) {
      memcpy(A, M + blk_pack[b], sizeof(double) * n * n);
      for (int r = 0; r < n; ++r) col[r] = r == c ? 1.0 : 0.0;
      if (!chol_solve(n, A, col)) { for (int r = 0; r < n; ++r) col[r] = r == c ? 1.0 : 0.0; }
      for (int r = 0; r < n; ++r) Minv[blk_pack[b] + r * n + c] = col[r];
    }
  }
  free(M);
}

/* ------------------------------------------------------------------------- the solve */
int ba_oracle_solve_with_position_priors(const b200ba_options* o, b200ba_problem* p, const b200ba_position_priors* pr, b200ba_summary* sum) {
  memset(sum, 0, sizeof(*sum));
  sum->termination_type = B200BA_FAILURE;
  const int npr = pr ? pr->num_priors : 0;
  for (int k = 0; k < npr; ++k) {
    if (pr->pose_idx[k] < 0 || pr->pose_idx[k] >= p->num_poses) return -2;
    const int s = pr->sensor_idx ? pr->sensor_idx[k] : -1;
    if (s < -1 || s >= p->num_sensors) return -2;
  }
  ba_flat F; memset(&F, 0, sizeof(F)); F.o = o; F.p = p;
  if (flatten(&F) != 0) return -2;
  prior_set S; memset(&S, 0, sizeof(S));
  S.loss = pr ? pr->loss_function_type : 0; S.scale = pr ? pr->loss_function_scale : 1.0;
  S.pi = (int*)malloc(sizeof(int) * (npr + 1)); S.si = (int*)malloc(sizeof(int) * (npr + 1));
  S.po = (int*)malloc(sizeof(int) * (npr + 1)); S.so = (int*)malloc(sizeof(int) * (npr + 1));
  S.c = (double*)malloc(sizeof(double) * (3 * npr + 1)); S.W = (double*)malloc(sizeof(double) * (9 * npr + 1));
  S.J = (double*)calloc(36 * npr + 1, sizeof(double)); S.r = (double*)calloc(3 * npr + 1, sizeof(double)); S.cost = (double*)calloc(npr + 1, sizeof(double));
  for (int k = 0; k < npr; ++k) {
    const int pi = pr->pose_idx[k], si = pr->sensor_idx ? pr->sensor_idx[k] : -1;
    const int po = F.pose_off[pi], so = si >= 0 ? F.sens_off[si] : -1;
    if (po < 0 && so < 0) continue;
    if (!weight_of(pr->covariance + 9 * k, S.W + 9 * S.n)) return -2;
    S.pi[S.n] = pi; S.si[S.n] = si; S.po[S.n] = po; S.so[S.n] = so;
    memcpy(S.c + 3 * S.n, pr->position + 3 * k, 24);
    S.n++;
  }
  sum->num_residuals = (int)(2 * F.nobs) + 3 * S.n;
  int64_t ncamparams = 0;
  for (int c = 0; c < p->num_cameras; ++c) { const int e = p->camera_param_offset[c] + model_num_params(p->camera_model_id[c]); if (e > ncamparams) ncamparams = e; }
  int neff = 0;
  for (int i = 0; i < p->num_poses; ++i) if (F.pose_off[i] >= 0) neff += __builtin_popcount(F.pose_mask[i]);
  for (int c = 0; c < p->num_cameras; ++c) neff += F.cam_nvar[c];
  for (int k = 0; k < p->num_sensors; ++k) if (F.sens_off[k] >= 0) neff += 6;
  neff += (int)(3 * F.nvpt);
  sum->num_effective_parameters = neff;
  int lst = o->linear_solver_type;
  if (lst == B200BA_AUTO) {
    int nimg = p->num_config_images;
    if (nimg <= 0) {
      unsigned char* used = (unsigned char*)calloc((size_t)p->num_poses + 1, 1);
      for (int64_t i = 0; i < p->num_observations; ++i) used[p->obs_pose_idx[i]] = 1;
      for (int i = 0; i < p->num_poses; ++i) nimg += used[i];
      free(used);
    }
    lst = nimg <= 50 ? B200BA_DENSE_SCHUR : (nimg <= 1000 ? B200BA_SPARSE_SCHUR : B200BA_ITERATIVE_SCHUR);
  }
  sum->linear_solver_type_used = lst;
  if (F.nobs == 0 || neff == 0) { sum->termination_type = B200BA_CONVERGENCE; sum->num_residuals = (int)(2 * F.nobs); return 0; }

  const int nc = F.nc; const int64_t np3 = 3 * F.nvpt;
  double* poses = (double*)malloc(sizeof(double) * 7 * p->num_poses); memcpy(poses, p->poses, sizeof(double) * 7 * p->num_poses);
  double* cams = (double*)malloc(sizeof(double) * (ncamparams + 1)); memcpy(cams, p->camera_params, sizeof(double) * ncamparams);
  double* pts = (double*)malloc(sizeof(double) * 3 * p->num_points); memcpy(pts, p->points, sizeof(double) * 3 * p->num_points);
  for (int i = 0; i < p->num_poses; ++i) if (F.pose_off[i] >= 0) { double* q = poses + 7 * i; const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]); for (int k = 0; k < 4; ++k) q[k] /= n; }
  double* sens = (double*)malloc(sizeof(double) * (7 * p->num_sensors + 1)); double* nsens = (double*)malloc(sizeof(double) * (7 * p->num_sensors + 1));
  if (p->num_sensors) memcpy(sens, p->sensor_from_rig, sizeof(double) * 7 * p->num_sensors);
  for (int i = 0; i < p->num_sensors; ++i) if (F.sens_off[i] >= 0) { double* q = sens + 7 * i; const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]); for (int k = 0; k < 4; ++k) q[k] /= n; }
  double* nposes = (double*)malloc(sizeof(double) * 7 * p->num_poses);
  double* ncams = (double*)malloc(sizeof(double) * (ncamparams + 1));
  double* npts = (double*)malloc(sizeof(double) * 3 * p->num_points);
  double* gc = (double*)malloc(sizeof(double) * (nc + 1)); double* gp = (double*)malloc(sizeof(double) * (np3 + 1));
  double* dc = (double*)malloc(sizeof(double) * (nc + 1)); double* dp = (double*)malloc(sizeof(double) * (np3 + 1));
  double* rhs = (double*)malloc(sizeof(double) * (nc + 1));
  ba_lin L; L.Hpp_inv = (double*)malloc(sizeof(double) * (9 * F.nvpt + 1)); L.Dc2 = (double*)malloc(sizeof(double) * (nc + 1)); L.Dp2 = (double*)malloc(sizeof(double) * (np3 + 1));
  double* diag_c = (double*)malloc(sizeof(double) * (nc + 1)); double* diag_p = (double*)malloc(sizeof(double) * (np3 + 1));
  int nblk = 0; int* blk_start = (int*)malloc(sizeof(int) * (p->num_poses + p->num_sensors + p->num_cameras + 2)); int* blk_pack = (int*)malloc(sizeof(int) * (p->num_poses + p->num_sensors + p->num_cameras + 2));
  { int pk = 0;
    for (int i = 0; i < p->num_poses; ++i) if (F.pose_off[i] >= 0) { blk_start[nblk] = F.pose_off[i]; blk_pack[nblk] = pk; pk += 36; nblk++; }
    for (int i = 0; i < p->num_sensors; ++i) if (F.sens_off[i] >= 0) { blk_start[nblk] = F.sens_off[i]; blk_pack[nblk] = pk; pk += 36; nblk++; }
    for (int c = 0; c < p->num_cameras; ++c) if (F.cam_off[c] >= 0) { blk_start[nblk] = F.cam_off[c]; blk_pack[nblk] = pk; pk += F.cam_nvar[c] * F.cam_nvar[c]; nblk++; }
    blk_start[nblk] = nc; blk_pack[nblk] = pk; }

  double cost = linearize_all(&F, &S, poses, sens, cams, pts, 1);
  sum->initial_cost = cost;
  double radius = o->initial_trust_region_radius, decrease_factor = 2.0;
  int iter = 0, have_scale = 0;
  sum->termination_type = B200BA_NO_CONVERGENCE;
  for (;;) {
    if (!have_scale) {   /* jacobi scaling over every residual row, the priors' included */
      for (int i = 0; i < nc; ++i) F.scale_c[i] = 0; for (int64_t i = 0; i < np3; ++i) F.scale_p[i] = 0;
      for (int64_t j = 0; j < F.nobs; ++j) {
        obs_blk B; obs_blocks(&F, j, &B); const double* Jc = F.Jc + 2 * JC * j;
        for (int w = 0; w < 3; ++w)
          if (B.off[w] >= 0) for (int c = 0; c < B.n[w]; ++c) F.scale_c[B.off[w] + c] += Jc[B.jo[w] + c] * Jc[B.jo[w] + c] + Jc[JC + B.jo[w] + c] * Jc[JC + B.jo[w] + c];
      }
      for (int k = 0; k < S.n; ++k)
        for (int j = 0; j < 12; ++j) { const int col = col_of(&S, k, j); const double* J = S.J + 36 * k; if (col >= 0) F.scale_c[col] += J[j] * J[j] + J[12 + j] * J[12 + j] + J[24 + j] * J[24 + j]; }
      for (int64_t k = 0; k < F.nvpt; ++k)
        for (int64_t j = F.pt_start[k]; j < F.pt_start[k + 1]; ++j) { const double* Jp = F.Jp + 6 * j; for (int c = 0; c < 3; ++c) F.scale_p[3 * k + c] += Jp[c] * Jp[c] + Jp[3 + c] * Jp[3 + c]; }
      for (int i = 0; i < nc; ++i) F.scale_c[i] = o->jacobi_scaling ? 1.0 / (1.0 + sqrt(F.scale_c[i])) : 1.0;
      for (int64_t i = 0; i < np3; ++i) F.scale_p[i] = o->jacobi_scaling ? 1.0 / (1.0 + sqrt(F.scale_p[i])) : 1.0;
      have_scale = 1;
    }
    memset(gc, 0, sizeof(double) * nc); memset(gp, 0, sizeof(double) * np3);
    memset(diag_c, 0, sizeof(double) * nc); memset(diag_p, 0, sizeof(double) * np3);
    for (int64_t j = 0; j < F.nobs; ++j) {
      jct_times_add(&F, j, F.r + 2 * j, gc);
      obs_blk B; obs_blocks(&F, j, &B); const double* Jc = F.Jc + 2 * JC * j;
      for (int w = 0; w < 3; ++w)
        if (B.off[w] >= 0) for (int c = 0; c < B.n[w]; ++c) { const double sc = F.scale_c[B.off[w] + c]; diag_c[B.off[w] + c] += sc * sc * (Jc[B.jo[w] + c] * Jc[B.jo[w] + c] + Jc[JC + B.jo[w] + c] * Jc[JC + B.jo[w] + c]); }
    }
    for (int k = 0; k < S.n; ++k) {
      prior_t_times_add(&F, &S, k, S.r + 3 * k, gc);
      for (int j = 0; j < 12; ++j) { const int col = col_of(&S, k, j); const double* J = S.J + 36 * k; if (col >= 0) diag_c[col] += F.scale_c[col] * F.scale_c[col] * (J[j] * J[j] + J[12 + j] * J[12 + j] + J[24 + j] * J[24 + j]); }
    }
    for (int64_t pv = 0; pv < F.nvpt; ++pv)
      for (int64_t j = F.pt_start[pv]; j < F.pt_start[pv + 1]; ++j) {
        const double* Jp = F.Jp + 6 * j;
        for (int c = 0; c < 3; ++c) {
          const double s = F.scale_p[3 * pv + c];
          gp[3 * pv + c] += s * (Jp[c] * F.r[2 * j] + Jp[3 + c] * F.r[2 * j + 1]);
          diag_p[3 * pv + c] += s * s * (Jp[c] * Jp[c] + Jp[3 + c] * Jp[3 + c]);
        }
      }
    {
      double* ugc = dc; double* ugp = dp;
      for (int i = 0; i < nc; ++i) ugc[i] = gc[i] / F.scale_c[i];
      for (int64_t i = 0; i < np3; ++i) ugp[i] = gp[i] / F.scale_p[i];
      if (gradient_max_norm(&F, poses, sens, ugc, ugp) <= o->gradient_tolerance) { sum->termination_type = B200BA_CONVERGENCE; break; }
    }
    int accepted = 0;
    while (!accepted) {
      if (iter >= o->max_num_iterations) goto done;
      ++iter;
      for (int i = 0; i < nc; ++i) L.Dc2[i] = fmin(fmax(diag_c[i], o->min_lm_diagonal), o->max_lm_diagonal) / radius;
      for (int64_t i = 0; i < np3; ++i) L.Dp2[i] = fmin(fmax(diag_p[i], o->min_lm_diagonal), o->max_lm_diagonal) / radius;
      int ok = 1;
      for (int64_t k = 0; k < F.nvpt; ++k) {
        double H[9] = {0};
        for (int64_t j = F.pt_start[k]; j < F.pt_start[k + 1]; ++j) {
          const double* Jp = F.Jp + 6 * j;
          for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) H[3 * a + b] += F.scale_p[3 * k + a] * F.scale_p[3 * k + b] * (Jp[a] * Jp[b] + Jp[3 + a] * Jp[3 + b]);
        }
        for (int a = 0; a < 3; ++a) H[4 * a] += L.Dp2[3 * k + a];
        if (!chol3_inv(H, L.Hpp_inv + 9 * k)) ok = 0;
      }
      for (int i = 0; i < nc; ++i) rhs[i] = -gc[i];
      for (int64_t k = 0; k < F.nvpt; ++k) {
        const double* Hi = L.Hpp_inv + 9 * k; double w[3];
        for (int c = 0; c < 3; ++c) w[c] = Hi[3 * c] * gp[3 * k] + Hi[3 * c + 1] * gp[3 * k + 1] + Hi[3 * c + 2] * gp[3 * k + 2];
        for (int64_t j = F.pt_start[k]; j < F.pt_start[k + 1]; ++j) {
          const double* Jp = F.Jp + 6 * j; double u[2];
          for (int r = 0; r < 2; ++r) { double t = 0; for (int c = 0; c < 3; ++c) t += Jp[3 * r + c] * F.scale_p[3 * k + c] * w[c]; u[r] = t; }
          jct_times_add(&F, j, u, rhs);
        }
      }
      memset(dc, 0, sizeof(double) * nc);
      if (ok && nc > 0) {
        if (lst != B200BA_ITERATIVE_SCHUR) {
          double* Sm = (double*)malloc(sizeof(double) * (size_t)nc * nc); double* e = (double*)calloc(nc, sizeof(double)); double* col = (double*)malloc(sizeof(double) * nc);
          for (int i = 0; i < nc; ++i) { e[i] = 1.0; schur_apply_all(&F, &S, &L, e, col); e[i] = 0.0; for (int r = 0; r < nc; ++r) Sm[(size_t)r * nc + i] = col[r]; }
          memcpy(dc, rhs, sizeof(double) * nc);
          ok = chol_solve(nc, Sm, dc);
          free(Sm); free(e); free(col);
        } else {
          double* Minv = (double*)malloc(sizeof(double) * (blk_pack[nblk] + 1));
          schur_jacobi_all(&F, &S, &L, blk_start, nblk, Minv, blk_pack);
          double *r = (double*)malloc(sizeof(double) * nc), *z = (double*)malloc(sizeof(double) * nc), *pv = (double*)malloc(sizeof(double) * nc), *q = (double*)malloc(sizeof(double) * nc);
          memcpy(r, rhs, sizeof(double) * nc);
          double norm_b = 0; for (int i = 0; i < nc; ++i) norm_b += rhs[i] * rhs[i]; norm_b = sqrt(norm_b);
          double rho = 1.0, Q0 = 0.0;
          if (norm_b > 0) for (int it = 1; it <= o->max_linear_solver_iterations; ++it) {
            for (int b = 0; b < nblk; ++b) { const int n = blk_start[b + 1] - blk_start[b]; const double* Mb = Minv + blk_pack[b];
              for (int rr = 0; rr < n; ++rr) { double t = 0; for (int c = 0; c < n; ++c) t += Mb[rr * n + c] * r[blk_start[b] + c]; z[blk_start[b] + rr] = t; } }
            const double last_rho = rho; rho = 0; for (int i = 0; i < nc; ++i) rho += r[i] * z[i];
            if (it == 1) memcpy(pv, z, sizeof(double) * nc); else { const double beta = rho / last_rho; for (int i = 0; i < nc; ++i) pv[i] = z[i] + beta * pv[i]; }
            schur_apply_all(&F, &S, &L, pv, q);
            double pq = 0; for (int i = 0; i < nc; ++i) pq += pv[i] * q[i];
            if (!(pq > 0)) break;
            const double alpha = rho / pq;
            for (int i = 0; i < nc; ++i) { dc[i] += alpha * pv[i]; r[i] -= alpha * q[i]; }
            sum->num_linear_solver_iterations++;
            double Q1 = 0; for (int i = 0; i < nc; ++i) Q1 += dc[i] * (rhs[i] + r[i]); Q1 = -1.0 * Q1;
            const double zeta = it * (Q1 - Q0) / Q1;
            if (zeta < o->eta) break;
            Q0 = Q1;
            double nr = 0; for (int i = 0; i < nc; ++i) nr += r[i] * r[i];
            if (sqrt(nr) <= 1e-300) break;
          }
          free(Minv); free(r); free(z); free(pv); free(q);
        }
      }
      for (int64_t k = 0; k < F.nvpt; ++k) {
        double t[3] = {-gp[3 * k], -gp[3 * k + 1], -gp[3 * k + 2]};
        for (int64_t j = F.pt_start[k]; j < F.pt_start[k + 1]; ++j) {
          double y[2]; jc_times(&F, j, dc, y); const double* Jp = F.Jp + 6 * j;
          for (int c = 0; c < 3; ++c) t[c] -= F.scale_p[3 * k + c] * (Jp[c] * y[0] + Jp[3 + c] * y[1]);
        }
        const double* Hi = L.Hpp_inv + 9 * k;
        for (int c = 0; c < 3; ++c) dp[3 * k + c] = Hi[3 * c] * t[0] + Hi[3 * c + 1] * t[1] + Hi[3 * c + 2] * t[2];
      }
      double model = 0;
      for (int64_t j = 0; j < F.nobs; ++j) {
        double y[2]; jc_times(&F, j, dc, y);
        if (j < F.nobs_var) { const int64_t pv = F.pt_var[p->obs_point_idx[F.obs[j]]]; const double* Jp = F.Jp + 6 * j;
          for (int r = 0; r < 2; ++r) for (int c = 0; c < 3; ++c) y[r] += Jp[3 * r + c] * F.scale_p[3 * pv + c] * dp[3 * pv + c]; }
        model -= y[0] * (F.r[2 * j] + 0.5 * y[0]) + y[1] * (F.r[2 * j + 1] + 0.5 * y[1]);
      }
      for (int k = 0; k < S.n; ++k) { double y[3]; prior_times(&F, &S, k, dc, y); const double* r = S.r + 3 * k; model -= y[0] * (r[0] + 0.5 * y[0]) + y[1] * (r[1] + 0.5 * y[1]) + y[2] * (r[2] + 0.5 * y[2]); }
      double rho_q = 0.0, new_cost = cost;
      if (ok && model > 0) {
        double* udc = (double*)malloc(sizeof(double) * (nc + 1)); double* udp = (double*)malloc(sizeof(double) * (np3 + 1));
        for (int i = 0; i < nc; ++i) udc[i] = dc[i] * F.scale_c[i];
        for (int64_t i = 0; i < np3; ++i) udp[i] = dp[i] * F.scale_p[i];
        apply_step(&F, poses, sens, cams, pts, udc, udp, nposes, nsens, ncams, npts, ncamparams);
        free(udc); free(udp);
        new_cost = linearize_all(&F, &S, nposes, nsens, ncams, npts, 0);
        rho_q = (-F.cost_delta) / model;
      }
      if (getenv("BA_ORACLE_VERBOSE")) fprintf(stderr, "[prior oracle] it %d cost %.12g new %.12g model %.6g rho %.6g radius %.4g pcg_total %d\n", iter, cost, new_cost, model, rho_q, radius, sum->num_linear_solver_iterations);
      if (ok && model > 0 && rho_q > o->min_relative_decrease) {
        accepted = 1;
        sum->num_successful_steps++;
        memcpy(poses, nposes, sizeof(double) * 7 * p->num_poses); memcpy(cams, ncams, sizeof(double) * ncamparams); memcpy(pts, npts, sizeof(double) * 3 * p->num_points);
        memcpy(sens, nsens, sizeof(double) * 7 * p->num_sensors);
        const double cost_change = -F.cost_delta;
        cost = linearize_all(&F, &S, poses, sens, cams, pts, 1);
        const double t = 2.0 * rho_q - 1.0;
        radius = radius / fmax(1.0 / 3.0, 1.0 - t * t * t);
        radius = fmin(o->max_trust_region_radius, radius);
        decrease_factor = 2.0;
        if (fabs(cost_change) <= o->function_tolerance * cost) { sum->termination_type = B200BA_CONVERGENCE; goto done; }
      } else {
        sum->num_unsuccessful_steps++;
        radius = radius / decrease_factor;
        decrease_factor *= 2.0;
        if (radius < o->min_trust_region_radius) { sum->termination_type = B200BA_CONVERGENCE; goto done; }
      }
    }
  }
done:
  sum->final_cost = cost;
  for (int i = 0; i < p->num_poses; ++i) if (F.pose_off[i] >= 0) memcpy(p->poses + 7 * i, poses + 7 * i, 56);
  for (int i = 0; i < p->num_sensors; ++i) if (F.sens_off[i] >= 0) memcpy(p->sensor_from_rig + 7 * i, sens + 7 * i, 56);
  for (int c = 0; c < p->num_cameras; ++c) if (F.cam_off[c] >= 0) for (int k = 0; k < F.cam_nvar[c]; ++k) { const int idx = p->camera_param_offset[c] + F.cam_var[c][k]; p->camera_params[idx] = cams[idx]; }
  for (int64_t i = 0; i < p->num_points; ++i) if (F.pt_var[i] >= 0) memcpy(p->points + 3 * i, pts + 3 * i, 24);
  free(sens); free(nsens); free(F.sens_off);
  free(poses); free(cams); free(pts); free(nposes); free(ncams); free(npts); free(gc); free(gp); free(dc); free(dp); free(rhs);
  free(L.Hpp_inv); free(L.Dc2); free(L.Dp2); free(diag_c); free(diag_p); free(blk_start); free(blk_pack);
  free(F.pose_off); free(F.pose_mask); free(F.cam_off); free(F.cam_nvar); free(F.cam_var); free(F.pt_var); free(F.obs); free(F.pt_start);
  free(F.cost_obs); free(F.r); free(F.Jc); free(F.Jp); free(F.scale_c); free(F.scale_p);
  free(S.pi); free(S.si); free(S.po); free(S.so); free(S.c); free(S.W); free(S.J); free(S.r); free(S.cost);
  return 0;
}
