// sift_rays.cu — Camera::CamRayFromImgWithJac (scene/camera.h:355-371) on the host, for the essential-matrix filter of
// guided SIFT matching (sift_matching.cu).  The unprojection is the global positioner's (cam_rays.cuh) and the
// projection Jacobian is bundle adjustment's (ba_img_from_cam_any), so the eighteen models are written once.
#include "ba_common.cuh"
#include "cam_rays.cuh"

// out9: the unit ray, then d(ray) / d(pixel) as a row-major 3 x 2 matrix.  false where the reference returns nullopt:
// CamRayFromImg fails, ImgFromCamWithJac fails at the ray (cheirality checked), or CamRayFromImgJacobian's relative
// alpha test (models.h:2977-2997) rejects the point.
bool sm_cam_ray_with_jac(int id, const double* params, double x, double y, double* out9) {
  double ray[3];
  if (!cam_ray_from_img(id, params, x, y, ray)) return false;
  double px, py, Jp[2 * BA_MAXP], J[6];
  if (!ba_img_from_cam_any(id, params, ray[0], ray[1], ray[2], &px, &py, Jp, J)) return false;
  const double gx[3] = {J[0], J[1], J[2]}, gy[3] = {J[3], J[4], J[5]};
  const double c[3] = {gx[1] * gy[2] - gx[2] * gy[1], gx[2] * gy[0] - gx[0] * gy[2], gx[0] * gy[1] - gx[1] * gy[0]};
  const double alpha = ray[0] * c[0] + ray[1] * c[1] + ray[2] * c[2];
  const double sq = (gx[0] * gx[0] + gx[1] * gx[1] + gx[2] * gx[2]) + (gy[0] * gy[0] + gy[1] * gy[1] + gy[2] * gy[2]);
  if (!(fabs(alpha) > 1e-6 * sq)) return false;
  // column 0 = g_y x ray, column 1 = ray x g_x, both divided by alpha
  const double c0[3] = {gy[1] * ray[2] - gy[2] * ray[1], gy[2] * ray[0] - gy[0] * ray[2], gy[0] * ray[1] - gy[1] * ray[0]};
  const double c1[3] = {ray[1] * gx[2] - ray[2] * gx[1], ray[2] * gx[0] - ray[0] * gx[2], ray[0] * gx[1] - ray[1] * gx[0]};
  for (int k = 0; k < 3; ++k) {
    out9[k] = ray[k];
    out9[3 + 2 * k] = c0[k] / alpha;
    out9[4 + 2 * k] = c1[k] / alpha;
  }
  return true;
}
