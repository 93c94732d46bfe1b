// cam_rays.cuh — CamRayFromImg of the eighteen camera models on the host (sensor/models.h), shared by the global
// positioner (b200gp_cam_ray_from_img) and guided SIFT matching (b200sm_cam_ray_from_img_with_jac).
#pragma once
#include <float.h>
#include <math.h>

#include <algorithm>

#include "ba_models.cuh"

// Distortion(extra_params, u, v) of the models that undistort iteratively (sensor/models.h), in dual numbers so that
// the Newton step of IterativeUndistortion (models.h:1141-1190) gets its Jacobian.
template <typename S>
static bool gp_distortion(int id, const double* e, const S& u, const S& v, S* du, S* dv) {
  const S two(2.0);
  if (id == 2 || id == 8) {            // SIMPLE_RADIAL(_FISHEYE): k
    const S r = S(e[0]) * (u * u + v * v); *du = u * r; *dv = v * r;
  } else if (id == 3 || id == 9) {     // RADIAL(_FISHEYE): k1 k2
    const S r2 = u * u + v * v, r = S(e[0]) * r2 + S(e[1]) * r2 * r2; *du = u * r; *dv = v * r;
  } else if (id == 4) {                // OPENCV: k1 k2 p1 p2
    const S u2 = u * u, uv = u * v, v2 = v * v, r2 = u2 + v2, r = S(e[0]) * r2 + S(e[1]) * r2 * r2;
    *du = u * r + two * S(e[2]) * uv + S(e[3]) * (r2 + two * u2);
    *dv = v * r + two * S(e[3]) * uv + S(e[2]) * (r2 + two * v2);
  } else if (id == 5) {                // OPENCV_FISHEYE: k1..k4 on the fisheye coordinates
    const S t2 = u * u + v * v, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
    const S r = S(e[0]) * t2 + S(e[1]) * t4 + S(e[2]) * t6 + S(e[3]) * t8; *du = u * r; *dv = v * r;
  } else if (id == 6) {                // FULL_OPENCV: k1 k2 p1 p2 k3 k4 k5 k6
    const S u2 = u * u, uv = u * v, v2 = v * v, r2 = u2 + v2, r4 = r2 * r2, r6 = r4 * r2;
    const S r = (S(1.0) + S(e[0]) * r2 + S(e[1]) * r4 + S(e[4]) * r6) / (S(1.0) + S(e[5]) * r2 + S(e[6]) * r4 + S(e[7]) * r6);
    *du = u * r + two * S(e[2]) * uv + S(e[3]) * (r2 + two * u2) - u;
    *dv = v * r + two * S(e[3]) * uv + S(e[2]) * (r2 + two * v2) - v;
  } else if (id == 10) {               // THIN_PRISM_FISHEYE: k1 k2 p1 p2 k3 k4 sx1 sy1
    const S u2 = u * u, uv = u * v, v2 = v * v, r2 = u2 + v2, r4 = r2 * r2, r6 = r4 * r2, r8 = r6 * r2;
    const S r = S(e[0]) * r2 + S(e[1]) * r4 + S(e[4]) * r6 + S(e[5]) * r8;
    *du = u * r + two * S(e[2]) * uv + S(e[3]) * (r2 + two * u2) + S(e[6]) * r2;
    *dv = v * r + two * S(e[3]) * uv + S(e[2]) * (r2 + two * v2) + S(e[7]) * r2;
  } else if (id == 11) {               // RAD_TAN_THIN_PRISM_FISHEYE: k0..k5 p0 p1 s0..s3
    const S t2 = u * u + v * v;
    S radial(1.0), power(1.0);
    for (int i = 0; i < 6; ++i) { power = power * t2; radial = radial + S(e[i]) * power; }
    const S px = radial * u, py = radial * v;
    const S x2 = px * px, y2 = py * py, xy = px * py, r2 = x2 + y2, r4 = r2 * r2;
    *du = px + (two * S(e[7]) * xy + S(e[6]) * (r2 + two * x2)) + (S(e[8]) * r2 + S(e[9]) * r4) - u;
    *dv = py + (two * S(e[6]) * xy + S(e[7]) * (r2 + two * y2)) + (S(e[10]) * r2 + S(e[11]) * r4) - v;
  } else {
    return false;
  }
  return true;
}

static bool gp_iterative_undistortion(int id, const double* e, double* u, double* v) {
  const double x0[2] = {*u, *v};
  double x[2] = {*u, *v};
  for (int it = 0; it < 100; ++it) {
    typedef BaDual<2> D;
    D du, dv;
    gp_distortion<D>(id, e, D::variable(x[0], 0), D::variable(x[1], 1), &du, &dv);
    const double J00 = du.d[0] + 1, J01 = du.d[1], J10 = dv.d[0], J11 = dv.d[1] + 1;
    const double b0 = x[0] + du.v - x0[0], b1 = x[1] + dv.v - x0[1];
    // J.partialPivLu().solve(b) for 2x2: partial pivoting on the first column
    double s0, s1;
    if (fabs(J10) > fabs(J00)) {
      const double l = J00 / J10, u11 = J01 - l * J11;
      s1 = (b0 - l * b1) / u11; s0 = (b1 - J11 * s1) / J10;
    } else {
      const double l = J10 / J00, u11 = J11 - l * J01;
      s1 = (b1 - l * b0) / u11; s0 = (b0 - J01 * s1) / J00;
    }
    const double radius_sqr = std::max((x[0] * x[0] + x[1] * x[1]) * 0.01, 0.01);
    const double n2 = s0 * s0 + s1 * s1;
    if (n2 > radius_sqr) { const double f = sqrt(radius_sqr / n2); s0 *= f; s1 *= f; }
    x[0] -= s0; x[1] -= s1;
    if (s0 * s0 + s1 * s1 < 1e-10) { *u = x[0]; *v = x[1]; return true; }
  }
  *u = x[0]; *v = x[1];
  return false;
}

static void gp_normal_from_fisheye(double uu, double vv, double* u, double* v) {
  *u = uu; *v = vv;
  const double theta = sqrt(uu * uu + vv * vv), tct = theta * cos(theta);
  if (tct > DBL_EPSILON) { const double s = sin(theta) / tct; *u *= s; *v *= s; }
}

// CamFromImg of every model but EQUIRECTANGULAR's ray (models.h:1248-2900)
static bool gp_cam_from_img(int id, const double* p, double x, double y, double* u, double* v) {
  switch (id) {
    case 0: *u = (x - p[1]) / p[0]; *v = (y - p[2]) / p[0]; return true;
    case 1: *u = (x - p[2]) / p[0]; *v = (y - p[3]) / p[1]; return true;
    case 2: case 3: *u = (x - p[1]) / p[0]; *v = (y - p[2]) / p[0]; return gp_iterative_undistortion(id, p + 3, u, v);
    case 4: case 6: *u = (x - p[2]) / p[0]; *v = (y - p[3]) / p[1]; return gp_iterative_undistortion(id, p + 4, u, v);
    case 5: case 10: case 11: case 8: case 9: {
      const bool simple = id == 8 || id == 9;
      double uu = simple ? (x - p[1]) / p[0] : (x - p[2]) / p[0], vv = simple ? (y - p[2]) / p[0] : (y - p[3]) / p[1];
      if (!gp_iterative_undistortion(id, p + (simple ? 3 : 4), &uu, &vv)) return false;
      gp_normal_from_fisheye(uu, vv, u, v);
      return true;
    }
    case 7: {   // FOV: closed-form Undistortion (models.h:1891-1925)
      const double uu = (x - p[2]) / p[0], vv = (y - p[3]) / p[1], omega = p[4];
      const double r2 = uu * uu + vv * vv, o2 = omega * omega;
      double f;
      if (o2 < 1e-4) f = (o2 * r2) / 3.0 - o2 / 12.0 + 1.0;
      else if (r2 < 1e-4) f = (omega * (omega * omega * r2 + 3.0)) / (6.0 * tan(omega / 2.0));
      else { const double r = sqrt(r2); f = tan(r * omega) / (r * 2.0 * tan(omega / 2.0)); }
      *u = uu * f; *v = vv * f;
      return true;
    }
    case 12: case 13: {
      const bool s = id == 12;
      const double x0 = s ? (x - p[1]) / p[0] : (x - p[2]) / p[0], y0 = s ? (y - p[2]) / p[0] : (y - p[3]) / p[1];
      const double den = 1.0 + (s ? p[3] : p[4]) * (x0 * x0 + y0 * y0);
      *u = x0 / den; *v = y0 / den;
      return true;
    }
    case 14: gp_normal_from_fisheye((x - p[1]) / p[0], (y - p[2]) / p[0], u, v); return true;
    case 15: gp_normal_from_fisheye((x - p[2]) / p[0], (y - p[3]) / p[1], u, v); return true;
    case 16: {  // EUCM (models.h:2796-2830)
      *u = (x - p[2]) / p[0]; *v = (y - p[3]) / p[1];
      const double alpha = p[4], beta = p[5], r2 = *u * *u + *v * *v, gamma = 1.0 - alpha;
      const double rad = 1.0 - (alpha - gamma) * beta * r2;
      if (rad < 0) return false;
      const double hden = alpha * sqrt(rad) + gamma;
      if (hden < DBL_EPSILON) return false;
      const double h = (1.0 - alpha * alpha * beta * r2) / hden;
      if (h < DBL_EPSILON) return false;
      *u /= h; *v /= h;
      return true;
    }
    default: return false;
  }
}

// CameraModelCamRayFromImg (models.h:3029-3047): EQUIRECTANGULAR's own ray (models.h:809-829), else CamFromImg
// normalised.  false where the reference returns nullopt.
static bool cam_ray_from_img(int id, const double* p, double x, double y, double* ray) {
  if (id == 17) {
    const double theta = 2.0 * M_PI * (x / p[0] - 0.5), phi = M_PI * (0.5 - y / p[1]);
    const double cp = cos(phi);
    ray[0] = cp * sin(theta); ray[1] = -sin(phi); ray[2] = cp * cos(theta);
    return true;
  }
  double u = 0, v = 0;
  if (!gp_cam_from_img(id, p, x, y, &u, &v)) return false;
  const double n = sqrt(u * u + v * v + 1.0);
  ray[0] = u / n; ray[1] = v / n; ray[2] = 1.0 / n;
  return true;
}
