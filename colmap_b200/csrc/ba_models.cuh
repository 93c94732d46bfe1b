// ba_models.cuh — camera models with MORE than five parameters, as formulas only, differentiated by forward-mode dual
// numbers that live in registers (SURVEY.md section 8f rank 4).  The solve and the covariance estimate evaluate these
// models in every WIDE linearisation (ba_img_from_cam_any / ba_residual_any in ba_common.cuh); the <= 5-parameter
// models keep their hand-written Jacobians.  The CPU test hook b200ba_test_project_wide evaluates them on the host.
//
// Reference behaviour: ImgFromCam of the twelve models COLMAP has beyond the radial pinhole family - OPENCV,
// OPENCV_FISHEYE, FULL_OPENCV, FOV, THIN_PRISM_FISHEYE, RAD_TAN_THIN_PRISM_FISHEYE, SIMPLE_DIVISION, DIVISION,
// SIMPLE_FISHEYE, FISHEYE, EUCM, EQUIRECTANGULAR (src/colmap/sensor/models.h:1513-2880; FisheyeFromNormal :429-438;
// depth guard :281-285).  The reference carries ~1200 lines of hand-derived Jacobians for these models
// (sensor/models_jacobian.h:401-1565); here the derivative falls out of the value computation, the same source works on
// the host and on the device, and a new model is ten lines.
#pragma once
#include <math.h>

#ifndef BA_HD
#define BA_HD __host__ __device__ __forceinline__
#endif

template <int N>
struct BaDual {
  double v;
  double d[N];
  BA_HD BaDual() : v(0.0) { for (int i = 0; i < N; ++i) d[i] = 0.0; }
  BA_HD BaDual(double x) : v(x) { for (int i = 0; i < N; ++i) d[i] = 0.0; }   // constant
  BA_HD static BaDual variable(double x, int k) { BaDual r(x); r.d[k] = 1.0; return r; }
};
template <int N> BA_HD BaDual<N> operator+(const BaDual<N>& a, const BaDual<N>& b) { BaDual<N> r; r.v = a.v + b.v; for (int i = 0; i < N; ++i) r.d[i] = a.d[i] + b.d[i]; return r; }
template <int N> BA_HD BaDual<N> operator-(const BaDual<N>& a, const BaDual<N>& b) { BaDual<N> r; r.v = a.v - b.v; for (int i = 0; i < N; ++i) r.d[i] = a.d[i] - b.d[i]; return r; }
template <int N> BA_HD BaDual<N> operator-(const BaDual<N>& a) { BaDual<N> r; r.v = -a.v; for (int i = 0; i < N; ++i) r.d[i] = -a.d[i]; return r; }
template <int N> BA_HD BaDual<N> operator*(const BaDual<N>& a, const BaDual<N>& b) { BaDual<N> r; r.v = a.v * b.v; for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * b.v + a.v * b.d[i]; return r; }
template <int N> BA_HD BaDual<N> operator/(const BaDual<N>& a, const BaDual<N>& b) {
  BaDual<N> r; const double ib = 1.0 / b.v; r.v = a.v * ib;
  for (int i = 0; i < N; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) * ib;
  return r;
}
template <int N> BA_HD BaDual<N> ba_sqrt(const BaDual<N>& a) { BaDual<N> r; r.v = sqrt(a.v); const double s = 0.5 / r.v; for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * s; return r; }
template <int N> BA_HD BaDual<N> ba_atan(const BaDual<N>& a) { BaDual<N> r; r.v = atan(a.v); const double s = 1.0 / (1.0 + a.v * a.v); for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * s; return r; }
template <int N> BA_HD BaDual<N> ba_tan(const BaDual<N>& a) { BaDual<N> r; r.v = tan(a.v); const double s = 1.0 + r.v * r.v; for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * s; return r; }
template <int N> BA_HD BaDual<N> ba_atan2(const BaDual<N>& y, const BaDual<N>& x) {
  BaDual<N> r; r.v = atan2(y.v, x.v); const double s = 1.0 / (x.v * x.v + y.v * y.v);
  for (int i = 0; i < N; ++i) r.d[i] = (x.v * y.d[i] - y.v * x.d[i]) * s;
  return r;
}
BA_HD double ba_atan2(double y, double x) { return atan2(y, x); }
BA_HD double ba_sqrt(double a) { return sqrt(a); }
BA_HD double ba_atan(double a) { return atan(a); }
BA_HD double ba_tan(double a) { return tan(a); }
template <int N> BA_HD double ba_value(const BaDual<N>& a) { return a.v; }
BA_HD double ba_value(double a) { return a; }

BA_HD int ba_wide_model_num_params(int id) {
  switch (id) {
    case 4: case 5: return 8;      // OPENCV, OPENCV_FISHEYE
    case 6: case 10: return 12;    // FULL_OPENCV, THIN_PRISM_FISHEYE
    case 7: case 13: return 5;     // FOV, DIVISION
    case 11: return 16;            // RAD_TAN_THIN_PRISM_FISHEYE
    case 12: case 15: return 4;    // SIMPLE_DIVISION, FISHEYE
    case 14: return 3;             // SIMPLE_FISHEYE
    case 16: return 6;             // EUCM
    case 17: return 2;             // EQUIRECTANGULAR
    default: return -1;
  }
}

// equidistant fisheye mapping of the normalised point (identity for r -> 0)
template <typename S>
BA_HD void ba_fisheye_from_normal(const S& a, const S& b, S* fa, S* fb) {
  const S r = ba_sqrt(a * a + b * b);
  if (ba_value(r) > 2.220446049250313e-16) { const S s = ba_atan(r) / r; *fa = a * s; *fb = b * s; }
  else { *fa = a; *fb = b; }
}

// q: parameters (as S), (u, v, w): point in the camera frame; false if the depth guard fails
template <typename S>
BA_HD bool ba_project_wide(int id, const S* q, const S& u, const S& v, const S& w, S* x, S* y) {
  const S two(2.0), one(1.0);
  if (id == 12 || id == 13) {   // SIMPLE_DIVISION f cx cy k / DIVISION fx fy cx cy k: no depth guard, negative discriminant fails
    const S k = id == 12 ? q[3] : q[4];
    const S disc_sq = w * w - S(4.0) * (u * u + v * v) * k;
    if (ba_value(disc_sq) < 0.0) return false;
    const S r = two / (w + ba_sqrt(disc_sq));
    if (id == 12) { *x = q[0] * r * u + q[1]; *y = q[0] * r * v + q[2]; }
    else { *x = q[0] * r * u + q[2]; *y = q[1] * r * v + q[3]; }
    return true;
  }
  if (id == 17) {               // EQUIRECTANGULAR width height: azimuth / elevation of the ray, defined on the whole sphere
    const S horizontal = ba_sqrt(u * u + w * w);
    if (ba_value(horizontal) + fabs(ba_value(v)) < 2.220446049250313e-16) return false;
    const S theta = ba_atan2(u, w), phi = ba_atan2(-v, horizontal);
    *x = (theta / S(6.283185307179586476925286766559) + S(0.5)) * q[0];
    *y = (S(0.5) - phi / S(3.14159265358979323846264338327950288)) * q[1];
    return true;
  }
  if (!(ba_value(w) >= 2.220446049250313e-16)) return false;
  if (id == 16) {               // EUCM fx fy cx cy alpha beta
    const S rho2 = q[5] * (u * u + v * v) + w * w;
    if (ba_value(rho2) < 0.0) return false;
    const S den = q[4] * ba_sqrt(rho2) + (one - q[4]) * w;
    if (!(ba_value(den) >= 2.220446049250313e-16)) return false;
    *x = q[0] * (u / den) + q[2]; *y = q[1] * (v / den) + q[3];
    return true;
  }
  const S a = u / w, b = v / w;
  if (id == 14 || id == 15) {   // SIMPLE_FISHEYE f cx cy / FISHEYE fx fy cx cy: equidistant mapping, no distortion
    S fa, fb; ba_fisheye_from_normal(a, b, &fa, &fb);
    if (id == 14) { *x = q[0] * fa + q[1]; *y = q[0] * fb + q[2]; }
    else { *x = q[0] * fa + q[2]; *y = q[1] * fb + q[3]; }
    return true;
  }
  if (id == 11) {               // RAD_TAN_THIN_PRISM_FISHEYE fx fy cx cy k0..k5 p0 p1 s0..s3
    S fa, fb; ba_fisheye_from_normal(a, b, &fa, &fb);
    const S t2 = fa * fa + fb * fb;
    S radial = one, power = one;
    for (int i = 0; i < 6; ++i) { power = power * t2; radial = radial + q[4 + i] * power; }
    const S px = radial * fa, py = radial * fb;
    const S x2 = px * px, y2 = py * py, xy = px * py, r2 = x2 + y2, r4 = r2 * r2;
    const S xd = px + (two * q[11] * xy + q[10] * (r2 + two * x2)) + (q[12] * r2 + q[13] * r4);
    const S yd = py + (two * q[10] * xy + q[11] * (r2 + two * y2)) + (q[14] * r2 + q[15] * r4);
    *x = q[0] * xd + q[2]; *y = q[1] * yd + q[3];
    return true;
  }
  if (id == 4) {          // OPENCV: fx fy cx cy k1 k2 p1 p2
    const S a2 = a * a, ab = a * b, b2 = b * b, r2 = a2 + b2, radial = q[4] * r2 + q[5] * r2 * r2;
    const S du = a * radial + two * q[6] * ab + q[7] * (r2 + two * a2);
    const S dv = b * radial + two * q[7] * ab + q[6] * (r2 + two * b2);
    *x = q[0] * (a + du) + q[2]; *y = q[1] * (b + dv) + q[3];
  } else if (id == 5) {   // OPENCV_FISHEYE: fx fy cx cy k1 k2 k3 k4
    S fa, fb; ba_fisheye_from_normal(a, b, &fa, &fb);
    const S t2 = fa * fa + fb * fb, t4 = t2 * t2, t6 = t4 * t2, t8 = t4 * t4;
    const S radial = q[4] * t2 + q[5] * t4 + q[6] * t6 + q[7] * t8;
    *x = q[0] * (fa + fa * radial) + q[2]; *y = q[1] * (fb + fb * radial) + q[3];
  } else if (id == 6) {   // FULL_OPENCV: fx fy cx cy k1 k2 p1 p2 k3 k4 k5 k6
    const S a2 = a * a, ab = a * b, b2 = b * b, r2 = a2 + b2, r4 = r2 * r2, r6 = r4 * r2;
    const S radial = (one + q[4] * r2 + q[5] * r4 + q[8] * r6) / (one + q[9] * r2 + q[10] * r4 + q[11] * r6);
    const S xd = a * radial + two * q[6] * ab + q[7] * (r2 + two * a2);
    const S yd = b * radial + two * q[7] * ab + q[6] * (r2 + two * b2);
    *x = q[0] * xd + q[2]; *y = q[1] * yd + q[3];
  } else if (id == 7) {   // FOV: fx fy cx cy omega
    const S omega = q[4], r2 = a * a + b * b, o2 = omega * omega;
    S factor;
    if (ba_value(o2) < 1e-4) factor = (o2 * r2) / S(3.0) - o2 / S(12.0) + one;
    else if (ba_value(r2) < 1e-4) { const S t = ba_tan(omega / two); factor = (S(-2.0) * t * (S(4.0) * r2 * t * t - S(3.0))) / (S(3.0) * omega); }
    else { const S r = ba_sqrt(r2); factor = ba_atan(r * two * ba_tan(omega / two)) / (r * omega); }
    *x = q[0] * (a * factor) + q[2]; *y = q[1] * (b * factor) + q[3];
  } else if (id == 10) {  // THIN_PRISM_FISHEYE: fx fy cx cy k1 k2 p1 p2 k3 k4 sx1 sy1
    S fa, fb; ba_fisheye_from_normal(a, b, &fa, &fb);
    const S a2 = fa * fa, ab = fa * fb, b2 = fb * fb, r2 = a2 + b2, r4 = r2 * r2, r6 = r4 * r2, r8 = r6 * r2;
    const S radial = q[4] * r2 + q[5] * r4 + q[8] * r6 + q[9] * r8;
    const S du = fa * radial + two * q[6] * ab + q[7] * (r2 + two * a2) + q[10] * r2;
    const S dv = fb * radial + two * q[7] * ab + q[6] * (r2 + two * b2) + q[11] * r2;
    *x = q[0] * (fa + du) + q[2]; *y = q[1] * (fb + dv) + q[3];
  } else {
    return false;
  }
  return true;
}

// value + Jacobians wrt (u, v, w) [2x3] and the P parameters [2xP], all in one pass of duals with 3 + P derivative slots
template <int P>
BA_HD bool ba_project_wide_with_jac(int id, const double* params, double u, double v, double w, double* xy, double* J_uvw,
                                    double* J_params) {
  typedef BaDual<3 + P> D;
  D q[P];
  for (int k = 0; k < P; ++k) q[k] = D::variable(params[k], 3 + k);
  D x, y;
  if (!ba_project_wide<D>(id, q, D::variable(u, 0), D::variable(v, 1), D::variable(w, 2), &x, &y)) return false;
  xy[0] = x.v; xy[1] = y.v;
  for (int c = 0; c < 3; ++c) { J_uvw[c] = x.d[c]; J_uvw[3 + c] = y.d[c]; }
  for (int k = 0; k < P; ++k) { J_params[k] = x.d[3 + k]; J_params[P + k] = y.d[3 + k]; }
  return true;
}
