// camera_radial.h -- the RADIAL camera model of the bundle adjustment with intrinsics (bundle_adjust_intrinsics.cu):
// its projection, residual and Jacobians, and the undistortion of a pixel.  COLMAP's RADIAL model, five parameters
// k = (f, cx, cy, k1, k2) per intrinsics group:
//
//   p = R X + t,  u = (p0 / p2, p1 / p2),  s = u . u,  d = 1 + k1 s + k2 s^2,  x = f d u + (cx, cy)
//
// With k1 = k2 = 0 this is the pinhole projection through K = [[f, 0, cx], [0, f, cy], [0, 0, 1]].  One focal length
// (no fx != fy) and no skew, by design.  Pose parameters are those of absolute_pose.h (ap_jacobian, ap_step).
// tests/bundle_adjust_intrinsics_np.py restates every function here in numpy, and tests/bundle_adjust_intrinsics_host.cpp
// builds this header with g++.
#pragma once
#include "common.h"

namespace dg {

constexpr int kRadParams = 5;            // f, cx, cy, k1, k2
constexpr int kRadUndistortIters = 50;   // Newton (or bisection) steps of the undistortion at most

// Intrinsics a camera can use: every parameter finite and f > 0
DG_HD bool rad_valid(const double* k) {
  bool ok = k[0] > 0.0;
#pragma unroll
  for (int i = 0; i < kRadParams; ++i) ok = ok && fabs(k[i]) < INFINITY;
  return ok;
}

// The pixel residual r [2] of camera point p observed at (x, y)
DG_HD void rad_residual(const double* k, const double* p, double x, double y, double* r) {
  const double iz = 1.0 / p[2];
  const double u0 = p[0] * iz, u1 = p[1] * iz;
  const double s = u0 * u0 + u1 * u1;
  const double fd = k[0] * (1.0 + s * (k[3] + s * k[4]));
  r[0] = fd * u0 + k[1] - x;
  r[1] = fd * u1 + k[2] - y;
}

// e^2 of an observation of X under pose P [12], and whether its depth is positive
DG_HD double rad_sq_error(const double* P, const double* k, const double* X, double x, double y, bool* front) {
  double p[3], r[2];
#pragma unroll
  for (int i = 0; i < 3; ++i) p[i] = P[3 * i] * X[0] + P[3 * i + 1] * X[1] + P[3 * i + 2] * X[2] + P[9 + i];
  rad_residual(k, p, x, y, r);
  *front = p[2] > 0.0;
  return r[0] * r[0] + r[1] * r[1];
}

// r [2], J_cam [2][6] (by w, d at zero, as ap_jacobian), J_X [2][3] and J_k [2][5] (by f, cx, cy, k1, k2)
DG_HD void rad_jacobian(const double* P, const double* k, const double* X, double x, double y, double* r, double* Jc,
                        double* Jx, double* Jk) {
  double g[3], p[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) g[i] = P[3 * i] * X[0] + P[3 * i + 1] * X[1] + P[3 * i + 2] * X[2];   // R X
#pragma unroll
  for (int i = 0; i < 3; ++i) p[i] = g[i] + P[9 + i];
  const double iz = 1.0 / p[2];
  const double u0 = p[0] * iz, u1 = p[1] * iz;
  const double s = u0 * u0 + u1 * u1;
  const double d = 1.0 + s * (k[3] + s * k[4]);
  const double f = k[0], fd = f * d;
  r[0] = fd * u0 + k[1] - x;
  r[1] = fd * u1 + k[2] - y;
  // dx/du = f (d I + d'(s) 2 u u^T), d'(s) = k1 + 2 k2 s; du/dp = [[1, 0, -u0], [0, 1, -u1]] / p2
  const double c = 2.0 * f * (k[3] + 2.0 * s * k[4]);
  const double a00 = fd + c * u0 * u0, a01 = c * u0 * u1, a11 = fd + c * u1 * u1;
  const double Du[3] = {a00 * iz, a01 * iz, -(a00 * u0 + a01 * u1) * iz};
  const double Dv[3] = {a01 * iz, a11 * iz, -(a01 * u0 + a11 * u1) * iz};
  Jc[0] = Du[2] * g[1] - Du[1] * g[2];
  Jc[1] = Du[0] * g[2] - Du[2] * g[0];
  Jc[2] = Du[1] * g[0] - Du[0] * g[1];
  Jc[3] = Du[0]; Jc[4] = Du[1]; Jc[5] = Du[2];
  Jc[6] = Dv[2] * g[1] - Dv[1] * g[2];
  Jc[7] = Dv[0] * g[2] - Dv[2] * g[0];
  Jc[8] = Dv[1] * g[0] - Dv[0] * g[1];
  Jc[9] = Dv[0]; Jc[10] = Dv[1]; Jc[11] = Dv[2];
#pragma unroll
  for (int m = 0; m < 3; ++m) {
    Jx[m] = Du[0] * P[m] + Du[1] * P[3 + m] + Du[2] * P[6 + m];
    Jx[3 + m] = Dv[0] * P[m] + Dv[1] * P[3 + m] + Dv[2] * P[6 + m];
  }
  Jk[0] = d * u0; Jk[1] = 1.0; Jk[2] = 0.0; Jk[3] = f * s * u0; Jk[4] = f * s * s * u0;
  Jk[5] = d * u1; Jk[6] = 0.0; Jk[7] = 1.0; Jk[8] = f * s * u1; Jk[9] = f * s * s * u1;
}

// The first turning point of the distortion, the smallest radius rho > 0 where d/drho (rho d(rho^2)) = 1 + 3 k1 rho^2
// + 5 k2 rho^4 = 0; INFINITY when it has none
DG_HD double rad_max_radius(double k1, double k2) {
  double s = INFINITY;   // the smallest positive root of 5 k2 s^2 + 3 k1 s + 1
  if (k2 == 0.0) {
    if (k1 < 0.0) s = -1.0 / (3.0 * k1);
  } else {
    const double disc = 9.0 * k1 * k1 - 20.0 * k2;
    if (disc >= 0.0) {
      const double q = sqrt(disc);
      const double s1 = (-3.0 * k1 - q) / (10.0 * k2), s2 = (-3.0 * k1 + q) / (10.0 * k2);
      if (s1 > 0.0) s = s1;
      if (s2 > 0.0 && s2 < s) s = s2;
    }
  }
  return sqrt(s);
}

// The pinhole pixel f u + c of the raw pixel (x, y): the radius rho of u solves rho (1 + k1 rho^2 + k2 rho^4) = rd,
// rd = |(x, y) - c| / f, by Newton's method kept inside [0, the first turning point] (a step that leaves the bracket
// bisects it), until a Newton step is at most 1e-15 rho.  False, and (NaN, NaN), for invalid intrinsics, for rd at or
// beyond the turning point's image, or when after kRadUndistortIters steps |rho d(rho^2) - rd| > 1e-14 rd.
DG_HD bool rad_undistort(const double* k, double x, double y, double* out) {
  out[0] = out[1] = NAN;
  if (!rad_valid(k) || !(fabs(x) < INFINITY) || !(fabs(y) < INFINITY)) return false;
  const double f = k[0], k1 = k[3], k2 = k[4];
  const double dx = x - k[1], dy = y - k[2];
  const double rd = sqrt(dx * dx + dy * dy) / f;
  if (rd == 0.0) {
    out[0] = x;
    out[1] = y;
    return true;
  }
  const double rmax = rad_max_radius(k1, k2);
  double lo = 0.0, hi = rmax;
  if (rmax < INFINITY) {
    const double s = rmax * rmax;
    if (!(rd < rmax * (1.0 + s * (k1 + s * k2)))) return false;   // at or beyond the turning point's image
  }
  double rho = rd < hi ? rd : 0.5 * hi;
  for (int it = 0; it < kRadUndistortIters; ++it) {
    const double s = rho * rho;
    const double phi = rho * (1.0 + s * (k1 + s * k2)) - rd;
    if (phi == 0.0) break;
    if (phi > 0.0) hi = rho; else lo = rho;
    const double next = rho - phi / (1.0 + s * (3.0 * k1 + 5.0 * k2 * s));
    if (fabs(next - rho) <= 1e-15 * rho) {           // converged
      rho = next;
      break;
    }
    rho = next > lo && next < hi ? next : (hi < INFINITY ? 0.5 * (lo + hi) : 2.0 * rho);
  }
  const double s = rho * rho;
  if (!(fabs(rho * (1.0 + s * (k1 + s * k2)) - rd) <= 1e-14 * rd)) return false;   // not converged
  const double sc = rho / rd;
  out[0] = k[1] + dx * sc;
  out[1] = k[2] + dy * sc;
  return true;
}

}  // namespace dg
