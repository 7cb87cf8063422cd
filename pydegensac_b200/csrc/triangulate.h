// triangulate.h -- per-thread pieces of the multi-view track triangulation (triangulate_tracks_ragged_kernel,
// triangulate.cu): the camera table, the world rays, the two-ray midpoint hypothesis, the MSAC score of an
// observation, the enumeration of pairs and the local optimisation's Levenberg-Marquardt row.
//
//   camera c: x ~ K_c (R_c X + t_c),  centre C_c = -R_c^T t_c,  ray of an observation d = R_c^T normalize(K_c^-1 [x, y, 1])
//
// The score and the residual are those of absolute_pose.h (ap_msac, ap_camera, ap_residual) with the observation's
// camera as the pose and the track's point as the world point.  Local parameters: X <- X + D (3).
// tests/triangulate_np.py restates every function here in numpy.
#pragma once
#include "common.h"
#include "absolute_pose.h"

namespace dg {

constexpr int kTrParams = 3;
constexpr int kTrSums = 1 + kTrParams * (kTrParams + 1) / 2 + kTrParams;   // cost, J^T J (upper, by rows), J^T r
constexpr int kTrMinRows = 2;          // fewer usable observations: no model; fewer inliers: no local optimisation
constexpr int kTrLoRounds = 3;         // rounds of (LM on the inliers, re-selection of the inliers) at most

// One camera's row of the camera table: the pose P = (R [9], t [3]) as ap_camera takes it, K, K^-1, the centre and a
// flag (1.0 when the camera is registered: the 12 entries of (R, t) finite and det R > 0.5, else 0.0)
constexpr int kTrCamP = 0, kTrCamK = 12, kTrCamKi = 21, kTrCamC = 30, kTrCamOk = 33, kTrCamStride = 34;

DG_HD void tr_camera(const double* R, const double* t, const double* K, double* cam) {
  bool finite = true;
#pragma unroll
  for (int i = 0; i < 9; ++i) { cam[kTrCamP + i] = R[i]; finite = finite && fabs(R[i]) < INFINITY; }
#pragma unroll
  for (int i = 0; i < 3; ++i) { cam[kTrCamP + 9 + i] = t[i]; finite = finite && fabs(t[i]) < INFINITY; }
#pragma unroll
  for (int i = 0; i < 9; ++i) cam[kTrCamK + i] = K[i];
  ap_inv3(K, cam + kTrCamKi);
#pragma unroll
  for (int k = 0; k < 3; ++k) cam[kTrCamC + k] = -(R[k] * t[0] + R[3 + k] * t[1] + R[6 + k] * t[2]);
  double c[3];
  cross3(c, R + 3, R + 6);
  const double det = R[0] * c[0] + R[1] * c[1] + R[2] * c[2];
  cam[kTrCamOk] = finite && det > 0.5 ? 1.0 : 0.0;
}

// The world ray direction d = R^T ap_bearing(K^-1, x, y) of an observation at (x, y) in camera `cam`
DG_HD void tr_ray(const double* cam, double x, double y, double* d) {
  double b[3];
  ap_bearing(cam + kTrCamKi, x, y, b);
  const double* R = cam + kTrCamP;
#pragma unroll
  for (int k = 0; k < 3; ++k) d[k] = R[k] * b[0] + R[3 + k] * b[1] + R[6 + k] * b[2];
}

DG_HD double tr_dot(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// The hypothesis of the rays (Ci, di), (Cj, dj): the midpoint of their common perpendicular, when the angle between
// them is at least the gate's (b = di . dj <= cos_max, 1 - b^2 > 0) and both feet lie ahead of their centres
DG_HD bool tr_midpoint(const double* Ci, const double* di, const double* Cj, const double* dj, double cos_max,
                       double* X) {
  const double b = tr_dot(di, dj);
  const double den = 1.0 - b * b;
  if (b > cos_max || !(den > 0.0)) return false;
  const double w[3] = {Ci[0] - Cj[0], Ci[1] - Cj[1], Ci[2] - Cj[2]};
  const double pi = tr_dot(di, w), pj = tr_dot(dj, w);
  const double li = (b * pj - pi) / den, lj = (pj - b * pi) / den;
  if (!(li > 0.0) || !(lj > 0.0)) return false;
#pragma unroll
  for (int k = 0; k < 3; ++k) X[k] = 0.5 * ((Ci[k] + li * di[k]) + (Cj[k] + lj * dj[k]));
  return true;
}

// The MSAC term min(e^2, th^2) of an observation of X in camera `cam` (th^2 behind it), and its inlier flag
DG_HD double tr_msac(const double* cam, const double* X, double x, double y, double th2, bool* inlier) {
  return ap_msac(cam + kTrCamP, cam + kTrCamK, x, y, X[0], X[1], X[2], th2, inlier);
}

// Residual r [2] and Jacobian J [2][3] by X of an observation: d(u, v)/dp = [K0 - u K2; K1 - v K2] / q2 (K_i the rows
// of K), dp/dX = R
DG_HD void tr_jacobian(const double* cam, const double* X, double x, double y, double* r, double* J) {
  const double* R = cam + kTrCamP;
  const double* K = cam + kTrCamK;
  double p[3];
  ap_camera(R, X[0], X[1], X[2], p);
  const double q0 = K[0] * p[0] + K[1] * p[1] + K[2] * p[2];
  const double q1 = K[3] * p[0] + K[4] * p[1] + K[5] * p[2];
  const double q2 = K[6] * p[0] + K[7] * p[1] + K[8] * p[2];
  const double iz = 1.0 / q2;
  const double u = q0 * iz, v = q1 * iz;
  r[0] = u - x;
  r[1] = v - y;
  double Du[3], Dv[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) { Du[j] = (K[j] - u * K[6 + j]) * iz; Dv[j] = (K[3 + j] - v * K[6 + j]) * iz; }
#pragma unroll
  for (int m = 0; m < 3; ++m) {
    J[m] = Du[0] * R[m] + Du[1] * R[3 + m] + Du[2] * R[6 + m];
    J[3 + m] = Dv[0] * R[m] + Dv[1] * R[3 + m] + Dv[2] * R[6 + m];
  }
}

// One observation of the LM pass: adds |r|^2 to acc[0], J^T J (upper triangle by rows) to acc[1 .. 6], J^T r to
// acc[7 .. 9]
DG_HD void tr_row(const double* cam, const double* X, double x, double y, double* acc) {
  double r[2], J[6];
  tr_jacobian(cam, X, x, y, r, J);
  acc[0] += r[0] * r[0] + r[1] * r[1];
  int m = 1;
#pragma unroll
  for (int k = 0; k < kTrParams; ++k)
#pragma unroll
    for (int l = k; l < kTrParams; ++l) acc[m++] += J[k] * J[l] + J[3 + k] * J[3 + l];
#pragma unroll
  for (int k = 0; k < kTrParams; ++k) acc[m++] += J[k] * r[0] + J[3 + k] * r[1];
}

// The pair (i, j), i < j < n, s places after (i, j) in lexicographic order: (0, 1), (0, 2), ..., (0, n-1), (1, 2), ....
// Each step of the loop passes the rest of a row, so it runs at most s times.  Past the last pair, i reaches n - 1.
DG_HD void tr_pair_advance(int n, int s, int* i, int* j) {
  int a = *i, b = *j + s;
  while (b >= n && a < n - 1) {
    const int over = b - n;
    ++a;
    b = a + 1 + over;
  }
  *i = a;
  *j = b;
}

}  // namespace dg
