// absolute_pose.h -- per-thread pieces of the absolute-pose RANSAC (absolute_pose_ragged_kernel, absolute_pose.cu):
// the bearings of the minimal sample, the MSAC score of a row, the stopping rule and the local optimisation's
// Levenberg-Marquardt row and step.
//
//   camera point p = R X + t,  projection q = K p,  pixel residual r = (q0 / q2 - x, q1 / q2 - y),  e^2 = |r|^2
//
// A row whose depth p_z is not positive scores th^2; the MSAC cost of a pose is sum min(e^2, th^2) over the usable rows,
// and a row is an inlier when p_z > 0 and e^2 <= th^2.  Local parameters theta = (w [3], d [3]), re-centred at every
// accepted step: R <- exp([w]x) R, t <- t + d; at theta = 0, dp/dw = -[R X]x and dp/dd = I.  tests/absolute_pose_np.py
// restates every function here in numpy.
#pragma once
#include "common.h"
#include "pose_refine.h"

namespace dg {

constexpr int kApParams = 6;
constexpr int kApSums = 1 + kApParams * (kApParams + 1) / 2 + kApParams;   // cost, J^T J (upper triangle by rows), J^T r
constexpr int kApMinRows = 4;          // fewer usable rows: no model; fewer inliers: no local optimisation
constexpr int kApLoRounds = 3;         // rounds of (LM on the inliers, re-selection of the inliers) at most

// K^-1 [9] of K [9] (row-major) by its adjugate: the rows of K^-1 are the cross products of K's columns over det K
DG_HD void ap_inv3(const double* K, double* Ki) {
  const double c0[3] = {K[0], K[3], K[6]}, c1[3] = {K[1], K[4], K[7]}, c2[3] = {K[2], K[5], K[8]};
  cross3(Ki, c1, c2);
  cross3(Ki + 3, c2, c0);
  cross3(Ki + 6, c0, c1);
  const double det = c0[0] * Ki[0] + c0[1] * Ki[1] + c0[2] * Ki[2];
#pragma unroll
  for (int i = 0; i < 9; ++i) Ki[i] = Ki[i] / det;
}

// The unit bearing normalize(K^-1 [x, y, 1])
DG_HD void ap_bearing(const double* Ki, double x, double y, double* b) {
#pragma unroll
  for (int i = 0; i < 3; ++i) b[i] = Ki[3 * i] * x + Ki[3 * i + 1] * y + Ki[3 * i + 2];
  const double inv = 1.0 / sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
  b[0] *= inv; b[1] *= inv; b[2] *= inv;
}

// Camera point p of world point X under the pose P [12] = (R [9], t [3])
DG_HD void ap_camera(const double* P, double X, double Y, double Z, double* p) {
#pragma unroll
  for (int i = 0; i < 3; ++i) p[i] = P[3 * i] * X + P[3 * i + 1] * Y + P[3 * i + 2] * Z + P[9 + i];
}

// The pixel residual (r0, r1) of camera point p observed at (x, y) through K
DG_HD void ap_residual(const double* K, const double* p, double x, double y, double* r) {
  const double q0 = K[0] * p[0] + K[1] * p[1] + K[2] * p[2];
  const double q1 = K[3] * p[0] + K[4] * p[1] + K[5] * p[2];
  const double q2 = K[6] * p[0] + K[7] * p[1] + K[8] * p[2];
  r[0] = q0 / q2 - x;
  r[1] = q1 / q2 - y;
}

// e^2 of a row under pose P, and whether its depth is positive
DG_HD double ap_sq_error(const double* P, const double* K, double x, double y, double X, double Y, double Z,
                         bool* front) {
  double p[3], r[2];
  ap_camera(P, X, Y, Z, p);
  ap_residual(K, p, x, y, r);
  *front = p[2] > 0.0;
  return r[0] * r[0] + r[1] * r[1];
}

// The MSAC term min(e^2, th^2) of a row (th^2 behind the camera; fmin keeps th^2 for a NaN e^2), and its inlier flag
DG_HD double ap_msac(const double* P, const double* K, double x, double y, double X, double Y, double Z, double th2,
                     bool* inlier) {
  bool front;
  const double e2 = ap_sq_error(P, K, x, y, X, Y, Z, &front);
  *inlier = front && e2 <= th2;
  return front ? fmin(e2, th2) : th2;
}

// Residual r [2] and Jacobian J [2][6] (by w0, w1, w2, d0, d1, d2 at zero) of a row under pose P
DG_HD void ap_jacobian(const double* P, const double* K, double x, double y, double X, double Y, double Z, double* r,
                       double* J) {
  double g[3], p[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) g[i] = P[3 * i] * X + P[3 * i + 1] * Y + P[3 * i + 2] * Z;   // R X
#pragma unroll
  for (int i = 0; i < 3; ++i) p[i] = g[i] + P[9 + i];
  const double q0 = K[0] * p[0] + K[1] * p[1] + K[2] * p[2];
  const double q1 = K[3] * p[0] + K[4] * p[1] + K[5] * p[2];
  const double q2 = K[6] * p[0] + K[7] * p[1] + K[8] * p[2];
  const double iz = 1.0 / q2;
  const double u = q0 * iz, v = q1 * iz;
  r[0] = u - x;
  r[1] = v - y;
  // d(u, v)/dp = [K0 - u K2; K1 - v K2] / q2 (K_i the rows of K); dp/dw = -[g]x = [[0, g2, -g1], [-g2, 0, g0],
  // [g1, -g0, 0]], dp/dd = I
  double Du[3], Dv[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) { Du[j] = (K[j] - u * K[6 + j]) * iz; Dv[j] = (K[3 + j] - v * K[6 + j]) * iz; }
  J[0] = Du[2] * g[1] - Du[1] * g[2];
  J[1] = Du[0] * g[2] - Du[2] * g[0];
  J[2] = Du[1] * g[0] - Du[0] * g[1];
  J[3] = Du[0]; J[4] = Du[1]; J[5] = Du[2];
  J[6] = Dv[2] * g[1] - Dv[1] * g[2];
  J[7] = Dv[0] * g[2] - Dv[2] * g[0];
  J[8] = Dv[1] * g[0] - Dv[0] * g[1];
  J[9] = Dv[0]; J[10] = Dv[1]; J[11] = Dv[2];
}

// One row of the LM pass: adds |r|^2 to acc[0], J^T J (upper triangle by rows) to acc[1 .. 21], J^T r to acc[22 .. 27]
DG_HD void ap_row(const double* P, const double* K, double x, double y, double X, double Y, double Z, double* acc) {
  double r[2], J[12];
  ap_jacobian(P, K, x, y, X, Y, Z, r, J);
  acc[0] += r[0] * r[0] + r[1] * r[1];
  int m = 1;
#pragma unroll
  for (int k = 0; k < kApParams; ++k)
#pragma unroll
    for (int l = k; l < kApParams; ++l) acc[m++] += J[k] * J[l] + J[6 + k] * J[6 + l];
#pragma unroll
  for (int k = 0; k < kApParams; ++k) acc[m++] += J[k] * r[0] + J[6 + k] * r[1];
}

// The pose D = (w, d) away from P: R2 = exp([w]x) R (Rodrigues, as pr_step), t2 = t + d
DG_HD void ap_step(const double* P, const double* D, double* P2) {
  const double a = sqrt(D[0] * D[0] + D[1] * D[1] + D[2] * D[2]);
  double c1 = 1.0, c2 = 0.5;
  if (a != 0.0) {
    const double h = sin(0.5 * a) / a;
    c1 = sin(a) / a;
    c2 = 2.0 * h * h;
  }
  double W[9], W2[9], E[9];
  pr_skew(D, W);
  pr_mul3(W, W, W2);
#pragma unroll
  for (int i = 0; i < 9; ++i) E[i] = (i % 4 == 0 ? 1.0 : 0.0) + c1 * W[i] + c2 * W2[i];
  pr_mul3(E, P, P2);
#pragma unroll
  for (int i = 0; i < 3; ++i) P2[9 + i] = P[9 + i] + D[3 + i];
}

// w^S as ((w w) w) ...
template <int S>
DG_HD double ipow(double w) {
  if constexpr (S == 1) return w;
  else return ipow<S - 1>(w) * w;
}

// The iterations the sequential rule requires after an iteration k whose best model, fitted to samples of S rows, has
// `inl` of n inliers: min(max_iters, ceil(log(1 - conf) / log1p(-w^S))), w = inl / n; max_iters when conf == 1 or
// there is no best model yet (has_best false), k when w == 1.
template <int S>
DG_HD int required_iters(bool has_best, int inl, int n, double conf, int max_iters, int k) {
  if (!has_best || conf >= 1.0) return max_iters;
  if (inl >= n) return k;
  const double w = (double)inl / (double)n;
  const double q = ceil(log(1.0 - conf) / log1p(-ipow<S>(w)));
  return q < (double)max_iters ? (int)q : max_iters;
}
DG_HD int ap_required_iters(bool has_best, int inl, int n, double conf, int max_iters, int k) {
  return required_iters<3>(has_best, inl, n, conf, max_iters, k);
}

}  // namespace dg
