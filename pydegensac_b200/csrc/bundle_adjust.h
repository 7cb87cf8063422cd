// bundle_adjust.h -- per-thread pieces of the bundle adjustment of registered views and their tracks
// (bundle_adjust.cu): the robust weight, the projection with its Jacobians by the camera and the point, the damped 3 x 3
// point block and its inverse, the Schur products and the scale-gauge axis.
//
//   camera c: x ~ K_c (R_c X + t_c);  residual r = (q0 / q2 - x, q1 / q2 - y), q = K (R X + t),  e^2 = |r|^2
//   cost C = sum rho(e^2): rho(s) = s, or with a loss scale sigma the Cauchy loss sigma^2 log(1 + s / sigma^2)
//   IRLS weight w = rho'(e^2) at the linearisation: 1, or 1 / (1 + e^2 / sigma^2)
//
// Camera parameters are those of absolute_pose.h (ap_jacobian, ap_step): (w [3], d [3]), R <- exp([w]x) R, t <- t + d;
// point parameters X <- X + D.  The camera table is triangulate.h's (tr_camera).  tests/bundle_adjust_np.py restates
// every function here in numpy.
#pragma once
#include "common.h"
#include "absolute_pose.h"
#include "triangulate.h"

namespace dg {

constexpr int kBaMaxFree = 64;          // free cameras at most: the reduced camera system is dense, 6 x 64 unknowns
constexpr int kBaCamParams = 6;
constexpr int kBaMaxN = kBaCamParams * kBaMaxFree;

// One used observation's row of the linearisation: J_cam [2][6], r [2], w, W = w J_cam^T J_X [6][3] and
// Y = W V*^-1 [6][3] (the last written at every trial step, the rest after an accepted step)
constexpr int kBaObsJc = 0, kBaObsR = 12, kBaObsW = 14, kBaObsWm = 15, kBaObsY = 33, kBaObsStride = 51;
// One track's row: V = sum w J_X^T J_X (upper triangle by rows, 6), g_p = sum w J_X^T r (3), V*^-1 (upper, 6) and
// the track's cost at the trial point
constexpr int kBaTrkV = 0, kBaTrkG = 6, kBaTrkVi = 9, kBaTrkCost = 15, kBaTrkStride = 16;

// rho(s) and rho'(s) for the loss scale's square sig2 (0: the trivial loss)
DG_HD double ba_rho(double s, double sig2) { return sig2 > 0.0 ? sig2 * log1p(s / sig2) : s; }
DG_HD double ba_weight(double s, double sig2) { return sig2 > 0.0 ? 1.0 / (1.0 + s / sig2) : 1.0; }

// r [2], J_cam [2][6] (ap_jacobian) and J_X [2][3] = d(u, v)/dp R of an observation at (x, y) of X under pose P [12]
DG_HD void ba_jacobian(const double* P, const double* K, const double* X, double x, double y, double* r, double* Jc,
                       double* Jx) {
  ap_jacobian(P, K, x, y, X[0], X[1], X[2], r, Jc);
  // Jc[3 .. 5] and Jc[9 .. 11] are d(u, v)/dp
#pragma unroll
  for (int m = 0; m < 3; ++m) {
    Jx[m] = Jc[3] * P[m] + Jc[4] * P[3 + m] + Jc[5] * P[6 + m];
    Jx[3 + m] = Jc[9] * P[m] + Jc[10] * P[3 + m] + Jc[11] * P[6 + m];
  }
}

// V += w J_X^T J_X (upper triangle by rows) and g += w J_X^T r
DG_HD void ba_point_terms(const double* Jx, const double* r, double w, double* V, double* g) {
  int m = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int l = k; l < 3; ++l) V[m++] += w * (Jx[k] * Jx[l] + Jx[3 + k] * Jx[3 + l]);
#pragma unroll
  for (int k = 0; k < 3; ++k) g[k] += w * (Jx[k] * r[0] + Jx[3 + k] * r[1]);
}

// W = w J_cam^T J_X [6][3]
DG_HD void ba_cross_block(const double* Jc, const double* Jx, double w, double* W) {
#pragma unroll
  for (int k = 0; k < 6; ++k)
#pragma unroll
    for (int m = 0; m < 3; ++m) W[3 * k + m] = w * (Jc[k] * Jx[m] + Jc[6 + k] * Jx[3 + m]);
}

// Vi = (V + lam diag V)^-1 (both upper triangles by rows) by Cholesky; false at a pivot that is not positive
DG_HD bool ba_inv3(const double* V, double lam, double* Vi) {
  const double a00 = V[0] + lam * V[0], a01 = V[1], a02 = V[2], a11 = V[3] + lam * V[3], a12 = V[4],
               a22 = V[5] + lam * V[5];
  if (!(a00 > 0.0)) return false;
  const double l00 = sqrt(a00), l10 = a01 / l00, l20 = a02 / l00;
  const double d1 = a11 - l10 * l10;
  if (!(d1 > 0.0)) return false;
  const double l11 = sqrt(d1), l21 = (a12 - l20 * l10) / l11;
  const double d2 = a22 - l20 * l20 - l21 * l21;
  if (!(d2 > 0.0)) return false;
  const double l22 = sqrt(d2);
  // M = L^-1 (lower), V*^-1 = M^T M
  const double m00 = 1.0 / l00, m11 = 1.0 / l11, m22 = 1.0 / l22;
  const double m10 = -l10 * m00 / l11;
  const double m21 = -l21 * m11 / l22;
  const double m20 = -(l20 * m00 + l21 * m10) / l22;
  Vi[0] = m00 * m00 + m10 * m10 + m20 * m20;
  Vi[1] = m10 * m11 + m20 * m21;
  Vi[2] = m20 * m22;
  Vi[3] = m11 * m11 + m21 * m21;
  Vi[4] = m21 * m22;
  Vi[5] = m22 * m22;
  return true;
}

// y = Vi v for Vi symmetric (upper triangle by rows)
DG_HD void ba_sym3_mul(const double* Vi, const double* v, double* y) {
  y[0] = Vi[0] * v[0] + Vi[1] * v[1] + Vi[2] * v[2];
  y[1] = Vi[1] * v[0] + Vi[3] * v[1] + Vi[4] * v[2];
  y[2] = Vi[2] * v[0] + Vi[4] * v[1] + Vi[5] * v[2];
}

// Y = W Vi [6][3]
DG_HD void ba_schur_row(const double* W, const double* Vi, double* Y) {
#pragma unroll
  for (int k = 0; k < 6; ++k) ba_sym3_mul(Vi, W + 3 * k, Y + 3 * k);
}

// The axis of g's translation that the scale gauge holds: the largest |t_g + R_g c_a| (c_a the centre of the held
// camera a, from the camera table), the lower axis on ties
DG_HD int ba_gauge_axis(const double* Pg, const double* Ca) {
  double v[3];
  ap_camera(Pg, Ca[0], Ca[1], Ca[2], v);
  const double a0 = fabs(v[0]), a1 = fabs(v[1]), a2 = fabs(v[2]);
  return (a0 >= a1 && a0 >= a2) ? 0 : (a1 >= a2 ? 1 : 2);
}

}  // namespace dg
