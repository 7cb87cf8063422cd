// essential.h -- per-thread pieces of the essential-matrix RANSAC (essential_ragged_kernel, essential.cu): the
// normalised coordinates of the minimal sample, the calibrated F of an essential matrix, the MSAC score of a row and
// the start pose of the local optimisation.
//
//   x_n = K^-1 [x, y, 1],   x2_n^T E x1_n = 0,   F = K2^-T E K1^-1 (unit Frobenius norm),   e^2 = f_resid_sampson(F)
//
// A row is an inlier when e^2 < th^2 (the F RANSAC's Sampson rule in pixels); the MSAC cost of a model is
// sum min(e^2, th^2) over the usable rows.  The local optimisation is the Levenberg-Marquardt of refine_pose_ragged
// (pose_refine.h) over (R, t), |t| = 1.  tests/essential_np.py restates every function here in numpy.
#pragma once
#include "common.h"
#include "absolute_pose.h"
#include "five_point.h"
#include "pose_refine.h"

namespace dg {

constexpr int kEsMinRows = 5;          // fewer usable rows: no model
constexpr int kEsLoMinInliers = 6;     // fewer inliers: no local optimisation
constexpr int kEsLoRounds = 3;         // rounds of (LM on the inliers, re-selection of the inliers) at most

// K^-1 [x, y, 1]
DG_HD void es_normalise(const double* Ki, double x, double y, double* n) {
#pragma unroll
  for (int i = 0; i < 3; ++i) n[i] = Ki[3 * i] * x + Ki[3 * i + 1] * y + Ki[3 * i + 2];
}

// M [9] scaled to unit Frobenius norm (left at zero when it is zero), as refine_pose_ragged scales its F
DG_HD void es_unit9(double* M) {
  double nrm = 0.0;
#pragma unroll
  for (int i = 0; i < 9; ++i) nrm += M[i] * M[i];
  const double inv = nrm > 0.0 ? 1.0 / sqrt(nrm) : 0.0;
#pragma unroll
  for (int i = 0; i < 9; ++i) M[i] = M[i] * inv;
}

// F = A E Bk at unit norm, with A = K2^-T and Bk = K1^-1
DG_HD void es_fundamental(const double* E, const double* A, const double* Bk, double* F) {
  double AE[9];
  pr_mul3(A, E, AE);
  pr_mul3(AE, Bk, F);
  es_unit9(F);
}

// The MSAC term min(e^2, th^2) of a row under F (th^2 for a NaN e^2) and its inlier flag e^2 < th^2
DG_HD double es_msac(const double* F, double x1, double y1, double x2, double y2, double th2, bool* inlier) {
  const double e2 = f_resid_sampson(F, x1, y1, x2, y2);
  *inlier = e2 < th2;
  return fmin(e2, th2);
}

// One decomposition E ~ [t]x R (|t| = 1) of an essential matrix at unit norm (Horn 1990): t the unit vector orthogonal
// to E's columns (the largest of their three cross products), R = 2 cof(E) - sqrt(2) [t]x E, then orthonormalised.
// Any of the four decompositions gives +-E, and the Sampson error ignores the sign.  false for a rank < 2 E.
DG_HD bool es_pose(const double* E, double* R, double* t) {
  const double c[3][3] = {{E[0], E[3], E[6]}, {E[1], E[4], E[7]}, {E[2], E[5], E[8]}};
  double best = -1.0;
  for (int k = 0; k < 3; ++k) {
    double u[3];
    cross3(u, c[k == 2 ? 1 : 0], c[k == 0 ? 1 : 2]);
    const double nn = (u[0] * u[0] + u[1] * u[1]) + u[2] * u[2];
    if (nn > best) { best = nn; t[0] = u[0]; t[1] = u[1]; t[2] = u[2]; }
  }
  if (!(best > 0.0) || !(best < INFINITY)) return false;
  pr_unit3(t);
  double cof[9], T[9], TE[9];
  cross3(cof, E + 3, E + 6);
  cross3(cof + 3, E + 6, E);
  cross3(cof + 6, E, E + 3);
  pr_skew(t, T);
  pr_mul3(T, E, TE);
  const double r2 = sqrt(2.0);
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = 2.0 * cof[i] - r2 * TE[i];
  pr_orthonormalise(R);
  return true;
}

// E = [t]x R at unit norm
DG_HD void es_essential(const double* R, const double* t, double* E) {
  double T[9];
  pr_skew(t, T);
  pr_mul3(T, R, E);
  es_unit9(E);
}

DG_HD int es_required_iters(bool has_best, int inl, int n, double conf, int max_iters, int k) {
  return required_iters<5>(has_best, inl, n, conf, max_iters, k);
}

}  // namespace dg
