// refine_f.h -- per-thread pieces of the fundamental-matrix refinement (f_refine_ragged_kernel, frontend.cu):
// Levenberg-Marquardt on the Sampson error over the rank-2 matrices, in Hartley-normalised coordinates.
//
// F is row-major with x2^T F x1 = 0, as the F RANSAC returns it; a row's cost is f_resid_sampson(F, row), the residual
// of the F RANSAC's default inlier rule, and its Gauss-Newton residual r = c / sqrt(s) is pr_row's (pose_refine.h),
// which does not depend on the scale of F.  T1, T2 (rh_transform, refine_h.h) move the masked rows of image 1, 2 to
// their centroid and an RMS distance of sqrt(2); the normalised model is Fn = T2^-T F T1^-1 at |Fn|_F = 1, and the
// residuals are always evaluated in pixels through F = T2^T Fn T1.
//
// The 7 local parameters d are free of gauge.  The tangent space of the unit-norm rank-2 matrices at Fn is the
// complement in R^9 of vec(Fn) and of vec(cof Fn) (cof Fn = +-s1 s2 u3 v3^T for a rank-2 Fn, and <Fn, cof Fn> =
// 3 det Fn = 0).  B (9 x 7) is an orthonormal basis of it by two Householder reflections: the first, B1, maps e_9 to
// +-vec(Fn) (the reflection of rh_basis_column); the second, inside B1's 8 columns, maps e_8 to +-a, the coordinates
// a = B1^T c of the unit cofactor vector c.  B depends on Fn alone, through polynomials and the two reflections: no
// SVD sign or ordering enters it.  A step is the retraction Fn <- unit(rank2(Fn + B d)), rank2 the projection of
// la.h in its inlinable flavour enforce_rank2_inl (a call of the non-inlined enforce_rank2 from the kernel changes the
// register allocation of the svd3_onesided it shares with the pose kernels, and their SASS with it); to first order
// the retraction is the identity on the tangent space, so dFn / dd_k = B_k at d = 0 and dF_k = T2^T B_k T1.
// tests/refine_fundamental_np.py restates every function here in numpy.
#pragma once
#include "common.h"
#include "fgeom.h"
#include "la.h"
#include "pose_refine.h"   // pr_row_n, pr_cholesky_solve and the Levenberg-Marquardt schedule (kPrLambda0 ...), shared
#include "refine_h.h"      // rh_transform, rh_unit, shared

namespace dg {

constexpr int kRfSums = 36;       // per pass: cost, J^T J (upper triangle by rows, 28), J^T r (7)
constexpr int kRfMinRows = 8;     // fewer rows with mask != 0: F is passed through

// Fn = T2^-T F T1^-1 (row-major 3 x 3, not normalised); T as (s, mx, my) of rh_transform
DG_HD void rf_from_pixels(const double* T1, const double* T2, const double* F, double* Fn) {
  double Q[9];                                     // F T1^-1
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    Q[3 * i] = F[3 * i] / T1[0];
    Q[3 * i + 1] = F[3 * i + 1] / T1[0];
    Q[3 * i + 2] = T1[1] * F[3 * i] + T1[2] * F[3 * i + 1] + F[3 * i + 2];
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    Fn[j] = Q[j] / T2[0];
    Fn[3 + j] = Q[3 + j] / T2[0];
    Fn[6 + j] = T2[1] * Q[j] + T2[2] * Q[3 + j] + Q[6 + j];
  }
}

// F = T2^T Fn T1 (row-major)
DG_HD void rf_to_pixels(const double* T1, const double* T2, const double* Fn, double* F) {
  double P[9];                                     // Fn T1
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    P[3 * i] = T1[0] * Fn[3 * i];
    P[3 * i + 1] = T1[0] * Fn[3 * i + 1];
    P[3 * i + 2] = Fn[3 * i + 2] - T1[0] * T1[1] * Fn[3 * i] - T1[0] * T1[2] * Fn[3 * i + 1];
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    F[j] = T2[0] * P[j];
    F[3 + j] = T2[0] * P[3 + j];
    F[6 + j] = P[6 + j] - T2[0] * T2[1] * P[j] - T2[0] * T2[2] * P[3 + j];
  }
}

// The cofactor matrix of f, row-major (cof F = det(F) F^-T)
DG_HD void rf_cofactor(const double* f, double* c) {
  c[0] = f[4] * f[8] - f[5] * f[7]; c[1] = f[5] * f[6] - f[3] * f[8]; c[2] = f[3] * f[7] - f[4] * f[6];
  c[3] = f[2] * f[7] - f[1] * f[8]; c[4] = f[0] * f[8] - f[2] * f[6]; c[5] = f[1] * f[6] - f[0] * f[7];
  c[6] = f[1] * f[5] - f[2] * f[4]; c[7] = f[2] * f[3] - f[0] * f[5]; c[8] = f[0] * f[4] - f[1] * f[3];
}

// y = Q x for the first L - 1 columns Q of the Householder reflection that maps e_L to s m (m a unit L-vector,
// s = -sign(m_{L-1}), -1 at 0; the columns of rh_basis_column for L = 9): with u = 1 + |m_{L-1}| and md = m . x over
// j < L - 1, y_j = x_j - m_j md / u for j < L - 1 and y_{L-1} = s md.
template <int L>
DG_HD void rf_householder_apply(const double* m, const double* x, double* y) {
  const double u = 1.0 + fabs(m[L - 1]), s = m[L - 1] >= 0.0 ? -1.0 : 1.0;
  double md = 0.0;
#pragma unroll
  for (int j = 0; j < L - 1; ++j) md += m[j] * x[j];
#pragma unroll
  for (int j = 0; j < L - 1; ++j) y[j] = x[j] - m[j] * md / u;
  y[L - 1] = s * md;
}

// a [8]: the coordinates a = B1^T c of the unit cofactor vector c of Fn in the first reflection's columns, scaled to
// unit length (B1[j][k] = delta_jk - m_j m_k / u for j < 8 and B1[8][k] = s m_k, m = vec(Fn))
DG_HD void rf_cofactor_coords(const double* Fn, double* a) {
  double c[9];
  rf_cofactor(Fn, c);
  rh_unit(c);
  const double u = 1.0 + fabs(Fn[8]), s = Fn[8] >= 0.0 ? -1.0 : 1.0;
  double mc = 0.0;
#pragma unroll
  for (int j = 0; j < 8; ++j) mc += Fn[j] * c[j];
  double n2 = 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    a[k] = c[k] - Fn[k] * mc / u + s * Fn[k] * c[8];
    n2 += a[k] * a[k];
  }
  const double inv = 1.0 / sqrt(n2);
#pragma unroll
  for (int k = 0; k < 8; ++k) a[k] *= inv;
}

// v [9] = B d for d [7]: v = B1 (Q2 d), Q2 the first 7 columns of the reflection of a
DG_HD void rf_tangent(const double* Fn, const double* a, const double* d, double* v) {
  double q[8];
  rf_householder_apply<8>(a, d, q);
  rf_householder_apply<9>(Fn, q, v);
}

// The retraction: Fn2 = unit(rank2(Fn + B d))
DG_HD void rf_retract(const double* Fn, const double* d, double* Fn2) {
  double a[8], v[9], X[9];
  rf_cofactor_coords(Fn, a);
  rf_tangent(Fn, a, d, v);
#pragma unroll
  for (int i = 0; i < 9; ++i) X[i] = Fn[i] + v[i];
  enforce_rank2_inl(X);
  rh_unit(X);
#pragma unroll
  for (int i = 0; i < 9; ++i) Fn2[i] = X[i];
}

// False when F is all zero or holds a value that is not finite (no model)
DG_HD bool rf_has_model(const double* F) {
  bool zero = true, ok = true;
#pragma unroll
  for (int i = 0; i < 9; ++i) { zero &= F[i] == 0.0; ok &= fabs(F[i]) < INFINITY; }
  return ok && !zero;
}

// The start point Fn0 = unit(rank2(T2^-T F T1^-1)): F itself, up to rounding, when F has rank 2
DG_HD void rf_start(const double* T1, const double* T2, const double* F, double* Fn) {
  double X[9];
  rf_from_pixels(T1, T2, F, X);
  enforce_rank2_inl(X);
  rh_unit(X);
#pragma unroll
  for (int i = 0; i < 9; ++i) Fn[i] = X[i];
}

// F [9] and dF [7][9] (pixels, row-major): the model and its derivatives by the 7 local parameters at zero
DG_HD void rf_linearise(const double* T1, const double* T2, const double* Fn, double* F, double* dF) {
  double a[8];
  rf_cofactor_coords(Fn, a);
  rf_to_pixels(T1, T2, Fn, F);
  for (int k = 0; k < 7; ++k) {
    double d[7], b[9];
#pragma unroll
    for (int j = 0; j < 7; ++j) d[j] = j == k ? 1.0 : 0.0;
    rf_tangent(Fn, a, d, b);
    rf_to_pixels(T1, T2, b, dF + 9 * k);
  }
}

// The public F of Fn: T2^T Fn T1 at unit Frobenius norm, signed so that <F, F_in> >= 0
DG_HD void rf_output(const double* T1, const double* T2, const double* Fn, const double* F_in, double* F) {
  rf_to_pixels(T1, T2, Fn, F);
  rh_unit(F);
  double dot = 0.0;
#pragma unroll
  for (int i = 0; i < 9; ++i) dot += F[i] * F_in[i];
  if (dot < 0.0) {
#pragma unroll
    for (int i = 0; i < 9; ++i) F[i] = -F[i];
  }
}

}  // namespace dg
