// refine_h.h -- per-thread pieces of the homography refinement (h_refine_ragged_kernel, frontend.cu): Levenberg-Marquardt
// on the engine's Sampson error over the inlier rows, in Hartley-normalised coordinates.
//
// The model is G = H^-1 (image 2 -> image 1), stored column-major as hgeom.h expects (g[i + 3 j] = G_ij); a row's cost
// is h_resid_sampson(G, row), the residual of the H RANSAC's default inlier rule.  With the algebraic pair e = (r1, r2)
// and JJ^T = [[A, B], [B, D]] of h_resid_sampson, the whitened residuals
//
//   z1 = r1 / sqrt(A),   z2 = (r2 - (B / sqrt(A)) z1) / sqrt(D - B^2 / A),   |z|^2 = e^T (JJ^T)^-1 e
//
// are the Gauss-Newton residuals; e, A, B and D are linear or quadratic in G, so the Jacobian is analytic.  The 8 local
// parameters d live in normalised coordinates: T1, T2 move the masked rows of image 1, 2 to their centroid and an RMS
// distance of sqrt(2); the normalised model is M = T1 G T2^-1 / |.|_F and a step is M <- (M + B d) / |M + B d|_F with
// B (9 x 8) the orthonormal basis of the plane orthogonal to M given by the Householder reflection that maps e_9 to
// +-M.  The residuals are always evaluated in pixels, G = T1^-1 M T2.  z does not depend on the scale of G, so the
// unit-norm constraint adds no term: dG_k = T1^-1 B_k T2.  tests/refine_homography_np.py restates every function here
// in numpy.
#pragma once
#include "common.h"
#include "hgeom.h"
#include "pose_refine.h"   // pr_cholesky_solve and the Levenberg-Marquardt schedule (kPrLambda0 ...), shared

namespace dg {

constexpr int kRhSums = 45;       // per pass: cost, J^T J (upper triangle by rows, 36), J^T z (8)
constexpr int kRhNormSums = 8;    // per image: sum x, y, x^2, y^2 of the masked rows
constexpr int kRhMinRows = 5;     // fewer rows with mask != 0: H is passed through

// A normalising transform as (s, mx, my): T = [[s, 0, -s mx], [0, s, -s my], [0, 0, 1]], from the sums of x, y, x^2, y^2
// over n rows.  A pair without spread (or without rows) gets s = 1.
DG_HD void rh_transform(const double* sums, int n, double* T) {
  const double mx = n > 0 ? sums[0] / n : 0.0, my = n > 0 ? sums[1] / n : 0.0;
  const double var = n > 0 ? (sums[2] + sums[3]) / n - mx * mx - my * my : 0.0;
  T[0] = (var > 0.0 && var < INFINITY) ? sqrt(2.0 / var) : 1.0;
  T[1] = mx;
  T[2] = my;
}

// G = T1^-1 M T2 (column-major 3 x 3)
DG_HD void rh_to_pixels(const double* T1, const double* T2, const double* M, double* G) {
  double P[9];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    P[3 * j] = M[3 * j] / T1[0] + T1[1] * M[3 * j + 2];
    P[3 * j + 1] = M[3 * j + 1] / T1[0] + T1[2] * M[3 * j + 2];
    P[3 * j + 2] = M[3 * j + 2];
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    G[i] = T2[0] * P[i];
    G[3 + i] = T2[0] * P[3 + i];
    G[6 + i] = P[6 + i] - T2[0] * T2[1] * P[i] - T2[0] * T2[2] * P[3 + i];
  }
}

DG_HD void rh_unit(double* M) {
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < 9; ++i) s += M[i] * M[i];
  const double inv = 1.0 / sqrt(s);
#pragma unroll
  for (int i = 0; i < 9; ++i) M[i] *= inv;
}

// M = T1 G T2^-1 / |.|_F
DG_HD void rh_from_pixels(const double* T1, const double* T2, const double* G, double* M) {
  double Q[9];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    Q[3 * j] = T1[0] * (G[3 * j] - T1[1] * G[3 * j + 2]);
    Q[3 * j + 1] = T1[0] * (G[3 * j + 1] - T1[2] * G[3 * j + 2]);
    Q[3 * j + 2] = G[3 * j + 2];
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    M[i] = Q[i] / T2[0];
    M[3 + i] = Q[3 + i] / T2[0];
    M[6 + i] = T2[1] * Q[i] + T2[2] * Q[3 + i] + Q[6 + i];
  }
  rh_unit(M);
}

// C = adj(A), row-major in and out (A^-1 = C / det A)
DG_HD void rh_adjugate(const double* a, double* C) {
  C[0] = a[4] * a[8] - a[5] * a[7]; C[1] = a[2] * a[7] - a[1] * a[8]; C[2] = a[1] * a[5] - a[2] * a[4];
  C[3] = a[5] * a[6] - a[3] * a[8]; C[4] = a[0] * a[8] - a[2] * a[6]; C[5] = a[2] * a[3] - a[0] * a[5];
  C[6] = a[3] * a[7] - a[4] * a[6]; C[7] = a[1] * a[6] - a[0] * a[7]; C[8] = a[0] * a[4] - a[1] * a[3];
}

// The engine model of a public H (row-major, x2 ~ H x1): g = H^-1 = adj(H) / det(H), column-major.  False when H is all
// zero, holds a NaN, or its inverse is not finite (no model).
DG_HD bool rh_engine_model(const double* H, double* g) {
  bool zero = true, ok = true;
#pragma unroll
  for (int i = 0; i < 9; ++i) { zero &= H[i] == 0.0; ok &= H[i] == H[i]; }
  if (zero || !ok) return false;
  double C[9];
  rh_adjugate(H, C);
  const double det = H[0] * C[0] + H[1] * C[3] + H[2] * C[6];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      g[i + 3 * j] = C[3 * i + j] / det;
      ok &= fabs(g[i + 3 * j]) < INFINITY;
    }
  return ok;
}

// H scaled to unit Frobenius norm and det H > 0, in place
DG_HD void rh_unit_det_pos(double* H) {
  rh_unit(H);
  double C[9];
  rh_adjugate(H, C);
  if (H[0] * C[0] + H[1] * C[3] + H[2] * C[6] < 0.0) {
#pragma unroll
    for (int i = 0; i < 9; ++i) H[i] = -H[i];
  }
}

// The public H (row-major, x2 ~ H x1, unit Frobenius norm, det > 0) of a column-major engine model g: adj(G) is H up to
// scale, and read as row-major the column-major g is G^T, whose adjugate is adj(G)^T.
DG_HD void rh_public_model(const double* g, double* H) {
  double C[9];
  rh_adjugate(g, C);
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) H[3 * i + j] = C[3 * j + i];
  rh_unit_det_pos(H);
}

// Column k (< 8) of the Householder basis of the plane orthogonal to the unit 9-vector m: with s = -sign(m_8) (-1 at
// m_8 = 0) and u = 1 + |m_8|, B_k[j] = delta_jk - m_j m_k / u for j < 8 and B_k[8] = s m_k.
DG_HD void rh_basis_column(const double* m, int k, double* b) {
  const double u = 1.0 + fabs(m[8]), s = m[8] >= 0.0 ? -1.0 : 1.0;
#pragma unroll
  for (int j = 0; j < 8; ++j) b[j] = (j == k ? 1.0 : 0.0) - m[j] * m[k] / u;
  b[8] = s * m[k];
}

// G [9] and dG [8][9] (pixels, column-major): the model and its derivatives by the 8 local parameters at zero
DG_HD void rh_linearise(const double* T1, const double* T2, const double* M, double* G, double* dG) {
  rh_to_pixels(T1, T2, M, G);
  for (int k = 0; k < 8; ++k) {
    double b[9];
    rh_basis_column(M, k, b);
    rh_to_pixels(T1, T2, b, dG + 9 * k);
  }
}

// A read of the linearisation that the compiler may not hoist out of the row loop: the 81 entries of (G, dG) kept in
// registers across rows would take the registers the 45 sums need, and spill.
#if DG_DEVICE_PASS
DG_HD void rh_load9(const double* p, double* g) {
#pragma unroll
  for (int i = 0; i < 9; ++i) g[i] = *(const volatile double*)(p + i);
}
#else
DG_HD void rh_load9(const double* p, double* g) {
  for (int i = 0; i < 9; ++i) g[i] = p[i];
}
#endif

// The algebraic pair and the entries of the Sampson Jacobian of one row under gp (the operations of h_resid_sampson)
DG_HD void rh_terms(const double* gp, double x1, double y1, double x2, double y2, double* t) {
  double g[9];
  rh_load9(gp, g);
  double r1 = 0.0, r2 = 0.0;
  r1 += g[0] * x2;
  r2 += g[1] * x2;
  r1 += g[2] * (-x1 * x2);
  r2 += g[2] * (-y1 * x2);
  r1 += g[3] * y2;
  r2 += g[4] * y2;
  r1 += g[5] * (-x1 * y2);
  r2 += g[5] * (-y1 * y2);
  r1 += g[6] * 1.0;
  r2 += g[7] * 1.0;
  r1 += g[8] * (-x1 * 1.0);
  r2 += g[8] * (-y1 * 1.0);
  t[0] = r1;
  t[1] = r2;
  t[2] = g[0] - g[2] * x1;            // a
  t[3] = g[3] - g[5] * x1;            // b
  t[4] = -g[8] - g[2] * x2 - g[5] * y2;   // c
  t[5] = g[1] - g[2] * y1;            // d
  t[6] = g[4] - g[5] * y1;            // e
}

// One row at the linearisation (G, dG): adds h_resid_sampson(G, row) to acc[0], J_k J_l (k <= l, both whitened
// residuals) to acc[1 .. 36] and J_k . z to acc[37 .. 44].
DG_HD void rh_row(const double* G, const double* dG, double x1, double y1, double x2, double y2, double* acc) {
  acc[0] += h_resid_sampson(G, x1, y1, x2, y2);
  double t[7];
  rh_terms(G, x1, y1, x2, y2, t);
  const double a = t[2], b = t[3], c = t[4], d = t[5], e = t[6];
  const double A = a * a + b * b + c * c, B = a * d + b * e, D = d * d + e * e + c * c;
  const double sA = sqrt(A), iA = 1.0 / sA, be = B * iA;
  const double sS = sqrt(D - be * be), iS = 1.0 / sS;
  const double z1 = t[0] * iA, z2 = (t[1] - be * z1) * iS;
  double J1[8], J2[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    double q[7];
    rh_terms(dG + 9 * k, x1, y1, x2, y2, q);
    const double dA = 2.0 * (a * q[2] + b * q[3] + c * q[4]);
    const double dB = a * q[5] + d * q[2] + b * q[6] + e * q[3];
    const double dD = 2.0 * (d * q[5] + e * q[6] + c * q[4]);
    const double dz1 = (q[0] - z1 * dA * 0.5 * iA) * iA;
    const double dbe = (dB - be * dA * 0.5 * iA) * iA;
    const double dS = dD - 2.0 * be * dbe;
    J1[k] = dz1;
    J2[k] = (q[1] - dbe * z1 - be * dz1 - z2 * dS * 0.5 * iS) * iS;
  }
  int m = 1;
#pragma unroll
  for (int k = 0; k < 8; ++k)
#pragma unroll
    for (int l = k; l < 8; ++l) acc[m++] += J1[k] * J1[l] + J2[k] * J2[l];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[37 + k] += J1[k] * z1 + J2[k] * z2;
}

// The model D away from M: (M + B D) / |M + B D|_F
DG_HD void rh_step(const double* M, const double* D, double* M2) {
  const double u = 1.0 + fabs(M[8]), s = M[8] >= 0.0 ? -1.0 : 1.0;
  double md = 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) md += M[k] * D[k];
#pragma unroll
  for (int j = 0; j < 8; ++j) M2[j] = M[j] + D[j] - M[j] * md / u;
  M2[8] = M[8] + s * md;
  rh_unit(M2);
}

}  // namespace dg
