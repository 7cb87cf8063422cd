// p3p.h -- the minimal solver of the absolute-pose RANSAC (absolute_pose.cu): Lambda Twist P3P (M. Persson and
// K. Nordberg, "Lambda Twist: An Accurate Fast Robust Perspective Three Point (P3P) Solver", ECCV 2018), in FP64.
//
// Three unit bearings y_i (camera frame) and three world points x_i give the depths l_i > 0 of the points along their
// bearings from the three distance constraints
//   l_i^2 + l_j^2 + b_ij l_i l_j = a_ij,   b_ij = -2 y_i . y_j,   a_ij = |x_i - x_j|^2   ((i, j) = (1,2), (1,3), (2,3)).
// Lambda Twist combines two of them, D1 = a23 M12 - a12 M23 and D2 = a23 M13 - a13 M23 (M_ij the quadratic form of
// constraint ij), into D0 = D1 - g D2 with det D0 = 0: one real root g of a cubic.  D0 is then rank 2, so
// lambda^T D0 lambda = 0 factors into two planes through the origin, l1 = w0 l2 + w1 l3; each plane and the constraint
// a13 (12) - a12 (13) give a quadratic in tau = l3 / l2, and (23) fixes the scale.  Up to 4 solutions, each polished by
// Newton's method on the three constraints; then R = [y-triangle] [x-triangle]^-1 and t = l1 y1 - R x1 (x ~ R X + t).
//
// Only +, -, *, / and sqrt, in a fixed order: a host build with -ffp-contract=off (tests/absolute_pose_host.cpp) and
// the device build with -fmad=false give the same bits, and tests/absolute_pose_np.py restates every line with
// Python floats.
#pragma once
#include "common.h"

namespace dg {

constexpr int kP3pCubicIters = 50;     // Newton steps on the cubic at most; at least 7 before the residual test
constexpr int kP3pNewtonIters = 5;     // Newton steps on the depths
constexpr double kP3pOrthoTol = 1e-6;  // a solution with max |R R^T - I| above this is dropped (degenerate triple)
constexpr double kP3pDegenerate = 1e-20;   // a triple with sin^2 of its world triangle's angle at x1, or det^2 of its
                                           // bearings, at most this has no pose (collinear or coincident points,
                                           // coincident or coplanar bearings)

DG_HD double p3p_dot(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
DG_HD void p3p_cross(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// The two roots of x^2 + b x + c (false and no roots when they are not real); r1 is the one of larger magnitude.
DG_HD bool p3p_root2(double b, double c, double* r1, double* r2) {
  const double v = b * b - 4.0 * c;
  if (!(v >= 0.0)) return false;
  const double y = sqrt(v);
  const double q = b < 0.0 ? -0.5 * (b - y) : -0.5 * (b + y);
  *r1 = q;
  *r2 = q != 0.0 ? c / q : 0.0;
  return true;
}

// One real root of x^3 + b x^2 + c x + d: a start on the outer side of the stationary points (or at the inflection),
// then Newton's method.
DG_HD double p3p_cubic_root(double b, double c, double d) {
  double r;
  if (b * b >= 3.0 * c) {
    const double v = sqrt(b * b - 3.0 * c);
    const double t1 = (-b - v) / 3.0;
    const double k1 = ((t1 + b) * t1 + c) * t1 + d;
    if (k1 > 0.0) {
      r = t1 - sqrt(-k1 / (3.0 * t1 + b));
    } else {
      const double t2 = (-b + v) / 3.0;
      const double k2 = ((t2 + b) * t2 + c) * t2 + d;
      r = t2 + sqrt(-k2 / (3.0 * t2 + b));
    }
  } else {
    r = -b / 3.0;
    if (fabs((3.0 * r + 2.0 * b) * r + c) < 1e-4) r += 1.0;
  }
  for (int i = 0; i < kP3pCubicIters; ++i) {
    const double f = ((r + b) * r + c) * r + d;
    if (i >= 7 && !(fabs(f) > 1e-13)) break;
    const double fp = (3.0 * r + 2.0 * b) * r + c;
    r -= f / fp;
  }
  return r;
}

// Newton's method on the three distance constraints, from l [3]
DG_HD void p3p_refine_depths(double* l, double a12, double a13, double a23, double b12, double b13, double b23) {
  for (int it = 0; it < kP3pNewtonIters; ++it) {
    const double l1 = l[0], l2 = l[1], l3 = l[2];
    const double r1 = l1 * l1 + l2 * l2 + b12 * l1 * l2 - a12;
    const double r2 = l1 * l1 + l3 * l3 + b13 * l1 * l3 - a13;
    const double r3 = l2 * l2 + l3 * l3 + b23 * l2 * l3 - a23;
    if (r1 == 0.0 && r2 == 0.0 && r3 == 0.0) break;
    // J = [[p, q, 0], [r, 0, s], [0, u, w]]
    const double p = 2.0 * l1 + b12 * l2, q = 2.0 * l2 + b12 * l1;
    const double r = 2.0 * l1 + b13 * l3, s = 2.0 * l3 + b13 * l1;
    const double u = 2.0 * l2 + b23 * l3, w = 2.0 * l3 + b23 * l2;
    const double det = -(p * s * u) - q * r * w;
    if (det == 0.0) break;
    const double d1 = (-(s * u) * r1 - q * w * r2 + q * s * r3) / det;
    const double d2 = (-(r * w) * r1 + p * w * r2 - p * s * r3) / det;
    const double d3 = (r * u * r1 - p * u * r2 - q * r * r3) / det;
    const double n1 = l1 - d1, n2 = l2 - d2, n3 = l3 - d3;
    if (!(fabs(n1) + fabs(n2) + fabs(n3) < INFINITY)) break;
    l[0] = n1; l[1] = n2; l[2] = n3;
  }
}

// The eigenvectors v1, v2 (unit, third component positive) of the symmetric rank-2 matrix A [6] = (A00, A01, A02, A11,
// A12, A22) for its two eigenvalues e1, e2 other than 0, |e1| >= |e2|.  false when they are not real.
DG_HD bool p3p_eig_rank2(const double* A, double* v1, double* v2, double* e1, double* e2) {
  const double a00 = A[0], a01 = A[1], a02 = A[2], a11 = A[3], a12 = A[4], a22 = A[5];
  const double b = -a00 - a11 - a22;
  const double c = -(a01 * a01) - a02 * a02 - a12 * a12 + a00 * (a11 + a22) + a11 * a22;
  double x1, x2;
  if (!p3p_root2(b, c, &x1, &x2)) return false;
  if (fabs(x1) < fabs(x2)) { const double tmp = x1; x1 = x2; x2 = tmp; }
  *e1 = x1; *e2 = x2;
  const double pr0 = a01 * a12 - a02 * a11, pr1 = a01 * a02 - a00 * a12;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const double e = k == 0 ? x1 : x2;
    double* v = k == 0 ? v1 : v2;
    const double det = e * e - e * (a00 + a11) + a00 * a11 - a01 * a01;
    const double c1 = (e * a02 + pr0) / det, c2 = (e * a12 + pr1) / det;
    const double inv = 1.0 / sqrt(c1 * c1 + c2 * c2 + 1.0);
    v[0] = c1 * inv; v[1] = c2 * inv; v[2] = inv;
  }
  return true;
}

DG_HD bool p3p_finite(double v) { return fabs(v) < INFINITY; }

// Poses x ~ R X + t (R [9] row-major, t [3]) of bearings y [3][3] (unit) and world points X [3][3]: 0 to 4 of them in
// R [4][9], t [4][3], each with positive depths l_i for its three points and finite entries.  A degenerate triple
// (collinear or coincident points, coincident bearings) has none.
DG_HDN int p3p_lambda_twist(const double* y, const double* X, double* R, double* t) {
  const double* y1 = y; const double* y2 = y + 3; const double* y3 = y + 6;
  const double* x1 = X; const double* x2 = X + 3; const double* x3 = X + 6;
  const double b12 = -2.0 * p3p_dot(y1, y2), b13 = -2.0 * p3p_dot(y1, y3), b23 = -2.0 * p3p_dot(y2, y3);
  double d12[3], d13[3], d23[3], dx[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) { d12[i] = x1[i] - x2[i]; d13[i] = x1[i] - x3[i]; d23[i] = x2[i] - x3[i]; }
  p3p_cross(d12, d13, dx);
  const double a12 = p3p_dot(d12, d12), a13 = p3p_dot(d13, d13), a23 = p3p_dot(d23, d23);
  double yx[3];
  p3p_cross(y2, y3, yx);
  const double vol = p3p_dot(y1, yx);
  if (!(p3p_dot(dx, dx) > kP3pDegenerate * a12 * a13) || !(vol * vol > kP3pDegenerate)) return 0;
  const double c31 = -0.5 * b13, c23 = -0.5 * b23, c12 = -0.5 * b12;
  const double blob = c12 * c23 * c31 - 1.0;
  const double s31 = 1.0 - c31 * c31, s23 = 1.0 - c23 * c23, s12 = 1.0 - c12 * c12;
  // det(D1 - g D2) = a23 (p3 g^3 + p2 g^2 + p1 g + p0)
  const double p3 = a13 * (a23 * s31 - a13 * s23);
  const double p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23 + a23 * (a23 - a12) * s31;
  const double p1 = a23 * (a13 - a23) * s12 - a12 * a12 * s23 - 2.0 * a12 * (blob * a23 + a13 * s23);
  const double p0 = a12 * (a12 * s23 - a23 * s12);
  const double g = fabs(p3) >= fabs(p0) ? p3p_cubic_root(p2 / p3, p1 / p3, p0 / p3)
                                        : 1.0 / p3p_cubic_root(p1 / p0, p2 / p0, p3 / p0);
  // D0 = D1 - g D2 (upper triangle by rows)
  const double A[6] = {a23 * (1.0 - g), a23 * b12 * 0.5, a23 * b13 * g * -0.5,
                       a23 - a12 + a13 * g, b23 * (a13 * g - a12) * 0.5, g * (a13 - a23) - a12};
  double v1[3], v2[3], e1, e2;
  if (!p3p_eig_rank2(A, v1, v2, &e1, &e2)) return 0;
  const double sv = sqrt(fmax(0.0, -e2 / e1));
  double L[4][3];
  int m = 0;
#pragma unroll
  for (int side = 0; side < 2; ++side) {      // the two planes v1 . l = +-sv (v2 . l)
    const double s = side == 0 ? sv : -sv;
    const double w2 = 1.0 / (s * v2[0] - v1[0]);
    const double w0 = (v1[1] - s * v2[1]) * w2;
    const double w1 = (v1[2] - s * v2[2]) * w2;
    const double ia = 1.0 / ((a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12);
    const double qb = (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13)) * ia;
    const double qc = ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13) * ia;
    double tau[2];
    if (!p3p_root2(qb, qc, tau, tau + 1)) continue;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      if (!(tau[j] > 0.0)) continue;
      const double d = a23 / (tau[j] * (b23 + tau[j]) + 1.0);
      if (!(d > 0.0)) continue;
      const double l2 = sqrt(d);
      const double l3 = tau[j] * l2;
      const double l1 = w0 * l2 + w1 * l3;
      if (!(l1 > 0.0)) continue;
      L[m][0] = l1; L[m][1] = l2; L[m][2] = l3;
      ++m;
    }
  }
  // [d12, d13, d12 x d13]^-1: its rows are the cross products of its columns over its determinant
  double Xi[9];
  p3p_cross(d13, dx, Xi);
  p3p_cross(dx, d12, Xi + 3);
  p3p_cross(d12, d13, Xi + 6);
  const double det = p3p_dot(d12, Xi);
#pragma unroll
  for (int i = 0; i < 9; ++i) Xi[i] = Xi[i] / det;
  int n = 0;
  for (int k = 0; k < m; ++k) {
    double l[3] = {L[k][0], L[k][1], L[k][2]};
    p3p_refine_depths(l, a12, a13, a23, b12, b13, b23);
    if (!(l[0] > 0.0 && l[1] > 0.0 && l[2] > 0.0)) continue;
    double yd1[3], yd2[3], yc[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) { yd1[i] = y1[i] * l[0] - y2[i] * l[1]; yd2[i] = y1[i] * l[0] - y3[i] * l[2]; }
    p3p_cross(yd1, yd2, yc);
    double* Rk = R + 9 * n;
    double* tk = t + 3 * n;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) Rk[3 * i + j] = yd1[i] * Xi[j] + yd2[i] * Xi[3 + j] + yc[i] * Xi[6 + j];
#pragma unroll
    for (int i = 0; i < 3; ++i) tk[i] = y1[i] * l[0] - (Rk[3 * i] * x1[0] + Rk[3 * i + 1] * x1[1] + Rk[3 * i + 2] * x1[2]);
    bool ok = true;
#pragma unroll
    for (int i = 0; i < 9; ++i) ok = ok && p3p_finite(Rk[i]);
#pragma unroll
    for (int i = 0; i < 3; ++i) ok = ok && p3p_finite(tk[i]);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = i; j < 3; ++j) {
        const double v = Rk[3 * i] * Rk[3 * j] + Rk[3 * i + 1] * Rk[3 * j + 1] + Rk[3 * i + 2] * Rk[3 * j + 2] -
                         (i == j ? 1.0 : 0.0);
        ok = ok && fabs(v) <= kP3pOrthoTol;
      }
    if (ok) ++n;
  }
  return n;
}

}  // namespace dg
