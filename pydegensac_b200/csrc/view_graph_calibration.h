// view_graph_calibration.h -- per-thread pieces of the view-graph calibration (view_graph_calibration.cu): the edge
// validity test, an edge's twelve constants from its fundamental matrix, its two Kruppa residuals and their Jacobian,
// the robust weight, and the write-back of a group's focal length.  Host-compilable: tests/view_graph_calibration_host.cpp
// builds it with g++ and tests/view_graph_calibration_np.py restates every function here in numpy.
//
// Edge e = (i, j) carries F with x_j^T F x_i = 0.  With K0 the start intrinsics of a view's group and K = K0 D,
// D = diag(e^theta, e^theta, 1), G = K0_j^T F K0_i is the fundamental matrix of calibration D_i, D_j, whose dual image
// of the absolute conic is omega = D D^T = diag(e^{2 theta}, e^{2 theta}, 1).  From G = U S V^T (unit Frobenius norm,
// s1 >= s2 >= s3) the simplified Kruppa equations (Hartley, PAMI 1997) say A ~ B with
//   A = (s1^2 v1^T w_i v1, s1 s2 v1^T w_i v2, s2^2 v2^T w_i v2),  B = (u2^T w_j u2, -u1^T w_j u2, u1^T w_j u1),
// each A_k = alpha_k e^{2 theta_i} + beta_k and each B_k = gamma_k e^{2 theta_j} + delta_k.
#pragma once
#include "common.h"
#include "la.h"

namespace dg {

constexpr double kVgMinS2 = 1e-6;        // s2 at most this share of s1: F is too close to rank 1 to be an edge
// An edge's constants: alpha [3], beta [3], gamma [3], delta [3]
constexpr int kVgAlpha = 0, kVgBeta = 3, kVgGamma = 6, kVgDelta = 9, kVgConsts = 12;

// Whether a group's start intrinsics (f0, cx, cy, k1, k2) are finite with f0 > 0
DG_HD bool vg_intrinsics_ok(const double* k) {
  for (int m = 0; m < 5; ++m)
    if (!(fabs(k[m]) < INFINITY)) return false;
  return k[0] > 0.0;
}

// Whether the pair (i, j) over n_views views, with view groups gi, gj over n_groups groups, can be an edge: i != j,
// both views and both groups in range, the mask set and F [9] finite (the intrinsics and the rank are tested apart)
DG_HD bool vg_edge_ok(int i, int j, int n_views, int gi, int gj, int n_groups, bool mask_set, const double* F) {
  if (i == j || i < 0 || j < 0 || i >= n_views || j >= n_views || !mask_set) return false;
  if (gi < 0 || gj < 0 || gi >= n_groups || gj >= n_groups) return false;
  for (int m = 0; m < 9; ++m)
    if (!(fabs(F[m]) < INFINITY)) return false;
  return true;
}

// The constants c [kVgConsts] of F [9] between the start intrinsics ki of view i and kj of view j; false (c not
// written) when G has no finite non-zero norm or s2 <= kVgMinS2 s1
DG_HD bool vg_constants(const double* F, const double* ki, const double* kj, double* c) {
  double T[9], G[9];
#pragma unroll
  for (int r = 0; r < 3; ++r) {                      // T = F K0_i
    T[3 * r] = F[3 * r] * ki[0];
    T[3 * r + 1] = F[3 * r + 1] * ki[0];
    T[3 * r + 2] = F[3 * r] * ki[1] + F[3 * r + 1] * ki[2] + F[3 * r + 2];
  }
#pragma unroll
  for (int m = 0; m < 3; ++m) {                      // G = K0_j^T T
    G[m] = kj[0] * T[m];
    G[3 + m] = kj[0] * T[3 + m];
    G[6 + m] = kj[1] * T[m] + kj[2] * T[3 + m] + T[6 + m];
  }
  double n2 = 0.0;
#pragma unroll
  for (int m = 0; m < 9; ++m) n2 += G[m] * G[m];
  const double n = sqrt(n2);
  if (!(n > 0.0) || !(n < INFINITY)) return false;
  const double inv = 1.0 / n;
#pragma unroll
  for (int m = 0; m < 9; ++m) G[m] *= inv;
  double Gv[9], V[9], sv[3];
  svd3_onesided(G, Gv, V, sv);                       // Gv = G V, its columns s_k u_k
  int o0 = 0, o1 = 1, o2 = 2, t;                     // singular values, largest first (pose_candidates' order)
  if (sv[o1] > sv[o0]) { t = o0; o0 = o1; o1 = t; }
  if (sv[o2] > sv[o0]) { t = o0; o0 = o2; o2 = t; }
  if (sv[o2] > sv[o1]) { t = o1; o1 = o2; o2 = t; }
  const double s1 = sv[o0], s2 = sv[o1];
  if (!(s2 > kVgMinS2 * s1)) return false;
  const double v1[3] = {V[o0], V[3 + o0], V[6 + o0]}, v2[3] = {V[o1], V[3 + o1], V[6 + o1]};
  const double i1 = 1.0 / s1, i2 = 1.0 / s2;
  const double u1[3] = {Gv[o0] * i1, Gv[3 + o0] * i1, Gv[6 + o0] * i1};
  const double u2[3] = {Gv[o1] * i2, Gv[3 + o1] * i2, Gv[6 + o1] * i2};
  c[kVgAlpha] = s1 * s1 * (v1[0] * v1[0] + v1[1] * v1[1]);
  c[kVgAlpha + 1] = s1 * s2 * (v1[0] * v2[0] + v1[1] * v2[1]);
  c[kVgAlpha + 2] = s2 * s2 * (v2[0] * v2[0] + v2[1] * v2[1]);
  c[kVgBeta] = s1 * s1 * (v1[2] * v1[2]);
  c[kVgBeta + 1] = s1 * s2 * (v1[2] * v2[2]);
  c[kVgBeta + 2] = s2 * s2 * (v2[2] * v2[2]);
  c[kVgGamma] = u2[0] * u2[0] + u2[1] * u2[1];
  c[kVgGamma + 1] = -(u1[0] * u2[0] + u1[1] * u2[1]);
  c[kVgGamma + 2] = u1[0] * u1[0] + u1[1] * u1[1];
  c[kVgDelta] = u2[2] * u2[2];
  c[kVgDelta + 1] = -(u1[2] * u2[2]);
  c[kVgDelta + 2] = u1[2] * u1[2];
  return true;
}

// The residuals r [2] of an edge with constants c at (theta_i, theta_j), and when J is not null their Jacobian J [4]
// row-major, J = [[dr1/dti, dr1/dtj], [dr2/dti, dr2/dtj]].  Returns s = r1^2 + r2^2.
//   r1 = (A0 B2 - A2 B0) / (A0 B2 + A2 B0),  r2 = (A1 / sqrt(A0 A2) - B1 / sqrt(B0 B2)) / 2
DG_HD double vg_residuals(const double* c, double ti, double tj, double* r, double* J) {
  const double a = exp(2.0 * ti), b = exp(2.0 * tj);
  double A[3], B[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    A[k] = c[kVgAlpha + k] * a + c[kVgBeta + k];
    B[k] = c[kVgGamma + k] * b + c[kVgDelta + k];
  }
  const double P = A[0] * B[2], Q = A[2] * B[0], den = P + Q;
  const double qa = 1.0 / sqrt(A[0] * A[2]), qb = 1.0 / sqrt(B[0] * B[2]);
  const double ra = A[1] * qa, rb = B[1] * qb;
  r[0] = (P - Q) / den;
  r[1] = 0.5 * (ra - rb);
  if (J) {
    double dA[3], dB[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      dA[k] = 2.0 * c[kVgAlpha + k] * a;
      dB[k] = 2.0 * c[kVgGamma + k] * b;
    }
    const double id2 = 2.0 / (den * den);
    J[0] = id2 * (Q * (dA[0] * B[2]) - P * (dA[2] * B[0]));
    J[1] = id2 * (Q * (A[0] * dB[2]) - P * (A[2] * dB[0]));
    J[2] = 0.5 * (dA[1] * qa - 0.5 * ra * (dA[0] / A[0] + dA[2] / A[2]));
    J[3] = -0.5 * (dB[1] * qb - 0.5 * rb * (dB[0] / B[0] + dB[2] / B[2]));
  }
  return r[0] * r[0] + r[1] * r[1];
}

// The Cauchy loss rho(s) = sig2 log(1 + s / sig2) of an edge's s and its IRLS weight rho'(s) = 1 / (1 + s / sig2)
// (bundle_adjust.h's ba_rho and ba_weight); sig2 = 0: the squared loss, weight 1
DG_HD double vg_rho(double s, double sig2) { return sig2 > 0.0 ? sig2 * log1p(s / sig2) : s; }
DG_HD double vg_weight(double s, double sig2) { return sig2 > 0.0 ? 1.0 / (1.0 + s / sig2) : 1.0; }

// An edge's term of the cost at a trial point: rho(s), +inf when s is not finite
DG_HD double vg_cost(double s, double sig2) { return s < INFINITY ? vg_rho(s, sig2) : INFINITY; }

// Whether a group with (has_edge) or without a used edge is refined at theta: f / f0 = e^theta within [1 / max_ratio,
// max_ratio].  k_out [5] is then k_in with f = f0 e^theta, and otherwise k_in bit for bit.
DG_HD bool vg_write_back(const double* k_in, double theta, bool has_edge, double max_ratio, double* k_out) {
  const double ratio = exp(theta);
  const bool refined = has_edge && ratio >= 1.0 / max_ratio && ratio <= max_ratio;
#pragma unroll
  for (int m = 0; m < 5; ++m) k_out[m] = k_in[m];
  if (refined) k_out[0] = k_in[0] * ratio;
  return refined;
}

}  // namespace dg
