// rotation_averaging.h -- per-thread pieces of the rotation averaging (rotation_averaging.cu): the validity and
// preparation of an edge's relative rotation, the composition along a spanning-tree edge, the edge residual and its log
// map, the IRLS weights and the update of a view.  Host-compilable: tests/rotation_averaging_host.cpp builds it with
// g++ and tests/rotation_averaging_np.py restates every function here in numpy.
//
// Edge e = (i, j) carries R_e with x_j ~ R_e x_i, so R_e ~ R_j R_i^T for world-to-camera rotations R_v.  The residual
// of e is dR_e = R_j^T R_e R_i and r_e = log dR_e; a view moves by a right perturbation R_v <- R_v exp([w_v]x), which
// changes r_e by -w_j + w_i to first order.
#pragma once
#include "common.h"
#include "pose_refine.h"
#include "absolute_pose.h"

namespace dg {

constexpr double kRaSmall = 1e-4;        // below this angle the log map takes its Taylor series
constexpr double kRaNearPi = 1e-3;       // within this of pi the axis comes from the symmetric part
constexpr double kRaL1Floor = 1e-3;      // the smallest angle an L1 weight 1 / theta divides by
constexpr double kRaMinDet = 0.5;        // det R_e at most this (a failed pose's R = 0 among them): not an edge

// Whether R_e [9] is finite with det R_e > kRaMinDet
DG_HD bool ra_edge_ok(const double* R) {
  for (int k = 0; k < 9; ++k)
    if (!(fabs(R[k]) < INFINITY)) return false;
  const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) +
                     R[2] * (R[3] * R[7] - R[4] * R[6]);
  return det > kRaMinDet;
}

// A valid R_e as the estimator uses it: re-orthonormalised when it drifts more than kPrOrthoTol
DG_HD void ra_prepare(double* R) {
  if (pr_ortho_drift(R) > kPrOrthoTol) pr_orthonormalise(R);
}

// C = A^T B (row-major)
DG_HD void ra_mul3_tn(const double* A, const double* B, double* C) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
}

// The child's rotation from its tree parent's Rp across edge e = (i, j): R_j = R_e R_i when the child is j, R_i =
// R_e^T R_j when it is i
DG_HD void ra_compose(const double* Re, const double* Rp, bool child_is_j, double* Rc) {
  if (child_is_j) pr_mul3(Re, Rp, Rc);
  else ra_mul3_tn(Re, Rp, Rc);
}

// dR = R_j^T (R_e R_i)
DG_HD void ra_relative(const double* Ri, const double* Rj, const double* Re, double* dR) {
  double T[9];
  pr_mul3(Re, Ri, T);
  ra_mul3_tn(Rj, T, dR);
}

// r = log dR [3] of a rotation matrix, and theta = |r| in [0, pi].  With a = (dR32 - dR23, dR13 - dR31, dR21 -
// dR12) (1-based; 2 sin theta times the axis): theta = atan2(|a|, tr dR - 1); r = theta / (2 sin theta) a, by its
// Taylor series below kRaSmall; within kRaNearPi of pi the axis is the largest-diagonal column of S - cos(theta) I,
// S = (dR + dR^T) / 2 = cos(theta) I + (1 - cos(theta)) n n^T, normalised and signed as a (any sign at theta = pi).
// Finite for every rotation.
DG_HD double ra_log(const double* dR, double* r) {
  const double a[3] = {dR[7] - dR[5], dR[2] - dR[6], dR[3] - dR[1]};
  const double s = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
  const double c2 = dR[0] + dR[4] + dR[8] - 1.0;         // 2 cos theta
  const double th = atan2(s, c2);
  if (th < kRaSmall) {
    const double t2 = th * th;
    const double f = 0.5 * (1.0 + t2 / 6.0 + 7.0 * t2 * t2 / 360.0);
    r[0] = f * a[0]; r[1] = f * a[1]; r[2] = f * a[2];
  } else if (th <= M_PI - kRaNearPi) {
    const double f = th / (2.0 * sin(th));
    r[0] = f * a[0]; r[1] = f * a[1]; r[2] = f * a[2];
  } else {
    const double c = 0.5 * c2;
    const int k = (dR[0] >= dR[4] && dR[0] >= dR[8]) ? 0 : (dR[4] >= dR[8] ? 1 : 2);
    double n[3];
#pragma unroll
    for (int m = 0; m < 3; ++m) n[m] = 0.5 * (dR[3 * m + k] + dR[3 * k + m]) - (m == k ? c : 0.0);
    const double inv = 1.0 / sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
    const double sg = (n[0] * a[0] + n[1] * a[1] + n[2] * a[2]) < 0.0 ? -inv : inv;
    r[0] = th * sg * n[0]; r[1] = th * sg * n[1]; r[2] = th * sg * n[2];
  }
  return th;
}

// The IRLS weight of an edge with residual angle theta: phase 0 (L1, Weiszfeld) 1 / max(theta, kRaL1Floor); phase 1
// (Geman-McClure, rho(theta) = sig2 theta^2 / (sig2 + theta^2)) (sig2 / (sig2 + theta^2))^2
DG_HD double ra_weight(int phase, double th, double sig2) {
  if (phase == 0) return 1.0 / (th > kRaL1Floor ? th : kRaL1Floor);
  const double q = sig2 / (sig2 + th * th);
  return q * q;
}

// R2 = R exp([w]x) = exp([R w]x) R (ap_step's left step), re-orthonormalised when it drifts more than kPrOrthoTol
DG_HD void ra_update(const double* R, const double* w, double* R2) {
  double P[12], D[6], P2[12];
#pragma unroll
  for (int k = 0; k < 9; ++k) P[k] = R[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    P[9 + k] = 0.0;
    D[k] = R[3 * k] * w[0] + R[3 * k + 1] * w[1] + R[3 * k + 2] * w[2];
    D[3 + k] = 0.0;
  }
  ap_step(P, D, P2);
  if (pr_ortho_drift(P2) > kPrOrthoTol) pr_orthonormalise(P2);
#pragma unroll
  for (int k = 0; k < 9; ++k) R2[k] = P2[k];
}

}  // namespace dg
