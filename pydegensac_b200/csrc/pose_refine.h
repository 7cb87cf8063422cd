// pose_refine.h -- per-thread pieces of the relative-pose refinement (pose_refine_ragged_kernel, frontend.cu):
// Levenberg-Marquardt on the pixel-domain Sampson residual over the 5-parameter essential manifold.
//
//   F = K2^-T [t]x R K1^-1,   r = (p2^T F p1) / sqrt(s),   s = (F p1)_0^2 + (F p1)_1^2 + (F^T p2)_0^2 + (F^T p2)_1^2
//
// so r^2 is f_resid_sampson (fgeom.h).  Local parameters theta = (w [3], d [2]), re-centred at every accepted step:
// R <- exp([w]x) R,  t <- (t + B d) / |t + B d| with B = (b1, b2) an orthonormal basis of the plane orthogonal to t.
// At theta = 0 the derivatives of E = [t]x R are [t]x [e_k]x R (k = 0, 1, 2) and [b_j]x R (j = 0, 1); r does not
// depend on the scale of F, so the normalisation of t adds no term.  tests/pose_refine_np.py restates every function
// here in numpy.
#pragma once
#include "common.h"
#include "fgeom.h"
#include "la.h"

namespace dg {

constexpr int kPrSums = 21;             // per pass: cost, J^T J (upper triangle by rows, 15), J^T r (5)
constexpr int kPrMinRows = 6;           // fewer rows with mask != 0: the pose is passed through
constexpr double kPrLambda0 = 1e-3, kPrLambdaMin = 1e-12, kPrLambdaMax = 1e8;
constexpr double kPrRelDecrease = 1e-12;   // a trial step that moves the cost by less than this share of it stops
constexpr double kPrOrthoTol = 1e-12;      // largest |R R^T - I| entry left alone after the last accepted step

DG_HD void pr_mul3(const double* A, const double* B, double* C) {   // row-major C = A B
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
DG_HD void pr_skew(const double* v, double* S) {
  S[0] = 0.0; S[1] = -v[2]; S[2] = v[1];
  S[3] = v[2]; S[4] = 0.0; S[5] = -v[0];
  S[6] = -v[1]; S[7] = v[0]; S[8] = 0.0;
}
DG_HD void pr_unit3(double* v) {
  const double inv = 1.0 / sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  v[0] *= inv; v[1] *= inv; v[2] *= inv;
}

// b1 = t x e / |t x e| with e the coordinate axis of t's smallest |component| (the first on ties), b2 = t x b1 / |..|
DG_HD void pr_basis(const double* t, double* b1, double* b2) {
  const double a0 = fabs(t[0]), a1 = fabs(t[1]), a2 = fabs(t[2]);
  const int ax = (a0 <= a1 && a0 <= a2) ? 0 : (a1 <= a2 ? 1 : 2);
  const double e[3] = {ax == 0 ? 1.0 : 0.0, ax == 1 ? 1.0 : 0.0, ax == 2 ? 1.0 : 0.0};
  cross3(b1, t, e);
  pr_unit3(b1);
  cross3(b2, t, b1);
  pr_unit3(b2);
}

// F = A [t]x R Bk with A = K2^-T, Bk = K1^-1 (not normalised)
DG_HD void pr_fundamental(const double* R, const double* t, const double* A, const double* Bk, double* F) {
  double T[9], AT[9], RB[9];
  pr_skew(t, T);
  pr_mul3(A, T, AT);
  pr_mul3(R, Bk, RB);
  pr_mul3(AT, RB, F);
}

// F [9] and dF [5][9], the derivatives of F by (w0, w1, w2, d0, d1) at zero
DG_HD void pr_linearise(const double* R, const double* t, const double* A, const double* Bk, double* F, double* dF) {
  double T[9], AT[9], RB[9], S[9], M[9], b[2][3];
  pr_skew(t, T);
  pr_mul3(A, T, AT);
  pr_mul3(R, Bk, RB);
  pr_mul3(AT, RB, F);
#pragma unroll
  for (int k = 0; k < 3; ++k) {           // A [t]x [e_k]x R Bk
    const double e[3] = {k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0};
    pr_skew(e, S);
    pr_mul3(AT, S, M);
    pr_mul3(M, RB, dF + 9 * k);
  }
  pr_basis(t, b[0], b[1]);
#pragma unroll
  for (int j = 0; j < 2; ++j) {           // A [b_j]x R Bk
    pr_skew(b[j], S);
    pr_mul3(A, S, M);
    pr_mul3(M, RB, dF + 9 * (3 + j));
  }
}

// 9 entries of a linearisation in shared memory at p: p itself, or with kReread (device code) a copy in buf by a read
// that the compiler may not hoist out of the row loop -- 7 x 9 derivatives kept in registers across rows take the
// registers the sums need, and spill.
template <bool kReread>
DG_HD const double* pr_lin9(const double* p, double* buf) {
  if constexpr (kReread && DG_DEVICE_PASS) {
#pragma unroll
    for (int i = 0; i < 9; ++i) buf[i] = *(const volatile double*)(p + i);
    return buf;
  } else {
    return p;
  }
}

// One correspondence at the linearisation (F, dF [N][9]): adds its r^2 to acc[0] (the operations of f_resid_sampson),
// J_k J_l (k <= l) to acc[1 .. N (N + 1) / 2] and J_k r to the N sums after them, with J_k = dr/dtheta_k = dc_k / sqrt(s)
// - c (ds_k / 2) / (s sqrt(s)), dc_k = p2^T dF_k p1, ds_k / 2 = (F p1)_{0,1} . (dF_k p1)_{0,1} + (F^T p2)_{0,1} .
// (dF_k^T p2)_{0,1}.  (N = 7: the fundamental-matrix refinement, refine_f.h.)  With kReread the linearisation is read
// afresh for each row (pr_lin9), as the F refinement needs it.
template <int N, bool kReread = false>
DG_HD void pr_row_n(const double* F, const double* dF, double x1, double y1, double x2, double y2, double* acc) {
  double fbuf[9];
  const FRes q = f_res_terms(pr_lin9<kReread>(F, fbuf), x1, y1, x2, y2);
  const double s = q.rxc * q.rxc + q.ryc * q.ryc + q.rx * q.rx + q.ry * q.ry;
  acc[0] += q.r * q.r / s;
  const double inv = 1.0 / sqrt(s);
  const double r = q.r * inv, w = r * inv * inv;
  double J[N];
#pragma unroll
  for (int k = 0; k < N; ++k) {
    double dbuf[9];
    const double* d = pr_lin9<kReread>(dF + 9 * k, dbuf);
    const double u0 = d[0] * x1 + d[1] * y1 + d[2], u1 = d[3] * x1 + d[4] * y1 + d[5], u2 = d[6] * x1 + d[7] * y1 + d[8];
    const double v0 = d[0] * x2 + d[3] * y2 + d[6], v1 = d[1] * x2 + d[4] * y2 + d[7];
    const double dc = x2 * u0 + y2 * u1 + u2;
    const double hs = q.rx * u0 + q.ry * u1 + q.rxc * v0 + q.ryc * v1;
    J[k] = dc * inv - w * hs;
  }
  int m = 1;
#pragma unroll
  for (int k = 0; k < N; ++k)
#pragma unroll
    for (int l = k; l < N; ++l) acc[m++] += J[k] * J[l];
#pragma unroll
  for (int k = 0; k < N; ++k) acc[1 + N * (N + 1) / 2 + k] += J[k] * r;
}
DG_HD void pr_row(const double* F, const double* dF, double x1, double y1, double x2, double y2, double* acc) {
  pr_row_n<5>(F, dF, x1, y1, x2, y2, acc);
}

// D [N] of (H + lam diag(H)) D = -g by Cholesky; H: upper triangle by rows [N (N + 1) / 2].  false at a pivot that is
// not positive.  (N = 8: the homography refinement, refine_h.h.)
template <int N>
DG_HD bool pr_cholesky_solve(const double* H, const double* g, double lam, double* D) {
  double L[N][N];
  int m = 0;
#pragma unroll
  for (int k = 0; k < N; ++k)
#pragma unroll
    for (int l = k; l < N; ++l) { L[l][k] = (l == k) ? H[m] + lam * H[m] : H[m]; ++m; }
#pragma unroll
  for (int j = 0; j < N; ++j) {
    double d = L[j][j];
#pragma unroll
    for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
    if (!(d > 0.0)) return false;
    L[j][j] = sqrt(d);
#pragma unroll
    for (int i = j + 1; i < N; ++i) {
      double v = L[i][j];
#pragma unroll
      for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
      L[i][j] = v / L[j][j];
    }
  }
  double y[N];
#pragma unroll
  for (int i = 0; i < N; ++i) {
    double v = -g[i];
#pragma unroll
    for (int k = 0; k < i; ++k) v -= L[i][k] * y[k];
    y[i] = v / L[i][i];
  }
#pragma unroll
  for (int i = N - 1; i >= 0; --i) {
    double v = y[i];
#pragma unroll
    for (int k = i + 1; k < N; ++k) v -= L[k][i] * D[k];
    D[i] = v / L[i][i];
  }
  return true;
}
DG_HD bool pr_solve(const double* H, const double* g, double lam, double* D) { return pr_cholesky_solve<5>(H, g, lam, D); }

// The factor / apply pair of the same Cholesky, for one matrix and many right-hand sides (N = 6: the block-Jacobi
// preconditioner of bundle_adjust_pcg.cu).  pr_cholesky_factor: A (upper triangle by rows [N (N + 1) / 2]) = L L^T,
// L (lower triangle by rows, L[i][k] at i (i + 1) / 2 + k); false at a pivot that is not positive.
// pr_cholesky_apply: x = A^-1 b from L (x may alias b).
template <int N>
DG_HD bool pr_cholesky_factor(const double* A, double* Lp) {
  double L[N][N];
  int m = 0;
#pragma unroll
  for (int k = 0; k < N; ++k)
#pragma unroll
    for (int l = k; l < N; ++l) L[l][k] = A[m++];
#pragma unroll
  for (int j = 0; j < N; ++j) {
    double d = L[j][j];
#pragma unroll
    for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
    if (!(d > 0.0)) return false;
    L[j][j] = sqrt(d);
#pragma unroll
    for (int i = j + 1; i < N; ++i) {
      double v = L[i][j];
#pragma unroll
      for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
      L[i][j] = v / L[j][j];
    }
  }
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int k = 0; k <= i; ++k) Lp[i * (i + 1) / 2 + k] = L[i][k];
  return true;
}
template <int N>
DG_HD void pr_cholesky_apply(const double* Lp, const double* b, double* x) {
  double y[N];
#pragma unroll
  for (int i = 0; i < N; ++i) {
    double v = b[i];
#pragma unroll
    for (int k = 0; k < i; ++k) v -= Lp[i * (i + 1) / 2 + k] * y[k];
    y[i] = v / Lp[i * (i + 1) / 2 + i];
  }
#pragma unroll
  for (int i = N - 1; i >= 0; --i) {
    double v = y[i];
#pragma unroll
    for (int k = i + 1; k < N; ++k) v -= Lp[k * (k + 1) / 2 + i] * y[k];
    y[i] = v / Lp[i * (i + 1) / 2 + i];
  }
#pragma unroll
  for (int i = 0; i < N; ++i) x[i] = y[i];
}

// The pose D = (w, d) away from (R, t): exp([w]x) = I + (sin a / a) [w]x + (2 sin^2(a/2) / a^2) [w]x^2, a = |w|
DG_HD void pr_step(const double* R, const double* t, const double* D, double* R2, double* t2) {
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
  pr_mul3(E, R, R2);
  double b1[3], b2[3];
  pr_basis(t, b1, b2);
#pragma unroll
  for (int i = 0; i < 3; ++i) t2[i] = t[i] + b1[i] * D[3] + b2[i] * D[4];
  pr_unit3(t2);
}

// Largest |R R^T - I| entry
DG_HD double pr_ortho_drift(const double* R) {
  double worst = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = i; j < 3; ++j) {
      const double v = R[3 * i] * R[3 * j] + R[3 * i + 1] * R[3 * j + 1] + R[3 * i + 2] * R[3 * j + 2] - (i == j ? 1.0 : 0.0);
      worst = fabs(v) > worst ? fabs(v) : worst;
    }
  return worst;
}

// Gram-Schmidt on the rows, the third row their cross product (det +1)
DG_HD void pr_orthonormalise(double* R) {
  pr_unit3(R);
  const double p = R[0] * R[3] + R[1] * R[4] + R[2] * R[5];
#pragma unroll
  for (int i = 0; i < 3; ++i) R[3 + i] -= p * R[i];
  pr_unit3(R + 3);
  cross3(R + 6, R, R + 3);
}

}  // namespace dg
