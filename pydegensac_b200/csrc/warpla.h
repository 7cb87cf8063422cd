// warpla.h -- warp-cooperative small dense solves (one warp, operands in a per-warp shared-memory tile).
//
// The LO and DEGENSAC steps are latency chains of 9x9 eigen-problems and 9x8 null-vector problems; run by a
// single thread they dominate the pair time.  Here one warp does them:
//   * symmetric 9x9 eigen-decomposition by PARALLEL-ORDER Jacobi: in each of the 9 rounds of a sweep the
//     4 disjoint index pairs {(r+k) mod 9, (r-k) mod 9} are rotated at once (36+36 two-element updates
//     spread over the lanes), replacing LAPACK dsyev_ on the reference side (lapwrap.c:67);
//   * Householder QR of the 9 x len (len <= 8) system with one lane per column, giving the vector
//     orthogonal to all columns, replacing CCMATH svduv's "last column of U" (Ftools.c:373,383).
// The code is SPMD over `lane` in [0, W): W = 32 on the device, W = 1 in the host emulation, where every
// strided loop degenerates to the sequential order -- same arithmetic, same results.
#pragma once
#include <stddef.h>
#include "common.h"
#include "la.h"

namespace dg {

struct WarpScratch {
  double A[81];
  double V[81];
  double aux[168];   // second Jacobi buffer (A and V) / DLT rows / Householder vectors
  double cs[16];
};

static_assert(offsetof(WarpScratch, V) == 81 * sizeof(double), "[A|V] must be contiguous");

#if DG_DEVICE_PASS
#define DG_WSYNC() __syncwarp()
DG_ENG inline double wl_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
#else
#define DG_WSYNC() ((void)0)
inline double wl_sum(double v) { return v; }
#endif

#if DG_DEVICE_PASS
DG_ENG inline double dg_rsqrt(double x) { return rsqrt(x); }
#else
inline double dg_rsqrt(double x) { return 1.0 / sqrt(x); }
#endif

// Eigen-decomposition of the symmetric matrix in ws->A (full 9x9 row-major).  On return ws->A holds the
// eigenvalues on its diagonal and column k of ws->V the eigenvector of A[k][k].
// Per round: (1) four lanes compute the rotations of the four disjoint pairs (one sqrt, one division and
// one rsqrt each); (2) every lane rebuilds its entries of J^T A J directly from the four old entries they
// depend on (A is double-buffered between ws->A and ws->aux) and rotates its entries of V.
DG_ENGN void warp_jacobi_eig9(WarpScratch* ws, int lane, int W) {
  // [A | V] lives in ws->A..ws->V (162 contiguous doubles) and ping-pongs with ws->aux
  double* cur = ws->A;
  double* nxt = ws->aux;
  #pragma unroll 1
  for (int t = lane; t < 81; t += W) cur[81 + t] = (t / 9 == t % 9) ? 1.0 : 0.0;
  DG_WSYNC();
  #pragma unroll 1
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0, dia = 0.0;
    #pragma unroll 1
    for (int t = lane; t < 81; t += W) {
      const int r = t / 9, cc = t % 9;
      const double v = cur[t];
      if (r < cc) off += v * v;
      else if (r == cc) dia += v * v;
    }
    off = wl_sum(off);
    dia = wl_sum(dia);
    if (!(off > 4e-30 * dia) || off == 0.0) break;  // off-norm at rounding level: converged
    for (int r = 0; r < 9; ++r) {
      #pragma unroll 1
      for (int k = lane; k < 4; k += W) {
        const int i = (r + k + 1) % 9, j = (r + 9 - k - 1) % 9;
        const int p = i < j ? i : j, q = i < j ? j : i;
        const double apq = cur[p * 9 + q];
        double c = 1.0, s = 0.0;
        if (apq != 0.0) {
          const double zeta = cur[q * 10] - cur[p * 10];
          const double h = sqrt(zeta * zeta + 4.0 * apq * apq);
          const double tt = (zeta >= 0.0 ? 2.0 * apq : -2.0 * apq) / (fabs(zeta) + h);
          c = dg_rsqrt(tt * tt + 1.0);
          s = tt * c;
        }
        ws->cs[2 * k] = c;
        ws->cs[2 * k + 1] = s;
      }
      DG_WSYNC();
      // Index x != r is rotated with partner 2r-x (mod 9): x' = c*x -/+ s*partner (- for the smaller index).
      // new A[i][j] = sum over {i,pi} x {j,pj} of J[a][i] * A[a][b] * J[b][j];  new V[:,j] = c*V[:,j] -/+ s*V[:,pj]
      #pragma unroll 1
      for (int t = lane; t < 162; t += W) {
        const int u = (t < 81) ? t : t - 81;
        const int i = u / 9, j = u % 9;
        int pj = j;
        double cj = 1.0, sj = 0.0;
        if (j != r) {
          const int d = (j - r + 9) % 9;
          const int k = (d <= 4) ? d - 1 : 8 - d;
          pj = (2 * r - j + 18) % 9;
          const double c = ws->cs[2 * k], s = ws->cs[2 * k + 1];
          cj = c;
          sj = (j < pj) ? -s : s;
        }
        if (t < 81) {
          int pi = i;
          double ci = 1.0, si = 0.0;
          if (i != r) {
            const int d = (i - r + 9) % 9;
            const int k = (d <= 4) ? d - 1 : 8 - d;
            pi = (2 * r - i + 18) % 9;
            const double c = ws->cs[2 * k], s = ws->cs[2 * k + 1];
            ci = c;
            si = (i < pi) ? -s : s;
          }
          const double u0 = ci * cur[i * 9 + j] + si * cur[pi * 9 + j];
          const double u1 = ci * cur[i * 9 + pj] + si * cur[pi * 9 + pj];
          nxt[t] = cj * u0 + sj * u1;
        } else {
          nxt[t] = cj * cur[81 + i * 9 + j] + sj * cur[81 + i * 9 + pj];
        }
      }
      DG_WSYNC();
      double* tmp = cur; cur = nxt; nxt = tmp;
    }
  }
  if (cur != ws->A) {
    #pragma unroll 1
    for (int t = lane; t < 162; t += W) ws->A[t] = cur[t];
    DG_WSYNC();
  }
}

#if DG_DEVICE_PASS
DG_ENG inline double shfl_d(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }

// ---------------------------------------------------------------------------------------------
// Device flavour of warp_smallest_eigvec9: lane i (< 9) keeps ROW i of the matrix in registers, pivots and pivot
// rows travel by warp shuffles, the elimination is fully unrolled (~1.3k warp instructions per call; the
// shared-memory version below spent ~10k on index decoding, __syncwarp and shared-memory round trips).
//   * L D L^T of (A - sigma I), sigma = 0 first;
//   * start vector L^-T e_8 (exact null vector when the last pivot vanishes), inverse iteration;
//   * when the iterate still moves by > 1e-5 after two solves (clustered small eigenvalues) the shift is raised to
//     rho - |A x - rho x| (a lower bound of the eigenvalue nearest the Rayleigh quotient rho) and the matrix is
//     refactored: quadratic convergence instead of the Jacobi fallback.  A non-positive pivot of a shifted
//     factorisation means the bound overshot lambda_min: the last good shift is restored.
// On the LO / DEGENSAC matrices of the benchmark scenes: 4.6 solves and 1.4 factorisations per call, no fallback.
// Returns true with the unit eigenvector in ws->cs[0..8]; false (ws->A untouched) sends the caller to Jacobi.
// ---------------------------------------------------------------------------------------------
// One pivot of the L D L^T factorisation (template so that all indices into a[] are literals, cf. pairsolve_step).
template <int K>
__device__ __forceinline__ void eig9_factor_step(double (&a)[9], int lane, double tiny, bool& neg, double& dsel) {
  double dk = shfl_d(a[K], K);
  if (!(dk > tiny)) { dk = tiny; neg = true; }   // singular / negative pivot: regularise (and report)
  const double inv = 1.0 / dk;
  if (lane == K) { a[K] = dk; dsel = dk; }
  const double lik = a[K] * inv;
#pragma unroll
  for (int j = K + 1; j < 9; ++j) {
    const double akj = shfl_d(a[j], K);
    if (lane > K) a[j] = fma(-lik, akj, a[j]);
  }
  if (lane > K) a[K] = lik;
}
__device__ __forceinline__ bool eig9_factor_reg(const double* A, int r, int lane, double sigma, double tiny,
                                                double* T, double (&a)[9], double (&ct)[9], double& dinv) {
  // (a lane-keyed select chain over a[] would be turned into a[lane] -- a dynamic index that drags the array
  //  into local memory; every access keeps a literal index)
  a[0] = A[r * 9 + 0] - ((lane == 0) ? sigma : 0.0); a[1] = A[r * 9 + 1] - ((lane == 1) ? sigma : 0.0);
  a[2] = A[r * 9 + 2] - ((lane == 2) ? sigma : 0.0); a[3] = A[r * 9 + 3] - ((lane == 3) ? sigma : 0.0);
  a[4] = A[r * 9 + 4] - ((lane == 4) ? sigma : 0.0); a[5] = A[r * 9 + 5] - ((lane == 5) ? sigma : 0.0);
  a[6] = A[r * 9 + 6] - ((lane == 6) ? sigma : 0.0); a[7] = A[r * 9 + 7] - ((lane == 7) ? sigma : 0.0);
  a[8] = A[r * 9 + 8] - ((lane == 8) ? sigma : 0.0);
  bool neg = false;
  double dsel = 1.0;
  eig9_factor_step<0>(a, lane, tiny, neg, dsel); eig9_factor_step<1>(a, lane, tiny, neg, dsel);
  eig9_factor_step<2>(a, lane, tiny, neg, dsel); eig9_factor_step<3>(a, lane, tiny, neg, dsel);
  eig9_factor_step<4>(a, lane, tiny, neg, dsel); eig9_factor_step<5>(a, lane, tiny, neg, dsel);
  eig9_factor_step<6>(a, lane, tiny, neg, dsel); eig9_factor_step<7>(a, lane, tiny, neg, dsel);
  eig9_factor_step<8>(a, lane, tiny, neg, dsel);
  // lane i now holds L[i][k] (k < i) and d_i; the transposed factor comes back through shared memory
  dinv = 1.0 / dsel;
  __syncwarp();
  if (lane < 9) {
    double* t = T + lane * 9;
    t[0] = a[0]; t[1] = a[1]; t[2] = a[2]; t[3] = a[3]; t[4] = a[4]; t[5] = a[5]; t[6] = a[6]; t[7] = a[7]; t[8] = a[8];
  }
  __syncwarp();
  ct[0] = T[0 * 9 + r]; ct[1] = T[1 * 9 + r]; ct[2] = T[2 * 9 + r]; ct[3] = T[3 * 9 + r]; ct[4] = T[4 * 9 + r];
  ct[5] = T[5 * 9 + r]; ct[6] = T[6 * 9 + r]; ct[7] = T[7 * 9 + r]; ct[8] = T[8 * 9 + r];      // L[k][i], used for k > i
  return neg;
}

// The residual test accepts ANY eigenpair: a start vector without a component along v_min (L^-T e_8 misses v_min when
// its last entry vanishes) converges to the next eigenvector.  x with Rayleigh quotient rho belongs to the smallest
// eigenvalue (to 32 eps |A|_F) exactly when A - (rho - 32 eps |A|_F) I is positive definite: no non-positive pivot.
__device__ __forceinline__ bool eig9_nothing_below(const double* A, int r, int lane, double rho, double fro, double tiny,
                                                   double* T) {
  double a[9], ct[9], dinv;
  return !eig9_factor_reg(A, r, lane, rho - 32.0 * 2.220446049250313e-16 * sqrt(fro), tiny, T, a, ct, dinv);
}

__device__ __noinline__ bool warp_smallest_eigvec9_reg(WarpScratch* ws, int lane) {
  const bool act = lane < 9;
  const int r = act ? lane : 0;            // idle lanes shadow row 0 (their values are never read)
  const double* A = ws->A;
  double fro = 0.0;
#pragma unroll
  for (int j = 0; j < 9; ++j) { const double v = A[r * 9 + j]; fro += v * v; }
  fro = wl_sum(act ? fro : 0.0);
  if (!((fro > 0.0) && (fro < 1e300))) return false;
  const double tiny = sqrt(fro) * 1e-30;
  double a[9], ct[9], dinv = 1.0, x = 0.0;
  double sigma = 0.0, good = 0.0;
  bool need = true, have_x = false, done = false;
  int nfac = 0, allow_at = 1;
#pragma unroll 1
  for (int it = 0; it < 16 && !done; ++it) {
#pragma unroll 1
    while (need) {
      const bool neg = eig9_factor_reg(A, r, lane, sigma, tiny, ws->aux, a, ct, dinv);
      ++nfac;
      if (sigma > good && neg) { sigma = good; allow_at = it + 2; continue; }   // overshoot: back to the last good shift
      good = sigma;
      need = false;
    }
    if (!have_x) {                           // x = L^-T e_8, normalised
      double y = (lane == 8) ? 1.0 : 0.0;
#pragma unroll
      for (int k = 8; k > 0; --k) {
        const double yk = shfl_d(y, k);
        if (lane < k) y = fma(-ct[k], yk, y);
      }
      if (!act) y = 0.0;
      const double n2 = wl_sum(y * y);
      if (!(n2 > 0.0) || !(n2 < 1e300)) return false;
      x = y * rsqrt(n2);
      have_x = true;
    }
    double y = x;
#pragma unroll
    for (int k = 0; k < 8; ++k) {           // forward substitution, unit lower factor
      const double yk = shfl_d(y, k);
      if (lane > k) y = fma(-a[k], yk, y);
    }
    y *= dinv;
#pragma unroll
    for (int k = 8; k > 0; --k) {           // backward substitution, transposed factor
      const double yk = shfl_d(y, k);
      if (lane < k) y = fma(-ct[k], yk, y);
    }
    if (!act) y = 0.0;
    const double n2 = wl_sum(y * y);
    const double dot = wl_sum(y * x);
    if (!(n2 > 0.0) || !(n2 < 1e300)) return false;
    const double xn = y * ((dot < 0.0 ? -1.0 : 1.0) * rsqrt(n2));
    const double df = xn - x;
    x = xn;
    const double ch = wl_sum(df * df);
    if (ch < 1e-28) { done = true; break; }
    if (it >= allow_at && ch > 1e-10 && nfac < 8) {
      double s = 0.0;
#pragma unroll
      for (int j = 0; j < 9; ++j) s = fma(A[r * 9 + j], shfl_d(x, j), s);
      if (!act) s = 0.0;
      const double rho = wl_sum(s * x);
      const double rr = s - rho * x;
      const double shift = rho - sqrt(wl_sum(rr * rr));
      if (shift > sigma) { sigma = shift; need = true; }
    }
  }
  if (!done) return false;
  // Rayleigh residual against the ORIGINAL matrix
  double s = 0.0;
#pragma unroll
  for (int j = 0; j < 9; ++j) s = fma(A[r * 9 + j], shfl_d(x, j), s);
  if (!act) s = 0.0;
  const double rho = wl_sum(s * x);
  const double rr = s - rho * x;
  const double r2 = wl_sum(rr * rr);
  if (!(r2 <= 1e-28 * fro)) return false;
  if (!eig9_nothing_below(A, r, lane, rho, fro, tiny, ws->aux)) return false;
  if (act) ws->cs[lane] = x;
  __syncwarp();
  return true;
}

// ---------------------------------------------------------------------------------------------
// Inverse iteration on the EXPLICIT inverse.  One warp runs the eigen-solver while the rest of the CTA waits, and a
// lone warp is paid in dependent-instruction latency: the substitution version above spends 16 shuffle + FMA steps and
// three butterflies per solve, ~4 000 dynamic instructions per call (tools/prof_phases.py times it in situ).  Here the factorisation is followed by nine column solves run side by side -- lane i solves
// L D L^T z = e_i entirely in its own registers (the factor is broadcast from shared memory) and keeps z = row i of
// M = (A - sigma I)^-1 -- after which one inverse-iteration step is a single matrix-vector product: nine independent
// shuffles and nine FMAs per lane instead of two sequential triangular sweeps.  Same start vector (M e_8 is parallel to
// L^-T e_8), same convergence rule, same Rayleigh-shift refactorisation for clustered small eigenvalues, and the same
// final test of |A x - rho x| against the ORIGINAL matrix, so a wrong answer cannot get out: failure sends the caller
// to the substitution version / Jacobi.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool eig9_inverse_rows(const double* A, int r, int lane, bool act, double sigma, double tiny,
                                                  double* T, double* Dv, double (&m)[9]) {
  double a[9];
  a[0] = A[r * 9 + 0] - ((lane == 0) ? sigma : 0.0); a[1] = A[r * 9 + 1] - ((lane == 1) ? sigma : 0.0);
  a[2] = A[r * 9 + 2] - ((lane == 2) ? sigma : 0.0); a[3] = A[r * 9 + 3] - ((lane == 3) ? sigma : 0.0);
  a[4] = A[r * 9 + 4] - ((lane == 4) ? sigma : 0.0); a[5] = A[r * 9 + 5] - ((lane == 5) ? sigma : 0.0);
  a[6] = A[r * 9 + 6] - ((lane == 6) ? sigma : 0.0); a[7] = A[r * 9 + 7] - ((lane == 7) ? sigma : 0.0);
  a[8] = A[r * 9 + 8] - ((lane == 8) ? sigma : 0.0);
  bool neg = false;
  double dsel = 1.0;
  eig9_factor_step<0>(a, lane, tiny, neg, dsel); eig9_factor_step<1>(a, lane, tiny, neg, dsel);
  eig9_factor_step<2>(a, lane, tiny, neg, dsel); eig9_factor_step<3>(a, lane, tiny, neg, dsel);
  eig9_factor_step<4>(a, lane, tiny, neg, dsel); eig9_factor_step<5>(a, lane, tiny, neg, dsel);
  eig9_factor_step<6>(a, lane, tiny, neg, dsel); eig9_factor_step<7>(a, lane, tiny, neg, dsel);
  eig9_factor_step<8>(a, lane, tiny, neg, dsel);
  __syncwarp();
  if (act) {
    double* t = T + lane * 9;     // row i: L[i][k] for k < i
    t[0] = a[0]; t[1] = a[1]; t[2] = a[2]; t[3] = a[3]; t[4] = a[4]; t[5] = a[5]; t[6] = a[6]; t[7] = a[7]; t[8] = a[8];
    Dv[lane] = 1.0 / dsel;
  }
  __syncwarp();
  // column r of the inverse: forward sweep (unit lower factor), diagonal, backward sweep (transposed factor); every index
  // into m[] is a literal, every factor entry one broadcast shared-memory load
#pragma unroll
  for (int i = 0; i < 9; ++i) m[i] = (r == i) ? 1.0 : 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k)
#pragma unroll
    for (int i = k + 1; i < 9; ++i) m[i] = fma(-T[i * 9 + k], m[k], m[i]);
#pragma unroll
  for (int i = 0; i < 9; ++i) m[i] *= Dv[i];
#pragma unroll
  for (int k = 8; k > 0; --k)
#pragma unroll
    for (int i = 0; i < k; ++i) m[i] = fma(-T[k * 9 + i], m[k], m[i]);
  return neg;
}

__device__ __noinline__ bool warp_smallest_eigvec9_inv(WarpScratch* ws, int lane) {
  const bool act = lane < 9;
  const int r = act ? lane : 0;            // idle lanes shadow row 0 (their values are never read)
  const double* A = ws->A;
  double* T = ws->aux;
  double* Dv = ws->aux + 81;
  double fro = 0.0;
#pragma unroll
  for (int j = 0; j < 9; ++j) { const double v = A[r * 9 + j]; fro += v * v; }
  fro = wl_sum(act ? fro : 0.0);
  if (!((fro > 0.0) && (fro < 1e300))) return false;
  const double tiny = sqrt(fro) * 1e-30;
  double m[9], x = 0.0, mx2 = 0.0;         // mx2: |M x|^2 of the last step
  double sigma = 0.0, good = 0.0;
  bool need = true, have_x = false, done = false;
  int nfac = 0, allow_at = 1;
#pragma unroll 1
  for (int it = 0; it < 16 && !done; ++it) {
#pragma unroll 1
    while (need) {
      const bool neg = eig9_inverse_rows(A, r, lane, act, sigma, tiny, T, Dv, m);
      ++nfac;
      if (sigma > good && neg) { sigma = good; allow_at = it + 2; continue; }   // overshoot: back to the last good shift
      good = sigma;
      need = false;
    }
    if (!have_x) {                           // x = M e_8 (parallel to L^-T e_8), normalised
      double y = act ? m[8] : 0.0;
      const double n2 = wl_sum(y * y);
      if (!(n2 > 0.0) || !(n2 < 1e300)) return false;
      x = y * rsqrt(n2);
      have_x = true;
    }
    double y0 = m[0] * shfl_d(x, 0), y1 = m[1] * shfl_d(x, 1), y2 = m[2] * shfl_d(x, 2);
    y0 = fma(m[3], shfl_d(x, 3), y0); y1 = fma(m[4], shfl_d(x, 4), y1); y2 = fma(m[5], shfl_d(x, 5), y2);
    y0 = fma(m[6], shfl_d(x, 6), y0); y1 = fma(m[7], shfl_d(x, 7), y1); y2 = fma(m[8], shfl_d(x, 8), y2);
    double y = (y0 + y1) + y2;
    if (!act) y = 0.0;
    double n2 = y * y, dot = y * x;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      n2 += __shfl_xor_sync(0xffffffffu, n2, o);
      dot += __shfl_xor_sync(0xffffffffu, dot, o);
    }
    if (!(n2 > 0.0) || !(n2 < 1e300)) return false;
    mx2 = n2;
    const double xn = y * ((dot < 0.0 ? -1.0 : 1.0) * rsqrt(n2));
    const double df = xn - x;
    x = xn;
    const double ch = wl_sum(df * df);
    if (ch < 1e-28) { done = true; break; }
    if (it >= allow_at && ch > 1e-10 && nfac < 8) {
      double s = 0.0;
#pragma unroll
      for (int j = 0; j < 9; ++j) s = fma(A[r * 9 + j], shfl_d(x, j), s);
      if (!act) s = 0.0;
      const double rho = wl_sum(s * x);
      const double rr = s - rho * x;
      const double shift = rho - sqrt(wl_sum(rr * rr));
      if (shift > sigma) { sigma = shift; need = true; }
    }
  }
  if (!done) return false;
  // Rayleigh residual against the ORIGINAL matrix
  double s = 0.0;
#pragma unroll
  for (int j = 0; j < 9; ++j) s = fma(A[r * 9 + j], shfl_d(x, j), s);
  if (!act) s = 0.0;
  const double rho = wl_sum(s * x);
  const double rr = s - rho * x;
  const double r2 = wl_sum(rr * rr);
  if (!(r2 <= 1e-28 * fro)) return false;
  // M = (A - good I)^-1 has the eigenvalues 1 / (lambda_i - good) > 0, so an x of a larger eigenvalue has
  // trace(M) >= 2 |M x|: a well-separated lambda_min is settled here, the others by the inertia count
  double tr = 0.0;
#pragma unroll
  for (int j = 0; j < 9; ++j) tr += shfl_d(m[j], j);
  if (!(tr > 0.0 && tr * tr <= 1.5625 * mx2) && !eig9_nothing_below(A, r, lane, rho, fro, tiny, ws->aux)) return false;
  if (act) ws->cs[lane] = x;
  __syncwarp();
  return true;
}

// ---------------------------------------------------------------------------------------------
// Device flavour of warp_null_8x9: lane l keeps row (l & 7) of the 8 x 9 system in registers (four redundant
// copies across the warp, so xor-shuffles over 4,2,1 leave every lane with the pivot choice), Gauss-Jordan with
// partial pivoting by ROLE instead of row swaps: the pivot row of column c stays where it is and is marked used.
// ---------------------------------------------------------------------------------------------
// Core on registers: lane l holds row (l & 7) in m[0..8]; on success every lane gets the unit null vector n[0..8]
// (last component positive).
__device__ __forceinline__ bool null_8x9_core(double (&m)[9], int lane, double (&n)[9]) {
  const unsigned full = 0xffffffffu;
  const int r = lane & 7;
  bool used = false;
  int whoarr[8];
#pragma unroll
  for (int col = 0; col < 8; ++col) {
    double mag = used ? -1.0 : fabs(m[col]);
    if (!(mag == mag)) mag = 1e308 * 10.0;   // NaN -> +inf: wins the search and fails the test below
    int who = r;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      const double m2 = __shfl_xor_sync(full, mag, o);
      const int w2 = __shfl_xor_sync(full, who, o);
      if (m2 > mag || (m2 == mag && w2 < who)) { mag = m2; who = w2; }
    }
    if (!(mag > 0.0) || !(mag < 1e300)) return false;
    whoarr[col] = who;
    const double p = shfl_d(m[col], who);
    const double inv = 1.0 / p;
    const double f = m[col];
#pragma unroll
    for (int j = col + 1; j < 9; ++j) {
      const double pj = shfl_d(m[j], who) * inv;
      m[j] = (r == who) ? pj : fma(-f, pj, m[j]);
    }
    if (r == who) used = true;
  }
  double n2 = m[8] * m[8];
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) n2 += __shfl_xor_sync(full, n2, o);
  const double sc = rsqrt(1.0 + n2);
  const double mine = -m[8] * sc;
#pragma unroll
  for (int col = 0; col < 8; ++col) n[col] = shfl_d(mine, whoarr[col]);
  n[8] = sc;
  return true;
}

__device__ __noinline__ bool warp_null_8x9_reg(WarpScratch* ws, int lane) {
  const int r = lane & 7;
  double m[9], n[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) m[j] = ws->A[j * 8 + r];
  if (!null_8x9_core(m, lane, n)) return false;
  __syncwarp();
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < 9; ++j) ws->cs[j] = n[j];
  }
  __syncwarp();
  return true;
}
#endif

// ---------------------------------------------------------------------------------------------
// Eigenvector of the SMALLEST eigenvalue of the symmetric positive semi-definite 9x9 matrix in ws->A, written
// to ws->cs[0..8] (visible to the whole warp on return).  This is all the LSQ fits need (the reference takes
// column `argmin D` of LAPACK dsyev_, Ftools.c:376-389, Htools.c:126-127).
//
// Fast path: L D L^T factorisation (no pivoting: the matrix is a Gram matrix) followed by inverse iteration
// x <- A^-1 x, which converges like (lambda_min / lambda_next)^k -- for an over-determined fit of noisy
// correspondences that ratio is tiny, so 3-5 solves reach rounding level.  The result is accepted only if the
// Rayleigh residual |A x - rho x| <= 1e-14 |A|_F; otherwise (clustered small eigenvalues, breakdown, NaN) the
// parallel-order Jacobi above is used.  Dependent long-latency operations: ~9 divisions + a few solves,
// instead of ~190 (sqrt, div, rsqrt) x 3 for seven Jacobi sweeps.
// ---------------------------------------------------------------------------------------------
#ifdef DG_EIG_STATS
static long g_eig_calls = 0, g_eig_fallbacks = 0, g_eig_iters = 0;
#endif
DG_ENGN void warp_smallest_eigvec9(WarpScratch* ws, int lane, int W) {
#ifdef DG_EIG_STATS
  ++g_eig_calls;
  if (const char* dump = getenv("DG_EIG_DUMP")) { FILE* fp = fopen(dump, "ab"); if (fp) { fwrite(ws->A, sizeof(double), 81, fp); fclose(fp); } }
#endif
#if DG_DEVICE_PASS
#ifndef DG_EIG_SUBST
  if (warp_smallest_eigvec9_inv(ws, lane)) return;
#endif
  if (warp_smallest_eigvec9_reg(ws, lane)) return;
  {
    warp_jacobi_eig9(ws, lane, W);
    DG_WSYNC();
    if (lane == 0) {
      int m = 0;
      for (int i = 1; i < 9; ++i)
        if (ws->A[i * 10] < ws->A[m * 10]) m = i;
      for (int i = 0; i < 9; ++i) ws->cs[i] = ws->V[i * 9 + m];
    }
    DG_WSYNC();
    return;
  }
#endif
  const double* A = ws->A;
  double* L = ws->aux;          // 81: factor (lower triangle), unit diagonal implied
  double* d = ws->aux + 81;     // 9 pivots
  double* x = ws->aux + 90;     // 9 iterate
  double* y = ws->aux + 99;     // 9 work
  double* red = ws->aux + 108;  // scalars
  double fro = 0.0;
#pragma unroll 1
  for (int t = lane; t < 81; t += W) { const double v = A[t]; L[t] = v; fro += v * v; }
  fro = wl_sum(fro);
  DG_WSYNC();
  bool ok = (fro > 0.0) && (fro == fro) && (fro < 1e300);
  const double tiny = sqrt(fro) * 1e-30;
  if (ok) {
    for (int k = 0; k < 9; ++k) {
      double dk = L[k * 10];
      if (!(dk > tiny)) dk = tiny;          // exactly singular / rounding-negative pivot: regularise
      const double inv = 1.0 / dk;
      if (lane == 0) d[k] = dk;
      // trailing update of the lower triangle: L[i][j] -= L[i][k] * L[j][k] / dk   (k < j <= i)
      const int m = 8 - k;                  // trailing size
      const int ntask = m * (m + 1) / 2;
#pragma unroll 1
      for (int t = lane; t < ntask; t += W) {
        int ii = 0;
        while ((ii + 1) * (ii + 2) / 2 <= t) ++ii;
        const int jj = t - ii * (ii + 1) / 2;
        const int i = k + 1 + ii, j = k + 1 + jj;
        L[i * 9 + j] -= (L[i * 9 + k] * inv) * L[j * 9 + k];
      }
      DG_WSYNC();
#pragma unroll 1
      for (int i = k + 1 + lane; i < 9; i += W) L[i * 9 + k] *= inv;
      DG_WSYNC();
    }
#pragma unroll 1
    for (int i = lane; i < 9; i += W) x[i] = 1.0 / 3.0;
    DG_WSYNC();
    double prev_change = 1.0;
#pragma unroll 1
    for (int it = 0; it < 12; ++it) {
#ifdef DG_EIG_STATS
      ++g_eig_iters;
#endif
#pragma unroll 1
      for (int i = lane; i < 9; i += W) y[i] = x[i];
      DG_WSYNC();
      for (int k = 0; k < 8; ++k) {          // forward substitution with the unit lower factor
#pragma unroll 1
        for (int i = k + 1 + lane; i < 9; i += W) y[i] -= L[i * 9 + k] * y[k];
        DG_WSYNC();
      }
#pragma unroll 1
      for (int i = lane; i < 9; i += W) y[i] /= d[i];
      DG_WSYNC();
#pragma unroll 1
      for (int k = 8; k > 0; --k) {          // backward substitution with the transposed factor
#pragma unroll 1
        for (int i = lane; i < k; i += W) y[i] -= L[k * 9 + i] * y[k];
        DG_WSYNC();
      }
      double n2 = 0.0, dot = 0.0;
#pragma unroll 1
      for (int i = lane; i < 9; i += W) { n2 += y[i] * y[i]; dot += y[i] * x[i]; }
      n2 = wl_sum(n2);
      dot = wl_sum(dot);
      if (!(n2 > 0.0) || !(n2 < 1e300)) { ok = false; break; }
      const double sc = (dot < 0.0 ? -1.0 : 1.0) / sqrt(n2);
      double ch = 0.0;
#pragma unroll 1
      for (int i = lane; i < 9; i += W) {
        const double xn = y[i] * sc;
        const double df = xn - x[i];
        ch += df * df;
        x[i] = xn;
      }
      ch = wl_sum(ch);
      DG_WSYNC();
      if (ch < 1e-31) break;                 // iterate unchanged to rounding level
      if (it >= 6 && ch > 0.25 * prev_change) { ok = false; break; }   // slow: clustered eigenvalues -> Jacobi
      prev_change = ch;
    }
  }
  if (ok) {   // Rayleigh residual against the ORIGINAL matrix
    double rho = 0.0;
#pragma unroll 1
    for (int i = lane; i < 9; i += W) {
      double s = 0.0;
      for (int j = 0; j < 9; ++j) s += A[i * 9 + j] * x[j];
      y[i] = s;
      rho += s * x[i];
    }
    rho = wl_sum(rho);
    DG_WSYNC();
    double r2 = 0.0;
#pragma unroll 1
    for (int i = lane; i < 9; i += W) { const double r = y[i] - rho * x[i]; r2 += r * r; }
    r2 = wl_sum(r2);
    ok = (r2 <= 1e-28 * fro);
  }
  DG_WSYNC();
  if (ok) {
#pragma unroll 1
    for (int i = lane; i < 9; i += W) ws->cs[i] = x[i];
    DG_WSYNC();
    return;
  }
#ifdef DG_EIG_STATS
  ++g_eig_fallbacks;
#endif
  warp_jacobi_eig9(ws, lane, W);
  DG_WSYNC();
  if (lane == 0) {
    int m = 0;
    for (int i = 1; i < 9; ++i)
      if (ws->A[i * 10] < ws->A[m * 10]) m = i;
    for (int i = 0; i < 9; ++i) ws->cs[i] = ws->V[i * 9 + m];
  }
  DG_WSYNC();
}

// Eigenvector of the smallest eigenvalue of the symmetric matrix whose lower triangle (row-major packed,
// 45 entries: (0,0),(1,0),(1,1),(2,0)...) is in `packed`; result in ws->cs[0..8] (visible after DG_WSYNC).
DG_ENGN void warp_min_eigvec9_packed(WarpScratch* ws, const double* packed, int lane, int W) {
#pragma unroll 1
  for (int t = lane; t < 45; t += W) {
    int i = 0;
    while ((i + 1) * (i + 2) / 2 <= t) ++i;
    const int j = t - i * (i + 1) / 2;
    const double v = packed[t];
    ws->A[9 * i + j] = v;
    ws->A[9 * j + i] = v;
  }
  DG_WSYNC();
  warp_smallest_eigvec9(ws, lane, W);
}

// ---------------------------------------------------------------------------------------------
// Unit null vector of the 8 x 9 system whose rows are the 8 columns of the 9 x 8 row-major matrix Z in
// ws->A[0..72) (i.e. the vector orthogonal to all eight correspondences' coefficient columns), by Gauss-Jordan
// elimination with partial pivoting spread over the lanes (every lane owns 2-3 matrix entries; per pivot:
// search, one division per lane, one fused update).  ~8 dependent divisions instead of the ~16 sqrt/div plus
// long dot-product chains of the Householder route below.  Returns false (all lanes) when a pivot vanishes
// (rank-deficient sample): the caller then uses the Householder route.  Result in ws->cs[0..8].
// ---------------------------------------------------------------------------------------------
DG_ENGN bool warp_null_8x9(WarpScratch* ws, int lane, int W) {
#if DG_DEVICE_PASS
  return warp_null_8x9_reg(ws, lane);
#endif
  double* M = ws->aux;          // 8 x 9 row-major working copy (row = correspondence)
  double* mult = ws->aux + 80;  // multipliers of the current pivot column
  int* piv = reinterpret_cast<int*>(ws->aux + 96);
#pragma unroll 1
  for (int t = lane; t < 72; t += W) {
    const int r = t / 9, cc = t % 9;
    M[t] = ws->A[cc * 8 + r];
  }
  DG_WSYNC();
  bool ok = true;
  for (int col = 0; col < 8; ++col) {
    if (lane == 0) {
      int best = col;
      double mag = fabs(M[col * 9 + col]);
#pragma unroll
      for (int r = 1; r < 8; ++r) {
        const int rr = col + r;
        if (rr < 8) {
          const double v = fabs(M[rr * 9 + col]);
          if (v > mag) { mag = v; best = rr; }
        }
      }
      piv[0] = (mag > 0.0 && mag == mag) ? best : -1;
    }
    DG_WSYNC();
    const int best = piv[0];
    if (best < 0) { ok = false; break; }
    // swap rows col <-> best, scale the pivot row, publish the multipliers
    const double p = M[best * 9 + col];
#pragma unroll 1
    for (int cc = lane; cc < 9; cc += W) {
      const double a = M[col * 9 + cc], b = M[best * 9 + cc];
      M[best * 9 + cc] = a;
      M[col * 9 + cc] = b / p;
    }
    DG_WSYNC();
#pragma unroll 1
    for (int r = lane; r < 8; r += W) mult[r] = M[r * 9 + col];
    DG_WSYNC();
#pragma unroll 1
    for (int t = lane; t < 72; t += W) {
      const int r = t / 9, cc = t % 9;
      if (r != col && cc >= col) M[t] -= mult[r] * M[col * 9 + cc];
    }
    DG_WSYNC();
  }
  if (ok) {
    double n2 = 1.0;
#pragma unroll
    for (int r = 0; r < 8; ++r) n2 += M[r * 9 + 8] * M[r * 9 + 8];
    const double sc = 1.0 / sqrt(n2);
    DG_WSYNC();
#pragma unroll 1
    for (int i = lane; i < 9; i += W) ws->cs[i] = (i < 8) ? -M[i * 9 + 8] * sc : sc;
  }
  DG_WSYNC();
  return ok;
}

// Unit vector orthogonal to the `len` (1..8) columns of the 9 x len row-major matrix in ws->A[0 .. 9*len)
// (destroyed); result in ws->cs[0..8].  Same Householder arithmetic as left_null_9xk (la.h), with the
// reflector applied to the trailing columns one lane per column.
DG_ENGN void warp_left_null_9xk(WarpScratch* ws, int len, int lane, int W) {
  double* Z = ws->A;
  double* vs = ws->aux;        // len x 9 reflectors
  double* beta = ws->aux + 80;
  #pragma unroll 1
  for (int c = 0; c < len; ++c) {
    if (lane == 0) {
      double nrm = 0.0;
      #pragma unroll 1
      for (int r = c; r < 9; ++r) nrm += Z[r * len + c] * Z[r * len + c];
      nrm = sqrt(nrm);
      for (int r = 0; r < 9; ++r) vs[c * 9 + r] = 0.0;
      if (nrm == 0.0) {
        beta[c] = 0.0;
      } else {
        const double x0 = Z[c * len + c];
        const double alpha = (x0 >= 0.0) ? -nrm : nrm;
        #pragma unroll 1
        for (int r = c; r < 9; ++r) vs[c * 9 + r] = Z[r * len + c];
        vs[c * 9 + c] = x0 - alpha;
        double vn = 0.0;
        #pragma unroll 1
        for (int r = c; r < 9; ++r) vn += vs[c * 9 + r] * vs[c * 9 + r];
        beta[c] = (vn > 0.0) ? 2.0 / vn : 0.0;
      }
    }
    DG_WSYNC();
    if (beta[c] != 0.0) {
      #pragma unroll 1
      for (int cc = c + lane; cc < len; cc += W) {
        double dot = 0.0;
        #pragma unroll 1
        for (int r = c; r < 9; ++r) dot += vs[c * 9 + r] * Z[r * len + cc];
        dot *= beta[c];
        #pragma unroll 1
        for (int r = c; r < 9; ++r) Z[r * len + cc] -= dot * vs[c * 9 + r];
      }
    }
    DG_WSYNC();
  }
  if (lane == 0) {
    double q[9];
    for (int r = 0; r < 9; ++r) q[r] = 0.0;
    q[8] = 1.0;
    #pragma unroll 1
    for (int c = len - 1; c >= 0; --c) {
      double dot = 0.0;
      #pragma unroll 1
      for (int r = c; r < 9; ++r) dot += vs[c * 9 + r] * q[r];
      dot *= beta[c];
      #pragma unroll 1
      for (int r = c; r < 9; ++r) q[r] -= dot * vs[c * 9 + r];
    }
    for (int r = 0; r < 9; ++r) ws->cs[r] = q[r];
  }
  DG_WSYNC();
}

}  // namespace dg
