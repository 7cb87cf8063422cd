// global_positioning.h -- per-thread pieces of the global positioning (global_positioning.cu): the world ray of an
// observation, the random start, the residual, the Huber loss and its IRLS weight, one observation's linearisation with
// its scale eliminated, the products with the eliminated 3 x 3 blocks, the scale's back-substitution and projection, and
// the angle of an observation at the output.  Host-compilable: tests/global_positioning_host.cpp builds it with g++ and
// tests/global_positioning_np.py restates every function here in numpy.
//
//   observation o of camera i and track j: ray v = normalise(R_i^T K_i^-1 (x, y, 1)), a = X_j - c_i,
//   residual r = d_o a - v (BATA's pairwise direction error), cost rho(|r|^2), rho Huber of scale delta.
//
// With B = [-I, I] over (c_i, X_j) the observation's Jacobian is [d B, a] over (c_i, X_j, d_o).  Under the Marquardt
// damping lambda diag(w J^T J), eliminating d_o (H_dd* = (1 + lambda) w |a|^2) leaves m B^T P B in the (c, X) block
// with s = w d^2, u = a / |a|, P = I - u u^T / (1 + lambda), and w d B^T (r - u (u . r) / (1 + lambda)) as its gradient.
#pragma once
#include "common.h"
#include "bundle_adjust.h"
#include "rng.h"
#include "triangulate.h"

namespace dg {

constexpr double kGpMinScale = 1e-5;     // d_min: the smallest scale of an observation
constexpr uint32_t kGpKindView = 0, kGpKindTrack = 1;   // the Philox counter word that keeps views and tracks apart

// The world ray of an observation at (x, y) of camera `cam` (a row of triangulate.h's table): normalise(R^T K^-1 (x,
// y, 1))
DG_HD void gp_ray(const double* cam, double x, double y, double* v) {
  const double* Ki = cam + kTrCamKi;
  const double* R = cam + kTrCamP;
  double b[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) b[i] = Ki[3 * i] * x + Ki[3 * i + 1] * y + Ki[3 * i + 2];
#pragma unroll
  for (int k = 0; k < 3; ++k) v[k] = R[k] * b[0] + R[3 + k] * b[1] + R[6 + k] * b[2];
  const double inv = 1.0 / sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  v[0] *= inv; v[1] *= inv; v[2] *= inv;
}

// The random start of item `index` of `kind` (a view's centre or a track's point): coordinate k is init_scale (2 u_k -
// 1), u_k = (o[k] + 1/2) 2^-32, o = philox4x32_10(ctr = (0, index, kind, 0), key = (seed_lo, seed_hi))
DG_HD void gp_start(uint64_t seed, uint32_t kind, uint32_t index, double init_scale, double* out) {
  uint32_t o[4];
  philox4x32_10(0u, index, kind, 0u, (uint32_t)seed, (uint32_t)(seed >> 32), o);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double u = ((double)o[k] + 0.5) * 2.3283064365386963e-10;
    out[k] = init_scale * (2.0 * u - 1.0);
  }
}

// a = X - c and r = d a - v; returns |r|^2
DG_HD double gp_residual(const double* c, const double* X, double d, const double* v, double* a, double* r) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    a[k] = X[k] - c[k];
    r[k] = d * a[k] - v[k];
  }
  return r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
}

// The Huber loss of scale delta (0: the trivial loss) on s = |r|^2: s for s <= delta^2, else 2 delta sqrt(s) - delta^2
DG_HD double gp_rho(double s, double delta) {
  if (delta > 0.0 && s > delta * delta) return 2.0 * delta * sqrt(s) - delta * delta;
  return s;
}

// Its IRLS weight rho'(s) = min(1, delta / |r|) (1 for the trivial loss)
DG_HD double gp_weight(double s, double delta) {
  if (delta > 0.0 && s > delta * delta) return delta / sqrt(s);
  return 1.0;
}

// One observation's linearisation at (a, r, d, w): u = a / |a|, n = |a|, s = w d^2, h = w d r, ar = a . r.  False when
// |a| is 0 or not finite (the linearisation is not defined there).
DG_HD bool gp_obs_terms(const double* a, const double* r, double d, double w, double* u, double* n, double* s,
                        double* h, double* ar) {
  const double na = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
  if (!(na > 0.0) || !(na < INFINITY)) return false;
  const double inv = 1.0 / na;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    u[k] = a[k] * inv;
    h[k] = w * d * r[k];
  }
  *n = na;
  *s = w * d * d;
  *ar = a[0] * r[0] + a[1] * r[1] + a[2] * r[2];
  return true;
}

// out = s (p - f u (u . p)), f = 1 / (1 + lambda): the eliminated block m = s P times p
DG_HD void gp_m_apply(const double* u, double s, double f, const double* p, double* out) {
  const double up = f * (u[0] * p[0] + u[1] * p[1] + u[2] * p[2]);
#pragma unroll
  for (int k = 0; k < 3; ++k) out[k] = s * (p[k] - up * u[k]);
}

// The damped 3 x 3 block of a centre or a point (upper triangle by rows) from its sums S = sum s and Q = sum s u u^T
// (upper, 6): (1 + lambda) S I - Q / (1 + lambda), i.e. sum m + lambda diag(sum w d^2 B^T B)
DG_HD void gp_block(double S, const double* Q, double lam, double* out) {
  const double f = 1.0 / (1.0 + lam), g = (1.0 + lam) * S;
#pragma unroll
  for (int m = 0; m < 6; ++m) out[m] = (m == 0 || m == 3 || m == 5 ? g : 0.0) - f * Q[m];
}

// Q += s u u^T (upper triangle by rows)
DG_HD void gp_add_outer(const double* u, double s, double* Q) {
  int m = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int l = k; l < 3; ++l) Q[m++] += s * u[k] * u[l];
}

// A += m = s (I - f u u^T) (upper triangle by rows)
DG_HD void gp_m_add(const double* u, double s, double f, double* A) {
  int m = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int l = k; l < 3; ++l, ++m) A[m] += s * ((k == l ? 1.0 : 0.0) - f * u[k] * u[l]);
}

// out += A Vi A for symmetric A and Vi (upper triangles by rows), column by column: A (Vi (A e_l))
DG_HD void gp_sandwich(const double* A, const double* Vi, double* out) {
  const double F[9] = {A[0], A[1], A[2], A[1], A[3], A[4], A[2], A[4], A[5]};
  double col[3][3];
#pragma unroll
  for (int l = 0; l < 3; ++l) {
    const double a[3] = {F[l], F[3 + l], F[6 + l]};
    double w[3];
    ba_sym3_mul(Vi, a, w);
    ba_sym3_mul(A, w, col[l]);
  }
  int m = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int l = k; l < 3; ++l) out[m++] += col[l][k];
}

// The scale's back-substitution: dd = -(a . r + d |a| u . (dX - dc)) / ((1 + lambda) |a|^2), w cancelled, then the
// projected trial scale max(d + dd, d_min)
DG_HD double gp_scale_step(double ar, double n, double d, const double* u, const double* dXc, double lam) {
  const double ud = u[0] * dXc[0] + u[1] * dXc[1] + u[2] * dXc[2];
  const double dd = -(ar + d * n * ud) / ((1.0 + lam) * (n * n));
  const double t = d + dd;
  return t > kGpMinScale ? t : kGpMinScale;
}

// The angle between the ray v and a = X - c, atan2(|v x a|, v . a), in [0, pi]
DG_HD double gp_angle(const double* v, const double* a) {
  const double x0 = v[1] * a[2] - v[2] * a[1], x1 = v[2] * a[0] - v[0] * a[2], x2 = v[0] * a[1] - v[1] * a[0];
  return atan2(sqrt(x0 * x0 + x1 * x1 + x2 * x2), v[0] * a[0] + v[1] * a[1] + v[2] * a[2]);
}

}  // namespace dg
