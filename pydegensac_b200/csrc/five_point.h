// five_point.h -- the five-point relative-pose solver: every essential matrix E with x2^T E x1 = 0 for five
// correspondences in normalised coordinates x = K^-1 [u, v, 1].  Nistér (PAMI 2004) in the formulation of Stewénius,
// Engels and Nistér (2006):
//   1. the 4-dimensional null space X, Y, Z, W of the 5 x 9 epipolar constraint matrix (Householder QR of its
//      transpose), so that E = x X + y Y + z Z + W;
//   2. the ten cubic constraints det E = 0 and 2 E E^T E - tr(E E^T) E = 0 over the 20 monomials of (x, y, z) in
//      Nistér's order x^3, y^3, x^2y, xy^2, x^2z, x^2, y^2z, y^2, xyz, xy | xz^2, xz, x, yz^2, yz, y, z^3, z^2, z, 1;
//   3. Gauss-Jordan elimination of the 10 x 20 system (partial pivoting) and the 3 x 3 polynomial matrix
//      B(z) [x, y, 1]^T = 0 of rows <e> - z <f>, <g> - z <h>, <i> - z <j>, whose determinant is of degree 10 in z;
//   4. its real roots: counted and isolated by a Sturm sequence, refined by a fixed number of bisections on the sign;
//   5. back-substitution: [x, y, 1] from the cross product of two rows of B(z), polished by a few Gauss-Newton steps
//      on the ten constraints (the elimination loses digits that the polynomial's roots alone do not recover), E at
//      unit Frobenius norm.
// Only +, -, *, / and sqrt, so the host build and tests/essential_np.py agree to the bit.  A degenerate sample (a
// rank-deficient constraint matrix, a zero pivot, a Sturm sequence that loses a degree) gives no solution.
#pragma once
#include "common.h"

namespace dg {

constexpr int kFpMaxSolutions = 10;
constexpr int kFpIsolateSteps = 128;   // Sturm halvings at most to isolate one root
constexpr int kFpRefineSteps = 100;    // sign halvings of each isolated root
constexpr int kFpPolishSteps = 3;      // Gauss-Newton steps on the ten constraints at most per solution

// Index of the product of linear monomials a, b in (x, y, z, 1) among x^2, xy, xz, x, y^2, yz, y, z^2, z, 1
DG_HD int fp_q(int a, int b) {
  const int t[16] = {0, 1, 2, 3, 1, 4, 5, 6, 2, 5, 7, 8, 3, 6, 8, 9};
  return t[4 * a + b];
}

// Index of the product of quadratic monomial q and linear monomial a among the 20 cubic monomials (Nistér's order)
DG_HD int fp_c(int q, int a) {
  const int t[40] = {0, 2, 4, 5,  2, 3, 8, 9,  4, 8, 10, 11,  5, 9, 11, 12,  3, 1, 6, 7,
                     8, 6, 13, 14,  9, 7, 14, 15,  10, 13, 16, 17,  11, 14, 17, 18,  12, 15, 18, 19};
  return t[4 * q + a];
}

// q [10] += s (a b), a and b linear [4]
DG_HD void fp_mul11(const double* a, const double* b, double s, double* q) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) q[fp_q(i, j)] += s * (a[i] * b[j]);
}

// c [20] += q l, q quadratic [10], l linear [4]
DG_HD void fp_mul21(const double* q, const double* l, double* c) {
#pragma unroll
  for (int i = 0; i < 10; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) c[fp_c(i, j)] += q[i] * l[j];
}

// Polynomial c [na + nb - 1] += a [na] b [nb] (coefficients in ascending powers)
template <int NA, int NB>
DG_HD void fp_pmul(const double* a, const double* b, double* c) {
#pragma unroll
  for (int i = 0; i < NA; ++i)
#pragma unroll
    for (int j = 0; j < NB; ++j) c[i + j] += a[i] * b[j];
}

// Horner evaluation of p [deg + 1] at z
DG_HD double fp_horner(const double* p, int deg, double z) {
  double v = p[deg];
  for (int i = deg - 1; i >= 0; --i) v = v * z + p[i];
  return v;
}

// Sign variations of the Sturm sequence s (11 polynomials of degrees 10 .. 0, packed) at z, zeros skipped
DG_HD int fp_variations(const double* s, double z) {
  int count = 0, last = 0;
  int off = 0;
  for (int k = 0; k <= 10; ++k) {
    const int deg = 10 - k;
    const double v = fp_horner(s + off, deg, z);
    off += deg + 1;
    const int sg = v > 0.0 ? 1 : (v < 0.0 ? -1 : 0);
    if (sg != 0) {
      if (last != 0 && sg != last) ++count;
      last = sg;
    }
  }
  return count;
}

// Null space of the 5 x 9 constraint matrix of x1 [5][3], x2 [5][3]: N [4][9], orthonormal; false when the matrix is
// rank deficient (a zero Householder column).
DG_HD bool fp_null_space(const double* x1, const double* x2, double* N) {
  double M[9][5], V[5][9], beta[5];
#pragma unroll
  for (int c = 0; c < 5; ++c)
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) M[3 * i + j][c] = x2[3 * c + i] * x1[3 * c + j];
  for (int c = 0; c < 5; ++c) {
    double s = 0.0;
    for (int r = c; r < 9; ++r) s += M[r][c] * M[r][c];
    if (!(s > 0.0)) return false;
    const double nrm = sqrt(s);
    const double alpha = M[c][c] < 0.0 ? nrm : -nrm;    // v = x - alpha e_c, without cancellation
    for (int r = 0; r < 9; ++r) V[c][r] = r < c ? 0.0 : M[r][c];
    V[c][c] = V[c][c] - alpha;
    double vv = 0.0;
    for (int r = c; r < 9; ++r) vv += V[c][r] * V[c][r];
    if (!(vv > 0.0)) return false;
    beta[c] = 2.0 / vv;
    for (int k = c + 1; k < 5; ++k) {
      double w = 0.0;
      for (int r = c; r < 9; ++r) w += V[c][r] * M[r][k];
      const double f = beta[c] * w;
      for (int r = c; r < 9; ++r) M[r][k] = M[r][k] - f * V[c][r];
    }
  }
  // N_j = H_0 H_1 ... H_4 e_{5 + j}: the last four columns of the orthogonal factor
  for (int j = 0; j < 4; ++j) {
    double y[9];
    for (int r = 0; r < 9; ++r) y[r] = r == 5 + j ? 1.0 : 0.0;
    for (int c = 4; c >= 0; --c) {
      double w = 0.0;
      for (int r = c; r < 9; ++r) w += V[c][r] * y[r];
      const double f = beta[c] * w;
      for (int r = c; r < 9; ++r) y[r] = y[r] - f * V[c][r];
    }
    for (int r = 0; r < 9; ++r) N[9 * j + r] = y[r];
  }
  return true;
}

// The ten cubic constraints of E = x X + y Y + z Z + W (N [4][9] = X, Y, Z, W): C [10][20], row 0 det E, rows 1 .. 9
// the entries (i, j) of 2 E E^T E - tr(E E^T) E in row-major order
DG_HD void fp_constraints(const double* N, double (*C)[20]) {
  double E[9][4];
#pragma unroll
  for (int e = 0; e < 9; ++e)
#pragma unroll
    for (int a = 0; a < 4; ++a) E[e][a] = N[9 * a + e];
  for (int r = 0; r < 10; ++r)
    for (int m = 0; m < 20; ++m) C[r][m] = 0.0;
  // det E = e0 . (e1 x e2) by the cofactors of row 0
  {
    double cof[3][10];
    for (int j = 0; j < 3; ++j) {
      for (int m = 0; m < 10; ++m) cof[j][m] = 0.0;
      const int j1 = (j + 1) % 3, j2 = (j + 2) % 3;
      fp_mul11(E[3 + j1], E[6 + j2], 1.0, cof[j]);
      fp_mul11(E[3 + j2], E[6 + j1], -1.0, cof[j]);
    }
    for (int j = 0; j < 3; ++j) fp_mul21(cof[j], E[j], C[0]);
  }
  double Q[3][3][10], tr[10], T[10];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      for (int m = 0; m < 10; ++m) Q[i][j][m] = 0.0;
      for (int k = 0; k < 3; ++k) fp_mul11(E[3 * i + k], E[3 * j + k], 1.0, Q[i][j]);
    }
  for (int m = 0; m < 10; ++m) tr[m] = (Q[0][0][m] + Q[1][1][m]) + Q[2][2][m];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      for (int k = 0; k < 3; ++k) {
        for (int m = 0; m < 10; ++m) T[m] = i == k ? 2.0 * Q[i][k][m] - tr[m] : 2.0 * Q[i][k][m];
        fp_mul21(T, E[3 * k + j], C[1 + 3 * i + j]);
      }
}

// Gauss-Jordan elimination of C [10][20] on its first 10 columns (partial pivoting, the first largest |pivot|);
// false at a zero (or NaN) pivot
DG_HD bool fp_eliminate(double (*C)[20]) {
  for (int c = 0; c < 10; ++c) {
    int p = c;
    double best = fabs(C[c][c]);
    for (int r = c + 1; r < 10; ++r)
      if (fabs(C[r][c]) > best) { best = fabs(C[r][c]); p = r; }
    if (!(best > 0.0)) return false;
    if (p != c)
      for (int k = c; k < 20; ++k) { const double t = C[c][k]; C[c][k] = C[p][k]; C[p][k] = t; }
    const double piv = C[c][c];
    for (int k = c; k < 20; ++k) C[c][k] = C[c][k] / piv;
    for (int r = 0; r < 10; ++r) {
      if (r == c) continue;
      const double f = C[r][c];
      for (int k = c; k < 20; ++k) C[r][k] = C[r][k] - f * C[c][k];
    }
  }
  return true;
}

// The rows <a> - z <b> of B(z): x-, y- (degree 3) and 1-polynomial (degree 4) from the eliminated rows a, b, whose
// last 10 columns multiply xz^2, xz, x, yz^2, yz, y, z^3, z^2, z, 1
DG_HD void fp_brow(const double* ra, const double* rb, double* px, double* py, double* p1) {
  px[0] = ra[12]; px[1] = ra[11] - rb[12]; px[2] = ra[10] - rb[11]; px[3] = -rb[10];
  py[0] = ra[15]; py[1] = ra[14] - rb[15]; py[2] = ra[13] - rb[14]; py[3] = -rb[13];
  p1[0] = ra[19]; p1[1] = ra[18] - rb[19]; p1[2] = ra[17] - rb[18]; p1[3] = ra[16] - rb[17]; p1[4] = -rb[16];
}

// The Sturm sequence of the monic a [11] (packed: degrees 10, 9, ..., 0); false when a remainder loses a degree
DG_HD bool fp_sturm(const double* a, double* s) {
  for (int i = 0; i < 11; ++i) s[i] = a[i];
  for (int i = 0; i < 10; ++i) s[11 + i] = (double)(i + 1) * a[i + 1];
  int offA = 0, offB = 11;
  for (int d = 9; d >= 1; --d) {                 // A of degree d + 1, B of degree d -> -rem(A, B) of degree d - 1
    const double* A = s + offA;
    const double* B = s + offB;
    double* R = s + offB + d + 1;
    if (!(B[d] != 0.0)) return false;
    const double q1 = A[d + 1] / B[d];
    const double q0 = (A[d] - q1 * B[d - 1]) / B[d];
    for (int i = 0; i < d; ++i) {
      double r = A[i] - q0 * B[i];
      if (i > 0) r = r - q1 * B[i - 1];
      R[i] = -r;
    }
    offA = offB;
    offB = offB + d + 1;
  }
  return s[65] != 0.0;
}

// The ten constraints C [10][20] (before elimination) at (x, y, z): r [10], J [10][3] = dr / d(x, y, z); returns |r|^2
DG_HD double fp_residual(const double (*C)[20], double x, double y, double z, double* r, double (*J)[3]) {
  const double xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
  const double m[20] = {xx * x, yy * y, xx * y, x * yy, xx * z, xx, yy * z, yy, xy * z, xy,
                        x * zz, xz, x, y * zz, yz, y, zz * z, zz, z, 1.0};
  const double mx[20] = {3.0 * xx, 0.0, 2.0 * xy, yy, 2.0 * xz, 2.0 * x, 0.0, 0.0, yz, y,
                         zz, z, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  const double my[20] = {0.0, 3.0 * yy, xx, 2.0 * xy, 0.0, 0.0, 2.0 * yz, 2.0 * y, xz, x,
                         0.0, 0.0, 0.0, zz, z, 1.0, 0.0, 0.0, 0.0, 0.0};
  const double mz[20] = {0.0, 0.0, 0.0, 0.0, xx, 0.0, yy, 0.0, xy, 0.0,
                         2.0 * xz, x, 0.0, 2.0 * yz, y, 0.0, 3.0 * zz, 2.0 * z, 1.0, 0.0};
  double rr = 0.0;
  for (int i = 0; i < 10; ++i) {
    double v = 0.0, a = 0.0, b = 0.0, c = 0.0;
    for (int k = 0; k < 20; ++k) {
      v += C[i][k] * m[k];
      a += C[i][k] * mx[k];
      b += C[i][k] * my[k];
      c += C[i][k] * mz[k];
    }
    r[i] = v; J[i][0] = a; J[i][1] = b; J[i][2] = c;
    rr += v * v;
  }
  return rr;
}

// Gauss-Newton on the ten constraints from (x, y, z): a step is taken while it lowers |r|^2
DG_HD void fp_polish(const double (*C)[20], double* x, double* y, double* z) {
  double r[10], J[10][3];
  double rr = fp_residual(C, *x, *y, *z, r, J);
  for (int it = 0; it < kFpPolishSteps; ++it) {
    double H[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, g[3] = {0.0, 0.0, 0.0};
    for (int i = 0; i < 10; ++i) {
      H[0] += J[i][0] * J[i][0]; H[1] += J[i][0] * J[i][1]; H[2] += J[i][0] * J[i][2];
      H[3] += J[i][1] * J[i][1]; H[4] += J[i][1] * J[i][2]; H[5] += J[i][2] * J[i][2];
      g[0] += J[i][0] * r[i]; g[1] += J[i][1] * r[i]; g[2] += J[i][2] * r[i];
    }
    // (J^T J) D = -g by Cholesky
    if (!(H[0] > 0.0)) return;
    const double l00 = sqrt(H[0]), l10 = H[1] / l00, l20 = H[2] / l00;
    const double d1 = H[3] - l10 * l10;
    if (!(d1 > 0.0)) return;
    const double l11 = sqrt(d1), l21 = (H[4] - l20 * l10) / l11;
    const double d2 = (H[5] - l20 * l20) - l21 * l21;
    if (!(d2 > 0.0)) return;
    const double l22 = sqrt(d2);
    const double y0 = -g[0] / l00, y1 = (-g[1] - l10 * y0) / l11, y2 = ((-g[2] - l20 * y0) - l21 * y1) / l22;
    const double D2 = y2 / l22, D1 = (y1 - l21 * D2) / l11, D0 = ((y0 - l10 * D1) - l20 * D2) / l00;
    const double xn = *x + D0, yn = *y + D1, zn = *z + D2;
    const double rn = fp_residual(C, xn, yn, zn, r, J);
    if (!(rn < rr)) return;
    *x = xn; *y = yn; *z = zn;
    rr = rn;
  }
}

// Every essential matrix of five correspondences x1 [5][3], x2 [5][3] (x2^T E x1 = 0): Es [10][9], each at unit
// Frobenius norm; returns their number (0 for a degenerate sample)
DG_HDN int five_point(const double* x1, const double* x2, double* Es) {
  double N[36];
  if (!fp_null_space(x1, x2, N)) return 0;
  double C0[10][20], C[10][20];
  fp_constraints(N, C0);
  for (int r = 0; r < 10; ++r)
    for (int m = 0; m < 20; ++m) C[r][m] = C0[r][m];
  if (!fp_eliminate(C)) return 0;
  // B(z) from rows e, f (4, 5), g, h (6, 7), i, j (8, 9); its determinant
  double Bp[3][3][5];
  for (int r = 0; r < 3; ++r) fp_brow(C[4 + 2 * r], C[5 + 2 * r], Bp[r][0], Bp[r][1], Bp[r][2]);
  double p[11];
  {
    double u[8], v[8], w[7], t[11];
    for (int m = 0; m < 11; ++m) p[m] = 0.0;
    // + kx (ly m1 - l1 my) - ky (lx m1 - l1 mx) + k1 (lx my - ly mx)
    for (int m = 0; m < 8; ++m) { u[m] = 0.0; v[m] = 0.0; }
    fp_pmul<4, 5>(Bp[1][1], Bp[2][2], u);
    fp_pmul<5, 4>(Bp[1][2], Bp[2][1], v);
    for (int m = 0; m < 8; ++m) u[m] = u[m] - v[m];
    for (int m = 0; m < 11; ++m) t[m] = 0.0;
    fp_pmul<4, 8>(Bp[0][0], u, t);
    for (int m = 0; m < 11; ++m) p[m] = p[m] + t[m];
    for (int m = 0; m < 8; ++m) { u[m] = 0.0; v[m] = 0.0; }
    fp_pmul<4, 5>(Bp[1][0], Bp[2][2], u);
    fp_pmul<5, 4>(Bp[1][2], Bp[2][0], v);
    for (int m = 0; m < 8; ++m) u[m] = u[m] - v[m];
    for (int m = 0; m < 11; ++m) t[m] = 0.0;
    fp_pmul<4, 8>(Bp[0][1], u, t);
    for (int m = 0; m < 11; ++m) p[m] = p[m] - t[m];
    for (int m = 0; m < 7; ++m) { w[m] = 0.0; v[m] = 0.0; }
    fp_pmul<4, 4>(Bp[1][0], Bp[2][1], w);
    fp_pmul<4, 4>(Bp[1][1], Bp[2][0], v);
    for (int m = 0; m < 7; ++m) w[m] = w[m] - v[m];
    for (int m = 0; m < 11; ++m) t[m] = 0.0;
    fp_pmul<5, 7>(Bp[0][2], w, t);
    for (int m = 0; m < 11; ++m) p[m] = p[m] + t[m];
  }
  // monic, the Cauchy bound, the Sturm sequence
  if (!(fabs(p[10]) > 0.0) || !(fabs(p[10]) < INFINITY)) return 0;
  double a[11], bound = 0.0;
  for (int m = 0; m < 10; ++m) {
    a[m] = p[m] / p[10];
    if (!(fabs(a[m]) < INFINITY)) return 0;
    bound = fabs(a[m]) > bound ? fabs(a[m]) : bound;
  }
  a[10] = 1.0;
  bound = 1.0 + bound;
  double s[66];
  if (!fp_sturm(a, s)) return 0;
  const int v_lo = fp_variations(s, -bound);
  const int n_roots = v_lo - fp_variations(s, bound);
  int ns = 0;
  for (int j = 0; j < n_roots && j < kFpMaxSolutions; ++j) {
    // isolate root j (0-based, ascending): N(lo) <= j < N(hi), N(z) = roots in (-bound, z]
    double lo = -bound, hi = bound;
    int nlo = 0, nhi = n_roots;
    for (int step = 0; step < kFpIsolateSteps && !(nlo == j && nhi == j + 1); ++step) {
      const double mid = 0.5 * (lo + hi);
      const int c = v_lo - fp_variations(s, mid);
      if (c > j) { hi = mid; nhi = c; } else { lo = mid; nlo = c; }
    }
    double flo = fp_horner(a, 10, lo);
    const double fhi = fp_horner(a, 10, hi);
    if (!((flo <= 0.0 && fhi >= 0.0) || (flo >= 0.0 && fhi <= 0.0))) continue;   // no sign change: no root kept
    for (int step = 0; step < kFpRefineSteps; ++step) {
      const double mid = 0.5 * (lo + hi);
      const double fm = fp_horner(a, 10, mid);
      if ((fm < 0.0) == (flo < 0.0)) { lo = mid; flo = fm; } else { hi = mid; }
    }
    double z = 0.5 * (lo + hi);
    // [x, y, 1] ~ the null vector of B(z): the cross product of two of its rows, the largest of the three
    double b[3][3];
    for (int r = 0; r < 3; ++r) {
      b[r][0] = fp_horner(Bp[r][0], 3, z);
      b[r][1] = fp_horner(Bp[r][1], 3, z);
      b[r][2] = fp_horner(Bp[r][2], 4, z);
    }
    double best[3] = {0.0, 0.0, 0.0}, best_n = -1.0;
    for (int r = 0; r < 3; ++r) {
      const double* u = b[r == 2 ? 1 : 0];
      const double* w = b[r == 0 ? 1 : 2];
      const double c[3] = {u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0]};
      const double nn = (c[0] * c[0] + c[1] * c[1]) + c[2] * c[2];
      if (nn > best_n) { best_n = nn; best[0] = c[0]; best[1] = c[1]; best[2] = c[2]; }
    }
    if (!(best[2] != 0.0)) continue;
    double x = best[0] / best[2], y = best[1] / best[2];
    fp_polish(C0, &x, &y, &z);
    double* E = Es + 9 * ns;
    double nrm = 0.0;
    for (int e = 0; e < 9; ++e) {
      E[e] = ((x * N[e] + y * N[9 + e]) + z * N[18 + e]) + N[27 + e];
      nrm += E[e] * E[e];
    }
    if (!(nrm > 0.0) || !(nrm < INFINITY)) continue;
    const double inv = 1.0 / sqrt(nrm);
    for (int e = 0; e < 9; ++e) E[e] = E[e] * inv;
    ++ns;
  }
  return ns;
}

}  // namespace dg
