// Host build of csrc/bundle_adjust.h, the per-thread pieces of the bundle-adjustment kernels -- TEST HELPER ONLY
// (tests/test_bundle_adjust.py compiles it with g++ -ffp-contract=off into a temporary directory and compares it with
// tests/bundle_adjust_np.py).
#include "../pydegensac_b200/csrc/bundle_adjust.h"

extern "C" {

// Per observation of X [n][3] in pose P [n][12] and K [n][9] at pts [n][2]: r [n][2], J_cam [n][2][6], J_X [n][2][3]
void bah_jacobian(const double* P, const double* K, const double* X, const double* pts, int n, double* r, double* Jc,
                  double* Jx) {
  for (int i = 0; i < n; ++i)
    dg::ba_jacobian(P + 12 * i, K + 9 * i, X + 3 * i, pts[2 * i], pts[2 * i + 1], r + 2 * i, Jc + 12 * i, Jx + 6 * i);
}

void bah_loss(const double* s, int n, double sig2, double* rho, double* w) {
  for (int i = 0; i < n; ++i) {
    rho[i] = dg::ba_rho(s[i], sig2);
    w[i] = dg::ba_weight(s[i], sig2);
  }
}

// V [6] and g [3] summed over n observations (J_X [n][2][3], r [n][2], w [n]) in order
void bah_point_terms(const double* Jx, const double* r, const double* w, int n, double* V, double* g) {
  for (int k = 0; k < 6; ++k) V[k] = 0.0;
  for (int k = 0; k < 3; ++k) g[k] = 0.0;
  for (int i = 0; i < n; ++i) dg::ba_point_terms(Jx + 6 * i, r + 2 * i, w[i], V, g);
}

int bah_inv3(const double* V, double lam, double* Vi) { return dg::ba_inv3(V, lam, Vi) ? 1 : 0; }

void bah_schur_row(const double* W, const double* Vi, double* Y) { dg::ba_schur_row(W, Vi, Y); }

void bah_cross_block(const double* Jc, const double* Jx, double w, double* W) { dg::ba_cross_block(Jc, Jx, w, W); }

int bah_gauge_axis(const double* Pg, const double* Ca) { return dg::ba_gauge_axis(Pg, Ca); }

}  // extern "C"
