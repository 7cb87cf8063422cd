// Host build of csrc/refine_f.h, the per-thread pieces of f_refine_ragged_kernel -- TEST HELPER ONLY
// (tests/test_refine_fundamental.py compiles it with g++ into a temporary directory and compares it with
// tests/refine_fundamental_np.py).
#include "../pydegensac_b200/csrc/refine_f.h"

extern "C" {

// From a public F and n rows, as the kernel's first passes form them (one thread): T [6] = (T1, T2), the start point
// Fn [9], the linearisation F [9], dF [63] and the sums [36] (cost, J^T J upper triangle by rows, J^T r).  Returns 0
// when F is no model.
int rfh_pass(const double* F_in, const double* p1, const double* p2, int n, double* T, double* Fn, double* F,
             double* dF, double* sums) {
  if (!dg::rf_has_model(F_in)) return 0;
  double ns[dg::kRhNormSums] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < n; ++i) {
    const double x1 = p1[2 * i], y1 = p1[2 * i + 1], x2 = p2[2 * i], y2 = p2[2 * i + 1];
    ns[0] += x1; ns[1] += y1; ns[2] += x1 * x1; ns[3] += y1 * y1;
    ns[4] += x2; ns[5] += y2; ns[6] += x2 * x2; ns[7] += y2 * y2;
  }
  dg::rh_transform(ns, n, T);
  dg::rh_transform(ns + 4, n, T + 3);
  dg::rf_start(T, T + 3, F_in, Fn);
  dg::rf_linearise(T, T + 3, Fn, F, dF);
  for (int j = 0; j < dg::kRfSums; ++j) sums[j] = 0.0;
  for (int i = 0; i < n; ++i) dg::pr_row_n<7, true>(F, dF, p1[2 * i], p1[2 * i + 1], p2[2 * i], p2[2 * i + 1], sums);
  return 1;
}

// B [7][9]: the basis columns at Fn
void rfh_basis(const double* Fn, double* B) {
  double a[8];
  dg::rf_cofactor_coords(Fn, a);
  for (int k = 0; k < 7; ++k) {
    double d[7] = {0, 0, 0, 0, 0, 0, 0};
    d[k] = 1.0;
    dg::rf_tangent(Fn, a, d, B + 9 * k);
  }
}

void rfh_rank2(double* F) { dg::enforce_rank2_inl(*reinterpret_cast<double(*)[9]>(F)); }

int rfh_solve(const double* H, const double* g, double lam, double* D) {
  return dg::pr_cholesky_solve<7>(H, g, lam, D) ? 1 : 0;
}

void rfh_retract(const double* Fn, const double* D, double* Fn2) { dg::rf_retract(Fn, D, Fn2); }

// the public F of the normalised model Fn under T [6], signed against F_in
void rfh_output(const double* T, const double* Fn, const double* F_in, double* F) {
  dg::rf_output(T, T + 3, Fn, F_in, F);
}

void rfh_constants(double* c) {
  c[0] = dg::kPrLambda0; c[1] = dg::kPrLambdaMin; c[2] = dg::kPrLambdaMax; c[3] = dg::kPrRelDecrease;
  c[4] = dg::kRfMinRows; c[5] = dg::kRfSums;
}

}  // extern "C"
