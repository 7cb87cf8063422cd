// Host build of csrc/refine_h.h, the per-thread pieces of h_refine_ragged_kernel -- TEST HELPER ONLY
// (tests/test_refine_homography.py compiles it with g++ into a temporary directory and compares it with
// tests/refine_homography_np.py).
#include "../pydegensac_b200/csrc/refine_h.h"

extern "C" {

// From a public H and n rows, as the kernel's first passes form them (one thread): the engine model g [9] (returns 0 when
// there is none), T [6] = (T1, T2), the normalised model M [9], the linearisation G [9], dG [72] and the sums [45]
// (cost, J^T J upper triangle by rows, J^T z).
int rhh_pass(const double* H, const double* p1, const double* p2, int n, double* g, double* T, double* M, double* G,
             double* dG, double* sums) {
  if (!dg::rh_engine_model(H, g)) return 0;
  double ns[dg::kRhNormSums] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < n; ++i) {
    const double x1 = p1[2 * i], y1 = p1[2 * i + 1], x2 = p2[2 * i], y2 = p2[2 * i + 1];
    ns[0] += x1; ns[1] += y1; ns[2] += x1 * x1; ns[3] += y1 * y1;
    ns[4] += x2; ns[5] += y2; ns[6] += x2 * x2; ns[7] += y2 * y2;
  }
  dg::rh_transform(ns, n, T);
  dg::rh_transform(ns + 4, n, T + 3);
  dg::rh_from_pixels(T, T + 3, g, M);
  dg::rh_linearise(T, T + 3, M, G, dG);
  for (int j = 0; j < dg::kRhSums; ++j) sums[j] = 0.0;
  for (int i = 0; i < n; ++i) dg::rh_row(G, dG, p1[2 * i], p1[2 * i + 1], p2[2 * i], p2[2 * i + 1], sums);
  return 1;
}

int rhh_solve(const double* H, const double* g, double lam, double* D) {
  return dg::pr_cholesky_solve<8>(H, g, lam, D) ? 1 : 0;
}

void rhh_step(const double* M, const double* D, double* M2) { dg::rh_step(M, D, M2); }

// the public H of the normalised model M under T [6]
void rhh_public(const double* T, const double* M, double* H) {
  double G[9];
  dg::rh_to_pixels(T, T + 3, M, G);
  dg::rh_public_model(G, H);
}

void rhh_constants(double* c) {
  c[0] = dg::kPrLambda0; c[1] = dg::kPrLambdaMin; c[2] = dg::kPrLambdaMax; c[3] = dg::kPrRelDecrease;
  c[4] = dg::kRhMinRows; c[5] = dg::kRhSums;
}

}  // extern "C"
