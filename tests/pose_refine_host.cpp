// Host build of csrc/pose_refine.h, the per-thread pieces of pose_refine_ragged_kernel -- TEST HELPER ONLY
// (tests/test_pose_refine.py compiles it with g++ into a temporary directory and compares it with tests/pose_refine_np.py).
#include "../pydegensac_b200/csrc/pose_refine.h"

extern "C" {

// sums [21] (cost, J^T J upper triangle by rows, J^T r) over n rows at (R, t), as one thread would accumulate them;
// F [9] and dF [45] of the linearisation.  A = K2^-T, Bk = K1^-1.
void prh_pass(const double* R, const double* t, const double* A, const double* Bk, const double* p1, const double* p2, int n,
              double* F, double* dF, double* sums) {
  dg::pr_linearise(R, t, A, Bk, F, dF);
  for (int j = 0; j < dg::kPrSums; ++j) sums[j] = 0.0;
  for (int i = 0; i < n; ++i) dg::pr_row(F, dF, p1[2 * i], p1[2 * i + 1], p2[2 * i], p2[2 * i + 1], sums);
}

int prh_solve(const double* H, const double* g, double lam, double* D) { return dg::pr_solve(H, g, lam, D) ? 1 : 0; }

void prh_step(const double* R, const double* t, const double* D, double* R2, double* t2) { dg::pr_step(R, t, D, R2, t2); }

double prh_orthonormalise(double* R) {
  const double drift = dg::pr_ortho_drift(R);
  dg::pr_orthonormalise(R);
  return drift;
}

void prh_constants(double* c) {
  c[0] = dg::kPrLambda0; c[1] = dg::kPrLambdaMin; c[2] = dg::kPrLambdaMax; c[3] = dg::kPrRelDecrease;
  c[4] = dg::kPrMinRows; c[5] = dg::kPrOrthoTol;
}

}  // extern "C"
