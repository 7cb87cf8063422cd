// Host build of csrc/p3p.h, csrc/absolute_pose.h and the minimal sample of csrc/rng.h, the per-thread pieces of
// absolute_pose_ragged_kernel -- TEST HELPER ONLY (tests/test_absolute_pose.py compiles it with g++ -ffp-contract=off
// into a temporary directory and compares it with tests/absolute_pose_np.py).
#include "../pydegensac_b200/csrc/absolute_pose.h"
#include "../pydegensac_b200/csrc/p3p.h"
#include "../pydegensac_b200/csrc/rng.h"

extern "C" {

// Lambda Twist on bearings y [9] and world points X [9]: the number of poses, R [4][9], t [4][3]
int aph_p3p(const double* y, const double* X, double* R, double* t) { return dg::p3p_lambda_twist(y, X, R, t); }

void aph_sample(unsigned long long seed, unsigned k, int n, int* sel) { dg::minimal_sample<3>(seed, k, n, sel); }

void aph_inv3(const double* K, double* Ki) { dg::ap_inv3(K, Ki); }

void aph_bearing(const double* Ki, double x, double y, double* b) { dg::ap_bearing(Ki, x, y, b); }

// Per row of x [n][2], X [n][3] under pose P [12]: the MSAC term and the inlier flag
void aph_msac(const double* P, const double* K, const double* x, const double* X, int n, double th2, double* term,
              int* inlier) {
  for (int i = 0; i < n; ++i) {
    bool in;
    term[i] = dg::ap_msac(P, K, x[2 * i], x[2 * i + 1], X[3 * i], X[3 * i + 1], X[3 * i + 2], th2, &in);
    inlier[i] = in ? 1 : 0;
  }
}

// Per row: r [n][2] and J [n][2][6]
void aph_jacobian(const double* P, const double* K, const double* x, const double* X, int n, double* r, double* J) {
  for (int i = 0; i < n; ++i)
    dg::ap_jacobian(P, K, x[2 * i], x[2 * i + 1], X[3 * i], X[3 * i + 1], X[3 * i + 2], r + 2 * i, J + 12 * i);
}

// The LM sums [28] over the rows, in row order
void aph_sums(const double* P, const double* K, const double* x, const double* X, int n, double* sums) {
  for (int j = 0; j < dg::kApSums; ++j) sums[j] = 0.0;
  for (int i = 0; i < n; ++i) dg::ap_row(P, K, x[2 * i], x[2 * i + 1], X[3 * i], X[3 * i + 1], X[3 * i + 2], sums);
}

int aph_solve(const double* H, const double* g, double lam, double* D) {
  return dg::pr_cholesky_solve<dg::kApParams>(H, g, lam, D) ? 1 : 0;
}

void aph_step(const double* P, const double* D, double* P2) { dg::ap_step(P, D, P2); }

int aph_required_iters(int has_best, int inl, int n, double conf, int max_iters, int k) {
  return dg::ap_required_iters(has_best != 0, inl, n, conf, max_iters, k);
}

}  // extern "C"
