// Host build of csrc/five_point.h, csrc/essential.h and the minimal sample of csrc/rng.h, the per-thread pieces of
// essential_ragged_kernel -- TEST HELPER ONLY (tests/test_essential.py compiles it with g++ -ffp-contract=off into a
// temporary directory and compares it with tests/essential_np.py).
#include "../pydegensac_b200/csrc/essential.h"
#include "../pydegensac_b200/csrc/rng.h"

extern "C" {

// The five-point solver on x1 [5][3], x2 [5][3]: the number of solutions, Es [10][9]
int esh_five_point(const double* x1, const double* x2, double* Es) { return dg::five_point(x1, x2, Es); }

void esh_sample(unsigned long long seed, unsigned k, int n, int* sel) { dg::minimal_sample<5>(seed, k, n, sel); }

void esh_normalise(const double* Ki, double x, double y, double* out) { dg::es_normalise(Ki, x, y, out); }

void esh_fundamental(const double* E, const double* A, const double* Bk, double* F) { dg::es_fundamental(E, A, Bk, F); }

// Per row of p1 [n][2], p2 [n][2] under F [9]: the MSAC term and the inlier flag
void esh_msac(const double* F, const double* p1, const double* p2, int n, double th2, double* term, int* inlier) {
  for (int i = 0; i < n; ++i) {
    bool in;
    term[i] = dg::es_msac(F, p1[2 * i], p1[2 * i + 1], p2[2 * i], p2[2 * i + 1], th2, &in);
    inlier[i] = in ? 1 : 0;
  }
}

int esh_pose(const double* E, double* R, double* t) { return dg::es_pose(E, R, t) ? 1 : 0; }

void esh_essential(const double* R, const double* t, double* E) { dg::es_essential(R, t, E); }

int esh_required_iters(int has_best, int inl, int n, double conf, int max_iters, int k) {
  return dg::es_required_iters(has_best != 0, inl, n, conf, max_iters, k);
}

}  // extern "C"
