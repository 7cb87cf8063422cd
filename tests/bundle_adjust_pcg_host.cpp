// g++ host build of the per-thread functions that bundle_adjust_pcg.cu adds: the Cholesky factor / apply pair of
// csrc/pose_refine.h at N = 6, the preconditioner block's.  tests/test_bundle_adjust_pcg.py checks it against numpy.
#include <math.h>

#include "../pydegensac_b200/csrc/pose_refine.h"

extern "C" {

// A (upper triangle by rows, 21) -> L (lower by rows, 21) and x = A^-1 b; 0 at a non-positive pivot
int pcgh_solve(const double* A, double* L, const double* b, double* x) {
  if (!dg::pr_cholesky_factor<6>(A, L)) return 0;
  dg::pr_cholesky_apply<6>(L, b, x);
  return 1;
}

}  // extern "C"
