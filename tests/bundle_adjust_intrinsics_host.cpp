// g++ host build of csrc/camera_radial.h, the RADIAL camera model of bundle_adjust_intrinsics.cu: its projection, its
// Jacobians and its undistortion.  tests/test_bundle_adjust_intrinsics.py checks it against central differences and
// against tests/bundle_adjust_intrinsics_np.py.
#include <math.h>

#include "../pydegensac_b200/csrc/camera_radial.h"

extern "C" {

// r [2], J_cam [12], J_X [6], J_k [10] of X observed at (x, y) through pose P [12] and intrinsics k [5]
void radh_jacobian(const double* P, const double* k, const double* X, double x, double y, double* r, double* Jc,
                   double* Jx, double* Jk) {
  dg::rad_jacobian(P, k, X, x, y, r, Jc, Jx, Jk);
}

double radh_sq_error(const double* P, const double* k, const double* X, double x, double y, int* front) {
  bool f;
  const double e2 = dg::rad_sq_error(P, k, X, x, y, &f);
  *front = f ? 1 : 0;
  return e2;
}

// out [n][2] the pinhole pixels of pts [n][2]; returns how many rows converged
int radh_undistort(const double* k, const double* pts, int n, double* out) {
  int ok = 0;
  for (int i = 0; i < n; ++i) ok += dg::rad_undistort(k, pts[2 * i], pts[2 * i + 1], out + 2 * i) ? 1 : 0;
  return ok;
}

double radh_max_radius(double k1, double k2) { return dg::rad_max_radius(k1, k2); }

}  // extern "C"
