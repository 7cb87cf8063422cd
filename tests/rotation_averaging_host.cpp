// g++ host build of csrc/rotation_averaging.h, the per-edge and per-view pieces of the rotation averaging -- TEST HELPER
// ONLY (tests/test_rotation_averaging.py compiles it into a temporary directory and checks it against
// tests/rotation_averaging_np.py).  Every function takes n items of row-major 3 x 3 matrices.
#include "../pydegensac_b200/csrc/rotation_averaging.h"

extern "C" {

// ok [n] = ra_edge_ok; R [n][9] prepared in place where ok
void rah_prepare(int n, double* R, int* ok) {
  for (int e = 0; e < n; ++e) {
    ok[e] = dg::ra_edge_ok(R + 9 * e) ? 1 : 0;
    if (ok[e]) dg::ra_prepare(R + 9 * e);
  }
}

// r [n][3] and theta [n] of ra_log
void rah_log(int n, const double* dR, double* r, double* th) {
  for (int e = 0; e < n; ++e) th[e] = dg::ra_log(dR + 9 * e, r + 3 * e);
}

// dR [n][9] = ra_relative(Ri, Rj, Re)
void rah_relative(int n, const double* Ri, const double* Rj, const double* Re, double* dR) {
  for (int e = 0; e < n; ++e) dg::ra_relative(Ri + 9 * e, Rj + 9 * e, Re + 9 * e, dR + 9 * e);
}

// Rc [n][9] = ra_compose(Re, Rp, child_is_j)
void rah_compose(int n, const double* Re, const double* Rp, const int* child_is_j, double* Rc) {
  for (int e = 0; e < n; ++e) dg::ra_compose(Re + 9 * e, Rp + 9 * e, child_is_j[e] != 0, Rc + 9 * e);
}

// w [n] = ra_weight(phase, theta, sig2)
void rah_weight(int n, int phase, const double* th, double sig2, double* w) {
  for (int e = 0; e < n; ++e) w[e] = dg::ra_weight(phase, th[e], sig2);
}

// R2 [n][9] = ra_update(R, w)
void rah_update(int n, const double* R, const double* w, double* R2) {
  for (int v = 0; v < n; ++v) dg::ra_update(R + 9 * v, w + 3 * v, R2 + 9 * v);
}

}  // extern "C"
