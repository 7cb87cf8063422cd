// g++ host build of csrc/view_graph_calibration.h, the per-edge and per-group pieces of the view-graph calibration --
// TEST HELPER ONLY (tests/test_view_graph_calibration.py compiles it into a temporary directory and checks it against
// tests/view_graph_calibration_np.py).  Every function takes n items.
#include "../pydegensac_b200/csrc/view_graph_calibration.h"

extern "C" {

// ok [n] = vg_edge_ok(ij[2e], ij[2e+1], n_views, g[2e], g[2e+1], n_groups, mask[e], F + 9e)
void vgh_edge_ok(int n, const int* ij, int n_views, const int* g, int n_groups, const int* mask, const double* F,
                 int* ok) {
  for (int e = 0; e < n; ++e)
    ok[e] = dg::vg_edge_ok(ij[2 * e], ij[2 * e + 1], n_views, g[2 * e], g[2 * e + 1], n_groups, mask[e] != 0,
                           F + 9 * e) ? 1 : 0;
}

// ok [n] = vg_intrinsics_ok(k + 5e)
void vgh_intrinsics_ok(int n, const double* k, int* ok) {
  for (int e = 0; e < n; ++e) ok[e] = dg::vg_intrinsics_ok(k + 5 * e) ? 1 : 0;
}

// c [n][12] = vg_constants(F, ki, kj) where ok [n]
void vgh_constants(int n, const double* F, const double* ki, const double* kj, double* c, int* ok) {
  for (int e = 0; e < n; ++e) ok[e] = dg::vg_constants(F + 9 * e, ki + 5 * e, kj + 5 * e, c + 12 * e) ? 1 : 0;
}

// r [n][2], J [n][4] and s [n] = vg_residuals(c, ti, tj)
void vgh_residuals(int n, const double* c, const double* ti, const double* tj, double* r, double* J, double* s) {
  for (int e = 0; e < n; ++e) s[e] = dg::vg_residuals(c + 12 * e, ti[e], tj[e], r + 2 * e, J + 4 * e);
}

// rho [n], w [n] of s [n]
void vgh_loss(int n, const double* s, double sig2, double* rho, double* w) {
  for (int e = 0; e < n; ++e) {
    rho[e] = dg::vg_rho(s[e], sig2);
    w[e] = dg::vg_weight(s[e], sig2);
  }
}

// k_out [n][5] and refined [n] = vg_write_back(k_in, theta, has_edge, max_ratio)
void vgh_write_back(int n, const double* k_in, const double* theta, const int* has_edge, double max_ratio,
                    double* k_out, int* refined) {
  for (int g = 0; g < n; ++g)
    refined[g] = dg::vg_write_back(k_in + 5 * g, theta[g], has_edge[g] != 0, max_ratio, k_out + 5 * g) ? 1 : 0;
}

}  // extern "C"
