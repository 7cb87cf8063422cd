// Host build of csrc/triangulate.h, the stopping rule of csrc/absolute_pose.h and the minimal sample of csrc/rng.h, the
// per-thread pieces of triangulate_tracks_ragged_kernel -- TEST HELPER ONLY (tests/test_triangulate.py compiles it
// with g++ -ffp-contract=off into a temporary directory and compares it with tests/triangulate_np.py).
#include "../pydegensac_b200/csrc/triangulate.h"
#include "../pydegensac_b200/csrc/rng.h"

extern "C" {

void trh_camera(const double* R, const double* t, const double* K, double* cam) { dg::tr_camera(R, t, K, cam); }

void trh_ray(const double* cam, double x, double y, double* d) { dg::tr_ray(cam, x, y, d); }

int trh_midpoint(const double* Ci, const double* di, const double* Cj, const double* dj, double cos_max, double* X) {
  return dg::tr_midpoint(Ci, di, Cj, dj, cos_max, X) ? 1 : 0;
}

// Per observation of X, in camera tab[cams[i]] at pts [n][2]: the MSAC term and the inlier flag
void trh_msac(const double* tab, const int* cams, const double* pts, int n, const double* X, double th2, double* term,
              int* inlier) {
  for (int i = 0; i < n; ++i) {
    bool in;
    term[i] = dg::tr_msac(tab + dg::kTrCamStride * cams[i], X, pts[2 * i], pts[2 * i + 1], th2, &in);
    inlier[i] = in ? 1 : 0;
  }
}

// Per observation: r [n][2] and J [n][2][3]
void trh_jacobian(const double* tab, const int* cams, const double* pts, int n, const double* X, double* r, double* J) {
  for (int i = 0; i < n; ++i)
    dg::tr_jacobian(tab + dg::kTrCamStride * cams[i], X, pts[2 * i], pts[2 * i + 1], r + 2 * i, J + 6 * i);
}

// The LM sums [10] over the observations, in row order
void trh_sums(const double* tab, const int* cams, const double* pts, int n, const double* X, double* sums) {
  for (int j = 0; j < dg::kTrSums; ++j) sums[j] = 0.0;
  for (int i = 0; i < n; ++i) dg::tr_row(tab + dg::kTrCamStride * cams[i], X, pts[2 * i], pts[2 * i + 1], sums);
}

int trh_solve(const double* H, const double* g, double lam, double* D) {
  return dg::pr_cholesky_solve<dg::kTrParams>(H, g, lam, D) ? 1 : 0;
}

void trh_pair_advance(int n, int s, int* i, int* j) { dg::tr_pair_advance(n, s, i, j); }

void trh_sample(unsigned long long seed, unsigned k, int n, int* sel) { dg::minimal_sample<2>(seed, k, n, sel); }

int trh_required_iters(int s, int has_best, int inl, int n, double conf, int max_iters, int k) {
  return s == 2 ? dg::required_iters<2>(has_best != 0, inl, n, conf, max_iters, k)
                : dg::required_iters<3>(has_best != 0, inl, n, conf, max_iters, k);
}

int trh_ap_required_iters(int has_best, int inl, int n, double conf, int max_iters, int k) {
  return dg::ap_required_iters(has_best != 0, inl, n, conf, max_iters, k);
}

}  // extern "C"
