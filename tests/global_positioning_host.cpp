// g++ host build of csrc/global_positioning.h, the per-observation pieces of the global positioning -- TEST HELPER
// ONLY (tests/test_global_positioning.py compiles it into a temporary directory and checks it against
// tests/global_positioning_np.py).  Every function takes n rows.
#include "../pydegensac_b200/csrc/global_positioning.h"

extern "C" {

// v [n][3] = gp_ray of pixel (x, y) of a camera with rotation R [n][9] and intrinsics K [n][9]
void gph_ray(int n, const double* R, const double* K, const double* xy, double* v) {
  for (int i = 0; i < n; ++i) {
    double cam[dg::kTrCamStride];
    const double t0[3] = {0.0, 0.0, 0.0};
    dg::tr_camera(R + 9 * i, t0, K + 9 * i, cam);
    dg::gp_ray(cam, xy[2 * i], xy[2 * i + 1], v + 3 * i);
  }
}

// out [n][3] = gp_start(seed, kind, index[i], init_scale)
void gph_start(int n, unsigned long long seed, unsigned kind, const unsigned* index, double init_scale, double* out) {
  for (int i = 0; i < n; ++i) dg::gp_start(seed, kind, index[i], init_scale, out + 3 * i);
}

// a, r [n][3], s2 [n] = gp_residual; rho [n], w [n] = gp_rho, gp_weight of s2 at delta; the linearisation ok [n], u
// [n][3], nrm, s [n], h [n][3], ar [n] = gp_obs_terms(a, r, d, w)
void gph_terms(int n, const double* c, const double* X, const double* d, const double* v, double delta, double* a,
               double* r, double* s2, double* rho, double* w, int* ok, double* u, double* nrm, double* s, double* h,
               double* ar) {
  for (int i = 0; i < n; ++i) {
    s2[i] = dg::gp_residual(c + 3 * i, X + 3 * i, d[i], v + 3 * i, a + 3 * i, r + 3 * i);
    rho[i] = dg::gp_rho(s2[i], delta);
    w[i] = dg::gp_weight(s2[i], delta);
    ok[i] = dg::gp_obs_terms(a + 3 * i, r + 3 * i, d[i], w[i], u + 3 * i, nrm + i, s + i, h + 3 * i, ar + i) ? 1 : 0;
  }
}

// out [n][3] = gp_m_apply(u, s, f, p); blk [n][6] = gp_block(s, Q = s u u^T by gp_add_outer, lam); dn [n] =
// gp_scale_step(ar, nrm, d, u, p, lam); th [n] = gp_angle(u, p)
void gph_blocks(int n, const double* u, const double* s, double lam, const double* p, const double* ar,
                const double* nrm, const double* d, double* out, double* blk, double* dn, double* th) {
  for (int i = 0; i < n; ++i) {
    dg::gp_m_apply(u + 3 * i, s[i], 1.0 / (1.0 + lam), p + 3 * i, out + 3 * i);
    double Q[6] = {0, 0, 0, 0, 0, 0};
    dg::gp_add_outer(u + 3 * i, s[i], Q);
    dg::gp_block(s[i], Q, lam, blk + 6 * i);
    dn[i] = dg::gp_scale_step(ar[i], nrm[i], d[i], u + 3 * i, p + 3 * i, lam);
    th[i] = dg::gp_angle(u + 3 * i, p + 3 * i);
  }
}

}  // extern "C"
