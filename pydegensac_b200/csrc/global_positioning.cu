// global_positioning.cu -- global positioning, device resident: the views' centres and the tracks' points from the
// views' rotations and the tracks' rays (GLOMAP's global positioner with point-to-camera constraints; the pairwise
// direction error of BATA).  Levenberg-Marquardt from a random start over the centres, the points and one scale per
// observation, each trial step solved through a nested Schur complement: every observation's scale is eliminated into
// its (centre, point) block, every track's point into the centres' reduced system, which conjugate gradients solve
// matrix-free with a block-Jacobi preconditioner (as bundle_adjust_pcg.cu, with 3-parameter cameras).  A translation
// unit of its own, so that adding it changes no instruction of the other sources' kernels.  The estimator is specified
// in include/degensac_b200.h; the per-thread pieces are in global_positioning.h.
//
// Once per call:
//   gp_cameras_kernel    one thread per view: the camera table (triangulate.h's, with t = 0), the union-find's roots;
//   gp_mark_kernel       one warp per track: the usable observations and their rays, whether the track is used, and
//                        tk_link (tracks.h) of the cameras of its used observations;
//   gp_compress_kernel   one thread per view: tk_compress, so each view points at its component's smallest view;
//   gp_key_kernel,       the camera-major list of the used observations of the views that move (every active view but
//   gp_count_kernel,     the anchors), ascending observation order within a view, by the one-digit stable counting
//   gp_scan_kernel,      sort of bundle_adjust_device.h (ba_sort_*);
//   gp_scatter_kernel
//   gp_start_views_kernel, gp_start_tracks_kernel  the random start and its cost;
//   gp_init_kernel       one CTA: cost0, n_used and the LM state.
// Per trial step (the host launches max_iters steps; each kernel returns at once when the state says the call stopped):
//   gp_linearise_kernel  one warp per used track, after an accepted step: each observation's linearisation (u, s, |a|,
//                        a . r by observation; u, s, h camera-major) and the track's sums;
//   gp_points_kernel     one thread per used track: V*_j^-1 and t_j = V*_j^-1 g_j;
//   gp_precond_kernel    one warp per view: U*, the preconditioner block M (S's diagonal block) and its Cholesky
//                        factor, the right-hand side and the start of PCG;
//   gp_solve_kernel      the whole PCG loop in one cooperative launch (grid.sync between the phases), then the trial
//                        centres;
//   gp_backsub_kernel    one warp per used track: the trial point, the trial scales and the track's trial cost;
//   gp_decide_kernel     one CTA: ba_decide_step.
// After the last step gp_finish_views_kernel, gp_finish_tracks_kernel and gp_finish_obs_kernel write the outputs.
//
// One PCG iteration: A, one thread per track: y_j = V*_j^-1 sum m_o p_i(o); B, one warp per view: q_i = U*_i p_i -
// sum m_o y_j(o) over its camera-major list, p_i . q_i; C, one thread per view: x += alpha p, r -= alpha q, z = M^-1 r;
// r . r and r . z; the loop is pcg_run (pcg_device.h), whose dot products every CTA sums itself in one fixed order, so
// they do not depend on the grid.  No floating-point atomics anywhere: a rerun gives the same bytes.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/degensac_b200.h"
#include "entry_error.h"
#include "bundle_adjust_args.h"
#include "common.h"
#include "global_positioning.h"
#include "tracks.h"
#include "device_util.h"
#include "bundle_adjust_device.h"
#include "pcg_device.h"
#include "adjust_host.h"

namespace cg = cooperative_groups;

namespace {

thread_local char g_err[256] = "";
int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err, code, what, e); }

constexpr int kGpThreads = 128;                   // the one-thread-per-item kernels
constexpr int kGpWarps = 4;                       // tracks or views per CTA of the one-warp-per-item kernels
constexpr int kGpSolveThreads = 256;              // the cooperative kernel
constexpr int kGpRange = 4096;                    // observations per warp of the counting sort

// One observation's linearisation in observation order (u [3], s = w d^2, |a|, a . r) and camera-major (u [3], s,
// h = w d r [3]); structure of arrays, [k][obs]
constexpr int kLoU = 0, kLoS = 3, kLoN = 4, kLoAR = 5, kLoRows = 6;
constexpr int kLcU = 0, kLcS = 3, kLcH = 4, kLcRows = 7;
// One track's sums at the linearisation: Q = sum s u u^T (upper, 6), sum h, sum u (u . h), sum s; the trial cost at
// bundle_adjust.h's kBaTrkCost, so that ba_decide_step reads it
constexpr int kGtQ = 0, kGtH = 6, kGtUH = 9, kGtS = 12;
static_assert(dg::kBaTrkCost == 15 && dg::kBaTrkStride == 16, "the track record shares bundle_adjust.h's cost slot");
// One track's V*^-1 (upper, 6) and t = V*^-1 g (3)
constexpr int kGvVi = 0, kGvT = 6, kGvStride = 9;
// One view's record: U* (upper, 6), the preconditioner's Cholesky factor L (lower, 6), then its PCG vectors
// (pcg_device.h): b, x, r, z (3 each), p in two buffers (6), q (3)
constexpr int kGcU = 0, kGcL = 6, kGcB = 12, kGcX = 15, kGcP = 24, kGcQ = 30, kGcStride = 33;

struct GpArgs {
  const int* cams; const double* pts;                      // [obs], [obs][2]
  const double* R; const double* K;
  int k_per_camera, n_cams;
  const int* offsets; const unsigned char* mask;           // [T+1], [obs] or null
  int n_tracks, obs, n_ranges, cg_max_iters;
  unsigned long long seed;
  double init_scale, delta, max_angle, cg_tol2;
  // workspace
  double* tab;       // [n_cams][kTrCamStride]
  double* cen;       // [2][n_cams][3]: current and trial centres
  double* Xb;        // [2][T][3]
  double* dsc;       // [2][obs]: the scales
  double* ray;       // [3][obs]
  double* lo;        // [kLoRows][obs]
  double* lc;        // [kLcRows][obs], camera-major
  double* trk;       // [T][kBaTrkStride]
  double* tv;        // [T][kGvStride]
  double* y;         // [T][3]
  double* rec;       // [n_cams][kGcStride]
  double* part;      // [kPcgParts][n_cams]
  BaState* state;
  int* cg_iters;     // [1]
  int* linbad;       // [1]: the linearisation has an observation with |a| = 0 or not finite
  int* parent;       // [n_cams]
  int* active;       // [n_cams]: the view has a used observation
  int* key;          // [obs]: the view of a used observation of a view that moves, or -1
  int* track_of;     // [obs]
  int* pos_of;       // [obs]
  int* ctrk;         // [obs]: the track of each camera-major entry
  int* hist;         // [n_cams][n_ranges]
  int* list_off;     // [n_cams + 1]
  int* trk_used;     // [T]: used observations of the track (0: not used)
  unsigned char* used;   // [obs]
  // outputs
  double* t_out; double* X_out; int* comp_out; double* angle_out; unsigned char* inl_out;
  double* cost0_out; double* cost_out; int* iters_out; int* n_used_out; int* cg_iters_out;
};

__device__ __forceinline__ double* centre(const GpArgs& a, int buf, int c) {
  return a.cen + 3 * ((size_t)buf * a.n_cams + c);
}
__device__ __forceinline__ double* point_of(const GpArgs& a, int buf, int j) {
  return a.Xb + 3 * ((size_t)buf * a.n_tracks + j);
}
__device__ __forceinline__ double* view_rec(const GpArgs& a, int c) { return a.rec + kGcStride * (size_t)c; }
__device__ __forceinline__ void load_ray(const GpArgs& a, int r, double* v) {
  const size_t no = (size_t)a.obs;
  v[0] = a.ray[r]; v[1] = a.ray[no + r]; v[2] = a.ray[2 * no + r];
}
__device__ __forceinline__ bool span_ok(const GpArgs& a, int b, int e) { return b >= 0 && b <= e && e <= a.obs; }

// ---------------------------------------------------------------------------------------------- once per call
__global__ void __launch_bounds__(kGpThreads) gp_cameras_kernel(GpArgs a) {
  const int c = blockIdx.x * kGpThreads + threadIdx.x;
  if (c >= a.n_cams) return;
  const double t0[3] = {0.0, 0.0, 0.0};
  dg::tr_camera(a.R + 9 * (size_t)c, t0, a.K + (a.k_per_camera ? 9 * (size_t)c : 0),
                a.tab + dg::kTrCamStride * (size_t)c);
  a.parent[c] = c;
  a.active[c] = 0;
}

// One warp per track: usable rows (mask, camera in range and registered, finite pixel) get their ray; the track is used
// when they come from at least 2 distinct cameras, and then its usable rows are used and their cameras linked
__global__ void __launch_bounds__(32 * kGpWarps) gp_mark_kernel(GpArgs a) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kGpWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks) return;                       // (warp-uniform)
  if (lane == 0) a.trk_used[j] = 0;
  const int b = a.offsets[j], e = a.offsets[j + 1];
  if (!span_ok(a, b, e)) return;                     // malformed span: no row read or written
  const size_t no = (size_t)a.obs;
  int first_cam = -1, n = 0;
  bool two = false;
  for (int c0 = b; c0 < e; c0 += 32) {
    const int r = c0 + lane;
    bool ok = false;
    int cm = -1;
    if (r < e) {
      cm = a.cams[r];
      const double x = a.pts[2 * (size_t)r], y = a.pts[2 * (size_t)r + 1];
      ok = (!a.mask || a.mask[r]) && cm >= 0 && cm < a.n_cams && finite(x) && finite(y) &&
           a.tab[dg::kTrCamStride * (size_t)cm + dg::kTrCamOk] != 0.0;
      if (ok) {
        double v[3];
        dg::gp_ray(a.tab + dg::kTrCamStride * (size_t)cm, x, y, v);
        a.ray[r] = v[0]; a.ray[no + r] = v[1]; a.ray[2 * no + r] = v[2];
      }
      a.used[r] = ok ? 1 : 0;
    }
    const unsigned bal = __ballot_sync(kFull, ok);
    if (bal) {
      if (first_cam < 0) first_cam = __shfl_sync(kFull, cm, __ffs(bal) - 1);
      two = two || __any_sync(kFull, ok && cm != first_cam);
    }
    n += __popc(bal);
  }
  __syncwarp();
  for (int r = b + lane; r < e; r += 32) {           // (the rows this lane wrote above)
    const unsigned char u = two ? a.used[r] : 0;
    a.used[r] = u;
    a.track_of[r] = j;
    if (u) {
      const int cm = a.cams[r];
      a.active[cm] = 1;                              // (the same store from every thread that makes it)
      dg::tk_link(a.parent, cm, first_cam);
    }
  }
  if (two && lane == 0) a.trk_used[j] = n;
}

__global__ void __launch_bounds__(kGpThreads) gp_compress_kernel(GpArgs a) {
  const int c = blockIdx.x * kGpThreads + threadIdx.x;
  if (c < a.n_cams) dg::tk_compress(a.parent, c);
}

__global__ void __launch_bounds__(kGpThreads) gp_key_kernel(GpArgs a) {
  const int r = blockIdx.x * kGpThreads + threadIdx.x;
  if (r >= a.obs) return;
  int k = -1;
  if (a.used[r]) {
    const int cm = a.cams[r];
    if (a.parent[cm] != cm) k = cm;                  // an anchor does not move
  }
  a.key[r] = k;
}

__global__ void __launch_bounds__(32 * kGpWarps) gp_count_kernel(GpArgs a) {
  const int w = blockIdx.x * kGpWarps + (threadIdx.x >> 5);
  if (w >= a.n_ranges) return;                       // (warp-uniform)
  ba_sort_count(a.key, a.obs, kGpRange, a.hist, a.n_ranges, w, threadIdx.x & 31);
}

__global__ void __launch_bounds__(kBaCta) gp_scan_kernel(GpArgs a) {
  __shared__ int sh[kBaCta];
  ba_sort_scan(a.hist, a.n_cams, a.n_ranges, a.list_off, sh);
}

__global__ void __launch_bounds__(32 * kGpWarps) gp_scatter_kernel(GpArgs a) {
  const int w = blockIdx.x * kGpWarps + (threadIdx.x >> 5);
  if (w >= a.n_ranges) return;                       // (warp-uniform)
  ba_sort_scatter(a.key, a.obs, kGpRange, a.hist, a.n_ranges, a.track_of, a.pos_of, a.ctrk, w, threadIdx.x & 31);
}

// Both centre buffers: NaN for an inactive view, 0 for an anchor, else the random start
__global__ void __launch_bounds__(kGpThreads) gp_start_views_kernel(GpArgs a) {
  const int c = blockIdx.x * kGpThreads + threadIdx.x;
  if (c >= a.n_cams) return;
  double s[3] = {0.0, 0.0, 0.0};
  if (!a.active[c]) s[0] = s[1] = s[2] = qnan();
  else if (a.parent[c] != c) dg::gp_start(a.seed, dg::kGpKindView, (uint32_t)c, a.init_scale, s);
  for (int buf = 0; buf < 2; ++buf)
    for (int k = 0; k < 3; ++k) centre(a, buf, c)[k] = s[k];
}

// One warp per track: both point buffers (NaN for a track that is not used), d = 1 in both scale buffers, the start
// cost
__global__ void __launch_bounds__(32 * kGpWarps) gp_start_tracks_kernel(GpArgs a) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kGpWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks) return;                       // (warp-uniform)
  const bool use = a.trk_used[j] > 0;
  double X[3] = {qnan(), qnan(), qnan()};
  if (use) dg::gp_start(a.seed, dg::kGpKindTrack, (uint32_t)j, a.init_scale, X);
  if (lane < 3) {
    point_of(a, 0, j)[lane] = X[lane];
    point_of(a, 1, j)[lane] = X[lane];
  }
  double c = 0.0;
  if (use) {
    const int b = a.offsets[j], e = a.offsets[j + 1];
    for (int r = b + lane; r < e; r += 32) {
      if (!a.used[r]) continue;
      a.dsc[r] = 1.0;
      a.dsc[(size_t)a.obs + r] = 1.0;
      double v[3], av[3], rr[3];
      load_ray(a, r, v);
      c += dg::gp_rho(dg::gp_residual(centre(a, 0, a.cams[r]), X, 1.0, v, av, rr), a.delta);
    }
    c = warp_sum(c);
  }
  if (lane == 0) a.trk[dg::kBaTrkStride * (size_t)j + dg::kBaTrkCost] = c;
}

__global__ void __launch_bounds__(kBaCta) gp_init_kernel(GpArgs a) {
  __shared__ double shd[kBaCta];
  __shared__ int shi[kBaCta / 32];
  double c = 0.0;
  int u = 0;
  for (int j = threadIdx.x; j < a.n_tracks; j += kBaCta) {
    c += a.trk[dg::kBaTrkStride * (size_t)j + dg::kBaTrkCost];
    u += a.trk_used[j];
  }
  c = block_sum_double(c, shd);
  u = block_sum_int(u, shi);
  if (threadIdx.x == 0) {
    BaState* st = a.state;
    st->lam = dg::kPrLambda0;
    st->cost = c;
    st->cost0 = c;
    st->cur = 0;
    st->stop = 0;
    st->lin = 1;
    st->bad = 0;
    st->iters = 0;
    st->n_used = u;
    st->hold_row = -1;
    a.cg_iters[0] = 0;
    a.linbad[0] = 0;
  }
}

// ---------------------------------------------------------------------------------------------- one trial step
__global__ void __launch_bounds__(32 * kGpWarps) gp_linearise_kernel(GpArgs a) {
  const BaState* st = a.state;
  if (st->stop || !st->lin) return;
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kGpWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks || a.trk_used[j] == 0) return;   // (warp-uniform)
  const int cur = st->cur;
  const double* X = point_of(a, cur, j);
  const int b = a.offsets[j], e = a.offsets[j + 1];
  const size_t no = (size_t)a.obs;
  double Q[6] = {0, 0, 0, 0, 0, 0}, H[3] = {0, 0, 0}, UH[3] = {0, 0, 0}, S = 0.0;
  bool bad = false;
  for (int r = b + lane; r < e; r += 32) {
    if (!a.used[r]) continue;
    const int cm = a.cams[r];
    const double d = a.dsc[(size_t)cur * no + r];
    double v[3], av[3], rr[3], u[3], h[3], n, s, ar;
    load_ray(a, r, v);
    const double w = dg::gp_weight(dg::gp_residual(centre(a, cur, cm), X, d, v, av, rr), a.delta);
    if (!dg::gp_obs_terms(av, rr, d, w, u, &n, &s, h, &ar)) {
      bad = true;
      continue;
    }
    a.lo[kLoU * no + r] = u[0]; a.lo[(kLoU + 1) * no + r] = u[1]; a.lo[(kLoU + 2) * no + r] = u[2];
    a.lo[kLoS * no + r] = s; a.lo[kLoN * no + r] = n; a.lo[kLoAR * no + r] = ar;
    const int k = a.key[r];
    if (k >= 0) {
      const size_t pos = (size_t)a.pos_of[r];
#pragma unroll
      for (int m = 0; m < 3; ++m) {
        a.lc[(kLcU + m) * no + pos] = u[m];
        a.lc[(kLcH + m) * no + pos] = h[m];
      }
      a.lc[kLcS * no + pos] = s;
    }
    dg::gp_add_outer(u, s, Q);
    const double uh = u[0] * h[0] + u[1] * h[1] + u[2] * h[2];
#pragma unroll
    for (int m = 0; m < 3; ++m) {
      H[m] += h[m];
      UH[m] += u[m] * uh;
    }
    S += s;
  }
#pragma unroll
  for (int m = 0; m < 6; ++m) Q[m] = warp_sum(Q[m]);
#pragma unroll
  for (int m = 0; m < 3; ++m) {
    H[m] = warp_sum(H[m]);
    UH[m] = warp_sum(UH[m]);
  }
  S = warp_sum(S);
  bad = __any_sync(kFull, bad);
  if (lane == 0) {
    double* tk = a.trk + dg::kBaTrkStride * (size_t)j;
#pragma unroll
    for (int m = 0; m < 6; ++m) tk[kGtQ + m] = Q[m];
#pragma unroll
    for (int m = 0; m < 3; ++m) {
      tk[kGtH + m] = H[m];
      tk[kGtUH + m] = UH[m];
    }
    tk[kGtS] = S;
    if (bad) a.linbad[0] = 1;
  }
}

// V*_j = (1 + lambda) S I - Q / (1 + lambda), its inverse, and t_j = V*_j^-1 g_j with g_j = sum h - sum u (u . h) /
// (1 + lambda), the point's gradient once the scales are eliminated
__global__ void __launch_bounds__(kGpThreads) gp_points_kernel(GpArgs a) {
  BaState* st = a.state;
  if (st->stop) return;
  const int j = blockIdx.x * kGpThreads + threadIdx.x;
  if (j == 0 && a.linbad[0]) st->bad = 1;            // the step is rejected
  if (j >= a.n_tracks || a.trk_used[j] == 0) return;
  const double lam = st->lam, f = 1.0 / (1.0 + lam);
  const double* tk = a.trk + dg::kBaTrkStride * (size_t)j;
  double Vs[6], Vi[6];
  dg::gp_block(tk[kGtS], tk + kGtQ, lam, Vs);
  if (!dg::ba_inv3(Vs, 0.0, Vi)) {
    st->bad = 1;                                     // the step is rejected
    return;
  }
  const double g[3] = {tk[kGtH] - f * tk[kGtUH], tk[kGtH + 1] - f * tk[kGtUH + 1], tk[kGtH + 2] - f * tk[kGtUH + 2]};
  double* o = a.tv + kGvStride * (size_t)j;
#pragma unroll
  for (int m = 0; m < 6; ++m) o[kGvVi + m] = Vi[m];
  dg::ba_sym3_mul(Vi, g, o + kGvT);
}

// One warp per view over its camera-major list: U* = (1 + lambda) S I - Q / (1 + lambda), M = U* - sum_j W_ij V*_j^-1
// W_ij^T with W_ij = sum of m over the view's observations of track j (S's diagonal block), and
// b = sum (e - m t), e = h - u (u . h) / (1 + lambda); a view without a list (inactive or an anchor) gets U* = 0, M = I
// and b = 0.  Then the start of PCG: x = 0, r = b, z = M^-1 r, both p buffers 0, and the view's r . z and b . b.
__global__ void __launch_bounds__(32 * kGpWarps) gp_precond_kernel(GpArgs a) {
  BaState* st = a.state;
  if (st->stop || st->bad) return;
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kGpWarps + (threadIdx.x >> 5);
  if (c >= a.n_cams) return;                         // (warp-uniform)
  const size_t no = (size_t)a.obs;
  const double lam = st->lam, f = 1.0 / (1.0 + lam);
  double S = 0.0, Q[6] = {0, 0, 0, 0, 0, 0}, Mv[6] = {0, 0, 0, 0, 0, 0}, bv[3] = {0, 0, 0};
  const int i0 = a.list_off[c], i1 = a.list_off[c + 1];
  for (int i = i0 + lane; i < i1; i += 32) {
    const double u[3] = {a.lc[kLcU * no + i], a.lc[(kLcU + 1) * no + i], a.lc[(kLcU + 2) * no + i]};
    const double h[3] = {a.lc[kLcH * no + i], a.lc[(kLcH + 1) * no + i], a.lc[(kLcH + 2) * no + i]};
    const double s = a.lc[kLcS * no + i];
    const int j = a.ctrk[i];
    const double* tv = a.tv + kGvStride * (size_t)j;
    double mt[3];
    dg::gp_m_apply(u, s, f, tv + kGvT, mt);
    const double uh = f * (u[0] * h[0] + u[1] * h[1] + u[2] * h[2]);
#pragma unroll
    for (int m = 0; m < 3; ++m) bv[m] += (h[m] - uh * u[m]) - mt[m];
    // W_ij V*_j^-1 W_ij^T once per (view, track): the entry that starts a run of the track's observations in this view
    // (adjacent in the list, which keeps observation order) sums m over the run, so that M is S's diagonal block
    if (i == i0 || a.ctrk[i - 1] != j) {
      double A[6] = {0, 0, 0, 0, 0, 0};
      for (int k = i; k < i1 && a.ctrk[k] == j; ++k) {
        const double uk[3] = {a.lc[kLcU * no + k], a.lc[(kLcU + 1) * no + k], a.lc[(kLcU + 2) * no + k]};
        dg::gp_m_add(uk, a.lc[kLcS * no + k], f, A);
      }
      dg::gp_sandwich(A, tv + kGvVi, Mv);
    }
    dg::gp_add_outer(u, s, Q);
    S += s;
  }
  S = warp_sum(S);
#pragma unroll
  for (int m = 0; m < 6; ++m) {
    Q[m] = warp_sum(Q[m]);
    Mv[m] = warp_sum(Mv[m]);
  }
#pragma unroll
  for (int m = 0; m < 3; ++m) bv[m] = warp_sum(bv[m]);
  if (lane != 0) return;
  const bool act = i1 > i0;
  double U[6], M[6];
  dg::gp_block(S, Q, lam, U);
#pragma unroll
  for (int m = 0; m < 6; ++m) M[m] = act ? U[m] - Mv[m] : (m == 0 || m == 3 || m == 5 ? 1.0 : 0.0);
  double* rec = view_rec(a, c);
  if (!dg::pr_cholesky_factor<3>(M, rec + kGcL)) {
    st->bad = 1;                                     // the step is rejected
    return;
  }
  double b[3], z[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) b[k] = act ? bv[k] : 0.0;
  dg::pr_cholesky_apply<3>(rec + kGcL, b, z);
  pcg_start<3>(rec + kGcB, b, z, a.part, a.n_cams, c);
#pragma unroll
  for (int m = 0; m < 6; ++m) rec[kGcU + m] = act ? U[m] : 0.0;
}

// pcg_run's S p and phase C over the views.  product: A, one thread per track, y_j = V*_j^-1 sum m_o p_i(o); grid.sync;
// B, one warp per view, q_c = U*_c p_c - sum m_o y_j(o), p_c stored, p_c . q_c.  update: one thread per view.
struct GpSchur {
  const GpArgs& a;
  int tid, nthr, lane, warp, nwarps;
  double f;

  __device__ __forceinline__ void product(cg::grid_group& grid, int cur, int prev, double beta) const {
    const int nc = a.n_cams;
    const size_t no = (size_t)a.obs;
    for (int j = tid; j < a.n_tracks; j += nthr) {
      if (a.trk_used[j] == 0) continue;
      const int b = a.offsets[j], e = a.offsets[j + 1];
      double acc[3] = {0.0, 0.0, 0.0};
      for (int r = b; r < e; ++r) {
        const int k = a.key[r];
        if (k < 0) continue;
        double p[3], mp[3];
        pcg_direction<3>(view_rec(a, k) + kGcB, prev, beta, p);
        const double u[3] = {__ldg(a.lo + kLoU * no + r), __ldg(a.lo + (kLoU + 1) * no + r),
                             __ldg(a.lo + (kLoU + 2) * no + r)};
        dg::gp_m_apply(u, __ldg(a.lo + kLoS * no + r), f, p, mp);
        acc[0] += mp[0]; acc[1] += mp[1]; acc[2] += mp[2];
      }
      double yv[3];
      dg::ba_sym3_mul(a.tv + kGvStride * (size_t)j + kGvVi, acc, yv);
#pragma unroll
      for (int m = 0; m < 3; ++m) a.y[3 * (size_t)j + m] = yv[m];
    }
    grid.sync();
    for (int c = warp; c < nc; c += nwarps) {
      double acc[3] = {0.0, 0.0, 0.0};
      const int i0 = a.list_off[c], i1 = a.list_off[c + 1];
      for (int i = i0 + lane; i < i1; i += 32) {
        const double* yp = a.y + 3 * (size_t)a.ctrk[i];
        const double yv[3] = {__ldcg(yp), __ldcg(yp + 1), __ldcg(yp + 2)};
        const double u[3] = {__ldg(a.lc + kLcU * no + i), __ldg(a.lc + (kLcU + 1) * no + i),
                             __ldg(a.lc + (kLcU + 2) * no + i)};
        double my[3];
        dg::gp_m_apply(u, __ldg(a.lc + kLcS * no + i), f, yv, my);
        acc[0] += my[0]; acc[1] += my[1]; acc[2] += my[2];
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) acc[k] = warp_sum(acc[k]);
      if (lane == 0) {
        double p[3], Up[3];
        double* rec = view_rec(a, c);
        pcg_direction<3>(rec + kGcB, prev, beta, p);
        dg::ba_sym3_mul(rec + kGcU, p, Up);
        double pq = 0.0;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double q = Up[k] - acc[k];
          rec[kGcQ + k] = q;
          rec[kGcP + 3 * cur + k] = p[k];
          pq += p[k] * q;
        }
        a.part[kPartPQ * (size_t)nc + c] = pq;
      }
    }
  }

  __device__ __forceinline__ void update(int cur, int /*prev*/, double /*beta*/, double alpha) const {
    const int nc = a.n_cams;
    for (int c = tid; c < nc; c += nthr) {
      double* rec = view_rec(a, c);
      double p[3], q[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        p[k] = __ldcg(rec + kGcP + 3 * cur + k);
        q[k] = __ldcg(rec + kGcQ + k);
      }
      const double2 rz = pcg_update<3>(rec + kGcB, p, q, alpha, [rec](const double* r, double* z) {
        dg::pr_cholesky_apply<3>(rec + kGcL, r, z);
      });
      a.part[kPartRR * (size_t)nc + c] = rz.x;
      a.part[kPartRZ * (size_t)nc + c] = rz.y;
    }
  }
};

// The PCG loop of one trial step (pcg_run), then the trial centres
__global__ void __launch_bounds__(kGpSolveThreads) gp_solve_kernel(GpArgs a) {
  __shared__ double sh[2 * kGpSolveThreads];
  BaState* st = a.state;
  if (st->stop || st->bad) return;                   // (grid-uniform: nothing below writes them before a grid.sync)
  cg::grid_group grid = cg::this_grid();
  const int tid = blockIdx.x * kGpSolveThreads + threadIdx.x, nthr = gridDim.x * kGpSolveThreads;
  const int nc = a.n_cams;
  const GpSchur op{a, tid, nthr, (int)threadIdx.x & 31, tid >> 5, nthr >> 5, 1.0 / (1.0 + st->lam)};
  const PcgResult res = pcg_run<kGpSolveThreads>(grid, a.part, nc, a.cg_tol2, a.cg_max_iters, sh, op);
  // the trial centres of the views that move (x of a view was last written by this thread, in phase C)
  const int cur = st->cur;
  if (!res.reject)
    for (int c = tid; c < nc; c += nthr) {
      if (a.list_off[c + 1] == a.list_off[c]) continue;
      const double* x = view_rec(a, c) + kGcX;
      const double* c0 = centre(a, cur, c);
      double* c1 = centre(a, 1 - cur, c);
      for (int k = 0; k < 3; ++k) c1[k] = c0[k] + x[k];
    }
  if (tid == 0) {
    a.cg_iters[0] += res.iters;
    if (res.reject) st->bad = 1;
  }
}

// One warp per used track: dX = -t + V*^-1 sum m_o dc_i(o); each used observation's trial scale max(d + dd, d_min);
// the track's trial cost, +inf when an observation's |a| is 0 or not finite there
__global__ void __launch_bounds__(32 * kGpWarps) gp_backsub_kernel(GpArgs a) {
  const BaState* st = a.state;
  if (st->stop || st->bad) return;
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kGpWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks || a.trk_used[j] == 0) return;   // (warp-uniform)
  const int cur = st->cur, b = a.offsets[j], e = a.offsets[j + 1];
  const size_t no = (size_t)a.obs;
  const double lam = st->lam, f = 1.0 / (1.0 + lam);
  double acc[3] = {0.0, 0.0, 0.0};
  for (int r = b + lane; r < e; r += 32) {
    const int k = a.key[r];
    if (k < 0) continue;
    const double u[3] = {a.lo[kLoU * no + r], a.lo[(kLoU + 1) * no + r], a.lo[(kLoU + 2) * no + r]};
    double md[3];
    dg::gp_m_apply(u, a.lo[kLoS * no + r], f, view_rec(a, k) + kGcX, md);
    acc[0] += md[0]; acc[1] += md[1]; acc[2] += md[2];
  }
#pragma unroll
  for (int m = 0; m < 3; ++m) acc[m] = warp_sum(acc[m]);
  const double* tv = a.tv + kGvStride * (size_t)j;
  double D[3];
  dg::ba_sym3_mul(tv + kGvVi, acc, D);
  const double dX[3] = {D[0] - tv[kGvT], D[1] - tv[kGvT + 1], D[2] - tv[kGvT + 2]};
  const double* X0 = point_of(a, cur, j);
  const double X[3] = {X0[0] + dX[0], X0[1] + dX[1], X0[2] + dX[2]};
  if (lane < 3) point_of(a, 1 - cur, j)[lane] = X[lane];
  double c = 0.0;
  for (int r = b + lane; r < e; r += 32) {
    if (!a.used[r]) continue;
    const int cm = a.cams[r], k = a.key[r];
    const double* dc = view_rec(a, cm) + kGcX;
    const double dXc[3] = {k >= 0 ? dX[0] - dc[0] : dX[0], k >= 0 ? dX[1] - dc[1] : dX[1],
                           k >= 0 ? dX[2] - dc[2] : dX[2]};
    const double u[3] = {a.lo[kLoU * no + r], a.lo[(kLoU + 1) * no + r], a.lo[(kLoU + 2) * no + r]};
    const double d = dg::gp_scale_step(a.lo[kLoAR * no + r], a.lo[kLoN * no + r], a.dsc[(size_t)cur * no + r], u, dXc,
                                       lam);
    a.dsc[(size_t)(1 - cur) * no + r] = d;
    double v[3], av[3], rr[3];
    load_ray(a, r, v);
    const double s2 = dg::gp_residual(centre(a, 1 - cur, cm), X, d, v, av, rr);
    const double na = sqrt(av[0] * av[0] + av[1] * av[1] + av[2] * av[2]);
    c += (na > 0.0 && na < INFINITY) ? dg::gp_rho(s2, a.delta) : INFINITY;
  }
  c = warp_sum(c);
  if (lane == 0) a.trk[dg::kBaTrkStride * (size_t)j + dg::kBaTrkCost] = c;
}

__global__ void __launch_bounds__(kBaCta) gp_decide_kernel(GpArgs a) {
  __shared__ double shd[kBaCta];
  if (a.state->stop) return;                         // (block-uniform)
  ba_decide_step(a, shd);
}

// ---------------------------------------------------------------------------------------------- outputs
__global__ void __launch_bounds__(kGpThreads) gp_finish_views_kernel(GpArgs a) {
  const int c = blockIdx.x * kGpThreads + threadIdx.x;
  const BaState* st = a.state;
  if (c == 0) {
    a.cost0_out[0] = st->cost0;
    a.cost_out[0] = st->cost;
    a.iters_out[0] = st->iters;
    a.n_used_out[0] = st->n_used;
    a.cg_iters_out[0] = a.cg_iters[0];
  }
  if (c >= a.n_cams) return;
  const bool act = a.active[c] != 0;
  const double* R = a.R + 9 * (size_t)c;
  const double* x = centre(a, st->cur, c);
  for (int k = 0; k < 3; ++k)
    a.t_out[3 * (size_t)c + k] = act ? -(R[3 * k] * x[0] + R[3 * k + 1] * x[1] + R[3 * k + 2] * x[2]) : qnan();
  a.comp_out[c] = act ? a.parent[c] : -1;
}

__global__ void __launch_bounds__(kGpThreads) gp_finish_tracks_kernel(GpArgs a) {
  const int j = blockIdx.x * kGpThreads + threadIdx.x;
  if (j >= a.n_tracks) return;
  const double* X = point_of(a, a.state->cur, j);   // (NaN for a track that is not used)
  for (int k = 0; k < 3; ++k) a.X_out[3 * (size_t)j + k] = X[k];
}

__global__ void __launch_bounds__(kGpThreads) gp_finish_obs_kernel(GpArgs a) {
  const int r = blockIdx.x * kGpThreads + threadIdx.x;
  if (r >= a.obs) return;
  double th = qnan();
  if (a.used[r]) {
    const int cur = a.state->cur;
    const double* X = point_of(a, cur, a.track_of[r]);
    const double* c = centre(a, cur, a.cams[r]);
    double v[3];
    load_ray(a, r, v);
    const double av[3] = {X[0] - c[0], X[1] - c[1], X[2] - c[2]};
    th = dg::gp_angle(v, av);
  }
  a.angle_out[r] = th;
  a.inl_out[r] = th <= a.max_angle ? 1 : 0;          // (false for NaN)
}

}  // namespace

extern "C" {

const char* dgb200_global_positioning_last_error(void) { return g_err; }

int dgb200_global_positioning_ragged_dev(const int32_t* d_cams, const double* d_pts, const double* d_R,
                                         const double* d_K, int k_per_camera, int n_cams, const int32_t* d_offsets,
                                         int n_tracks, int obs, const uint8_t* d_mask, uint64_t seed,
                                         double init_scale, double loss_scale, int max_iters, double max_angle,
                                         int cg_max_iters, double cg_tol, double* d_t_out, double* d_X_out,
                                         int32_t* d_component_out, double* d_angle_out, uint8_t* d_inliers_out,
                                         double* d_cost0_out, double* d_cost_out, int32_t* d_iters_out,
                                         int32_t* d_n_used_out, int32_t* d_cg_iters_out, void* stream) {
  int gauge_slot = -1, held_cam = -1;
  // the bundle adjustments' shared checks, in their order; no camera list and no scale gauge here, and no pixel
  // threshold (1.0 passes its check)
  const char* bad = ba_arg_error(!d_R || !d_K || !d_offsets || !d_t_out || !d_X_out || !d_component_out ||
                                     !d_cost0_out || !d_cost_out || !d_iters_out || !d_n_used_out || !d_cg_iters_out,
                                 !d_cams || !d_pts || !d_angle_out || !d_inliers_out, n_tracks, obs, n_cams, nullptr,
                                 0, 0, "", -1, loss_scale, max_iters, 1.0, &gauge_slot, &held_cam);
  if (bad) return fail(DGB200_E_ARG, bad);
  if (!(init_scale >= 0.0) || !(init_scale < INFINITY))
    return fail(DGB200_E_ARG, "init_scale must be a non-negative finite number");
  if (!(max_angle >= 0.0) || !(max_angle < INFINITY))
    return fail(DGB200_E_ARG, "max_angle must be a non-negative finite number");
  if (cg_max_iters < 1) return fail(DGB200_E_ARG, "cg_max_iters must be at least 1");
  if (!(cg_tol >= 0.0) || !(cg_tol < INFINITY)) return fail(DGB200_E_ARG, "cg_tol must be a non-negative finite number");
  const cudaStream_t st = (cudaStream_t)stream;
  int sms = 0, per_sm = 0;
  cudaError_t e = cudaSuccess;
  if (const char* m = coop_sms(&sms, &e)) return fail(DGB200_E_CUDA, m, e);
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gp_solve_kernel, kGpSolveThreads, 0));
  if (per_sm < 1) return fail(DGB200_E_CUDA, "gp_solve_kernel does not fit on an SM");
  const int n_ranges = obs > 0 ? blocks((size_t)obs, kGpRange) : 1;
  const size_t no = (size_t)(obs > 0 ? obs : 1), nt = (size_t)n_tracks, nc = (size_t)n_cams;
  GpArgs a;
  a.cams = d_cams; a.pts = d_pts; a.R = d_R; a.K = d_K; a.k_per_camera = k_per_camera; a.n_cams = n_cams;
  a.offsets = d_offsets; a.mask = d_mask; a.n_tracks = n_tracks; a.obs = obs; a.n_ranges = n_ranges;
  a.cg_max_iters = cg_max_iters; a.seed = seed; a.init_scale = init_scale; a.delta = loss_scale;
  a.max_angle = max_angle; a.cg_tol2 = cg_tol * cg_tol;
  auto lay_out = [&](char* base) {
    Carve w{base};
    a.tab = w.take<double>(dg::kTrCamStride * nc);
    a.cen = w.take<double>(6 * nc);
    a.Xb = w.take<double>(6 * nt);
    a.dsc = w.take<double>(2 * no);
    a.ray = w.take<double>(3 * no);
    a.lo = w.take<double>(kLoRows * no);
    a.lc = w.take<double>(kLcRows * no);
    a.trk = w.take<double>(dg::kBaTrkStride * nt);
    a.tv = w.take<double>(kGvStride * nt);
    a.y = w.take<double>(3 * nt);
    a.rec = w.take<double>(kGcStride * nc);
    a.part = w.take<double>(kPcgParts * nc);
    a.state = w.take<BaState>(1);
    a.cg_iters = w.take<int>(1);
    a.linbad = w.take<int>(1);
    a.parent = w.take<int>(nc);
    a.active = w.take<int>(nc);
    a.key = w.take<int>(no);
    a.track_of = w.take<int>(no);
    a.pos_of = w.take<int>(no);
    a.ctrk = w.take<int>(no);
    a.hist = w.take<int>(nc * (size_t)n_ranges);
    a.list_off = w.take<int>(nc + 1);
    a.trk_used = w.take<int>(nt);
    a.used = w.take<unsigned char>(no);
    return w.bytes;
  };
  char* ws = nullptr;
  const size_t bytes = lay_out(nullptr);
  CU(cudaMallocAsync((void**)&ws, bytes, st));
  lay_out(ws);
  a.t_out = d_t_out; a.X_out = d_X_out; a.comp_out = d_component_out; a.angle_out = d_angle_out;
  a.inl_out = d_inliers_out; a.cost0_out = d_cost0_out; a.cost_out = d_cost_out; a.iters_out = d_iters_out;
  a.n_used_out = d_n_used_out; a.cg_iters_out = d_cg_iters_out;
  const int cam_grid = blocks(nc, kGpThreads), cam_warp_grid = blocks(nc, kGpWarps);
  const int trk_grid = blocks(nt, kGpWarps), trk_thread_grid = blocks(nt, kGpThreads);
  const int obs_grid = blocks(no, kGpThreads), range_grid = blocks((size_t)n_ranges, kGpWarps);
  void* solve_args[] = {&a};
  cudaError_t launch = cudaSuccess;
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.used, 0, no, st));              // rows outside every span are not used
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.track_of, 0xff, sizeof(int) * no, st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.list_off, 0, sizeof(int) * (nc + 1), st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.hist, 0, sizeof(int) * nc * (size_t)n_ranges, st));
  ADJ_LAUNCH((gp_cameras_kernel<<<cam_grid, kGpThreads, 0, st>>>(a)));
  ADJ_LAUNCH((gp_mark_kernel<<<trk_grid, 32 * kGpWarps, 0, st>>>(a)));
  ADJ_LAUNCH((gp_compress_kernel<<<cam_grid, kGpThreads, 0, st>>>(a)));
  if (obs > 0) {
    ADJ_LAUNCH((gp_key_kernel<<<obs_grid, kGpThreads, 0, st>>>(a)));
    ADJ_LAUNCH((gp_count_kernel<<<range_grid, 32 * kGpWarps, 0, st>>>(a)));
    ADJ_LAUNCH((gp_scan_kernel<<<1, kBaCta, 0, st>>>(a)));
    ADJ_LAUNCH((gp_scatter_kernel<<<range_grid, 32 * kGpWarps, 0, st>>>(a)));
  }
  ADJ_LAUNCH((gp_start_views_kernel<<<cam_grid, kGpThreads, 0, st>>>(a)));
  ADJ_LAUNCH((gp_start_tracks_kernel<<<trk_grid, 32 * kGpWarps, 0, st>>>(a)));
  ADJ_LAUNCH((gp_init_kernel<<<1, kBaCta, 0, st>>>(a)));
  for (int it = 0; it < max_iters && launch == cudaSuccess; ++it) {
    ADJ_LAUNCH((gp_linearise_kernel<<<trk_grid, 32 * kGpWarps, 0, st>>>(a)));
    ADJ_LAUNCH((gp_points_kernel<<<trk_thread_grid, kGpThreads, 0, st>>>(a)));
    ADJ_LAUNCH((gp_precond_kernel<<<cam_warp_grid, 32 * kGpWarps, 0, st>>>(a)));
    ADJ_LAUNCH(launch = cudaLaunchCooperativeKernel((const void*)gp_solve_kernel, per_sm * sms, kGpSolveThreads,
                                                    solve_args, 0, st));
    ADJ_LAUNCH((gp_backsub_kernel<<<trk_grid, 32 * kGpWarps, 0, st>>>(a)));
    ADJ_LAUNCH((gp_decide_kernel<<<1, kBaCta, 0, st>>>(a)));
  }
  ADJ_LAUNCH((gp_finish_views_kernel<<<cam_grid, kGpThreads, 0, st>>>(a)));
  ADJ_LAUNCH((gp_finish_tracks_kernel<<<trk_thread_grid, kGpThreads, 0, st>>>(a)));
  if (obs > 0) ADJ_LAUNCH((gp_finish_obs_kernel<<<obs_grid, kGpThreads, 0, st>>>(a)));
  CU(cudaFreeAsync(ws, st));
  CU(launch);
  return 0;
}

}  // extern "C"
