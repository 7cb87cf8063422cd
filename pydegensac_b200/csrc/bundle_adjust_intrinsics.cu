// bundle_adjust_intrinsics.cu -- bundle adjustment that also refines the intrinsics, device resident: the inexact
// Levenberg-Marquardt of bundle_adjust_pcg.cu over the free cameras' poses and the free intrinsics groups' RADIAL
// parameters (camera_radial.h), and the undistortion of pixels through those intrinsics.  A translation unit of its own,
// so that adding it changes no instruction of the other sources' kernels.
//
// The reduced system is over [free poses; free groups' intrinsics].  Each group slot has 5 coordinates; those the call
// does not refine, and every coordinate of a group without a used observation, are pinned (identity row and column,
// zero right-hand side), as the pose solver pins its held coordinate.  U is no longer block-diagonal: camera a of group
// g adds E_a = sum_{i in a} w J_pose,i^T J_intr,i.  S p = U* p - sum_p W_p V*_p^-1 W_p^T p stays matrix-free, and the
// E_a products are formed per observation from the stored Jacobians, so E_a is never stored.
//
// Once per call:
//   bai_cameras_kernel   the camera table (pinhole K of the camera's group; a camera of an invalid group is not
//                        registered) and both pose buffers;
//   bai_slots_kernel     the maps from camera to free slot and from group to free group slot, both intrinsics buffers;
//   bai_mark_kernel      one warp per track: ba_mark_track with the RADIAL model;
//   bai_slot_obs_kernel  the free slot and the free group slot of each used observation (-1: none);
//   bai_hist/scan/scatter_kernel, twice: the camera-major and the group-major lists of the used observations
//                        (ba_sort_*, bundle_adjust_device.h);
//   bai_chunks_kernel    one thread: the fixed partition of each group's list into chunks of kBaiChunk observations;
//   bai_init_kernel      one CTA: cost0, n_used, the scale gauge's axis, the LM state (ba_init_state).
// Per trial step (8 launches; each returns at once when the state says the call stopped):
//   bai_linearise_kernel one warp per track, after an accepted step: V_p, g_p; W_pose, W_intr by observation and the
//                        Jacobians, residuals and weights in camera-major and group-major order;
//   bai_points_kernel    one thread per track: V*_p^-1;
//   bai_precond_kernel   one warp per free slot: U_a, g_a, M_a = U*_a - sum W V*^-1 W^T, its Cholesky factor, b_a;
//   bai_gchunk_kernel    one warp per chunk: the chunk's partial sums of U_g, g_g, sum W_intr V*^-1 W_intr^T and
//                        sum W_intr V*^-1 g_p;
//   bai_group_kernel     one warp per free group: the fixed-order sum of its chunks' partials, M_g, its Cholesky
//                        factor and b_g (Ceres' SCHUR_JACOBI: the cross blocks are left out of the preconditioner);
//   bai_solve_kernel     the whole PCG loop in one cooperative launch, then the trial poses and intrinsics;
//   bai_backsub_kernel   one warp per track: the trial point and its cost (+inf when a group's trial f <= 0);
//   bai_decide_kernel    one CTA: ba_decide_step.
// After the last step bai_finish_*_kernel write the outputs and the inlier mask at the refined intrinsics.
//
// One PCG iteration (three grid.sync), each phase a grid-stride loop over a fixed partition of the work:
//   A  one thread per track: y_p = V*_p^-1 sum_i (W_pose,i^T p_cam(i) + W_intr,i^T p_grp(i));
//   B  one warp per free slot: q_a = U*_a p_a + E_a p_g(a) - sum W_pose,i y; and one warp per chunk of a group's
//      list: its share of E_a^T p_a - W_intr,i y (the group's first chunk also adds U*_g p_g), and of p . q;
//   C  one thread per free slot, one warp per free group (q_g = its chunks' shares in a fixed order): x += alpha p,
//      r -= alpha q, z = M^-1 r.
// The loop is pcg_run (pcg_device.h).  The dot products are sums of per-slot, per-group and per-chunk terms that every
// CTA sums itself in one fixed order, so nothing depends on the grid and there are no floating-point atomics: a rerun
// gives the same bytes.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/degensac_b200.h"
#include "entry_error.h"
#include "bundle_adjust_args.h"
#include "common.h"
#include "absolute_pose.h"
#include "pose_refine.h"
#include "triangulate.h"
#include "bundle_adjust.h"
#include "camera_radial.h"
#include "device_util.h"
#include "bundle_adjust_device.h"
#include "pcg_device.h"
#include "adjust_host.h"

namespace cg = cooperative_groups;

namespace {

thread_local char g_err[256] = "";
thread_local char g_err_ud[256] = "";
int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err, code, what, e); }
int fail_ud(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err_ud, code, what, e); }

constexpr int kBaiWarps = 4;                      // tracks, slots or chunks per CTA, one per warp
constexpr int kBaiThreads = 32 * kBaiWarps;
constexpr int kBaiCamThreads = 128;
constexpr int kBaiSolveThreads = 256;             // the cooperative kernel
constexpr int kBaiRange = 4096;                   // observations per warp of the counting sorts
constexpr int kBaiChunk = 256;                    // observations per chunk of a group's list
constexpr int kNK = dg::kRadParams;               // 5
constexpr int kNK2 = kNK * (kNK + 1) / 2;         // 15

// Per observation, by observation: W_pose [6][3] (kWp), W_intr [5][3] (kWk).  Camera-major: W_pose (18), J_cam (12),
// r (2), w, J_intr (10) = 43 (kCm*).  Group-major: W_intr (15), J_intr (10), J_cam (12), r (2), w = 40 (kGm*).
constexpr int kWp = 18, kWk = 15;
constexpr int kCmW = 0, kCmJc = 18, kCmR = 30, kCmWt = 32, kCmJk = 33, kCm = 43;
constexpr int kGmW = 0, kGmJk = 15, kGmJc = 25, kGmR = 37, kGmWt = 39, kGm = 40;

// A free slot's record: U (21), g_c (6), L (21), then its PCG vectors (pcg_device.h): b, x, r, z (6 each), p in two
// buffers (12), q (6)
constexpr int kPcU = 0, kPcG = 21, kPcL = 27, kPcB = 48, kPcX = 54, kPcP = 72, kPcQ = 84, kPcStride = 90;
// A free group's record: U (15), g (5), L (15), then b, x, r, z (5 each), p in two buffers (10); no q, which its chunks
// hold
constexpr int kGrU = 0, kGrG = 15, kGrL = 20, kGrB = 35, kGrX = 40, kGrP = 55, kGrStride = 65;
// A chunk's partials: U (15), g (5), sum W V*^-1 W^T (15), sum W V*^-1 g_p (5); in the PCG loop its q share (5)
constexpr int kChU = 0, kChG = 15, kChM = 20, kChH = 35, kChStride = 40;
// The terms of the dot products (pcg_device.h): kPcgParts arrays of n_part = n_free + n_gfree + chunk capacity entries

struct BaiArgs {
  const int* cams; const double* pts;                      // [obs], [obs][2]
  const double* R; const double* t;
  const int* groups; const double* intr_in;                // [n_cams], [n_groups][5]
  int n_cams, n_groups;
  const int* offsets; const unsigned char* mask;           // [T+1], [obs] or null
  const double* X;                                         // [T][3]
  int n_tracks, obs, n_free, n_gfree, refine, gauge_slot, held_cam, n_ranges, n_chunks, n_part, cg_max_iters;
  double sig2, th2, cg_tol2;
  const int* free; const int* gfree;                       // [n_free], [n_gfree], on the device
  // workspace
  double* tab;       // [n_cams][kTrCamStride]
  double* poses;     // [2][n_cams][12]: current and trial
  double* intr;      // [2][n_groups][5]: current and trial
  double* Xb;        // [2][T][3]
  double* trk;       // [T][kBaTrkStride]
  double* y;         // [T][3]
  double* Wo;        // [kWp + kWk][obs]: W_pose, W_intr by observation
  double* Cm;        // [kCm][obs]: camera-major
  double* Gm;        // [kGm][obs]: group-major
  double* slot;      // [n_free][kPcStride]
  double* grp;       // [n_gfree][kGrStride]
  double* chk;       // [n_chunks][kChStride]
  double* part;      // [kPcgParts][n_part]
  BaState* state;
  int* cg_iters;     // [1]
  int* slot_of;      // [n_cams]
  int* gslot_of;     // [n_groups]
  int* track_of;     // [obs]
  int* sl; int* gsl; // [obs]: the free slot / free group slot of a used observation, or -1
  int* pos_of; int* gpos_of;   // [obs]: its position in the camera-major / group-major list
  int* ctrk; int* gtrk;        // [obs]: the track of each camera-major / group-major entry
  int* gcs;          // [obs]: the free slot of each group-major entry's camera (-1: held)
  int* hist;         // [max(n_free, n_gfree)][n_ranges]: counts, then cursors
  int* list_off;     // [n_free + 1]
  int* glist_off;    // [n_gfree + 1]
  int* chunk_off;    // [n_gfree + 1]: the chunks of free group q are chunk_off[q] .. chunk_off[q + 1] - 1
  int* chunk_beg;    // [n_chunks]: a chunk's first group-major position (its end: the next chunk's, or the group's)
  int* trk_used;     // [T]
  unsigned char* usable; unsigned char* used;   // [obs]
  // outputs
  double* R_out; double* t_out; double* X_out; double* intr_out; unsigned char* mask_out;
  double* cost0_out; double* cost_out; int* iters_out; int* n_used_out; int* cg_iters_out;
};

__device__ __forceinline__ const double* pose_of(const BaiArgs& a, int buf, int c) {
  return a.poses + 12 * ((size_t)buf * a.n_cams + c);
}
__device__ __forceinline__ double* point_of(const BaiArgs& a, int buf, int j) {
  return a.Xb + 3 * ((size_t)buf * a.n_tracks + j);
}
// The intrinsics of camera c (a usable camera: its group is valid) in buffer buf
__device__ __forceinline__ const double* intr_of(const BaiArgs& a, int buf, int c) {
  return a.intr + kNK * ((size_t)buf * a.n_groups + a.groups[c]);
}
__device__ __forceinline__ double* slot_rec(const BaiArgs& a, int s) { return a.slot + kPcStride * (size_t)s; }
__device__ __forceinline__ double* grp_rec(const BaiArgs& a, int q) { return a.grp + kGrStride * (size_t)q; }
__device__ __forceinline__ double* part_of(const BaiArgs& a, int kind) { return a.part + kind * (size_t)a.n_part; }
// Whether coordinate k of a free group's intrinsics is refined: f (bit 0), cx, cy (bit 1), k1, k2 (bit 2)
__device__ __forceinline__ bool refined(int refine, int k) {
  return (refine >> (k == 0 ? 0 : (k < 3 ? 1 : 2))) & 1;
}
__device__ __forceinline__ int chunk_end(const BaiArgs& a, int q, int c) {
  return c + 1 < a.chunk_off[q + 1] ? a.chunk_beg[c + 1] : a.glist_off[q + 1];
}

// The RADIAL model for the shared marking and output mask
struct BaRadial {
  static __device__ __forceinline__ void point_row(const BaiArgs& a, const double* P, int cm, int buf, const double* X,
                                                   double x, double y, double* r, double* Jx) {
    double Jc[12], Jk[10];
    dg::rad_jacobian(P, intr_of(a, buf, cm), X, x, y, r, Jc, Jx, Jk);
  }
  static __device__ __forceinline__ double sq_error(const BaiArgs& a, const double* P, int cm, int buf, const double* X,
                                                    double x, double y, bool* front) {
    return dg::rad_sq_error(P, intr_of(a, buf, cm), X, x, y, front);
  }
};

// ---------------------------------------------------------------------------------------------- once per call
__global__ void __launch_bounds__(kBaiCamThreads) bai_cameras_kernel(BaiArgs a) {
  const int c = blockIdx.x * kBaiCamThreads + threadIdx.x;
  if (c >= a.n_cams) return;
  const double* R = a.R + 9 * (size_t)c;
  const double* t = a.t + 3 * (size_t)c;
  const int g = a.groups[c];
  const double* k = a.intr_in + kNK * (size_t)(g >= 0 && g < a.n_groups ? g : 0);
  const bool ok = g >= 0 && g < a.n_groups && dg::rad_valid(k);
  const double K[9] = {ok ? k[0] : 1.0, 0.0, ok ? k[1] : 0.0, 0.0, ok ? k[0] : 1.0, ok ? k[2] : 0.0, 0.0, 0.0, 1.0};
  double* tab = a.tab + dg::kTrCamStride * (size_t)c;
  dg::tr_camera(R, t, K, tab);
  if (!ok) tab[dg::kTrCamOk] = 0.0;                    // an invalid group: the camera is not registered
  for (int buf = 0; buf < 2; ++buf) {
    double* P = a.poses + 12 * ((size_t)buf * a.n_cams + c);
    for (int i = 0; i < 9; ++i) P[i] = R[i];
    for (int i = 0; i < 3; ++i) P[9 + i] = t[i];
  }
}

__global__ void __launch_bounds__(kBaiCamThreads) bai_slots_kernel(BaiArgs a) {
  const int q = blockIdx.x * kBaiCamThreads + threadIdx.x;
  if (q < a.n_free) a.slot_of[a.free[q]] = q;
  if (q < a.n_gfree) a.gslot_of[a.gfree[q]] = q;
  if (q < a.n_groups)
    for (int buf = 0; buf < 2; ++buf)
      for (int i = 0; i < kNK; ++i) a.intr[kNK * ((size_t)buf * a.n_groups + q) + i] = a.intr_in[kNK * (size_t)q + i];
}

__global__ void __launch_bounds__(kBaiThreads) bai_mark_kernel(BaiArgs a) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kBaiWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks) return;                       // (warp-uniform)
  ba_mark_track<BaiArgs, BaRadial>(a, j, lane);
}

__global__ void __launch_bounds__(kBaiCamThreads) bai_slot_obs_kernel(BaiArgs a) {
  const int r = blockIdx.x * kBaiCamThreads + threadIdx.x;
  if (r >= a.obs) return;
  const bool u = a.used[r];                            // (a used observation's camera and group are valid)
  a.sl[r] = u ? a.slot_of[a.cams[r]] : -1;
  a.gsl[r] = u ? a.gslot_of[a.groups[a.cams[r]]] : -1;
}

// key: sl (camera-major) or gsl (group-major)
__global__ void __launch_bounds__(kBaiThreads) bai_hist_kernel(BaiArgs a, const int* key) {
  const int lane = threadIdx.x & 31;
  const int w = blockIdx.x * kBaiWarps + (threadIdx.x >> 5);
  if (w >= a.n_ranges) return;                       // (warp-uniform)
  ba_sort_count(key, a.obs, kBaiRange, a.hist, a.n_ranges, w, lane);
}

__global__ void __launch_bounds__(kBaCta) bai_scan_kernel(BaiArgs a, int n_keys, int* list_off) {
  __shared__ int sh[kBaCta];
  ba_sort_scan(a.hist, n_keys, a.n_ranges, list_off, sh);
}

__global__ void __launch_bounds__(kBaiThreads) bai_scatter_kernel(BaiArgs a, const int* key, int* pos_of, int* item) {
  const int lane = threadIdx.x & 31;
  const int w = blockIdx.x * kBaiWarps + (threadIdx.x >> 5);
  if (w >= a.n_ranges) return;                       // (warp-uniform)
  ba_sort_scatter(key, a.obs, kBaiRange, a.hist, a.n_ranges, a.track_of, pos_of, item, w, lane);
}

// One thread: chunk_off and chunk_beg; and the camera slot of each group-major entry (all threads)
__global__ void __launch_bounds__(kBaiCamThreads) bai_chunks_kernel(BaiArgs a) {
  const int r = blockIdx.x * kBaiCamThreads + threadIdx.x;
  if (r < a.obs && a.gsl[r] >= 0) a.gcs[a.gpos_of[r]] = a.sl[r];
  if (r != 0) return;
  int c = 0;
  for (int q = 0; q < a.n_gfree; ++q) {
    a.chunk_off[q] = c;
    for (int i = a.glist_off[q]; i < a.glist_off[q + 1]; i += kBaiChunk) a.chunk_beg[c++] = i;
  }
  a.chunk_off[a.n_gfree] = c;
}

__global__ void __launch_bounds__(kBaCta) bai_init_kernel(BaiArgs a) {
  ba_init_state(a);
  if (threadIdx.x == 0) a.cg_iters[0] = 0;
}

// ---------------------------------------------------------------------------------------------- one trial step
__global__ void __launch_bounds__(kBaiThreads) bai_linearise_kernel(BaiArgs a) {
  const BaState* st = a.state;
  if (st->stop || !st->lin) return;
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kBaiWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks || a.trk_used[j] == 0) return;   // (warp-uniform)
  const int cur = st->cur;
  const double* X = point_of(a, cur, j);
  const int b = a.offsets[j], e = a.offsets[j + 1];
  const size_t no = (size_t)a.obs;
  double V[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
  for (int r = b + lane; r < e; r += 32) {
    if (!a.used[r]) continue;
    const int cm = a.cams[r];
    double rr[2], Jc[12], Jx[6], Jk[10];
    dg::rad_jacobian(pose_of(a, cur, cm), intr_of(a, cur, cm), X, a.pts[2 * (size_t)r], a.pts[2 * (size_t)r + 1], rr,
                     Jc, Jx, Jk);
    const double w = dg::ba_weight(rr[0] * rr[0] + rr[1] * rr[1], a.sig2);
    dg::ba_point_terms(Jx, rr, w, V, g);
    if (a.sl[r] >= 0) {
      double W[kWp];
      dg::ba_cross_block(Jc, Jx, w, W);
      double* C = a.Cm + (size_t)a.pos_of[r];
#pragma unroll
      for (int k = 0; k < kWp; ++k) {
        a.Wo[k * no + r] = W[k];
        C[(kCmW + k) * no] = W[k];
      }
#pragma unroll
      for (int k = 0; k < 12; ++k) C[(kCmJc + k) * no] = Jc[k];
      C[kCmR * no] = rr[0];
      C[(kCmR + 1) * no] = rr[1];
      C[kCmWt * no] = w;
#pragma unroll
      for (int k = 0; k < 10; ++k) C[(kCmJk + k) * no] = Jk[k];
    }
    if (a.gsl[r] >= 0) {
      double* G = a.Gm + (size_t)a.gpos_of[r];
#pragma unroll
      for (int k = 0; k < kNK; ++k)
#pragma unroll
        for (int m = 0; m < 3; ++m) {
          const double v = w * (Jk[k] * Jx[m] + Jk[5 + k] * Jx[3 + m]);
          a.Wo[(kWp + 3 * k + m) * no + r] = v;
          G[(kGmW + 3 * k + m) * no] = v;
        }
#pragma unroll
      for (int k = 0; k < 10; ++k) G[(kGmJk + k) * no] = Jk[k];
#pragma unroll
      for (int k = 0; k < 12; ++k) G[(kGmJc + k) * no] = Jc[k];
      G[kGmR * no] = rr[0];
      G[(kGmR + 1) * no] = rr[1];
      G[kGmWt * no] = w;
    }
  }
#pragma unroll
  for (int s = 0; s < 6; ++s) V[s] = warp_sum(V[s]);
#pragma unroll
  for (int s = 0; s < 3; ++s) g[s] = warp_sum(g[s]);
  if (lane == 0) {
    double* tk = a.trk + dg::kBaTrkStride * (size_t)j;
#pragma unroll
    for (int s = 0; s < 6; ++s) tk[dg::kBaTrkV + s] = V[s];
#pragma unroll
    for (int s = 0; s < 3; ++s) tk[dg::kBaTrkG + s] = g[s];
  }
}

__global__ void __launch_bounds__(kBaiThreads) bai_points_kernel(BaiArgs a) {
  BaState* st = a.state;
  if (st->stop) return;
  const int j = blockIdx.x * kBaiThreads + threadIdx.x;
  if (j >= a.n_tracks || a.trk_used[j] == 0) return;
  double* tk = a.trk + dg::kBaTrkStride * (size_t)j;
  double Vi[6];
  if (!dg::ba_inv3(tk + dg::kBaTrkV, st->lam, Vi)) {
    st->bad = 1;                                       // the step is rejected
    return;
  }
#pragma unroll
  for (int s = 0; s < 6; ++s) tk[dg::kBaTrkVi + s] = Vi[s];
}

// One warp per free slot: the pose block of bundle_adjust_pcg.cu's pcg_precond_kernel, over this unit's camera-major
// layout (the held coordinate and inactive slots pinned), and the start of PCG
__global__ void __launch_bounds__(kBaiThreads) bai_precond_kernel(BaiArgs a) {
  BaState* st = a.state;
  if (st->stop || st->bad) return;
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x * kBaiWarps + (threadIdx.x >> 5);
  if (s >= a.n_free) return;                           // (warp-uniform)
  const size_t no = (size_t)a.obs;
  double U[21], gc[6], Mw[21], h[6];
#pragma unroll
  for (int m = 0; m < 21; ++m) { U[m] = 0.0; Mw[m] = 0.0; }
#pragma unroll
  for (int k = 0; k < 6; ++k) { gc[k] = 0.0; h[k] = 0.0; }
  const int i0 = a.list_off[s], i1 = a.list_off[s + 1];
  for (int i = i0 + lane; i < i1; i += 32) {
    const double* C = a.Cm + i;
    double Jc[12], W[kWp], Y[kWp];
#pragma unroll
    for (int k = 0; k < 12; ++k) Jc[k] = C[(kCmJc + k) * no];
    const double e0 = C[kCmR * no], e1 = C[(kCmR + 1) * no], w = C[kCmWt * no];
#pragma unroll
    for (int k = 0; k < kWp; ++k) W[k] = C[(kCmW + k) * no];
    const double* tk = a.trk + dg::kBaTrkStride * (size_t)a.ctrk[i];
    dg::ba_schur_row(W, tk + dg::kBaTrkVi, Y);
    const double* gp = tk + dg::kBaTrkG;
    int m = 0;
#pragma unroll
    for (int k = 0; k < 6; ++k)
#pragma unroll
      for (int l = k; l < 6; ++l, ++m) {
        U[m] += w * (Jc[k] * Jc[l] + Jc[6 + k] * Jc[6 + l]);
        Mw[m] += Y[3 * k] * W[3 * l] + Y[3 * k + 1] * W[3 * l + 1] + Y[3 * k + 2] * W[3 * l + 2];
      }
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      gc[k] += w * (Jc[k] * e0 + Jc[6 + k] * e1);
      h[k] += Y[3 * k] * gp[0] + Y[3 * k + 1] * gp[1] + Y[3 * k + 2] * gp[2];
    }
  }
#pragma unroll
  for (int m = 0; m < 21; ++m) { U[m] = warp_sum(U[m]); Mw[m] = warp_sum(Mw[m]); }
#pragma unroll
  for (int k = 0; k < 6; ++k) { gc[k] = warp_sum(gc[k]); h[k] = warp_sum(h[k]); }
  if (lane != 0) return;
  const int hold = st->hold_row - dg::kBaCamParams * s;
  const bool active = i1 > i0;
  const double lam = st->lam;
  double M[21], b[6];
  int m = 0;
#pragma unroll
  for (int k = 0; k < 6; ++k)
#pragma unroll
    for (int l = k; l < 6; ++l, ++m) {
      double v = (k == l ? U[m] + lam * U[m] : U[m]) - Mw[m];
      if (!active || k == hold || l == hold) v = k == l ? 1.0 : 0.0;
      M[m] = v;
    }
#pragma unroll
  for (int k = 0; k < 6; ++k) b[k] = (!active || k == hold) ? 0.0 : -(gc[k] - h[k]);
  double* rec = slot_rec(a, s);
  if (!dg::pr_cholesky_factor<6>(M, rec + kPcL)) {
    st->bad = 1;                                       // the step is rejected
    return;
  }
  double z[6];
  dg::pr_cholesky_apply<6>(rec + kPcL, b, z);
  pcg_start<6>(rec + kPcB, b, z, a.part, a.n_part, s);
#pragma unroll
  for (int k = 0; k < 6; ++k) rec[kPcG + k] = gc[k];
#pragma unroll
  for (int q = 0; q < 21; ++q) rec[kPcU + q] = active ? U[q] : 0.0;
}

// One warp per chunk of a free group's group-major list: the chunk's partial sums (a fixed tree over the lanes)
__global__ void __launch_bounds__(kBaiThreads) bai_gchunk_kernel(BaiArgs a) {
  const BaState* st = a.state;
  if (st->stop || st->bad) return;
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kBaiWarps + (threadIdx.x >> 5);
  if (c >= a.n_chunks) return;                         // (warp-uniform)
  const int i0 = a.chunk_beg[c];
  // the chunk's group: the last q with chunk_off[q] <= c (chunks past the last one are empty and skipped)
  if (c >= a.chunk_off[a.n_gfree]) return;
  int lo = 0, hi = a.n_gfree - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.chunk_off[mid] <= c) lo = mid; else hi = mid - 1;
  }
  const int i1 = chunk_end(a, lo, c);
  const size_t no = (size_t)a.obs;
  double U[kNK2], Mw[kNK2], gg[kNK], h[kNK];
#pragma unroll
  for (int m = 0; m < kNK2; ++m) { U[m] = 0.0; Mw[m] = 0.0; }
#pragma unroll
  for (int k = 0; k < kNK; ++k) { gg[k] = 0.0; h[k] = 0.0; }
  for (int i = i0 + lane; i < i1; i += 32) {
    const double* G = a.Gm + i;
    double Jk[10], W[kWk], Y[kWk];
#pragma unroll
    for (int k = 0; k < 10; ++k) Jk[k] = G[(kGmJk + k) * no];
    const double e0 = G[kGmR * no], e1 = G[(kGmR + 1) * no], w = G[kGmWt * no];
#pragma unroll
    for (int k = 0; k < kWk; ++k) W[k] = G[(kGmW + k) * no];
    const double* tk = a.trk + dg::kBaTrkStride * (size_t)a.gtrk[i];
#pragma unroll
    for (int k = 0; k < kNK; ++k) dg::ba_sym3_mul(tk + dg::kBaTrkVi, W + 3 * k, Y + 3 * k);
    const double* gp = tk + dg::kBaTrkG;
    int m = 0;
#pragma unroll
    for (int k = 0; k < kNK; ++k)
#pragma unroll
      for (int l = k; l < kNK; ++l, ++m) {
        U[m] += w * (Jk[k] * Jk[l] + Jk[5 + k] * Jk[5 + l]);
        Mw[m] += Y[3 * k] * W[3 * l] + Y[3 * k + 1] * W[3 * l + 1] + Y[3 * k + 2] * W[3 * l + 2];
      }
#pragma unroll
    for (int k = 0; k < kNK; ++k) {
      gg[k] += w * (Jk[k] * e0 + Jk[5 + k] * e1);
      h[k] += Y[3 * k] * gp[0] + Y[3 * k + 1] * gp[1] + Y[3 * k + 2] * gp[2];
    }
  }
#pragma unroll
  for (int m = 0; m < kNK2; ++m) { U[m] = warp_sum(U[m]); Mw[m] = warp_sum(Mw[m]); }
#pragma unroll
  for (int k = 0; k < kNK; ++k) { gg[k] = warp_sum(gg[k]); h[k] = warp_sum(h[k]); }
  if (lane != 0) return;
  double* ch = a.chk + kChStride * (size_t)c;
#pragma unroll
  for (int m = 0; m < kNK2; ++m) { ch[kChU + m] = U[m]; ch[kChM + m] = Mw[m]; }
#pragma unroll
  for (int k = 0; k < kNK; ++k) { ch[kChG + k] = gg[k]; ch[kChH + k] = h[k]; }
}

// One warp per free group: its chunks' partials summed in a fixed order (lane l takes chunks l, l + 32, ..., then a
// fixed tree over the lanes), M_g = U*_g - sum W_intr V*^-1 W_intr^T (pinned rows and columns of the identity), its
// Cholesky factor, b_g and the start of PCG
__global__ void __launch_bounds__(kBaiThreads) bai_group_kernel(BaiArgs a) {
  BaState* st = a.state;
  if (st->stop || st->bad) return;
  const int lane = threadIdx.x & 31;
  const int q = blockIdx.x * kBaiWarps + (threadIdx.x >> 5);
  if (q >= a.n_gfree) return;                          // (warp-uniform)
  double U[kNK2], Mw[kNK2], gg[kNK], h[kNK];
#pragma unroll
  for (int m = 0; m < kNK2; ++m) { U[m] = 0.0; Mw[m] = 0.0; }
#pragma unroll
  for (int k = 0; k < kNK; ++k) { gg[k] = 0.0; h[k] = 0.0; }
  for (int c = a.chunk_off[q] + lane; c < a.chunk_off[q + 1]; c += 32) {
    const double* ch = a.chk + kChStride * (size_t)c;
#pragma unroll
    for (int m = 0; m < kNK2; ++m) { U[m] += ch[kChU + m]; Mw[m] += ch[kChM + m]; }
#pragma unroll
    for (int k = 0; k < kNK; ++k) { gg[k] += ch[kChG + k]; h[k] += ch[kChH + k]; }
  }
#pragma unroll
  for (int m = 0; m < kNK2; ++m) { U[m] = warp_sum(U[m]); Mw[m] = warp_sum(Mw[m]); }
#pragma unroll
  for (int k = 0; k < kNK; ++k) { gg[k] = warp_sum(gg[k]); h[k] = warp_sum(h[k]); }
  if (lane != 0) return;
  const bool active = a.glist_off[q + 1] > a.glist_off[q];
  const double lam = st->lam;
  double M[kNK2], b[kNK];
  int m = 0;
#pragma unroll
  for (int k = 0; k < kNK; ++k)
#pragma unroll
    for (int l = k; l < kNK; ++l, ++m) {
      double v = (k == l ? U[m] + lam * U[m] : U[m]) - Mw[m];
      if (!active || !refined(a.refine, k) || !refined(a.refine, l)) v = k == l ? 1.0 : 0.0;
      M[m] = v;
    }
#pragma unroll
  for (int k = 0; k < kNK; ++k) b[k] = (!active || !refined(a.refine, k)) ? 0.0 : -(gg[k] - h[k]);
  double* rec = grp_rec(a, q);
  if (!dg::pr_cholesky_factor<kNK>(M, rec + kGrL)) {
    st->bad = 1;                                       // the step is rejected
    return;
  }
  double z[kNK];
  dg::pr_cholesky_apply<kNK>(rec + kGrL, b, z);
  pcg_start<kNK>(rec + kGrB, b, z, a.part, a.n_part, a.n_free + q);
#pragma unroll
  for (int k = 0; k < kNK; ++k) rec[kGrG + k] = gg[k];
#pragma unroll
  for (int i = 0; i < kNK2; ++i) rec[kGrU + i] = active ? U[i] : 0.0;
}

// p = z + beta p' of slot s / free group q, p' in buffer `prev`
__device__ __forceinline__ void direction(const BaiArgs& a, int s, int prev, double beta, double* p) {
  pcg_direction<6>(slot_rec(a, s) + kPcB, prev, beta, p);
}
__device__ __forceinline__ void gdirection(const BaiArgs& a, int q, int prev, double beta, double* p) {
  pcg_direction<kNK>(grp_rec(a, q) + kGrB, prev, beta, p);
}

// U* p of a packed upper triangle U [n (n + 1) / 2], damped on the diagonal
template <int N>
__device__ __forceinline__ double damped_row(const double* U, double lam, const double* p, int k) {
  double v = 0.0;
#pragma unroll
  for (int l = 0; l < N; ++l) {
    const int m = k <= l ? k * N - k * (k - 1) / 2 + (l - k) : l * N - l * (l - 1) / 2 + (k - l);
    v += __ldcg(U + m) * p[l];
  }
  const int d = k * N - k * (k - 1) / 2;
  return v + lam * __ldcg(U + d) * p[k];
}

// pcg_run's S p and phase C over [free slots; free groups].  product: A, one thread per track, y_p = V*_p^-1
// sum_i (W_pose,i^T p_s(i) + W_intr,i^T p_g(i)); grid.sync; B, one warp per free slot, then one per chunk.  update:
// one thread per free slot, one warp per free group.
struct BaiSchur {
  const BaiArgs& a;
  int tid, nthr, lane, warp, nwarps;
  double lam;
  int hold_row;

  __device__ __forceinline__ void product(cg::grid_group& grid, int cur, int prev, double beta) const {
    const int nf = a.n_free, ng = a.n_gfree;
    const size_t no = (size_t)a.obs;
    for (int j = tid; j < a.n_tracks; j += nthr) {
      if (a.trk_used[j] == 0) continue;
      const int b = a.offsets[j], e = a.offsets[j + 1];
      double u[3] = {0.0, 0.0, 0.0};
      for (int r = b; r < e; ++r) {
        const int s = a.sl[r], q = a.gsl[r];
        if (s >= 0) {
          double p[6];
          direction(a, s, prev, beta, p);
#pragma unroll
          for (int k = 0; k < 6; ++k)
#pragma unroll
            for (int m = 0; m < 3; ++m) u[m] += __ldg(a.Wo + (3 * k + m) * no + r) * p[k];
        }
        if (q >= 0) {
          double p[kNK];
          gdirection(a, q, prev, beta, p);
#pragma unroll
          for (int k = 0; k < kNK; ++k)
#pragma unroll
            for (int m = 0; m < 3; ++m) u[m] += __ldg(a.Wo + (kWp + 3 * k + m) * no + r) * p[k];
        }
      }
      double yv[3];
      dg::ba_sym3_mul(a.trk + dg::kBaTrkStride * (size_t)j + dg::kBaTrkVi, u, yv);
#pragma unroll
      for (int m = 0; m < 3; ++m) a.y[3 * (size_t)j + m] = yv[m];
    }
    grid.sync();
    for (int v = warp; v < nf + a.n_chunks; v += nwarps) {
      if (v < nf) {
        const int s = v;
        const bool active = a.list_off[s + 1] > a.list_off[s];
        const int gq = active ? a.gslot_of[a.groups[a.free[s]]] : -1;   // (an active slot's group is valid)
        double pg[kNK] = {0.0, 0.0, 0.0, 0.0, 0.0};
        if (gq >= 0) gdirection(a, gq, prev, beta, pg);
        double acc[6] = {0, 0, 0, 0, 0, 0};
        const int i0 = a.list_off[s], i1 = a.list_off[s + 1];
        for (int i = i0 + lane; i < i1; i += 32) {
          const double* C = a.Cm + i;
          const double* yp = a.y + 3 * (size_t)a.ctrk[i];
          const double y0 = __ldcg(yp), y1 = __ldcg(yp + 1), y2 = __ldcg(yp + 2);
          // E_a p_g: w J_cam^T (J_intr p_g)
          double e0 = 0.0, e1 = 0.0;
          if (gq >= 0) {
#pragma unroll
            for (int k = 0; k < kNK; ++k) {
              e0 += __ldg(C + (kCmJk + k) * no) * pg[k];
              e1 += __ldg(C + (kCmJk + 5 + k) * no) * pg[k];
            }
            const double w = __ldg(C + kCmWt * no);
            e0 *= w;
            e1 *= w;
          }
#pragma unroll
          for (int k = 0; k < 6; ++k)
            acc[k] += __ldg(C + (kCmW + 3 * k) * no) * y0 + __ldg(C + (kCmW + 3 * k + 1) * no) * y1 +
                      __ldg(C + (kCmW + 3 * k + 2) * no) * y2 -
                      (__ldg(C + (kCmJc + k) * no) * e0 + __ldg(C + (kCmJc + 6 + k) * no) * e1);
        }
#pragma unroll
        for (int k = 0; k < 6; ++k) acc[k] = warp_sum(acc[k]);
        if (lane == 0) {
          double p[6];
          direction(a, s, prev, beta, p);
          double* rec = slot_rec(a, s);
          const int hold = hold_row - dg::kBaCamParams * s;
          double pq = 0.0;
#pragma unroll
          for (int k = 0; k < 6; ++k) {
            double q = damped_row<6>(rec + kPcU, lam, p, k) - acc[k];
            if (k == hold) q = p[k];
            rec[kPcQ + k] = q;
            rec[kPcP + 6 * cur + k] = p[k];
            pq += p[k] * q;
          }
          part_of(a, kPartPQ)[s] = pq;
        }
      } else {
        const int c = v - nf;
        if (c >= a.chunk_off[ng]) continue;          // past the last chunk (warp-uniform)
        int lo = 0, hi = ng - 1;
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (a.chunk_off[mid] <= c) lo = mid; else hi = mid - 1;
        }
        const int q = lo, i0 = a.chunk_beg[c], i1 = chunk_end(a, q, c);
        double pg[kNK];
        gdirection(a, q, prev, beta, pg);
        double acc[kNK] = {0.0, 0.0, 0.0, 0.0, 0.0};
        for (int i = i0 + lane; i < i1; i += 32) {
          const double* G = a.Gm + i;
          const double* yp = a.y + 3 * (size_t)a.gtrk[i];
          const double y0 = __ldcg(yp), y1 = __ldcg(yp + 1), y2 = __ldcg(yp + 2);
          const int s = a.gcs[i];
          double e0 = 0.0, e1 = 0.0;
          if (s >= 0) {                              // E_a^T p_a: w J_intr^T (J_cam p_a)
            double p[6];
            direction(a, s, prev, beta, p);
#pragma unroll
            for (int k = 0; k < 6; ++k) {
              e0 += __ldg(G + (kGmJc + k) * no) * p[k];
              e1 += __ldg(G + (kGmJc + 6 + k) * no) * p[k];
            }
            const double w = __ldg(G + kGmWt * no);
            e0 *= w;
            e1 *= w;
          }
#pragma unroll
          for (int k = 0; k < kNK; ++k)
            acc[k] += __ldg(G + (kGmJk + k) * no) * e0 + __ldg(G + (kGmJk + 5 + k) * no) * e1 -
                      (__ldg(G + (kGmW + 3 * k) * no) * y0 + __ldg(G + (kGmW + 3 * k + 1) * no) * y1 +
                       __ldg(G + (kGmW + 3 * k + 2) * no) * y2);
        }
#pragma unroll
        for (int k = 0; k < kNK; ++k) acc[k] = warp_sum(acc[k]);
        if (lane == 0) {
          const double* rec = grp_rec(a, q);
          const bool first = c == a.chunk_off[q];
          double* ch = a.chk + kChStride * (size_t)c;
          double pq = 0.0;
#pragma unroll
          for (int k = 0; k < kNK; ++k) {
            double v = acc[k] + (first ? damped_row<kNK>(rec + kGrU, lam, pg, k) : 0.0);
            if (!refined(a.refine, k)) v = 0.0;      // (p_g is 0 there: q_g = p_g)
            ch[k] = v;
            pq += pg[k] * v;
          }
          part_of(a, kPartPQ)[nf + ng + c] = pq;
        }
      }
    }
  }

  __device__ __forceinline__ void update(int cur, int prev, double beta, double alpha) const {
    const int nf = a.n_free, ng = a.n_gfree;
    for (int v = tid; v < nf; v += nthr) {
      double* rec = slot_rec(a, v);
      double p[6], q[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        p[k] = __ldcg(rec + kPcP + 6 * cur + k);
        q[k] = __ldcg(rec + kPcQ + k);
      }
      const double2 rz = pcg_update<6>(rec + kPcB, p, q, alpha, [rec](const double* r, double* z) {
        dg::pr_cholesky_apply<6>(rec + kPcL, r, z);
      });
      part_of(a, kPartRR)[v] = rz.x;
      part_of(a, kPartRZ)[v] = rz.y;
    }
    // one warp per free group: q_g = its chunks' shares summed in a fixed order (lane l takes chunks l, l + 32, ...,
    // then a fixed tree), then x, r, z as for a slot
    for (int q = warp; q < ng; q += nwarps) {
      double qv[kNK] = {0.0, 0.0, 0.0, 0.0, 0.0};
      for (int c = a.chunk_off[q] + lane; c < a.chunk_off[q + 1]; c += 32)
#pragma unroll
        for (int k = 0; k < kNK; ++k) qv[k] += __ldcg(a.chk + kChStride * (size_t)c + k);
#pragma unroll
      for (int k = 0; k < kNK; ++k) qv[k] = warp_sum(qv[k]);
      if (lane == 0) {
        double* rec = grp_rec(a, q);
        double p[kNK];
        gdirection(a, q, prev, beta, p);
#pragma unroll
        for (int k = 0; k < kNK; ++k) rec[kGrP + kNK * cur + k] = p[k];
        const double2 rz = pcg_update<kNK>(rec + kGrB, p, qv, alpha, [rec](const double* r, double* z) {
          dg::pr_cholesky_apply<kNK>(rec + kGrL, r, z);
        });
        part_of(a, kPartRR)[nf + q] = rz.x;
        part_of(a, kPartRZ)[nf + q] = rz.y;
      }
    }
  }
};

// The PCG loop of one trial step (pcg_run), then the trial poses and intrinsics
__global__ void __launch_bounds__(kBaiSolveThreads) bai_solve_kernel(BaiArgs a) {
  __shared__ double sh[2 * kBaiSolveThreads];
  BaState* st = a.state;
  if (st->stop || st->bad) return;                     // (grid-uniform: nothing below writes them before a grid.sync)
  cg::grid_group grid = cg::this_grid();
  const int tid = blockIdx.x * kBaiSolveThreads + threadIdx.x, nthr = gridDim.x * kBaiSolveThreads;
  const int nf = a.n_free, ng = a.n_gfree;
  const BaiSchur op{a, tid, nthr, (int)threadIdx.x & 31, tid >> 5, nthr >> 5, st->lam, st->hold_row};
  const PcgResult res = pcg_run<kBaiSolveThreads>(grid, a.part, a.n_part, a.cg_tol2, a.cg_max_iters, sh, op);
  // the trial poses and intrinsics (x was last written in a phase C that a grid.sync has closed)
  const int cur = st->cur;
  if (!res.reject)
    for (int v = tid; v < nf + ng; v += nthr) {
      if (v < nf) {
        if (a.list_off[v + 1] == a.list_off[v]) continue;
        const int c = a.free[v];
        double P2[12];
        dg::ap_step(pose_of(a, cur, c), slot_rec(a, v) + kPcX, P2);
        if (dg::pr_ortho_drift(P2) > dg::kPrOrthoTol) dg::pr_orthonormalise(P2);
        double* out = a.poses + 12 * ((size_t)(1 - cur) * a.n_cams + c);
        for (int i = 0; i < 12; ++i) out[i] = P2[i];
      } else {
        const int q = v - nf;
        if (a.glist_off[q + 1] == a.glist_off[q]) continue;
        const int g = a.gfree[q];
        const double* k0 = a.intr + kNK * ((size_t)cur * a.n_groups + g);
        double* k1 = a.intr + kNK * ((size_t)(1 - cur) * a.n_groups + g);
        const double* x = grp_rec(a, q) + kGrX;
        for (int i = 0; i < kNK; ++i) k1[i] = k0[i] + __ldcg(x + i);
      }
    }
  if (tid == 0) {
    a.cg_iters[0] += res.iters;
    if (res.reject) st->bad = 1;
  }
}

__global__ void __launch_bounds__(kBaiThreads) bai_backsub_kernel(BaiArgs a) {
  const BaState* st = a.state;
  if (st->stop || st->bad) return;
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kBaiWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks || a.trk_used[j] == 0) return;   // (warp-uniform)
  const int cur = st->cur, b = a.offsets[j], e = a.offsets[j + 1];
  const size_t no = (size_t)a.obs;
  double acc[3] = {0.0, 0.0, 0.0};
  for (int r = b + lane; r < e; r += 32) {
    const int s = a.sl[r], q = a.gsl[r];
    if (s >= 0) {
      const double* d = slot_rec(a, s) + kPcX;
#pragma unroll
      for (int m = 0; m < 3; ++m)
#pragma unroll
        for (int k = 0; k < 6; ++k) acc[m] += a.Wo[(3 * k + m) * no + r] * d[k];
    }
    if (q >= 0) {
      const double* d = grp_rec(a, q) + kGrX;
#pragma unroll
      for (int m = 0; m < 3; ++m)
#pragma unroll
        for (int k = 0; k < kNK; ++k) acc[m] += a.Wo[(kWp + 3 * k + m) * no + r] * d[k];
    }
  }
#pragma unroll
  for (int m = 0; m < 3; ++m) acc[m] = warp_sum(acc[m]);
  const double* tk = a.trk + dg::kBaTrkStride * (size_t)j;
  const double v[3] = {tk[dg::kBaTrkG] + acc[0], tk[dg::kBaTrkG + 1] + acc[1], tk[dg::kBaTrkG + 2] + acc[2]};
  double D[3];
  dg::ba_sym3_mul(tk + dg::kBaTrkVi, v, D);
  const double* X0 = point_of(a, cur, j);
  const double X[3] = {X0[0] - D[0], X0[1] - D[1], X0[2] - D[2]};
  if (lane < 3) point_of(a, 1 - cur, j)[lane] = X[lane];
  double c = 0.0;
  for (int r = b + lane; r < e; r += 32) {
    if (!a.used[r]) continue;
    const int cm = a.cams[r];
    const double* k = intr_of(a, 1 - cur, cm);
    bool front;
    const double e2 = dg::rad_sq_error(pose_of(a, 1 - cur, cm), k, X, a.pts[2 * (size_t)r], a.pts[2 * (size_t)r + 1],
                                       &front);
    c += front && k[0] > 0.0 ? dg::ba_rho(e2, a.sig2) : INFINITY;
  }
  c = warp_sum(c);
  if (lane == 0) a.trk[dg::kBaTrkStride * (size_t)j + dg::kBaTrkCost] = c;
}

__global__ void __launch_bounds__(kBaCta) bai_decide_kernel(BaiArgs a) {
  __shared__ double shd[kBaCta];
  if (a.state->stop) return;                           // (block-uniform)
  ba_decide_step(a, shd);
}

// ---------------------------------------------------------------------------------------------- outputs
__global__ void __launch_bounds__(kBaiCamThreads) bai_finish_cameras_kernel(BaiArgs a) {
  const int c = blockIdx.x * kBaiCamThreads + threadIdx.x;
  if (c == 0) a.cg_iters_out[0] = a.cg_iters[0];
  if (c < a.n_groups) {
    const double* k = a.intr + kNK * ((size_t)a.state->cur * a.n_groups + c);
    for (int i = 0; i < kNK; ++i) a.intr_out[kNK * (size_t)c + i] = k[i];
  }
  ba_finish_camera(a, c);
}

__global__ void __launch_bounds__(kBaiThreads) bai_finish_tracks_kernel(BaiArgs a) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kBaiWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks) return;
  ba_finish_track<BaiArgs, BaRadial>(a, j, lane);
}

// ---------------------------------------------------------------------------------------------- undistortion
__global__ void __launch_bounds__(kBaiCamThreads) undistort_kernel(const double* pts, const int* cams, int rows,
                                                                    const int* groups, int n_cams,
                                                                    const double* intr, int n_groups, double* out) {
  const int r = blockIdx.x * kBaiCamThreads + threadIdx.x;
  if (r >= rows) return;
  const int c = cams[r];
  const int g = c >= 0 && c < n_cams ? groups[c] : -1;
  double o[2] = {NAN, NAN};
  if (g >= 0 && g < n_groups) dg::rad_undistort(intr + kNK * (size_t)g, pts[2 * (size_t)r], pts[2 * (size_t)r + 1], o);
  out[2 * (size_t)r] = o[0];
  out[2 * (size_t)r + 1] = o[1];
}

}  // namespace

extern "C" {

const char* dgb200_bundle_adjust_intrinsics_last_error(void) { return g_err; }
const char* dgb200_undistort_last_error(void) { return g_err_ud; }

int dgb200_bundle_adjust_intrinsics_ragged_dev(
    const int32_t* d_cams, const double* d_pts, const double* d_R, const double* d_t, const int32_t* d_groups,
    const double* d_intrinsics, int n_groups, int n_cams, const int32_t* d_offsets, int n_tracks, int obs,
    const double* d_X, const uint8_t* d_mask, const int32_t* h_free, int n_free, const int32_t* h_free_groups,
    int n_free_groups, int refine, int scale_gauge, double loss_scale, int max_iters, double px_th, int cg_max_iters,
    double cg_tol, double* d_R_out, double* d_t_out, double* d_X_out, double* d_intrinsics_out, uint8_t* d_mask_out,
    double* d_cost0_out, double* d_cost_out, int32_t* d_iters_out, int32_t* d_n_used_out, int32_t* d_cg_iters_out,
    void* stream) {
  int gauge_slot = -1, held_cam = -1;
  const char* bad = ba_arg_error(!d_R || !d_t || !d_groups || !d_intrinsics || !d_offsets || !d_X || !d_R_out ||
                                     !d_t_out || !d_X_out || !d_intrinsics_out || !d_cost0_out || !d_cost_out ||
                                     !d_iters_out || !d_n_used_out || !d_cg_iters_out,
                                 !d_cams || !d_pts || !d_mask_out, n_tracks, obs, n_cams, h_free, n_free, n_cams,
                                 "n_free must lie in [0, n_cams]", scale_gauge, loss_scale, max_iters, px_th,
                                 &gauge_slot, &held_cam);
  if (bad) return fail(DGB200_E_ARG, bad);
  if (cg_max_iters < 1) return fail(DGB200_E_ARG, "cg_max_iters must be at least 1");
  if (!(cg_tol >= 0.0) || !(cg_tol < INFINITY)) return fail(DGB200_E_ARG, "cg_tol must be a non-negative finite number");
  if (n_groups < 1) return fail(DGB200_E_ARG, "need n_groups >= 1");
  if (n_free_groups < 0 || n_free_groups > n_groups) return fail(DGB200_E_ARG, "n_free_groups must lie in [0, n_groups]");
  if (n_free_groups > 0 && !h_free_groups) return fail(DGB200_E_ARG, "null free-group list");
  {
    std::vector<unsigned char> seen((size_t)n_groups, 0);
    for (int q = 0; q < n_free_groups; ++q) {
      if (h_free_groups[q] < 0 || h_free_groups[q] >= n_groups) return fail(DGB200_E_ARG, "free group index out of range");
      if (seen[h_free_groups[q]]) return fail(DGB200_E_ARG, "free group index repeated");
      seen[h_free_groups[q]] = 1;
    }
  }
  if (refine & ~(DGB200_REFINE_FOCAL | DGB200_REFINE_PRINCIPAL_POINT | DGB200_REFINE_DISTORTION))
    return fail(DGB200_E_ARG, "refine must be a set of DGB200_REFINE_* bits");
  const cudaStream_t st = (cudaStream_t)stream;
  int sms = 0, per_sm = 0;
  cudaError_t e = cudaSuccess;
  if (const char* m = coop_sms(&sms, &e)) return fail(DGB200_E_CUDA, m, e);
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bai_solve_kernel, kBaiSolveThreads, 0));
  if (per_sm < 1) return fail(DGB200_E_CUDA, "bai_solve_kernel does not fit on an SM");
  // a free group with no refined coordinate changes nothing: no group is free then
  const int ngf = refine ? n_free_groups : 0;
  const int n_ranges = obs > 0 ? blocks((size_t)obs, kBaiRange) : 1;
  const size_t no = (size_t)(obs > 0 ? obs : 1), nt = (size_t)n_tracks, nc = (size_t)n_cams, ng = (size_t)n_groups;
  const size_t nf = (size_t)(n_free > 0 ? n_free : 1), nq = (size_t)(ngf > 0 ? ngf : 1);
  const size_t nch = (size_t)obs / kBaiChunk + nq;    // chunks at most: sum over groups of ceil(n_q / kBaiChunk)
  const size_t npart = (size_t)n_free + (size_t)ngf + nch;
  const size_t nkey = nf > nq ? nf : nq;
  BaiArgs a;
  a.cams = d_cams; a.pts = d_pts; a.R = d_R; a.t = d_t; a.groups = d_groups; a.intr_in = d_intrinsics;
  a.n_cams = n_cams; a.n_groups = n_groups; a.offsets = d_offsets; a.mask = d_mask; a.X = d_X;
  a.n_tracks = n_tracks; a.obs = obs; a.n_free = n_free; a.n_gfree = ngf; a.refine = refine;
  a.gauge_slot = gauge_slot; a.held_cam = held_cam; a.n_ranges = n_ranges; a.n_chunks = (int)nch;
  a.n_part = (int)npart; a.cg_max_iters = cg_max_iters;
  a.sig2 = loss_scale * loss_scale; a.th2 = px_th * px_th; a.cg_tol2 = cg_tol * cg_tol;
  int *d_free = nullptr, *d_gfree = nullptr;
  auto lay_out = [&](char* base) {
    Carve w{base};
    a.tab = w.take<double>(dg::kTrCamStride * nc);
    a.poses = w.take<double>(24 * nc);
    a.intr = w.take<double>(2 * kNK * ng);
    a.Xb = w.take<double>(6 * nt);
    a.trk = w.take<double>(dg::kBaTrkStride * nt);
    a.y = w.take<double>(3 * nt);
    a.Wo = w.take<double>((kWp + kWk) * no);
    a.Cm = w.take<double>(kCm * no);
    a.Gm = w.take<double>(kGm * no);
    a.slot = w.take<double>(kPcStride * nf);
    a.grp = w.take<double>(kGrStride * nq);
    a.chk = w.take<double>(kChStride * nch);
    a.part = w.take<double>(kPcgParts * npart);
    a.state = w.take<BaState>(1);
    a.cg_iters = w.take<int>(1);
    d_free = w.take<int>(nf);
    d_gfree = w.take<int>(nq);
    a.slot_of = w.take<int>(nc);
    a.gslot_of = w.take<int>(ng);
    a.track_of = w.take<int>(no);
    a.sl = w.take<int>(no);
    a.gsl = w.take<int>(no);
    a.pos_of = w.take<int>(no);
    a.gpos_of = w.take<int>(no);
    a.ctrk = w.take<int>(no);
    a.gtrk = w.take<int>(no);
    a.gcs = w.take<int>(no);
    a.hist = w.take<int>(nkey * (size_t)n_ranges);
    a.list_off = w.take<int>(nf + 1);
    a.glist_off = w.take<int>(nq + 1);
    a.chunk_off = w.take<int>(nq + 1);
    a.chunk_beg = w.take<int>(nch);
    a.trk_used = w.take<int>(nt);
    a.usable = w.take<unsigned char>(no);
    a.used = w.take<unsigned char>(no);
    return w.bytes;
  };
  char* ws = nullptr;
  const size_t bytes = lay_out(nullptr);
  CU(cudaMallocAsync((void**)&ws, bytes, st));
  lay_out(ws);
  a.free = d_free; a.gfree = d_gfree;
  a.R_out = d_R_out; a.t_out = d_t_out; a.X_out = d_X_out; a.intr_out = d_intrinsics_out; a.mask_out = d_mask_out;
  a.cost0_out = d_cost0_out; a.cost_out = d_cost_out; a.iters_out = d_iters_out; a.n_used_out = d_n_used_out;
  a.cg_iters_out = d_cg_iters_out;
  const int cam_grid = blocks(nc > ng ? nc : ng, kBaiCamThreads);
  const int trk_grid = blocks(nt, kBaiWarps);
  const int obs_grid = blocks(no, kBaiCamThreads);
  const int range_grid = blocks((size_t)n_ranges, kBaiWarps);
  const size_t hist_bytes = sizeof(int) * nkey * (size_t)n_ranges;
  void* solve_args[] = {&a};
  cudaError_t launch = cudaSuccess;
  if (n_free > 0)
    ADJ_LAUNCH(launch = cudaMemcpyAsync(d_free, h_free, sizeof(int) * (size_t)n_free, cudaMemcpyHostToDevice, st));
  if (ngf > 0)
    ADJ_LAUNCH(launch = cudaMemcpyAsync(d_gfree, h_free_groups, sizeof(int) * (size_t)ngf, cudaMemcpyHostToDevice, st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.usable, 0, no, st));   // rows outside every span are neither usable nor used
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.used, 0, no, st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.slot_of, 0xff, sizeof(int) * nc, st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.gslot_of, 0xff, sizeof(int) * ng, st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.list_off, 0, sizeof(int) * (nf + 1), st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.glist_off, 0, sizeof(int) * (nq + 1), st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.chunk_off, 0, sizeof(int) * (nq + 1), st));
  // entries no one writes stay 0
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.part, 0, sizeof(double) * kPcgParts * npart, st));
  ADJ_LAUNCH((bai_cameras_kernel<<<blocks(nc, kBaiCamThreads), kBaiCamThreads, 0, st>>>(a)));
  ADJ_LAUNCH((bai_slots_kernel<<<cam_grid, kBaiCamThreads, 0, st>>>(a)));
  ADJ_LAUNCH((bai_mark_kernel<<<trk_grid, kBaiThreads, 0, st>>>(a)));
  if (obs > 0) ADJ_LAUNCH((bai_slot_obs_kernel<<<obs_grid, kBaiCamThreads, 0, st>>>(a)));
  if (n_free > 0 && obs > 0) {
    ADJ_LAUNCH(launch = cudaMemsetAsync(a.hist, 0, hist_bytes, st));
    ADJ_LAUNCH((bai_hist_kernel<<<range_grid, kBaiThreads, 0, st>>>(a, a.sl)));
    ADJ_LAUNCH((bai_scan_kernel<<<1, kBaCta, 0, st>>>(a, n_free, a.list_off)));
    ADJ_LAUNCH((bai_scatter_kernel<<<range_grid, kBaiThreads, 0, st>>>(a, a.sl, a.pos_of, a.ctrk)));
  }
  if (ngf > 0 && obs > 0) {
    ADJ_LAUNCH(launch = cudaMemsetAsync(a.hist, 0, hist_bytes, st));
    ADJ_LAUNCH((bai_hist_kernel<<<range_grid, kBaiThreads, 0, st>>>(a, a.gsl)));
    ADJ_LAUNCH((bai_scan_kernel<<<1, kBaCta, 0, st>>>(a, ngf, a.glist_off)));
    ADJ_LAUNCH((bai_scatter_kernel<<<range_grid, kBaiThreads, 0, st>>>(a, a.gsl, a.gpos_of, a.gtrk)));
    ADJ_LAUNCH((bai_chunks_kernel<<<obs_grid, kBaiCamThreads, 0, st>>>(a)));
  }
  ADJ_LAUNCH((bai_init_kernel<<<1, kBaCta, 0, st>>>(a)));
  for (int it = 0; it < max_iters && launch == cudaSuccess; ++it) {
    ADJ_LAUNCH((bai_linearise_kernel<<<trk_grid, kBaiThreads, 0, st>>>(a)));
    ADJ_LAUNCH((bai_points_kernel<<<blocks(nt, kBaiThreads), kBaiThreads, 0, st>>>(a)));
    if (n_free > 0 || ngf > 0) {
      if (n_free > 0) ADJ_LAUNCH((bai_precond_kernel<<<blocks(nf, kBaiWarps), kBaiThreads, 0, st>>>(a)));
      if (ngf > 0) {
        ADJ_LAUNCH((bai_gchunk_kernel<<<blocks(nch, kBaiWarps), kBaiThreads, 0, st>>>(a)));
        ADJ_LAUNCH((bai_group_kernel<<<blocks(nq, kBaiWarps), kBaiThreads, 0, st>>>(a)));
      }
      ADJ_LAUNCH(launch = cudaLaunchCooperativeKernel((const void*)bai_solve_kernel, per_sm * sms, kBaiSolveThreads,
                                                      solve_args, 0, st));
    }
    ADJ_LAUNCH((bai_backsub_kernel<<<trk_grid, kBaiThreads, 0, st>>>(a)));
    ADJ_LAUNCH((bai_decide_kernel<<<1, kBaCta, 0, st>>>(a)));
  }
  if (obs > 0) ADJ_LAUNCH(launch = cudaMemsetAsync(d_mask_out, 0, (size_t)obs, st));   // rows outside every span
  ADJ_LAUNCH((bai_finish_cameras_kernel<<<cam_grid, kBaiCamThreads, 0, st>>>(a)));
  ADJ_LAUNCH((bai_finish_tracks_kernel<<<trk_grid, kBaiThreads, 0, st>>>(a)));
  CU(cudaFreeAsync(ws, st));
  CU(launch);
  return 0;
}

int dgb200_undistort_points_dev(const double* d_pts, const int32_t* d_cams, int rows, const int32_t* d_groups,
                                int n_cams, const double* d_intrinsics, int n_groups, double* d_out, void* stream) {
  if (!d_groups || !d_intrinsics) return fail_ud(DGB200_E_ARG, "null buffer");
  if (rows > 0 && (!d_pts || !d_cams || !d_out)) return fail_ud(DGB200_E_ARG, "null row buffer");
  if (rows < 0 || n_cams < 1 || n_groups < 1)
    return fail_ud(DGB200_E_ARG, "need rows >= 0, n_cams >= 1 and n_groups >= 1");
  if (rows == 0) return 0;
  undistort_kernel<<<blocks((size_t)rows, kBaiCamThreads), kBaiCamThreads, 0, (cudaStream_t)stream>>>(
      d_pts, d_cams, rows, d_groups, n_cams, d_intrinsics, n_groups, d_out);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail_ud(DGB200_E_CUDA, "undistort_kernel", e);
  return 0;
}

}  // extern "C"
