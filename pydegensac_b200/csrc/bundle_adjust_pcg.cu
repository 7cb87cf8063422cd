// bundle_adjust_pcg.cu -- bundle adjustment of any number of cameras, device resident: the Levenberg-Marquardt of
// bundle_adjust.cu with the reduced camera system solved inexactly by conjugate gradients on the implicit Schur
// complement with a block-Jacobi preconditioner (Ceres' ITERATIVE_SCHUR with SCHUR_JACOBI; Agarwal et al., "Bundle
// Adjustment in the Large").  S is never formed: S p = U* p - sum_p W_p V*_p^-1 (W_p^T p) is one pass over the tracks
// and one over the cameras.  A translation unit of its own, so that adding it changes no instruction of the other
// sources' kernels.
//
// Once per call:
//   pcg_cameras_kernel   the camera table and both pose buffers; pcg_slots_kernel the map from camera to free slot;
//   pcg_mark_kernel      one warp per track: ba_mark_track (bundle_adjust_device.h);
//   pcg_slot_obs_kernel  the free slot of each used observation (-1: none);
//   pcg_hist_kernel,     the camera-major list of the used observations of the free cameras, ascending observation
//   pcg_scan_kernel,     order within a camera, by the one-digit stable counting sort of bundle_adjust_device.h
//   pcg_scatter_kernel   (ba_sort_*): one warp per range of kPcgRange observations counts its observations per slot,
//                        one CTA scans the counts slot after slot, and each warp scatters its range in order;
//   pcg_init_kernel      one CTA: cost0, n_used, the scale gauge's axis, the LM state (ba_init_state).
// Per trial step (the host launches max_iters steps; each kernel returns at once when the state says the call stopped):
//   pcg_linearise_kernel one warp per track, after an accepted step: V_p and g_p per track; W = w J_cam^T J_X per
//                        observation in observation order, and W, J_cam, r, w in camera-major order;
//   pcg_points_kernel    one thread per track: V*_p^-1;
//   pcg_precond_kernel   one warp per free slot: U_a, g_a, the preconditioner block M_a = U*_a - sum W_i V*^-1 W_i^T
//                        and its Cholesky factor, the right-hand side b_a and the start of PCG;
//   pcg_solve_kernel     the whole PCG loop in one cooperative launch (grid.sync between the phases), then the trial
//                        poses of the free cameras;
//   pcg_backsub_kernel   one warp per track: dX_p = -V*_p^-1 (g_p + sum W_i^T dc), the trial point and its cost;
//   pcg_decide_kernel    one CTA: ba_decide_step.
// After the last step pcg_finish_cameras_kernel and pcg_finish_tracks_kernel write the outputs and the inlier mask.
//
// One PCG iteration, each phase a grid-stride loop over a fixed partition of the work:
//   A  one thread per track: p_s = z_s + beta p'_s gathered by camera, y_p = V*_p^-1 sum W_i^T p_s(i);
//   B  one warp per free slot: q_a = U*_a p_a - sum W_i y_p(i) over the slot's camera-major list; p_a stored; p_a . q_a;
//   C  one thread per free slot: x += alpha p, r -= alpha q, z = M^-1 r; r . r and r . z.
// The loop itself, the dot products' fixed-order CTA sums and the record helpers are pcg_run and its helpers in
// pcg_device.h.  No floating-point atomics anywhere: a rerun gives the same bytes.
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
#include "device_util.h"
#include "bundle_adjust_device.h"
#include "pcg_device.h"
#include "adjust_host.h"

namespace cg = cooperative_groups;

namespace {

thread_local char g_err[256] = "";
int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err, code, what, e); }

constexpr int kPcgWarps = 4;                      // tracks or slots per CTA, one per warp
constexpr int kPcgThreads = 32 * kPcgWarps;
constexpr int kPcgCamThreads = 128;
constexpr int kPcgSolveThreads = 256;             // the cooperative kernel
constexpr int kPcgRange = 4096;                   // observations per warp of the counting sort
constexpr int kPcgW = 18;                         // W [6][3] per observation

// One free slot's record: U (upper by rows, 21), g_c (6), the preconditioner's Cholesky factor L (lower by rows, 21),
// then its PCG vectors (pcg_device.h): b, x, r, z (6 each), p in two buffers (12), q (6)
constexpr int kPcU = 0, kPcG = 21, kPcL = 27, kPcB = 48, kPcX = 54, kPcP = 72, kPcQ = 84, kPcStride = 90;

struct PcgArgs {
  const int* cams; const double* pts;                      // [obs], [obs][2]
  const double* R; const double* t; const double* K;
  int k_per_camera, n_cams;
  const int* offsets; const unsigned char* mask;           // [T+1], [obs] or null
  const double* X;                                         // [T][3]
  int n_tracks, obs, n_free, gauge_slot, held_cam, n_ranges, cg_max_iters;
  double sig2, th2, cg_tol2;
  const int* free;   // [n_free], on the device
  // workspace
  double* tab;       // [n_cams][kTrCamStride]
  double* poses;     // [2][n_cams][12]: current and trial
  double* Xb;        // [2][T][3]
  double* trk;       // [T][kBaTrkStride]
  double* y;         // [T][3]
  double* Wt;        // [18][obs]: W of the used observations of free cameras, by observation
  double* Wc;        // [18][obs]: the same, camera-major (the first list_off[n_free] columns)
  double* Jr;        // [15][obs]: J_cam, r, w, camera-major
  double* slot;      // [n_free][kPcStride]
  double* part;      // [kPcgParts][n_free]
  BaState* state;
  int* cg_iters;     // [1]
  int* slot_of;      // [n_cams]
  int* track_of;     // [obs]
  int* sl;           // [obs]: the free slot of a used observation, or -1
  int* pos_of;       // [obs]: its position in the camera-major list
  int* ctrk;         // [obs]: the track of each camera-major entry
  int* hist;         // [n_free][n_ranges]: counts, then cursors
  int* list_off;     // [n_free + 1]
  int* trk_used;     // [T]: used observations of the track (0: not optimised)
  unsigned char* usable; unsigned char* used;   // [obs]
  // outputs
  double* R_out; double* t_out; double* X_out; unsigned char* mask_out;
  double* cost0_out; double* cost_out; int* iters_out; int* n_used_out; int* cg_iters_out;
};

__device__ __forceinline__ const double* pose_of(const PcgArgs& a, int buf, int c) {
  return a.poses + 12 * ((size_t)buf * a.n_cams + c);
}
__device__ __forceinline__ double* point_of(const PcgArgs& a, int buf, int j) {
  return a.Xb + 3 * ((size_t)buf * a.n_tracks + j);
}
__device__ __forceinline__ double* slot_rec(const PcgArgs& a, int s) { return a.slot + kPcStride * (size_t)s; }
__device__ __forceinline__ bool slot_active(const PcgArgs& a, int s) { return a.list_off[s + 1] > a.list_off[s]; }

// ---------------------------------------------------------------------------------------------- once per call
__global__ void __launch_bounds__(kPcgCamThreads) pcg_cameras_kernel(PcgArgs a) {
  const int c = blockIdx.x * kPcgCamThreads + threadIdx.x;
  if (c >= a.n_cams) return;
  const double* R = a.R + 9 * (size_t)c;
  const double* t = a.t + 3 * (size_t)c;
  dg::tr_camera(R, t, a.K + (a.k_per_camera ? 9 * (size_t)c : 0), a.tab + dg::kTrCamStride * (size_t)c);
  for (int buf = 0; buf < 2; ++buf) {
    double* P = a.poses + 12 * ((size_t)buf * a.n_cams + c);
    for (int i = 0; i < 9; ++i) P[i] = R[i];
    for (int i = 0; i < 3; ++i) P[9 + i] = t[i];
  }
}

__global__ void __launch_bounds__(kPcgCamThreads) pcg_slots_kernel(PcgArgs a) {
  const int q = blockIdx.x * kPcgCamThreads + threadIdx.x;
  if (q < a.n_free) a.slot_of[a.free[q]] = q;
}

__global__ void __launch_bounds__(kPcgThreads) pcg_mark_kernel(PcgArgs a) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kPcgWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks) return;                       // (warp-uniform)
  ba_mark_track(a, j, lane);
}

__global__ void __launch_bounds__(kPcgCamThreads) pcg_slot_obs_kernel(PcgArgs a) {
  const int r = blockIdx.x * kPcgCamThreads + threadIdx.x;
  if (r < a.obs) a.sl[r] = a.used[r] ? a.slot_of[a.cams[r]] : -1;
}

// The camera-major list by ba_sort_* (bundle_adjust_device.h), keyed by the free slot
__global__ void __launch_bounds__(kPcgThreads) pcg_hist_kernel(PcgArgs a) {
  const int w = blockIdx.x * kPcgWarps + (threadIdx.x >> 5);
  if (w >= a.n_ranges) return;                       // (warp-uniform)
  ba_sort_count(a.sl, a.obs, kPcgRange, a.hist, a.n_ranges, w, threadIdx.x & 31);
}

__global__ void __launch_bounds__(kBaCta) pcg_scan_kernel(PcgArgs a) {
  __shared__ int sh[kBaCta];
  ba_sort_scan(a.hist, a.n_free, a.n_ranges, a.list_off, sh);
}

__global__ void __launch_bounds__(kPcgThreads) pcg_scatter_kernel(PcgArgs a) {
  const int w = blockIdx.x * kPcgWarps + (threadIdx.x >> 5);
  if (w >= a.n_ranges) return;                       // (warp-uniform)
  ba_sort_scatter(a.sl, a.obs, kPcgRange, a.hist, a.n_ranges, a.track_of, a.pos_of, a.ctrk, w, threadIdx.x & 31);
}

__global__ void __launch_bounds__(kBaCta) pcg_init_kernel(PcgArgs a) {
  ba_init_state(a);
  if (threadIdx.x == 0) a.cg_iters[0] = 0;
}

// ---------------------------------------------------------------------------------------------- one trial step
__global__ void __launch_bounds__(kPcgThreads) pcg_linearise_kernel(PcgArgs a) {
  const BaState* st = a.state;
  if (st->stop || !st->lin) return;
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kPcgWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks || a.trk_used[j] == 0) return;   // (warp-uniform)
  const int cur = st->cur;
  const double* X = point_of(a, cur, j);
  const int b = a.offsets[j], e = a.offsets[j + 1];
  const size_t no = (size_t)a.obs;
  double V[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
  for (int r = b + lane; r < e; r += 32) {
    if (!a.used[r]) continue;
    const int cm = a.cams[r];
    double rr[2], Jc[12], Jx[6];
    dg::ba_jacobian(pose_of(a, cur, cm), a.tab + dg::kTrCamStride * (size_t)cm + dg::kTrCamK, X, a.pts[2 * (size_t)r],
                    a.pts[2 * (size_t)r + 1], rr, Jc, Jx);
    const double w = dg::ba_weight(rr[0] * rr[0] + rr[1] * rr[1], a.sig2);
    dg::ba_point_terms(Jx, rr, w, V, g);
    if (a.sl[r] >= 0) {
      double W[kPcgW];
      dg::ba_cross_block(Jc, Jx, w, W);
      const size_t pos = (size_t)a.pos_of[r];
#pragma unroll
      for (int k = 0; k < kPcgW; ++k) {
        a.Wt[k * no + r] = W[k];
        a.Wc[k * no + pos] = W[k];
      }
#pragma unroll
      for (int k = 0; k < 12; ++k) a.Jr[k * no + pos] = Jc[k];
      a.Jr[12 * no + pos] = rr[0];
      a.Jr[13 * no + pos] = rr[1];
      a.Jr[14 * no + pos] = w;
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

__global__ void __launch_bounds__(kPcgThreads) pcg_points_kernel(PcgArgs a) {
  BaState* st = a.state;
  if (st->stop) return;
  const int j = blockIdx.x * kPcgThreads + threadIdx.x;
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

// One warp per free slot: U, g_c, M = U* - sum W V*^-1 W^T and b = -(g_c - sum W V*^-1 g_p) over the slot's list; the
// held coordinate's row and column of M become the identity's and its b is 0; an inactive slot gets U = 0, M = I, b = 0.
// Then the start of PCG: x = 0, r = b, z = M^-1 r, both p buffers 0, and the slot's r . z and b . b.
__global__ void __launch_bounds__(kPcgThreads) pcg_precond_kernel(PcgArgs a) {
  BaState* st = a.state;
  if (st->stop || st->bad) return;
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x * kPcgWarps + (threadIdx.x >> 5);
  if (s >= a.n_free) return;                           // (warp-uniform)
  const size_t no = (size_t)a.obs;
  double U[21], gc[6], Mw[21], h[6];
#pragma unroll
  for (int m = 0; m < 21; ++m) { U[m] = 0.0; Mw[m] = 0.0; }
#pragma unroll
  for (int k = 0; k < 6; ++k) { gc[k] = 0.0; h[k] = 0.0; }
  const int i0 = a.list_off[s], i1 = a.list_off[s + 1];
  for (int i = i0 + lane; i < i1; i += 32) {
    double Jc[12], W[kPcgW], Y[kPcgW];
#pragma unroll
    for (int k = 0; k < 12; ++k) Jc[k] = a.Jr[k * no + i];
    const double e0 = a.Jr[12 * no + i], e1 = a.Jr[13 * no + i], w = a.Jr[14 * no + i];
#pragma unroll
    for (int k = 0; k < kPcgW; ++k) W[k] = a.Wc[k * no + i];
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
  const int hold = st->hold_row - dg::kBaCamParams * s;   // the held coordinate in this slot, or outside [0, 6)
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
  pcg_start<6>(rec + kPcB, b, z, a.part, a.n_free, s);
#pragma unroll
  for (int k = 0; k < 6; ++k) rec[kPcG + k] = gc[k];
#pragma unroll
  for (int q = 0; q < 21; ++q) rec[kPcU + q] = active ? U[q] : 0.0;
}

// pcg_run's S p and phase C over the free slots.  product: A, one thread per track, y_p = V*_p^-1 sum W_i^T p_s(i);
// grid.sync; B, one warp per free slot, q_a = U*_a p_a - sum W_i y_p(i), p_a stored, p_a . q_a.  update: one thread
// per free slot.
struct PcgSchur {
  const PcgArgs& a;
  int tid, nthr, lane, warp, nwarps;
  double lam;
  int hold_row;

  __device__ __forceinline__ void product(cg::grid_group& grid, int cur, int prev, double beta) const {
    const int nf = a.n_free;
    const size_t no = (size_t)a.obs;
    for (int j = tid; j < a.n_tracks; j += nthr) {
      if (a.trk_used[j] == 0) continue;
      const int b = a.offsets[j], e = a.offsets[j + 1];
      double u[3] = {0.0, 0.0, 0.0};
      for (int r = b; r < e; ++r) {
        const int s = a.sl[r];
        if (s < 0) continue;
        double p[6];
        pcg_direction<6>(slot_rec(a, s) + kPcB, prev, beta, p);
#pragma unroll
        for (int k = 0; k < 6; ++k)
#pragma unroll
          for (int m = 0; m < 3; ++m) u[m] += __ldg(a.Wt + (3 * k + m) * no + r) * p[k];
      }
      double yv[3];
      dg::ba_sym3_mul(a.trk + dg::kBaTrkStride * (size_t)j + dg::kBaTrkVi, u, yv);
#pragma unroll
      for (int m = 0; m < 3; ++m) a.y[3 * (size_t)j + m] = yv[m];
    }
    grid.sync();
    for (int s = warp; s < nf; s += nwarps) {
      double acc[6] = {0, 0, 0, 0, 0, 0};
      const int i0 = a.list_off[s], i1 = a.list_off[s + 1];
      for (int i = i0 + lane; i < i1; i += 32) {
        const double* yp = a.y + 3 * (size_t)a.ctrk[i];
        const double y0 = __ldcg(yp), y1 = __ldcg(yp + 1), y2 = __ldcg(yp + 2);
#pragma unroll
        for (int k = 0; k < 6; ++k)
          acc[k] += __ldg(a.Wc + (3 * k) * no + i) * y0 + __ldg(a.Wc + (3 * k + 1) * no + i) * y1 +
                    __ldg(a.Wc + (3 * k + 2) * no + i) * y2;
      }
#pragma unroll
      for (int k = 0; k < 6; ++k) acc[k] = warp_sum(acc[k]);
      if (lane == 0) {
        double p[6];
        double* rec = slot_rec(a, s);
        pcg_direction<6>(rec + kPcB, prev, beta, p);
        const double* U = rec + kPcU;
        const int hold = hold_row - dg::kBaCamParams * s;
        double pq = 0.0;
#pragma unroll
        for (int k = 0; k < 6; ++k) {
          double v = -acc[k];
#pragma unroll
          for (int l = 0; l < 6; ++l) {
            const int m = k <= l ? k * 6 - k * (k - 1) / 2 + (l - k) : l * 6 - l * (l - 1) / 2 + (k - l);
            v += U[m] * p[l];
          }
          const int d = k * 6 - k * (k - 1) / 2;
          v += lam * U[d] * p[k];
          if (k == hold) v = p[k];
          rec[kPcQ + k] = v;
          rec[kPcP + 6 * cur + k] = p[k];
          pq += p[k] * v;
        }
        a.part[kPartPQ * (size_t)nf + s] = pq;
      }
    }
  }

  __device__ __forceinline__ void update(int cur, int /*prev*/, double /*beta*/, double alpha) const {
    const int nf = a.n_free;
    for (int s = tid; s < nf; s += nthr) {
      double* rec = slot_rec(a, s);
      double p[6], q[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        p[k] = __ldcg(rec + kPcP + 6 * cur + k);
        q[k] = __ldcg(rec + kPcQ + k);
      }
      const double2 rz = pcg_update<6>(rec + kPcB, p, q, alpha, [rec](const double* r, double* z) {
        dg::pr_cholesky_apply<6>(rec + kPcL, r, z);
      });
      a.part[kPartRR * (size_t)nf + s] = rz.x;
      a.part[kPartRZ * (size_t)nf + s] = rz.y;
    }
  }
};

// The PCG loop of one trial step (pcg_run), then the trial poses of the free cameras
__global__ void __launch_bounds__(kPcgSolveThreads) pcg_solve_kernel(PcgArgs a) {
  __shared__ double sh[2 * kPcgSolveThreads];
  BaState* st = a.state;
  if (st->stop || st->bad) return;                     // (grid-uniform: nothing below writes them before a grid.sync)
  cg::grid_group grid = cg::this_grid();
  const int tid = blockIdx.x * kPcgSolveThreads + threadIdx.x, nthr = gridDim.x * kPcgSolveThreads;
  const int nf = a.n_free;
  const PcgSchur op{a, tid, nthr, (int)threadIdx.x & 31, tid >> 5, nthr >> 5, st->lam, st->hold_row};
  const PcgResult res = pcg_run<kPcgSolveThreads>(grid, a.part, nf, a.cg_tol2, a.cg_max_iters, sh, op);
  // the trial poses (x of a slot was last written by this thread, in phase C)
  const int cur = st->cur;
  if (!res.reject)
    for (int s = tid; s < nf; s += nthr) {
      if (!slot_active(a, s)) continue;
      const int c = a.free[s];
      double P2[12];
      dg::ap_step(pose_of(a, cur, c), slot_rec(a, s) + kPcX, P2);
      if (dg::pr_ortho_drift(P2) > dg::kPrOrthoTol) dg::pr_orthonormalise(P2);
      double* out = a.poses + 12 * ((size_t)(1 - cur) * a.n_cams + c);
      for (int i = 0; i < 12; ++i) out[i] = P2[i];
    }
  if (tid == 0) {
    a.cg_iters[0] += res.iters;
    if (res.reject) st->bad = 1;
  }
}

__global__ void __launch_bounds__(kPcgThreads) pcg_backsub_kernel(PcgArgs a) {
  const BaState* st = a.state;
  if (st->stop || st->bad) return;
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kPcgWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks || a.trk_used[j] == 0) return;   // (warp-uniform)
  const int cur = st->cur, b = a.offsets[j], e = a.offsets[j + 1];
  const size_t no = (size_t)a.obs;
  double acc[3] = {0.0, 0.0, 0.0};
  for (int r = b + lane; r < e; r += 32) {
    const int s = a.sl[r];
    if (s < 0) continue;
    const double* d = slot_rec(a, s) + kPcX;
#pragma unroll
    for (int m = 0; m < 3; ++m)
#pragma unroll
      for (int k = 0; k < 6; ++k) acc[m] += a.Wt[(3 * k + m) * no + r] * d[k];
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
    bool front;
    const double e2 = dg::ap_sq_error(pose_of(a, 1 - cur, cm), a.tab + dg::kTrCamStride * (size_t)cm + dg::kTrCamK,
                                      a.pts[2 * (size_t)r], a.pts[2 * (size_t)r + 1], X[0], X[1], X[2], &front);
    c += front ? dg::ba_rho(e2, a.sig2) : INFINITY;
  }
  c = warp_sum(c);
  if (lane == 0) a.trk[dg::kBaTrkStride * (size_t)j + dg::kBaTrkCost] = c;
}

__global__ void __launch_bounds__(kBaCta) pcg_decide_kernel(PcgArgs a) {
  __shared__ double shd[kBaCta];
  if (a.state->stop) return;                           // (block-uniform)
  ba_decide_step(a, shd);
}

// ---------------------------------------------------------------------------------------------- outputs
__global__ void __launch_bounds__(kPcgCamThreads) pcg_finish_cameras_kernel(PcgArgs a) {
  const int c = blockIdx.x * kPcgCamThreads + threadIdx.x;
  if (c == 0) a.cg_iters_out[0] = a.cg_iters[0];
  ba_finish_camera(a, c);
}

__global__ void __launch_bounds__(kPcgThreads) pcg_finish_tracks_kernel(PcgArgs a) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kPcgWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks) return;
  ba_finish_track(a, j, lane);
}

}  // namespace

extern "C" {

const char* dgb200_bundle_adjust_pcg_last_error(void) { return g_err; }

int dgb200_bundle_adjust_pcg_ragged_dev(const int32_t* d_cams, const double* d_pts, const double* d_R,
                                        const double* d_t, const double* d_K, int k_per_camera, int n_cams,
                                        const int32_t* d_offsets, int n_tracks, int obs, const double* d_X,
                                        const uint8_t* d_mask, const int32_t* h_free, int n_free, int scale_gauge,
                                        double loss_scale, int max_iters, double px_th, int cg_max_iters,
                                        double cg_tol, double* d_R_out, double* d_t_out, double* d_X_out,
                                        uint8_t* d_mask_out, double* d_cost0_out, double* d_cost_out,
                                        int32_t* d_iters_out, int32_t* d_n_used_out, int32_t* d_cg_iters_out,
                                        void* stream) {
  int gauge_slot = -1, held_cam = -1;
  const char* bad = ba_arg_error(!d_R || !d_t || !d_K || !d_offsets || !d_X || !d_R_out || !d_t_out || !d_X_out ||
                                     !d_cost0_out || !d_cost_out || !d_iters_out || !d_n_used_out || !d_cg_iters_out,
                                 !d_cams || !d_pts || !d_mask_out, n_tracks, obs, n_cams, h_free, n_free, n_cams,
                                 "n_free must lie in [0, n_cams]", scale_gauge, loss_scale, max_iters, px_th,
                                 &gauge_slot, &held_cam);
  if (bad) return fail(DGB200_E_ARG, bad);
  if (cg_max_iters < 1) return fail(DGB200_E_ARG, "cg_max_iters must be at least 1");
  if (!(cg_tol >= 0.0) || !(cg_tol < INFINITY)) return fail(DGB200_E_ARG, "cg_tol must be a non-negative finite number");
  const cudaStream_t st = (cudaStream_t)stream;
  int sms = 0, per_sm = 0;
  cudaError_t e = cudaSuccess;
  if (const char* m = coop_sms(&sms, &e)) return fail(DGB200_E_CUDA, m, e);
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pcg_solve_kernel, kPcgSolveThreads, 0));
  if (per_sm < 1) return fail(DGB200_E_CUDA, "pcg_solve_kernel does not fit on an SM");
  const int n_ranges = obs > 0 ? blocks((size_t)obs, kPcgRange) : 1;
  const size_t no = (size_t)(obs > 0 ? obs : 1), nt = (size_t)n_tracks, nc = (size_t)n_cams;
  const size_t nf = (size_t)(n_free > 0 ? n_free : 1);
  PcgArgs a;
  a.cams = d_cams; a.pts = d_pts; a.R = d_R; a.t = d_t; a.K = d_K; a.k_per_camera = k_per_camera; a.n_cams = n_cams;
  a.offsets = d_offsets; a.mask = d_mask; a.X = d_X; a.n_tracks = n_tracks; a.obs = obs; a.n_free = n_free;
  a.gauge_slot = gauge_slot; a.held_cam = held_cam; a.n_ranges = n_ranges; a.cg_max_iters = cg_max_iters;
  a.sig2 = loss_scale * loss_scale; a.th2 = px_th * px_th; a.cg_tol2 = cg_tol * cg_tol;
  int* d_free = nullptr;
  auto lay_out = [&](char* base) {
    Carve w{base};
    a.tab = w.take<double>(dg::kTrCamStride * nc);
    a.poses = w.take<double>(24 * nc);
    a.Xb = w.take<double>(6 * nt);
    a.trk = w.take<double>(dg::kBaTrkStride * nt);
    a.y = w.take<double>(3 * nt);
    a.Wt = w.take<double>(kPcgW * no);
    a.Wc = w.take<double>(kPcgW * no);
    a.Jr = w.take<double>(15 * no);
    a.slot = w.take<double>(kPcStride * nf);
    a.part = w.take<double>(kPcgParts * nf);
    a.state = w.take<BaState>(1);
    a.cg_iters = w.take<int>(1);
    d_free = w.take<int>(nf);
    a.slot_of = w.take<int>(nc);
    a.track_of = w.take<int>(no);
    a.sl = w.take<int>(no);
    a.pos_of = w.take<int>(no);
    a.ctrk = w.take<int>(no);
    a.hist = w.take<int>(nf * (size_t)n_ranges);
    a.list_off = w.take<int>(nf + 1);
    a.trk_used = w.take<int>(nt);
    a.usable = w.take<unsigned char>(no);
    a.used = w.take<unsigned char>(no);
    return w.bytes;
  };
  char* ws = nullptr;
  const size_t bytes = lay_out(nullptr);
  CU(cudaMallocAsync((void**)&ws, bytes, st));
  lay_out(ws);
  a.free = d_free;
  a.R_out = d_R_out; a.t_out = d_t_out; a.X_out = d_X_out; a.mask_out = d_mask_out;
  a.cost0_out = d_cost0_out; a.cost_out = d_cost_out; a.iters_out = d_iters_out; a.n_used_out = d_n_used_out;
  a.cg_iters_out = d_cg_iters_out;
  const int cam_grid = blocks(nc, kPcgCamThreads);
  const int trk_grid = blocks(nt, kPcgWarps);
  const int obs_grid = blocks(no, kPcgCamThreads);
  const int range_grid = blocks((size_t)n_ranges, kPcgWarps);
  const int slot_grid = blocks(nf, kPcgWarps);
  void* solve_args[] = {&a};
  cudaError_t launch = cudaSuccess;
  if (n_free > 0)
    ADJ_LAUNCH(launch = cudaMemcpyAsync(d_free, h_free, sizeof(int) * (size_t)n_free, cudaMemcpyHostToDevice, st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.usable, 0, no, st));   // rows outside every span are neither usable nor used
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.used, 0, no, st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.slot_of, 0xff, sizeof(int) * nc, st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.list_off, 0, sizeof(int) * (nf + 1), st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.hist, 0, sizeof(int) * nf * (size_t)n_ranges, st));
  ADJ_LAUNCH((pcg_cameras_kernel<<<cam_grid, kPcgCamThreads, 0, st>>>(a)));
  if (n_free > 0) ADJ_LAUNCH((pcg_slots_kernel<<<blocks(nf, kPcgCamThreads), kPcgCamThreads, 0, st>>>(a)));
  ADJ_LAUNCH((pcg_mark_kernel<<<trk_grid, kPcgThreads, 0, st>>>(a)));
  if (obs > 0) ADJ_LAUNCH((pcg_slot_obs_kernel<<<obs_grid, kPcgCamThreads, 0, st>>>(a)));
  if (n_free > 0 && obs > 0) {
    ADJ_LAUNCH((pcg_hist_kernel<<<range_grid, kPcgThreads, 0, st>>>(a)));
    ADJ_LAUNCH((pcg_scan_kernel<<<1, kBaCta, 0, st>>>(a)));
    ADJ_LAUNCH((pcg_scatter_kernel<<<range_grid, kPcgThreads, 0, st>>>(a)));
  }
  ADJ_LAUNCH((pcg_init_kernel<<<1, kBaCta, 0, st>>>(a)));
  for (int it = 0; it < max_iters && launch == cudaSuccess; ++it) {
    ADJ_LAUNCH((pcg_linearise_kernel<<<trk_grid, kPcgThreads, 0, st>>>(a)));
    ADJ_LAUNCH((pcg_points_kernel<<<blocks(nt, kPcgThreads), kPcgThreads, 0, st>>>(a)));
    if (n_free > 0) {
      ADJ_LAUNCH((pcg_precond_kernel<<<slot_grid, kPcgThreads, 0, st>>>(a)));
      ADJ_LAUNCH(launch = cudaLaunchCooperativeKernel((const void*)pcg_solve_kernel, per_sm * sms, kPcgSolveThreads,
                                                      solve_args, 0, st));
    }
    ADJ_LAUNCH((pcg_backsub_kernel<<<trk_grid, kPcgThreads, 0, st>>>(a)));
    ADJ_LAUNCH((pcg_decide_kernel<<<1, kBaCta, 0, st>>>(a)));
  }
  if (obs > 0) ADJ_LAUNCH(launch = cudaMemsetAsync(d_mask_out, 0, (size_t)obs, st));   // rows outside every span
  ADJ_LAUNCH((pcg_finish_cameras_kernel<<<cam_grid, kPcgCamThreads, 0, st>>>(a)));
  ADJ_LAUNCH((pcg_finish_tracks_kernel<<<trk_grid, kPcgThreads, 0, st>>>(a)));
  CU(cudaFreeAsync(ws, st));
  CU(launch);
  return 0;
}

}  // extern "C"
