// bundle_adjust.cu -- bundle adjustment of registered views and their tracks, device resident: Levenberg-Marquardt
// over the free cameras' poses and the tracks' points jointly, with the points eliminated by the Schur complement
// (what an incremental reconstruction runs after registering a view).  A translation unit of its own, so that adding
// it changes no instruction of the kernels in degensac_b200.cu, frontend.cu, absolute_pose.cu and triangulate.cu.
//
// Once per call:
//   ba_cameras_kernel   the camera table (triangulate.h: pose, K, centre, registered), both pose buffers and the map
//                       from camera to free slot;
//   ba_mark_kernel      one warp per track: the usable observations, whether the track is optimised (2 distinct
//                       cameras, V_p at the start has a positive Cholesky factor), its start cost, both point buffers;
//   ba_count_kernel,    one CTA per free slot: the slot's used observations, then their camera-major list in
//   ba_list_kernel      observation order by a block ballot scan;
//   ba_init_kernel      one CTA: cost0 and n_used by fixed-order sums, the scale gauge's axis, the LM state.
// Per trial step (the host launches max_iters steps; each kernel returns at once when the state says the call stopped):
//   ba_linearise_kernel one warp per track, after an accepted step: J_cam, r, w and W = w J_cam^T J_X per observation,
//                       V_p and g_p per track;
//   ba_points_kernel    one warp per track: V*_p^-1 and Y_i = W_i V*_p^-1;
//   ba_schur_kernel     one warp per upper block (a, b) of S: lanes stride over slot a's list, find the partners from
//                       camera b in the same track span and reduce by butterfly; diagonal blocks add U*_a and the
//                       reduced right-hand side;
//   ba_solve_kernel     one CTA: dense Cholesky of S, the two triangular solves and the free cameras' trial poses;
//   ba_backsub_kernel   one warp per track: dX_p = -V*_p^-1 (g_p + sum W_i^T dc), the trial point and its cost;
//   ba_decide_kernel    one CTA: fixed-order sum of the track costs, accept / reject / stop, lambda, buffer swap.
// After the last step ba_finish_cameras_kernel and ba_finish_tracks_kernel write the outputs and the inlier mask.
// No floating-point atomics anywhere: every sum has a fixed order, so a rerun gives the same bytes.  The bodies of the
// mark, init, decide and finish kernels are in bundle_adjust_device.h, the argument checks in bundle_adjust_args.h
// and the launch plumbing in adjust_host.h, shared with the iterative solver of bundle_adjust_pcg.cu.
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
#include "adjust_host.h"

namespace {

thread_local char g_err[256] = "";
int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err, code, what, e); }

constexpr int kBaWarps = 4;                       // tracks (or Schur blocks) per CTA, one per warp
constexpr int kBaThreads = 32 * kBaWarps;
constexpr int kBaCamThreads = 128;

struct BaArgs {
  const int* cams; const double* pts;                      // [obs], [obs][2]
  const double* R; const double* t; const double* K;       // inputs, read by ba_cameras_kernel only
  int k_per_camera, n_cams;
  const int* offsets; const unsigned char* mask;           // [T+1], [obs] or null
  const double* X;                                         // [T][3], read by ba_mark_kernel only
  int n_tracks, obs, n_free, n, gauge_slot, held_cam, n_blocks;
  int free[dg::kBaMaxFree];
  double sig2, th2;
  // workspace
  double* tab;       // [n_cams][kTrCamStride]
  double* poses;     // [2][n_cams][12]: current and trial
  double* Xb;        // [2][T][3]
  double* obsd;      // [obs][kBaObsStride]
  double* trk;       // [T][kBaTrkStride]
  double* S;         // [n][n]
  double* rhs;       // [n]
  BaState* state;
  int* slot_of;      // [n_cams]
  int* track_of;     // [obs]
  int* list;         // [obs]: the used observations of each free slot, slot after slot
  int* counts;       // [n_free]
  int* list_off;     // [n_free + 1]
  int* trk_used;     // [T]: used observations of the track (0: not optimised)
  unsigned char* usable; unsigned char* used;   // [obs]
  // outputs
  double* R_out; double* t_out; double* X_out; unsigned char* mask_out;
  double* cost0_out; double* cost_out; int* iters_out; int* n_used_out;
};

__device__ __forceinline__ const double* pose_of(const BaArgs& a, int buf, int c) {
  return a.poses + 12 * ((size_t)buf * a.n_cams + c);
}
__device__ __forceinline__ double* point_of(const BaArgs& a, int buf, int j) {
  return a.Xb + 3 * ((size_t)buf * a.n_tracks + j);
}
__device__ __forceinline__ bool slot_active(const BaArgs& a, int s) { return a.list_off[s + 1] > a.list_off[s]; }

__global__ void __launch_bounds__(kBaCamThreads) ba_cameras_kernel(BaArgs a) {
  const int c = blockIdx.x * kBaCamThreads + threadIdx.x;
  if (c >= a.n_cams) return;
  const double* R = a.R + 9 * (size_t)c;
  const double* t = a.t + 3 * (size_t)c;
  dg::tr_camera(R, t, a.K + (a.k_per_camera ? 9 * (size_t)c : 0), a.tab + dg::kTrCamStride * (size_t)c);
  for (int buf = 0; buf < 2; ++buf) {
    double* P = a.poses + 12 * ((size_t)buf * a.n_cams + c);
    for (int i = 0; i < 9; ++i) P[i] = R[i];
    for (int i = 0; i < 3; ++i) P[9 + i] = t[i];
  }
  int s = -1;
  for (int q = 0; q < a.n_free; ++q) s = a.free[q] == c ? q : s;
  a.slot_of[c] = s;
}

// Usable observations, whether the track is optimised, its start cost, both point buffers
__global__ void __launch_bounds__(kBaThreads) ba_mark_kernel(BaArgs a) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kBaWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks) return;                       // (warp-uniform)
  ba_mark_track(a, j, lane);
}

__device__ __forceinline__ bool in_slot(const BaArgs& a, int r, int s) { return a.used[r] && a.slot_of[a.cams[r]] == s; }

__global__ void __launch_bounds__(kBaCta) ba_count_kernel(BaArgs a) {
  __shared__ int sh[kBaCta / 32];
  const int s = blockIdx.x;
  int c = 0;
  for (int r = threadIdx.x; r < a.obs; r += kBaCta) c += in_slot(a, r, s) ? 1 : 0;
  c = block_sum_int(c, sh);
  if (threadIdx.x == 0) a.counts[s] = c;
}

__global__ void __launch_bounds__(kBaCta) ba_list_kernel(BaArgs a) {
  __shared__ int warp_n[kBaCta / 32];
  const int s = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int base = 0;
  for (int q = 0; q < s; ++q) base += a.counts[q];
  if (threadIdx.x == 0) {
    a.list_off[s] = base;
    if (s == a.n_free - 1) a.list_off[a.n_free] = base + a.counts[s];
  }
  for (int c0 = 0; c0 < a.obs; c0 += kBaCta) {
    const int r = c0 + threadIdx.x;
    const bool f = r < a.obs && in_slot(a, r, s);
    const unsigned bal = __ballot_sync(kFull, f);
    if (lane == 0) warp_n[wid] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int q = 0; q < kBaCta / 32; ++q) {
      before += q < wid ? warp_n[q] : 0;
      total += warp_n[q];
    }
    if (f) a.list[base + before + __popc(bal & ((1u << lane) - 1u))] = r;
    base += total;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kBaCta) ba_init_kernel(BaArgs a) { ba_init_state(a); }

// ---------------------------------------------------------------------------------------------- one trial step
__global__ void __launch_bounds__(kBaThreads) ba_linearise_kernel(BaArgs a) {
  const BaState* st = a.state;
  if (st->stop || !st->lin) return;
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kBaWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks || a.trk_used[j] == 0) return;   // (warp-uniform)
  const int cur = st->cur;
  const double* X = point_of(a, cur, j);
  const int b = a.offsets[j], e = a.offsets[j + 1];
  double V[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
  for (int r = b + lane; r < e; r += 32) {
    if (!a.used[r]) continue;
    const int cm = a.cams[r];
    double* o = a.obsd + dg::kBaObsStride * (size_t)r;
    double Jx[6];
    dg::ba_jacobian(pose_of(a, cur, cm), a.tab + dg::kTrCamStride * (size_t)cm + dg::kTrCamK, X, a.pts[2 * (size_t)r],
                    a.pts[2 * (size_t)r + 1], o + dg::kBaObsR, o + dg::kBaObsJc, Jx);
    const double* rr = o + dg::kBaObsR;
    const double w = dg::ba_weight(rr[0] * rr[0] + rr[1] * rr[1], a.sig2);
    o[dg::kBaObsW] = w;
    dg::ba_point_terms(Jx, rr, w, V, g);
    if (a.slot_of[cm] >= 0) dg::ba_cross_block(o + dg::kBaObsJc, Jx, w, o + dg::kBaObsWm);
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

__global__ void __launch_bounds__(kBaThreads) ba_points_kernel(BaArgs a) {
  BaState* st = a.state;
  if (st->stop) return;
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kBaWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks || a.trk_used[j] == 0) return;   // (warp-uniform)
  double* tk = a.trk + dg::kBaTrkStride * (size_t)j;
  double Vi[6];
  if (!dg::ba_inv3(tk + dg::kBaTrkV, st->lam, Vi)) {
    if (lane == 0) st->bad = 1;                        // the step is rejected
    return;
  }
  if (lane < 6) tk[dg::kBaTrkVi + lane] = Vi[lane];
  const int b = a.offsets[j], e = a.offsets[j + 1];
  for (int r = b + lane; r < e; r += 32) {
    if (!a.used[r] || a.slot_of[a.cams[r]] < 0) continue;
    double* o = a.obsd + dg::kBaObsStride * (size_t)r;
    dg::ba_schur_row(o + dg::kBaObsWm, Vi, o + dg::kBaObsY);
  }
}

// S[row][col] = v, with the held coordinate's row and column replaced by those of the identity
__device__ __forceinline__ void put_s(const BaArgs& a, int hold, int row, int col, double v) {
  if (row == hold || col == hold) v = row == col ? 1.0 : 0.0;
  a.S[(size_t)row * a.n + col] = v;
}

__global__ void __launch_bounds__(kBaThreads) ba_schur_kernel(BaArgs a) {
  const BaState* st = a.state;
  if (st->stop || st->bad) return;
  const int lane = threadIdx.x & 31;
  const int q = blockIdx.x * kBaWarps + (threadIdx.x >> 5);
  if (q >= a.n_blocks) return;                         // (warp-uniform)
  int A = 0, rem = q;                                  // block q of the upper triangle, by rows
  while (rem >= a.n_free - A) { rem -= a.n_free - A; ++A; }
  const int B = A + rem;
  const int hold = st->hold_row;
  const int r0 = dg::kBaCamParams * A, c0 = dg::kBaCamParams * B;
  if (!slot_active(a, A) || !slot_active(a, B)) {      // a camera without used observations is held: identity rows
    for (int m = lane; m < 36; m += 32) {
      const int k = m / 6, l = m % 6;
      const double v = (A == B && k == l) ? 1.0 : 0.0;
      a.S[(size_t)(r0 + k) * a.n + c0 + l] = v;
      if (A != B) a.S[(size_t)(c0 + l) * a.n + r0 + k] = v;
      if (A == B && l == 0) a.rhs[r0 + k] = 0.0;
    }
    return;
  }
  const int la0 = a.list_off[A], la1 = a.list_off[A + 1];
  if (A == B) {                                        // U*_a and the reduced right-hand side
    double U[21], h[6];
#pragma unroll
    for (int s = 0; s < 21; ++s) U[s] = 0.0;
#pragma unroll
    for (int s = 0; s < 6; ++s) h[s] = 0.0;
    for (int i = la0 + lane; i < la1; i += 32) {
      const int r = a.list[i];
      const double* o = a.obsd + dg::kBaObsStride * (size_t)r;
      const double* Jc = o + dg::kBaObsJc;
      const double w = o[dg::kBaObsW], e0 = o[dg::kBaObsR], e1 = o[dg::kBaObsR + 1];
      const double* gp = a.trk + dg::kBaTrkStride * (size_t)a.track_of[r] + dg::kBaTrkG;
      const double* Y = o + dg::kBaObsY;
      int m = 0;
#pragma unroll
      for (int k = 0; k < 6; ++k)
#pragma unroll
        for (int l = k; l < 6; ++l) U[m++] += w * (Jc[k] * Jc[l] + Jc[6 + k] * Jc[6 + l]);
#pragma unroll
      for (int k = 0; k < 6; ++k)
        h[k] += w * (Jc[k] * e0 + Jc[6 + k] * e1) - (Y[3 * k] * gp[0] + Y[3 * k + 1] * gp[1] + Y[3 * k + 2] * gp[2]);
    }
#pragma unroll
    for (int s = 0; s < 21; ++s) U[s] = warp_sum(U[s]);
#pragma unroll
    for (int s = 0; s < 6; ++s) h[s] = warp_sum(h[s]);
    if (lane == 0) {
      const double lam = st->lam;
      int m = 0;
#pragma unroll
      for (int k = 0; k < 6; ++k)
#pragma unroll
        for (int l = k; l < 6; ++l, ++m) {
          const double v = k == l ? U[m] + lam * U[m] : U[m];
          a.S[(size_t)(r0 + k) * a.n + r0 + l] = v;
          a.S[(size_t)(r0 + l) * a.n + r0 + k] = v;
        }
#pragma unroll
      for (int k = 0; k < 6; ++k) a.rhs[r0 + k] = r0 + k == hold ? 0.0 : -h[k];
    }
  }
  // - sum over the pairs (i in slot a, k from camera b in i's track) of Y_i W_k^T
  double M[36];
#pragma unroll
  for (int s = 0; s < 36; ++s) M[s] = 0.0;
  const int cb = a.free[B];
  for (int i = la0 + lane; i < la1; i += 32) {
    const int r = a.list[i];
    const int p = a.track_of[r];
    const double* Y = a.obsd + dg::kBaObsStride * (size_t)r + dg::kBaObsY;
    const int e = a.offsets[p + 1];
    for (int k = a.offsets[p]; k < e; ++k) {
      if (!a.used[k] || a.cams[k] != cb) continue;
      const double* W = a.obsd + dg::kBaObsStride * (size_t)k + dg::kBaObsWm;
#pragma unroll
      for (int kk = 0; kk < 6; ++kk)
#pragma unroll
        for (int l = 0; l < 6; ++l)
          M[6 * kk + l] += Y[3 * kk] * W[3 * l] + Y[3 * kk + 1] * W[3 * l + 1] + Y[3 * kk + 2] * W[3 * l + 2];
    }
  }
#pragma unroll
  for (int s = 0; s < 36; ++s) M[s] = warp_sum(M[s]);
  __syncwarp();                                        // lane 0's U*_a is written
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 6; ++k)
#pragma unroll
      for (int l = 0; l < 6; ++l) {
        const double base = A == B ? a.S[(size_t)(r0 + k) * a.n + c0 + l] : 0.0;
        const double v = base - M[6 * k + l];
        put_s(a, hold, r0 + k, c0 + l, v);
        if (A != B) put_s(a, hold, c0 + l, r0 + k, v);
      }
  }
}

// Dense Cholesky S = L L^T in place (lower triangle, right-looking, one column at a time), L y = rhs, L^T dc = y, then
// the trial poses of the free cameras
__global__ void __launch_bounds__(kBaCta) ba_solve_kernel(BaArgs a) {
  BaState* st = a.state;
  if (st->stop || st->bad) return;
  __shared__ double col[dg::kBaMaxN];
  __shared__ double vec[dg::kBaMaxN];
  __shared__ int fail;
  const int n = a.n, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  double* S = a.S;
  for (int j = 0; j < n; ++j) {
    if (tid == 0) {
      const double d = S[(size_t)j * n + j];
      fail = !(d > 0.0);
      col[j] = sqrt(d);
      S[(size_t)j * n + j] = col[j];
    }
    __syncthreads();
    if (fail) {                                        // (block-uniform)
      if (tid == 0) st->bad = 1;
      return;
    }
    for (int i = j + 1 + tid; i < n; i += kBaCta) {
      const double v = S[(size_t)i * n + j] / col[j];
      S[(size_t)i * n + j] = v;
      col[i] = v;
    }
    __syncthreads();
    for (int i = j + 1 + wid; i < n; i += kBaCta / 32) {
      const double li = col[i];
      double* row = S + (size_t)i * n;
      for (int k = j + 1 + lane; k <= i; k += 32) row[k] -= li * col[k];
    }
    __syncthreads();
  }
  for (int i = tid; i < n; i += kBaCta) vec[i] = a.rhs[i];
  __syncthreads();
  for (int j = 0; j < n; ++j) {
    if (tid == 0) vec[j] = vec[j] / S[(size_t)j * n + j];
    __syncthreads();
    for (int i = j + 1 + tid; i < n; i += kBaCta) vec[i] -= S[(size_t)i * n + j] * vec[j];
    __syncthreads();
  }
  for (int j = n - 1; j >= 0; --j) {
    if (tid == 0) vec[j] = vec[j] / S[(size_t)j * n + j];
    __syncthreads();
    for (int i = tid; i < j; i += kBaCta) vec[i] -= S[(size_t)j * n + i] * vec[j];
    __syncthreads();
  }
  for (int i = tid; i < n; i += kBaCta) a.rhs[i] = vec[i];   // dc, read by ba_backsub_kernel
  const int cur = st->cur;
  if (tid < a.n_free && slot_active(a, tid)) {
    const int c = a.free[tid];
    double P2[12];
    dg::ap_step(pose_of(a, cur, c), vec + dg::kBaCamParams * tid, P2);
    if (dg::pr_ortho_drift(P2) > dg::kPrOrthoTol) dg::pr_orthonormalise(P2);
    double* out = a.poses + 12 * ((size_t)(1 - cur) * a.n_cams + c);
    for (int i = 0; i < 12; ++i) out[i] = P2[i];
  }
}

__global__ void __launch_bounds__(kBaThreads) ba_backsub_kernel(BaArgs a) {
  const BaState* st = a.state;
  if (st->stop || st->bad) return;
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kBaWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks || a.trk_used[j] == 0) return;   // (warp-uniform)
  const int cur = st->cur, b = a.offsets[j], e = a.offsets[j + 1];
  const double* dc = a.rhs;
  double acc[3] = {0.0, 0.0, 0.0};
  for (int r = b + lane; r < e; r += 32) {
    if (!a.used[r]) continue;
    const int s = a.slot_of[a.cams[r]];
    if (s < 0 || !slot_active(a, s)) continue;
    const double* W = a.obsd + dg::kBaObsStride * (size_t)r + dg::kBaObsWm;
    const double* d = dc + dg::kBaCamParams * s;
#pragma unroll
    for (int m = 0; m < 3; ++m)
#pragma unroll
      for (int k = 0; k < 6; ++k) acc[m] += W[3 * k + m] * d[k];
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

__global__ void __launch_bounds__(kBaCta) ba_decide_kernel(BaArgs a) {
  __shared__ double shd[kBaCta];
  if (a.state->stop) return;                           // (block-uniform)
  ba_decide_step(a, shd);
}

// ---------------------------------------------------------------------------------------------- outputs
__global__ void __launch_bounds__(kBaCamThreads) ba_finish_cameras_kernel(BaArgs a) {
  ba_finish_camera(a, blockIdx.x * kBaCamThreads + threadIdx.x);
}

__global__ void __launch_bounds__(kBaThreads) ba_finish_tracks_kernel(BaArgs a) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kBaWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks) return;
  ba_finish_track(a, j, lane);
}

}  // namespace

extern "C" {

const char* dgb200_bundle_adjust_last_error(void) { return g_err; }

int dgb200_bundle_adjust_ragged_dev(const int32_t* d_cams, const double* d_pts, const double* d_R, const double* d_t,
                                    const double* d_K, int k_per_camera, int n_cams, const int32_t* d_offsets,
                                    int n_tracks, int obs, const double* d_X, const uint8_t* d_mask,
                                    const int32_t* h_free, int n_free, int scale_gauge, double loss_scale,
                                    int max_iters, double px_th, double* d_R_out, double* d_t_out, double* d_X_out,
                                    uint8_t* d_mask_out, double* d_cost0_out, double* d_cost_out,
                                    int32_t* d_iters_out, int32_t* d_n_used_out, void* stream) {
  int gauge_slot = -1, held_cam = -1;
  const char* bad = ba_arg_error(!d_R || !d_t || !d_K || !d_offsets || !d_X || !d_R_out || !d_t_out || !d_X_out ||
                                     !d_cost0_out || !d_cost_out || !d_iters_out || !d_n_used_out,
                                 !d_cams || !d_pts || !d_mask_out, n_tracks, obs, n_cams, h_free, n_free,
                                 dg::kBaMaxFree, "n_free must lie in [0, 64]", scale_gauge, loss_scale, max_iters, px_th,
                                 &gauge_slot, &held_cam);
  if (bad) return fail(DGB200_E_ARG, bad);
  const cudaStream_t st = (cudaStream_t)stream;
  const int n = dg::kBaCamParams * n_free;
  const size_t no = (size_t)(obs > 0 ? obs : 1), nt = (size_t)n_tracks, nc = (size_t)n_cams;
  const size_t nn = (size_t)(n > 0 ? n : 1);
  BaArgs a;
  a.cams = d_cams; a.pts = d_pts; a.R = d_R; a.t = d_t; a.K = d_K; a.k_per_camera = k_per_camera; a.n_cams = n_cams;
  a.offsets = d_offsets; a.mask = d_mask; a.X = d_X; a.n_tracks = n_tracks; a.obs = obs; a.n_free = n_free; a.n = n;
  a.gauge_slot = gauge_slot; a.held_cam = held_cam; a.n_blocks = n_free * (n_free + 1) / 2;
  for (int q = 0; q < dg::kBaMaxFree; ++q) a.free[q] = q < n_free ? h_free[q] : -1;
  a.sig2 = loss_scale * loss_scale; a.th2 = px_th * px_th;
  auto lay_out = [&](char* base) {
    Carve w{base};
    a.tab = w.take<double>(dg::kTrCamStride * nc);
    a.poses = w.take<double>(24 * nc);
    a.Xb = w.take<double>(6 * nt);
    a.obsd = w.take<double>(dg::kBaObsStride * no);
    a.trk = w.take<double>(dg::kBaTrkStride * nt);
    a.S = w.take<double>(nn * nn);
    a.rhs = w.take<double>(nn);
    a.state = w.take<BaState>(1);
    a.slot_of = w.take<int>(nc);
    a.track_of = w.take<int>(no);
    a.list = w.take<int>(no);
    a.counts = w.take<int>(n_free + 1);
    a.list_off = w.take<int>(n_free + 1);
    a.trk_used = w.take<int>(nt);
    a.usable = w.take<unsigned char>(no);
    a.used = w.take<unsigned char>(no);
    return w.bytes;
  };
  char* ws = nullptr;
  const size_t bytes = lay_out(nullptr);
  CU(cudaMallocAsync((void**)&ws, bytes, st));
  lay_out(ws);
  a.R_out = d_R_out; a.t_out = d_t_out; a.X_out = d_X_out; a.mask_out = d_mask_out;
  a.cost0_out = d_cost0_out; a.cost_out = d_cost_out; a.iters_out = d_iters_out; a.n_used_out = d_n_used_out;
  const int cam_grid = blocks(nc, kBaCamThreads);
  const int trk_grid = blocks(nt, kBaWarps);
  cudaError_t launch = cudaSuccess;
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.usable, 0, no, st));   // rows outside every span are neither usable nor used
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.used, 0, no, st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.list_off, 0, sizeof(int) * (n_free + 1), st));
  ADJ_LAUNCH((ba_cameras_kernel<<<cam_grid, kBaCamThreads, 0, st>>>(a)));
  ADJ_LAUNCH((ba_mark_kernel<<<trk_grid, kBaThreads, 0, st>>>(a)));
  if (n_free > 0) {
    ADJ_LAUNCH((ba_count_kernel<<<n_free, kBaCta, 0, st>>>(a)));
    ADJ_LAUNCH((ba_list_kernel<<<n_free, kBaCta, 0, st>>>(a)));
  }
  ADJ_LAUNCH((ba_init_kernel<<<1, kBaCta, 0, st>>>(a)));
  const int schur_grid = blocks((size_t)a.n_blocks, kBaWarps);
  for (int it = 0; it < max_iters && launch == cudaSuccess; ++it) {
    ADJ_LAUNCH((ba_linearise_kernel<<<trk_grid, kBaThreads, 0, st>>>(a)));
    ADJ_LAUNCH((ba_points_kernel<<<trk_grid, kBaThreads, 0, st>>>(a)));
    if (n_free > 0) {
      ADJ_LAUNCH((ba_schur_kernel<<<schur_grid, kBaThreads, 0, st>>>(a)));
      ADJ_LAUNCH((ba_solve_kernel<<<1, kBaCta, 0, st>>>(a)));
    }
    ADJ_LAUNCH((ba_backsub_kernel<<<trk_grid, kBaThreads, 0, st>>>(a)));
    ADJ_LAUNCH((ba_decide_kernel<<<1, kBaCta, 0, st>>>(a)));
  }
  if (obs > 0) ADJ_LAUNCH(launch = cudaMemsetAsync(d_mask_out, 0, (size_t)obs, st));   // rows outside every span
  ADJ_LAUNCH((ba_finish_cameras_kernel<<<cam_grid, kBaCamThreads, 0, st>>>(a)));
  ADJ_LAUNCH((ba_finish_tracks_kernel<<<trk_grid, kBaThreads, 0, st>>>(a)));
  CU(cudaFreeAsync(ws, st));
  CU(launch);
  return 0;
}

}  // extern "C"
