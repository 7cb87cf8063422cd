// bundle_adjust_device.h -- the kernel bodies that the dense bundle adjustment (bundle_adjust.cu) and the iterative one
// (bundle_adjust_pcg.cu) share, with the one that also refines the intrinsics (bundle_adjust_intrinsics.cu): the LM
// state, the fixed-order CTA sums, the counting sort of the observations (not bundle_adjust.cu), the marking of the
// usable observations and optimised tracks, the start state, the step decision and the outputs.  Device code, in the anonymous namespace of the
// including translation unit (after device_util.h), as each kernel source keeps its own.
//
// The templates take the translation unit's argument block A, which has the members used here with the meaning they
// have in bundle_adjust.cu's BaArgs: the inputs (cams, pts, mask, offsets, X, n_cams, n_tracks, obs, sig2, th2), the
// free list (free, gauge_slot, held_cam), the workspace (tab, poses [2][n_cams][12], Xb [2][T][3], trk, usable, used,
// track_of, trk_used, state) and the outputs.  The marking and the output mask also take the camera model Cam: BaPinhole,
// the camera table's K, unless the caller passes its own (bundle_adjust_intrinsics.cu: the RADIAL model).
#pragma once
#include <cuda_runtime.h>

#include "bundle_adjust.h"
#include "pose_refine.h"
#include "triangulate.h"

namespace {

constexpr int kBaCta = 1024;                      // the one-CTA kernels

// The LM state of the call, in the workspace; only the start and the decision write it (bad: also the kernels that
// find a non-positive pivot)
struct BaState {
  double lam, cost, cost0;
  int cur, stop, lin, bad, iters, n_used, hold_row;
};

// The pinhole model of the camera table: an observation's residual r [2] and J_X [2][3] under pose P, and its e^2
struct BaPinhole {
  template <class A>
  static __device__ __forceinline__ void point_row(const A& a, const double* P, int cm, int /*buf*/, const double* X,
                                                   double x, double y, double* r, double* Jx) {
    double Jc[12];
    dg::ba_jacobian(P, a.tab + dg::kTrCamStride * (size_t)cm + dg::kTrCamK, X, x, y, r, Jc, Jx);
  }
  template <class A>
  static __device__ __forceinline__ double sq_error(const A& a, const double* P, int cm, int /*buf*/, const double* X,
                                                    double x, double y, bool* front) {
    return dg::ap_sq_error(P, a.tab + dg::kTrCamStride * (size_t)cm + dg::kTrCamK, x, y, X[0], X[1], X[2], front);
  }
};

__device__ int block_sum_int(int v, int* sh) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = warp_sum(v);
  if (lane == 0) sh[wid] = v;
  __syncthreads();
  int total = 0;
  for (int q = 0; q < kBaCta / 32; ++q) total += sh[q];
  __syncthreads();
  return total;
}

// A fixed-order sum over the CTA: thread i adds its terms in turn, then a tree over the threads
__device__ double block_sum_double(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = kBaCta / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  const double total = sh[0];
  __syncthreads();
  return total;
}

// The one-digit stable counting sort of the observations by a key in [0, n_keys) (-1: left out), in three passes.
// Warp w owns observations [w range, (w + 1) range) and column w of hist [n_keys][n_ranges], so its updates need no
// atomics.  ba_sort_count: the counts; ba_sort_scan (one CTA of kBaCta threads, sh: kBaCta ints): their exclusive
// prefix sum in key-major order, in place, and list_off [n_keys + 1] the start of each key; ba_sort_scatter: pos_of
// [obs] the position of each observation in the key-major list, ascending observation order within a key, and item
// [position] = track_of of its observation.
__device__ __forceinline__ void ba_sort_count(const int* key, int obs, int range, int* hist, int n_ranges, int w,
                                              int lane) {
  const int r0 = w * range, r1 = min(r0 + range, obs);
  for (int c0 = r0; c0 < r1; c0 += 32) {
    const int r = c0 + lane;
    const int s = r < r1 ? key[r] : -1;
    const unsigned peers = __match_any_sync(kFull, s);
    if (s >= 0 && lane == __ffs(peers) - 1) hist[(size_t)s * n_ranges + w] += __popc(peers);
    __syncwarp();
  }
}

__device__ __forceinline__ void ba_sort_scan(int* hist, int n_keys, int n_ranges, int* list_off, int* sh) {
  const size_t n = (size_t)n_keys * n_ranges;
  const size_t per = (n + kBaCta - 1) / kBaCta;
  const size_t b = per * threadIdx.x, e = min(b + per, n);
  int sum = 0;
  for (size_t i = b; i < e; ++i) sum += hist[i];
  sh[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {                            // 1024 partial sums, scanned in order by one thread
    int run = 0;
    for (int q = 0; q < kBaCta; ++q) {
      const int v = sh[q];
      sh[q] = run;
      run += v;
    }
    list_off[n_keys] = run;
  }
  __syncthreads();
  int run = sh[threadIdx.x];
  for (size_t i = b; i < e; ++i) {
    const int v = hist[i];
    hist[i] = run;
    if (i % n_ranges == 0) list_off[i / n_ranges] = run;
    run += v;
  }
}

__device__ __forceinline__ void ba_sort_scatter(const int* key, int obs, int range, int* hist, int n_ranges,
                                                const int* track_of, int* pos_of, int* item, int w, int lane) {
  const int r0 = w * range, r1 = min(r0 + range, obs);
  for (int c0 = r0; c0 < r1; c0 += 32) {
    const int r = c0 + lane;
    const int s = r < r1 ? key[r] : -1;
    const unsigned peers = __match_any_sync(kFull, s);
    if (s >= 0) {
      int* cursor = hist + (size_t)s * n_ranges + w;
      const int base = *cursor;
      const int pos = base + __popc(peers & ((1u << lane) - 1u));
      pos_of[r] = pos;
      item[pos] = track_of[r];
      __syncwarp(peers);                               // every peer has read the cursor before the first one moves it
      if (lane == __ffs(peers) - 1) *cursor = base + __popc(peers);
    }
    __syncwarp();
  }
}

// One warp per track j: the usable observations, whether the track is optimised, its start cost, both point buffers
template <class A, class Cam = BaPinhole>
__device__ __forceinline__ void ba_mark_track(const A& a, int j, int lane) {
  const double X[3] = {a.X[3 * (size_t)j], a.X[3 * (size_t)j + 1], a.X[3 * (size_t)j + 2]};
  if (lane < 3) {
    a.Xb[3 * (size_t)j + lane] = X[lane];
    a.Xb[3 * ((size_t)a.n_tracks + j) + lane] = X[lane];
  }
  if (lane == 0) {
    a.trk_used[j] = 0;
    a.trk[dg::kBaTrkStride * (size_t)j + dg::kBaTrkCost] = 0.0;
  }
  const int b = a.offsets[j], e = a.offsets[j + 1];
  if (!(b >= 0 && b <= e && e <= a.obs)) return;     // malformed span: no row read or written
  const bool xok = finite(X[0]) && finite(X[1]) && finite(X[2]);
  // the usable observations; the camera of the first one and whether another camera sees the track too
  int first_cam = -1, n = 0;
  bool two = false;
  double V[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0}, cost = 0.0;
  for (int c0 = b; c0 < e; c0 += 32) {
    const int r = c0 + lane;
    bool ok = false;
    int cm = -1;
    if (r < e) {
      cm = a.cams[r];
      const double x = a.pts[2 * (size_t)r], y = a.pts[2 * (size_t)r + 1];
      ok = xok && (!a.mask || a.mask[r]) && cm >= 0 && cm < a.n_cams && finite(x) && finite(y) &&
           a.tab[dg::kTrCamStride * (size_t)cm + dg::kTrCamOk] != 0.0;
      if (ok) {
        const double* P = a.poses + 12 * (size_t)cm;
        double p[3];
        dg::ap_camera(P, X[0], X[1], X[2], p);
        ok = p[2] > 0.0;
        if (ok) {
          double rr[2], Jx[6];
          Cam::point_row(a, P, cm, 0, X, x, y, rr, Jx);
          const double e2 = rr[0] * rr[0] + rr[1] * rr[1];
          cost += dg::ba_rho(e2, a.sig2);
          dg::ba_point_terms(Jx, rr, dg::ba_weight(e2, a.sig2), V, g);
        }
      }
      a.usable[r] = ok ? 1 : 0;
    }
    const unsigned bal = __ballot_sync(kFull, ok);
    if (bal) {
      if (first_cam < 0) first_cam = __shfl_sync(kFull, cm, __ffs(bal) - 1);
      two = two || __any_sync(kFull, ok && cm != first_cam);
    }
    n += __popc(bal);
  }
#pragma unroll
  for (int s = 0; s < 6; ++s) V[s] = warp_sum(V[s]);
  cost = warp_sum(cost);
  double Vi[6];
  const bool opt = two && dg::ba_inv3(V, 0.0, Vi);
  __syncwarp();
  for (int r = b + lane; r < e; r += 32) {
    const unsigned char u = opt ? a.usable[r] : 0;
    a.used[r] = u;
    a.track_of[r] = j;
  }
  if (opt && lane == 0) {
    a.trk_used[j] = n;
    a.trk[dg::kBaTrkStride * (size_t)j + dg::kBaTrkCost] = cost;
  }
}

// One CTA of kBaCta threads: cost0 and n_used by fixed-order sums, the scale gauge's axis, the LM state
template <class A>
__device__ __forceinline__ void ba_init_state(const A& a) {
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
    int hold = -1;
    if (a.gauge_slot >= 0) {
      const int ax = dg::ba_gauge_axis(a.poses + 12 * (size_t)a.free[a.gauge_slot],
                                       a.tab + dg::kTrCamStride * (size_t)a.held_cam + dg::kTrCamC);
      hold = dg::kBaCamParams * a.gauge_slot + 3 + ax;
    }
    st->hold_row = hold;
  }
}

// One CTA of kBaCta threads (shd: kBaCta doubles of shared memory), once the call has not stopped (the kernel returns
// first when st->stop): the schedule of pose_refine_ragged_kernel on the summed cost of the tracks.
template <class A>
__device__ __forceinline__ void ba_decide_step(const A& a, double* shd) {
  BaState* st = a.state;
  const bool go = !st->bad;
  double c = 0.0;
  if (go)
    for (int j = threadIdx.x; j < a.n_tracks; j += kBaCta) c += a.trk[dg::kBaTrkStride * (size_t)j + dg::kBaTrkCost];
  c = block_sum_double(c, shd);                        // (every thread reads st before thread 0 writes it)
  if (threadIdx.x == 0) {
    const double c_old = st->cost, c_new = go ? c : c_old;
    const bool better = go && c_new < c_old;
    const bool flat = go && fabs(c_old - c_new) < dg::kPrRelDecrease * c_old;
    st->iters += 1;
    st->bad = 0;
    if (better) {
      st->cost = c_new;
      st->cur = 1 - st->cur;
      st->lam = fmax(st->lam / 10.0, dg::kPrLambdaMin);
      st->lin = 1;
      if (flat) st->stop = 1;
    } else {
      st->lin = 0;
      st->lam *= 10.0;
      if (flat || st->lam > dg::kPrLambdaMax) st->stop = 1;
    }
  }
}

// Camera c's output pose, and the scalars (c = 0)
template <class A>
__device__ __forceinline__ void ba_finish_camera(const A& a, int c) {
  const BaState* st = a.state;
  if (c == 0) {
    a.cost0_out[0] = st->cost0;
    a.cost_out[0] = st->cost;
    a.iters_out[0] = st->iters;
    a.n_used_out[0] = st->n_used;
  }
  if (c >= a.n_cams) return;
  const double* P = a.poses + 12 * ((size_t)st->cur * a.n_cams + c);
  for (int i = 0; i < 9; ++i) a.R_out[9 * (size_t)c + i] = P[i];
  for (int i = 0; i < 3; ++i) a.t_out[3 * (size_t)c + i] = P[9 + i];
}

// One warp per track j: the output point and the track's rows of the output mask
template <class A, class Cam = BaPinhole>
__device__ __forceinline__ void ba_finish_track(const A& a, int j, int lane) {
  const int cur = a.state->cur;
  const double* X = a.Xb + 3 * ((size_t)cur * a.n_tracks + j);
  if (lane < 3) a.X_out[3 * (size_t)j + lane] = X[lane];
  const int b = a.offsets[j], e = a.offsets[j + 1];
  if (!(b >= 0 && b <= e && e <= a.obs)) return;
  for (int r = b + lane; r < e; r += 32) {
    unsigned char f = 0;
    if (a.usable[r]) {
      const int cm = a.cams[r];
      bool front;
      const double e2 = Cam::sq_error(a, a.poses + 12 * ((size_t)cur * a.n_cams + cm), cm, cur, X,
                                      a.pts[2 * (size_t)r], a.pts[2 * (size_t)r + 1], &front);
      f = front && e2 <= a.th2 ? 1 : 0;
    }
    a.mask_out[r] = f;
  }
}

}  // namespace
