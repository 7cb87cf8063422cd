// triangulate.cu -- multi-view triangulation of tracks across registered views, device resident: two-ray midpoint
// MSAC-RANSAC with local optimisation over ragged batches of tracks (what an incremental reconstruction does track by
// track on the host after registering a view).  A translation unit of its own, so that adding it changes no
// instruction of the kernels in degensac_b200.cu, frontend.cu and absolute_pose.cu.
//
//   cameras      triangulate_cameras_kernel writes one row of the camera table per camera (triangulate.h: the pose, K,
//                K^-1, the centre, whether it is registered) into the call's workspace.
//   tracks       triangulate_tracks_ragged_kernel: one warp per track, kTrWarps warps per CTA; warps never wait for
//                each other, so a track's result does not depend on the warp or CTA it lands in.
//     usable     a ballot scan lists the track's usable observations in row order in the workspace (n entries);
//                hypotheses and scores see only that list.
//     RANSAC     waves of 32 iterations: lane l owns iteration k0 + l, builds its hypothesis (the l-th pair after the
//                wave's first in lexicographic order, or a Philox sample) and scores it over the list sequentially.
//                The warp then applies the sequential rule in iteration order, every lane keeping the same state, and
//                drops everything after the stop: the result does not depend on the wave width.
//     LO         up to kTrLoRounds rounds of Levenberg-Marquardt on the inliers (3 parameters, the schedule of
//                pose_refine_ragged_kernel) and re-selection; lanes take the observations l, l + 32, ... and the
//                sums are reduced by a butterfly, a fixed order; kept when its MSAC cost is at most the RANSAC point's.
// The inlier flags of the point being optimised live in the output mask; the last pass writes the output's flags.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/degensac_b200.h"
#include "entry_error.h"
#include "common.h"
#include "rng.h"
#include "absolute_pose.h"
#include "pose_refine.h"
#include "triangulate.h"
#include "device_util.h"

namespace {

thread_local char g_err[256] = "";
int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err, code, what, e); }

constexpr int kTrWarps = 4;                       // tracks per CTA, one per warp
constexpr int kTrThreads = 32 * kTrWarps;
constexpr int kTrCamThreads = 128;

struct TriArgs {
  const int* cams; const double* pts; const double* tab;   // [obs], [obs][2], camera table [n_cams][kTrCamStride]
  int n_cams;
  const int* offsets; const unsigned char* mask;           // [T+1], [obs] or null
  int n_tracks, obs, max_iters, refine_iters;
  double th2, cos_max, conf;
  const uint64_t* seeds;                                   // [T]
  int* list;                                               // [obs] workspace: the usable rows of each track's span
  double* X_out; unsigned char* mask_out;                  // [T][3], [obs]
  int* n_inliers; int* iters; double* cost0; double* cost; double* angle;   // [T]
};

__global__ void __launch_bounds__(kTrCamThreads) triangulate_cameras_kernel(const double* R, const double* t,
                                                                            const double* K, int k_per_camera,
                                                                            int n_cams, double* tab) {
  const int c = blockIdx.x * kTrCamThreads + threadIdx.x;
  if (c >= n_cams) return;
  dg::tr_camera(R + 9 * (size_t)c, t + 3 * (size_t)c, K + (k_per_camera ? 9 * (size_t)c : 0),
                tab + dg::kTrCamStride * (size_t)c);
}

struct Select { double cost; int inliers, changed; };

// One pass over the usable observations under point X: writes every row's inlier flag to mask_out, and returns the
// MSAC cost, the number of inliers and the number of flags that changed (the same in every lane).
__device__ Select select_pass(const TriArgs& a, const int* list, int n, const double* X) {
  double c = 0.0;
  int inl = 0, chg = 0;
  for (int i = threadIdx.x & 31; i < n; i += 32) {
    const size_t r = (size_t)list[i];
    bool in;
    c += dg::tr_msac(a.tab + dg::kTrCamStride * (size_t)a.cams[r], X, a.pts[2 * r], a.pts[2 * r + 1], a.th2, &in);
    const unsigned char f = in ? 1 : 0;
    inl += f;
    chg += a.mask_out[r] != f;
    a.mask_out[r] = f;
  }
  Select s;
  s.cost = warp_sum(c);
  s.inliers = warp_sum(inl);
  s.changed = warp_sum(chg);
  return s;
}

// One LM pass over the rows flagged in mask_out under point X: the cost, J^T J and J^T r (dg::tr_row), each summed
// over the warp by a butterfly; every lane gets out[kTrSums].
__device__ void lm_pass(const TriArgs& a, const int* list, int n, const double* X, double* out) {
#pragma unroll
  for (int s = 0; s < dg::kTrSums; ++s) out[s] = 0.0;
  for (int i = threadIdx.x & 31; i < n; i += 32) {
    const size_t r = (size_t)list[i];
    if (!a.mask_out[r]) continue;
    dg::tr_row(a.tab + dg::kTrCamStride * (size_t)a.cams[r], X, a.pts[2 * r], a.pts[2 * r + 1], out);
  }
#pragma unroll
  for (int s = 0; s < dg::kTrSums; ++s) out[s] = warp_sum(out[s]);
}

// Lane's hypothesis of list entries (i, j): false when both come from one camera or tr_midpoint gives none
__device__ bool hypothesis(const TriArgs& a, const int* list, int i, int j, double* X) {
  const size_t ri = (size_t)list[i], rj = (size_t)list[j];
  const int ci = a.cams[ri], cj = a.cams[rj];
  if (ci == cj) return false;
  const double* cam_i = a.tab + dg::kTrCamStride * (size_t)ci;
  const double* cam_j = a.tab + dg::kTrCamStride * (size_t)cj;
  double di[3], dj[3];
  dg::tr_ray(cam_i, a.pts[2 * ri], a.pts[2 * ri + 1], di);
  dg::tr_ray(cam_j, a.pts[2 * rj], a.pts[2 * rj + 1], dj);
  return dg::tr_midpoint(cam_i + dg::kTrCamC, di, cam_j + dg::kTrCamC, dj, a.cos_max, X);
}

__global__ void __launch_bounds__(kTrThreads) triangulate_tracks_ragged_kernel(TriArgs a) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * kTrWarps + (threadIdx.x >> 5);
  if (j >= a.n_tracks) return;                       // (warp-uniform)
  const int b = a.offsets[j], e = a.offsets[j + 1];
  if (!(b >= 0 && b <= e && e <= a.obs)) {           // malformed span: no model, no row read or written
    if (lane < 3) a.X_out[3 * (size_t)j + lane] = qnan();
    if (lane == 0) {
      a.n_inliers[j] = 0;
      a.iters[j] = 0;
      a.cost0[j] = qnan();
      a.cost[j] = qnan();
      a.angle[j] = qnan();
    }
    return;
  }
  const int len = e - b;
  int* list = a.list + b;
  // usable observations, in row order; every row of the span starts outside the mask
  int n = 0;
  for (int c = 0; c < len; c += 32) {
    const int i = c + lane;
    bool ok = false;
    if (i < len) {
      const size_t r = (size_t)b + i;
      const int cm = a.cams[r];
      ok = (!a.mask || a.mask[r]) && cm >= 0 && cm < a.n_cams && finite(a.pts[2 * r]) && finite(a.pts[2 * r + 1]) &&
           a.tab[dg::kTrCamStride * (size_t)cm + dg::kTrCamOk] != 0.0;
      a.mask_out[r] = 0;
    }
    const unsigned bal = __ballot_sync(kFull, ok);
    if (ok) list[n + __popc(bal & ((1u << lane) - 1u))] = b + i;
    n += __popc(bal);
  }
  __syncwarp();                                      // the list and the cleared flags are seen by every lane
  // RANSAC: waves of 32 iterations, the sequential rule applied in iteration order
  const long long pairs = (long long)n * (n - 1) / 2;
  const bool enumerate = pairs <= a.max_iters;
  const int kmax = enumerate ? (int)pairs : a.max_iters;
  const uint64_t seed = a.seeds[j];
  double best[3] = {0.0, 0.0, 0.0}, best_cost = INFINITY;
  int best_inl = 0, iters = 0, req = kmax;
  bool has_best = false;
  if (n >= dg::kTrMinRows) {
    int wi = 0, wj = 1;                              // the wave's first pair (enumeration)
    for (int k0 = 1, stop = 0; !stop; k0 += 32) {    // (warp-uniform: every lane keeps the same state)
      const int k = k0 + lane;
      bool valid = false;
      double c = 0.0, X[3] = {0.0, 0.0, 0.0};
      int q = 0;
      if (k <= kmax) {
        int sel[2] = {wi, wj};
        if (enumerate) dg::tr_pair_advance(n, lane, &sel[0], &sel[1]);
        else dg::minimal_sample<2>(seed, (uint32_t)k, n, sel);
        valid = hypothesis(a, list, sel[0], sel[1], X);
        if (valid) {
          for (int m = 0; m < n; ++m) {
            const size_t r = (size_t)list[m];
            bool in;
            c += dg::tr_msac(a.tab + dg::kTrCamStride * (size_t)a.cams[r], X, a.pts[2 * r], a.pts[2 * r + 1], a.th2,
                             &in);
            q += in ? 1 : 0;
          }
        }
      }
      for (int l = 0; l < 32; ++l) {
        const int kl = k0 + l;                       // iteration kl runs: kl - 1 < N_req after iteration kl - 1
        const bool vl = __shfl_sync(kFull, (int)valid, l) != 0;
        const double cl = __shfl_sync(kFull, c, l);
        if (vl && cl < best_cost) {                  // N_req changes only with the best point
          best_cost = cl;
          best_inl = __shfl_sync(kFull, q, l);
#pragma unroll
          for (int s = 0; s < 3; ++s) best[s] = __shfl_sync(kFull, X[s], l);
          has_best = true;
          req = dg::required_iters<2>(true, best_inl, n, a.conf, kmax, kl);
        }
        iters = kl;
        if (!(kl < req)) { stop = 1; break; }
      }
      if (enumerate) dg::tr_pair_advance(n, 32, &wi, &wj);
    }
  }
  if (!has_best) {                                   // no model: n < 2 or no valid hypothesis
    if (lane < 3) a.X_out[3 * (size_t)j + lane] = qnan();
    if (lane == 0) {
      a.n_inliers[j] = 0;
      a.iters[j] = iters;
      a.cost0[j] = qnan();
      a.cost[j] = qnan();
      a.angle[j] = qnan();
    }
    return;
  }
  const double cost0 = best_cost;
  double X[3] = {best[0], best[1], best[2]};
  Select sel = select_pass(a, list, n, X);
  double cost = cost0;
  int inliers = sel.inliers;
  if (a.refine_iters > 0 && sel.inliers >= dg::kTrMinRows) {
    for (int round = 0; round < dg::kTrLoRounds; ++round) {
      // Levenberg-Marquardt on the rows flagged now, from X: the schedule of pose_refine_ragged_kernel
      double cur[dg::kTrSums], trial[dg::kTrSums];
      lm_pass(a, list, n, X, cur);
      double lam = dg::kPrLambda0;
      for (int it = 0; it < a.refine_iters;) {
        ++it;
        double D[dg::kTrParams], X2[3];
        const bool go = dg::pr_cholesky_solve<dg::kTrParams>(cur + 1, cur + 1 + dg::kTrParams * (dg::kTrParams + 1) / 2,
                                                             lam, D);
        if (go) {
#pragma unroll
          for (int s = 0; s < 3; ++s) X2[s] = X[s] + D[s];
          lm_pass(a, list, n, X2, trial);
        }
        const double c_old = cur[0], c_new = go ? trial[0] : c_old;
        const bool better = go && c_new < c_old;
        const bool flat = go && fabs(c_old - c_new) < dg::kPrRelDecrease * c_old;
        if (better) {
#pragma unroll
          for (int s = 0; s < dg::kTrSums; ++s) cur[s] = trial[s];
#pragma unroll
          for (int s = 0; s < 3; ++s) X[s] = X2[s];
          lam = fmax(lam / 10.0, dg::kPrLambdaMin);
          if (flat) break;
        } else {
          lam *= 10.0;
          if (flat || lam > dg::kPrLambdaMax) break;
        }
      }
      sel = select_pass(a, list, n, X);
      if (sel.changed == 0 || sel.inliers < dg::kTrMinRows) break;
    }
    if (sel.cost <= cost0) {
      cost = sel.cost;
      inliers = sel.inliers;
    } else {                                         // the RANSAC point stays: its flags go back to the mask
#pragma unroll
      for (int s = 0; s < 3; ++s) X[s] = best[s];
      inliers = select_pass(a, list, n, X).inliers;
    }
  }
  __syncwarp();                                      // every lane reads the flags of the other lanes' rows
  // the largest triangulation angle at X over pairs of inliers from distinct cameras (0 without such a pair)
  double ang = 0.0;
  for (int i = lane; i < n; i += 32) {
    const size_t ri = (size_t)list[i];
    if (!a.mask_out[ri]) continue;
    const int ci = a.cams[ri];
    const double* Ci = a.tab + dg::kTrCamStride * (size_t)ci + dg::kTrCamC;
    const double u[3] = {X[0] - Ci[0], X[1] - Ci[1], X[2] - Ci[2]};
    for (int m = i + 1; m < n; ++m) {
      const size_t rm = (size_t)list[m];
      const int cm = a.cams[rm];
      if (!a.mask_out[rm] || cm == ci) continue;
      const double* Cm = a.tab + dg::kTrCamStride * (size_t)cm + dg::kTrCamC;
      const double v[3] = {X[0] - Cm[0], X[1] - Cm[1], X[2] - Cm[2]};
      double w[3];
      dg::cross3(w, u, v);
      ang = fmax(ang, atan2(sqrt(dg::tr_dot(w, w)), dg::tr_dot(u, v)));
    }
  }
  for (int o = 16; o > 0; o >>= 1) ang = fmax(ang, __shfl_xor_sync(kFull, ang, o));
  if (lane < 3) a.X_out[3 * (size_t)j + lane] = X[lane];
  if (lane == 0) {
    a.n_inliers[j] = inliers;
    a.iters[j] = iters;
    a.cost0[j] = cost0;
    a.cost[j] = cost;
    a.angle[j] = ang;
  }
}

}  // namespace

extern "C" {

const char* dgb200_triangulate_last_error(void) { return g_err; }

int dgb200_triangulate_tracks_ragged_dev(const int32_t* d_cams, const double* d_pts, const double* d_R,
                                         const double* d_t, const double* d_K, int k_per_camera, int n_cams,
                                         const int32_t* d_offsets, int n_tracks, int obs, const uint8_t* d_mask,
                                         double px_th, double min_angle, double conf, int max_iters, int refine_iters,
                                         const uint64_t* d_seeds, double* d_X_out, uint8_t* d_mask_out,
                                         int32_t* d_n_inliers_out, int32_t* d_iters_out, double* d_cost0_out,
                                         double* d_cost_out, double* d_angle_out, void* stream) {
  if (!d_R || !d_t || !d_K || !d_offsets || !d_seeds || !d_X_out || !d_n_inliers_out || !d_iters_out ||
      !d_cost0_out || !d_cost_out || !d_angle_out)
    return fail(DGB200_E_ARG, "null buffer");
  if (obs > 0 && (!d_cams || !d_pts || !d_mask_out)) return fail(DGB200_E_ARG, "null observation buffer");
  if (n_tracks < 1 || obs < 0 || n_cams < 1) return fail(DGB200_E_ARG, "need n_tracks >= 1, obs >= 0 and n_cams >= 1");
  if (!(px_th > 0.0) || !(px_th < INFINITY)) return fail(DGB200_E_ARG, "px_th must be a positive number");
  if (!(min_angle >= 0.0 && min_angle < M_PI)) return fail(DGB200_E_ARG, "min_angle must lie in [0, pi)");
  if (!(conf > 0.0 && conf <= 1.0)) return fail(DGB200_E_ARG, "conf must lie in (0, 1]");
  if (max_iters < 1) return fail(DGB200_E_ARG, "max_iters must be at least 1");
  if (refine_iters < 0) return fail(DGB200_E_ARG, "refine_iters must not be negative");
  const cudaStream_t st = (cudaStream_t)stream;
  const size_t tab_bytes = sizeof(double) * dg::kTrCamStride * (size_t)n_cams;
  char* ws = nullptr;
  CU(cudaMallocAsync((void**)&ws, tab_bytes + sizeof(int) * (size_t)(obs > 0 ? obs : 1), st));
  TriArgs a;
  a.cams = d_cams; a.pts = d_pts; a.tab = (const double*)ws; a.n_cams = n_cams; a.offsets = d_offsets; a.mask = d_mask;
  a.n_tracks = n_tracks; a.obs = obs; a.max_iters = max_iters; a.refine_iters = refine_iters;
  a.th2 = px_th * px_th; a.cos_max = cos(min_angle); a.conf = conf; a.seeds = d_seeds; a.list = (int*)(ws + tab_bytes);
  a.X_out = d_X_out; a.mask_out = d_mask_out; a.n_inliers = d_n_inliers_out; a.iters = d_iters_out;
  a.cost0 = d_cost0_out; a.cost = d_cost_out; a.angle = d_angle_out;
  triangulate_cameras_kernel<<<(n_cams + kTrCamThreads - 1) / kTrCamThreads, kTrCamThreads, 0, st>>>(
      d_R, d_t, d_K, k_per_camera, n_cams, (double*)ws);
  cudaError_t launch = cudaGetLastError();
  if (launch == cudaSuccess) {
    triangulate_tracks_ragged_kernel<<<(n_tracks + kTrWarps - 1) / kTrWarps, kTrThreads, 0, st>>>(a);
    launch = cudaGetLastError();
  }
  CU(cudaFreeAsync(ws, st));
  CU(launch);
  return 0;
}

}  // extern "C"
