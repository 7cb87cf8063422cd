// absolute_pose.cu -- registering a view against known 3D points, device resident: P3P MSAC-RANSAC with local
// optimisation over ragged batches of 2D-3D correspondences (what cv2.solvePnPRansac does for one view on the host).
// A translation unit of its own, so that adding it changes no instruction of the kernels in degensac_b200.cu and
// frontend.cu.
//
// One CTA of kApThreads per pair.
//   usable rows  an ordered block scan lists the pair's rows with mask != 0 and five finite coordinates, in row order,
//                in a workspace of the call; sampling and scoring see only that list (n entries).
//   RANSAC       waves of kApWarps iterations: warp w owns iteration k0 + w.  Lane 0 draws dg::minimal_sample<3>,
//                forms the bearings and solves Lambda Twist (p3p.h, 0 to 4 poses); the 32 lanes then score every pose
//                in one pass over the list (FP64 MSAC sums, lane l taking entries l, l + 32, ..., then a butterfly
//                over the warp: a fixed order that does not depend on the wave width).  Thread 0 then applies the
//                sequential rule to the wave in iteration order and drops everything after the stop.
//   LO           up to kApLoRounds rounds of Levenberg-Marquardt on the inliers (6 parameters, the schedule of
//                pose_refine_ragged_kernel) and re-selection of the inliers, with block-wide passes reduced in a
//                fixed order; kept when its MSAC cost is at most the RANSAC pose's.
// The inlier flags of the pose being optimised live in the output mask; the last pass writes the output's flags.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/degensac_b200.h"
#include "entry_error.h"
#include "common.h"
#include "rng.h"
#include "p3p.h"
#include "absolute_pose.h"
#include "device_util.h"

namespace {

thread_local char g_err[256] = "";
int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err, code, what, e); }

constexpr int kApThreads = 128;
constexpr int kApWarps = kApThreads / 32;     // the wave width: iterations evaluated side by side

struct AbsPoseArgs {
  const double* x; const double* X; const double* K;      // [rows][2], [rows][3]; K [9] shared or [P][9]
  int k_per_pair;
  const int* offsets; const unsigned char* mask;           // [P+1], [rows] or null
  int n_pairs, rows, max_iters, refine_iters;
  double th2, conf;
  const uint64_t* seeds;                                   // [P]
  int* list;                                               // [rows] workspace: the usable rows of each pair's span
  double* R_out; double* t_out; unsigned char* mask_out;   // [P][9], [P][3], [rows]
  int* n_inliers; int* iters; double* cost0; double* cost; // [P]
};

// Exclusive rank of `flag` among the CTA's threads in thread order, and the CTA's total in *total.  Called by all
// threads; two barriers.
__device__ __forceinline__ int block_rank(bool flag, int* wsum, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned b = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) wsum[wid] = __popc(b);
  __syncthreads();
  int before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kApWarps; ++w) { before += w < wid ? wsum[w] : 0; all += wsum[w]; }
  __syncthreads();
  *total = all;
  return before + __popc(b & ((1u << lane) - 1u));
}

// Sum of per-thread values over the CTA in a fixed order (butterfly in each warp, then the warps in order); every
// thread gets it.  Two barriers.
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* wpart) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) wpart[wid] = v;
  __syncthreads();
  T s = wpart[0];
#pragma unroll
  for (int w = 1; w < kApWarps; ++w) s += wpart[w];
  __syncthreads();
  return s;
}

struct Select { double cost; int inliers, changed; };

// One pass over the usable rows under pose P: writes every row's inlier flag to mask_out, and returns the MSAC cost,
// the number of inliers and the number of flags that changed.
__device__ Select select_pass(const AbsPoseArgs& a, const int* list, int n, const double* P, const double* K,
                              double* dpart, int* ipart) {
  double c = 0.0;
  int inl = 0, chg = 0;
  for (int i = threadIdx.x; i < n; i += kApThreads) {
    const int r = list[i];
    bool in;
    c += dg::ap_msac(P, K, a.x[2 * (size_t)r], a.x[2 * (size_t)r + 1], a.X[3 * (size_t)r], a.X[3 * (size_t)r + 1],
                     a.X[3 * (size_t)r + 2], a.th2, &in);
    const unsigned char f = in ? 1 : 0;
    inl += f;
    chg += a.mask_out[r] != f;
    a.mask_out[r] = f;
  }
  Select s;
  s.cost = block_sum(c, dpart);
  s.inliers = block_sum(inl, ipart);
  s.changed = block_sum(chg, ipart);
  return s;
}

// One LM pass over the rows flagged in mask_out under pose P: the cost, J^T J and J^T r (dg::ap_row) summed over the
// CTA into out[kApSums] in a fixed order (butterfly in each warp, thread j < kApSums adds the warps' partials of sum j
// in warp order).  Called by all threads; ends with a barrier.
__device__ void lm_pass(const AbsPoseArgs& a, const int* list, int n, const double* P, const double* K,
                        double (*wpart)[dg::kApSums], double* out) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  double acc[dg::kApSums];
#pragma unroll
  for (int j = 0; j < dg::kApSums; ++j) acc[j] = 0.0;
  for (int i = tid; i < n; i += kApThreads) {
    const int r = list[i];
    if (!a.mask_out[r]) continue;
    dg::ap_row(P, K, a.x[2 * (size_t)r], a.x[2 * (size_t)r + 1], a.X[3 * (size_t)r], a.X[3 * (size_t)r + 1],
               a.X[3 * (size_t)r + 2], acc);
  }
#pragma unroll
  for (int j = 0; j < dg::kApSums; ++j)
    for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < dg::kApSums; ++j) wpart[wid][j] = acc[j];
  }
  __syncthreads();
  if (tid < dg::kApSums) {
    double s = wpart[0][tid];
    for (int w = 1; w < kApWarps; ++w) s += wpart[w][tid];
    out[tid] = s;
  }
  __syncthreads();
}

// Thread 0's trial step: solve (H + lam diag H) D = -g and move pose[0] to pose[1]; false when a pivot is not positive
__device__ __noinline__ bool lm_trial(const double* cur, double lam, const double* P, double* P2) {
  double D[dg::kApParams];
  if (!dg::pr_cholesky_solve<dg::kApParams>(cur + 1, cur + 1 + dg::kApParams * (dg::kApParams + 1) / 2, lam, D))
    return false;
  dg::ap_step(P, D, P2);
  return true;
}

// Lane 0's hypothesis generation for iteration k: the sample, its bearings and world points, Lambda Twist; the poses
// go to P [4][12], the count is returned.
__device__ __noinline__ int hypotheses(const AbsPoseArgs& a, const int* list, int n, uint64_t seed, int k,
                                       const double* Ki, double* P) {
  int sel[3];
  dg::minimal_sample<3>(seed, (uint32_t)k, n, sel);
  double y[9], X[9], R[36], t[12];
  for (int j = 0; j < 3; ++j) {
    const size_t r = (size_t)list[sel[j]];
    dg::ap_bearing(Ki, a.x[2 * r], a.x[2 * r + 1], y + 3 * j);
    X[3 * j] = a.X[3 * r]; X[3 * j + 1] = a.X[3 * r + 1]; X[3 * j + 2] = a.X[3 * r + 2];
  }
  const int ns = dg::p3p_lambda_twist(y, X, R, t);
  for (int s = 0; s < ns; ++s) {
    for (int i = 0; i < 9; ++i) P[12 * s + i] = R[9 * s + i];
    for (int i = 0; i < 3; ++i) P[12 * s + 9 + i] = t[3 * s + i];
  }
  return ns;
}

__global__ void __launch_bounds__(kApThreads) absolute_pose_ragged_kernel(AbsPoseArgs a) {
  __shared__ double sK[9], sKi[9];
  __shared__ double hyp[kApWarps][4 * 12];             // the poses of each warp's iteration
  __shared__ double hcost[kApWarps][4];
  __shared__ int hinl[kApWarps][4], hn[kApWarps];
  __shared__ double best[12], pose[2][12];             // the RANSAC pose; the LO's current and trial poses
  __shared__ double cur[dg::kApSums], trial[dg::kApSums];
  __shared__ double wpart[kApWarps][dg::kApSums];
  __shared__ double dpart[kApWarps];
  __shared__ int ipart[kApWarps];
  __shared__ double s_best_cost;
  __shared__ int s_best_inl, s_has_best, s_iters, s_stop, s_go;
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int b = a.offsets[p], e = a.offsets[p + 1];
  const bool span_ok = b >= 0 && b <= e && e <= a.rows;
  const int r0 = span_ok ? b : 0, len = span_ok ? e - b : 0;
  int* list = a.list + r0;
  // usable rows, in row order; every row of the span starts outside the mask
  int n = 0;
  for (int c = 0; c < len; c += kApThreads) {
    const int i = c + tid;
    bool ok = false;
    if (i < len) {
      const size_t r = (size_t)r0 + i;
      ok = (!a.mask || a.mask[r]) && finite(a.x[2 * r]) && finite(a.x[2 * r + 1]) && finite(a.X[3 * r]) &&
           finite(a.X[3 * r + 1]) && finite(a.X[3 * r + 2]);
      a.mask_out[r] = 0;
    }
    int total;
    const int rank = block_rank(ok, ipart, &total);
    if (ok) list[n + rank] = r0 + i;
    n += total;
  }
  if (tid < 9) sK[tid] = a.K[(a.k_per_pair ? (size_t)p * 9 : 0) + tid];
  if (tid == 0) { s_best_cost = INFINITY; s_best_inl = 0; s_has_best = 0; s_iters = 0; s_stop = 0; }
  __syncthreads();
  if (tid == 0) dg::ap_inv3(sK, sKi);
  __syncthreads();
  const uint64_t seed = a.seeds[p];
  // RANSAC: waves of kApWarps iterations, the sequential rule applied in iteration order
  if (n >= dg::kApMinRows) {
    for (int k0 = 1; !s_stop; k0 += kApWarps) {      // (block-uniform: s_stop changes between two barriers)
      const int k = k0 + wid;
      int ns = 0;
      if (k <= a.max_iters) {
        if (lane == 0) ns = hypotheses(a, list, n, seed, k, sKi, hyp[wid]);
        ns = __shfl_sync(0xffffffffu, ns, 0);
        __syncwarp();
        double c[4] = {0.0, 0.0, 0.0, 0.0};
        int q[4] = {0, 0, 0, 0};
        for (int i = lane; i < n; i += 32) {
          const size_t r = (size_t)list[i];
          const double x = a.x[2 * r], y = a.x[2 * r + 1], X = a.X[3 * r], Y = a.X[3 * r + 1], Z = a.X[3 * r + 2];
#pragma unroll
          for (int s = 0; s < 4; ++s) {
            if (s < ns) {
              bool in;
              c[s] += dg::ap_msac(hyp[wid] + 12 * s, sK, x, y, X, Y, Z, a.th2, &in);
              q[s] += in ? 1 : 0;
            }
          }
        }
#pragma unroll
        for (int s = 0; s < 4; ++s)
          for (int o = 16; o > 0; o >>= 1) {
            c[s] += __shfl_xor_sync(0xffffffffu, c[s], o);
            q[s] += __shfl_xor_sync(0xffffffffu, q[s], o);
          }
        if (lane == 0) {
          hn[wid] = ns;
#pragma unroll
          for (int s = 0; s < 4; ++s) { hcost[wid][s] = c[s]; hinl[wid][s] = q[s]; }
        }
      }
      __syncthreads();
      if (tid == 0) {
        for (int w = 0; w < kApWarps; ++w) {
          const int kw = k0 + w;                     // iteration kw runs: kw - 1 < N_req after iteration kw - 1
          for (int s = 0; s < hn[w]; ++s)
            if (hcost[w][s] < s_best_cost) {
              s_best_cost = hcost[w][s];
              s_best_inl = hinl[w][s];
              s_has_best = 1;
              for (int i = 0; i < 12; ++i) best[i] = hyp[w][12 * s + i];
            }
          s_iters = kw;
          const int req = dg::ap_required_iters(s_has_best != 0, s_best_inl, n, a.conf, a.max_iters, kw);
          if (!(kw < req)) { s_stop = 1; break; }
        }
      }
      __syncthreads();
    }
  }
  const bool has_best = s_has_best != 0;
  if (!has_best) {                                   // no usable model: n < 4, no pose found, or bad offsets
    if (tid < 9) a.R_out[(size_t)p * 9 + tid] = 0.0;
    if (tid < 3) a.t_out[(size_t)p * 3 + tid] = 0.0;
    if (tid == 0) {
      a.n_inliers[p] = 0;
      a.iters[p] = s_iters;
      a.cost0[p] = qnan();
      a.cost[p] = qnan();
    }
    return;
  }
  const double cost0 = s_best_cost;
  if (tid < 12) pose[0][tid] = best[tid];
  __syncthreads();
  Select sel = select_pass(a, list, n, best, sK, dpart, ipart);
  double cost = cost0;
  int inliers = sel.inliers;
  if (a.refine_iters > 0 && sel.inliers >= dg::kApMinRows) {
    for (int round = 0; round < dg::kApLoRounds; ++round) {
      // Levenberg-Marquardt on the rows flagged now, from pose[0]: the schedule of pose_refine_ragged_kernel
      lm_pass(a, list, n, pose[0], sK, wpart, cur);
      double lam = dg::kPrLambda0;
      int it = 0, accepted = 0;
      while (it < a.refine_iters) {                  // (block-uniform: every thread keeps the same lam, it)
        ++it;
        if (tid == 0) s_go = lm_trial(cur, lam, pose[0], pose[1]) ? 1 : 0;
        __syncthreads();
        const bool go = s_go != 0;
        if (go) lm_pass(a, list, n, pose[1], sK, wpart, trial);
        const double c_old = cur[0], c_new = trial[0];
        const bool better = go && c_new < c_old;
        const bool flat = go && fabs(c_old - c_new) < dg::kPrRelDecrease * c_old;
        __syncthreads();                             // s_go, cur[0], trial[0] are read: they may change
        if (better) {
          if (tid < dg::kApSums) cur[tid] = trial[tid];
          if (tid < 12) pose[0][tid] = pose[1][tid];
        }
        __syncthreads();
        if (better) {
          lam = fmax(lam / 10.0, dg::kPrLambdaMin);
          ++accepted;
          if (flat) break;
        } else {
          lam *= 10.0;
          if (flat || lam > dg::kPrLambdaMax) break;
        }
      }
      if (tid == 0 && accepted && dg::pr_ortho_drift(pose[0]) > dg::kPrOrthoTol) dg::pr_orthonormalise(pose[0]);
      __syncthreads();
      sel = select_pass(a, list, n, pose[0], sK, dpart, ipart);
      if (sel.changed == 0 || sel.inliers < dg::kApMinRows) break;
    }
    if (sel.cost <= cost0) {
      cost = sel.cost;
      inliers = sel.inliers;
    } else {                                         // the RANSAC pose stays: its flags go back to the mask
      if (tid < 12) pose[0][tid] = best[tid];
      inliers = select_pass(a, list, n, best, sK, dpart, ipart).inliers;
    }
  }
  __syncthreads();
  if (tid < 9) a.R_out[(size_t)p * 9 + tid] = pose[0][tid];
  if (tid < 3) a.t_out[(size_t)p * 3 + tid] = pose[0][9 + tid];
  if (tid == 0) {
    a.n_inliers[p] = inliers;
    a.iters[p] = s_iters;
    a.cost0[p] = cost0;
    a.cost[p] = cost;
  }
}

}  // namespace

extern "C" {

const char* dgb200_absolute_pose_last_error(void) { return g_err; }

int dgb200_find_absolute_pose_ragged_dev(const double* d_x, const double* d_X, const double* d_K, int k_per_pair,
                                         const int32_t* d_offsets, int n_pairs, int rows, const uint8_t* d_mask,
                                         double px_th, double conf, int max_iters, int refine_iters,
                                         const uint64_t* d_seeds, double* d_R_out, double* d_t_out,
                                         uint8_t* d_mask_out, int32_t* d_n_inliers_out, int32_t* d_iters_out,
                                         double* d_cost0_out, double* d_cost_out, void* stream) {
  if (!d_K || !d_offsets || !d_seeds || !d_R_out || !d_t_out || !d_n_inliers_out || !d_iters_out || !d_cost0_out ||
      !d_cost_out)
    return fail(DGB200_E_ARG, "null buffer");
  if (rows > 0 && (!d_x || !d_X || !d_mask_out)) return fail(DGB200_E_ARG, "null row buffer");
  if (n_pairs < 1 || rows < 0) return fail(DGB200_E_ARG, "need n_pairs >= 1 and rows >= 0");
  if (!(px_th > 0.0) || !(px_th < INFINITY)) return fail(DGB200_E_ARG, "px_th must be a positive number");
  if (!(conf > 0.0 && conf <= 1.0)) return fail(DGB200_E_ARG, "conf must lie in (0, 1]");
  if (max_iters < 1) return fail(DGB200_E_ARG, "max_iters must be at least 1");
  if (refine_iters < 0) return fail(DGB200_E_ARG, "refine_iters must not be negative");
  const cudaStream_t st = (cudaStream_t)stream;
  int* list = nullptr;
  CU(cudaMallocAsync((void**)&list, sizeof(int) * (size_t)(rows > 0 ? rows : 1), st));
  AbsPoseArgs a;
  a.x = d_x; a.X = d_X; a.K = d_K; a.k_per_pair = k_per_pair; a.offsets = d_offsets; a.mask = d_mask;
  a.n_pairs = n_pairs; a.rows = rows; a.max_iters = max_iters; a.refine_iters = refine_iters;
  a.th2 = px_th * px_th; a.conf = conf; a.seeds = d_seeds; a.list = list;
  a.R_out = d_R_out; a.t_out = d_t_out; a.mask_out = d_mask_out; a.n_inliers = d_n_inliers_out; a.iters = d_iters_out;
  a.cost0 = d_cost0_out; a.cost = d_cost_out;
  absolute_pose_ragged_kernel<<<n_pairs, kApThreads, 0, st>>>(a);
  const cudaError_t launch = cudaGetLastError();
  CU(cudaFreeAsync(list, st));
  CU(launch);
  return 0;
}

}  // extern "C"
