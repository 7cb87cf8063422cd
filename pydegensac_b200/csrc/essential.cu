// essential.cu -- relative pose of calibrated image pairs, device resident: five-point MSAC-RANSAC with local
// optimisation over ragged batches of correspondences (what cv2.findEssentialMat does for one pair on the host).  A
// translation unit of its own, so that adding it changes no instruction of the other kernels.
//
// One CTA of kEsThreads per pair.
//   usable rows  an ordered block scan lists the pair's rows with mask != 0 and four finite coordinates, in row order,
//                in a workspace of the call; sampling and scoring see only that list (n entries).
//   RANSAC       waves of kEsWarps iterations: warp w owns iteration k0 + w.  Lane 0 draws dg::minimal_sample<5>,
//                normalises the sample by K1^-1 and K2^-1 and solves it (five_point.h, 0 to 10 essential matrices);
//                lanes s < ns form the calibrated F_s = K2^-T E_s K1^-1; the 32 lanes then score every F in one pass
//                over the list (FP64 MSAC sums of the Sampson error, lane l taking entries l, l + 32, ..., then a
//                butterfly over the warp: a fixed order that does not depend on the wave width).  Thread 0 then
//                applies the sequential rule to the wave in iteration order and drops everything after the stop.
//   LO           from one decomposition of the best E, up to kEsLoRounds rounds of Levenberg-Marquardt over (R, t) on
//                the inliers (refine_pose_ragged's rows, solve and step) and re-selection of the inliers, with
//                block-wide passes reduced in a fixed order; kept when its MSAC cost is at most the RANSAC model's.
// The inlier flags of the model being optimised live in the output mask; the last pass writes the output's flags.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/degensac_b200.h"
#include "entry_error.h"
#include "common.h"
#include "rng.h"
#include "essential.h"
#include "device_util.h"

namespace {

thread_local char g_err[256] = "";
int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err, code, what, e); }

constexpr int kEsThreads = 128;
constexpr int kEsWarps = kEsThreads / 32;     // the wave width: iterations evaluated side by side
constexpr int kEsMax = dg::kFpMaxSolutions;

struct EssentialArgs {
  const double* x1; const double* x2; const double* K1; const double* K2;   // [rows][2] each; K [9] or [P][9]
  int k_per_pair;
  const int* offsets; const unsigned char* mask;           // [P+1], [rows] or null
  int n_pairs, rows, max_iters, refine_iters;
  double th2, conf;
  const uint64_t* seeds;                                   // [P]
  int* list;                                               // [rows] workspace: the usable rows of each pair's span
  double* E_out; double* F_out; unsigned char* mask_out;   // [P][9], [P][9], [rows]
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
  for (int w = 0; w < kEsWarps; ++w) { before += w < wid ? wsum[w] : 0; all += wsum[w]; }
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
  for (int w = 1; w < kEsWarps; ++w) s += wpart[w];
  __syncthreads();
  return s;
}

struct Select { double cost; int inliers, changed; };

// One pass over the usable rows under F: writes every row's inlier flag to mask_out, and returns the MSAC cost, the
// number of inliers and the number of flags that changed.
__device__ Select select_pass(const EssentialArgs& a, const int* list, int n, const double* F, double* dpart,
                              int* ipart) {
  double c = 0.0;
  int inl = 0, chg = 0;
  for (int i = threadIdx.x; i < n; i += kEsThreads) {
    const size_t r = (size_t)list[i];
    bool in;
    c += dg::es_msac(F, a.x1[2 * r], a.x1[2 * r + 1], a.x2[2 * r], a.x2[2 * r + 1], a.th2, &in);
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

// One LM pass over the rows flagged in mask_out at the linearisation lin = (F [9], dF [5][9]): the cost, J^T J and
// J^T r (dg::pr_row) summed over the CTA into out[kPrSums] in a fixed order (butterfly in each warp, thread j < kPrSums
// adds the warps' partials of sum j in warp order).  Called by all threads; ends with a barrier.
__device__ void lm_pass(const EssentialArgs& a, const int* list, int n, const double* lin,
                        double (*wpart)[dg::kPrSums], double* out) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  double acc[dg::kPrSums];
#pragma unroll
  for (int j = 0; j < dg::kPrSums; ++j) acc[j] = 0.0;
  for (int i = tid; i < n; i += kEsThreads) {
    const size_t r = (size_t)list[i];
    if (!a.mask_out[r]) continue;
    dg::pr_row(lin, lin + 9, a.x1[2 * r], a.x1[2 * r + 1], a.x2[2 * r], a.x2[2 * r + 1], acc);
  }
#pragma unroll
  for (int j = 0; j < dg::kPrSums; ++j)
    for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < dg::kPrSums; ++j) wpart[wid][j] = acc[j];
  }
  __syncthreads();
  if (tid < dg::kPrSums) {
    double s = wpart[0][tid];
    for (int w = 1; w < kEsWarps; ++w) s += wpart[w][tid];
    out[tid] = s;
  }
  __syncthreads();
}

// Lane 0's hypothesis generation for iteration k: the sample, its normalised coordinates, the five-point solver; the
// essential matrices go to Es [10][9], their count is returned.
__device__ __noinline__ int hypotheses(const EssentialArgs& a, const int* list, int n, uint64_t seed, int k,
                                       const double* K1i, const double* K2i, double* Es) {
  int sel[5];
  dg::minimal_sample<5>(seed, (uint32_t)k, n, sel);
  double y1[15], y2[15];
  for (int j = 0; j < 5; ++j) {
    const size_t r = (size_t)list[sel[j]];
    dg::es_normalise(K1i, a.x1[2 * r], a.x1[2 * r + 1], y1 + 3 * j);
    dg::es_normalise(K2i, a.x2[2 * r], a.x2[2 * r + 1], y2 + 3 * j);
  }
  return dg::five_point(y1, y2, Es);
}

// Thread 0's pieces of the LO, kept out of line so that their frames stay out of the scoring loop's registers.
// lo_start: the start pose P [12] = (R, t) of E and its linearisation lin = (F, dF [5][9]); false for a rank < 2 E.
__device__ __noinline__ bool lo_start(const double* E, const double* A, const double* Bk, double* P, double* lin) {
  if (!dg::es_pose(E, P, P + 9)) return false;
  dg::pr_linearise(P, P + 9, A, Bk, lin, lin + 9);
  return true;
}

// lo_trial: solve (H + lam diag H) D = -g from the sums cur, move P to P2 and linearise there; false when a pivot is
// not positive
__device__ __noinline__ bool lo_trial(const double* cur, double lam, const double* P, const double* A, const double* Bk,
                                      double* P2, double* lin) {
  double D[5];
  if (!dg::pr_solve(cur + 1, cur + 16, lam, D)) return false;
  dg::pr_step(P, P + 9, D, P2, P2 + 9);
  dg::pr_linearise(P2, P2 + 9, A, Bk, lin, lin + 9);
  return true;
}

// lo_model: after a round, R re-orthonormalised when an accepted step left it off, the model (E [9], F [9]) of P and
// the linearisation of the next round
__device__ __noinline__ void lo_model(bool accepted, double* P, const double* A, const double* Bk, double* model,
                                      double* lin) {
  if (accepted && dg::pr_ortho_drift(P) > dg::kPrOrthoTol) dg::pr_orthonormalise(P);
  dg::es_essential(P, P + 9, model);
  dg::es_fundamental(model, A, Bk, model + 9);
  dg::pr_linearise(P, P + 9, A, Bk, lin, lin + 9);
}

__global__ void __launch_bounds__(kEsThreads) essential_ragged_kernel(EssentialArgs a) {
  __shared__ double sK1i[9], sK2i[9], sA[9];           // K1^-1, K2^-1, K2^-T
  __shared__ double hypE[kEsWarps][kEsMax * 9];        // the essential matrices of each warp's iteration
  __shared__ double hypF[kEsWarps][kEsMax * 9];        // and their calibrated F
  __shared__ double hcost[kEsWarps][kEsMax];
  __shared__ int hinl[kEsWarps][kEsMax], hn[kEsWarps];
  __shared__ double bestE[9], bestF[9];                // the RANSAC model
  __shared__ double pose[2][12];                       // the LO's current and trial (R [9], t [3])
  __shared__ double lin[54];                           // F [9], dF [5][9] of the LM pass to come
  __shared__ double model[18];                         // the LO's E [9] and F [9]
  __shared__ double cur[dg::kPrSums], trial[dg::kPrSums];
  __shared__ double wpart[kEsWarps][dg::kPrSums];
  __shared__ double dpart[kEsWarps];
  __shared__ int ipart[kEsWarps];
  __shared__ double s_best_cost;
  __shared__ int s_best_inl, s_has_best, s_iters, s_stop, s_go, s_pose;
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int b = a.offsets[p], e = a.offsets[p + 1];
  const bool span_ok = b >= 0 && b <= e && e <= a.rows;
  const int r0 = span_ok ? b : 0, len = span_ok ? e - b : 0;
  int* list = a.list + r0;
  // usable rows, in row order; every row of the span starts outside the mask
  int n = 0;
  for (int c = 0; c < len; c += kEsThreads) {
    const int i = c + tid;
    bool ok = false;
    if (i < len) {
      const size_t r = (size_t)r0 + i;
      ok = (!a.mask || a.mask[r]) && finite(a.x1[2 * r]) && finite(a.x1[2 * r + 1]) && finite(a.x2[2 * r]) &&
           finite(a.x2[2 * r + 1]);
      a.mask_out[r] = 0;
    }
    int total;
    const int rank = block_rank(ok, ipart, &total);
    if (ok) list[n + rank] = r0 + i;
    n += total;
  }
  if (tid < 9) sK1i[tid] = a.K1[(a.k_per_pair ? (size_t)p * 9 : 0) + tid];
  else if (tid < 18) sK2i[tid - 9] = a.K2[(a.k_per_pair ? (size_t)p * 9 : 0) + tid - 9];
  if (tid == 0) { s_best_cost = INFINITY; s_best_inl = 0; s_has_best = 0; s_iters = 0; s_stop = 0; }
  __syncthreads();
  if (tid == 0) {
    double K[9];
    for (int i = 0; i < 9; ++i) K[i] = sK1i[i];
    dg::ap_inv3(K, sK1i);
    for (int i = 0; i < 9; ++i) K[i] = sK2i[i];
    dg::ap_inv3(K, sK2i);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) sA[3 * i + j] = sK2i[3 * j + i];
  }
  __syncthreads();
  const uint64_t seed = a.seeds[p];
  // RANSAC: waves of kEsWarps iterations, the sequential rule applied in iteration order
  if (n >= dg::kEsMinRows) {
    for (int k0 = 1; !s_stop; k0 += kEsWarps) {      // (block-uniform: s_stop changes between two barriers)
      const int k = k0 + wid;
      int ns = 0;
      if (k <= a.max_iters) {
        if (lane == 0) ns = hypotheses(a, list, n, seed, k, sK1i, sK2i, hypE[wid]);
        ns = __shfl_sync(0xffffffffu, ns, 0);
        __syncwarp();
        if (lane < ns) dg::es_fundamental(hypE[wid] + 9 * lane, sA, sK1i, hypF[wid] + 9 * lane);
        __syncwarp();
        double c[kEsMax];
        int q[kEsMax];
#pragma unroll
        for (int s = 0; s < kEsMax; ++s) { c[s] = 0.0; q[s] = 0; }
        for (int i = lane; i < n; i += 32) {
          const size_t r = (size_t)list[i];
          const double x1 = a.x1[2 * r], y1 = a.x1[2 * r + 1], x2 = a.x2[2 * r], y2 = a.x2[2 * r + 1];
#pragma unroll
          for (int s = 0; s < kEsMax; ++s) {
            if (s < ns) {
              bool in;
              double fbuf[9];          // F read afresh per row: ten models kept in registers across rows spill
              c[s] += dg::es_msac(dg::pr_lin9<true>(hypF[wid] + 9 * s, fbuf), x1, y1, x2, y2, a.th2, &in);
              q[s] += in ? 1 : 0;
            }
          }
        }
#pragma unroll
        for (int s = 0; s < kEsMax; ++s)
          for (int o = 16; o > 0; o >>= 1) {
            c[s] += __shfl_xor_sync(0xffffffffu, c[s], o);
            q[s] += __shfl_xor_sync(0xffffffffu, q[s], o);
          }
        if (lane == 0) {
          hn[wid] = ns;
#pragma unroll
          for (int s = 0; s < kEsMax; ++s) { hcost[wid][s] = c[s]; hinl[wid][s] = q[s]; }
        }
      }
      __syncthreads();
      if (tid == 0) {
        for (int w = 0; w < kEsWarps; ++w) {
          const int kw = k0 + w;                     // iteration kw runs: kw - 1 < N_req after iteration kw - 1
          for (int s = 0; s < hn[w]; ++s)
            if (hcost[w][s] < s_best_cost) {
              s_best_cost = hcost[w][s];
              s_best_inl = hinl[w][s];
              s_has_best = 1;
              for (int i = 0; i < 9; ++i) { bestE[i] = hypE[w][9 * s + i]; bestF[i] = hypF[w][9 * s + i]; }
            }
          s_iters = kw;
          const int req = dg::es_required_iters(s_has_best != 0, s_best_inl, n, a.conf, a.max_iters, kw);
          if (!(kw < req)) { s_stop = 1; break; }
        }
      }
      __syncthreads();
    }
  }
  const bool has_best = s_has_best != 0;
  if (!has_best) {                                   // no model: n < 5, no solution found, or bad offsets
    if (tid < 9) { a.E_out[(size_t)p * 9 + tid] = 0.0; a.F_out[(size_t)p * 9 + tid] = 0.0; }
    if (tid == 0) {
      a.n_inliers[p] = 0;
      a.iters[p] = s_iters;
      a.cost0[p] = qnan();
      a.cost[p] = qnan();
    }
    return;
  }
  const double cost0 = s_best_cost;
  Select sel = select_pass(a, list, n, bestF, dpart, ipart);
  double cost = cost0;
  int inliers = sel.inliers;
  bool lo_kept = false;
  if (a.refine_iters > 0 && sel.inliers >= dg::kEsLoMinInliers) {
    if (tid == 0) s_pose = lo_start(bestE, sA, sK1i, pose[0], lin) ? 1 : 0;
    __syncthreads();
    if (s_pose) {
      for (int round = 0; round < dg::kEsLoRounds; ++round) {
        // Levenberg-Marquardt on the rows flagged now, from pose[0]: the schedule of pose_refine_ragged_kernel
        lm_pass(a, list, n, lin, wpart, cur);
        double lam = dg::kPrLambda0;
        int it = 0, accepted = 0;
        while (it < a.refine_iters) {                // (block-uniform: every thread keeps the same lam, it)
          ++it;
          if (tid == 0) s_go = lo_trial(cur, lam, pose[0], sA, sK1i, pose[1], lin) ? 1 : 0;
          __syncthreads();
          const bool go = s_go != 0;
          if (go) lm_pass(a, list, n, lin, wpart, trial);
          const double c_old = cur[0], c_new = trial[0];
          const bool better = go && c_new < c_old;
          const bool flat = go && fabs(c_old - c_new) < dg::kPrRelDecrease * c_old;
          __syncthreads();                           // s_go, cur[0], trial[0] are read: they may change
          if (better) {
            if (tid < dg::kPrSums) cur[tid] = trial[tid];
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
        if (tid == 0) lo_model(accepted != 0, pose[0], sA, sK1i, model, lin);
        __syncthreads();
        sel = select_pass(a, list, n, model + 9, dpart, ipart);
        if (sel.changed == 0 || sel.inliers < dg::kEsLoMinInliers) break;
      }
      if (sel.cost <= cost0) {
        cost = sel.cost;
        inliers = sel.inliers;
        lo_kept = true;
      } else {                                       // the RANSAC model stays: its flags go back to the mask
        inliers = select_pass(a, list, n, bestF, dpart, ipart).inliers;
      }
    }
  }
  __syncthreads();
  const double* E = lo_kept ? model : bestE;
  const double* F = lo_kept ? model + 9 : bestF;
  if (tid < 9) { a.E_out[(size_t)p * 9 + tid] = E[tid]; a.F_out[(size_t)p * 9 + tid] = F[tid]; }
  if (tid == 0) {
    a.n_inliers[p] = inliers;
    a.iters[p] = s_iters;
    a.cost0[p] = cost0;
    a.cost[p] = cost;
  }
}

}  // namespace

extern "C" {

const char* dgb200_essential_last_error(void) { return g_err; }

int dgb200_find_essential_ragged_dev(const double* d_x1, const double* d_x2, const double* d_K1, const double* d_K2,
                                     int k_per_pair, const int32_t* d_offsets, int n_pairs, int rows,
                                     const uint8_t* d_mask, double px_th, double conf, int max_iters, int refine_iters,
                                     const uint64_t* d_seeds, double* d_E_out, double* d_F_out, uint8_t* d_mask_out,
                                     int32_t* d_n_inliers_out, int32_t* d_iters_out, double* d_cost0_out,
                                     double* d_cost_out, void* stream) {
  if (!d_K1 || !d_K2 || !d_offsets || !d_seeds || !d_E_out || !d_F_out || !d_n_inliers_out || !d_iters_out ||
      !d_cost0_out || !d_cost_out)
    return fail(DGB200_E_ARG, "null buffer");
  if (rows > 0 && (!d_x1 || !d_x2 || !d_mask_out)) return fail(DGB200_E_ARG, "null row buffer");
  if (n_pairs < 1 || rows < 0) return fail(DGB200_E_ARG, "need n_pairs >= 1 and rows >= 0");
  if (!(px_th > 0.0) || !(px_th < INFINITY)) return fail(DGB200_E_ARG, "px_th must be a positive number");
  if (!(conf > 0.0 && conf <= 1.0)) return fail(DGB200_E_ARG, "conf must lie in (0, 1]");
  if (max_iters < 1) return fail(DGB200_E_ARG, "max_iters must be at least 1");
  if (refine_iters < 0) return fail(DGB200_E_ARG, "refine_iters must not be negative");
  const cudaStream_t st = (cudaStream_t)stream;
  int* list = nullptr;
  CU(cudaMallocAsync((void**)&list, sizeof(int) * (size_t)(rows > 0 ? rows : 1), st));
  EssentialArgs a;
  a.x1 = d_x1; a.x2 = d_x2; a.K1 = d_K1; a.K2 = d_K2; a.k_per_pair = k_per_pair; a.offsets = d_offsets;
  a.mask = d_mask; a.n_pairs = n_pairs; a.rows = rows; a.max_iters = max_iters; a.refine_iters = refine_iters;
  a.th2 = px_th * px_th; a.conf = conf; a.seeds = d_seeds; a.list = list;
  a.E_out = d_E_out; a.F_out = d_F_out; a.mask_out = d_mask_out; a.n_inliers = d_n_inliers_out;
  a.iters = d_iters_out; a.cost0 = d_cost0_out; a.cost = d_cost_out;
  essential_ragged_kernel<<<n_pairs, kEsThreads, 0, st>>>(a);
  const cudaError_t launch = cudaGetLastError();
  CU(cudaFreeAsync(list, st));
  CU(launch);
  return 0;
}

}  // extern "C"
