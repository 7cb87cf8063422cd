// rotation_averaging.cu -- rotation averaging over a view graph, device resident: every view gets a world rotation from
// the relative rotations of its verified pairs (the first step of global SfM, as in GLOMAP, Theia and OpenMVG).  A
// maximum-spanning-forest start, then IRLS on the linearised problem, each step a Jacobi-preconditioned CG solve of the
// weighted graph Laplacian.  A translation unit of its own, so that adding it changes no instruction of the other
// sources' kernels.  The estimator is specified in include/degensac_b200.h; the per-thread pieces are in
// rotation_averaging.h.
//
// Once per call:
//   ra_edges_kernel      one thread per edge: validity, the prepared R_e, the two entries (i and j) of the view-major
//                        list's sort keys;
//   ra_views_kernel      one thread per view: the union-find and Boruvka's per-component minimum;
//   ra_count_kernel,     the view-major list of the valid edges' entries, ascending edge order within a view, by the
//   ra_scan_kernel,      one-digit stable counting sort of bundle_adjust_device.h (ba_sort_*);
//   ra_scatter_kernel
//   Boruvka rounds (ceil(log2 n_views) + 1 of them, so the host never reads back):
//     ra_min_edge_kernel one thread per valid edge joining two trees: the 64-bit key ((INT32_MAX - w) << 32) | e into
//                        both trees' minimum by an integer atomicMin (the smallest key wins whatever the order);
//     ra_hook_kernel     one thread per tree with a minimum: its edge joins the forest, tk_link (tracks.h);
//     ra_compress_kernel one thread per view: tk_compress, so each view points at its tree's smallest view;
//   ra_tree_kernel       one cooperative launch: each root gets R = I, then a level-synchronous walk down the forest
//                        (grid.sync between levels), each view composed from its tree parent's rotation.
// Per IRLS iteration (the host launches l1_iters + max_iters of them; each kernel returns at once once the state says
// the call has stopped):
//   ra_residual_kernel   one thread per valid edge: r_e and its weight;
//   ra_rhs_kernel        one warp per view: the Laplacian's diagonal and the right-hand side, the start of PCG;
//   ra_solve_kernel      the whole PCG loop in one cooperative launch (grid.sync between the phases), then the update
//                        of every view and its step length;
//   ra_decide_kernel     one CTA: the largest step, the iteration counts and the phase.
// After the last iteration ra_finish_edges_kernel and ra_finish_views_kernel write the outputs.
//
// One PCG iteration: B, one warp per view: q_v = d_v p_v - sum_{e in v} w_e p_other over the view's list (a root's q_v
// = p_v), p_v . q_v; C, one thread per view: x += alpha p, r -= alpha q, z = r / d; r . r and r . z.  The loop is
// pcg_run (pcg_device.h), whose dot products every CTA sums itself in one fixed order, so they do not depend on the
// grid.  No floating-point atomics anywhere: a rerun gives the same bytes.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/degensac_b200.h"
#include "entry_error.h"
#include "common.h"
#include "rotation_averaging.h"
#include "tracks.h"
#include "device_util.h"
#include "bundle_adjust_device.h"
#include "pcg_device.h"
#include "adjust_host.h"

namespace cg = cooperative_groups;

namespace {

thread_local char g_err[256] = "";
int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err, code, what, e); }

constexpr int kRaThreads = 256;                   // the one-thread-per-item kernels
constexpr int kRaWarps = 4;                       // views per CTA of the one-warp-per-view kernel
constexpr int kRaSolveThreads = 256;              // the cooperative kernels
constexpr int kRaRange = 4096;                    // entries per warp of the counting sort
constexpr unsigned long long kRaNoEdge = ~0ull;

// One view's record: the Laplacian's diagonal d, then its PCG vectors (pcg_device.h): b, x, r, z, p in two buffers
// and q (3 each)
constexpr int kRvD = 0, kRvB = 1, kRvX = 4, kRvP = 13, kRvQ = 19, kRvStride = 22;
// The per-view terms of the dot products (pcg_device.h), then the step lengths: kRaParts arrays of n_views
constexpr int kPartStep = kPcgParts, kRaParts = kPcgParts + 1;
constexpr int kPhaseDone = 2;

struct RaState {
  int phase, iters[2], cg_iters, reject;
};

struct RaArgs {
  int n_views, n_pairs, n_entries, n_ranges, l1_iters, max_iters, cg_max_iters;
  double sig2, step_tol, cg_tol2;
  const int2* pairs;                 // [P], device copy
  const double* R_rel;               // [P][9]
  const unsigned char* mask;         // [P] or null
  const int* weights;                // [P] or null
  // workspace
  double* Re;                        // [P][9]: the prepared relative rotations
  double* er;                        // [P][4]: r_e and w_e of the current iteration
  unsigned char* valid;              // [P]
  unsigned char* in_tree;            // [P]
  int* key;                          // [2P]: entry 2e + s (s = 0: view i, 1: view j) -> its view, or -1
  int* ent;                          // [2P]: the entry's own index (the sort's item)
  int* pos_of;                       // [2P]
  int* item;                         // [2P]: the view-major list of entries
  int* hist;                         // [n_views][n_ranges]
  int* list_off;                     // [n_views + 1]
  int* parent;                       // [n_views]
  unsigned long long* best;          // [n_views]
  int* level;                        // [n_views]
  int* flag;                         // [3]
  double* R;                         // [n_views][9]
  double* rec;                       // [n_views][kRvStride]
  double* part;                      // [kRaParts][n_views]
  RaState* state;
  // outputs
  double* R_out; int* comp_out; double* res_out; int* iters_out; int* cg_iters_out;
};

__device__ __forceinline__ double* view_rec(const RaArgs& a, int v) { return a.rec + kRvStride * (size_t)v; }
__device__ __forceinline__ bool pinned(const RaArgs& a, int v) { return a.parent[v] == v; }   // a root or isolated
__device__ __forceinline__ int other_view(const RaArgs& a, int entry) {
  const int2 pr = a.pairs[entry >> 1];
  return (entry & 1) ? pr.x : pr.y;
}

// ---------------------------------------------------------------------------------------------- once per call
__global__ void __launch_bounds__(kRaThreads) ra_edges_kernel(RaArgs a) {
  const int e = blockIdx.x * kRaThreads + threadIdx.x;
  if (e >= a.n_pairs) return;
  const int2 pr = a.pairs[e];
  double R[9];
  for (int k = 0; k < 9; ++k) R[k] = a.R_rel[9 * (size_t)e + k];
  const bool ok = pr.x != pr.y && (!a.mask || a.mask[e]) && (!a.weights || a.weights[e] >= 0) && dg::ra_edge_ok(R);
  if (ok) dg::ra_prepare(R);
  for (int k = 0; k < 9; ++k) a.Re[9 * (size_t)e + k] = R[k];
  a.valid[e] = ok ? 1 : 0;
  a.in_tree[e] = 0;
  a.key[2 * e] = ok ? pr.x : -1;
  a.key[2 * e + 1] = ok ? pr.y : -1;
  a.ent[2 * e] = 2 * e;
  a.ent[2 * e + 1] = 2 * e + 1;
}

__global__ void __launch_bounds__(kRaThreads) ra_views_kernel(RaArgs a) {
  const int v = blockIdx.x * kRaThreads + threadIdx.x;
  if (v < 3) a.flag[v] = 0;
  if (v == 0) {
    RaState* st = a.state;
    st->phase = a.l1_iters > 0 ? 0 : (a.max_iters > 0 ? 1 : kPhaseDone);
    st->iters[0] = 0;
    st->iters[1] = 0;
    st->cg_iters = 0;
    st->reject = 0;
  }
  if (v >= a.n_views) return;
  a.parent[v] = v;
  a.best[v] = kRaNoEdge;
  a.level[v] = -1;
}

__global__ void __launch_bounds__(32 * kRaWarps) ra_count_kernel(RaArgs a) {
  const int w = blockIdx.x * kRaWarps + (threadIdx.x >> 5);
  if (w >= a.n_ranges) return;                       // (warp-uniform)
  ba_sort_count(a.key, a.n_entries, kRaRange, a.hist, a.n_ranges, w, threadIdx.x & 31);
}

__global__ void __launch_bounds__(kBaCta) ra_scan_kernel(RaArgs a) {
  __shared__ int sh[kBaCta];
  ba_sort_scan(a.hist, a.n_views, a.n_ranges, a.list_off, sh);
}

__global__ void __launch_bounds__(32 * kRaWarps) ra_scatter_kernel(RaArgs a) {
  const int w = blockIdx.x * kRaWarps + (threadIdx.x >> 5);
  if (w >= a.n_ranges) return;                       // (warp-uniform)
  ba_sort_scatter(a.key, a.n_entries, kRaRange, a.hist, a.n_ranges, a.ent, a.pos_of, a.item, w, threadIdx.x & 31);
}

// Boruvka: every parent[] entry is its tree's root here (ra_compress_kernel ran last)
__global__ void __launch_bounds__(kRaThreads) ra_min_edge_kernel(RaArgs a) {
  const int e = blockIdx.x * kRaThreads + threadIdx.x;
  if (e >= a.n_pairs || !a.valid[e]) return;
  const int2 pr = a.pairs[e];
  const int ri = a.parent[pr.x], rj = a.parent[pr.y];
  if (ri == rj) return;
  const int w = a.weights ? a.weights[e] : 0;
  const unsigned long long k = ((unsigned long long)(unsigned)(INT32_MAX - w) << 32) | (unsigned)e;
  if (k < a.best[ri]) atomicMin(a.best + ri, k);
  if (k < a.best[rj]) atomicMin(a.best + rj, k);
}

__global__ void __launch_bounds__(kRaThreads) ra_hook_kernel(RaArgs a) {
  const int v = blockIdx.x * kRaThreads + threadIdx.x;
  if (v >= a.n_views) return;
  const unsigned long long k = a.best[v];
  if (k == kRaNoEdge) return;
  a.best[v] = kRaNoEdge;
  const int e = (int)(k & 0xffffffffull);
  a.in_tree[e] = 1;                                  // (both trees may pick e: the same store)
  const int2 pr = a.pairs[e];
  dg::tk_link(a.parent, pr.x, pr.y);
}

__global__ void __launch_bounds__(kRaThreads) ra_compress_kernel(RaArgs a) {
  const int v = blockIdx.x * kRaThreads + threadIdx.x;
  if (v < a.n_views) dg::tk_compress(a.parent, v);
}

// The start: R = I at each root (a view with a valid edge and parent[v] == v), NaN at a view without a valid edge;
// then level d + 1 is every unplaced view with a tree edge to a view of level d, composed across that edge (a forest:
// one such edge per view).  The level counter is grid-uniform: every CTA reads the same flag after the grid.sync.
__global__ void __launch_bounds__(kRaSolveThreads) ra_tree_kernel(RaArgs a) {
  cg::grid_group grid = cg::this_grid();
  const int tid = blockIdx.x * kRaSolveThreads + threadIdx.x, nthr = gridDim.x * kRaSolveThreads;
  for (int v = tid; v < a.n_views; v += nthr) {
    const bool has = a.list_off[v + 1] > a.list_off[v];
    double* R = a.R + 9 * (size_t)v;
    if (!has) {
      for (int k = 0; k < 9; ++k) R[k] = qnan();
    } else if (a.parent[v] == v) {
      for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0) ? 1.0 : 0.0;
      a.level[v] = 0;
    }
  }
  grid.sync();
  for (int d = 0;; ++d) {
    if (tid == 0) a.flag[(d + 1) % 3] = 0;           // read last at level d - 2, written next at level d + 1
    for (int v = tid; v < a.n_views; v += nthr) {
      if (__ldcg(a.level + v) >= 0) continue;
      const int i0 = a.list_off[v], i1 = a.list_off[v + 1];
      for (int i = i0; i < i1; ++i) {
        const int entry = a.item[i], e = entry >> 1;
        if (!a.in_tree[e]) continue;
        const int u = other_view(a, entry);
        if (__ldcg(a.level + u) != d) continue;
        double Rp[9], Rc[9];
        for (int k = 0; k < 9; ++k) Rp[k] = __ldcg(a.R + 9 * (size_t)u + k);
        dg::ra_compose(a.Re + 9 * (size_t)e, Rp, (entry & 1) == 1, Rc);
        for (int k = 0; k < 9; ++k) a.R[9 * (size_t)v + k] = Rc[k];
        a.level[v] = d + 1;
        a.flag[d % 3] = 1;
        break;
      }
    }
    grid.sync();
    if (__ldcg(a.flag + d % 3) == 0) break;
  }
}

// ---------------------------------------------------------------------------------------------- one IRLS iteration
__global__ void __launch_bounds__(kRaThreads) ra_residual_kernel(RaArgs a) {
  const int phase = a.state->phase;
  if (phase == kPhaseDone) return;
  const int e = blockIdx.x * kRaThreads + threadIdx.x;
  if (e >= a.n_pairs || !a.valid[e]) return;
  const int2 pr = a.pairs[e];
  double dR[9], r[3];
  dg::ra_relative(a.R + 9 * (size_t)pr.x, a.R + 9 * (size_t)pr.y, a.Re + 9 * (size_t)e, dR);
  const double th = dg::ra_log(dR, r);
  double* out = a.er + 4 * (size_t)e;
  out[0] = r[0]; out[1] = r[1]; out[2] = r[2];
  out[3] = dg::ra_weight(phase, th, a.sig2);
}

// One warp per view: d_v = sum w_e and b_v = sum (+-) w_e r_e over its list (+ where v is the edge's j); a pinned view
// gets d = 1, b = 0.  Then the start of PCG: x = 0, r = b, z = b / d, both p buffers 0, and the view's r . z and b . b.
__global__ void __launch_bounds__(32 * kRaWarps) ra_rhs_kernel(RaArgs a) {
  if (a.state->phase == kPhaseDone) return;
  const int lane = threadIdx.x & 31;
  const int v = blockIdx.x * kRaWarps + (threadIdx.x >> 5);
  if (v >= a.n_views) return;                        // (warp-uniform)
  double d = 0.0, b[3] = {0.0, 0.0, 0.0};
  const int i0 = a.list_off[v], i1 = a.list_off[v + 1];
  for (int i = i0 + lane; i < i1; i += 32) {
    const int entry = a.item[i];
    const double* er = a.er + 4 * (size_t)(entry >> 1);
    const double w = er[3], sw = (entry & 1) ? w : -w;
    d += w;
    b[0] += sw * er[0]; b[1] += sw * er[1]; b[2] += sw * er[2];
  }
  d = warp_sum(d);
#pragma unroll
  for (int k = 0; k < 3; ++k) b[k] = warp_sum(b[k]);
  if (lane != 0) return;
  if (pinned(a, v)) {
    d = 1.0;
    b[0] = b[1] = b[2] = 0.0;
  }
  double* rec = view_rec(a, v);
  rec[kRvD] = d;
  const double z[3] = {b[0] / d, b[1] / d, b[2] / d};
  pcg_start<3>(rec + kRvB, b, z, a.part, a.n_views, v);
}

// pcg_run's S p and phase C over the views.  product: B, one warp per view, q_v = d_v p_v - sum_e w_e p_other, p_v
// stored, p_v . q_v.  update: one thread per view.
struct RaLaplacian {
  const RaArgs& a;
  int tid, nthr, lane, warp, nwarps;

  __device__ __forceinline__ void product(cg::grid_group& /*grid*/, int cur, int prev, double beta) const {
    const int n = a.n_views;
    for (int v = warp; v < n; v += nwarps) {
      double acc[3] = {0.0, 0.0, 0.0};
      const bool pin = pinned(a, v);
      if (!pin) {
        const int i0 = a.list_off[v], i1 = a.list_off[v + 1];
        for (int i = i0 + lane; i < i1; i += 32) {
          const int entry = a.item[i];
          const double w = a.er[4 * (size_t)(entry >> 1) + 3];
          double po[3];
          pcg_direction<3>(view_rec(a, other_view(a, entry)) + kRvB, prev, beta, po);
          acc[0] += w * po[0]; acc[1] += w * po[1]; acc[2] += w * po[2];
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) acc[k] = warp_sum(acc[k]);
      }
      if (lane == 0) {
        double p[3];
        double* rec = view_rec(a, v);
        pcg_direction<3>(rec + kRvB, prev, beta, p);
        const double d = rec[kRvD];
        double pq = 0.0;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double q = pin ? p[k] : d * p[k] - acc[k];
          rec[kRvQ + k] = q;
          rec[kRvP + 3 * cur + k] = p[k];
          pq += p[k] * q;
        }
        a.part[kPartPQ * (size_t)n + v] = pq;
      }
    }
  }

  __device__ __forceinline__ void update(int cur, int /*prev*/, double /*beta*/, double alpha) const {
    const int n = a.n_views;
    for (int v = tid; v < n; v += nthr) {
      double* rec = view_rec(a, v);
      const double d = rec[kRvD];
      double p[3], q[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        p[k] = __ldcg(rec + kRvP + 3 * cur + k);
        q[k] = __ldcg(rec + kRvQ + k);
      }
      const double2 rz = pcg_update<3>(rec + kRvB, p, q, alpha, [d](const double* r, double* z) {
#pragma unroll
        for (int k = 0; k < 3; ++k) z[k] = r[k] / d;
      });
      a.part[kPartRR * (size_t)n + v] = rz.x;
      a.part[kPartRZ * (size_t)n + v] = rz.y;
    }
  }
};

// The PCG loop of one iteration (pcg_run), then the update of every view that is not pinned and its step length |w_v|
__global__ void __launch_bounds__(kRaSolveThreads) ra_solve_kernel(RaArgs a) {
  __shared__ double sh[2 * kRaSolveThreads];
  RaState* st = a.state;
  if (st->phase == kPhaseDone) return;               // (grid-uniform: written only by ra_decide_kernel)
  cg::grid_group grid = cg::this_grid();
  const int tid = blockIdx.x * kRaSolveThreads + threadIdx.x, nthr = gridDim.x * kRaSolveThreads;
  const int n = a.n_views;
  const RaLaplacian op{a, tid, nthr, (int)threadIdx.x & 31, tid >> 5, nthr >> 5};
  const PcgResult res = pcg_run<kRaSolveThreads>(grid, a.part, n, a.cg_tol2, a.cg_max_iters, sh, op);
  // the update (x of a view was last written by this thread, in phase C)
  for (int v = tid; v < n; v += nthr) {
    double step = 0.0;
    if (!res.reject && !pinned(a, v)) {
      const double* x = view_rec(a, v) + kRvX;
      const double w[3] = {x[0], x[1], x[2]};
      double* R = a.R + 9 * (size_t)v;
      double R2[9];
      dg::ra_update(R, w, R2);
      for (int k = 0; k < 9; ++k) R[k] = R2[k];
      step = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    }
    a.part[kPartStep * (size_t)n + v] = step;
  }
  if (tid == 0) {
    st->cg_iters += res.iters;
    st->reject = res.reject ? 1 : 0;
  }
}

// One CTA: the iteration is counted in its phase; the phase ends after a rejected first CG iteration, once the largest
// step is at most step_tol, or after its iteration limit
__global__ void __launch_bounds__(kBaCta) ra_decide_kernel(RaArgs a) {
  __shared__ double sh[kBaCta];
  RaState* st = a.state;
  const int phase = st->phase;
  if (phase == kPhaseDone) return;                   // (block-uniform)
  double m = 0.0;
  for (int v = threadIdx.x; v < a.n_views; v += kBaCta) m = fmax(m, a.part[kPartStep * (size_t)a.n_views + v]);
  sh[threadIdx.x] = m;
  __syncthreads();
  for (int s = kBaCta / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] = fmax(sh[threadIdx.x], sh[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  const int n_it = ++st->iters[phase];
  const int limit = phase == 0 ? a.l1_iters : a.max_iters;
  if (st->reject || sh[0] <= a.step_tol || n_it >= limit) st->phase = (phase == 0 && a.max_iters > 0) ? 1 : kPhaseDone;
}

// ---------------------------------------------------------------------------------------------- outputs
__global__ void __launch_bounds__(kRaThreads) ra_finish_edges_kernel(RaArgs a) {
  const int e = blockIdx.x * kRaThreads + threadIdx.x;
  if (e >= a.n_pairs) return;
  double th = qnan();
  if (a.valid[e]) {
    const int2 pr = a.pairs[e];
    double dR[9], r[3];
    dg::ra_relative(a.R + 9 * (size_t)pr.x, a.R + 9 * (size_t)pr.y, a.Re + 9 * (size_t)e, dR);
    th = dg::ra_log(dR, r);
  }
  a.res_out[e] = th;
}

__global__ void __launch_bounds__(kRaThreads) ra_finish_views_kernel(RaArgs a) {
  const int v = blockIdx.x * kRaThreads + threadIdx.x;
  if (v == 0) {
    a.iters_out[0] = a.state->iters[0];
    a.iters_out[1] = a.state->iters[1];
    a.cg_iters_out[0] = a.state->cg_iters;
  }
  if (v >= a.n_views) return;
  for (int k = 0; k < 9; ++k) a.R_out[9 * (size_t)v + k] = a.R[9 * (size_t)v + k];
  a.comp_out[v] = a.list_off[v + 1] > a.list_off[v] ? a.parent[v] : -1;
}

}  // namespace

extern "C" {

const char* dgb200_rotation_averaging_last_error(void) { return g_err; }

int dgb200_average_rotations_dev(const int32_t* h_pairs, int n_pairs, int n_views, const double* d_R_rel,
                                 const uint8_t* d_mask, const int32_t* d_weights, double sigma, int l1_iters,
                                 int max_iters, double step_tol, int cg_max_iters, double cg_tol, double* d_R_out,
                                 int32_t* d_component_out, double* d_residual_out, int32_t* d_iters_out,
                                 int32_t* d_cg_iters_out, void* stream) {
  if (!d_R_rel || !d_R_out || !d_component_out || !d_residual_out || !d_iters_out || !d_cg_iters_out)
    return fail(DGB200_E_ARG, "null buffer");
  if (n_views < 1 || n_pairs < 1) return fail(DGB200_E_ARG, "need n_views >= 1 and n_pairs >= 1");
  if (!h_pairs) return fail(DGB200_E_ARG, "null pair table");
  for (int e = 0; e < 2 * n_pairs; ++e)
    if (h_pairs[e] < 0 || h_pairs[e] >= n_views) return fail(DGB200_E_ARG, "pair view index out of range");
  if (!(sigma > 0.0) || !(sigma < INFINITY)) return fail(DGB200_E_ARG, "sigma must be a positive finite number");
  if (l1_iters < 0 || max_iters < 0) return fail(DGB200_E_ARG, "l1_iters and max_iters must not be negative");
  if (!(step_tol >= 0.0) || !(step_tol < INFINITY))
    return fail(DGB200_E_ARG, "step_tol must be a non-negative finite number");
  if (cg_max_iters < 1) return fail(DGB200_E_ARG, "cg_max_iters must be at least 1");
  if (!(cg_tol >= 0.0) || !(cg_tol < INFINITY)) return fail(DGB200_E_ARG, "cg_tol must be a non-negative finite number");
  const cudaStream_t st = (cudaStream_t)stream;
  int sms = 0, per_sm_tree = 0, per_sm_solve = 0;
  cudaError_t e = cudaSuccess;
  if (const char* m = coop_sms(&sms, &e)) return fail(DGB200_E_CUDA, m, e);
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_tree, ra_tree_kernel, kRaSolveThreads, 0));
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_solve, ra_solve_kernel, kRaSolveThreads, 0));
  if (per_sm_tree < 1 || per_sm_solve < 1) return fail(DGB200_E_CUDA, "a cooperative kernel does not fit on an SM");
  const size_t np = (size_t)n_pairs, nv = (size_t)n_views, ne = 2 * np;
  const int n_ranges = blocks(ne, kRaRange);
  int rounds = 0;                                    // ceil(log2 n_views) + 1
  while ((1ll << rounds) < (long long)n_views) ++rounds;
  ++rounds;
  RaArgs a;
  a.n_views = n_views; a.n_pairs = n_pairs; a.n_entries = (int)ne; a.n_ranges = n_ranges;
  a.l1_iters = l1_iters; a.max_iters = max_iters; a.cg_max_iters = cg_max_iters;
  a.sig2 = sigma * sigma; a.step_tol = step_tol; a.cg_tol2 = cg_tol * cg_tol;
  a.R_rel = d_R_rel; a.mask = d_mask; a.weights = d_weights;
  int2* d_pairs = nullptr;
  auto lay_out = [&](char* base) {
    Carve w{base};
    d_pairs = w.take<int2>(np);
    a.Re = w.take<double>(9 * np);
    a.er = w.take<double>(4 * np);
    a.valid = w.take<unsigned char>(np);
    a.in_tree = w.take<unsigned char>(np);
    a.key = w.take<int>(ne);
    a.ent = w.take<int>(ne);
    a.pos_of = w.take<int>(ne);
    a.item = w.take<int>(ne);
    a.hist = w.take<int>(nv * (size_t)n_ranges);
    a.list_off = w.take<int>(nv + 1);
    a.parent = w.take<int>(nv);
    a.best = w.take<unsigned long long>(nv);
    a.level = w.take<int>(nv);
    a.flag = w.take<int>(3);
    a.R = w.take<double>(9 * nv);
    a.rec = w.take<double>(kRvStride * nv);
    a.part = w.take<double>(kRaParts * nv);
    a.state = w.take<RaState>(1);
    return w.bytes;
  };
  char* ws = nullptr;
  const size_t bytes = lay_out(nullptr);
  CU(cudaMallocAsync((void**)&ws, bytes, st));
  lay_out(ws);
  a.pairs = d_pairs;
  a.R_out = d_R_out; a.comp_out = d_component_out; a.res_out = d_residual_out; a.iters_out = d_iters_out;
  a.cg_iters_out = d_cg_iters_out;
  const int edge_grid = blocks(np, kRaThreads), view_grid = blocks(nv, kRaThreads);
  const int range_grid = blocks((size_t)n_ranges, kRaWarps), warp_grid = blocks(nv, kRaWarps);
  void* coop_args[] = {&a};
  cudaError_t launch = cudaSuccess;
  ADJ_LAUNCH(launch = cudaMemcpyAsync(d_pairs, h_pairs, sizeof(int2) * np, cudaMemcpyHostToDevice, st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.hist, 0, sizeof(int) * nv * (size_t)n_ranges, st));
  ADJ_LAUNCH((ra_edges_kernel<<<edge_grid, kRaThreads, 0, st>>>(a)));
  ADJ_LAUNCH((ra_views_kernel<<<view_grid, kRaThreads, 0, st>>>(a)));
  ADJ_LAUNCH((ra_count_kernel<<<range_grid, 32 * kRaWarps, 0, st>>>(a)));
  ADJ_LAUNCH((ra_scan_kernel<<<1, kBaCta, 0, st>>>(a)));
  ADJ_LAUNCH((ra_scatter_kernel<<<range_grid, 32 * kRaWarps, 0, st>>>(a)));
  for (int r = 0; r < rounds; ++r) {
    ADJ_LAUNCH((ra_min_edge_kernel<<<edge_grid, kRaThreads, 0, st>>>(a)));
    ADJ_LAUNCH((ra_hook_kernel<<<view_grid, kRaThreads, 0, st>>>(a)));
    ADJ_LAUNCH((ra_compress_kernel<<<view_grid, kRaThreads, 0, st>>>(a)));
  }
  ADJ_LAUNCH(launch = cudaLaunchCooperativeKernel((const void*)ra_tree_kernel, per_sm_tree * sms, kRaSolveThreads,
                                                  coop_args, 0, st));
  for (int it = 0; it < l1_iters + max_iters && launch == cudaSuccess; ++it) {
    ADJ_LAUNCH((ra_residual_kernel<<<edge_grid, kRaThreads, 0, st>>>(a)));
    ADJ_LAUNCH((ra_rhs_kernel<<<warp_grid, 32 * kRaWarps, 0, st>>>(a)));
    ADJ_LAUNCH(launch = cudaLaunchCooperativeKernel((const void*)ra_solve_kernel, per_sm_solve * sms, kRaSolveThreads,
                                                    coop_args, 0, st));
    ADJ_LAUNCH((ra_decide_kernel<<<1, kBaCta, 0, st>>>(a)));
  }
  ADJ_LAUNCH((ra_finish_edges_kernel<<<edge_grid, kRaThreads, 0, st>>>(a)));
  ADJ_LAUNCH((ra_finish_views_kernel<<<view_grid, kRaThreads, 0, st>>>(a)));
  CU(cudaFreeAsync(ws, st));
  CU(launch);
  return 0;
}

}  // extern "C"
