// view_graph_calibration.cu -- view-graph calibration, device resident: each camera group's focal length from the
// fundamental matrices of the verified pairs (GLOMAP's first step), by robust Levenberg-Marquardt on the pairs' Kruppa
// residuals over one log focal length per group, each trial step a Jacobi-preconditioned CG solve over the groups.  A
// translation unit of its own, so that adding it changes no instruction of the other sources' kernels.  The estimator
// is specified in include/degensac_b200.h; the per-thread pieces are in view_graph_calibration.h.
//
// Once per call:
//   vg_groups_kernel     one thread per group: whether its intrinsics can be used, theta = 0 in both buffers;
//   vg_edges_kernel      one thread per edge: validity, the twelve constants, the start cost and the two entries of
//                        the group-major list's sort keys (one entry for an edge inside one group);
//   vg_count_kernel,     the group-major list of the used edges' entries, ascending edge order within a group, by the
//   vg_scan_kernel,      one-digit stable counting sort of bundle_adjust_device.h (ba_sort_*);
//   vg_scatter_kernel
//   vg_nchunks_kernel,   each group's list cut into chunks of kVgChunk entries: the chunk count of each group, their
//   vg_chunk_scan_kernel, prefix (ba_sort_scan again) and the group of every chunk, so that one group holding every
//   vg_chunk_map_kernel  edge is gathered by many warps;
//   vg_init_kernel       one CTA: cost0, n_used and the LM state.
// Per trial step (the host launches max_iters steps; each kernel returns at once when the state says the call stopped):
//   vg_linearise_kernel  one thread per used edge, after an accepted step: the residuals, the Jacobian and the weight;
//                        each entry's diagonal and gradient term at its list position;
//   vg_rhs_chunk_kernel  one warp per chunk: its entries' diagonal and gradient terms, summed;
//   vg_rhs_kernel        one warp per group: its chunks' sums in chunk order, the Jacobi diagonal (1 + lambda) D and
//                        the right-hand side, the start of PCG;
//   vg_solve_kernel      the whole PCG loop in one cooperative launch (grid.sync between the phases), then the trial
//                        thetas;
//   vg_trial_kernel      one thread per used edge: its cost at the trial thetas;
//   vg_decide_kernel     one CTA: ba_decide_step.
// After the last step vg_finish_groups_kernel and vg_finish_edges_kernel write the outputs.
//
// One PCG iteration: A, one thread per used edge: u = J_e (p_gi, p_gj), and w J_e^T u for each of its entries at the
// entry's list position; B1, one warp per chunk: the sum of its entries; B2, one warp per group: q_g = sum of its
// chunks in chunk order + lambda D_g p_g (q_g = p_g for a group without a used edge), p_g . q_g; C, one thread per
// group: x += alpha p, r -= alpha q, z = r / ((1 + lambda) D); r . r and r . z.  The loop is pcg_run (pcg_device.h),
// whose dot products every CTA sums itself in one fixed order.  No floating-point atomics anywhere: a rerun gives the
// same bytes.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/degensac_b200.h"
#include "entry_error.h"
#include "common.h"
#include "view_graph_calibration.h"
#include "device_util.h"
#include "bundle_adjust_device.h"
#include "pcg_device.h"
#include "adjust_host.h"

namespace cg = cooperative_groups;

namespace {

thread_local char g_err[256] = "";
int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err, code, what, e); }

constexpr int kVgThreads = 256;                   // the one-thread-per-item kernels
constexpr int kVgWarps = 4;                       // chunks or groups per CTA of the one-warp-per-item kernels
constexpr int kVgSolveThreads = 256;              // the cooperative kernel
constexpr int kVgRange = 4096;                    // entries per warp of the counting sort
constexpr int kVgChunk = 256;                     // entries per chunk of a group's list

// One edge's record: its constants, then the trial cost at bundle_adjust.h's kBaTrkCost, so that ba_decide_step reads
// it (the edges stand in for its tracks)
constexpr int kVeC = 0;
static_assert(dg::kVgConsts <= dg::kBaTrkCost && dg::kBaTrkStride == 16, "the edge record shares the cost slot");
// One edge's linearisation: the Jacobian's columns for view i's group and view j's group (2 each; an edge inside one
// group keeps the sum in the first and 0 in the second), and its weight
constexpr int kVlJi = 0, kVlJj = 2, kVlW = 4, kVlStride = 5;
// One group's record: D = diag(H), then its PCG vectors (pcg_device.h): b, x, r, z, p in two buffers, q (1 each)
constexpr int kVrD = 0, kVrB = 1, kVrX = 2, kVrP = 5, kVrQ = 7, kVrStride = 8;

struct VgArgs {
  int n_views, n_groups, n_pairs, n_entries, n_ranges, max_chunks, cg_max_iters;
  double sig2, max_error, max_ratio, cg_tol2;
  const int2* pairs;                 // [P], device copy
  const double* F;                   // [P][9]
  const unsigned char* mask;         // [P] or null
  const int* groups;                 // [n_views]
  const double* kin;                 // [G][5]
  // workspace; n_tracks and trk are the names ba_decide_step reads
  int n_tracks;                      // = n_pairs
  double* trk;                       // [P][kBaTrkStride]: the constants and the trial cost
  double* lin;                       // [P][kVlStride]
  unsigned char* used;               // [P]
  unsigned char* gok;                // [G]: the group's intrinsics can be used
  int* key;                          // [2P]: entry 2e + s (s = 0: view i, 1: view j) -> its group, or -1
  int* ent;                          // [2P]: the entry's own index (the sort's item)
  int* pos_of;                       // [2P]
  int* item;                         // [2P]: the group-major list of entries
  int* hist;                         // [G][n_ranges]
  int* list_off;                     // [G + 1]
  int* nch;                          // [G]: chunks of the group's list, then their prefix (in place)
  int* chunk_off;                    // [G + 1]
  int* chunk_grp;                    // [max_chunks]
  double* ed;                        // [2P]: each entry's diagonal term, at its list position
  double* eg;                        // [2P]: each entry's gradient term
  double* ey;                        // [2P]: each entry's term of S p
  double* cd;                        // [max_chunks]: the chunk sums of the diagonal terms
  double* cgr;                       // [max_chunks]: the chunk sums of the gradient terms
  double* cy;                        // [max_chunks]: the chunk sums of S p
  double* theta;                     // [2][G]
  double* rec;                       // [G][kVrStride]
  double* part;                      // [kPcgParts][G]
  BaState* state;
  int* cg_iters;                     // [1]
  // outputs
  double* k_out; unsigned char* refined_out; double* err_out; unsigned char* inl_out;
  double* cost0_out; double* cost_out; int* iters_out; int* n_used_out; int* cg_iters_out;
};

__device__ __forceinline__ double* group_rec(const VgArgs& a, int g) { return a.rec + kVrStride * (size_t)g; }
__device__ __forceinline__ double* theta_of(const VgArgs& a, int buf) { return a.theta + (size_t)buf * a.n_groups; }
__device__ __forceinline__ bool has_list(const VgArgs& a, int g) { return a.list_off[g + 1] > a.list_off[g]; }
// The groups of edge e's views (valid for a used edge)
__device__ __forceinline__ int2 edge_groups(const VgArgs& a, int e) {
  const int2 pr = a.pairs[e];
  return make_int2(a.groups[pr.x], a.groups[pr.y]);
}

// ---------------------------------------------------------------------------------------------- once per call
__global__ void __launch_bounds__(kVgThreads) vg_groups_kernel(VgArgs a) {
  const int g = blockIdx.x * kVgThreads + threadIdx.x;
  if (g >= a.n_groups) return;
  a.gok[g] = dg::vg_intrinsics_ok(a.kin + 5 * (size_t)g) ? 1 : 0;
  theta_of(a, 0)[g] = 0.0;
  theta_of(a, 1)[g] = 0.0;
}

__global__ void __launch_bounds__(kVgThreads) vg_edges_kernel(VgArgs a) {
  const int e = blockIdx.x * kVgThreads + threadIdx.x;
  if (e >= a.n_pairs) return;
  const int2 pr = a.pairs[e];
  const int gi = a.groups[pr.x], gj = a.groups[pr.y];   // (the host checked that both views lie in [0, C))
  double F[9];
  for (int k = 0; k < 9; ++k) F[k] = a.F[9 * (size_t)e + k];
  double* rc = a.trk + dg::kBaTrkStride * (size_t)e;
  bool ok = dg::vg_edge_ok(pr.x, pr.y, a.n_views, gi, gj, a.n_groups, !a.mask || a.mask[e], F) && a.gok[gi] &&
            a.gok[gj];
  if (ok) ok = dg::vg_constants(F, a.kin + 5 * (size_t)gi, a.kin + 5 * (size_t)gj, rc + kVeC);
  double c = 0.0;
  if (ok) {
    double r[2];
    c = dg::vg_cost(dg::vg_residuals(rc + kVeC, 0.0, 0.0, r, nullptr), a.sig2);
  }
  rc[dg::kBaTrkCost] = c;
  a.used[e] = ok ? 1 : 0;
  a.key[2 * e] = ok ? gi : -1;
  a.key[2 * e + 1] = ok && gj != gi ? gj : -1;
  a.ent[2 * e] = 2 * e;
  a.ent[2 * e + 1] = 2 * e + 1;
}

__global__ void __launch_bounds__(32 * kVgWarps) vg_count_kernel(VgArgs a) {
  const int w = blockIdx.x * kVgWarps + (threadIdx.x >> 5);
  if (w >= a.n_ranges) return;                       // (warp-uniform)
  ba_sort_count(a.key, a.n_entries, kVgRange, a.hist, a.n_ranges, w, threadIdx.x & 31);
}

__global__ void __launch_bounds__(kBaCta) vg_scan_kernel(VgArgs a) {
  __shared__ int sh[kBaCta];
  ba_sort_scan(a.hist, a.n_groups, a.n_ranges, a.list_off, sh);
}

__global__ void __launch_bounds__(32 * kVgWarps) vg_scatter_kernel(VgArgs a) {
  const int w = blockIdx.x * kVgWarps + (threadIdx.x >> 5);
  if (w >= a.n_ranges) return;                       // (warp-uniform)
  ba_sort_scatter(a.key, a.n_entries, kVgRange, a.hist, a.n_ranges, a.ent, a.pos_of, a.item, w, threadIdx.x & 31);
}

__global__ void __launch_bounds__(kVgThreads) vg_nchunks_kernel(VgArgs a) {
  const int g = blockIdx.x * kVgThreads + threadIdx.x;
  if (g < a.n_groups) a.nch[g] = (a.list_off[g + 1] - a.list_off[g] + kVgChunk - 1) / kVgChunk;
}

__global__ void __launch_bounds__(kBaCta) vg_chunk_scan_kernel(VgArgs a) {
  __shared__ int sh[kBaCta];
  ba_sort_scan(a.nch, a.n_groups, 1, a.chunk_off, sh);
}

// One warp per group: the group of each of its chunks
__global__ void __launch_bounds__(32 * kVgWarps) vg_chunk_map_kernel(VgArgs a) {
  const int g = blockIdx.x * kVgWarps + (threadIdx.x >> 5);
  if (g >= a.n_groups) return;
  for (int k = a.chunk_off[g] + (threadIdx.x & 31); k < a.chunk_off[g + 1]; k += 32) a.chunk_grp[k] = g;
}

__global__ void __launch_bounds__(kBaCta) vg_init_kernel(VgArgs a) {
  __shared__ double shd[kBaCta];
  __shared__ int shi[kBaCta / 32];
  double c = 0.0;
  int u = 0;
  for (int e = threadIdx.x; e < a.n_pairs; e += kBaCta) {
    c += a.trk[dg::kBaTrkStride * (size_t)e + dg::kBaTrkCost];
    u += a.used[e];
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
  }
}

// ---------------------------------------------------------------------------------------------- one trial step
// One thread per used edge at the current thetas: J's columns, w, and at each entry's list position its diagonal term
// w |J_col|^2 and gradient term w J_col^T r
__global__ void __launch_bounds__(kVgThreads) vg_linearise_kernel(VgArgs a) {
  const BaState* st = a.state;
  if (st->stop || !st->lin) return;
  const int e = blockIdx.x * kVgThreads + threadIdx.x;
  if (e >= a.n_pairs || !a.used[e]) return;
  const int2 g = edge_groups(a, e);
  const double* th = theta_of(a, st->cur);
  double r[2], J[4];
  const double s = dg::vg_residuals(a.trk + dg::kBaTrkStride * (size_t)e + kVeC, th[g.x], th[g.y], r, J);
  const double w = dg::vg_weight(s, a.sig2);
  const bool one = g.x == g.y;
  const double ci[2] = {one ? J[0] + J[1] : J[0], one ? J[2] + J[3] : J[2]};
  const double cj[2] = {one ? 0.0 : J[1], one ? 0.0 : J[3]};
  double* l = a.lin + kVlStride * (size_t)e;
  l[kVlJi] = ci[0]; l[kVlJi + 1] = ci[1];
  l[kVlJj] = cj[0]; l[kVlJj + 1] = cj[1];
  l[kVlW] = w;
  const int p0 = a.pos_of[2 * e];
  a.ed[p0] = w * (ci[0] * ci[0] + ci[1] * ci[1]);
  a.eg[p0] = w * (ci[0] * r[0] + ci[1] * r[1]);
  if (!one) {
    const int p1 = a.pos_of[2 * e + 1];
    a.ed[p1] = w * (cj[0] * cj[0] + cj[1] * cj[1]);
    a.eg[p1] = w * (cj[0] * r[0] + cj[1] * r[1]);
  }
}

// The first and one-past-last list positions of chunk k of group g
__device__ __forceinline__ int2 chunk_span(const VgArgs& a, int k, int g) {
  const int b = a.list_off[g] + (k - a.chunk_off[g]) * kVgChunk;
  return make_int2(b, min(b + kVgChunk, a.list_off[g + 1]));
}

// One warp per chunk: the sums of its entries' diagonal and gradient terms
__global__ void __launch_bounds__(32 * kVgWarps) vg_rhs_chunk_kernel(VgArgs a) {
  const BaState* st = a.state;
  if (st->stop || !st->lin) return;                  // (the sums of a rejected step's linearisation stay)
  const int k = blockIdx.x * kVgWarps + (threadIdx.x >> 5);
  const int n_chunks = a.chunk_off[a.n_groups];
  if (k >= n_chunks) return;                         // (warp-uniform)
  const int lane = threadIdx.x & 31;
  const int2 sp = chunk_span(a, k, a.chunk_grp[k]);
  double d = 0.0, g = 0.0;
  for (int i = sp.x + lane; i < sp.y; i += 32) {
    d += a.ed[i];
    g += a.eg[i];
  }
  d = warp_sum(d);
  g = warp_sum(g);
  if (lane == 0) {
    a.cd[k] = d;
    a.cgr[k] = g;
  }
}

// One warp per group: D = the sum of its chunks' diagonal sums in chunk order, b = -(the gradient's); a group without a
// used edge gets D = 1, b = 0.  A D or b that is not finite, or a D that is not positive, rejects the step.  Then the
// start of PCG: x = 0, r = b, z = b / ((1 + lambda) D), both p buffers 0, and the group's r . z and b . b.
__global__ void __launch_bounds__(32 * kVgWarps) vg_rhs_kernel(VgArgs a) {
  BaState* st = a.state;
  if (st->stop) return;
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * kVgWarps + (threadIdx.x >> 5);
  if (g >= a.n_groups) return;                       // (warp-uniform)
  const int k0 = a.chunk_off[g], k1 = a.chunk_off[g + 1];
  double d = 0.0, gr = 0.0;
  for (int k = k0 + lane; k < k1; k += 32) {
    d += a.cd[k];
    gr += a.cgr[k];
  }
  d = warp_sum(d);
  gr = warp_sum(gr);
  if (lane != 0) return;
  double b = -gr, m = (1.0 + st->lam) * d;
  if (k1 == k0) {
    d = 1.0;
    m = 1.0;
    b = 0.0;
  } else if (!(d > 0.0) || !(m < INFINITY) || !(fabs(b) < INFINITY)) {
    st->bad = 1;                                     // the step is rejected
    return;
  }
  double* rec = group_rec(a, g);
  rec[kVrD] = d;
  const double z = b / m;
  pcg_start<1>(rec + kVrB, &b, &z, a.part, a.n_groups, g);
}

// pcg_run's S p and phase C over the groups.  product: A, one thread per used edge, u = J_e (p_gi, p_gj), w J_e^T u at
// its entries' list positions; grid.sync; B1, one warp per chunk, the chunk's sum; grid.sync; B2, one warp per group,
// q_g = its chunks' sums in chunk order + lambda D_g p_g, p_g stored, p_g . q_g.  update: one thread per group.
struct VgNormal {
  const VgArgs& a;
  int tid, nthr, lane, warp, nwarps;
  double lam;

  __device__ __forceinline__ void product(cg::grid_group& grid, int cur, int prev, double beta) const {
    const int ng = a.n_groups;
    for (int e = tid; e < a.n_pairs; e += nthr) {
      if (!a.used[e]) continue;
      const int2 g = edge_groups(a, e);
      const double* l = a.lin + kVlStride * (size_t)e;
      double pi, pj;
      pcg_direction<1>(group_rec(a, g.x) + kVrB, prev, beta, &pi);
      pcg_direction<1>(group_rec(a, g.y) + kVrB, prev, beta, &pj);
      const double w = __ldg(l + kVlW);
      const double ji[2] = {__ldg(l + kVlJi), __ldg(l + kVlJi + 1)}, jj[2] = {__ldg(l + kVlJj), __ldg(l + kVlJj + 1)};
      if (g.x == g.y) pj = 0.0;                       // (one column: jj = 0)
      const double u[2] = {ji[0] * pi + jj[0] * pj, ji[1] * pi + jj[1] * pj};
      a.ey[a.pos_of[2 * e]] = w * (ji[0] * u[0] + ji[1] * u[1]);
      if (g.x != g.y) a.ey[a.pos_of[2 * e + 1]] = w * (jj[0] * u[0] + jj[1] * u[1]);
    }
    grid.sync();
    const int n_chunks = a.chunk_off[ng];
    for (int k = warp; k < n_chunks; k += nwarps) {
      const int2 sp = chunk_span(a, k, a.chunk_grp[k]);
      double acc = 0.0;
      for (int i = sp.x + lane; i < sp.y; i += 32) acc += __ldcg(a.ey + i);
      acc = warp_sum(acc);
      if (lane == 0) a.cy[k] = acc;
    }
    grid.sync();
    for (int g = warp; g < ng; g += nwarps) {
      const int k0 = a.chunk_off[g], k1 = a.chunk_off[g + 1];
      double acc = 0.0;
      for (int k = k0 + lane; k < k1; k += 32) acc += __ldcg(a.cy + k);
      acc = warp_sum(acc);
      if (lane == 0) {
        double p;
        double* rec = group_rec(a, g);
        pcg_direction<1>(rec + kVrB, prev, beta, &p);
        const double q = k1 > k0 ? acc + lam * rec[kVrD] * p : p;
        rec[kVrQ] = q;
        rec[kVrP + cur] = p;
        a.part[kPartPQ * (size_t)ng + g] = p * q;
      }
    }
  }

  __device__ __forceinline__ void update(int cur, int /*prev*/, double /*beta*/, double alpha) const {
    const int ng = a.n_groups;
    for (int g = tid; g < ng; g += nthr) {
      double* rec = group_rec(a, g);
      const double m = a.chunk_off[g + 1] > a.chunk_off[g] ? (1.0 + lam) * rec[kVrD] : 1.0;
      const double p = __ldcg(rec + kVrP + cur), q = __ldcg(rec + kVrQ);
      const double2 rz = pcg_update<1>(rec + kVrB, &p, &q, alpha, [m](const double* r, double* z) { z[0] = r[0] / m; });
      a.part[kPartRR * (size_t)ng + g] = rz.x;
      a.part[kPartRZ * (size_t)ng + g] = rz.y;
    }
  }
};

// The PCG loop of one trial step (pcg_run), then the trial thetas of the groups with a used edge
__global__ void __launch_bounds__(kVgSolveThreads) vg_solve_kernel(VgArgs a) {
  __shared__ double sh[2 * kVgSolveThreads];
  BaState* st = a.state;
  if (st->stop || st->bad) return;                   // (grid-uniform: nothing below writes them before a grid.sync)
  cg::grid_group grid = cg::this_grid();
  const int tid = blockIdx.x * kVgSolveThreads + threadIdx.x, nthr = gridDim.x * kVgSolveThreads;
  const int ng = a.n_groups;
  const VgNormal op{a, tid, nthr, (int)threadIdx.x & 31, tid >> 5, nthr >> 5, st->lam};
  const PcgResult res = pcg_run<kVgSolveThreads>(grid, a.part, ng, a.cg_tol2, a.cg_max_iters, sh, op);
  // (x of a group was last written by this thread, in phase C)
  const int cur = st->cur;
  if (!res.reject)
    for (int g = tid; g < ng; g += nthr)
      if (has_list(a, g)) theta_of(a, 1 - cur)[g] = theta_of(a, cur)[g] + group_rec(a, g)[kVrX];
  if (tid == 0) {
    a.cg_iters[0] += res.iters;
    if (res.reject) st->bad = 1;
  }
}

__global__ void __launch_bounds__(kVgThreads) vg_trial_kernel(VgArgs a) {
  const BaState* st = a.state;
  if (st->stop || st->bad) return;
  const int e = blockIdx.x * kVgThreads + threadIdx.x;
  if (e >= a.n_pairs || !a.used[e]) return;
  const int2 g = edge_groups(a, e);
  const double* th = theta_of(a, 1 - st->cur);
  double* rc = a.trk + dg::kBaTrkStride * (size_t)e;
  double r[2];
  rc[dg::kBaTrkCost] = dg::vg_cost(dg::vg_residuals(rc + kVeC, th[g.x], th[g.y], r, nullptr), a.sig2);
}

__global__ void __launch_bounds__(kBaCta) vg_decide_kernel(VgArgs a) {
  __shared__ double shd[kBaCta];
  if (a.state->stop) return;                         // (block-uniform)
  ba_decide_step(a, shd);
}

// ---------------------------------------------------------------------------------------------- outputs
// The theta a group's output stands for: the solved one when the group is refined, else 0
__device__ __forceinline__ double result_theta(const VgArgs& a, int g) {
  double k[5];
  const double th = theta_of(a, a.state->cur)[g];
  return dg::vg_write_back(a.kin + 5 * (size_t)g, th, has_list(a, g), a.max_ratio, k) ? th : 0.0;
}

__global__ void __launch_bounds__(kVgThreads) vg_finish_groups_kernel(VgArgs a) {
  const int g = blockIdx.x * kVgThreads + threadIdx.x;
  const BaState* st = a.state;
  if (g == 0) {
    a.cost0_out[0] = st->cost0;
    a.cost_out[0] = st->cost;
    a.iters_out[0] = st->iters;
    a.n_used_out[0] = st->n_used;
    a.cg_iters_out[0] = a.cg_iters[0];
  }
  if (g >= a.n_groups) return;
  double k[5];
  const bool ref = dg::vg_write_back(a.kin + 5 * (size_t)g, theta_of(a, st->cur)[g], has_list(a, g), a.max_ratio, k);
  for (int m = 0; m < 5; ++m) a.k_out[5 * (size_t)g + m] = k[m];
  a.refined_out[g] = ref ? 1 : 0;
}

__global__ void __launch_bounds__(kVgThreads) vg_finish_edges_kernel(VgArgs a) {
  const int e = blockIdx.x * kVgThreads + threadIdx.x;
  if (e >= a.n_pairs) return;
  double err = qnan();
  if (a.used[e]) {
    const int2 g = edge_groups(a, e);
    double r[2];
    err = sqrt(dg::vg_residuals(a.trk + dg::kBaTrkStride * (size_t)e + kVeC, result_theta(a, g.x),
                                result_theta(a, g.y), r, nullptr));
  }
  a.err_out[e] = err;
  a.inl_out[e] = err <= a.max_error ? 1 : 0;         // (false for NaN)
}

}  // namespace

extern "C" {

const char* dgb200_view_graph_calibration_last_error(void) { return g_err; }

int dgb200_calibrate_view_graph_dev(const int32_t* h_pairs, int n_pairs, int n_views, const double* d_F,
                                    const uint8_t* d_mask, const int32_t* d_groups, const double* d_intrinsics,
                                    int n_groups, double loss_scale, double max_error, double max_ratio, int max_iters,
                                    int cg_max_iters, double cg_tol, double* d_intrinsics_out, uint8_t* d_refined_out,
                                    double* d_error_out, uint8_t* d_inliers_out, double* d_cost0_out,
                                    double* d_cost_out, int32_t* d_iters_out, int32_t* d_n_used_out,
                                    int32_t* d_cg_iters_out, void* stream) {
  if (!d_F || !d_groups || !d_intrinsics || !d_intrinsics_out || !d_refined_out || !d_error_out || !d_inliers_out ||
      !d_cost0_out || !d_cost_out || !d_iters_out || !d_n_used_out || !d_cg_iters_out)
    return fail(DGB200_E_ARG, "null buffer");
  if (n_views < 1 || n_pairs < 1 || n_groups < 1)
    return fail(DGB200_E_ARG, "need n_views >= 1, n_pairs >= 1 and n_groups >= 1");
  if (!h_pairs) return fail(DGB200_E_ARG, "null pair table");
  for (int e = 0; e < 2 * n_pairs; ++e)
    if (h_pairs[e] < 0 || h_pairs[e] >= n_views) return fail(DGB200_E_ARG, "pair view index out of range");
  if (!(loss_scale >= 0.0) || !(loss_scale < INFINITY))
    return fail(DGB200_E_ARG, "loss_scale must be a non-negative finite number");
  if (!(max_error >= 0.0) || !(max_error < INFINITY))
    return fail(DGB200_E_ARG, "max_error must be a non-negative finite number");
  if (!(max_ratio >= 1.0) || !(max_ratio < INFINITY))
    return fail(DGB200_E_ARG, "max_ratio must be a finite number >= 1");
  if (max_iters < 0) return fail(DGB200_E_ARG, "max_iters must not be negative");
  if (cg_max_iters < 1) return fail(DGB200_E_ARG, "cg_max_iters must be at least 1");
  if (!(cg_tol >= 0.0) || !(cg_tol < INFINITY)) return fail(DGB200_E_ARG, "cg_tol must be a non-negative finite number");
  const cudaStream_t st = (cudaStream_t)stream;
  int sms = 0, per_sm = 0;
  cudaError_t e = cudaSuccess;
  if (const char* m = coop_sms(&sms, &e)) return fail(DGB200_E_CUDA, m, e);
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, vg_solve_kernel, kVgSolveThreads, 0));
  if (per_sm < 1) return fail(DGB200_E_CUDA, "vg_solve_kernel does not fit on an SM");
  const size_t np = (size_t)n_pairs, ng = (size_t)n_groups, ne = 2 * np;
  const int n_ranges = blocks(ne, kVgRange);
  // every group's chunks: at most ne / kVgChunk full ones and one partial one per group
  const size_t max_chunks = ne / kVgChunk + ng;
  VgArgs a;
  a.n_views = n_views; a.n_groups = n_groups; a.n_pairs = n_pairs; a.n_entries = (int)ne; a.n_ranges = n_ranges;
  a.max_chunks = (int)max_chunks; a.cg_max_iters = cg_max_iters;
  a.sig2 = loss_scale * loss_scale; a.max_error = max_error; a.max_ratio = max_ratio; a.cg_tol2 = cg_tol * cg_tol;
  a.F = d_F; a.mask = d_mask; a.groups = d_groups; a.kin = d_intrinsics; a.n_tracks = n_pairs;
  int2* d_pairs = nullptr;
  auto lay_out = [&](char* base) {
    Carve w{base};
    d_pairs = w.take<int2>(np);
    a.trk = w.take<double>(dg::kBaTrkStride * np);
    a.lin = w.take<double>(kVlStride * np);
    a.used = w.take<unsigned char>(np);
    a.gok = w.take<unsigned char>(ng);
    a.key = w.take<int>(ne);
    a.ent = w.take<int>(ne);
    a.pos_of = w.take<int>(ne);
    a.item = w.take<int>(ne);
    a.hist = w.take<int>(ng * (size_t)n_ranges);
    a.list_off = w.take<int>(ng + 1);
    a.nch = w.take<int>(ng);
    a.chunk_off = w.take<int>(ng + 1);
    a.chunk_grp = w.take<int>(max_chunks);
    a.ed = w.take<double>(ne);
    a.eg = w.take<double>(ne);
    a.ey = w.take<double>(ne);
    a.cd = w.take<double>(max_chunks);
    a.cgr = w.take<double>(max_chunks);
    a.cy = w.take<double>(max_chunks);
    a.theta = w.take<double>(2 * ng);
    a.rec = w.take<double>(kVrStride * ng);
    a.part = w.take<double>(kPcgParts * ng);
    a.state = w.take<BaState>(1);
    a.cg_iters = w.take<int>(1);
    return w.bytes;
  };
  char* ws = nullptr;
  const size_t bytes = lay_out(nullptr);
  CU(cudaMallocAsync((void**)&ws, bytes, st));
  lay_out(ws);
  a.pairs = d_pairs;
  a.k_out = d_intrinsics_out; a.refined_out = d_refined_out; a.err_out = d_error_out; a.inl_out = d_inliers_out;
  a.cost0_out = d_cost0_out; a.cost_out = d_cost_out; a.iters_out = d_iters_out; a.n_used_out = d_n_used_out;
  a.cg_iters_out = d_cg_iters_out;
  const int edge_grid = blocks(np, kVgThreads), group_grid = blocks(ng, kVgThreads);
  const int range_grid = blocks((size_t)n_ranges, kVgWarps), group_warp_grid = blocks(ng, kVgWarps);
  const int chunk_grid = blocks(max_chunks, kVgWarps);
  void* solve_args[] = {&a};
  cudaError_t launch = cudaSuccess;
  ADJ_LAUNCH(launch = cudaMemcpyAsync(d_pairs, h_pairs, sizeof(int2) * np, cudaMemcpyHostToDevice, st));
  ADJ_LAUNCH(launch = cudaMemsetAsync(a.hist, 0, sizeof(int) * ng * (size_t)n_ranges, st));
  ADJ_LAUNCH((vg_groups_kernel<<<group_grid, kVgThreads, 0, st>>>(a)));
  ADJ_LAUNCH((vg_edges_kernel<<<edge_grid, kVgThreads, 0, st>>>(a)));
  ADJ_LAUNCH((vg_count_kernel<<<range_grid, 32 * kVgWarps, 0, st>>>(a)));
  ADJ_LAUNCH((vg_scan_kernel<<<1, kBaCta, 0, st>>>(a)));
  ADJ_LAUNCH((vg_scatter_kernel<<<range_grid, 32 * kVgWarps, 0, st>>>(a)));
  ADJ_LAUNCH((vg_nchunks_kernel<<<group_grid, kVgThreads, 0, st>>>(a)));
  ADJ_LAUNCH((vg_chunk_scan_kernel<<<1, kBaCta, 0, st>>>(a)));
  ADJ_LAUNCH((vg_chunk_map_kernel<<<group_warp_grid, 32 * kVgWarps, 0, st>>>(a)));
  ADJ_LAUNCH((vg_init_kernel<<<1, kBaCta, 0, st>>>(a)));
  for (int it = 0; it < max_iters && launch == cudaSuccess; ++it) {
    ADJ_LAUNCH((vg_linearise_kernel<<<edge_grid, kVgThreads, 0, st>>>(a)));
    ADJ_LAUNCH((vg_rhs_chunk_kernel<<<chunk_grid, 32 * kVgWarps, 0, st>>>(a)));
    ADJ_LAUNCH((vg_rhs_kernel<<<group_warp_grid, 32 * kVgWarps, 0, st>>>(a)));
    ADJ_LAUNCH(launch = cudaLaunchCooperativeKernel((const void*)vg_solve_kernel, per_sm * sms, kVgSolveThreads,
                                                    solve_args, 0, st));
    ADJ_LAUNCH((vg_trial_kernel<<<edge_grid, kVgThreads, 0, st>>>(a)));
    ADJ_LAUNCH((vg_decide_kernel<<<1, kBaCta, 0, st>>>(a)));
  }
  ADJ_LAUNCH((vg_finish_groups_kernel<<<group_grid, kVgThreads, 0, st>>>(a)));
  ADJ_LAUNCH((vg_finish_edges_kernel<<<edge_grid, kVgThreads, 0, st>>>(a)));
  CU(cudaFreeAsync(ws, st));
  CU(launch);
  return 0;
}

}  // extern "C"
