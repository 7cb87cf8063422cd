// pcg_device.h -- the preconditioned conjugate gradients loop that the iterative solvers run in one cooperative launch
// (bundle_adjust_pcg.cu, bundle_adjust_intrinsics.cu, rotation_averaging.cu, global_positioning.cu): the fixed-order
// CTA sums of the dot products, the block helpers over a record's PCG vectors and the loop itself.  Device code, in
// the anonymous namespace of the including translation unit (after device_util.h), as each kernel source keeps its own.
//
// A record of N coordinates keeps its PCG vectors at a base v: b, x, r, z at v + {0, 1, 2, 3} N, p in two buffers at
// v + 4 N and v + 5 N, q at v + 6 N.  The per-record terms of the dot products are kPcgParts arrays of n entries at
// part + kind n.
#pragma once
#include <cooperative_groups.h>
#include <cuda_runtime.h>

namespace {

constexpr int kPartPQ = 0, kPartRR = 1, kPartRZ = 2, kPartBB = 3, kPcgParts = 4;

// The fixed-order sums of up to two arrays of n entries, the same in every CTA of kThreads threads (sh: 2 kThreads
// doubles): thread t adds entries t, t + kThreads, ... in turn, then a tree over the threads.  Every thread gets the
// sums, so alpha and beta are the same in every CTA and do not depend on the grid.
template <int kThreads>
__device__ void cta_sum2(const double* u, const double* v, int n, double* sh, double* su, double* sv) {
  double x = 0.0, y = 0.0;
  for (int i = threadIdx.x; i < n; i += kThreads) {
    x += __ldcg(u + i);
    if (v) y += __ldcg(v + i);
  }
  sh[threadIdx.x] = x;
  sh[kThreads + threadIdx.x] = y;
  __syncthreads();
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) {
      sh[threadIdx.x] += sh[threadIdx.x + s];
      sh[kThreads + threadIdx.x] += sh[kThreads + threadIdx.x + s];
    }
    __syncthreads();
  }
  *su = sh[0];
  *sv = sh[kThreads];
  __syncthreads();
}

// p = z + beta p', p' in buffer `prev`
template <int N>
__device__ __forceinline__ void pcg_direction(const double* v, int prev, double beta, double* p) {
#pragma unroll
  for (int k = 0; k < N; ++k) p[k] = __ldcg(v + 3 * N + k) + beta * __ldcg(v + 4 * N + N * prev + k);
}

// The start of PCG from the right-hand side b and z = M^-1 b: x = 0, r = b, both p buffers 0; the record's r . z and
// b . b into the part arrays at entry i
template <int N>
__device__ __forceinline__ void pcg_start(double* v, const double* b, const double* z, double* part, int n, int i) {
  double rz = 0.0, bb = 0.0;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    v[k] = b[k];
    v[N + k] = 0.0;
    v[2 * N + k] = b[k];
    v[3 * N + k] = z[k];
    v[4 * N + k] = 0.0;
    v[5 * N + k] = 0.0;
    rz += b[k] * z[k];
    bb += b[k] * b[k];
  }
  part[kPartRZ * (size_t)n + i] = rz;
  part[kPartBB * (size_t)n + i] = bb;
}

// Phase C of one record: x += alpha p, r -= alpha q, z = M^-1 r through apply(r, z); returns r . r and r . z
template <int N, class Apply>
__device__ __forceinline__ double2 pcg_update(double* v, const double* p, const double* q, double alpha,
                                              const Apply& apply) {
  double r[N], z[N];
#pragma unroll
  for (int k = 0; k < N; ++k) {
    v[N + k] = __ldcg(v + N + k) + alpha * p[k];
    r[k] = __ldcg(v + 2 * N + k) - alpha * q[k];
  }
  apply(r, z);
  double rr = 0.0, rz = 0.0;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    v[2 * N + k] = r[k];
    v[3 * N + k] = z[k];
    rr += r[k] * r[k];
    rz += r[k] * z[k];
  }
  return make_double2(rr, rz);
}

struct PcgResult {
  int iters;
  bool reject;                                         // the first iteration found p . q not positive or not finite
};

// The PCG loop over the n records whose terms are in part, from the start the caller's preceding kernel wrote.  Each
// iteration: op.product(grid, cur, prev, beta) writes q = S p, stores p in buffer cur and the records' p . q terms
// (its own grid.sync() calls between its phases); grid.sync; alpha; op.update(cur, prev, beta, alpha), phase C, writes
// the r . r and r . z terms; grid.sync; the stop test, then beta.  Data written inside the launch must be read with
// __ldcg (L2), as other CTAs wrote it; every CTA computes the same scalars, so every CTA takes the same branches and
// meets the same grid.sync() calls.  sh: 2 kThreads doubles of shared memory.
template <int kThreads, class Op>
__device__ __forceinline__ PcgResult pcg_run(cooperative_groups::grid_group& grid, const double* part, int n,
                                             double cg_tol2, int cg_max_iters, double* sh, const Op& op) {
  double bb, rho;
  cta_sum2<kThreads>(part + kPartBB * (size_t)n, part + kPartRZ * (size_t)n, n, sh, &bb, &rho);
  int it = 0;
  bool reject = false;
  if (bb > 0.0) {
    double beta = 0.0;
    for (;;) {
      const int cur = it & 1, prev = cur ^ 1;
      op.product(grid, cur, prev, beta);
      grid.sync();
      double kappa, unused;
      cta_sum2<kThreads>(part + kPartPQ * (size_t)n, nullptr, n, sh, &kappa, &unused);
      ++it;
      if (!(kappa > 0.0) || !finite(kappa)) {
        reject = it == 1;
        break;
      }
      const double alpha = rho / kappa;
      op.update(cur, prev, beta, alpha);
      grid.sync();
      double rr, rz;
      cta_sum2<kThreads>(part + kPartRR * (size_t)n, part + kPartRZ * (size_t)n, n, sh, &rr, &rz);
      if (rr <= cg_tol2 * bb || it >= cg_max_iters) break;
      beta = rz / rho;
      rho = rz;
    }
  }
  return {it, reject};
}

}  // namespace
