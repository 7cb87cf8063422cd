// frontend.cu -- the steps either side of the RANSAC path (SURVEY.md section 8(f).3 and 8(f).4), device resident:
//
//   BEFORE  descriptor matching: brute-force L2 two-nearest-neighbour search + SNN ratio test (+ optional mutual
//           check) producing the [N,2] correspondence arrays the RANSAC kernel consumes -- what the reference's
//           pipeline does on the host with cv2.BFMatcher.knnMatch(k=2) and `m.distance < 0.9 * n.distance`
//           (examples/simple-example.py:46-53), so that src_pts/dst_pts never visit the host.  Binary descriptors
//           (ORB, AKAZE, BRISK, FREAK) take the same path with the Hamming distance (cv2.NORM_HAMMING): one XOR and one
//           POPC per 32 bits in place of the FP32 FMAs.
//           The train descriptors are streamed through shared memory with Hopper BULK ASYNC COPIES
//           (cp.async.bulk global->shared, completion on an mbarrier; UBLKCP in SASS), double buffered behind the math.
//   AFTER   pose from a fundamental matrix: E = K2^T F K1, the four (R, t) candidates, cheirality vote over the
//           inliers (one warp per pair);  the reference stops at F (the survey lists E/pose as the step after).
//           Pose and scene plane from a homography (planar scenes, pure rotations): the decompositions of
//           K2^-1 H K1, cheirality vote, the two best candidates; the rows and median of the F path.
//           Refinement on the inliers of the pose (Sampson error of F = K2^-T [t]x R K1^-1), of a homography
//           (the engine's Sampson error of H) and of a fundamental matrix (its Sampson error over the rank-2
//           matrices), batched Levenberg-Marquardt.
//   ALSO    the reference's alternative 7-point null-space solver nullspace_qr7x9 (Ftools.c:594, USE_QR) as a batch
//           kernel over many samples (la.h restates LAPACK's dgeqp3 kernel).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <vector>

#include "../../include/degensac_b200.h"
#include "entry_error.h"
#include "common.h"
#include "la.h"
#include "hgeom.h"
#include "pose_refine.h"
#include "refine_h.h"
#include "refine_f.h"
#include "rng.h"
#include "device_util.h"

namespace {

thread_local char g_err[256] = "";
int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err, code, what, e); }

// ------------------------------------------------------------------------------------------------ matcher
constexpr int kTQ = 32;          // query descriptors per CTA
constexpr int kTT = 64;          // train descriptors per shared-memory stage
constexpr int kMatchThreads = 128;   // 32 queries x 4 train groups

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!done);
}
// 1-D bulk async copy global -> shared (TMA engine, no tensor map needed): size and both addresses 16-byte aligned
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// One matcher work unit per image pair.  Built on the host from the image offsets and the pair table, copied to the
// device with the call; entry n_pairs holds the totals.
struct PairMeta {
  int qrow, n1;     // query descriptors: rows qrow .. qrow+n1-1 of the query bank
  int trow, n2;     // train descriptors: rows trow .. trow+n2-1 of the train bank
  int tile0;        // first 2-NN work item: prefix of ceil(n1 / kTQ); a degenerate pair (n1 < 1 or n2 < 2) has none
  int row0;         // first per-query slot (nn_idx / nn_d1 / nn_d2): prefix of n1, which is also the output capacity
  int col0;         // first col_best slot: prefix of n2, so that a train image shared by several pairs keeps them apart
  int pad;
};

struct MatchArgs {
  const float* qbank; const float* tbank;   // [rows][D]: the query and train descriptors of every pair (binary rows:
                                            // 32-bit words, read through Dist::Elem)
  const PairMeta* meta;                     // [n_pairs + 1]
  int n_pairs, D;
  int use_bulk;                       // train rows are 16-byte aligned: stage them with cp.async.bulk
  int mutual;                         // also track, per train descriptor, its nearest query (col_best)
  int* nn_idx; float* nn_d1; float* nn_d2;          // per query: nearest train index, distances of the two nearest
  unsigned long long* col_best;       // per train descriptor: (distance bits << 32 | query index), atomicMin
  // guided matching only (a gate other than NoGate): per-pair models [n_pairs][9], keypoint rows of the banks'
  // images [rows][kp_dim] (x, y in columns 0-1) and the squared pixel threshold
  const double* models; const double* kq; const double* kt; int kp_dim; double th;
};

// ------------------------------------------------------------------------------------------------ guided matching
// Gate policies of the matcher: which train descriptors of a pair count as candidates of a query.  A policy splits its
// predicate into query terms (Q, registers of the query's thread), row terms (kTerms doubles per train row, computed
// once per CTA and staged in shared memory beside the descriptors) and pass(), which combines them in exactly the
// operation order of the unsplit expression (the library is compiled with -fmad=false), so that the gate is bit for bit
// the expression written out in the header.  Every comparison is written so that NaN fails it.
struct NoGate {             // plain matching: every train descriptor is a candidate
  static constexpr bool kOn = false;
  static constexpr int kTerms = 0;
  struct Q {};
};

// F (x_t^T F x_q = 0): the engine's Sampson residual dg::f_resid_sampson(F, xq, yq, xt, yt) <= th -- the rule that
// makes a correspondence an inlier of the RANSAC mask.  f_res_terms: rxc, ryc, rwc depend on the train point only, rx,
// ry on the query only; the denominator sums (((rxc^2 + ryc^2) + rx^2) + ry^2) left to right, so rxc^2 + ryc^2 is a
// row term as well.
struct EpipolarGate {
  static constexpr bool kOn = true;
  static constexpr int kTerms = 4;                     // rxc, ryc, rwc, rxc^2 + ryc^2
  struct Q { double xq, yq, rx2, ry2; };
  __device__ __forceinline__ static Q query(const double* F, double x, double y, bool valid) {
    if (!valid) return Q{qnan(), qnan(), qnan(), qnan()};
    const double rx = F[0] * x + F[1] * y + F[2];
    const double ry = F[3] * x + F[4] * y + F[5];
    return Q{x, y, rx * rx, ry * ry};
  }
  __device__ __forceinline__ static void row(const double* F, double x, double y, double* o) {
    const double rxc = F[0] * x + F[3] * y + F[6];
    const double ryc = F[1] * x + F[4] * y + F[7];
    o[0] = rxc; o[1] = ryc; o[2] = F[2] * x + F[5] * y + F[8]; o[3] = rxc * rxc + ryc * ryc;
  }
  __device__ __forceinline__ static bool pass(const Q& q, const double* o, double th) {
    const double r = q.xq * o[0] + q.yq * o[1] + o[2];
    const double num = r * r;
    const double den = o[3] + q.rx2 + q.ry2;
    // Division-free pre-test on the same operands.  When t = th * den is a normal double it is at least
    // th * den * (1 - 2^-53) (den > 0 then, since th >= 0), so num > 2 t means num / den > 2 (1 - 2^-53) th >= 1.5 th.
    // The gap above any positive double is at most the double itself, so 1.5 th lies at or beyond the midpoint
    // between th and its successor: the rounded quotient exceeds th and the exact test below would fail too.  2 t is
    // exact or +inf (no rejection).  A zero, subnormal, infinite or NaN t, or a NaN num, goes to the exact test.
    const double t = th * den;
    if (t >= 2.2250738585072014e-308 && num > 2.0 * t) return false;
    return num / den <= th;
  }
};

// H (x_t ~ H x_q, row-major): the query's transfer (px, py) lies within px_th of the train point.  The transfer
// depends on the query only; w = 0 or a NaN model gives a NaN or infinite distance, which fails.
struct TransferGate {
  static constexpr bool kOn = true;
  static constexpr int kTerms = 2;                     // xt, yt
  struct Q { double px, py; };
  __device__ __forceinline__ static Q query(const double* H, double x, double y, bool valid) {
    if (!valid) return Q{qnan(), qnan()};
    const double w = H[6] * x + H[7] * y + H[8];
    return Q{(H[0] * x + H[1] * y + H[2]) / w, (H[3] * x + H[4] * y + H[5]) / w};
  }
  __device__ __forceinline__ static void row(const double*, double x, double y, double* o) { o[0] = x; o[1] = y; }
  __device__ __forceinline__ static bool pass(const Q& q, const double* o, double th) {
    const double dx = o[0] - q.px, dy = o[1] - q.py;
    return dx * dx + dy * dy <= th;
  }
};

// The gate of one pair as nn2_tile sees it: the model, the query and train images' keypoint rows, th.
struct GateCtx { const double* model; const double* kq; const double* kt; int kp_dim; double th; };

// The distances of the matcher.  Each has a 4-byte element, reads rows 16 bytes at a time and accumulates four train
// rows against one query row; key() maps a distance to 32 bits that order like it (the high word of col_best).
// The distance is kept as a float in nn_d1 / nn_d2 and in the selection: exact for Hamming, which is <= 2048.
struct L2Dist {             // squared L2 over float rows, FP32, accumulated in descriptor order
  using Elem = float;
  using Acc = float;
  __device__ __forceinline__ static void acc4(const float* A, const float* B0, int r1, int r2, int r3, int D, float& s0,
                                              float& s1, float& s2, float& s3) {
    for (int k = 0; k < D; k += 4) {
      const float4 av = *reinterpret_cast<const float4*>(A + k);
      const float4 v0 = *reinterpret_cast<const float4*>(B0 + k);
      const float4 v1 = *reinterpret_cast<const float4*>(B0 + (size_t)r1 * D + k);
      const float4 v2 = *reinterpret_cast<const float4*>(B0 + (size_t)r2 * D + k);
      const float4 v3 = *reinterpret_cast<const float4*>(B0 + (size_t)r3 * D + k);
      float d;
      d = av.x - v0.x; s0 = fmaf(d, d, s0); d = av.y - v0.y; s0 = fmaf(d, d, s0); d = av.z - v0.z; s0 = fmaf(d, d, s0); d = av.w - v0.w; s0 = fmaf(d, d, s0);
      d = av.x - v1.x; s1 = fmaf(d, d, s1); d = av.y - v1.y; s1 = fmaf(d, d, s1); d = av.z - v1.z; s1 = fmaf(d, d, s1); d = av.w - v1.w; s1 = fmaf(d, d, s1);
      d = av.x - v2.x; s2 = fmaf(d, d, s2); d = av.y - v2.y; s2 = fmaf(d, d, s2); d = av.z - v2.z; s2 = fmaf(d, d, s2); d = av.w - v2.w; s2 = fmaf(d, d, s2);
      d = av.x - v3.x; s3 = fmaf(d, d, s3); d = av.y - v3.y; s3 = fmaf(d, d, s3); d = av.z - v3.z; s3 = fmaf(d, d, s3); d = av.w - v3.w; s3 = fmaf(d, d, s3);
    }
  }
  __device__ __forceinline__ static uint32_t key(float s) { return __float_as_uint(s); }   // s >= 0
};
struct HammingDist {        // differing bits of binary rows of 32-bit words: one XOR and one POPC per word
  using Elem = uint32_t;
  using Acc = uint32_t;
  __device__ __forceinline__ static void acc4(const uint32_t* A, const uint32_t* B0, int r1, int r2, int r3, int D,
                                              uint32_t& s0, uint32_t& s1, uint32_t& s2, uint32_t& s3) {
    for (int k = 0; k < D; k += 4) {
      const uint4 av = *reinterpret_cast<const uint4*>(A + k);
      const uint4 v0 = *reinterpret_cast<const uint4*>(B0 + k);
      const uint4 v1 = *reinterpret_cast<const uint4*>(B0 + (size_t)r1 * D + k);
      const uint4 v2 = *reinterpret_cast<const uint4*>(B0 + (size_t)r2 * D + k);
      const uint4 v3 = *reinterpret_cast<const uint4*>(B0 + (size_t)r3 * D + k);
      s0 += __popc(av.x ^ v0.x) + __popc(av.y ^ v0.y) + __popc(av.z ^ v0.z) + __popc(av.w ^ v0.w);
      s1 += __popc(av.x ^ v1.x) + __popc(av.y ^ v1.y) + __popc(av.z ^ v1.z) + __popc(av.w ^ v1.w);
      s2 += __popc(av.x ^ v2.x) + __popc(av.y ^ v2.y) + __popc(av.z ^ v2.z) + __popc(av.w ^ v2.w);
      s3 += __popc(av.x ^ v3.x) + __popc(av.y ^ v3.y) + __popc(av.z ^ v3.z) + __popc(av.w ^ v3.w);
    }
  }
  __device__ __forceinline__ static uint32_t key(uint32_t s) { return s; }
};

// Two nearest train descriptors of the queries q0 .. q0+kTQ-1 of one pair under the distance Dist (ties go to the
// lowest train index), among the candidates the gate admits (NoGate: all).  d1 [n1][D], d2 [n2][D] elements; nn_* and
// col_best are the pair's own segments.  Called by all kMatchThreads threads of the CTA.
template <class Dist, class Gate>
__device__ __forceinline__ void nn2_tile(const typename Dist::Elem* d1, int n1, const typename Dist::Elem* d2, int n2,
                                         int D, int q0, int use_bulk, int mutual, int* nn_idx, float* nn_d1,
                                         float* nn_d2, unsigned long long* col_best, const GateCtx& gc) {
  using T = typename Dist::Elem;
  using Acc = typename Dist::Acc;
  extern __shared__ __align__(128) unsigned char msm[];
  __shared__ __align__(8) uint64_t bar[2];
  const int qs = D + 4;                                 // padded query row: conflict-free 128-bit reads across queries
  T* tq = reinterpret_cast<T*>(msm);                    // [kTQ][D + 4]
  T* tt = tq + kTQ * qs;                                // 2 stages x [kTT][D]
  const size_t stage_elems = (size_t)kTT * D;
  // gated: 2 stages x [kTT][kTerms] row terms (double buffered with the descriptors), then the pair's model [9]
  double* gt = reinterpret_cast<double*>(tt + 2 * stage_elems);
  double* gm = gt + 2 * kTT * Gate::kTerms;
  const int tid = threadIdx.x, q = tid & 31, g = tid >> 5;
  for (int i = tid; i < kTQ * D; i += kMatchThreads) {
    const int r = i / D, c = i % D;
    tq[r * qs + c] = (q0 + r < n1) ? d1[(size_t)(q0 + r) * D + c] : T(0);
  }
  if constexpr (Gate::kOn) {
    if (tid < 9) gm[tid] = gc.model[tid];
  }
  if (tid == 0) { mbar_init(&bar[0], 1); mbar_init(&bar[1], 1); }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  const int ntiles = (n2 + kTT - 1) / kTT;
  auto issue = [&](int t) {          // stage tile t (one elected thread; or cooperative loads when unaligned)
    const int rows = min(kTT, n2 - t * kTT);
    T* dst = tt + (size_t)(t & 1) * stage_elems;
    if (use_bulk) {
      if (tid == 0) {
        const uint32_t bytes = (uint32_t)(rows * D * sizeof(T));
        mbar_expect_tx(&bar[t & 1], bytes);
        bulk_g2s(dst, d2 + (size_t)t * kTT * D, bytes, &bar[t & 1]);
      }
    } else {
      const T* src = d2 + (size_t)t * kTT * D;
      for (int i = tid; i < rows * D; i += kMatchThreads) dst[i] = src[i];
    }
    if constexpr (Gate::kOn) {       // the gate's row terms of the tile, one thread per train row
      if (tid < rows) {
        const double* kp = gc.kt + ((size_t)t * kTT + tid) * gc.kp_dim;
        Gate::row(gm, kp[0], kp[1], gt + ((size_t)(t & 1) * kTT + tid) * Gate::kTerms);
      }
    }
  };
  typename Gate::Q gq;
  if constexpr (Gate::kOn) {
    const bool valid = q0 + q < n1;
    const double* kp = gc.kq + (size_t)(valid ? q0 + q : 0) * gc.kp_dim;
    gq = Gate::query(gm, kp[0], kp[1], valid);      // a query past n1 gets NaN terms: no candidate
  }
  float b1 = INFINITY, b2 = INFINITY;
  int i1 = -1;
  if (ntiles > 0) issue(0);
  if constexpr (Gate::kOn) __syncthreads();           // tile 0's row terms (later tiles: the loop's barrier)
  for (int t = 0; t < ntiles; ++t) {
    if (t + 1 < ntiles) issue(t + 1);                 // next tile in flight behind this one's math
    if (use_bulk) mbar_wait(&bar[t & 1], (uint32_t)((t >> 1) & 1)); else __syncthreads();
    const int rows = min(kTT, n2 - t * kTT);
    const T* B = tt + (size_t)(t & 1) * stage_elems;
    const T* A = tq + q * qs;
    // this thread: train rows g*16 .. g*16+15 of the tile, four at a time (query chunk loaded once per four rows)
    for (int jb = g * 16; jb < g * 16 + 16 && jb < rows; jb += 4) {
      bool ok[4] = {true, true, true, true};
      if constexpr (Gate::kOn) {
        // the gate of the four rows, then a warp vote: when it admits none of them for any of the warp's queries the
        // warp skips their distances (warp-uniform branch)
        const double* G = gt + ((size_t)(t & 1) * kTT + jb) * Gate::kTerms;
        bool any = false;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          ok[u] = jb + u < rows && Gate::pass(gq, G + u * Gate::kTerms, gc.th);
          any |= ok[u];
        }
        if (!__any_sync(0xffffffffu, any)) continue;
      }
      Acc s0 = 0, s1 = 0, s2 = 0, s3 = 0;
      const T* B0 = B + (size_t)jb * D;
      const int r1 = (jb + 1 < rows) ? 1 : 0, r2 = (jb + 2 < rows) ? 2 : 0, r3 = (jb + 3 < rows) ? 3 : 0;
      Dist::acc4(A, B0, r1, r2, r3, D, s0, s1, s2, s3);
      const Acc sv[4] = {s0, s1, s2, s3};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int j = jb + u;
        if (j < rows) {                                // (warp-uniform: g and rows are)
          const float s = (float)sv[u];
          const int gj = t * kTT + j;
          if (ok[u]) {                                 // (NoGate: always) a rejected candidate updates nothing
            if (s < b1 || (s == b1 && gj < i1)) { b2 = b1; b1 = s; i1 = gj; }
            else if (s < b2) b2 = s;
          }
          if (mutual) {
            // nearest QUERY of train descriptor gj among this warp's 32 queries, then one atomic per warp and row
            unsigned long long key = (ok[u] && q0 + q < n1)
                                         ? (((unsigned long long)Dist::key(sv[u]) << 32) | (unsigned)(q0 + q))
                                         : 0xffffffffffffffffull;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
              key = other < key ? other : key;
            }
            if (q == 0) atomicMin(col_best + gj, key);
          }
        }
      }
    }
    __syncthreads();    // everybody is done with stage t&1 before tile t+2 overwrites it
  }
  // merge the four train groups of each query (shared memory reuse: the query tile is dead)
  float* m1 = reinterpret_cast<float*>(msm);
  float* m2 = m1 + kMatchThreads;
  int* mi = reinterpret_cast<int*>(m2 + kMatchThreads);
  m1[tid] = b1; m2[tid] = b2; mi[tid] = i1;
  __syncthreads();
  if (g == 0 && q0 + q < n1) {
    float c1 = INFINITY, c2 = INFINITY;
    int ci = -1;
    for (int gg = 0; gg < 4; ++gg) {
      const float x1 = m1[gg * 32 + q], x2 = m2[gg * 32 + q];
      const int xi = mi[gg * 32 + q];
      if (xi >= 0 && (x1 < c1 || (x1 == c1 && xi < ci))) { c2 = c1; c1 = x1; ci = xi; }
      else if (x1 < c2) c2 = x1;
      if (x2 < c2) c2 = x2;
    }
    nn_idx[q0 + q] = ci; nn_d1[q0 + q] = c1; nn_d2[q0 + q] = c2;
  }
}

// One flat grid over the (pair, kTQ-query tile) work items of the whole batch: CTA b finds its pair by binary search
// over the tile prefix (the last pair whose first tile is <= b: pairs without tiles share their successor's prefix).
template <class Dist, class Gate>
__global__ void __launch_bounds__(kMatchThreads) nn2_kernel(MatchArgs a) {
  using T = typename Dist::Elem;
  const int b = blockIdx.x;
  int lo = 0, hi = a.n_pairs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.meta[mid].tile0 <= b) lo = mid; else hi = mid - 1;
  }
  const PairMeta m = a.meta[lo];
  GateCtx gc{};
  if constexpr (Gate::kOn)
    gc = GateCtx{a.models + (size_t)lo * 9, a.kq + (size_t)m.qrow * a.kp_dim, a.kt + (size_t)m.trow * a.kp_dim, a.kp_dim,
                 a.th};
  nn2_tile<Dist, Gate>((const T*)(a.qbank + (size_t)m.qrow * a.D), m.n1, (const T*)(a.tbank + (size_t)m.trow * a.D), m.n2,
                       a.D, (b - m.tile0) * kTQ, a.use_bulk, a.mutual, a.nn_idx + m.row0, a.nn_d1 + m.row0,
                       a.nn_d2 + m.row0, a.col_best + m.col0, gc);
}

// shared memory of nn2_kernel<Dist, Gate>: the query tile, two descriptor stages, and when gated two stages of row
// terms and the model (every element type of the descriptors is 4 bytes)
size_t nn2_smem_bytes(int D, int terms) {
  return sizeof(float) * ((size_t)kTQ * (D + 4) + 2 * (size_t)kTT * D) +
         (terms ? sizeof(double) * (2 * (size_t)kTT * terms + 9) : 0);
}

constexpr int kSelThreads = 512;

struct SelectArgs {
  const PairMeta* meta;
  const int* nn_idx; const float* nn_d1; const float* nn_d2;
  const unsigned long long* col_best;
  float ratio2; int mutual;
  int hamming; double ratio;                    // integer distances: the ratio test in FP64 on the distances themselves
  int* counts;                                  // [n_pairs] accepted matches per pair
};

// SNN ratio test (+ mutual check) of query q of the pair described by m; the accepted train index in *j
__device__ __forceinline__ bool accept_match(const SelectArgs& a, const PairMeta& m, int q, int* j) {
  *j = a.nn_idx[m.row0 + q];
  bool ok = *j >= 0;
  if (ok) {
    // d1 < ratio * d2 on the distances (simple-example.py:50): squared L2 against ratio^2 in FP32; Hamming distances
    // exactly as the example evaluates them on cv2's, in double
    const float d1 = a.nn_d1[m.row0 + q], d2 = a.nn_d2[m.row0 + q];
    ok = a.hamming ? (double)d1 < a.ratio * (double)d2 : d1 < a.ratio2 * d2;
  }
  if (ok && a.mutual) ok = (unsigned)(a.col_best[m.col0 + *j] & 0xffffffffu) == (unsigned)q;
  return ok;
}

// one CTA per pair: how many of its queries pass
__global__ void __launch_bounds__(kSelThreads) count_kernel(SelectArgs a) {
  __shared__ int wsum[kSelThreads / 32];
  const PairMeta m = a.meta[blockIdx.x];
  const int tid = threadIdx.x;
  int c = 0;
  if (m.n1 >= 1 && m.n2 >= 2)                   // degenerate pairs were not matched: zero matches
    for (int q = tid; q < m.n1; q += kSelThreads) { int j; c += accept_match(a, m, q, &j) ? 1 : 0; }
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((tid & 31) == 0) wsum[tid >> 5] = c;
  __syncthreads();
  if (tid == 0) {
    int tot = 0;
    for (int w = 0; w < kSelThreads / 32; ++w) tot += wsum[w];
    a.counts[blockIdx.x] = tot;
  }
}

// exclusive scan of the per-pair counts in one CTA: offsets[0] = 0, offsets[p+1] = offsets[p] + counts[p]; *count_out
// (when given) = min(offsets[n_pairs], cap)
__global__ void __launch_bounds__(1024) scan_kernel(const int* counts, int n_pairs, int* offsets, int cap, int* count_out) {
  __shared__ int wsum[32];
  __shared__ int base;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) { base = 0; offsets[0] = 0; }
  __syncthreads();
  for (int p0 = 0; p0 < n_pairs; p0 += 1024) {
    const int p = p0 + tid;
    const int v = p < n_pairs ? counts[p] : 0;
    int x = v;                                   // inclusive scan within the warp
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    int off = base;
    for (int w = 0; w < wid; ++w) off += wsum[w];
    if (p < n_pairs) offsets[p + 1] = off + x;
    __syncthreads();
    if (tid == 0) { int tot = 0; for (int w = 0; w < 32; ++w) tot += wsum[w]; base += tot; }
    __syncthreads();
  }
  if (tid == 0 && count_out) *count_out = base < cap ? base : cap;
}

struct WriteArgs {
  SelectArgs s;
  const int* offsets;                          // [n_pairs + 1] from scan_kernel
  const double* kq; const double* kt; int kp_dim;   // keypoint banks (rows like the descriptor banks) or nullptr
  int* match_q; int* match_t; double* x1y1; double* x2y2; int out_dim, cap;
};

// one CTA per pair: ORDERED compaction of its accepted matches into rows offsets[p] .. offsets[p+1]-1 (ascending query
// order), indices local to each image; gathers the keypoint coordinates into the float64 arrays the RANSAC entry
// points take.  Rows at or past `cap` are not written.
__global__ void __launch_bounds__(kSelThreads) write_kernel(WriteArgs a) {
  __shared__ int wsum[kSelThreads / 32];
  __shared__ int base;
  const PairMeta m = a.s.meta[blockIdx.x];
  if (m.n1 < 1 || m.n2 < 2) return;            // (block-uniform)
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) base = a.offsets[blockIdx.x];
  __syncthreads();
  for (int q0 = 0; q0 < m.n1; q0 += kSelThreads) {
    const int q = q0 + tid;
    int j = -1;
    const bool ok = q < m.n1 && accept_match(a.s, m, q, &j);
    const unsigned msk = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) wsum[wid] = __popc(msk);
    __syncthreads();
    int off = base;
    for (int w = 0; w < wid; ++w) off += wsum[w];
    off += __popc(msk & ((1u << lane) - 1u));
    if (ok && off < a.cap) {
      a.match_q[off] = q; a.match_t[off] = j;
      if (a.x1y1) {
        const double* k1 = a.kq + ((size_t)m.qrow + q) * a.kp_dim;
        const double* k2 = a.kt + ((size_t)m.trow + j) * a.kp_dim;
        for (int c = 0; c < a.out_dim; ++c) {
          a.x1y1[(size_t)off * a.out_dim + c] = k1[c];
          a.x2y2[(size_t)off * a.out_dim + c] = k2[c];
        }
      }
    }
    __syncthreads();
    if (tid == 0) { int tot = 0; for (int w = 0; w < kSelThreads / 32; ++w) tot += wsum[w]; base += tot; }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ pose from F
struct PoseArgs {
  const double* F; const double* K1; const double* K2;   // [P][9] row-major; K: [9] shared or [P][9]
  int k_per_pair;
  const double* x1y1; const double* x2y2; const unsigned char* mask;   // [P][n][dim], [P][n]
  int n_pairs, n, dim;
  double* R; double* t; int* good;   // [P][9], [P][3], [P]
};

__device__ inline void mat3_mul(const double* A, const double* B, double* C) {   // row-major C = A B
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
__device__ inline double det3r(const double* A) {
  return A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
}

// The pieces of pose from F that the dense and the ragged kernel share, so that both give the same bits.
// E = K2^T F K1, factored by the one-sided Jacobi SVD (la.h), and its four (R, t) candidates into cand[4][12] =
// (R row-major [9], t [3]) in the order (R1,+t), (R1,-t), (R2,+t), (R2,-t); t = the third column of U, unit length.
__device__ __forceinline__ void pose_candidates(const double* F, const double* K1, const double* K2, double* cand) {
  double K2t[9], tmp[9], E[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) K2t[3 * i + j] = K2[3 * j + i];
  mat3_mul(K2t, F, tmp);
  mat3_mul(tmp, K1, E);
  // E = U S V^T with G = E V (orthogonal columns, norms = singular values)
  double G[9], V[9], sv[3];
  dg::svd3_onesided(E, G, V, sv);
  int o[3] = {0, 1, 2};                   // sort singular values, largest first
  for (int i = 0; i < 3; ++i) for (int j = i + 1; j < 3; ++j) if (sv[o[j]] > sv[o[i]]) { const int tt = o[i]; o[i] = o[j]; o[j] = tt; }
  double U[9], Vs[9];
  for (int c = 0; c < 2; ++c) {
    const int k = o[c];
    const double inv = sv[k] > 0 ? 1.0 / sv[k] : 0.0;
    for (int r = 0; r < 3; ++r) { U[3 * r + c] = G[3 * r + k] * inv; Vs[3 * r + c] = V[3 * r + k]; }
  }
  {  // third columns: cross products (unit, orthogonal), so that det(U) = det(V) = +1
    const double u0[3] = {U[0], U[3], U[6]}, u1[3] = {U[1], U[4], U[7]}, v0[3] = {Vs[0], Vs[3], Vs[6]}, v1[3] = {Vs[1], Vs[4], Vs[7]};
    double cu[3], cv[3];
    dg::cross3(cu, u0, u1); dg::cross3(cv, v0, v1);
    for (int r = 0; r < 3; ++r) { U[3 * r + 2] = cu[r]; Vs[3 * r + 2] = cv[r]; }
  }
  const double W[9] = {0, -1, 0, 1, 0, 0, 0, 0, 1}, Wt[9] = {0, 1, 0, -1, 0, 0, 0, 0, 1};
  double Vt[9], UW[9], R1[9], R2[9];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Vt[3 * i + j] = Vs[3 * j + i];
  mat3_mul(U, W, UW); mat3_mul(UW, Vt, R1);
  mat3_mul(U, Wt, UW); mat3_mul(UW, Vt, R2);
  for (int c = 0; c < 4; ++c) {
    const double* Rc = (c < 2) ? R1 : R2;
    const double sgn = (c & 1) ? -1.0 : 1.0;
    for (int i = 0; i < 9; ++i) cand[12 * c + i] = Rc[i];
    for (int r = 0; r < 3; ++r) cand[12 * c + 9 + r] = sgn * U[3 * r + 2];
  }
}

// Normalised ray x = ki [px; py; 1] of a pixel.
__device__ __forceinline__ void pose_ray(const double* ki, double px, double py, double* x) {
  x[0] = ki[0] * px + ki[1] * py + ki[2];
  x[1] = ki[3] * px + ki[4] * py + ki[5];
  x[2] = ki[6] * px + ki[7] * py + ki[8];
}

// Two-view triangulation under (R, t): the least-squares depths (l1, l2) of l1 R x1 + t = l2 x2.
__device__ __forceinline__ void pose_depths(const double* Rc, const double* tc, const double* x1, const double* x2,
                                            double* l1, double* l2) {
  const double a1[3] = {Rc[0] * x1[0] + Rc[1] * x1[1] + Rc[2] * x1[2], Rc[3] * x1[0] + Rc[4] * x1[1] + Rc[5] * x1[2],
                        Rc[6] * x1[0] + Rc[7] * x1[1] + Rc[8] * x1[2]};
  // minimise | l1 a1 - l2 x2 + t |: normal equations of the 3 x 2 system [a1, -x2] (l1, l2)^T = -t
  const double aa = a1[0] * a1[0] + a1[1] * a1[1] + a1[2] * a1[2];
  const double bb = x2[0] * x2[0] + x2[1] * x2[1] + x2[2] * x2[2];
  const double ab = a1[0] * x2[0] + a1[1] * x2[1] + a1[2] * x2[2];
  const double at = a1[0] * tc[0] + a1[1] * tc[1] + a1[2] * tc[2];
  const double bt = x2[0] * tc[0] + x2[1] * tc[1] + x2[2] * tc[2];
  const double det = aa * bb - ab * ab;
  *l1 = (-at * bb + ab * bt) / det;
  *l2 = (aa * bt - ab * at) / det;
}

// One warp per pair.  Lane 0 factors E and builds the four candidates; all lanes vote: a correspondence supports
// (R, t) when its two-view triangulation (pose_depths) has both depths positive.  Result: the candidate with the most
// supporters (first in the order (R1,+t), (R1,-t), (R2,+t), (R2,-t) on ties), t of unit length.
__global__ void pose_kernel(PoseArgs a) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= a.n_pairs) return;
  const int p = warp;
  __shared__ double sh[8][4 * 12];        // per warp: 4 candidates x (R[9], t[3])
  double* cand = sh[(threadIdx.x >> 5) & 7];
  const double* K1 = a.K1 + (a.k_per_pair ? (size_t)p * 9 : 0);
  const double* K2 = a.K2 + (a.k_per_pair ? (size_t)p * 9 : 0);
  double k1i[9], k2i[9];
  {   // inverse of an upper-triangular-ish calibration matrix: general 3x3 inverse
    double m[9];
    for (int i = 0; i < 9; ++i) m[i] = K1[i];
    dg::inv3(m);
    for (int i = 0; i < 9; ++i) k1i[i] = m[i];
    for (int i = 0; i < 9; ++i) m[i] = K2[i];
    dg::inv3(m);
    for (int i = 0; i < 9; ++i) k2i[i] = m[i];
  }
  if (lane == 0) pose_candidates(a.F + (size_t)p * 9, K1, K2, cand);
  __syncwarp();
  int votes[4] = {0, 0, 0, 0};
  const double* g1 = a.x1y1 + (size_t)p * a.n * a.dim;
  const double* g2 = a.x2y2 + (size_t)p * a.n * a.dim;
  const unsigned char* mk = a.mask ? a.mask + (size_t)p * a.n : nullptr;
  for (int i = lane; i < a.n; i += 32) {
    if (mk && !mk[i]) continue;
    double x1[3], x2[3];
    pose_ray(k1i, g1[(size_t)i * a.dim], g1[(size_t)i * a.dim + 1], x1);
    pose_ray(k2i, g2[(size_t)i * a.dim], g2[(size_t)i * a.dim + 1], x2);
    for (int c = 0; c < 4; ++c) {
      double l1, l2;
      pose_depths(cand + 12 * c, cand + 12 * c + 9, x1, x2, &l1, &l2);
      if (l1 > 0 && l2 > 0) ++votes[c];
    }
  }
  for (int c = 0; c < 4; ++c)
    for (int o = 16; o > 0; o >>= 1) votes[c] += __shfl_xor_sync(0xffffffffu, votes[c], o);
  if (lane == 0) {
    int best = 0;
    for (int c = 1; c < 4; ++c) if (votes[c] > votes[best]) best = c;
    for (int i = 0; i < 9; ++i) a.R[(size_t)p * 9 + i] = cand[12 * best + i];
    for (int i = 0; i < 3; ++i) a.t[(size_t)p * 3 + i] = cand[12 * best + 9 + i];
    if (a.good) a.good[p] = votes[best];
  }
}

// ------------------------------------------------------------------------------------------------ pose, ragged
constexpr int kPoseThreads = 256;     // = the 256 bins of the median's radix select: one bin per thread

// The ragged layout and the per-row outputs that the two ragged pose kernels (from F, from H) share.
struct PoseRows {
  const double* K1; const double* K2;                      // K: [9] shared or [P][9], row-major
  int k_per_pair;
  const double* x1y1; const double* x2y2; const int* offsets; const unsigned char* mask;   // [rows][dim], [P+1], [rows]
  int n_pairs, rows, dim;
  double* points; unsigned char* in_front; double* angle;   // [rows][3], [rows], [rows]
  double* median;                                         // [P]
};

struct PoseRaggedArgs {
  PoseRows w;
  const double* F;                                        // [P][9] row-major
  double* R; double* t; int* good;                        // [P][9], [P][3], [P] (or null)
};

struct PoseHRaggedArgs {
  PoseRows w;
  const double* H;                                        // [P][9] row-major, x2 ~ H x1
  double* R; double* t; double* plane; int* good;         // [P][2][9], [P][2][3], [P][2][4], [P][2] (or null)
  unsigned char* rotation_only;                           // [P]
};

// Exclusive prefix of v over the CTA's threads (in thread order) and the CTA's total; ws: kPoseThreads / 32 ints.
// Called by all threads; ends with a barrier after which ws may be reused.
__device__ __forceinline__ int pose_block_scan(int v, int* ws, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) ws[wid] = x;
  __syncthreads();
  int off = 0, tot = 0;
  for (int w = 0; w < kPoseThreads / 32; ++w) { if (w < wid) off += ws[w]; tot += ws[w]; }
  __syncthreads();
  *total = tot;
  return off + x - v;
}

// Pair p's rows r0 .. r0 + n - 1; offsets that decrease, are negative or pass `rows` make an empty pair.
__device__ __forceinline__ void pose_span(const PoseRows& w, int p, int* r0, int* n) {
  const int b = w.offsets[p], e = w.offsets[p + 1];
  const bool span_ok = b >= 0 && b <= e && e <= w.rows;
  *r0 = span_ok ? b : 0;
  *n = span_ok ? e - b : 0;
}

// The rows of a pair without a model: NaN points and angles, in_front = 0.
__device__ __forceinline__ void pose_rows_void(const PoseRows& w, int r0, int n) {
  for (int i = threadIdx.x; i < n; i += kPoseThreads) {
    const size_t r = (size_t)r0 + i;
    for (int c = 0; c < 3; ++c) w.points[3 * r + c] = qnan();
    w.in_front[r] = 0;
    w.angle[r] = qnan();
  }
}

// The inverse calibrations K1^-1, K2^-1 of pair p into kinv[18] (dg::inv3, as pose_kernel).
__device__ __forceinline__ void pose_kinv(const PoseRows& w, int p, double* kinv) {
  const double* K1 = w.K1 + (w.k_per_pair ? (size_t)p * 9 : 0);
  const double* K2 = w.K2 + (w.k_per_pair ? (size_t)p * 9 : 0);
  for (int i = 0; i < 9; ++i) { kinv[i] = K1[i]; kinv[9 + i] = K2[i]; }
  dg::inv3(kinv);
  dg::inv3(kinv + 9);
}

// y = R^T x.
__device__ __forceinline__ void pose_back_rotate(const double* R, const double* x, double* y) {
  for (int c = 0; c < 3; ++c) y[c] = R[c] * x[0] + R[3 + c] * x[1] + R[6 + c] * x[2];
}

// The block's vote: per candidate c < NC, the rows with mask != 0 whose rays x1, x2 `supports(c, x1, x2)` accepts.
// Counted per thread, reduced per warp by shuffles and over the warps in a fixed order; the totals tot[NC] are valid
// in thread 0.  Called by all threads; ends with a barrier.
template <int NC, class Supports>
__device__ __forceinline__ void pose_vote(const PoseRows& w, int r0, int n, const double* kinv, Supports supports,
                                          int (*wvotes)[NC], int* tot) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const unsigned char* mk = w.mask;
  const double* g1 = w.x1y1;
  const double* g2 = w.x2y2;
  const int dim = w.dim;
  int votes[NC];
  for (int c = 0; c < NC; ++c) votes[c] = 0;
  for (int i = tid; i < n; i += kPoseThreads) {
    const size_t r = (size_t)r0 + i;
    if (mk && !mk[r]) continue;
    double x1[3], x2[3];
    pose_ray(kinv, g1[r * dim], g1[r * dim + 1], x1);
    pose_ray(kinv + 9, g2[r * dim], g2[r * dim + 1], x2);
    for (int c = 0; c < NC; ++c)
      if (supports(c, x1, x2)) ++votes[c];
  }
  for (int c = 0; c < NC; ++c)
    for (int o = 16; o > 0; o >>= 1) votes[c] += __shfl_xor_sync(0xffffffffu, votes[c], o);
  if (lane == 0) for (int c = 0; c < NC; ++c) wvotes[wid][c] = votes[c];
  __syncthreads();
  if (tid == 0) {
    for (int c = 0; c < NC; ++c) tot[c] = 0;
    for (int v = 0; v < kPoseThreads / 32; ++v) for (int c = 0; c < NC; ++c) tot[c] += wvotes[v][c];
  }
}

// Per row under the pose (R, t): the parallax angle atan2(|x1 x R^T x2|, x1 . R^T x2) and
//   translation (rotation = false): in_front = mask && l1 > 0 && l2 > 0 with (l1, l2) of pose_depths, the midpoint
//     0.5 (l1 x1 + R^T (l2 x2 - t)) in camera 1's frame;
//   pure rotation (rotation = true, t unused): in_front = mask && x1 . R^T x2 > 0, NaN points (no depth).
__device__ __forceinline__ void pose_rows_under(const PoseRows& w, int r0, int n, const double* kinv, const double* Rb,
                                                const double* tb, bool rotation) {
  const unsigned char* mk = w.mask;
  const double* g1 = w.x1y1;
  const double* g2 = w.x2y2;
  const int dim = w.dim;
  for (int i = threadIdx.x; i < n; i += kPoseThreads) {
    const size_t r = (size_t)r0 + i;
    double x1[3], x2[3], y[3];                     // y = R^T x2
    pose_ray(kinv, g1[r * dim], g1[r * dim + 1], x1);
    pose_ray(kinv + 9, g2[r * dim], g2[r * dim + 1], x2);
    if (rotation) {
      pose_back_rotate(Rb, x2, y);
      w.in_front[r] = (!mk || mk[r]) && x1[0] * y[0] + x1[1] * y[1] + x1[2] * y[2] > 0;
      for (int c = 0; c < 3; ++c) w.points[3 * r + c] = qnan();
    } else {
      double l1, l2, q[3];                         // q = l2 x2 - t
      pose_depths(Rb, tb, x1, x2, &l1, &l2);
      w.in_front[r] = (!mk || mk[r]) && l1 > 0 && l2 > 0;
      for (int c = 0; c < 3; ++c) {
        y[c] = Rb[c] * x2[0] + Rb[3 + c] * x2[1] + Rb[6 + c] * x2[2];
        q[c] = l2 * x2[c] - tb[c];
      }
      for (int c = 0; c < 3; ++c)
        w.points[3 * r + c] = 0.5 * (l1 * x1[c] + (Rb[c] * q[0] + Rb[3 + c] * q[1] + Rb[6 + c] * q[2]));
    }
    const double cx = x1[1] * y[2] - x1[2] * y[1], cy = x1[2] * y[0] - x1[0] * y[2], cz = x1[0] * y[1] - x1[1] * y[0];
    w.angle[r] = atan2(sqrt(cx * cx + cy * cy + cz * cz), x1[0] * y[0] + x1[1] * y[1] + x1[2] * y[2]);
  }
}

// The median of the angles of the pair's in-front rows, count > 0 of them, read back from global memory after a
// barrier: a radix select over the bit patterns of the (non-negative) doubles, eight 8-bit digits from the top, which
// needs no workspace and no bound on the row count.  An even count averages the two middle values as np.median does.
// Called by all threads after the row pass; the result is valid in thread 0.
__device__ __forceinline__ double pose_median(const PoseRows& w, int r0, int n, int count) {
  __shared__ int ws[kPoseThreads / 32];
  __shared__ unsigned hist[256];
  __shared__ int s_digit, s_below, s_eq;
  __shared__ unsigned long long s_min[kPoseThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  __syncthreads();                                 // this CTA's angle / in_front rows are visible to all its threads

  // k-th smallest key (k = (count - 1) / 2) among the in-front rows: fix 8 bits per pass, from the top
  int k = (count - 1) >> 1;
  unsigned long long prefix = 0, known = 0;
  for (int shift = 56; shift >= 0; shift -= 8) {
    hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += kPoseThreads) {
      const size_t r = (size_t)r0 + i;
      if (!w.in_front[r]) continue;
      const unsigned long long key = (unsigned long long)__double_as_longlong(w.angle[r]);
      if ((key & known) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    const int h = (int)hist[tid];
    int tot;
    const int below = pose_block_scan(h, ws, &tot);
    if (below <= k && k < below + h) { s_digit = tid; s_below = below; s_eq = h; }
    __syncthreads();
    k -= s_below;
    prefix |= (unsigned long long)s_digit << shift;
    known |= 255ull << shift;
  }
  const double lo = __longlong_as_double((long long)prefix);
  if (count & 1) return lo;
  // even count: the next order statistic is lo again when lo has further copies, else the smallest key above it
  double hi = lo;
  if (k + 1 >= s_eq) {                             // (block-uniform)
    unsigned long long m = ~0ull;
    for (int i = tid; i < n; i += kPoseThreads) {
      const size_t r = (size_t)r0 + i;
      if (!w.in_front[r]) continue;
      const unsigned long long key = (unsigned long long)__double_as_longlong(w.angle[r]);
      if (key > prefix && key < m) m = key;
    }
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, m, o);
      m = other < m ? other : m;
    }
    if (lane == 0) s_min[wid] = m;
    __syncthreads();
    if (tid == 0) {
      for (int v = 1; v < kPoseThreads / 32; ++v) m = s_min[v] < m ? s_min[v] : m;
      hi = __longlong_as_double((long long)m);
    }
  }
  return (lo + hi) / 2.0;
}

// The rows and the median of a pair under its chosen pose (pose_rows_under, then pose_median); count = the pair's
// in-front rows, known from the vote.  Called by all threads.
__device__ __forceinline__ void pose_rows_and_median(const PoseRows& w, int p, int r0, int n, const double* kinv,
                                                     const double* Rb, const double* tb, bool rotation, int count) {
  pose_rows_under(w, r0, n, kinv, Rb, tb, rotation);
  if (count == 0) {                                // (block-uniform)
    if (threadIdx.x == 0) w.median[p] = qnan();
    return;
  }
  const double med = pose_median(w, r0, n, count);
  if (threadIdx.x == 0) w.median[p] = med;
}

// One CTA per pair p, rows b = offsets[p] .. e = offsets[p+1]-1.
//   pass 1: thread 0 builds the four candidates (pose_candidates), thread 1 the inverse calibrations;
//   pass 2: the block votes over the rows with mask != 0 (pose_depths), first candidate wins ties -- the arithmetic and
//           tie rule of pose_kernel, so R, t, good are those of a dense call on the pair alone;
//   pass 3: per row under the chosen (R, t) (pose_rows_under);
//   pass 4: the median of the angles of the in-front rows (pose_median).
// A pair whose F is all zero (no model) or holds a NaN gets R = t = 0, good = 0, NaN points and angles, in_front = 0,
// median NaN.  Offsets that decrease, are negative or pass `rows` make an empty pair: no row is read or written.
__global__ void __launch_bounds__(kPoseThreads) pose_ragged_kernel(PoseRaggedArgs a) {
  __shared__ double cand[4 * 12];
  __shared__ double kinv[18];
  __shared__ int wvotes[kPoseThreads / 32][4];
  __shared__ int s_best;
  const int p = blockIdx.x, tid = threadIdx.x;
  int r0, n;
  pose_span(a.w, p, &r0, &n);
  const double* F = a.F + (size_t)p * 9;
  bool zero = true, has_nan = false;
  for (int i = 0; i < 9; ++i) { zero &= F[i] == 0.0; has_nan |= F[i] != F[i]; }
  if (zero || has_nan) {                          // (block-uniform)
    pose_rows_void(a.w, r0, n);
    if (tid < 9) a.R[(size_t)p * 9 + tid] = 0.0;
    if (tid < 3) a.t[(size_t)p * 3 + tid] = 0.0;
    if (tid == 0) {
      if (a.good) a.good[p] = 0;
      a.w.median[p] = qnan();
    }
    return;
  }
  if (tid == 0)
    pose_candidates(F, a.w.K1 + (a.w.k_per_pair ? (size_t)p * 9 : 0), a.w.K2 + (a.w.k_per_pair ? (size_t)p * 9 : 0),
                    cand);
  if (tid == 1) pose_kinv(a.w, p, kinv);
  __syncthreads();

  int tot[4];
  pose_vote<4>(a.w, r0, n, kinv, [&](int c, const double* x1, const double* x2) {
    double l1, l2;
    pose_depths(cand + 12 * c, cand + 12 * c + 9, x1, x2, &l1, &l2);
    return l1 > 0 && l2 > 0;
  }, wvotes, tot);
  if (tid == 0) {
    int best = 0;
    for (int c = 1; c < 4; ++c) if (tot[c] > tot[best]) best = c;
    s_best = best;
    wvotes[0][0] = tot[best];
    if (a.good) a.good[p] = tot[best];
  }
  __syncthreads();
  const int best = s_best, count = wvotes[0][0];
  const double* Rb = cand + 12 * best;
  const double* tb = Rb + 9;
  if (tid < 9) a.R[(size_t)p * 9 + tid] = Rb[tid];
  if (tid < 3) a.t[(size_t)p * 3 + tid] = tb[tid];
  pose_rows_and_median(a.w, p, r0, n, kinv, Rb, tb, false, count);
}

// ------------------------------------------------------------------------------------------------ pose from H, ragged
constexpr double kRotationTol = 1e-3;   // max |Hn^T Hn - I| below which Hn is taken for a rotation (cv2's rule)

// Candidates of pose from a homography, FP64 on one thread, into cand[4][16] = (R row-major [9], t [3], n [3], d).
// Hn = K2^-1 H K1 divided by its middle singular value (dg::svd3_onesided) and negated when det(Hn) < 0.
//   max |S_ij| < kRotationTol with S = Hn^T Hn - I: a pure rotation, ONE candidate: R = U V^T (the rotation nearest to
//     Hn), t = 0, n = d = NaN.  Returns 1.
//   otherwise the four decompositions Hn = R + t' n^T, |n| = 1, of Malis & Vargas (INRIA RR-6303, 2007, section 4, the
//     analytical method) in the order (Ra, t'a, na), (Ra, -t'a, -na), (Rb, t'b, nb), (Rb, -t'b, -nb) -- the order of
//     cv2.decomposeHomographyMat -- stored as t = t' / |t'| and the plane n^T X = d, d = 1 / |t'|.  Returns 4.
__device__ int pose_h_candidates(const double* H, const double* K1, const double* K2, double* cand) {
  double Hn[9];
  {
    double K2i[9], T[9];
    for (int i = 0; i < 9; ++i) K2i[i] = K2[i];
    dg::inv3(K2i);
    mat3_mul(K2i, H, T);
    mat3_mul(T, K1, Hn);
  }
  double G[9], V[9], sv[3];
  dg::svd3_onesided(Hn, G, V, sv);
  const double mid = fmax(fmin(sv[0], sv[1]), fmin(fmax(sv[0], sv[1]), sv[2]));
  for (int i = 0; i < 9; ++i) Hn[i] /= mid;
  if (det3r(Hn) < 0) for (int i = 0; i < 9; ++i) Hn[i] = -Hn[i];
  double S[9], smax = 0.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      S[3 * i + j] = Hn[i] * Hn[j] + Hn[3 + i] * Hn[3 + j] + Hn[6 + i] * Hn[6 + j] - (i == j ? 1.0 : 0.0);
      smax = fmax(smax, fabs(S[3 * i + j]));
    }
  if (smax < kRotationTol) {
    dg::svd3_onesided(Hn, G, V, sv);               // Hn = U diag(sv) V^T, U = G diag(1 / sv)
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j)
        cand[3 * i + j] = G[3 * i] / sv[0] * V[3 * j] + G[3 * i + 1] / sv[1] * V[3 * j + 1] +
                          G[3 * i + 2] / sv[2] * V[3 * j + 2];
    for (int i = 9; i < 12; ++i) cand[i] = 0.0;
    for (int i = 12; i < 16; ++i) cand[i] = qnan();
    return 1;
  }
  // opposites of the principal minors of S (>= 0), and of the off-diagonal ones (their signs pick the roots)
  const double s11 = S[0], s12 = S[1], s13 = S[2], s22 = S[4], s23 = S[5], s33 = S[8];
  const double m11 = s23 * s23 - s22 * s33, m22 = s13 * s13 - s11 * s33, m33 = s12 * s12 - s11 * s22;
  const double m12 = s23 * s13 - s12 * s33, m13 = s22 * s13 - s12 * s23, m23 = s12 * s13 - s11 * s23;
  const double r11 = sqrt(fmax(m11, 0.0)), r22 = sqrt(fmax(m22, 0.0)), r33 = sqrt(fmax(m33, 0.0));
  const double d1 = fabs(s11), d2 = fabs(s22), d3 = fabs(s33);
  const int ii = (d1 >= d2 && d1 >= d3) ? 0 : (d2 >= d3 ? 1 : 2);   // the largest |s_ii| keeps n' away from zero
  double na[3], nb[3], es;
  if (ii == 0) {
    const double e = m23 >= 0 ? 1.0 : -1.0;
    na[0] = s11; na[1] = s12 + r33; na[2] = s13 + e * r22;
    nb[0] = s11; nb[1] = s12 - r33; nb[2] = s13 - e * r22;
    es = s11 >= 0 ? 1.0 : -1.0;
  } else if (ii == 1) {
    const double e = m13 >= 0 ? 1.0 : -1.0;
    na[0] = s12 + r33; na[1] = s22; na[2] = s23 - e * r11;
    nb[0] = s12 - r33; nb[1] = s22; nb[2] = s23 + e * r11;
    es = s22 >= 0 ? 1.0 : -1.0;
  } else {
    const double e = m12 >= 0 ? 1.0 : -1.0;
    na[0] = s13 + e * r22; na[1] = s23 + r11; na[2] = s33;
    nb[0] = s13 - e * r22; nb[1] = s23 - r11; nb[2] = s33;
    es = s33 >= 0 ? 1.0 : -1.0;
  }
  const double la = sqrt(na[0] * na[0] + na[1] * na[1] + na[2] * na[2]);
  const double lb = sqrt(nb[0] * nb[0] + nb[1] * nb[1] + nb[2] * nb[2]);
  for (int i = 0; i < 3; ++i) { na[i] /= la; nb[i] /= lb; }
  const double tr = s11 + s22 + s33;
  const double nu = 2.0 * sqrt(fmax(1.0 + tr - m11 - m22 - m33, 0.0));
  const double rho = sqrt(2.0 + tr + nu);
  const double te = sqrt(fmax(2.0 + tr - nu, 0.0));
  for (int s = 0; s < 2; ++s) {                    // s = 0: (Ra, t'a, na), s = 1: (Rb, t'b, nb)
    const double* n1 = s ? nb : na;
    const double* n2 = s ? na : nb;
    double ts[3], R[9], t[3];                      // ts = R^T t': t' in camera 1's frame
    for (int i = 0; i < 3; ++i) ts[i] = 0.5 * te * (es * rho * n2[i] - te * n1[i]);
    {
      double M[9];                                 // R = Hn (I - (2 / nu) ts n^T)
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) M[3 * i + j] = (i == j ? 1.0 : 0.0) - (2.0 / nu) * ts[i] * n1[j];
      mat3_mul(Hn, M, R);
    }
    for (int i = 0; i < 3; ++i) t[i] = R[3 * i] * ts[0] + R[3 * i + 1] * ts[1] + R[3 * i + 2] * ts[2];
    const double tn = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    for (int c = 0; c < 2; ++c) {                  // c = 1: (R, -t', -n)
      double* o = cand + 16 * (2 * s + c);
      const double sg = c ? -1.0 : 1.0;
      for (int i = 0; i < 9; ++i) o[i] = R[i];
      for (int i = 0; i < 3; ++i) { o[9 + i] = sg * t[i] / tn; o[12 + i] = sg * n1[i]; }
      o[15] = 1.0 / tn;
    }
  }
  return 4;
}

// One CTA per pair p over the ragged layout of pose_ragged_kernel.
//   pass 1: thread 0 builds the candidates (pose_h_candidates), thread 1 the inverse calibrations;
//   pass 2: the block votes over the rows with mask != 0: a candidate (R, t) is supported by a row when pose_depths
//           gives both depths positive; the rotation by a row with x1 . R^T x2 > 0.  Candidate 0 is the one with the
//           most votes, candidate 1 the one with the most among the rest, ties to the earlier candidate;
//   passes 3, 4: the rows under candidate 0 and the median, as pose_ragged_kernel (pose_rows_and_median).
// A rotation-only pair's candidate 1 is R = t = 0, plane NaN, good 0.  A pair whose H is all zero (no model) or holds a
// NaN gets R = t = 0 and plane NaN for both candidates, good 0, NaN points and angles, in_front = 0, median NaN.  Offsets
// that decrease, are negative or pass `rows` make an empty pair: no row is read or written.
__global__ void __launch_bounds__(kPoseThreads) pose_h_ragged_kernel(PoseHRaggedArgs a) {
  __shared__ double cand[4 * 16];
  __shared__ double kinv[18];
  __shared__ int wvotes[kPoseThreads / 32][4];
  __shared__ int s_nc, s_first, s_count;
  const int p = blockIdx.x, tid = threadIdx.x;
  int r0, n;
  pose_span(a.w, p, &r0, &n);
  const double* H = a.H + (size_t)p * 9;
  bool zero = true, has_nan = false;
  for (int i = 0; i < 9; ++i) { zero &= H[i] == 0.0; has_nan |= H[i] != H[i]; }
  if (zero || has_nan) {                          // (block-uniform)
    pose_rows_void(a.w, r0, n);
    if (tid < 18) a.R[(size_t)p * 18 + tid] = 0.0;
    if (tid < 6) a.t[(size_t)p * 6 + tid] = 0.0;
    if (tid < 8) a.plane[(size_t)p * 8 + tid] = qnan();
    if (tid < 2 && a.good) a.good[(size_t)p * 2 + tid] = 0;
    if (tid == 0) {
      a.rotation_only[p] = 0;
      a.w.median[p] = qnan();
    }
    return;
  }
  if (tid == 0)
    s_nc = pose_h_candidates(H, a.w.K1 + (a.w.k_per_pair ? (size_t)p * 9 : 0),
                             a.w.K2 + (a.w.k_per_pair ? (size_t)p * 9 : 0), cand);
  if (tid == 1) pose_kinv(a.w, p, kinv);
  __syncthreads();

  const int nc = s_nc;
  const bool rotation = nc == 1;
  int tot[4];
  pose_vote<4>(a.w, r0, n, kinv, [&](int c, const double* x1, const double* x2) {
    if (c >= nc) return false;
    const double* Rc = cand + 16 * c;
    if (rotation) {
      double y[3];
      pose_back_rotate(Rc, x2, y);
      return x1[0] * y[0] + x1[1] * y[1] + x1[2] * y[2] > 0;
    }
    double l1, l2;
    pose_depths(Rc, Rc + 9, x1, x2, &l1, &l2);
    return l1 > 0 && l2 > 0;
  }, wvotes, tot);
  if (tid == 0) {
    int first = 0, second = -1;
    for (int c = 1; c < nc; ++c) if (tot[c] > tot[first]) first = c;
    for (int c = 0; c < nc; ++c) if (c != first && (second < 0 || tot[c] > tot[second])) second = c;
    for (int slot = 0; slot < 2; ++slot) {
      const int c = slot ? second : first;
      const double* o = cand + 16 * (c < 0 ? 0 : c);
      for (int i = 0; i < 9; ++i) a.R[(size_t)p * 18 + 9 * slot + i] = c < 0 ? 0.0 : o[i];
      for (int i = 0; i < 3; ++i) a.t[(size_t)p * 6 + 3 * slot + i] = c < 0 ? 0.0 : o[9 + i];
      for (int i = 0; i < 4; ++i) a.plane[(size_t)p * 8 + 4 * slot + i] = c < 0 ? qnan() : o[12 + i];
      if (a.good) a.good[(size_t)p * 2 + slot] = c < 0 ? 0 : tot[c];
    }
    a.rotation_only[p] = rotation;
    s_first = first;
    s_count = tot[first];
  }
  __syncthreads();
  const double* Rb = cand + 16 * s_first;
  pose_rows_and_median(a.w, p, r0, n, kinv, Rb, Rb + 9, rotation, s_count);
}

// ------------------------------------------------------------------------------------------------ pose refinement, ragged
struct PoseRefineArgs {
  const double* R; const double* t; const double* K1; const double* K2;   // [P][9], [P][3]; K: [9] shared or [P][9]
  int k_per_pair;
  const double* x1y1; const double* x2y2; const int* offsets; const unsigned char* mask;   // [rows][dim], [P+1], [rows]
  int n_pairs, rows, dim, max_iters;
  double th2;                                              // px_th^2 of the inlier rows
  double* R_out; double* t_out; double* F_out;             // [P][9], [P][3], [P][9]
  double* cost0; double* cost; int* n_used; int* iters;    // [P] (cost0, n_used, iters may be null)
  unsigned char* inliers;                                  // [rows] or null
};

// One pass over the pair's rows with mask != 0 at the linearisation (F, dF) in shared memory: the cost, J^T J and J^T r
// (dg::pr_row) summed over the CTA into out[kPrSums], the number of rows into *count.  A fixed-shape tree: butterfly
// shuffles inside each warp, then thread j < kPrSums adds the warps' partials of sum j in warp order -- no atomics, so
// the sums of a pair do not depend on the batch it is in or on the run.  Called by all threads; ends with a barrier.
__device__ __forceinline__ void pose_refine_pass(const PoseRefineArgs& a, int r0, int n, const double* F, const double* dF,
                                                 double (*wpart)[dg::kPrSums], int* wcount, double* out, int* count) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const unsigned char* mk = a.mask;
  const double* g1 = a.x1y1;
  const double* g2 = a.x2y2;
  const int dim = a.dim;
  double acc[dg::kPrSums];
#pragma unroll
  for (int j = 0; j < dg::kPrSums; ++j) acc[j] = 0.0;
  int cnt = 0;
  for (int i = tid; i < n; i += kPoseThreads) {
    const size_t r = (size_t)r0 + i;
    if (mk && !mk[r]) continue;
    ++cnt;
    dg::pr_row(F, dF, g1[r * dim], g1[r * dim + 1], g2[r * dim], g2[r * dim + 1], acc);
  }
#pragma unroll
  for (int j = 0; j < dg::kPrSums; ++j)
    for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < dg::kPrSums; ++j) wpart[wid][j] = acc[j];
    wcount[wid] = cnt;
  }
  __syncthreads();
  if (tid < dg::kPrSums) {
    double s = wpart[0][tid];
    for (int w = 1; w < kPoseThreads / 32; ++w) s += wpart[w][tid];
    out[tid] = s;
  } else if (tid == dg::kPrSums) {
    int c = 0;
    for (int w = 0; w < kPoseThreads / 32; ++w) c += wcount[w];
    *count = c;
  }
  __syncthreads();
}

// One CTA per pair p, rows b = offsets[p] .. e = offsets[p+1]-1: Levenberg-Marquardt with Marquardt scaling on the
// Sampson cost C(R, t) = sum of f_resid_sampson over the rows with mask != 0, from the pose given (pose_refine.h has the
// residual, its analytic Jacobian and the local parameters).
//   start:  thread 0 linearises at (R, t); one pass gives C, H = J^T J, g = J^T r there; lambda = 1e-3.
//   trial:  thread 0 solves (H + lambda diag H) D = -g (5 x 5 Cholesky; a pivot that is not positive rejects the step
//           without a pass), moves to the trial pose and linearises there; one pass gives the trial C', H', g'.
//           C' < C: the trial pose and its sums become current, lambda <- max(lambda / 10, 1e-12).  Otherwise the
//           current sums stay, lambda <- 10 lambda, stop when lambda > 1e8.  Either way |C - C'| < 1e-12 C stops the
//           refinement: at the minimum a trial step moves the cost by rounding only, up as often as down.
//   So k trial steps read the rows at most k + 1 times, from global memory (a pair's rows stay in L2).
//   end:    R re-orthonormalised if an accepted step left |R R^T - I| above 1e-12; F = K2^-T [t]x R K1^-1 scaled to unit
//           Frobenius norm; with inliers_out one more pass over ALL the pair's rows: f_resid_sampson(F, ..) <= th2.
// Fewer than kPrMinRows rows with mask != 0: the pose is passed through, cost0 = cost = its cost, iters = 0.  R all zero
// or a NaN in R or t (no model): R = t = F = 0, NaN costs, n_used = iters = 0, inlier rows 0.  Offsets that decrease, are
// negative or pass `rows`: the same per-pair outputs and no row is read or written.  R_out / t_out may be R / t: the
// pose is read into shared memory before the first barrier and written after it.
__global__ void __launch_bounds__(kPoseThreads) pose_refine_ragged_kernel(PoseRefineArgs a) {
  __shared__ double kinv[18];                      // K1^-1, K2^-1
  __shared__ double kA[9];                         // K2^-T
  __shared__ double pose[2][12];                   // current and trial (R [9], t [3])
  __shared__ double lin[54];                       // F [9], dF [5][9] of the pass to come; at the end the output F
  __shared__ double cur[dg::kPrSums], trial[dg::kPrSums];
  __shared__ double wpart[kPoseThreads / 32][dg::kPrSums];
  __shared__ int wcount[kPoseThreads / 32];
  __shared__ int s_count, s_go;
  const int p = blockIdx.x, tid = threadIdx.x;
  const int b = a.offsets[p], e = a.offsets[p + 1];
  const bool span_ok = b >= 0 && b <= e && e <= a.rows;
  const int r0 = span_ok ? b : 0, n = span_ok ? e - b : 0;
  if (tid < 9) pose[0][tid] = a.R[(size_t)p * 9 + tid];
  else if (tid < 12) pose[0][tid] = a.t[(size_t)p * 3 + tid - 9];
  __syncthreads();                                 // the pose is read: the outputs may overwrite it
  bool zero = true, has_nan = false;
  for (int i = 0; i < 12; ++i) { zero &= i >= 9 || pose[0][i] == 0.0; has_nan |= pose[0][i] != pose[0][i]; }
  if (!span_ok || zero || has_nan) {               // (block-uniform)
    if (a.inliers) for (int i = tid; i < n; i += kPoseThreads) a.inliers[(size_t)r0 + i] = 0;
    if (tid < 9) { a.R_out[(size_t)p * 9 + tid] = 0.0; a.F_out[(size_t)p * 9 + tid] = 0.0; }
    if (tid < 3) a.t_out[(size_t)p * 3 + tid] = 0.0;
    if (tid == 0) {
      a.cost[p] = qnan();
      if (a.cost0) a.cost0[p] = qnan();
      if (a.n_used) a.n_used[p] = 0;
      if (a.iters) a.iters[p] = 0;
    }
    return;
  }
  if (tid == 0) {                                  // the inverse calibrations (dg::inv3, as the pose kernels)
    const double* K1 = a.K1 + (a.k_per_pair ? (size_t)p * 9 : 0);
    const double* K2 = a.K2 + (a.k_per_pair ? (size_t)p * 9 : 0);
    for (int i = 0; i < 9; ++i) { kinv[i] = K1[i]; kinv[9 + i] = K2[i]; }
    dg::inv3(kinv);
    dg::inv3(kinv + 9);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) kA[3 * i + j] = kinv[9 + 3 * j + i];
    dg::pr_linearise(pose[0], pose[0] + 9, kA, kinv, lin, lin + 9);
  }
  __syncthreads();
  pose_refine_pass(a, r0, n, lin, lin + 9, wpart, wcount, cur, &s_count);
  const int n_used = s_count;
  const double cost0 = cur[0];
  double lam = dg::kPrLambda0;
  int iters = 0, accepted = 0;
  while (n_used >= dg::kPrMinRows && iters < a.max_iters) {   // (block-uniform: every thread keeps the same lam, iters)
    ++iters;
    if (tid == 0) {
      double D[5];
      s_go = dg::pr_solve(cur + 1, cur + 16, lam, D) ? 1 : 0;
      if (s_go) {
        dg::pr_step(pose[0], pose[0] + 9, D, pose[1], pose[1] + 9);
        dg::pr_linearise(pose[1], pose[1] + 9, kA, kinv, lin, lin + 9);
      }
    }
    __syncthreads();
    const bool go = s_go != 0;
    if (go) pose_refine_pass(a, r0, n, lin, lin + 9, wpart, wcount, trial, &s_count);
    const double c_old = cur[0], c_new = trial[0];
    const bool better = go && c_new < c_old;
    const bool flat = go && fabs(c_old - c_new) < dg::kPrRelDecrease * c_old;   // converged: the cost no longer moves
    __syncthreads();                               // s_go, cur[0], trial[0] are read: they may change
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
  if (tid == 0) {
    if (accepted && dg::pr_ortho_drift(pose[0]) > dg::kPrOrthoTol) dg::pr_orthonormalise(pose[0]);
    double F[9];
    dg::pr_fundamental(pose[0], pose[0] + 9, kA, kinv, F);
    double nrm = 0.0;
    for (int i = 0; i < 9; ++i) nrm += F[i] * F[i];
    const double inv = nrm > 0.0 ? 1.0 / sqrt(nrm) : 0.0;
    for (int i = 0; i < 9; ++i) lin[i] = F[i] * inv;
  }
  __syncthreads();
  if (tid < 9) { a.R_out[(size_t)p * 9 + tid] = pose[0][tid]; a.F_out[(size_t)p * 9 + tid] = lin[tid]; }
  if (tid < 3) a.t_out[(size_t)p * 3 + tid] = pose[0][9 + tid];
  if (tid == 0) {
    a.cost[p] = cur[0];
    if (a.cost0) a.cost0[p] = cost0;
    if (a.n_used) a.n_used[p] = n_used;
    if (a.iters) a.iters[p] = iters;
  }
  if (a.inliers) {
    const int dim = a.dim;
    for (int i = tid; i < n; i += kPoseThreads) {
      const size_t r = (size_t)r0 + i;
      a.inliers[r] = dg::f_resid_sampson(lin, a.x1y1[r * dim], a.x1y1[r * dim + 1], a.x2y2[r * dim], a.x2y2[r * dim + 1]) <= a.th2;
    }
  }
}

// ------------------------------------------------------------------------------------------------ H refinement, ragged
// The arguments of the H and F refinements: a 3 x 3 model per pair and its ragged rows
struct RefineArgs {
  const double* model;                                     // [P][9] row-major: H (x2 ~ H x1) or F (x2^T F x1 = 0)
  const double* x1y1; const double* x2y2; const int* offsets; const unsigned char* mask;   // [rows][dim], [P+1], [rows]
  int n_pairs, rows, dim, max_iters;
  double th2;                                              // px_th^2 of the inlier rows
  double* model_out; double* cost0; double* cost; int* n_used; int* iters;   // [P][9], [P] (cost0, n_used, iters may be null)
  unsigned char* inliers;                                  // [rows] or null
};

// One pass over the pair's rows with mask != 0: row(x1, y1, x2, y2, acc) adds the row's NS sums, which are reduced
// over the CTA into out[NS], the number of rows into *count -- the fixed-shape tree of pose_refine_pass (butterfly
// shuffles in each warp, then thread j < NS adds the warps' partials of sum j in warp order; no atomics).  Called by
// all threads; ends with a barrier.  wpart holds the largest NS of its callers, the 45 sums of the H refinement.
template <int NS, class Row>
__device__ __forceinline__ void refine_pass(const RefineArgs& a, int r0, int n, Row row,
                                            double (*wpart)[dg::kRhSums], int* wcount, double* out, int* count) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const unsigned char* mk = a.mask;
  const double* g1 = a.x1y1;
  const double* g2 = a.x2y2;
  const int dim = a.dim;
  double acc[NS];
#pragma unroll
  for (int j = 0; j < NS; ++j) acc[j] = 0.0;
  int cnt = 0;
  for (int i = tid; i < n; i += kPoseThreads) {
    const size_t r = (size_t)r0 + i;
    if (mk && !mk[r]) continue;
    ++cnt;
    row(g1[r * dim], g1[r * dim + 1], g2[r * dim], g2[r * dim + 1], acc);
  }
#pragma unroll
  for (int j = 0; j < NS; ++j)
    for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < NS; ++j) wpart[wid][j] = acc[j];
    wcount[wid] = cnt;
  }
  __syncthreads();
  if (tid < NS) {
    double s = wpart[0][tid];
    for (int w = 1; w < kPoseThreads / 32; ++w) s += wpart[w][tid];
    out[tid] = s;
  } else if (tid == NS) {
    int c = 0;
    for (int w = 0; w < kPoseThreads / 32; ++w) c += wcount[w];
    *count = c;
  }
  __syncthreads();
}

// The row of the first pass of both refinements: the sums x, y, x^2, y^2 of each image that rh_transform takes
struct RefineNormRow {
  __device__ __forceinline__ void operator()(double x1, double y1, double x2, double y2, double* acc) const {
    acc[0] += x1; acc[1] += y1; acc[2] += x1 * x1; acc[3] += y1 * y1;
    acc[4] += x2; acc[5] += y2; acc[6] += x2 * x2; acc[7] += y2 * y2;
  }
};

// Thread 0's serial part of a trial step: D of the damped normal equations (cur: the current sums), the trial model
// M2 = M (+) D and the linearisation there into lin.  0 when the solve rejects the step.  Not inlined: the 8 x 8 factor
// then lives in this function's frame instead of competing with the row passes for the kernel's registers.
__device__ __noinline__ int h_refine_trial(const double* cur, double lam, const double* tr, const double* M, double* M2,
                                           double* lin) {
  double D[8];
  if (!dg::pr_cholesky_solve<8>(cur + 1, cur + 37, lam, D)) return 0;
  dg::rh_step(M, D, M2);
  dg::rh_linearise(tr, tr + 3, M2, lin, lin + 9);
  return 1;
}

// One CTA per pair p, rows b = offsets[p] .. e = offsets[p+1]-1: Levenberg-Marquardt with Marquardt scaling on the
// Sampson cost C = sum of h_resid_sampson(G, row) over the rows with mask != 0, G = H^-1 the engine's image-2 -> image-1
// model (refine_h.h has the whitened residuals, their analytic Jacobian and the 8 local parameters).
//   start:  thread 0 takes G = adj(H) / det(H); one pass sums x, y, x^2, y^2 of the masked rows of each image, thread 0
//           forms T1, T2, M = T1 G T2^-1 / |.|_F and linearises there; one pass gives C, J^T J, J^T z; lambda = 1e-3.
//   trial:  the schedule of pose_refine_ragged_kernel with an 8 x 8 Cholesky solve: (J^T J + lambda diag J^T J) D =
//           -J^T z, a pivot that is not positive rejects the step without a pass; C' < C accepts it (lambda <-
//           max(lambda / 10, 1e-12)), else lambda <- 10 lambda, stop when lambda > 1e8; |C - C'| < 1e-12 C stops.
//   end:    H = adj(T1^-1 M T2) after an accepted step, else the input H; scaled to unit Frobenius norm, det H > 0.  With
//           inliers_out one more pass over ALL the pair's rows: h_resid_sampson(H_out^-1, row) <= th2.
// Fewer than kRhMinRows rows with mask != 0: H is passed through (normalised), cost0 = cost, iters = 0.  H all zero, a NaN
// in H or an inverse that is not finite (no model): H = 0, NaN costs, n_used = iters = 0, inlier rows 0.  Offsets that
// decrease, are negative or pass `rows`: the same per-pair outputs and no row is read or written.  H_out may be H: H
// is read into shared memory before the first barrier and written after it.
__global__ void __launch_bounds__(kPoseThreads) h_refine_ragged_kernel(RefineArgs a) {
  __shared__ double hio[9];                        // the input H; at the end the output H
  __shared__ double tr[6];                         // T1, T2 as (s, mx, my)
  __shared__ double model[2][9];                   // current and trial M
  __shared__ double lin[81];                       // G [9], dG [8][9] of the pass to come; at the end H_out^-1
  __shared__ double cur[dg::kRhSums], trial[dg::kRhSums];
  __shared__ double wpart[kPoseThreads / 32][dg::kRhSums];
  __shared__ int wcount[kPoseThreads / 32];
  __shared__ int s_count, s_go;
  const int p = blockIdx.x, tid = threadIdx.x;
  const int b = a.offsets[p], e = a.offsets[p + 1];
  const bool span_ok = b >= 0 && b <= e && e <= a.rows;
  const int r0 = span_ok ? b : 0, n = span_ok ? e - b : 0;
  if (tid < 9) hio[tid] = a.model[(size_t)p * 9 + tid];
  __syncthreads();                                 // H is read: the outputs may overwrite it
  if (tid == 0) s_go = dg::rh_engine_model(hio, lin) ? 1 : 0;
  __syncthreads();
  if (!span_ok || !s_go) {                         // (block-uniform)
    if (a.inliers) for (int i = tid; i < n; i += kPoseThreads) a.inliers[(size_t)r0 + i] = 0;
    if (tid < 9) a.model_out[(size_t)p * 9 + tid] = 0.0;
    if (tid == 0) {
      a.cost[p] = qnan();
      if (a.cost0) a.cost0[p] = qnan();
      if (a.n_used) a.n_used[p] = 0;
      if (a.iters) a.iters[p] = 0;
    }
    return;
  }
  refine_pass<dg::kRhNormSums>(a, r0, n, RefineNormRow(), wpart, wcount, trial, &s_count);
  const int n_used = s_count;
  auto lm_row = [](const double* G, const double* dG) {
    return [G, dG](double x1, double y1, double x2, double y2, double* acc) { dg::rh_row(G, dG, x1, y1, x2, y2, acc); };
  };
  if (tid == 0) {
    dg::rh_transform(trial, n_used, tr);
    dg::rh_transform(trial + 4, n_used, tr + 3);
    double G[9];
    for (int i = 0; i < 9; ++i) G[i] = lin[i];
    dg::rh_from_pixels(tr, tr + 3, G, model[0]);
    dg::rh_linearise(tr, tr + 3, model[0], lin, lin + 9);
  }
  __syncthreads();
  refine_pass<dg::kRhSums>(a, r0, n, lm_row(lin, lin + 9), wpart, wcount, cur, &s_count);
  const double cost0 = cur[0];
  double lam = dg::kPrLambda0;
  int iters = 0, accepted = 0;
  while (n_used >= dg::kRhMinRows && iters < a.max_iters) {   // (block-uniform: every thread keeps the same lam, iters)
    ++iters;
    if (tid == 0) s_go = h_refine_trial(cur, lam, tr, model[0], model[1], lin);
    __syncthreads();
    const bool go = s_go != 0;
    if (go) refine_pass<dg::kRhSums>(a, r0, n, lm_row(lin, lin + 9), wpart, wcount, trial, &s_count);
    const double c_old = cur[0], c_new = trial[0];
    const bool better = go && c_new < c_old;
    const bool flat = go && fabs(c_old - c_new) < dg::kPrRelDecrease * c_old;   // converged: the cost no longer moves
    __syncthreads();                               // s_go, cur[0], trial[0] are read: they may change
    if (better) {
      if (tid < dg::kRhSums) cur[tid] = trial[tid];
      if (tid < 9) model[0][tid] = model[1][tid];
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
  if (tid == 0) {
    if (accepted) {
      double G[9];
      dg::rh_to_pixels(tr, tr + 3, model[0], G);
      dg::rh_public_model(G, hio);
    } else {
      dg::rh_unit_det_pos(hio);
    }
    dg::rh_engine_model(hio, lin);
  }
  __syncthreads();
  if (tid < 9) a.model_out[(size_t)p * 9 + tid] = hio[tid];
  if (tid == 0) {
    a.cost[p] = cur[0];
    if (a.cost0) a.cost0[p] = cost0;
    if (a.n_used) a.n_used[p] = n_used;
    if (a.iters) a.iters[p] = iters;
  }
  if (a.inliers) {
    const int dim = a.dim;
    for (int i = tid; i < n; i += kPoseThreads) {
      const size_t r = (size_t)r0 + i;
      a.inliers[r] = dg::h_resid_sampson(lin, a.x1y1[r * dim], a.x1y1[r * dim + 1], a.x2y2[r * dim], a.x2y2[r * dim + 1]) <= a.th2;
    }
  }
}

// ------------------------------------------------------------------------------------------------ F refinement, ragged
// Thread 0's serial part of a trial step: D of the damped normal equations (cur: the current sums), the trial model
// Fn2 = unit(rank2(Fn + B D)) and the linearisation there into lin.  0 when the solve rejects the step.  Not inlined,
// as h_refine_trial: the 7 x 7 factor and the rank-2 projection live in this function's frame.
__device__ __noinline__ int f_refine_trial(const double* cur, double lam, const double* tr, const double* Fn, double* Fn2,
                                           double* lin) {
  double D[7];
  if (!dg::pr_cholesky_solve<7>(cur + 1, cur + 29, lam, D)) return 0;
  dg::rf_retract(Fn, D, Fn2);
  dg::rf_linearise(tr, tr + 3, Fn2, lin, lin + 9);
  return 1;
}

// Thread 0's start: T1, T2 from the sums ns [8] of n rows, the start point Fn0 = unit(rank2(T2^-T F T1^-1)) and the
// linearisation there into lin.  Not inlined, as f_refine_trial.
__device__ __noinline__ void f_refine_start(const double* ns, int n, const double* F, double* tr, double* Fn,
                                            double* lin) {
  dg::rh_transform(ns, n, tr);
  dg::rh_transform(ns + 4, n, tr + 3);
  dg::rf_start(tr, tr + 3, F, Fn);
  dg::rf_linearise(tr, tr + 3, Fn, lin, lin + 9);
}

// One CTA per pair p, rows b = offsets[p] .. e = offsets[p+1]-1: Levenberg-Marquardt with Marquardt scaling on the
// Sampson cost C = sum of f_resid_sampson(F, row) over the rows with mask != 0 (refine_f.h has the normalisation, the
// 7 local parameters over the rank-2 matrices and the retraction; the residual and its Jacobian are pr_row's).
//   start:  one pass sums x, y, x^2, y^2 of the masked rows of each image; thread 0 forms T1, T2, the start point
//           Fn0 = unit(rank2(T2^-T F T1^-1)) and linearises there; one pass gives C, J^T J, J^T r; lambda = 1e-3.
//   trial:  the schedule of h_refine_ragged_kernel with a 7 x 7 Cholesky solve and the step Fn <- unit(rank2(Fn + B d)).
//   end:    F = T2^T Fn T1 at unit Frobenius norm, signed so that <F, F_in> >= 0 (the start point when no step was
//           accepted).  With inliers_out one more pass over ALL the pair's rows: f_resid_sampson(F_out, row) <= th2.
// Fewer than kRfMinRows rows with mask != 0: the start point is passed through, cost0 = cost, iters = 0.  F all zero or
// not finite (no model): F = 0, NaN costs, n_used = iters = 0, inlier rows 0.  Offsets that decrease, are negative or
// pass `rows`: the same per-pair outputs and no row is read or written.  F_out may be F: F is read into shared memory
// before the first barrier and written after it.
__global__ void __launch_bounds__(kPoseThreads) f_refine_ragged_kernel(RefineArgs a) {
  __shared__ double fin[9];                        // the input F
  __shared__ double tr[6];                         // T1, T2 as (s, mx, my)
  __shared__ double model[2][9];                   // current and trial Fn
  __shared__ double lin[72];                       // F [9], dF [7][9] of the pass to come; at the end the output F
  __shared__ double cur[dg::kRfSums], trial[dg::kRfSums];
  __shared__ double wpart[kPoseThreads / 32][dg::kRhSums];
  __shared__ int wcount[kPoseThreads / 32];
  __shared__ int s_count, s_go;
  const int p = blockIdx.x, tid = threadIdx.x;
  const int b = a.offsets[p], e = a.offsets[p + 1];
  const bool span_ok = b >= 0 && b <= e && e <= a.rows;
  const int r0 = span_ok ? b : 0, n = span_ok ? e - b : 0;
  if (tid < 9) fin[tid] = a.model[(size_t)p * 9 + tid];
  __syncthreads();                                 // F is read: the outputs may overwrite it
  if (!span_ok || !dg::rf_has_model(fin)) {        // (block-uniform)
    if (a.inliers) for (int i = tid; i < n; i += kPoseThreads) a.inliers[(size_t)r0 + i] = 0;
    if (tid < 9) a.model_out[(size_t)p * 9 + tid] = 0.0;
    if (tid == 0) {
      a.cost[p] = qnan();
      if (a.cost0) a.cost0[p] = qnan();
      if (a.n_used) a.n_used[p] = 0;
      if (a.iters) a.iters[p] = 0;
    }
    return;
  }
  refine_pass<dg::kRhNormSums>(a, r0, n, RefineNormRow(), wpart, wcount, trial, &s_count);
  const int n_used = s_count;
  auto lm_row = [](const double* F, const double* dF) {
    return [F, dF](double x1, double y1, double x2, double y2, double* acc) { dg::pr_row_n<7, true>(F, dF, x1, y1, x2, y2, acc); };
  };
  if (tid == 0) f_refine_start(trial, n_used, fin, tr, model[0], lin);
  __syncthreads();
  refine_pass<dg::kRfSums>(a, r0, n, lm_row(lin, lin + 9), wpart, wcount, cur, &s_count);
  const double cost0 = cur[0];
  double lam = dg::kPrLambda0;
  int iters = 0;
  while (n_used >= dg::kRfMinRows && iters < a.max_iters) {   // (block-uniform: every thread keeps the same lam, iters)
    ++iters;
    if (tid == 0) s_go = f_refine_trial(cur, lam, tr, model[0], model[1], lin);
    __syncthreads();
    const bool go = s_go != 0;
    if (go) refine_pass<dg::kRfSums>(a, r0, n, lm_row(lin, lin + 9), wpart, wcount, trial, &s_count);
    const double c_old = cur[0], c_new = trial[0];
    const bool better = go && c_new < c_old;
    const bool flat = go && fabs(c_old - c_new) < dg::kPrRelDecrease * c_old;   // converged: the cost no longer moves
    __syncthreads();                               // s_go, cur[0], trial[0] are read: they may change
    if (better) {
      if (tid < dg::kRfSums) cur[tid] = trial[tid];
      if (tid < 9) model[0][tid] = model[1][tid];
    }
    __syncthreads();
    if (better) {
      lam = fmax(lam / 10.0, dg::kPrLambdaMin);
      if (flat) break;
    } else {
      lam *= 10.0;
      if (flat || lam > dg::kPrLambdaMax) break;
    }
  }
  if (tid == 0) dg::rf_output(tr, tr + 3, model[0], fin, lin);
  __syncthreads();
  if (tid < 9) a.model_out[(size_t)p * 9 + tid] = lin[tid];
  if (tid == 0) {
    a.cost[p] = cur[0];
    if (a.cost0) a.cost0[p] = cost0;
    if (a.n_used) a.n_used[p] = n_used;
    if (a.iters) a.iters[p] = iters;
  }
  if (a.inliers) {
    const int dim = a.dim;
    for (int i = tid; i < n; i += kPoseThreads) {
      const size_t r = (size_t)r0 + i;
      a.inliers[r] = dg::f_resid_sampson(lin, a.x1y1[r * dim], a.x1y1[r * dim + 1], a.x2y2[r * dim], a.x2y2[r * dim + 1]) <= a.th2;
    }
  }
}

// ------------------------------------------------------------------------------------------------ QR null space
__global__ void qr7x9_kernel(const double* A, double* N, int* rc, int count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  double a[63], n[18];
  for (int k = 0; k < 63; ++k) a[k] = A[(size_t)i * 63 + k];
  for (int k = 0; k < 18; ++k) n[k] = 0.0;
  const int r = dg::nullspace_qr7x9(a, n);
  for (int k = 0; k < 18; ++k) N[(size_t)i * 18 + k] = n[k];
  if (rc) rc[i] = r;
}

// ------------------------------------------------------------------------------------------------ division check
// Bit-for-bit comparison of the shared-reciprocal quotients used by h_pinvJ (hgeom.h) with IEEE division on random
// operands spanning 60 binary orders of magnitude; returns the number of mismatches in *bad.
__global__ void div_check_kernel(unsigned long long seed, long long count, unsigned long long* bad) {
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long local = 0;
  for (long long i = i0; i < count; i += (long long)gridDim.x * blockDim.x) {
    uint32_t o[4];
    dg::philox4x32_10((uint32_t)i, (uint32_t)(i >> 32), 7u, 0u, (uint32_t)seed, (uint32_t)(seed >> 32), o);
    // mantissas from 52 random bits, exponents in [-30, 30], random signs
    const unsigned long long mx = ((unsigned long long)o[0] << 20) ^ o[1], mn = ((unsigned long long)o[2] << 20) ^ o[3];
    const int ex = (int)(o[1] % 61u) - 30, en = (int)(o[3] % 61u) - 30;
    double x = __longlong_as_double((long long)(((unsigned long long)(1023 + ex) << 52) | (mx & 0xfffffffffffffull)));
    double n = __longlong_as_double((long long)(((unsigned long long)(1023 + en) << 52) | (mn & 0xfffffffffffffull)));
    if (o[0] & 1u) x = -x;
    if (o[2] & 1u) n = -n;
    const double q = dg::div_by_shared_rcp(x, n, __drcp_rn(n));
    if (__double_as_longlong(q) != __double_as_longlong(x / n)) ++local;
  }
  if (local) atomicAdd(bad, local);
}

// ------------------------------------------------------------------------------------------------ matcher, host side
// Workspace of a batch: per-pair metadata, counts and (single-pair calls) offsets, then col_best [sum n2] and the
// per-query 2-NN results [sum n1]; every segment 256-byte aligned.
size_t match_ws_bytes(long long sum_n1, long long sum_n2, int n_pairs) {
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  return al(sizeof(PairMeta) * ((size_t)n_pairs + 1)) + 2 * al(sizeof(int) * ((size_t)n_pairs + 1)) +
         al(sizeof(unsigned long long) * (size_t)sum_n2) + 3 * al(sizeof(int) * (size_t)sum_n1);
}

// Pair metadata from the image offsets of the query and train banks (equal for a batch over one bank) and the pair
// table [n_pairs][2] = (query image, train image).  Rejects malformed input; meta[n_pairs] holds the totals.
int build_meta(const int32_t* qoff, const int32_t* toff, int n_images, const int32_t* pairs, int n_pairs,
               std::vector<PairMeta>* meta) {
  if (!qoff || !toff || !pairs) return fail(DGB200_E_ARG, "null image offsets or pair table");
  if (n_images < 1 || n_pairs < 1) return fail(DGB200_E_ARG, "need n_images >= 1 and n_pairs >= 1");
  for (const int32_t* off : {qoff, toff}) {
    if (off[0] != 0) return fail(DGB200_E_ARG, "image offsets must start at 0");
    for (int i = 0; i < n_images; ++i)
      if (off[i + 1] < off[i]) return fail(DGB200_E_ARG, "image offsets must be non-decreasing");
  }
  meta->assign((size_t)n_pairs + 1, PairMeta{});
  long long tiles = 0, rows = 0, cols = 0;
  for (int p = 0; p < n_pairs; ++p) {
    const int qi = pairs[2 * p], ti = pairs[2 * p + 1];
    if (qi < 0 || qi >= n_images || ti < 0 || ti >= n_images) return fail(DGB200_E_ARG, "pair table: image index out of range");
    PairMeta& m = (*meta)[p];
    m.qrow = qoff[qi]; m.n1 = qoff[qi + 1] - qoff[qi];
    m.trow = toff[ti]; m.n2 = toff[ti + 1] - toff[ti];
    m.tile0 = (int)tiles; m.row0 = (int)rows; m.col0 = (int)cols;
    if (m.n1 >= 1 && m.n2 >= 2) tiles += (m.n1 + kTQ - 1) / kTQ;   // degenerate pairs: no work, zero matches
    rows += m.n1;
    cols += m.n2;
    if (rows > INT32_MAX || cols > INT32_MAX) return fail(DGB200_E_ARG, "batch too large: more than 2^31 - 1 rows");
  }
  PairMeta& e = (*meta)[n_pairs];
  e.tile0 = (int)tiles; e.row0 = (int)rows; e.col0 = (int)cols;
  return 0;
}

// The matcher over a checked batch, asynchronous on st: metadata upload, 2-NN over all work items, per-pair counts,
// scan, ordered write.  The banks hold float rows of D floats (squared L2; ratio is a float's value) or, when
// `hamming`, binary rows of D 32-bit words.  offsets == nullptr: a workspace segment holds them.  guide: kNoGuide, or
// DGB200_GUIDE_F / DGB200_GUIDE_H with per-pair models [P][9] and the squared threshold th (the keypoint banks then
// give the gate its coordinates).
constexpr int kNoGuide = -1;
int run_match(const void* qbank, const void* tbank, int D, int hamming, const std::vector<PairMeta>& meta, double ratio,
              int mutual, const double* kq, const double* kt, int kp_dim, int* match_q, int* match_t, double* x1y1,
              double* x2y2, int out_dim, int cap, int* offsets, int* count_out, void* workspace, cudaStream_t st,
              int guide = kNoGuide, const double* models = nullptr, double th = 0.0) {
  const int P = (int)meta.size() - 1;
  const PairMeta& tot = meta[P];
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  unsigned char* w = (unsigned char*)workspace;
  PairMeta* d_meta = (PairMeta*)w; w += al(sizeof(PairMeta) * ((size_t)P + 1));
  int* counts = (int*)w; w += al(sizeof(int) * ((size_t)P + 1));
  int* ws_offsets = (int*)w; w += al(sizeof(int) * ((size_t)P + 1));
  MatchArgs a;
  a.col_best = (unsigned long long*)w; w += al(sizeof(unsigned long long) * (size_t)tot.col0);
  a.nn_idx = (int*)w; w += al(sizeof(int) * (size_t)tot.row0);
  a.nn_d1 = (float*)w; w += al(sizeof(float) * (size_t)tot.row0);
  a.nn_d2 = (float*)w;
  if (!offsets) offsets = ws_offsets;
  a.qbank = (const float*)qbank; a.tbank = (const float*)tbank; a.meta = d_meta; a.n_pairs = P; a.D = D;
  a.use_bulk = (((uintptr_t)tbank) & 15) == 0 ? 1 : 0;   // every image's rows then are too (D % 4 == 0)
  a.mutual = mutual;
  a.models = models; a.kq = kq; a.kt = kt; a.kp_dim = kp_dim; a.th = th;
  // pageable source: the runtime stages it before returning, the copy itself is ordered on st like the kernels
  CU(cudaMemcpyAsync(d_meta, meta.data(), sizeof(PairMeta) * meta.size(), cudaMemcpyHostToDevice, st));
  if (tot.tile0 > 0) {
    if (mutual) CU(cudaMemsetAsync(a.col_best, 0xff, sizeof(unsigned long long) * (size_t)tot.col0, st));
    void (*kern)(MatchArgs);
    size_t smem;
    if (guide == DGB200_GUIDE_F) {
      kern = hamming ? nn2_kernel<HammingDist, EpipolarGate> : nn2_kernel<L2Dist, EpipolarGate>;
      smem = nn2_smem_bytes(D, EpipolarGate::kTerms);
    } else if (guide == DGB200_GUIDE_H) {
      kern = hamming ? nn2_kernel<HammingDist, TransferGate> : nn2_kernel<L2Dist, TransferGate>;
      smem = nn2_smem_bytes(D, TransferGate::kTerms);
    } else {
      kern = hamming ? nn2_kernel<HammingDist, NoGate> : nn2_kernel<L2Dist, NoGate>;
      smem = nn2_smem_bytes(D, 0);
    }
    CU(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<tot.tile0, kMatchThreads, smem, st>>>(a);
    CU(cudaGetLastError());
  }
  SelectArgs s;
  s.meta = d_meta; s.nn_idx = a.nn_idx; s.nn_d1 = a.nn_d1; s.nn_d2 = a.nn_d2; s.col_best = a.col_best;
  s.ratio2 = (float)ratio * (float)ratio; s.mutual = mutual; s.counts = counts;
  s.hamming = hamming; s.ratio = ratio;
  count_kernel<<<P, kSelThreads, 0, st>>>(s);
  CU(cudaGetLastError());
  scan_kernel<<<1, 1024, 0, st>>>(counts, P, offsets, cap, count_out);
  CU(cudaGetLastError());
  WriteArgs wa;
  wa.s = s; wa.offsets = offsets; wa.kq = kq; wa.kt = kt; wa.kp_dim = kp_dim;
  wa.match_q = match_q; wa.match_t = match_t; wa.x1y1 = x1y1; wa.x2y2 = x2y2; wa.out_dim = out_dim; wa.cap = cap;
  write_kernel<<<P, kSelThreads, 0, st>>>(wa);
  CU(cudaGetLastError());
  return 0;
}

// Row lengths: float rows of D floats, binary rows of n_words 32-bit words.  The error message, or nullptr when valid.
const char* float_len_error(int D) {
  return (D < 4 || D > 256 || (D & 3)) ? "descriptor length must be a multiple of 4 in [4, 256]" : nullptr;
}
const char* word_len_error(int n_words) {
  return (n_words < 4 || n_words > 64 || (n_words & 3)) ? "binary descriptor length must be a multiple of 4 in [4, 64] words"
                                                        : nullptr;
}

// One pair (dgb200_match_descriptors_dev and its binary twin): a batch of one pair, image 0 the query image in the
// first bank, image 1 the train image in the second.  len_err: the row length's float_len_error / word_len_error.
int match_single(const void* d_desc1, int n1, const void* d_desc2, int n2, int D, const char* len_err, int hamming,
                 double ratio, int mutual, const double* d_kp1, const double* d_kp2, int kp_dim, int* d_match_q,
                 int* d_match_t, double* d_x1y1, double* d_x2y2, int out_dim, int capacity, int* d_count,
                 void* d_workspace, void* stream) {
  if (!d_desc1 || !d_desc2 || !d_match_q || !d_match_t || !d_count || !d_workspace) return fail(DGB200_E_ARG, "null buffer");
  if (n1 < 1 || n2 < 2) return fail(DGB200_E_ARG, "need n1 >= 1 query and n2 >= 2 train descriptors");
  if (len_err) return fail(DGB200_E_ARG, len_err);
  if (d_x1y1 && (!d_kp1 || !d_kp2 || !d_x2y2 || out_dim < 2 || out_dim > kp_dim)) return fail(DGB200_E_ARG, "keypoint arrays / out_dim inconsistent");
  const int32_t qoff[3] = {0, n1, n1}, toff[3] = {0, 0, n2}, pair[2] = {0, 1};
  std::vector<PairMeta> meta;
  const int rc = build_meta(qoff, toff, 2, pair, 1, &meta);
  if (rc) return rc;
  return run_match(d_desc1, d_desc2, D, hamming, meta, ratio, mutual, d_kp1, d_kp2, kp_dim, d_match_q, d_match_t, d_x1y1,
                   d_x2y2, out_dim, capacity, nullptr, d_count, d_workspace, (cudaStream_t)stream);
}

// Many pairs over one bank (dgb200_match_descriptors_batch_dev and its binary twin; with a guide, the guided twins).
int match_batch(const void* d_bank, const int32_t* img_offsets, int n_images, int D, const char* len_err, int hamming,
                const int32_t* pairs, int n_pairs, double ratio, int mutual, const double* d_kp_bank, int kp_dim,
                int* d_match_q, int* d_match_t, double* d_x1y1, double* d_x2y2, int out_dim, int capacity,
                int32_t* d_offsets_out, void* d_workspace, void* stream, bool guided = false, int guide = kNoGuide,
                const double* d_models = nullptr, double px_th = 0.0) {
  if (!d_match_q || !d_match_t || !d_offsets_out || !d_workspace) return fail(DGB200_E_ARG, "null buffer");
  if (len_err) return fail(DGB200_E_ARG, len_err);
  if (d_x1y1 && (!d_kp_bank || !d_x2y2 || out_dim < 2 || out_dim > kp_dim)) return fail(DGB200_E_ARG, "keypoint arrays / out_dim inconsistent");
  if (guided) {
    if (!d_models) return fail(DGB200_E_ARG, "null model array");
    if (!d_kp_bank || kp_dim < 2) return fail(DGB200_E_ARG, "guided matching needs the keypoint bank (kp_dim >= 2)");
    if (guide != DGB200_GUIDE_F && guide != DGB200_GUIDE_H) return fail(DGB200_E_ARG, "guide must be DGB200_GUIDE_F or DGB200_GUIDE_H");
    if (!(px_th >= 0.0)) return fail(DGB200_E_ARG, "px_th must be a non-negative number");
  }
  std::vector<PairMeta> meta;
  const int rc = build_meta(img_offsets, img_offsets, n_images, pairs, n_pairs, &meta);
  if (rc) return rc;
  if (!d_bank && meta[n_pairs].tile0 > 0) return fail(DGB200_E_ARG, "null descriptor bank");
  if (capacity < meta[n_pairs].row0) return fail(DGB200_E_ARG, "capacity below the sum of the query images' descriptor counts");
  return run_match(d_bank, d_bank, D, hamming, meta, ratio, mutual, d_kp_bank, d_kp_bank, kp_dim, d_match_q, d_match_t,
                   d_x1y1, d_x2y2, out_dim, capacity, d_offsets_out, nullptr, d_workspace, (cudaStream_t)stream,
                   guided ? guide : kNoGuide, d_models, px_th * px_th);
}

PoseRows pose_rows_args(const double* K1, const double* K2, int k_per_pair, const double* x1y1, const double* x2y2,
                        const int32_t* offsets, int n_pairs, int rows, int dim, const uint8_t* mask, double* points,
                        uint8_t* in_front, double* angle, double* median) {
  PoseRows w;
  w.K1 = K1; w.K2 = K2; w.k_per_pair = k_per_pair; w.x1y1 = x1y1; w.x2y2 = x2y2; w.offsets = offsets; w.mask = mask;
  w.n_pairs = n_pairs; w.rows = rows; w.dim = dim; w.points = points; w.in_front = in_front; w.angle = angle;
  w.median = median;
  return w;
}

// The checks the ragged pose and refine entry points share, in their order, after each has refused its null required
// buffers: the message of the first that fails, or nullptr.  row_bufs: every row buffer is non-null (needed only when
// rows > 0).  The pose calls pass max_iters = 0 and no inliers.
const char* ragged_arg_error(int n_pairs, int rows, int dim, bool row_bufs, int max_iters, bool inliers, double px_th) {
  if (rows > 0 && !row_bufs) return "null row buffer";
  if (n_pairs < 1 || rows < 0 || dim < 2) return "need n_pairs >= 1, rows >= 0 and dim >= 2";
  if (max_iters < 0) return "max_iters must not be negative";
  if (inliers && !(px_th >= 0.0)) return "px_th must be a non-negative number";
  return nullptr;
}

// The refinement of one 3 x 3 model per pair (H or F) by `kernel`
int refine_model_ragged(void (*kernel)(RefineArgs), const double* d_M, const double* d_x1y1, const double* d_x2y2,
                        const int32_t* d_offsets, int n_pairs, int rows, int dim, const uint8_t* d_mask, int max_iters,
                        double px_th, double* d_M_out, double* d_cost0_out, double* d_cost_out, int32_t* d_n_used_out,
                        int32_t* d_iters_out, uint8_t* d_inliers_out, void* stream) {
  if (!d_M || !d_offsets || !d_M_out || !d_cost_out) return fail(DGB200_E_ARG, "null buffer");
  if (const char* err = ragged_arg_error(n_pairs, rows, dim, d_x1y1 && d_x2y2, max_iters, d_inliers_out, px_th))
    return fail(DGB200_E_ARG, err);
  RefineArgs a;
  a.model = d_M; a.x1y1 = d_x1y1; a.x2y2 = d_x2y2; a.offsets = d_offsets; a.mask = d_mask; a.n_pairs = n_pairs;
  a.rows = rows; a.dim = dim; a.max_iters = max_iters; a.th2 = d_inliers_out ? px_th * px_th : 0.0;
  a.model_out = d_M_out; a.cost0 = d_cost0_out; a.cost = d_cost_out; a.n_used = d_n_used_out; a.iters = d_iters_out;
  a.inliers = d_inliers_out;
  kernel<<<n_pairs, kPoseThreads, 0, (cudaStream_t)stream>>>(a);
  CU(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" {

int dgb200_debug_div_check(unsigned long long seed, long long count, unsigned long long* h_bad) {
  unsigned long long* d = nullptr;
  CU(cudaMalloc(&d, sizeof(unsigned long long)));
  CU(cudaMemset(d, 0, sizeof(unsigned long long)));
  div_check_kernel<<<1184, 256>>>(seed, count, d);
  CU(cudaGetLastError());
  CU(cudaMemcpy(h_bad, d, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  cudaFree(d);
  return 0;
}

const char* dgb200_frontend_last_error(void) { return g_err; }

size_t dgb200_match_workspace_bytes(int n1, int n2) {
  if (n1 < 0 || n2 < 0) return 0;
  return match_ws_bytes(n1, n2, 1);
}

size_t dgb200_match_batch_workspace_bytes(const int32_t* img_offsets, int n_images, const int32_t* pairs, int n_pairs) {
  std::vector<PairMeta> meta;
  if (build_meta(img_offsets, img_offsets, n_images, pairs, n_pairs, &meta)) return 0;
  return match_ws_bytes(meta[n_pairs].row0, meta[n_pairs].col0, n_pairs);
}

int dgb200_match_descriptors_dev(const float* d_desc1, int n1, const float* d_desc2, int n2, int D, float ratio, int mutual,
                                 const double* d_kp1, const double* d_kp2, int kp_dim, int* d_match_q, int* d_match_t,
                                 double* d_x1y1, double* d_x2y2, int out_dim, int capacity, int* d_count, void* d_workspace,
                                 void* stream) {
  return match_single(d_desc1, n1, d_desc2, n2, D, float_len_error(D), 0, ratio, mutual, d_kp1, d_kp2, kp_dim, d_match_q,
                      d_match_t, d_x1y1, d_x2y2, out_dim, capacity, d_count, d_workspace, stream);
}

int dgb200_match_descriptors_batch_dev(const float* d_bank, const int32_t* img_offsets, int n_images, int D,
                                       const int32_t* pairs, int n_pairs, float ratio, int mutual, const double* d_kp_bank,
                                       int kp_dim, int* d_match_q, int* d_match_t, double* d_x1y1, double* d_x2y2,
                                       int out_dim, int capacity, int32_t* d_offsets_out, void* d_workspace,
                                       void* stream) {
  return match_batch(d_bank, img_offsets, n_images, D, float_len_error(D), 0, pairs, n_pairs, ratio, mutual, d_kp_bank,
                     kp_dim, d_match_q, d_match_t, d_x1y1, d_x2y2, out_dim, capacity, d_offsets_out, d_workspace, stream);
}

int dgb200_match_binary_descriptors_dev(const uint32_t* d_desc1, int n1, const uint32_t* d_desc2, int n2, int n_words,
                                        double ratio, int mutual, const double* d_kp1, const double* d_kp2, int kp_dim,
                                        int* d_match_q, int* d_match_t, double* d_x1y1, double* d_x2y2, int out_dim,
                                        int capacity, int* d_count, void* d_workspace, void* stream) {
  return match_single(d_desc1, n1, d_desc2, n2, n_words, word_len_error(n_words), 1, ratio, mutual, d_kp1, d_kp2, kp_dim,
                      d_match_q, d_match_t, d_x1y1, d_x2y2, out_dim, capacity, d_count, d_workspace, stream);
}

int dgb200_match_binary_descriptors_batch_dev(const uint32_t* d_bank, const int32_t* img_offsets, int n_images,
                                              int n_words, const int32_t* pairs, int n_pairs, double ratio, int mutual,
                                              const double* d_kp_bank, int kp_dim, int* d_match_q, int* d_match_t,
                                              double* d_x1y1, double* d_x2y2, int out_dim, int capacity,
                                              int32_t* d_offsets_out, void* d_workspace, void* stream) {
  return match_batch(d_bank, img_offsets, n_images, n_words, word_len_error(n_words), 1, pairs, n_pairs, ratio, mutual,
                     d_kp_bank, kp_dim, d_match_q, d_match_t, d_x1y1, d_x2y2, out_dim, capacity, d_offsets_out,
                     d_workspace, stream);
}

int dgb200_match_descriptors_guided_batch_dev(const float* d_bank, const int32_t* img_offsets, int n_images, int D,
                                              const int32_t* pairs, int n_pairs, const double* d_models, int guide,
                                              double px_th, float ratio, int mutual, const double* d_kp_bank, int kp_dim,
                                              int* d_match_q, int* d_match_t, double* d_x1y1, double* d_x2y2,
                                              int out_dim, int capacity, int32_t* d_offsets_out, void* d_workspace,
                                              void* stream) {
  return match_batch(d_bank, img_offsets, n_images, D, float_len_error(D), 0, pairs, n_pairs, ratio, mutual, d_kp_bank,
                     kp_dim, d_match_q, d_match_t, d_x1y1, d_x2y2, out_dim, capacity, d_offsets_out, d_workspace, stream,
                     true, guide, d_models, px_th);
}

int dgb200_match_binary_descriptors_guided_batch_dev(const uint32_t* d_bank, const int32_t* img_offsets, int n_images,
                                                     int n_words, const int32_t* pairs, int n_pairs,
                                                     const double* d_models, int guide, double px_th, double ratio,
                                                     int mutual, const double* d_kp_bank, int kp_dim, int* d_match_q,
                                                     int* d_match_t, double* d_x1y1, double* d_x2y2, int out_dim,
                                                     int capacity, int32_t* d_offsets_out, void* d_workspace,
                                                     void* stream) {
  return match_batch(d_bank, img_offsets, n_images, n_words, word_len_error(n_words), 1, pairs, n_pairs, ratio, mutual,
                     d_kp_bank, kp_dim, d_match_q, d_match_t, d_x1y1, d_x2y2, out_dim, capacity, d_offsets_out,
                     d_workspace, stream, true, guide, d_models, px_th);
}

int dgb200_pose_from_fundamental_batch_dev(const double* d_F,const double* d_K1, const double* d_K2, int k_per_pair,
                                           const double* d_x1y1, const double* d_x2y2, const uint8_t* d_mask, int n_pairs,
                                           int n, int dim, double* d_R_out, double* d_t_out, int32_t* d_good_out,
                                           void* stream) {
  if (!d_F || !d_K1 || !d_K2 || !d_x1y1 || !d_x2y2 || !d_R_out || !d_t_out) return fail(DGB200_E_ARG, "null buffer");
  if (n_pairs < 1 || n < 1 || dim < 2) return fail(DGB200_E_ARG, "bad sizes");
  PoseArgs a;
  a.F = d_F; a.K1 = d_K1; a.K2 = d_K2; a.k_per_pair = k_per_pair; a.x1y1 = d_x1y1; a.x2y2 = d_x2y2; a.mask = d_mask;
  a.n_pairs = n_pairs; a.n = n; a.dim = dim; a.R = d_R_out; a.t = d_t_out; a.good = d_good_out;
  const int threads = 256;
  pose_kernel<<<(n_pairs * 32 + threads - 1) / threads, threads, 0, (cudaStream_t)stream>>>(a);
  CU(cudaGetLastError());
  return 0;
}

int dgb200_pose_from_fundamental_ragged_dev(const double* d_F, const double* d_K1, const double* d_K2, int k_per_pair,
                                            const double* d_x1y1, const double* d_x2y2, const int32_t* d_offsets,
                                            int n_pairs, int rows, int dim, const uint8_t* d_mask,
                                            double* d_R_out, double* d_t_out, int32_t* d_good_out,
                                            double* d_points_out, uint8_t* d_in_front_out, double* d_angle_out,
                                            double* d_median_angle_out, void* stream) {
  if (!d_F || !d_K1 || !d_K2 || !d_offsets || !d_R_out || !d_t_out || !d_median_angle_out) return fail(DGB200_E_ARG, "null buffer");
  if (const char* err = ragged_arg_error(n_pairs, rows, dim,
                                         d_x1y1 && d_x2y2 && d_points_out && d_in_front_out && d_angle_out, 0, false, 0.0))
    return fail(DGB200_E_ARG, err);
  PoseRaggedArgs a;
  a.w = pose_rows_args(d_K1, d_K2, k_per_pair, d_x1y1, d_x2y2, d_offsets, n_pairs, rows, dim, d_mask, d_points_out,
                       d_in_front_out, d_angle_out, d_median_angle_out);
  a.F = d_F; a.R = d_R_out; a.t = d_t_out; a.good = d_good_out;
  pose_ragged_kernel<<<n_pairs, kPoseThreads, 0, (cudaStream_t)stream>>>(a);
  CU(cudaGetLastError());
  return 0;
}

int dgb200_pose_from_homography_ragged_dev(const double* d_H, const double* d_K1, const double* d_K2, int k_per_pair,
                                           const double* d_x1y1, const double* d_x2y2, const int32_t* d_offsets,
                                           int n_pairs, int rows, int dim, const uint8_t* d_mask,
                                           double* d_R_out, double* d_t_out, double* d_plane_out, int32_t* d_good_out,
                                           uint8_t* d_rotation_only_out, double* d_points_out, uint8_t* d_in_front_out,
                                           double* d_angle_out, double* d_median_angle_out, void* stream) {
  if (!d_H || !d_K1 || !d_K2 || !d_offsets || !d_R_out || !d_t_out || !d_plane_out || !d_rotation_only_out ||
      !d_median_angle_out)
    return fail(DGB200_E_ARG, "null buffer");
  if (const char* err = ragged_arg_error(n_pairs, rows, dim,
                                         d_x1y1 && d_x2y2 && d_points_out && d_in_front_out && d_angle_out, 0, false, 0.0))
    return fail(DGB200_E_ARG, err);
  PoseHRaggedArgs a;
  a.w = pose_rows_args(d_K1, d_K2, k_per_pair, d_x1y1, d_x2y2, d_offsets, n_pairs, rows, dim, d_mask, d_points_out,
                       d_in_front_out, d_angle_out, d_median_angle_out);
  a.H = d_H; a.R = d_R_out; a.t = d_t_out; a.plane = d_plane_out; a.good = d_good_out;
  a.rotation_only = d_rotation_only_out;
  pose_h_ragged_kernel<<<n_pairs, kPoseThreads, 0, (cudaStream_t)stream>>>(a);
  CU(cudaGetLastError());
  return 0;
}

int dgb200_refine_pose_ragged_dev(const double* d_R, const double* d_t, const double* d_K1, const double* d_K2,
                                  int k_per_pair, const double* d_x1y1, const double* d_x2y2, const int32_t* d_offsets,
                                  int n_pairs, int rows, int dim, const uint8_t* d_mask, int max_iters, double px_th,
                                  double* d_R_out, double* d_t_out, double* d_F_out, double* d_cost0_out,
                                  double* d_cost_out, int32_t* d_n_used_out, int32_t* d_iters_out,
                                  uint8_t* d_inliers_out, void* stream) {
  if (!d_R || !d_t || !d_K1 || !d_K2 || !d_offsets || !d_R_out || !d_t_out || !d_F_out || !d_cost_out)
    return fail(DGB200_E_ARG, "null buffer");
  if (const char* err = ragged_arg_error(n_pairs, rows, dim, d_x1y1 && d_x2y2, max_iters, d_inliers_out, px_th))
    return fail(DGB200_E_ARG, err);
  PoseRefineArgs a;
  a.R = d_R; a.t = d_t; a.K1 = d_K1; a.K2 = d_K2; a.k_per_pair = k_per_pair; a.x1y1 = d_x1y1; a.x2y2 = d_x2y2;
  a.offsets = d_offsets; a.mask = d_mask; a.n_pairs = n_pairs; a.rows = rows; a.dim = dim; a.max_iters = max_iters;
  a.th2 = d_inliers_out ? px_th * px_th : 0.0;
  a.R_out = d_R_out; a.t_out = d_t_out; a.F_out = d_F_out; a.cost0 = d_cost0_out; a.cost = d_cost_out;
  a.n_used = d_n_used_out; a.iters = d_iters_out; a.inliers = d_inliers_out;
  pose_refine_ragged_kernel<<<n_pairs, kPoseThreads, 0, (cudaStream_t)stream>>>(a);
  CU(cudaGetLastError());
  return 0;
}

int dgb200_refine_homography_ragged_dev(const double* d_H, const double* d_x1y1, const double* d_x2y2,
                                        const int32_t* d_offsets, int n_pairs, int rows, int dim, const uint8_t* d_mask,
                                        int max_iters, double px_th, double* d_H_out, double* d_cost0_out,
                                        double* d_cost_out, int32_t* d_n_used_out, int32_t* d_iters_out,
                                        uint8_t* d_inliers_out, void* stream) {
  return refine_model_ragged(h_refine_ragged_kernel, d_H, d_x1y1, d_x2y2, d_offsets, n_pairs, rows, dim, d_mask,
                             max_iters, px_th, d_H_out, d_cost0_out, d_cost_out, d_n_used_out, d_iters_out,
                             d_inliers_out, stream);
}

int dgb200_refine_fundamental_ragged_dev(const double* d_F, const double* d_x1y1, const double* d_x2y2,
                                         const int32_t* d_offsets, int n_pairs, int rows, int dim, const uint8_t* d_mask,
                                         int max_iters, double px_th, double* d_F_out, double* d_cost0_out,
                                         double* d_cost_out, int32_t* d_n_used_out, int32_t* d_iters_out,
                                         uint8_t* d_inliers_out, void* stream) {
  return refine_model_ragged(f_refine_ragged_kernel, d_F, d_x1y1, d_x2y2, d_offsets, n_pairs, rows, dim, d_mask,
                             max_iters, px_th, d_F_out, d_cost0_out, d_cost_out, d_n_used_out, d_iters_out,
                             d_inliers_out, stream);
}

int dgb200_nullspace_qr7x9_batch_dev(const double* d_A, double* d_N, int32_t* d_rc, int count, void* stream) {
  if (!d_A || !d_N || count < 1) return fail(DGB200_E_ARG, "bad arguments");
  qr7x9_kernel<<<(count + 127) / 128, 128, 0, (cudaStream_t)stream>>>(d_A, d_N, d_rc, count);
  CU(cudaGetLastError());
  return 0;
}

}  // extern "C"
