// tracks.cu -- the track builder, device resident: the connected components of the graph whose nodes are keypoints and
// whose edges are verified matches, in the ragged track layout of dgb200_triangulate_tracks_ragged_dev (what
// OpenMVG's TracksBuilder and COLMAP's correspondence graph do on the host).  A translation unit of its own, so that
// adding it changes no instruction of the other kernels.
//
//   init         parent[g] = g, sizes 0, track_of = -1, stats 0
//   hook         one warp per pair, striding its rows: tk_link of every edge (tracks.h), lock-free
//   compress     parent[g] = tk_compress(g), the smallest node of g's component; size[root] += 1 (integer atomics)
//   scan 1       ordered reduce-then-scan over the nodes: each root with 2 <= size <= n_images gets a segment of `size`
//                slots, in root order (roots with a larger size are conflicting and only counted)
//   scatter      every node of such a root takes a slot of its segment (an atomic cursor: the slot depends on timing)
//   rank         one warp per segment: each node's rank is the number of smaller nodes in the segment, which sorts the
//                segment whatever the scatter's slots were; two nodes of one image flag the segment as conflicting
//   scan 2       ordered reduce-then-scan over the segments that survive (no conflict, size >= min_length): the track
//                index and the first observation of each
//   write        one warp per surviving segment: offsets, cams, kp, pts and track_of
//   finish       the padding past the last track and observation, and stats[0..1]
// The integer atomics are the hooks (whose result, the smallest node of each component, does not depend on their
// order), the sizes and the conflict counts (sums), and the scatter's cursors (undone by the rank): the output is a
// function of the edge set alone.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <vector>

#include "../../include/degensac_b200.h"
#include "entry_error.h"
#include "tracks.h"
#include "device_util.h"

namespace {

thread_local char g_err[256] = "";
int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return set_error(g_err, code, what, e); }

constexpr int kTkThreads = 256;                   // every kernel; the warp kernels take 8 pairs or segments per CTA
constexpr int kTkItems = 8;                       // items per thread of a scan tile
constexpr int kTkTile = kTkThreads * kTkItems;
constexpr int kTkMaxWarpCtas = 4096;              // grid of the grid-stride warp kernels

struct TkArgs {
  int n_nodes, n_images, n_pairs, rows, min_length, seg_cap, track_cap;
  const int* img_off;                             // [n_images + 1] (device copy)
  const int4* pair_tab;                           // [n_pairs]: (first node of q, count of q, first node of t, count of t)
  const int* idx1; const int* idx2; const int* offsets; const unsigned char* mask;
  const double* kp;                               // [n_nodes][2] or null
  int* parent;                                    // [n_nodes]
  int* aux;                                       // [n_nodes]: component size, then the segment cursor of a root (-1)
  int* nodes; int* sorted;                        // [n_nodes]: segment slots as scattered, then in node order
  int* seg_off;                                   // [seg_cap + 1]
  int2* seg;                                      // [seg_cap]: (survives, size), then (track, first observation) or -1
  int* cnt;                                       // [3]: segments, tracks, observations
  int* off_out; int* cams_out; int* kp_out; double* pts_out; int* track_of; int* stats;
};

__global__ void __launch_bounds__(kTkThreads) tk_init_kernel(TkArgs a) {
  const long long g = (long long)blockIdx.x * kTkThreads + threadIdx.x;
  if (g < 3) a.cnt[g] = 0;
  if (g < 4) a.stats[g] = 0;
  if (g >= a.n_nodes) return;
  a.parent[g] = g;
  a.aux[g] = 0;
  a.track_of[g] = -1;
}

// One warp per pair: a malformed pair is rejected once and none of its rows is read
__global__ void __launch_bounds__(kTkThreads) tk_hook_kernel(TkArgs a) {
  const int p = blockIdx.x * (kTkThreads / 32) + (threadIdx.x >> 5);
  if (p >= a.n_pairs) return;                     // (warp-uniform)
  const int b = a.offsets[p], e = a.offsets[p + 1];
  if (!(b >= 0 && b <= e && e <= a.rows)) return;
  const int4 pt = a.pair_tab[p];
  for (int r = b + (threadIdx.x & 31); r < e; r += 32) {
    if (a.mask && !a.mask[r]) continue;
    const int i = a.idx1[r], j = a.idx2[r];
    if (i < 0 || i >= pt.y || j < 0 || j >= pt.w) continue;
    dg::tk_link(a.parent, pt.x + i, pt.z + j);
  }
}

__global__ void __launch_bounds__(kTkThreads) tk_compress_kernel(TkArgs a) {
  const long long i = (long long)blockIdx.x * kTkThreads + threadIdx.x;
  if (i >= a.n_nodes) return;
  const int g = (int)i;
  atomicAdd(a.aux + dg::tk_compress(a.parent, g), 1);
}

// ------------------------------------------------------------------------ ordered reduce-then-scan of int2 values
// Scan 1 runs over the nodes (kMode 1), scan 2 over the segments (kMode 2).  Tile b holds items b * kTkTile ..;
// thread t of a tile its items t * kTkItems .. + kTkItems - 1, so the order is the item order.
template <int kMode>
__device__ __forceinline__ int2 tk_value(const TkArgs& a, long long i) {
  if (kMode == 1) {
    if (i >= a.n_nodes || a.parent[i] != i) return make_int2(0, 0);
    const int s = a.aux[i];
    return s >= 2 && s <= a.n_images ? make_int2(1, s) : make_int2(0, 0);
  }
  return i < a.cnt[0] ? a.seg[i] : make_int2(0, 0);
}

// v: the item's value, x: the exclusive prefix of its scan
template <int kMode>
__device__ __forceinline__ void tk_put(const TkArgs& a, long long i, int2 v, int2 x) {
  if (kMode == 1) {
    if (i >= a.n_nodes) return;
    if (v.x) a.seg_off[x.x] = x.y;
    else if (a.parent[i] == i && a.aux[i] > a.n_images) {   // conflicting by its size alone
      atomicAdd(a.stats + 2, 1);
      atomicAdd(a.stats + 3, a.aux[i]);
    }
    a.aux[i] = v.x ? x.y : -1;
  } else if (i < a.cnt[0]) {
    a.seg[i] = v.x ? x : make_int2(-1, 0);
  }
}

__device__ __forceinline__ int2 add2(int2 u, int2 v) { return make_int2(u.x + v.x, u.y + v.y); }

__device__ __forceinline__ int2 warp_incl(int2 v) {
  const int lane = threadIdx.x & 31;
  for (int o = 1; o < 32; o <<= 1) {
    const int x = __shfl_up_sync(kFull, v.x, o), y = __shfl_up_sync(kFull, v.y, o);
    if (lane >= o) { v.x += x; v.y += y; }
  }
  return v;
}

// Exclusive scan of one int2 per thread over the CTA (in thread order); *total gets the CTA's sum
__device__ int2 block_excl(int2 v, int2* total) {
  __shared__ int2 wsum[kTkThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int2 inc = warp_incl(v);
  if (lane == 31) wsum[wid] = inc;
  __syncthreads();
  int2 off = make_int2(0, 0), tot = make_int2(0, 0);
  for (int w = 0; w < kTkThreads / 32; ++w) {
    if (w < wid) off = add2(off, wsum[w]);
    tot = add2(tot, wsum[w]);
  }
  __syncthreads();                                // wsum may be reused by the caller's next call
  *total = tot;
  return make_int2(off.x + inc.x - v.x, off.y + inc.y - v.y);
}

template <int kMode>
__global__ void __launch_bounds__(kTkThreads) tk_scan_reduce_kernel(TkArgs a, int2* tile_sum) {
  const long long i0 = (long long)blockIdx.x * kTkTile + threadIdx.x * kTkItems;
  int2 s = make_int2(0, 0);
#pragma unroll
  for (int k = 0; k < kTkItems; ++k) s = add2(s, tk_value<kMode>(a, i0 + k));
  int2 tot;
  block_excl(s, &tot);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = tot;
}

// One CTA: the tiles' sums become their exclusive prefixes; the grand total goes to *total (and, for scan 1, the
// end of the last segment to seg_off[segments])
__global__ void __launch_bounds__(kTkThreads) tk_scan_tiles_kernel(TkArgs a, int2* tile_sum, int n_tiles, int mode) {
  int2 base = make_int2(0, 0);
  for (int b0 = 0; b0 < n_tiles; b0 += kTkThreads) {
    const int b = b0 + threadIdx.x;
    const int2 v = b < n_tiles ? tile_sum[b] : make_int2(0, 0);
    int2 tot;
    const int2 x = block_excl(v, &tot);
    if (b < n_tiles) tile_sum[b] = add2(base, x);
    base = add2(base, tot);
  }
  if (threadIdx.x == 0) {
    if (mode == 1) {
      a.cnt[0] = base.x;
      a.seg_off[base.x] = base.y;
    } else {
      a.cnt[1] = base.x;
      a.cnt[2] = base.y;
    }
  }
}

template <int kMode>
__global__ void __launch_bounds__(kTkThreads) tk_scan_write_kernel(TkArgs a, const int2* tile_off) {
  const long long i0 = (long long)blockIdx.x * kTkTile + threadIdx.x * kTkItems;
  int2 v[kTkItems], s = make_int2(0, 0);
#pragma unroll
  for (int k = 0; k < kTkItems; ++k) {
    v[k] = tk_value<kMode>(a, i0 + k);
    s = add2(s, v[k]);
  }
  int2 tot;
  int2 x = add2(tile_off[blockIdx.x], block_excl(s, &tot));
#pragma unroll
  for (int k = 0; k < kTkItems; ++k) {
    tk_put<kMode>(a, i0 + k, v[k], x);
    x = add2(x, v[k]);
  }
}

// ------------------------------------------------------------------------ segments
__global__ void __launch_bounds__(kTkThreads) tk_scatter_kernel(TkArgs a) {
  const long long i = (long long)blockIdx.x * kTkThreads + threadIdx.x;
  if (i >= a.n_nodes) return;
  const int g = (int)i;
  const int r = a.parent[g];
  if (a.aux[r] >= 0) a.nodes[atomicAdd(a.aux + r, 1)] = g;   // (a cursor only grows; -1 marks no segment)
}

// One warp per segment (grid-stride over the segments found): the segment in node order, and whether it survives
__global__ void __launch_bounds__(kTkThreads) tk_rank_kernel(TkArgs a) {
  const int lane = threadIdx.x & 31;
  const int n_seg = a.cnt[0];
  for (int k = (blockIdx.x * kTkThreads + threadIdx.x) >> 5; k < n_seg; k += (gridDim.x * kTkThreads) >> 5) {
    const int b = a.seg_off[k], len = a.seg_off[k + 1] - b;
    const int* nd = a.nodes + b;
    bool dup = false;
    for (int c = 0; c < len; c += 32) {          // lane: node c + lane, against every node of the segment
      const int i = c + lane;
      const int g = i < len ? nd[i] : -1;
      const int im = i < len ? dg::tk_image(a.img_off, a.n_images, g) : -1;
      int rank = 0;
      for (int c2 = 0; c2 < len; c2 += 32) {
        const int j = c2 + lane;
        const int h = j < len ? nd[j] : -1;
        const int ih = j < len ? dg::tk_image(a.img_off, a.n_images, h) : -2;
        const int m = len - c2 < 32 ? len - c2 : 32;
        for (int l = 0; l < m; ++l) {
          const int hl = __shfl_sync(kFull, h, l), il = __shfl_sync(kFull, ih, l);
          rank += hl < g;
          dup = dup || (il == im && hl != g);
        }
      }
      if (i < len) a.sorted[b + rank] = g;
    }
    dup = __any_sync(kFull, dup);
    const bool keep = !dup && len >= a.min_length;
    if (lane == 0) {
      a.seg[k] = keep ? make_int2(1, len) : make_int2(0, 0);
      if (dup) {
        atomicAdd(a.stats + 2, 1);
        atomicAdd(a.stats + 3, len);
      }
    }
  }
}

__global__ void __launch_bounds__(kTkThreads) tk_write_kernel(TkArgs a) {
  const int lane = threadIdx.x & 31;
  const int n_seg = a.cnt[0];
  for (int k = (blockIdx.x * kTkThreads + threadIdx.x) >> 5; k < n_seg; k += (gridDim.x * kTkThreads) >> 5) {
    const int2 to = a.seg[k];
    if (to.x < 0) continue;                       // (warp-uniform)
    const int b = a.seg_off[k], len = a.seg_off[k + 1] - b;
    if (lane == 0) a.off_out[to.x] = to.y;
    for (int i = lane; i < len; i += 32) {
      const int g = a.sorted[b + i], o = to.y + i;
      const int im = dg::tk_image(a.img_off, a.n_images, g);
      a.cams_out[o] = im;
      a.kp_out[o] = g - a.img_off[im];
      if (a.pts_out) {
        a.pts_out[2 * (size_t)o] = a.kp[2 * (size_t)g];
        a.pts_out[2 * (size_t)o + 1] = a.kp[2 * (size_t)g + 1];
      }
      a.track_of[g] = to.x;
    }
  }
}

// The padding: offsets[T .. track_cap] = n_obs, observations n_obs .. n_nodes - 1 empty; and stats[0..1]
__global__ void __launch_bounds__(kTkThreads) tk_finish_kernel(TkArgs a) {
  const long long i = (long long)blockIdx.x * kTkThreads + threadIdx.x;
  const int n_tracks = a.cnt[1], n_obs = a.cnt[2];
  if (i == 0) {
    a.stats[0] = n_tracks;
    a.stats[1] = n_obs;
  }
  if (i >= n_tracks && i <= a.track_cap) a.off_out[i] = n_obs;
  if (i >= n_obs && i < a.n_nodes) {
    a.cams_out[i] = -1;
    a.kp_out[i] = -1;
    if (a.pts_out) a.pts_out[2 * (size_t)i] = a.pts_out[2 * (size_t)i + 1] = qnan();
  }
}

int blocks(long long n, int per) { return (int)((n + per - 1) / per); }

}  // namespace

extern "C" {

const char* dgb200_tracks_last_error(void) { return g_err; }

int dgb200_build_tracks_ragged_dev(const int32_t* img_offsets, int n_images, const int32_t* pairs, int n_pairs,
                                   const int32_t* d_idx1, const int32_t* d_idx2, const int32_t* d_offsets, int rows,
                                   const uint8_t* d_mask, const double* d_kp, int min_length, int32_t* d_offsets_out,
                                   int32_t* d_cams_out, int32_t* d_kp_out, double* d_pts_out, int32_t* d_track_of_out,
                                   int32_t* d_stats_out, void* stream) {
  if (!img_offsets || !pairs || !d_offsets || !d_offsets_out || !d_stats_out) return fail(DGB200_E_ARG, "null buffer");
  if (n_images < 1 || n_pairs < 1 || rows < 0)
    return fail(DGB200_E_ARG, "need n_images >= 1, n_pairs >= 1 and rows >= 0");
  if (rows > 0 && (!d_idx1 || !d_idx2)) return fail(DGB200_E_ARG, "null row buffer");
  if (min_length < 2) return fail(DGB200_E_ARG, "min_length must be at least 2");
  if (img_offsets[0] != 0) return fail(DGB200_E_ARG, "img_offsets must start at 0 and must not decrease");
  for (int i = 0; i < n_images; ++i)
    if (img_offsets[i + 1] < img_offsets[i])
      return fail(DGB200_E_ARG, "img_offsets must start at 0 and must not decrease");
  const int n = img_offsets[n_images];
  if (n > 0 && (!d_cams_out || !d_kp_out || !d_track_of_out)) return fail(DGB200_E_ARG, "null keypoint buffer");
  if ((d_kp == nullptr) != (d_pts_out == nullptr) || (n == 0 && d_kp != nullptr))
    return fail(DGB200_E_ARG, "d_kp and d_pts_out must both be given (with keypoints) or both be null");
  std::vector<int4> tab((size_t)n_pairs);
  for (int p = 0; p < n_pairs; ++p) {
    const int q = pairs[2 * p], t = pairs[2 * p + 1];
    if (q < 0 || q >= n_images || t < 0 || t >= n_images) return fail(DGB200_E_ARG, "pairs: image index out of range");
    tab[p] = make_int4(img_offsets[q], img_offsets[q + 1] - img_offsets[q], img_offsets[t],
                       img_offsets[t + 1] - img_offsets[t]);
  }
  const cudaStream_t st = (cudaStream_t)stream;
  const int seg_cap = n / 2, track_cap = n / min_length;
  const int node_tiles = blocks(n, kTkTile) > 0 ? blocks(n, kTkTile) : 1;
  const int seg_tiles = blocks(seg_cap, kTkTile) > 0 ? blocks(seg_cap, kTkTile) : 1;
  const size_t n4 = sizeof(int) * (size_t)n;
  const size_t bytes = sizeof(int4) * (size_t)n_pairs + sizeof(int) * ((size_t)n_images + 1) + 4 * n4 +
                       sizeof(int) * ((size_t)seg_cap + 1) + sizeof(int2) * (size_t)seg_cap +
                       sizeof(int2) * (size_t)(node_tiles > seg_tiles ? node_tiles : seg_tiles) + sizeof(int) * 3;
  char* ws = nullptr;
  CU(cudaMallocAsync((void**)&ws, bytes, st));
  TkArgs a;
  a.n_nodes = n; a.n_images = n_images; a.n_pairs = n_pairs; a.rows = rows; a.min_length = min_length;
  a.seg_cap = seg_cap; a.track_cap = track_cap;
  char* w = ws;                                   // the 16- and 8-byte arrays first, then the int arrays
  int4* d_tab = (int4*)w; w += sizeof(int4) * (size_t)n_pairs;
  a.seg = (int2*)w; w += sizeof(int2) * (size_t)seg_cap;
  int2* tile_sum = (int2*)w; w += sizeof(int2) * (size_t)(node_tiles > seg_tiles ? node_tiles : seg_tiles);
  int* d_img = (int*)w; w += sizeof(int) * ((size_t)n_images + 1);
  a.parent = (int*)w; w += n4;
  a.aux = (int*)w; w += n4;
  a.nodes = (int*)w; w += n4;
  a.sorted = (int*)w; w += n4;
  a.seg_off = (int*)w; w += sizeof(int) * ((size_t)seg_cap + 1);
  a.cnt = (int*)w;
  a.img_off = d_img; a.pair_tab = d_tab;
  a.idx1 = d_idx1; a.idx2 = d_idx2; a.offsets = d_offsets; a.mask = d_mask; a.kp = d_kp;
  a.off_out = d_offsets_out; a.cams_out = d_cams_out; a.kp_out = d_kp_out; a.pts_out = d_pts_out;
  a.track_of = d_track_of_out; a.stats = d_stats_out;
  cudaError_t e = cudaMemcpyAsync(d_tab, tab.data(), sizeof(int4) * (size_t)n_pairs, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(d_img, img_offsets, sizeof(int) * ((size_t)n_images + 1), cudaMemcpyHostToDevice, st);
  const int node_blocks = blocks(n > 4 ? n : 4, kTkThreads);
  const int warp_blocks = blocks(seg_cap, kTkThreads / 32) < kTkMaxWarpCtas ? blocks(seg_cap, kTkThreads / 32)
                                                                            : kTkMaxWarpCtas;
  if (e == cudaSuccess) {
    tk_init_kernel<<<node_blocks, kTkThreads, 0, st>>>(a);
    if (n > 0) {
      tk_hook_kernel<<<blocks(n_pairs, kTkThreads / 32), kTkThreads, 0, st>>>(a);
      tk_compress_kernel<<<node_blocks, kTkThreads, 0, st>>>(a);
    }
    tk_scan_reduce_kernel<1><<<node_tiles, kTkThreads, 0, st>>>(a, tile_sum);
    tk_scan_tiles_kernel<<<1, kTkThreads, 0, st>>>(a, tile_sum, node_tiles, 1);
    tk_scan_write_kernel<1><<<node_tiles, kTkThreads, 0, st>>>(a, tile_sum);
    if (seg_cap > 0) {
      tk_scatter_kernel<<<node_blocks, kTkThreads, 0, st>>>(a);
      tk_rank_kernel<<<warp_blocks, kTkThreads, 0, st>>>(a);
    }
    tk_scan_reduce_kernel<2><<<seg_tiles, kTkThreads, 0, st>>>(a, tile_sum);
    tk_scan_tiles_kernel<<<1, kTkThreads, 0, st>>>(a, tile_sum, seg_tiles, 2);
    tk_scan_write_kernel<2><<<seg_tiles, kTkThreads, 0, st>>>(a, tile_sum);
    if (seg_cap > 0) tk_write_kernel<<<warp_blocks, kTkThreads, 0, st>>>(a);
    tk_finish_kernel<<<blocks((n > track_cap + 1 ? n : track_cap + 1), kTkThreads), kTkThreads, 0, st>>>(a);
    e = cudaGetLastError();
  }
  CU(cudaFreeAsync(ws, st));
  if (e != cudaSuccess) return fail(DGB200_E_CUDA, "dgb200_build_tracks_ragged_dev", e);
  return 0;
}

}  // extern "C"
