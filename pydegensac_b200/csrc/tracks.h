// tracks.h -- per-thread pieces of the track builder (tracks.cu): the lock-free union-find over keypoints and the
// image of a keypoint.  Host-compilable: tests/tracks_host.cpp runs tk_link / tk_find from several std::threads, with
// std::atomic_ref standing in for the device's atomicCAS.
//
// The forest `parent` holds, for every node g, parent[g] <= g, and parent[g] is a node of g's component; a root has
// parent[r] == r.  tk_link hooks the larger of two roots under the smaller with a compare-and-swap that succeeds only
// while the larger is still a root, and tk_find halves the path it walks (ECL-CC, Jaiganesh & Burtscher, HPDC 2018).
// Path halving writes an ancestor over a non-root's parent: the store may race with other halvings of the same node,
// but every value stored is a smaller node of the same component, so the invariant holds whichever store lands, and a
// node that stopped being a root never becomes one again.  So, whatever the interleaving, once every edge is linked
// each component is one tree whose root is its smallest node.
#pragma once
#include "common.h"

#if !defined(__CUDACC__)
#include <atomic>
#endif

namespace dg {

#if defined(__CUDACC__)
__device__ __forceinline__ int tk_load(int* p) { return *(volatile int*)p; }
__device__ __forceinline__ void tk_store(int* p, int v) { *(volatile int*)p = v; }
__device__ __forceinline__ int tk_cas(int* p, int expect, int want) { return atomicCAS(p, expect, want); }
#define DG_TK __device__ __forceinline__
#else
inline int tk_load(int* p) { return std::atomic_ref<int>(*p).load(std::memory_order_relaxed); }
inline void tk_store(int* p, int v) { std::atomic_ref<int>(*p).store(v, std::memory_order_relaxed); }
inline int tk_cas(int* p, int expect, int want) {
  std::atomic_ref<int>(*p).compare_exchange_strong(expect, want, std::memory_order_relaxed);
  return expect;                                     // the value found, as atomicCAS returns it
}
#define DG_TK inline
#endif

// The root of g's tree, halving the path on the way
DG_TK int tk_find(int* parent, int g) {
  int p = tk_load(parent + g);
  while (p != g) {
    const int gp = tk_load(parent + p);
    if (gp != p) tk_store(parent + g, gp);
    g = gp;
    p = tk_load(parent + g);
  }
  return g;
}

// Compression of g once every edge is linked: parent[g] = the root of g's tree, which it returns.  The walk does not
// halve: a halving store racing with another node's compression could put a non-root back over its root, so here
// every store is a root, and a walk that reads one meets an ancestor either way.
DG_TK int tk_compress(int* parent, int g) {
  int r = g, p = tk_load(parent + g);
  while (p != r) {
    r = p;
    p = tk_load(parent + r);
  }
  tk_store(parent + g, r);
  return r;
}

// Joins the trees of a and b: the larger root is hooked under the smaller one
DG_TK void tk_link(int* parent, int a, int b) {
  a = tk_find(parent, a);
  b = tk_find(parent, b);
  while (a != b) {
    if (a > b) { const int s = a; a = b; b = s; }
    const int seen = tk_cas(parent + b, b, a);
    if (seen == b) return;                           // b hooked under a
    b = tk_find(parent, seen);                       // b was hooked meanwhile: carry on from its new root
    a = tk_find(parent, a);
  }
}

// The image of node g: the largest i < n_images with img_off[i] <= g (empty images own no node)
DG_HD int tk_image(const int* img_off, int n_images, int g) {
  int lo = 0, hi = n_images - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (img_off[mid] <= g) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

}  // namespace dg
