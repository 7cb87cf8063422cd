// Host build of csrc/tracks.h, the union-find and the image lookup of the track builder -- TEST HELPER ONLY
// (tests/test_build_tracks.py compiles it with g++ -std=c++20 into a temporary directory).  std::atomic_ref stands in
// for atomicCAS, and several std::threads link the edges concurrently, as the warps of tk_hook_kernel do.
#include <numeric>
#include <thread>
#include <vector>

#include "../pydegensac_b200/csrc/tracks.h"

extern "C" {

// The forest after linking the m edges (a[e], b[e]) from n_threads threads (thread k takes the edges k, k + n_threads,
// ...) and compressing from as many threads: roots [n] = parent [n]
void tkh_roots(int n, const int* a, const int* b, int m, int n_threads, int* roots) {
  std::vector<int> parent((size_t)n);
  std::iota(parent.begin(), parent.end(), 0);
  int* par = parent.data();
  std::vector<std::thread> th;
  for (int k = 0; k < n_threads; ++k)
    th.emplace_back([=] { for (int e = k; e < m; e += n_threads) dg::tk_link(par, a[e], b[e]); });
  for (auto& t : th) t.join();
  th.clear();
  for (int k = 0; k < n_threads; ++k)
    th.emplace_back([=] {
      for (int g = k; g < n; g += n_threads) dg::tk_compress(par, g);
    });
  for (auto& t : th) t.join();
  for (int g = 0; g < n; ++g) roots[g] = par[g];     // the forest itself: every node must point at its root
}

// The image of every node g in [0, n): out [n]
void tkh_images(const int* img_off, int n_images, int n, int* out) {
  for (int g = 0; g < n; ++g) out[g] = dg::tk_image(img_off, n_images, g);
}

}  // extern "C"
