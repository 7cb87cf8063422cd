// blockleaf.cu -- TEST HELPER ONLY.  The block level of the device harness: the engine headers, unchanged, compiled by
// nvcc with the library's flags (sm_90a, -fmad=false), and one kernel per CTA-cooperative primitive.  Each kernel runs
// ONE CTA of `nt` threads (any multiple of 32 up to the pair kernel's 256) over a SoA pair in global memory with its
// BlockScratch in shared memory, as ransac_pairs_kernel sets them up, and calls one primitive.  Every launcher takes and
// returns host arrays and reports the CUDA status; tests/devleaf/blk.py loads it with ctypes.  Never loaded by the
// pydegensac_b200 package.
#include <cuda_runtime.h>
#include <string.h>
#include "../../pydegensac_b200/csrc/engine_f.h"
#include "../../pydegensac_b200/csrc/engine_h.h"

using namespace dg;

namespace {

__device__ void blk_ctx(Ctx& c, BlockScratch* sc, const double* soa, int N, int row) {
  memset(&c, 0, sizeof(c));
  c.tid = threadIdx.x; c.nt = blockDim.x; c.lane = c.tid & 31; c.wid = c.tid >> 5; c.nw = c.nt >> 5;
  c.N = N;
  if (soa) { c.x1 = soa; c.y1 = soa + row; c.x2 = soa + 2 * row; c.y2 = soa + 3 * row; }
  c.sc = sc;
}

enum { CMP_ONE = 0, CMP_TWO = 1 };
// mode CMP_ONE: two blk_inlidxs calls (thA, thB); CMP_TWO: one blk_inlidxs2.  J[0..1], I[0..1]; I[2] = blk_count_lt(thA)
__global__ void k_inlidxs(const double* err, int N, double thA, double thB, int mode, int* listA, int* listB, double* J,
                          int* I) {
  __shared__ BlockScratch sc;
  Ctx c;
  blk_ctx(c, &sc, nullptr, N, 0);
  Score SA, SB;
  if (mode == CMP_ONE) {
    SA = blk_inlidxs(c, err, thA, listA);
    SB = blk_inlidxs(c, err, thB, listB);
  } else {
    blk_inlidxs2(c, err, thA, listA, &SA, thB, listB, &SB);
  }
  const int cnt = blk_count_lt(c, err, thA);
  if (c.tid == 0) { J[0] = SA.J; J[1] = SB.J; I[0] = (int)SA.I; I[1] = (int)SB.I; I[2] = cnt; }
}

// Every thread's view of the reductions: vd[t], vi[t] are thread t's inputs, vv[48 t + i] its blk_sum_vec entries.
// od[3 nt + 48] = {blk_sum[t], blk_scan_sum J[t], 0, vec_out[0..k)};  oi[5 nt] = {blk_sum_i, blk_excl_scan_i offset,
// its total, blk_scan_sum offset, its total} per thread.
__global__ void k_reduce(const double* vd, const int* vi, const double* vv, int k, double* od, int* oi) {
  __shared__ BlockScratch sc;
  Ctx c;
  blk_ctx(c, &sc, nullptr, 0, 0);
  const int t = c.tid, nt = c.nt;
  od[t] = blk_sum(c, vd[t]);
  oi[t] = blk_sum_i(c, vi[t]);
  int tot = 0;
  oi[nt + t] = blk_excl_scan_i(c, vi[t], &tot);
  oi[2 * nt + t] = tot;
  DG_SYNC();
  int off = 0, tot2 = 0;
  double Jt = 0.0;
  blk_scan_sum(c, vi[t], vd[t], &off, &tot2, &Jt);
  oi[3 * nt + t] = off; oi[4 * nt + t] = tot2; od[nt + t] = Jt;
  double v[kVecRed];
  for (int i = 0; i < kVecRed; ++i) v[i] = vv[(size_t)kVecRed * t + i];
  blk_sum_vec(c, v, k);
  for (int i = t; i < k; i += nt) od[3 * nt + i] = c.sc->vec_out[i];
}

// blk_resid_F (weighted = 0) or blk_resid_w_F (weighted = 1, weights to w)
__global__ void k_resid_F(const double* soa, int N, int row, int metric, const double* F, int weighted, double* out,
                          double* w) {
  __shared__ BlockScratch sc;
  Ctx c;
  blk_ctx(c, &sc, soa, N, row);
  double f[9];
  for (int i = 0; i < 9; ++i) f[i] = F[i];
  if (weighted) blk_resid_w_F(c, metric, f, out, w);
  else blk_resid_F(c, metric, f, out);
}

// blk_resid_H with HParams {metric, th}; with_tile: the pair's FP32 tile is built first (c.t32 set, as the H kernel
// does for the Sampson metric), which turns on the two-step row for N >= kResidClassifyMinN.  list: N ints of scratch.
__global__ void k_resid_H(const double* soa, int N, int row, int metric, double th, const double* h, int with_tile,
                          float* tile, int* list, double* out) {
  __shared__ BlockScratch sc;
  Ctx c;
  blk_ctx(c, &sc, soa, N, row);
  Tile32 T;
  if (with_tile) {
    blk_prepare_tile32(c, reinterpret_cast<Pt32*>(tile), &T);
    c.t32 = &T;
  }
  HParams P;
  memset(&P, 0, sizeof(P));
  P.metric = metric; P.th = th;
  Workspace W;
  memset(&W, 0, sizeof(W));
  W.itmp[3] = list;
  double hh[9];
  for (int i = 0; i < 9; ++i) hh[i] = h[i];
  blk_resid_H(c, P, W, hh, out);
}

// Gate counts over list[0..n): out = {blk_sym_count_F, blk_laf_count_F, blk_sym_count_H, blk_laf_count_H(p1),
// blk_laf_count_H(p2)}.  laf: the eight helper rows, `row` apart.
__global__ void k_counts(const double* soa, const double* laf, int N, int row, const int* list, int n, const double* F,
                         const double* h, int fmetric, int hmetric, double sym_th, double th_laf, int* out) {
  __shared__ BlockScratch sc;
  Ctx c;
  blk_ctx(c, &sc, soa, N, row);
  for (int i = 0; i < 8; ++i) c.laf[i] = laf + (size_t)i * row;
  double f[9], hh[9];
  for (int i = 0; i < 9; ++i) { f[i] = F[i]; hh[i] = h[i]; }
  const unsigned a = blk_sym_count_F(c, f, list, n, sym_th);
  const unsigned b = blk_laf_count_F(c, fmetric, f, list, n, th_laf);
  const unsigned d = blk_sym_count_H(c, hh, list, n, sym_th);
  const int e0 = blk_laf_count_H(c, hmetric, hh, list, n, th_laf, 0);
  const int e1 = blk_laf_count_H(c, hmetric, hh, list, n, th_laf, 1);
  if (c.tid == 0) { out[0] = (int)a; out[1] = (int)b; out[2] = (int)d; out[3] = e0; out[4] = e1; }
}

// blk_fit_F (kind 0, weights w or nullptr) or blk_fit_H (kind 1) on idx[0..len); model to out[0..8]
__global__ void k_fit(const double* soa, int N, int row, const int* idx, int len, const double* w, int kind, double* out) {
  __shared__ BlockScratch sc;
  Ctx c;
  blk_ctx(c, &sc, soa, N, row);
  double m[9];
  for (int i = 0; i < 9; ++i) m[i] = NAN;
  if (kind == 0) blk_fit_F(c, idx, len, w, m);
  else blk_fit_H(c, idx, len, m);
  if (c.tid == 0) for (int i = 0; i < 9; ++i) out[i] = m[i];
}

// fused: blk_sample8_fit_F; split: blk_randsubset(8) then blk_fit_F(len 8) on the permuted tail.  list (max_sz ints)
// permuted in place; out[0..8] = F, cur[0] = the cursor's j after the call, cur[1] = warp_sample8_fit's fast flag (fused)
__global__ void k_sample8(const double* soa, int N, int row, int* list, int max_sz, const double* w, uint64_t seed,
                          uint32_t k, uint32_t j0, int fused, double* out, int* cur) {
  __shared__ BlockScratch sc;
  Ctx c;
  blk_ctx(c, &sc, soa, N, row);
  DrawCursor dc;
  dc.seed = seed; dc.k = k; dc.j = j0;
  double f[9];
  if (c.tid == 0) sc.bci[1] = -1;
  DG_SYNC();
  if (fused) {
    blk_sample8_fit_F(c, list, max_sz, w, dc, f);
  } else {
    blk_randsubset(c, list, max_sz, 8, dc);
    blk_fit_F(c, list + max_sz - 8, 8, w, f);
  }
  if (c.tid == 0) {
    for (int i = 0; i < 9; ++i) out[i] = f[i];
    cur[0] = (int)dc.j;
    cur[1] = fused ? sc.bci[1] : -1;
  }
}

// hash_seen_elsewhere on the table {hhash, hlen, hid}[0..*htn) of capacity hcap (updated in place, *htn too); the
// verdict (0 inserted, 1 already ours, 2 abort) to verdict[0] and the hash warp 0 computed is the one it inserted
__global__ void k_hash(const int* list, int n, int iterID, uint32_t* hhash, int* hlen, int* hid, int hcap, int* htn,
                       int* verdict) {
  __shared__ BlockScratch sc;
  Ctx c;
  blk_ctx(c, &sc, nullptr, 0, 0);
  Workspace W;
  memset(&W, 0, sizeof(W));
  W.hhash = hhash; W.hlen = hlen; W.hid = hid; W.hcap = hcap;
  HashTab ht;
  ht.n = *htn;
  DG_SYNC();
  const bool abort = hash_seen_elsewhere(c, W, ht, list, n, iterID);
  if (c.tid == 0) { *htn = ht.n; verdict[0] = sc.bci[0]; verdict[1] = abort ? 1 : 0; }
}

// ---- host side: device copies of the caller's arrays, freed on scope exit
struct Dev {
  void* p = nullptr;
  cudaError_t err = cudaSuccess;
  Dev(const void* host, size_t bytes) {
    err = cudaMalloc(&p, bytes ? bytes : 1);
    if (err == cudaSuccess && host) err = cudaMemcpy(p, host, bytes, cudaMemcpyHostToDevice);
  }
  ~Dev() { if (p) cudaFree(p); }
  template <class T> T* as() const { return static_cast<T*>(p); }
};

int finish(std::initializer_list<const Dev*> bufs) {
  for (const Dev* b : bufs) if (b->err != cudaSuccess) return (int)b->err;
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  return (int)e;
}
int back(void* host, const Dev& d, size_t bytes) { return (int)cudaMemcpy(host, d.p, bytes, cudaMemcpyDeviceToHost); }

}  // namespace

#define DL_CHECK(x) do { const int rc_ = (x); if (rc_) return rc_; } while (0)

extern "C" int dl_blk_inlidxs(const double* err, int N, double thA, double thB, int mode, int nthreads, int* listA,
                              int* listB, double* J, int* I) {
  Dev de(err, sizeof(double) * N), dA(nullptr, sizeof(int) * N), dB(nullptr, sizeof(int) * N),
      dJ(nullptr, sizeof(double) * 2), dI(nullptr, sizeof(int) * 3);
  if (de.err == cudaSuccess)
    k_inlidxs<<<1, nthreads>>>(de.as<double>(), N, thA, thB, mode, dA.as<int>(), dB.as<int>(), dJ.as<double>(), dI.as<int>());
  DL_CHECK(finish({&de, &dA, &dB, &dJ, &dI}));
  DL_CHECK(back(listA, dA, sizeof(int) * N));
  DL_CHECK(back(listB, dB, sizeof(int) * N));
  DL_CHECK(back(J, dJ, sizeof(double) * 2));
  return back(I, dI, sizeof(int) * 3);
}

extern "C" int dl_blk_reduce(const double* vd, const int* vi, const double* vv, int k, int nthreads, double* od, int* oi) {
  const size_t nd = 3 * (size_t)nthreads + kVecRed, ni = 5 * (size_t)nthreads;
  Dev dvd(vd, sizeof(double) * nthreads), dvi(vi, sizeof(int) * nthreads), dvv(vv, sizeof(double) * kVecRed * nthreads),
      dod(od, sizeof(double) * nd), doi(oi, sizeof(int) * ni);
  if (dvd.err == cudaSuccess && dvi.err == cudaSuccess && dvv.err == cudaSuccess && dod.err == cudaSuccess)
    k_reduce<<<1, nthreads>>>(dvd.as<double>(), dvi.as<int>(), dvv.as<double>(), k, dod.as<double>(), doi.as<int>());
  DL_CHECK(finish({&dvd, &dvi, &dvv, &dod, &doi}));
  DL_CHECK(back(od, dod, sizeof(double) * nd));
  return back(oi, doi, sizeof(int) * ni);
}

extern "C" int dl_blk_resid_F(const double* soa, int N, int row, int metric, const double* F, int weighted, int nthreads,
                              double* out, double* w) {
  Dev ds(soa, sizeof(double) * 4 * row), dF(F, sizeof(double) * 9), dout(out, sizeof(double) * N), dw(w, sizeof(double) * N);
  if (ds.err == cudaSuccess && dF.err == cudaSuccess && dout.err == cudaSuccess && dw.err == cudaSuccess)
    k_resid_F<<<1, nthreads>>>(ds.as<double>(), N, row, metric, dF.as<double>(), weighted, dout.as<double>(), dw.as<double>());
  DL_CHECK(finish({&ds, &dF, &dout, &dw}));
  DL_CHECK(back(out, dout, sizeof(double) * N));
  return back(w, dw, sizeof(double) * N);
}

extern "C" int dl_blk_resid_H(const double* soa, int N, int row, int metric, double th, const double* h, int with_tile,
                              int nthreads, double* out) {
  const size_t tb = 16 * ((size_t)N + 1);
  Dev ds(soa, sizeof(double) * 4 * row), dh(h, sizeof(double) * 9), dt(nullptr, tb), dl(nullptr, sizeof(int) * (N + 1)),
      dout(out, sizeof(double) * N);
  if (ds.err == cudaSuccess && dh.err == cudaSuccess && dt.err == cudaSuccess && dl.err == cudaSuccess && dout.err == cudaSuccess)
    k_resid_H<<<1, nthreads>>>(ds.as<double>(), N, row, metric, th, dh.as<double>(), with_tile, dt.as<float>(), dl.as<int>(),
                               dout.as<double>());
  DL_CHECK(finish({&ds, &dh, &dt, &dl, &dout}));
  return back(out, dout, sizeof(double) * N);
}

extern "C" int dl_blk_counts(const double* soa, const double* laf, int N, int row, const int* list, int n, const double* F,
                             const double* h, int fmetric, int hmetric, double sym_th, double th_laf, int nthreads, int* out) {
  Dev ds(soa, sizeof(double) * 4 * row), dl(laf, sizeof(double) * 8 * row), dli(list, sizeof(int) * n),
      dF(F, sizeof(double) * 9), dh(h, sizeof(double) * 9), dout(nullptr, sizeof(int) * 5);
  if (ds.err == cudaSuccess && dl.err == cudaSuccess && dli.err == cudaSuccess && dF.err == cudaSuccess && dh.err == cudaSuccess)
    k_counts<<<1, nthreads>>>(ds.as<double>(), dl.as<double>(), N, row, dli.as<int>(), n, dF.as<double>(), dh.as<double>(),
                              fmetric, hmetric, sym_th, th_laf, dout.as<int>());
  DL_CHECK(finish({&ds, &dl, &dli, &dF, &dh, &dout}));
  return back(out, dout, sizeof(int) * 5);
}

// w: N weights or nullptr
extern "C" int dl_blk_fit(const double* soa, int N, int row, const int* idx, int len, const double* w, int kind,
                          int nthreads, double* out) {
  Dev ds(soa, sizeof(double) * 4 * row), di(idx, sizeof(int) * len), dw(w, w ? sizeof(double) * N : 0),
      dout(nullptr, sizeof(double) * 9);
  if (ds.err == cudaSuccess && di.err == cudaSuccess && dw.err == cudaSuccess)
    k_fit<<<1, nthreads>>>(ds.as<double>(), N, row, di.as<int>(), len, w ? dw.as<double>() : nullptr, kind, dout.as<double>());
  DL_CHECK(finish({&ds, &di, &dw, &dout}));
  return back(out, dout, sizeof(double) * 9);
}

extern "C" int dl_blk_sample8(const double* soa, int N, int row, int* list, int max_sz, const double* w, uint64_t seed,
                              uint32_t k, uint32_t j0, int fused, int nthreads, double* out, int* cur) {
  Dev ds(soa, sizeof(double) * 4 * row), dli(list, sizeof(int) * max_sz), dw(w, w ? sizeof(double) * N : 0),
      dout(nullptr, sizeof(double) * 9), dc(nullptr, sizeof(int) * 2);
  if (ds.err == cudaSuccess && dli.err == cudaSuccess && dw.err == cudaSuccess)
    k_sample8<<<1, nthreads>>>(ds.as<double>(), N, row, dli.as<int>(), max_sz, w ? dw.as<double>() : nullptr, seed, k, j0,
                               fused, dout.as<double>(), dc.as<int>());
  DL_CHECK(finish({&ds, &dli, &dw, &dout, &dc}));
  DL_CHECK(back(list, dli, sizeof(int) * max_sz));
  DL_CHECK(back(out, dout, sizeof(double) * 9));
  return back(cur, dc, sizeof(int) * 2);
}

// table arrays of hcap entries, updated in place; htn in/out; verdict[2] = {bci[0], returned abort}
extern "C" int dl_blk_hash(const int* list, int n, int iterID, uint32_t* hhash, int* hlen, int* hid, int hcap, int* htn,
                           int nthreads, int* verdict) {
  Dev dli(list, sizeof(int) * n), dh(hhash, sizeof(uint32_t) * hcap), dl(hlen, sizeof(int) * hcap),
      di(hid, sizeof(int) * hcap), dn(htn, sizeof(int)), dv(nullptr, sizeof(int) * 2);
  if (dli.err == cudaSuccess && dh.err == cudaSuccess && dl.err == cudaSuccess && di.err == cudaSuccess && dn.err == cudaSuccess)
    k_hash<<<1, nthreads>>>(dli.as<int>(), n, iterID, dh.as<uint32_t>(), dl.as<int>(), di.as<int>(), hcap, dn.as<int>(),
                            dv.as<int>());
  DL_CHECK(finish({&dli, &dh, &dl, &di, &dn, &dv}));
  DL_CHECK(back(hhash, dh, sizeof(uint32_t) * hcap));
  DL_CHECK(back(hlen, dl, sizeof(int) * hcap));
  DL_CHECK(back(hid, di, sizeof(int) * hcap));
  DL_CHECK(back(htn, dn, sizeof(int)));
  return back(verdict, dv, sizeof(int) * 2);
}
