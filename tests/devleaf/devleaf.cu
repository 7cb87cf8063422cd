// devleaf.cu -- TEST HELPER ONLY.  The device twin of tests/hostemu/hostemu.cpp: the engine headers, unchanged, compiled
// by nvcc with the library's flags (sm_90a, -fmad=false), and one small kernel per DEVICE-ONLY leaf, run the way the
// engine runs it (one warp per 9x9 / 8x9 solve with its WarpScratch in shared memory, two threads per 7-point sample,
// one thread per 3x3 solve, one warp per FP32-scored model).  Every launcher takes and returns host arrays and reports
// the CUDA status; tests/devleaf/dev.py loads it with ctypes.  Never loaded by the pydegensac_b200 package.
#include <cuda_runtime.h>
#include <string.h>
#include "../../pydegensac_b200/csrc/engine_f.h"
#include "../../pydegensac_b200/csrc/engine_h.h"

using namespace dg;

namespace {

constexpr int kWarpsPerBlock = 4;

// warp-per-item launch geometry: item index of this warp, or -1
__device__ int warp_item(int n) {
  const int i = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  return i < n ? i : -1;
}
int warp_blocks(int n) { return (n + kWarpsPerBlock - 1) / kWarpsPerBlock; }

enum { EIG_DISPATCH = 0, EIG_INV = 1, EIG_REG = 2, EIG_JACOBI = 3 };

// x: ws->cs[0..8] on return; Aout / Vout: ws->A and ws->V on return; ok: the flavour's return value (1 for the others)
__global__ void k_eig9(const double* A, int n, int mode, double* x, double* Aout, double* Vout, int* ok) {
#if DG_DEVICE_PASS   // (the warp leaves exist in the device pass only)
  __shared__ WarpScratch tiles[kWarpsPerBlock];
  const int i = warp_item(n);
  if (i < 0) return;
  WarpScratch* ws = &tiles[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  for (int t = lane; t < 81; t += 32) { ws->A[t] = A[(size_t)i * 81 + t]; ws->V[t] = 0.0; }
  if (lane < 16) ws->cs[lane] = NAN;
  __syncwarp();
  bool r = true;
  if (mode == EIG_DISPATCH) warp_smallest_eigvec9(ws, lane, 32);
  else if (mode == EIG_INV) r = warp_smallest_eigvec9_inv(ws, lane);
  else if (mode == EIG_REG) r = warp_smallest_eigvec9_reg(ws, lane);
  else warp_jacobi_eig9(ws, lane, 32);
  __syncwarp();
  if (lane < 9) x[(size_t)i * 9 + lane] = ws->cs[lane];
  for (int t = lane; t < 81; t += 32) { Aout[(size_t)i * 81 + t] = ws->A[t]; Vout[(size_t)i * 81 + t] = ws->V[t]; }
  if (lane == 0) ok[i] = r ? 1 : 0;
#endif
}

enum { NULL_REG = 0, NULL_8X9 = 1, NULL_HOUSEHOLDER = 2, NULL_DISPATCH = 3 };

// Z: 9 x len row-major per item (72 doubles each); NULL_DISPATCH is the LSQ fit's choice (ffit.h): the lane-parallel
// Gauss-Jordan for len == 8, the Householder route when it declines or for shorter systems
__global__ void k_null9(const double* Z, const int* len, int n, int mode, double* q, int* ok) {
#if DG_DEVICE_PASS   // (the warp leaves exist in the device pass only)
  __shared__ WarpScratch tiles[kWarpsPerBlock];
  const int i = warp_item(n);
  if (i < 0) return;
  WarpScratch* ws = &tiles[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  for (int t = lane; t < 72; t += 32) ws->A[t] = Z[(size_t)i * 72 + t];
  if (lane < 16) ws->cs[lane] = NAN;
  __syncwarp();
  bool r = true;
  if (mode == NULL_REG) r = warp_null_8x9_reg(ws, lane);
  else if (mode == NULL_8X9) r = warp_null_8x9(ws, lane, 32);
  else if (mode == NULL_HOUSEHOLDER) warp_left_null_9xk(ws, len[i], lane, 32);
  else {
    bool have = false;
    if (len[i] == 8) have = warp_null_8x9(ws, lane, 32);
    if (!have) warp_left_null_9xk(ws, len[i], lane, 32);
  }
  __syncwarp();
  if (lane < 9) q[(size_t)i * 9 + lane] = ws->cs[lane];
  if (lane == 0) ok[i] = r ? 1 : 0;
#endif
}

// The wave's pair elimination for iterations kbeg..kend, with Ctx / FParams / Workspace set up as the pair kernel sets
// them up for it; one CTA of `nt` threads.
__global__ void k_pairsolve(const double* soa, int N, int row, uint64_t seed, int kbeg, int kend, double* nsbuf) {
#if DG_DEVICE_PASS   // (the warp leaves exist in the device pass only)
  Ctx c;
  memset(&c, 0, sizeof(c));
  c.tid = threadIdx.x; c.nt = blockDim.x; c.lane = c.tid & 31; c.wid = c.tid >> 5; c.nw = c.nt >> 5;
  c.N = N;
  c.x1 = soa; c.y1 = soa + row; c.x2 = soa + 2 * row; c.y2 = soa + 3 * row;
  FParams P;
  memset(&P, 0, sizeof(P));
  P.seed = seed;
  Workspace W;
  memset(&W, 0, sizeof(W));
  W.nsbuf = nsbuf;
  wave_F_pairsolve(c, P, W, kbeg, kend);
#endif
}

// one thread per 9x9 system: the one-thread null space (the wave's fallback for non-generic samples)
__global__ void k_nullspace9(const double* M, int n, double* ns, int* nfree) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double m[81], o[81];
  for (int t = 0; t < 81; ++t) m[t] = M[(size_t)i * 81 + t];
  nfree[i] = nullspace9(m, o);
  for (int t = 0; t < 18; ++t) ns[(size_t)i * 18 + t] = o[t];
}

// one thread per 3x3: out[52] = enforce_rank2 (9), enforce_rank2_slow (9), enforce_rank2_inl (9),
// smallest_right_sv3_fast (v 3, ok 1), svd3_onesided (G 9, V 9, sv 3)
constexpr int kSmall3Out = 52;
__global__ void k_small3(const double* F, int n, double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* f = F + (size_t)i * 9;
  double* o = out + (size_t)i * kSmall3Out;
  double a[9], b[9], cc[9], v[3], G[9], V[9], sv[3];
  for (int t = 0; t < 9; ++t) { a[t] = f[t]; b[t] = f[t]; cc[t] = f[t]; }
  enforce_rank2(a);
  enforce_rank2_slow(b);
  enforce_rank2_inl(cc);
  v[0] = v[1] = v[2] = NAN;
  const bool ok = smallest_right_sv3_fast(f, v);
  svd3_onesided(f, G, V, sv);
  for (int t = 0; t < 9; ++t) { o[t] = a[t]; o[9 + t] = b[t]; o[18 + t] = cc[t]; o[31 + t] = G[t]; o[40 + t] = V[t]; }
  for (int t = 0; t < 3; ++t) { o[27 + t] = v[t]; o[49 + t] = sv[t]; }
  o[30] = ok ? 1.0 : 0.0;
}

__global__ void k_pow2(const double* t, int n, double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = pow2_inv_exponent(t[i]);
}

// The pair's FP32 tile exactly as the pair kernel builds it (device branch: pair-interleaved, odd-N padding slot);
// cenbnd = Tile32::cen, Tile32::bnd
__global__ void k_tile32(const double* soa, int N, int row, float* tile, double* cenbnd) {
  __shared__ BlockScratch sc;
  Ctx c;
  memset(&c, 0, sizeof(c));
  c.tid = threadIdx.x; c.nt = blockDim.x; c.lane = c.tid & 31; c.wid = c.tid >> 5; c.nw = c.nt >> 5;
  c.N = N;
  c.x1 = soa; c.y1 = soa + row; c.x2 = soa + 2 * row; c.y2 = soa + 3 * row;
  c.sc = &sc;
  Tile32 T;
  blk_prepare_tile32(c, reinterpret_cast<Pt32*>(tile), &T);
  if (c.tid == 0)
    for (int k = 0; k < 4; ++k) { cenbnd[k] = T.cen[k]; cenbnd[4 + k] = T.bnd[k]; }
}

__device__ Tile32 tile_of(const float* tile, const double* cenbnd) {
  Tile32 T;
  T.pts = reinterpret_cast<const Pt32*>(tile);
  for (int k = 0; k < 4; ++k) { T.cen[k] = cenbnd[k]; T.bnd[k] = cenbnd[4 + k]; }
  return T;
}

// One warp per F model, the wave's stage-B loop (engine_f.h) with every gain stored: gains[m][2 npair], J[m] as the
// wave sums it (before the (1 + 2^-16) + 1e-3 of J_up).
__global__ void k_ffilter(const float* tile, const double* cenbnd, int N, int metric, double w, const double* F, int nm,
                          float* gains, float* J) {
#if DG_DEVICE_PASS   // (the warp leaves exist in the device pass only)
  const int m = warp_item(nm);
  if (m < 0) return;
  const int lane = threadIdx.x & 31;
  const Tile32 T = tile_of(tile, cenbnd);
  FFilter32 ff;
  f_filter_setup(metric, F + (size_t)m * 9, T, w, &ff);
  FFilter32x2 f2;
  f_filter_pack(ff, &f2);
  const float4* tp = reinterpret_cast<const float4*>(tile);
  const int npair = (N + 1) >> 1;
  const int last = (N & 1) ? npair - 1 : -1;
  float2* g = reinterpret_cast<float2*>(gains + (size_t)m * 2 * npair);
  f32x2 Ja = pk2(0.0f, 0.0f), Jb = pk2(0.0f, 0.0f);
  int i = lane;
  for (; i + 32 < npair; i += 64) {
    const f32x2 g0 = f_filter_gain2(f2, tp[2 * i], tp[2 * i + 1], i != last);
    const f32x2 g1 = f_filter_gain2(f2, tp[2 * i + 64], tp[2 * i + 65], i + 32 != last);
    g[i] = g0; g[i + 32] = g1;
    Ja = add2(Ja, g0);
    Jb = add2(Jb, g1);
  }
  if (i < npair) {
    const f32x2 g0 = f_filter_gain2(f2, tp[2 * i], tp[2 * i + 1], i != last);
    g[i] = g0;
    Ja = add2(Ja, g0);
  }
  float j0, j1;
  upk2(add2(Ja, Jb), j0, j1);
  float s = j0 + j1;
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) J[m] = s;
#endif
}

// One warp per H model (column-major h, image 2 -> image 1): gains and J at width w (the wave's stage B, engine_h.h),
// and the unclamped bound raw[m][2 npair] at width w_far (the residual-row classification of blk_resid_H).
__global__ void k_hfilter(const float* tile, const double* cenbnd, int N, double w, double w_far, const double* h, int nm,
                          float* gains, float* J, float* raw) {
#if DG_DEVICE_PASS   // (the warp leaves exist in the device pass only)
  const int m = warp_item(nm);
  if (m < 0) return;
  const int lane = threadIdx.x & 31;
  const Tile32 T = tile_of(tile, cenbnd);
  HFilter32 hf, hff;
  h_filter_setup(h + (size_t)m * 9, T, w, &hf);
  h_filter_setup(h + (size_t)m * 9, T, w_far, &hff);
  HFilter32x2 f2, f2far;
  h_filter_pack(hf, &f2);
  h_filter_pack(hff, &f2far);
  const float4* tp = reinterpret_cast<const float4*>(tile);
  const int npair = (N + 1) >> 1;
  const int last = (N & 1) ? npair - 1 : -1;
  float2* g = reinterpret_cast<float2*>(gains + (size_t)m * 2 * npair);
  float2* rw = reinterpret_cast<float2*>(raw + (size_t)m * 2 * npair);
  for (int q = lane; q < npair; q += 32) rw[q] = h_filter_raw2(f2far, tp[2 * q], tp[2 * q + 1]);
  f32x2 Ja = pk2(0.0f, 0.0f), Jb = pk2(0.0f, 0.0f);
  int i = lane;
  for (; i + 32 < npair; i += 64) {
    const f32x2 g0 = h_filter_gain2(f2, tp[2 * i], tp[2 * i + 1], i != last);
    const f32x2 g1 = h_filter_gain2(f2, tp[2 * i + 64], tp[2 * i + 65], i + 32 != last);
    g[i] = g0; g[i + 32] = g1;
    Ja = add2(Ja, g0);
    Jb = add2(Jb, g1);
  }
  if (i < npair) {
    const f32x2 g0 = h_filter_gain2(f2, tp[2 * i], tp[2 * i + 1], i != last);
    g[i] = g0;
    Ja = add2(Ja, g0);
  }
  float j0, j1;
  upk2(add2(Ja, Jb), j0, j1);
  float s = j0 + j1;
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) J[m] = s;
#endif
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

extern "C" int dl_eig9(const double* A, int n, int mode, double* x, double* Aout, double* Vout, int* ok) {
  Dev dA(A, sizeof(double) * 81 * n), dx(nullptr, sizeof(double) * 9 * n), dAo(nullptr, sizeof(double) * 81 * n),
      dV(nullptr, sizeof(double) * 81 * n), dok(nullptr, sizeof(int) * n);
  if (dA.err == cudaSuccess && n > 0)
    k_eig9<<<warp_blocks(n), 32 * kWarpsPerBlock>>>(dA.as<double>(), n, mode, dx.as<double>(), dAo.as<double>(),
                                                    dV.as<double>(), dok.as<int>());
  DL_CHECK(finish({&dA, &dx, &dAo, &dV, &dok}));
  DL_CHECK(back(x, dx, sizeof(double) * 9 * n));
  DL_CHECK(back(Aout, dAo, sizeof(double) * 81 * n));
  DL_CHECK(back(Vout, dV, sizeof(double) * 81 * n));
  return back(ok, dok, sizeof(int) * n);
}

extern "C" int dl_null9(const double* Z, const int* len, int n, int mode, double* q, int* ok) {
  Dev dZ(Z, sizeof(double) * 72 * n), dl(len, sizeof(int) * n), dq(nullptr, sizeof(double) * 9 * n),
      dok(nullptr, sizeof(int) * n);
  if (dZ.err == cudaSuccess && dl.err == cudaSuccess && n > 0)
    k_null9<<<warp_blocks(n), 32 * kWarpsPerBlock>>>(dZ.as<double>(), dl.as<int>(), n, mode, dq.as<double>(), dok.as<int>());
  DL_CHECK(finish({&dZ, &dl, &dq, &dok}));
  DL_CHECK(back(q, dq, sizeof(double) * 9 * n));
  return back(ok, dok, sizeof(int) * n);
}

// soa: x1, y1, x2, y2 rows of `row` doubles each; nsbuf: 16 doubles per iteration kbeg..kend
extern "C" int dl_pairsolve(const double* soa, int N, int row, uint64_t seed, int kbeg, int kend, int nthreads,
                            double* nsbuf) {
  const int n = kend - kbeg + 1;
  Dev ds(soa, sizeof(double) * 4 * row), dns(nsbuf, sizeof(double) * 16 * n);
  if (ds.err == cudaSuccess && dns.err == cudaSuccess)
    k_pairsolve<<<1, nthreads>>>(ds.as<double>(), N, row, seed, kbeg, kend, dns.as<double>());
  DL_CHECK(finish({&ds, &dns}));
  return back(nsbuf, dns, sizeof(double) * 16 * n);
}

extern "C" int dl_nullspace9(const double* M, int n, double* ns, int* nfree) {
  Dev dM(M, sizeof(double) * 81 * n), dns(nullptr, sizeof(double) * 18 * n), dnf(nullptr, sizeof(int) * n);
  if (dM.err == cudaSuccess && n > 0) k_nullspace9<<<(n + 63) / 64, 64>>>(dM.as<double>(), n, dns.as<double>(), dnf.as<int>());
  DL_CHECK(finish({&dM, &dns, &dnf}));
  DL_CHECK(back(ns, dns, sizeof(double) * 18 * n));
  return back(nfree, dnf, sizeof(int) * n);
}

extern "C" int dl_small3(const double* F, int n, double* out) {
  Dev dF(F, sizeof(double) * 9 * n), dout(nullptr, sizeof(double) * kSmall3Out * n);
  if (dF.err == cudaSuccess && n > 0) k_small3<<<(n + 127) / 128, 128>>>(dF.as<double>(), n, dout.as<double>());
  DL_CHECK(finish({&dF, &dout}));
  return back(out, dout, sizeof(double) * kSmall3Out * n);
}

extern "C" int dl_pow2_inv_exponent(const double* t, int n, double* out) {
  Dev dt(t, sizeof(double) * n), dout(nullptr, sizeof(double) * n);
  if (dt.err == cudaSuccess && n > 0) k_pow2<<<(n + 255) / 256, 256>>>(dt.as<double>(), n, dout.as<double>());
  DL_CHECK(finish({&dt, &dout}));
  return back(out, dout, sizeof(double) * n);
}

// tile: 8 floats per correspondence pair, pre-filled by the caller (slots the kernel leaves alone keep that content)
extern "C" int dl_tile32(const double* soa, int N, int row, int nthreads, float* tile, double* cenbnd) {
  const size_t tb = sizeof(float) * 8 * (size_t)((N + 1) / 2);
  Dev ds(soa, sizeof(double) * 4 * row), dt(tile, tb), dc(nullptr, sizeof(double) * 8);
  if (ds.err == cudaSuccess && dt.err == cudaSuccess)
    k_tile32<<<1, nthreads>>>(ds.as<double>(), N, row, dt.as<float>(), dc.as<double>());
  DL_CHECK(finish({&ds, &dt, &dc}));
  DL_CHECK(back(tile, dt, tb));
  return back(cenbnd, dc, sizeof(double) * 8);
}

extern "C" int dl_ffilter(const float* tile, const double* cenbnd, int N, int metric, double w, const double* F, int nm,
                          float* gains, float* J) {
  const size_t np = (size_t)((N + 1) / 2);
  Dev dt(tile, sizeof(float) * 8 * np), dc(cenbnd, sizeof(double) * 8), dF(F, sizeof(double) * 9 * nm),
      dg(nullptr, sizeof(float) * 2 * np * nm), dJ(nullptr, sizeof(float) * nm);
  if (dt.err == cudaSuccess && dc.err == cudaSuccess && dF.err == cudaSuccess && nm > 0)
    k_ffilter<<<warp_blocks(nm), 32 * kWarpsPerBlock>>>(dt.as<float>(), dc.as<double>(), N, metric, w, dF.as<double>(), nm,
                                                        dg.as<float>(), dJ.as<float>());
  DL_CHECK(finish({&dt, &dc, &dF, &dg, &dJ}));
  DL_CHECK(back(gains, dg, sizeof(float) * 2 * np * nm));
  return back(J, dJ, sizeof(float) * nm);
}

extern "C" int dl_hfilter(const float* tile, const double* cenbnd, int N, double w, double w_far, const double* h, int nm,
                          float* gains, float* J, float* raw) {
  const size_t np = (size_t)((N + 1) / 2);
  Dev dt(tile, sizeof(float) * 8 * np), dc(cenbnd, sizeof(double) * 8), dh(h, sizeof(double) * 9 * nm),
      dg(nullptr, sizeof(float) * 2 * np * nm), dJ(nullptr, sizeof(float) * nm), dr(nullptr, sizeof(float) * 2 * np * nm);
  if (dt.err == cudaSuccess && dc.err == cudaSuccess && dh.err == cudaSuccess && nm > 0)
    k_hfilter<<<warp_blocks(nm), 32 * kWarpsPerBlock>>>(dt.as<float>(), dc.as<double>(), N, w, w_far, dh.as<double>(), nm,
                                                        dg.as<float>(), dJ.as<float>(), dr.as<float>());
  DL_CHECK(finish({&dt, &dc, &dh, &dg, &dJ, &dr}));
  DL_CHECK(back(gains, dg, sizeof(float) * 2 * np * nm));
  DL_CHECK(back(raw, dr, sizeof(float) * 2 * np * nm));
  return back(J, dJ, sizeof(float) * nm);
}
