"""ctypes loader of the device leaf harness devleaf.cu (TEST HELPER ONLY).

The harness is compiled with the library's own nvcc flags (pydegensac_b200.build.NVCC_FLAGS: sm_90a, -fmad=false), so
each leaf it runs is the code the pair kernel runs.  __graft_entry__.build() builds it next to the library; here it is
rebuilt only when it is older than its source or an engine header."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "devleaf.cu")
_SO = os.path.join(_HERE, "libdevleaf.so")
_lib = None

EIG_DISPATCH, EIG_INV, EIG_REG, EIG_JACOBI = 0, 1, 2, 3
NULL_REG, NULL_8X9, NULL_HOUSEHOLDER, NULL_DISPATCH = 0, 1, 2, 3
CTA_THREADS = 256      # the pair kernel's CTA (degensac_b200.cu)


def _stale():
    from pydegensac_b200 import build as b
    deps = [_SRC] + [os.path.join(b.CSRC, f) for f in os.listdir(b.CSRC) if f.endswith(".h")]
    return not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(p) for p in deps)


def build(force=False):
    from pydegensac_b200 import build as b
    if force or _stale():
        nvcc = os.environ.get("NVCC", "nvcc")
        subprocess.check_call([nvcc] + b.NVCC_FLAGS + ["-o", _SO, _SRC])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_SO)
    return _lib


def _d(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def _f(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def _i(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))


def _check(rc):
    assert rc == 0, "CUDA error %d in the device leaf harness" % rc


def eig9(A, mode):
    """A: [n, 9, 9].  Returns (x [n, 9] = ws->cs, A after [n, 9, 9], V after [n, 9, 9], ok [n] bool)."""
    A = np.ascontiguousarray(A, dtype=np.float64).reshape(-1, 81)
    n = A.shape[0]
    x = np.zeros((n, 9)); Ao = np.zeros((n, 81)); Vo = np.zeros((n, 81)); ok = np.zeros(n, dtype=np.int32)
    _check(lib().dl_eig9(_d(A), n, int(mode), _d(x), _d(Ao), _d(Vo), _i(ok)))
    return x, Ao.reshape(n, 9, 9), Vo.reshape(n, 9, 9), ok.astype(bool)


def null9(Z, lens, mode):
    """Z: [n, 72] (9 x len row-major, zero padded).  Returns (q [n, 9] = ws->cs, ok [n] bool)."""
    Z = np.ascontiguousarray(Z, dtype=np.float64).reshape(-1, 72)
    n = Z.shape[0]
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    q = np.zeros((n, 9)); ok = np.zeros(n, dtype=np.int32)
    _check(lib().dl_null9(_d(Z), _i(lens), n, int(mode), _d(q), _i(ok)))
    return q, ok.astype(bool)


def _soa(p1, p2):
    n = p1.shape[0]
    row = ((8 * n + 127) // 128 * 128) // 8            # rows aligned like the engine's SoA copy
    soa = np.zeros(4 * row)
    for k, v in enumerate((p1[:, 0], p1[:, 1], p2[:, 0], p2[:, 1])):
        soa[k * row:k * row + n] = v
    return soa, row


def pairsolve(p1, p2, seed, kbeg, kend):
    """The wave's pair elimination (one CTA of the pair kernel's size): [kend - kbeg + 1, 16] =
    {-col7[0..6], -col8[0..6], generic, unused}."""
    soa, row = _soa(p1, p2)
    ns = np.full((kend - kbeg + 1, 16), np.nan)
    _check(lib().dl_pairsolve(_d(soa), p1.shape[0], row, ctypes.c_uint64(seed), int(kbeg), int(kend), CTA_THREADS, _d(ns)))
    return ns


def nullspace9(M):
    """One device thread per [9, 9] system: (ns [n, 18], nfree [n])."""
    M = np.ascontiguousarray(M, dtype=np.float64).reshape(-1, 81)
    n = M.shape[0]
    ns = np.zeros((n, 18)); nf = np.zeros(n, dtype=np.int32)
    _check(lib().dl_nullspace9(_d(M), n, _d(ns), _i(nf)))
    return ns, nf


def small3(F):
    """One device thread per 3x3 F: dict of enforce_rank2 / _slow / _inl results, smallest_right_sv3_fast (v, ok) and
    svd3_onesided (G, V, sv)."""
    F = np.ascontiguousarray(F, dtype=np.float64).reshape(-1, 9)
    n = F.shape[0]
    o = np.zeros((n, 52))
    _check(lib().dl_small3(_d(F), n, _d(o)))
    return dict(rank2=o[:, 0:9], rank2_slow=o[:, 9:18], rank2_inl=o[:, 18:27], v=o[:, 27:30], fast_ok=o[:, 30] != 0,
                G=o[:, 31:40], V=o[:, 40:49], sv=o[:, 49:52])


def pow2_inv_exponent(t):
    t = np.ascontiguousarray(t, dtype=np.float64)
    out = np.zeros_like(t)
    _check(lib().dl_pow2_inv_exponent(_d(t), t.size, _d(out)))
    return out


def tile32(p1, p2, fill=np.nan):
    """The pair kernel's FP32 tile: (tile [ceil(N/2), 8] floats {u0 u1 v0 v1 s0 s1 t0 t1}, cenbnd [8])."""
    soa, row = _soa(p1, p2)
    n = p1.shape[0]
    tile = np.full(((n + 1) // 2, 8), fill, dtype=np.float32)
    cb = np.zeros(8)
    _check(lib().dl_tile32(_d(soa), n, row, CTA_THREADS, _f(tile), _d(cb)))
    return tile, cb


def ffilter(tile, cb, n, metric, w, F):
    """Gains [m, 2 ceil(N/2)] and the wave's FP32 sum J [m] of the F models [m, 9] (row-major)."""
    F = np.ascontiguousarray(F, dtype=np.float64).reshape(-1, 9)
    m = F.shape[0]
    g = np.zeros((m, tile.shape[0] * 2), dtype=np.float32); J = np.zeros(m, dtype=np.float32)
    _check(lib().dl_ffilter(_f(tile), _d(cb), int(n), int(metric), ctypes.c_double(w), _d(F), m, _f(g), _f(J)))
    return g, J


def hfilter(tile, cb, n, w, w_far, h):
    """Gains, J (width w) and the unclamped bound raw (width w_far) of the H models [m, 9] (column-major h)."""
    h = np.ascontiguousarray(h, dtype=np.float64).reshape(-1, 9)
    m = h.shape[0]
    g = np.zeros((m, tile.shape[0] * 2), dtype=np.float32); J = np.zeros(m, dtype=np.float32)
    raw = np.zeros_like(g)
    _check(lib().dl_hfilter(_f(tile), _d(cb), int(n), ctypes.c_double(w), ctypes.c_double(w_far), _d(h), m, _f(g), _f(J),
                            _f(raw)))
    return g, J, raw
