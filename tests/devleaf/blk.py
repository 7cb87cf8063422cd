"""ctypes loader of the block-level device harness blockleaf.cu and of its host twin blockhost.cpp (TEST HELPERS ONLY).

blockleaf.cu is compiled with the library's own nvcc flags (pydegensac_b200.build.NVCC_FLAGS: sm_90a, -fmad=false), so
each primitive it runs is the code the pair kernel runs; blockhost.cpp builds the compaction of block.h with g++ as a
one-thread CTA.  __graft_entry__.build() builds both next to the library; here each is rebuilt only when it is older
than its source or an engine header."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "blockleaf.cu")
_SO = os.path.join(_HERE, "libblockleaf.so")
_HSRC = os.path.join(_HERE, "blockhost.cpp")
_HSO = os.path.join(_HERE, "libblockhost.so")
_lib = None
_hlib = None


def _stale(src, so):
    from pydegensac_b200 import build as b
    deps = [src] + [os.path.join(b.CSRC, f) for f in os.listdir(b.CSRC) if f.endswith(".h")]
    return not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(p) for p in deps)


def build(force=False):
    from pydegensac_b200 import build as b
    if force or _stale(_SRC, _SO):
        nvcc = os.environ.get("NVCC", "nvcc")
        subprocess.check_call([nvcc] + b.NVCC_FLAGS + ["-o", _SO, _SRC])
    if force or _stale(_HSRC, _HSO):
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-o", _HSO, _HSRC])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_SO)
    return _lib


def host_lib():
    global _hlib
    if _hlib is None:
        build()
        _hlib = ctypes.CDLL(_HSO)
    return _hlib


def _d(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def _i(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))


def _u32(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32))


def _check(rc):
    assert rc == 0, "CUDA error %d in the block-level harness" % rc


def _soa(p1, p2):
    n = p1.shape[0]
    row = ((8 * n + 127) // 128 * 128) // 8            # rows aligned like the engine's SoA copy
    soa = np.zeros(4 * row)
    for k, v in enumerate((p1[:, 0], p1[:, 1], p2[:, 0], p2[:, 1])):
        soa[k * row:k * row + n] = v
    return soa, row


def host_blk_inlidxs(err, thA, thB, two):
    """The one-thread build of blk_inlidxs (two calls, two=False) or blk_inlidxs2 (two=True): (listA, listB, J, I)."""
    err = np.ascontiguousarray(err, dtype=np.float64)
    n = err.size
    la = np.full(max(n, 1), -1, np.int32); lb = np.full(max(n, 1), -1, np.int32)
    J = np.zeros(2); I = np.zeros(3, np.int32)
    host_lib().hb_blk_inlidxs(_d(err), n, ctypes.c_double(thA), ctypes.c_double(thB), int(bool(two)), _i(la), _i(lb),
                              _d(J), _i(I))
    return la[:I[0]], lb[:I[1]], J, I


def blk_inlidxs(err, thA, thB, two, nt):
    """(listA, listB, J [2], I [3]): two blk_inlidxs calls (two=False) or one blk_inlidxs2 (two=True); I[2] is
    blk_count_lt(thA).  Lists are cut to their counts."""
    err = np.ascontiguousarray(err, dtype=np.float64)
    n = err.size
    la = np.full(max(n, 1), -1, np.int32); lb = np.full(max(n, 1), -1, np.int32)
    J = np.zeros(2); I = np.zeros(3, np.int32)
    _check(lib().dl_blk_inlidxs(_d(err), n, ctypes.c_double(thA), ctypes.c_double(thB), int(bool(two)), int(nt), _i(la),
                                _i(lb), _d(J), _i(I)))
    return la[:I[0]], lb[:I[1]], J, I


def blk_reduce(vd, vi, vv, k, nt):
    """Per-thread results: dict(sum [nt], scan_sum_J [nt], vec [k], sum_i, excl, excl_total, scan_off, scan_total)."""
    vd = np.ascontiguousarray(vd, np.float64); vi = np.ascontiguousarray(vi, np.int32)
    vv = np.ascontiguousarray(vv, np.float64).reshape(nt, 48)
    od = np.full(3 * nt + 48, np.nan); oi = np.full(5 * nt, -7, np.int32)
    _check(lib().dl_blk_reduce(_d(vd), _i(vi), _d(vv), int(k), int(nt), _d(od), _i(oi)))
    return dict(sum=od[:nt], scan_sum_J=od[nt:2 * nt], vec=od[3 * nt:3 * nt + k], sum_i=oi[:nt], excl=oi[nt:2 * nt],
                excl_total=oi[2 * nt:3 * nt], scan_off=oi[3 * nt:4 * nt], scan_total=oi[4 * nt:])


def blk_resid_F(p1, p2, metric, F, weighted, nt):
    """(row [N], weights [N] or None); entries the kernel does not write stay NaN."""
    soa, row = _soa(p1, p2)
    n = p1.shape[0]
    F = np.ascontiguousarray(F, np.float64).reshape(9)
    out = np.full(n, np.nan); w = np.full(n, np.nan)
    _check(lib().dl_blk_resid_F(_d(soa), n, row, int(metric), _d(F), int(bool(weighted)), int(nt), _d(out), _d(w)))
    return out, (w if weighted else None)


def blk_resid_H(p1, p2, metric, th, h, with_tile, nt):
    """Row [N] of blk_resid_H (h column-major, image 2 -> image 1); unwritten entries stay NaN."""
    soa, row = _soa(p1, p2)
    n = p1.shape[0]
    h = np.ascontiguousarray(h, np.float64).reshape(9)
    out = np.full(n, np.nan)
    _check(lib().dl_blk_resid_H(_d(soa), n, row, int(metric), ctypes.c_double(th), _d(h), int(bool(with_tile)), int(nt),
                                _d(out)))
    return out


def blk_counts(p1, p2, laf, lst, F, h, fmetric, hmetric, sym_th, th_laf, nt):
    """{sym_F, laf_F, sym_H, laf_H_p1, laf_H_p2} over lst; laf: [N, 8] helper rows (p1 x1 y1 x2 y2, p2 x1 y1 x2 y2)."""
    soa, row = _soa(p1, p2)
    n = p1.shape[0]
    lf = np.zeros(8 * row)
    for k in range(8):
        lf[k * row:k * row + n] = laf[:, k]
    lst = np.ascontiguousarray(lst, np.int32)
    F = np.ascontiguousarray(F, np.float64).reshape(9); h = np.ascontiguousarray(h, np.float64).reshape(9)
    out = np.zeros(5, np.int32)
    _check(lib().dl_blk_counts(_d(soa), _d(lf), n, row, _i(lst), lst.size, _d(F), _d(h), int(fmetric), int(hmetric),
                               ctypes.c_double(sym_th), ctypes.c_double(th_laf), int(nt), _i(out)))
    return out


def blk_fit(p1, p2, idx, w, kind, nt):
    """blk_fit_F (kind 0; F row-major) or blk_fit_H (kind 1; h column-major) on idx."""
    soa, row = _soa(p1, p2)
    n = p1.shape[0]
    idx = np.ascontiguousarray(idx, np.int32)
    wp = None
    if w is not None:
        w = np.ascontiguousarray(w, np.float64)
        wp = _d(w)
    out = np.full(9, np.nan)
    _check(lib().dl_blk_fit(_d(soa), n, row, _i(idx), idx.size, wp, int(kind), int(nt), _d(out)))
    return out


def blk_sample8(p1, p2, lst, w, seed, k, j0, fused, nt):
    """(permuted list, F [9], cursor j after, fast flag or -1) of blk_sample8_fit_F (fused) or blk_randsubset(8) +
    blk_fit_F(len 8)."""
    soa, row = _soa(p1, p2)
    n = p1.shape[0]
    lst = np.array(lst, np.int32)
    wp = None
    if w is not None:
        w = np.ascontiguousarray(w, np.float64)
        wp = _d(w)
    out = np.full(9, np.nan); cur = np.zeros(2, np.int32)
    _check(lib().dl_blk_sample8(_d(soa), n, row, _i(lst), lst.size, wp, ctypes.c_uint64(seed), ctypes.c_uint32(k),
                                ctypes.c_uint32(j0), int(bool(fused)), int(nt), _d(out), _i(cur)))
    return lst, out, int(cur[0]), int(cur[1])


def blk_hash(lst, iterID, table, nt):
    """hash_seen_elsewhere on `table` = dict(hash, len, id [hcap], n), updated in place; returns (verdict, abort)."""
    lst = np.ascontiguousarray(lst, np.int32)
    htn = np.array([table["n"]], np.int32)
    v = np.zeros(2, np.int32)
    _check(lib().dl_blk_hash(_i(lst) if lst.size else _i(np.zeros(1, np.int32)), lst.size, int(iterID), _u32(table["hash"]),
                             _i(table["len"]), _i(table["id"]), table["hash"].size, _i(htn), int(nt), _i(v)))
    table["n"] = int(htn[0])
    return int(v[0]), bool(v[1])
