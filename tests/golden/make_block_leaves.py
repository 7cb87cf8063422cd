"""Generates tests/golden/ref_block_leaves_v1.npz: outputs of the UNMODIFIED reference's own C leaves (oracle/_ref) on the
seeded inputs of tests/test_block_leaves.py -- the residual rows FDs, FDsSym, exFDs, exFDsSym, HDs, HDsSymMaxSq,
HDsSymMax, HDsSymSumSq, HDsSymSum, the fits u2f, u2fw, u2h, and SuperFastHash.  Needs oracle/_ref (oracle/build_ref.sh):

    python tests/golden/make_block_leaves.py
"""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref  # noqa: E402
from tests.test_block_leaves import (FIT_F_LENGTHS, FIT_H_LENGTHS, H_METRICS, _u6, f_resid_inputs, fit_inputs,  # noqa: E402
                                     fit_inputs_h, h_resid_inputs, hash_inputs)

dp = ctypes.POINTER(ctypes.c_double)
ip = ctypes.POINTER(ctypes.c_int)


def _p(a):
    return a.ctypes.data_as(dp)


def h_rows(L, p1, p2, h, name):
    u = np.ascontiguousarray(_u6(p1, p2))
    n = len(p1)
    lin = np.zeros(18 * n)
    inl = np.arange(n, dtype=np.int32)
    L.lin_hg(_p(u), _p(lin), inl.ctypes.data_as(ip), n)
    out = np.zeros(n)
    getattr(L, name)(_p(lin), _p(u), _p(np.ascontiguousarray(h)), _p(out), n)
    return out


def main():
    L = ref.lib()
    out = {}
    p1, p2, Fs = f_resid_inputs()
    u = np.ascontiguousarray(_u6(p1, p2))
    n = len(p1)
    for m, F in enumerate(Fs):
        F = np.ascontiguousarray(F)
        for key in ("FDs", "FDsSym"):
            r = np.zeros(n)
            getattr(L, key)(_p(u), _p(F), _p(r), n)
            out["%s_%d" % (key, m)] = r
        for key in ("exFDs", "exFDsSym"):
            r = np.zeros(n); w = np.zeros(n)
            getattr(L, key)(_p(u), _p(F), _p(r), _p(w), n)
            out["%s_e_%d" % (key, m)] = r; out["%s_w_%d" % (key, m)] = w
    (q1, q2), (b1, b2), hs = h_resid_inputs()
    for m, h in enumerate(hs):
        for key in H_METRICS:
            out["%s_%d" % (key, m)] = h_rows(L, q1, q2, h, key)
        out["HDs_big_%d" % m] = h_rows(L, b1, b2, h, "HDs")
    p1, p2, w, lists = fit_inputs()
    u = np.ascontiguousarray(_u6(p1, p2))
    for k in FIT_F_LENGTHS:
        idx = lists[k]
        buf = np.zeros(18 * k + 81)
        F = np.zeros(9)
        L.u2f(_p(u), idx.ctypes.data_as(ip), k, _p(F), _p(buf))
        out["u2f_%d" % k] = F.copy()
        L.u2fw(_p(u), idx.ctypes.data_as(ip), _p(w), k, _p(F), _p(buf))
        out["u2fw_%d" % k] = F.copy()
    p1, p2, lists = fit_inputs_h()
    u = np.ascontiguousarray(_u6(p1, p2))
    for k in FIT_H_LENGTHS:
        buf = np.zeros(18 * k + 81)
        H = np.zeros(9)
        L.u2h(_p(u), lists[k].ctypes.data_as(ip), k, _p(H), _p(buf))
        out["u2h_%d" % k] = H.copy()
    L.SuperFastHash.argtypes = [ctypes.c_char_p, ctypes.c_int]
    L.SuperFastHash.restype = ctypes.c_uint32
    out["hash"] = np.array([L.SuperFastHash(ix.tobytes(), 4 * len(ix)) for ix in hash_inputs()], np.uint32)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_block_leaves_v1.npz"), **out)


if __name__ == "__main__":
    main()
