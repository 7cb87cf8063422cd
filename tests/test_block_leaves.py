"""The replay's block-wide passes on the device, one primitive at a time, against exact references, at every CTA width.

Every O(N) pass of the replay and every LO fit goes through the CTA-cooperative routines of block.h, ffit.h, hfit.h and
engine_h.h.  The host emulation runs them as a one-thread CTA, where the ballot, parked-word, packed-count and
two-chains-per-thread spellings are not compiled at all, and the whole-call parity tests name a pair, not a pass.  Here
the harness tests/devleaf/blockleaf.cu runs each routine on ONE CTA of nt threads (every multiple of 32 up to the pair kernel's 256)
over row lengths chosen at the switches between its code paths, and compares it with:
  - numpy / math.fsum restatements (inlier lists, MSAC scores, scans, sums, gate counts, the hash table),
  - the unmodified reference's own leaves on the same inputs (FDs*, exFDs*, HDs*, u2f, u2fw, u2h, SuperFastHash),
    stored in tests/golden/ref_block_leaves_v1.npz by tests/golden/make_block_leaves.py.
The shipped kernels are also run at CTA widths 128 and 160 (DGB200_THREADS) against the recorded reference answers.
The oracles themselves, and the one-thread host build of the compaction (blockhost.cpp), are checked without a GPU."""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from pydegensac_b200.scenes import scene_F, scene_H
from tests.conftest import norm_model
from tests.devleaf import blk
from tests.hostemu import emu

EPS = 2.0 ** -52
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "ref_block_leaves_v1.npz")
ALL_WIDTHS = tuple(range(32, 257, 32))
SWEEP_WIDTHS = (32, 128, 160, 256)
H_METRICS = ("HDs", "HDsSymMaxSq", "HDsSymMax", "HDsSymSumSq", "HDsSymSum")   # HMetric ids 0..4 (common.h)
RESID_CLASSIFY_MIN_N = 2048   # engine_h.h kResidClassifyMinN in the device build
HASH_LENGTHS = (0, 1, 2, 3, 31, 32, 33, 64, 65, 1500)
FIT_F_LENGTHS = (8, 9, 12, 14, 15, 100, 2000, 20000)
FIT_H_LENGTHS = (4, 5, 12, 32, 33, 100, 2000)


def _dev():
    blk.lib()       # a missing or unbuildable harness is a failure, not a skip
    return blk


def _fixture():
    return np.load(FIXTURE)


# ------------------------------------------------------------------------------------------------------------------
# seeded inputs (the fixture holds the reference's outputs on exactly these)
# ------------------------------------------------------------------------------------------------------------------
def f_resid_inputs():
    """1001 correspondences (odd: the last trip's second chain is empty) and three F models (row-major)."""
    rng = np.random.default_rng(1201)
    p1, p2, _ = scene_F(1001, 0.5, 21)
    A = np.array([[x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0]
                  for (x1, y1), (x2, y2) in zip(p1[:400], p2[:400])])
    F0 = np.linalg.svd(A)[2][-1]
    return p1, p2, np.stack([F0, F0 * (1 + 1e-3 * rng.normal(size=9)), rng.normal(size=9)])


def h_resid_inputs():
    """(p1, p2, models) of the five-metric rows (N = 301) and of the two-step Sampson row (N = 2049, th = 1: a third of
    the correspondences sit within 2^-20 of 9/4 th and 18 th)."""
    from tests.test_device_leaves import h_filter_scene
    rng = np.random.default_rng(1202)
    small = scene_H(301, 150, 22)
    hs = []
    big = h_filter_scene(rng, 2049, 1.0, 0.0, 1.0)
    for m in big[2][[0, 1, 21]]:
        hs.append(m / np.abs(m).max())
    return (small[0], small[1]), (big[0], big[1]), np.stack(hs)


def fit_inputs():
    """20000 correspondences (40 % inliers), positive weights, and the index lists of the fits."""
    rng = np.random.default_rng(1203)
    p1, p2, _ = scene_F(20000, 0.4, 23)
    w = rng.uniform(0.1, 2.0, 20000)
    lists = {n: rng.permutation(20000)[:n].astype(np.int32) for n in sorted(set(FIT_F_LENGTHS + FIT_H_LENGTHS))}
    return p1, p2, w, lists


def fit_inputs_h():
    p1, p2, _ = scene_H(3000, 2500, 24, noise=0.5)
    rng = np.random.default_rng(1204)
    return p1, p2, {n: rng.permutation(3000)[:n].astype(np.int32) for n in FIT_H_LENGTHS}


def hash_inputs():
    rng = np.random.default_rng(1205)
    return [np.sort(rng.choice(5000, n, replace=False)).astype(np.int32) for n in HASH_LENGTHS]


def _u6(p1, p2):
    u = np.ones((len(p1), 6))
    u[:, 0:2] = p1
    u[:, 3:5] = p2
    return u


# ------------------------------------------------------------------------------------------------------------------
# numpy oracles
# ------------------------------------------------------------------------------------------------------------------
def trunc_quad_terms(err, th):
    """The reference's truncQuad (rtools.c:228-236) per entry, in float64."""
    if th == 0:
        return np.zeros_like(err)
    wq = th * 9 / 4
    with np.errstate(invalid="ignore", over="ignore"):
        return np.where(err >= wq, 0.0, 1 - err / wq)


def msac_oracle(err, th):
    """(list, J, J error bound): the ordered inlier list, the exact sum of the reference's gains and the rounding bound
    of the device's J: each gain 1 - e * (1 / wq) is within 2 eps of 1 - e / wq, the block sum adds (N - 1) eps of the
    sum of magnitudes."""
    t = trunc_quad_terms(err, th)
    if np.isnan(t).any():
        return np.flatnonzero(err <= th), math.nan, 0.0
    J = math.fsum(t.tolist())
    return np.flatnonzero(err <= th), J, 2 * EPS * np.count_nonzero(t) + (err.size + 1) * EPS * abs(J) + 1e-300


def msac_row(rng, N, th):
    """A residual row with entries exactly at th and 9/4 th, one ulp either side of each, +-0, subnormals, +inf and
    ordinary values below and above both thresholds."""
    wq = th * 9 / 4
    special = np.array([th, np.nextafter(th, 0), np.nextafter(th, np.inf), wq, np.nextafter(wq, 0), np.nextafter(wq, np.inf),
                        0.0, -0.0, 5e-324, 2.5e-308, np.inf, 1e300])
    e = rng.uniform(0, 3 * th if th > 0 else 1.0, N)
    pick = rng.random(N) < 0.4
    e[pick] = special[rng.integers(special.size, size=int(pick.sum()))]
    return e


def row_lengths(nt, rng):
    nw = nt // 32
    Ns = {1, 7, 8, 9, 31, 32, 33, nt - 1, nt, nt + 1, 8 * nt - 1, 8 * nt, 8 * nt + 1, 1024 * nw - 32, 1024 * nw + 32,
          65535, 65536, 70000}
    Ns.update(int(v) for v in rng.integers(2, 12000, 3))
    return sorted(n for n in Ns if n > 0)


def randsubset_oracle(lst, siz, seed, k, j0):
    """The reference's randsubset (rtools.c:25-39) on the engine's Philox stream (draw t = value31(seed, k, j0 + t),
    itself pinned to the reference harness in tests/test_hostemu_vs_ref.py)."""
    lst = np.array(lst, np.int32)
    L = emu.lib()
    L.emu_value31.restype = ctypes.c_uint32
    for i in range(siz):
        s = L.emu_value31(ctypes.c_uint64(seed), ctypes.c_uint32(k), ctypes.c_uint32(j0 + i)) % (lst.size - i)
        j = lst.size - i - 1
        lst[s], lst[j] = lst[j], lst[s]
    return lst


def host_hash(lst):
    """superfasthash_i32 of la.h, host build (pinned to the reference's SuperFastHash by the fixture)."""
    L = emu.lib()
    L.emu_hash.restype = ctypes.c_uint32
    return int(L.emu_hash(lst.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), lst.size))


class HashTable:
    """The LO de-duplication table (DESIGN section 4): (hash, len, iterID) entries, at most `cap`; a new entry past the
    cap is dropped.  Verdict 1: same hash and length under this iterID, 2: under another one only, 0: inserted."""

    def __init__(self, cap):
        self.cap, self.rows = cap, []

    def verdict(self, h, n, iterID):
        hits = [r for r in self.rows if r[0] == h and r[1] == n]
        if any(r[2] == iterID for r in hits):
            return 1
        if hits:
            return 2
        if len(self.rows) < self.cap:
            self.rows.append((h, n, iterID))
        return 0


def fit_tolerance(p1, p2, idx, w, kind):
    """Tolerance of a fitted model after norm_model, from the eigen-gap of its normalised normal matrix: rounding of
    the matrix (about len eps of its largest eigenvalue) moves the eigenvector by that over the gap."""
    a, b = p1[idx], p2[idx]

    def hart(x):
        c = x.mean(0)
        s = len(x) * math.sqrt(2) / np.sqrt(((x - c) ** 2).sum(1)).sum()
        return (x - c) * s
    a, b = hart(a), hart(b)
    if kind == 0:
        Z = np.stack([a[:, 0] * b[:, 0], a[:, 1] * b[:, 0], b[:, 0], a[:, 0] * b[:, 1], a[:, 1] * b[:, 1], b[:, 1],
                      a[:, 0], a[:, 1], np.ones(len(a))], 1)
        if w is not None:
            Z = Z * w[idx][:, None]
    else:
        o, z = np.ones(len(a)), np.zeros(len(a))
        Z = np.concatenate([np.stack([b[:, 0], z, -a[:, 0] * b[:, 0], b[:, 1], z, -a[:, 0] * b[:, 1], o, z, -a[:, 0]], 1),
                            np.stack([z, b[:, 0], -a[:, 1] * b[:, 0], z, b[:, 1], -a[:, 1] * b[:, 1], z, o, -a[:, 1]], 1)])
    ev = np.linalg.eigvalsh(Z.T @ Z)
    return 1e-8 + 1e3 * len(idx) * EPS * ev[-1] / max(ev[1] - ev[0], 1e-300)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the oracles and the host-emulation build against the fixture
# ------------------------------------------------------------------------------------------------------------------
def test_msac_oracle_and_host_compaction():
    """The numpy oracle of the compaction agrees with the one-thread build of blk_inlidxs / blk_inlidxs2 (list, I, the
    rounding bound of J), and the two-threshold pass equals two calls bit for bit there too."""
    rng = np.random.default_rng(5)
    for th in (1.0, 0.37, 3e-300, 0.0):
        for N in (1, 9, 257, 5000):
            e = msac_row(rng, N, th)
            thB = 2.5 * th
            for two in (False, True):
                la, lb, J, I = blk.host_blk_inlidxs(e, th, thB, two)
                for lst, j, t in ((la, J[0], th), (lb, J[1], thB)):
                    ol, oJ, bound = msac_oracle(e, t)
                    assert np.array_equal(lst, ol)
                    assert abs(j - oJ) <= bound, (th, N, j, oJ)
                assert I[2] == np.count_nonzero(e < th)
            one, two_ = blk.host_blk_inlidxs(e, th, thB, False), blk.host_blk_inlidxs(e, th, thB, True)
            assert all(np.array_equal(x, y) for x, y in zip(one[:2], two_[:2])) and one[2].tobytes() == two_[2].tobytes()
    e = msac_row(rng, 100, 1.0)
    e[17] = np.nan
    assert math.isnan(blk.host_blk_inlidxs(e, 1.0, 2.0, True)[2][0]) and math.isnan(msac_oracle(e, 1.0)[1])


def test_fixture_rows_against_exact_and_host_build():
    """The reference's FDs / FDsSym / HDs rows in the fixture are within a few ulp of the exact (rational) residuals,
    and the host build of the engine's residuals reproduces every entry of every row bit for bit."""
    from tests.test_device_leaves import f_sampson_exact, h_sampson_exact
    z = _fixture()
    p1, p2, Fs = f_resid_inputs()
    L = emu.lib()
    L.emu_f_resid.restype = ctypes.c_double
    L.emu_h_resid.restype = ctypes.c_double
    cd = ctypes.c_double
    for m, F in enumerate(Fs):
        Fc = np.ascontiguousarray(F)
        for metric, key in ((0, "FDs"), (1, "FDsSym")):
            ref = z["%s_%d" % (key, m)]
            host = np.array([L.emu_f_resid(metric, emu._dp(Fc), cd(a), cd(b), cd(c), cd(d))
                             for (a, b), (c, d) in zip(p1, p2)])
            assert host.tobytes() == ref.tobytes(), (key, m)
            for i in range(0, len(p1), 97):
                ex = f_sampson_exact(metric, F, p1[i, 0], p1[i, 1], p2[i, 0], p2[i, 1])
                assert abs(ref[i] - float(ex)) <= 1e-9 * abs(float(ex)) + 1e-12   # (the algebraic error cancels)
    (q1, q2), (b1, b2), hs = h_resid_inputs()
    for m, h in enumerate(hs):
        hc = np.ascontiguousarray(h)
        for metric, key in enumerate(H_METRICS):
            ref = z["%s_%d" % (key, m)]
            host = np.array([L.emu_h_resid(metric, emu._dp(hc), cd(a), cd(b), cd(c), cd(d)) for (a, b), (c, d) in zip(q1, q2)])
            assert host.tobytes() == ref.tobytes(), (key, m)
        ref = z["HDs_big_%d" % m]
        for i in range(0, len(b1), 61):
            ex = h_sampson_exact(h, b1[i, 0], b1[i, 1], b2[i, 0], b2[i, 1])
            assert abs(ref[i] - float(ex)) <= 1e-9 * abs(float(ex)) + 1e-12


def test_hash_and_subset_oracles():
    z = _fixture()
    for lst, h in zip(hash_inputs(), z["hash"]):
        assert host_hash(lst) == int(h)
    t = HashTable(2)
    assert [t.verdict(1, 3, 0), t.verdict(1, 3, 0), t.verdict(1, 3, 1), t.verdict(2, 3, 1), t.verdict(3, 3, 1),
            t.verdict(3, 3, 1)] == [0, 1, 2, 0, 0, 0]
    s = randsubset_oracle(np.arange(20), 8, 7, 3, 0)
    assert sorted(s.tolist()) == list(range(20))


# ------------------------------------------------------------------------------------------------------------------
# GPU: the primitives on one CTA
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_compaction_sweep_all_paths():
    """blk_inlidxs (segment / ballot-parked / ballot-reread / one-warp paths), blk_inlidxs2 (packed path and its
    N >= 65536 guard) and blk_count_lt: list = flatnonzero(err <= th) element for element, I its length, J within the
    rounding bound of fsum of the reference's gains; the two-threshold pass bit-identical to two calls."""
    dev = _dev()
    rng = np.random.default_rng(11)
    for nt in SWEEP_WIDTHS:
        for N in row_lengths(nt, rng):
            th = float(rng.choice([1.0, 0.25, 7.5]))
            thB = th * 2.5
            e = msac_row(rng, N, th)
            one = dev.blk_inlidxs(e, th, thB, False, nt)
            two = dev.blk_inlidxs(e, th, thB, True, nt)
            what = "nt=%d N=%d" % (nt, N)
            for lst, J, t in ((one[0], one[2][0], th), (one[1], one[2][1], thB)):
                ol, oJ, bound = msac_oracle(e, t)
                assert np.array_equal(lst, ol), what
                assert abs(J - oJ) <= bound, (what, J, oJ)
            assert one[3][0] == one[0].size and one[3][1] == one[1].size, what
            assert one[3][2] == np.count_nonzero(e < th), what
            assert np.array_equal(one[0], two[0]) and np.array_equal(one[1], two[1]), what
            assert one[2].tobytes() == two[2].tobytes() and np.array_equal(one[3], two[3]), what


@pytest.mark.gpu
def test_compaction_edges_every_width():
    """th = 0, all-NaN-free rows of zeros / subnormals / inf, and a NaN entry (NaN J, as the reference's truncQuad)."""
    dev = _dev()
    rng = np.random.default_rng(12)
    for nt in ALL_WIDTHS:
        for N in (1, 33, nt + 1, 8 * nt + 1, 3000):
            for th in (0.0, 1e-300, 1.0):
                e = msac_row(rng, N, th)
                for two in (False, True):
                    la, lb, J, I = dev.blk_inlidxs(e, th, 2 * th, two, nt)
                    assert np.array_equal(la, np.flatnonzero(e <= th)) and np.array_equal(lb, np.flatnonzero(e <= 2 * th))
                    ol, oJ, bound = msac_oracle(e, th)
                    assert abs(J[0] - oJ) <= bound, (nt, N, th, two)
            e = msac_row(rng, N, 1.0)
            e[rng.integers(N)] = np.nan
            for two in (False, True):
                la, lb, J, I = dev.blk_inlidxs(e, 1.0, 2.0, two, nt)
                assert math.isnan(J[0]) and math.isnan(J[1]), (nt, N)
                assert np.array_equal(la, np.flatnonzero(e <= 1.0))


@pytest.mark.gpu
@pytest.mark.xfail(strict=True, reason="known fault, DESIGN section 5: 1 / (9/4 th) overflows for th < 2^-1022 * 4/9 and "
                   "the hoisted gain e * (1 / wq) is NaN or -inf where the reference's e / wq is finite")
def test_compaction_subnormal_threshold():
    dev = _dev()
    e = np.array([0.0, 5e-324, 1e-323, 1.0])
    _, _, J, _ = dev.blk_inlidxs(e, 5e-324, 5e-324, False, 32)
    assert abs(J[0] - msac_oracle(e, 5e-324)[1]) <= 1e-15


@pytest.mark.gpu
def test_reductions_every_width():
    """blk_sum / blk_scan_sum's J within the fsum bound, blk_sum_i / blk_excl_scan_i / blk_scan_sum's offsets exact,
    blk_sum_vec for k = 1..48 within the fsum bound, every thread sees the same totals, same bytes on a rerun."""
    dev = _dev()
    rng = np.random.default_rng(13)
    for nt in ALL_WIDTHS:
        vd = rng.normal(size=nt) * 10.0 ** rng.uniform(-8, 8, nt)
        vi = rng.integers(0, 1000, nt).astype(np.int32)
        vv = rng.normal(size=(nt, 48)) * 10.0 ** rng.uniform(-6, 6, (nt, 48))
        S = math.fsum(vd.tolist())
        bound = nt * EPS * np.abs(vd).sum()
        for k in (1, 2, 4, 9, 31, 32, 33, 45, 48):
            r = dev.blk_reduce(vd, vi, vv, k, nt)
            assert np.all(r["sum"] == r["sum"][0]) and abs(r["sum"][0] - S) <= bound, nt
            assert np.all(r["scan_sum_J"] == r["scan_sum_J"][0]) and abs(r["scan_sum_J"][0] - S) <= bound, nt
            assert np.all(r["sum_i"] == vi.sum())
            excl = np.concatenate([[0], np.cumsum(vi)[:-1]])
            assert np.array_equal(r["excl"], excl) and np.all(r["excl_total"] == vi.sum()), nt
            assert np.array_equal(r["scan_off"], excl) and np.all(r["scan_total"] == vi.sum()), nt
            for i in range(k):
                col = vv[:, i]
                assert abs(r["vec"][i] - math.fsum(col.tolist())) <= nt * EPS * np.abs(col).sum(), (nt, k, i)
            again = dev.blk_reduce(vd, vi, vv, k, nt)
            assert all(np.asarray(r[x]).tobytes() == np.asarray(again[x]).tobytes() for x in r), (nt, k)


@pytest.mark.gpu
def test_resid_F_rows_bit_equal_reference():
    """blk_resid_F / blk_resid_w_F, both metrics, bit-equal to the reference's FDs, FDsSym, exFDs, exFDsSym at odd and
    even N around nt and 2 nt (the two chains of a trip), at every width."""
    dev = _dev()
    z = _fixture()
    p1, p2, Fs = f_resid_inputs()
    for nt in ALL_WIDTHS:
        for N in sorted({1, 7, 31, 33, nt - 1, nt, nt + 1, 2 * nt - 1, 2 * nt + 1, 1001}):
            for m, F in enumerate(Fs):
                for metric, key, exkey in ((0, "FDs", "exFDs"), (1, "FDsSym", "exFDsSym")):
                    out, _ = dev.blk_resid_F(p1[:N], p2[:N], metric, F, False, nt)
                    assert out.tobytes() == z["%s_%d" % (key, m)][:N].tobytes(), (nt, N, key, m)
                    out, w = dev.blk_resid_F(p1[:N], p2[:N], metric, F, True, nt)
                    assert out.tobytes() == z["%s_e_%d" % (exkey, m)][:N].tobytes(), (nt, N, exkey, m)
                    assert w.tobytes() == z["%s_w_%d" % (exkey, m)][:N].tobytes(), (nt, N, exkey, m)


@pytest.mark.gpu
def test_resid_H_rows_bit_equal_reference():
    """blk_resid_H, all five metrics, bit-equal to HDs, HDsSymMaxSq, HDsSymMax, HDsSymSumSq, HDsSymSum."""
    dev = _dev()
    z = _fixture()
    (q1, q2), _, hs = h_resid_inputs()
    for nt in ALL_WIDTHS:
        for N in sorted({1, 4, 33, nt - 1, nt + 1, 301}):
            for m, h in enumerate(hs):
                for metric, key in enumerate(H_METRICS):
                    out = dev.blk_resid_H(q1[:N], q2[:N], metric, 1.0, h, False, nt)
                    assert out.tobytes() == z["%s_%d" % (key, m)][:N].tobytes(), (nt, N, key, m)


@pytest.mark.gpu
def test_resid_H_two_step_sampson_row():
    """The two-step Sampson row (FP32 classification, then exact HDs on the near rows), N on both sides of the device's
    kResidClassifyMinN = 2048 and odd N (the padding slot of the pair-interleaved tile): every entry that is not +inf
    equals HDs bit for bit, every +inf entry has HDs >= 18 th (all of them are checked), and below the switch no entry
    is +inf."""
    dev = _dev()
    z = _fixture()
    _, (b1, b2), hs = h_resid_inputs()
    th = 1.0
    far_seen = 0
    for nt in SWEEP_WIDTHS + (64, 224):
        for N in (RESID_CLASSIFY_MIN_N - 1, RESID_CLASSIFY_MIN_N, RESID_CLASSIFY_MIN_N + 1):
            for m, h in enumerate(hs):
                ref = z["HDs_big_%d" % m][:N]
                out = dev.blk_resid_H(b1[:N], b2[:N], 0, th, h, True, nt)
                inf = np.isposinf(out)
                what = (nt, N, m)
                assert out[~inf].tobytes() == ref[~inf].tobytes(), what
                assert np.all(ref[inf] >= 18 * th), (what, ref[inf].min())
                if N < RESID_CLASSIFY_MIN_N:
                    assert not inf.any(), what
                far_seen += int(inf.sum())
    assert far_seen > 0


@pytest.mark.gpu
def test_gate_counts_match_recount():
    """blk_sym_count_F / blk_laf_count_F / blk_sym_count_H against a recount of the reference's own rows over the same
    list (the helper correspondences are other correspondences of the scene, so their rows are known too)."""
    dev = _dev()
    z = _fixture()
    p1, p2, Fs = f_resid_inputs()
    (q1, q2), _, hs = h_resid_inputs()
    rng = np.random.default_rng(14)
    N = 301
    p1, p2 = p1[:N], p2[:N]
    # H rows of q1/q2 (N = 301); F rows of p1/p2; the counts run over the same list on both point sets
    perm1, perm2 = rng.permutation(N), rng.permutation(N)
    fds = z["FDs_0"][:N]
    laf = np.stack([p1[perm1, 0], p1[perm1, 1], p2[perm1, 0], p2[perm1, 1],
                    p1[perm2, 0], p1[perm2, 1], p2[perm2, 0], p2[perm2, 1]], 1)
    symF = z["FDsSym_0"][:N]
    for nt in ALL_WIDTHS:
        for n in (0, 1, 31, 33, nt + 1, N):
            lst = np.sort(rng.choice(N, n, replace=False)).astype(np.int32)
            sym_th = float(np.median(symF))
            th_laf = float(np.median(fds))
            out = dev.blk_counts(p1, p2, laf, lst, Fs[0], hs[0], 0, 0, sym_th, th_laf, nt)
            assert out[0] == np.count_nonzero(symF[lst] <= sym_th), (nt, n)
            assert out[1] == min(np.count_nonzero(fds[perm1[lst]] <= th_laf), np.count_nonzero(fds[perm2[lst]] <= th_laf))
            hsym = z["HDsSymMax_0"][:N]
            hth = float(np.median(hsym))
            out = dev.blk_counts(q1, q2, laf, lst, Fs[0], hs[0], 0, 0, hth, th_laf, nt)
            assert out[2] == np.count_nonzero(hsym[lst] <= hth), (nt, n)


def _close_models(a, b, tol):
    return np.linalg.norm(norm_model(a) - norm_model(b)) <= tol


@pytest.mark.gpu
def test_fit_F_regimes_against_u2f_u2fw():
    """blk_fit_F in each regime (len <= 8: warp Householder / Gauss-Jordan; 9..14: warp_fit_F_small; 15+: block
    moments) against the reference's u2f and u2fw (with its stride-9 weight quirk at len 8), within a tolerance set by
    the eigen-gap of the normal matrix."""
    dev = _dev()
    z = _fixture()
    p1, p2, w, lists = fit_inputs()
    for nt in SWEEP_WIDTHS:
        for n in FIT_F_LENGTHS:
            idx = lists[n]
            for ww, key in ((None, "u2f"), (w, "u2fw")):
                F = dev.blk_fit(p1, p2, idx, ww, 0, nt)
                tol = fit_tolerance(p1, p2, idx, ww, 0) if n > 8 else 1e-8
                assert _close_models(F, z["%s_%d" % (key, n)], tol), (nt, n, key)


@pytest.mark.gpu
def test_fit_H_against_u2h():
    dev = _dev()
    z = _fixture()
    p1, p2, lists = fit_inputs_h()
    for nt in SWEEP_WIDTHS:
        for n in FIT_H_LENGTHS:
            h = dev.blk_fit(p1, p2, lists[n], None, 1, nt)
            tol = fit_tolerance(p1, p2, lists[n], None, 1) if n > 4 else 1e-8
            assert _close_models(h, z["u2h_%d" % n], tol), (nt, n)


@pytest.mark.gpu
def test_sample8_fused_equals_subset_then_fit():
    """blk_sample8_fit_F = blk_randsubset + blk_fit_F(len 8): the permuted list bit-equal to the reference's randsubset
    on the engine's stream, the cursor advanced by 8, F within tolerance; degenerate subsets (all eight the same point,
    or collinear points in both images) go down the fast = false route."""
    dev = _dev()
    p1, p2, w, _ = fit_inputs()
    rng = np.random.default_rng(15)
    for nt in SWEEP_WIDTHS:
        for trial in range(6):
            max_sz = int(rng.choice([8, 9, 40, 2000]))
            lst = rng.permutation(20000)[:max_sz].astype(np.int32)
            seed, k, j0 = int(rng.integers(1 << 40)), int(rng.integers(1 << 20)), int(rng.integers(1000))
            ww = w if trial % 2 else None
            lf, Ff, jf, fast = dev.blk_sample8(p1, p2, lst, ww, seed, k, j0, True, nt)
            ls, Fs, js, _ = dev.blk_sample8(p1, p2, lst, ww, seed, k, j0, False, nt)
            assert np.array_equal(lf, randsubset_oracle(lst, 8, seed, k, j0)), (nt, trial)
            assert np.array_equal(lf, ls) and jf == js == j0 + 8, (nt, trial)
            assert fast == 1 and _close_models(Ff, Fs, 1e-7), (nt, trial)
        # degenerate 8-subsets: one point repeated (rank 1, but rounding leaves non-zero pivots, so either route may
        # run), and image-1 points on the line x = 0, whose coefficient rows have exactly zero columns: no pivot is
        # left after the live columns, warp_sample8_fit gives up (fast = false) and the Householder route runs.
        q1 = np.tile(p1[:1], (20, 1)); q2 = np.tile(p2[:1], (20, 1))
        t = np.linspace(0, 1, 20)[:, None]
        c1 = np.concatenate([0 * t, 200 + 30 * t], 1); c2 = p2[:20]
        for case, (a, b) in enumerate(((q1, q2), (c1, c2))):
            lst = np.arange(20, dtype=np.int32)
            lf, Ff, jf, fast = dev.blk_sample8(a, b, lst, None, 3, 4, 5, True, nt)
            ls, Fs, js, _ = dev.blk_sample8(a, b, lst, None, 3, 4, 5, False, nt)
            assert np.array_equal(lf, ls) and jf == js == 13, (nt, case)
            if case == 1:
                assert fast == 0 and Ff.tobytes() == Fs.tobytes(), (nt, fast)


@pytest.mark.gpu
def test_hash_verdicts_against_table_model():
    """warp_hash_verdict / hash_seen_elsewhere: the inserted hash bit-equal to the reference's SuperFastHash at every
    length, and the verdicts equal the table model up to and past the 2048-entry cap."""
    dev = _dev()
    z = _fixture()
    cap = 2048
    for nt in SWEEP_WIDTHS:
        table = dict(hash=np.zeros(cap, np.uint32), len=np.zeros(cap, np.int32), id=np.zeros(cap, np.int32), n=0)
        model = HashTable(cap)
        for lst, h in zip(hash_inputs(), z["hash"]):
            v, ab = dev.blk_hash(lst, 1, table, nt)
            assert v == model.verdict(int(h), lst.size, 1) == 0 and not ab
            assert table["hash"][table["n"] - 1] == h and table["len"][table["n"] - 1] == lst.size, (nt, lst.size)
            assert dev.blk_hash(lst, 1, table, nt) == (model.verdict(int(h), lst.size, 1), False) == (1, False)
            assert dev.blk_hash(lst, 2, table, nt) == (2, True) and model.verdict(int(h), lst.size, 2) == 2
        # fill to the cap from the host with distinct (hash, len) pairs, then insert past it
        rng = np.random.default_rng(16)
        n0 = table["n"]
        fill = rng.integers(1, 1 << 32, cap - n0, dtype=np.uint64).astype(np.uint32)
        table["hash"][n0:] = fill; table["len"][n0:] = 999999; table["id"][n0:] = 5; table["n"] = cap
        for hv in fill:
            model.rows.append((int(hv), 999999, 5))
        extra = np.arange(7, dtype=np.int32)
        v, _ = dev.blk_hash(extra, 1, table, nt)
        hx = host_hash(extra)
        assert v == model.verdict(hx, 7, 1) == 0 and table["n"] == cap and len(model.rows) == cap
        v, _ = dev.blk_hash(extra, 1, table, nt)
        assert v == model.verdict(hx, 7, 1) == 0      # dropped, so not found again


# ------------------------------------------------------------------------------------------------------------------
# GPU: the shipped kernels at other CTA widths
# ------------------------------------------------------------------------------------------------------------------
PARITY_TESTS = ("test_F_configs_vs_reference or test_H_configs_vs_reference or "
                "test_randomised_small_configs_vs_reference or test_batch_of_distinct_pairs_vs_reference")


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [128, 160])
def test_shipped_kernels_at_cta_width(threads):
    """The F and H entry points launched with CTA width `threads` (DGB200_THREADS, read once per process, hence the
    subprocess) reproduce the recorded reference answers of the parity tests under their own rule (_cmp: same mask,
    model within 1e-6, same sample and LO counts).  The default width 256 is the parity tests themselves."""
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                        os.path.join("tests", "test_gpu_parity.py"), "-k", PARITY_TESTS],
                       cwd=ROOT, capture_output=True, text=True, timeout=1500,
                       env=dict(os.environ, DGB200_THREADS=str(threads)))
    assert r.returncode == 0 and "4 passed" in r.stdout, r.stdout[-4000:] + r.stderr[-2000:]
