"""Device-only leaves of the engine, one at a time, against exact references.

The host emulation (tests/hostemu) compiles only the code both passes share, and the whole-call parity tests reach the
device-only branches on a few scenes.  Here the harness tests/devleaf runs each device-only leaf as the pair kernel runs
it -- the 9x9 eigen-solver flavours, the wave's 7x9 pair elimination, the 32-lane null vectors, the rsqrt / bit-level 3x3
arithmetic, and the FP32 score bounds on the pair-interleaved tile -- and compares it with a plain high-precision
reference of the same operation (fractions.Fraction / mpmath on the exact float64 inputs).  The oracles themselves are
checked without a GPU."""
import ctypes
import math
import os
from fractions import Fraction

import mpmath
import numpy as np
import pytest

from pydegensac_b200.scenes import scene_F, scene_H
from tests.hostemu import emu

EPS = 2.0 ** -52


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def _dev():
    from tests.devleaf import dev
    dev.lib()       # a missing or unbuildable harness is a failure, not a skip
    return dev


# ------------------------------------------------------------------------------------------------------------------
# exact oracles
# ------------------------------------------------------------------------------------------------------------------
def mp_eigh(A, dps=40):
    """Eigenvalues (ascending, float) and unit eigenvectors (columns, float) of the exact symmetric float64 matrix A."""
    with mpmath.workdps(dps):
        E, Q = mpmath.eigsy(mpmath.matrix(np.asarray(A, dtype=np.float64).tolist()))
        order = sorted(range(9), key=lambda i: E[i])
        return (np.array([float(E[i]) for i in order]),
                np.array([[float(Q[r, i]) for i in order] for r in range(9)]))


def mp_rayleigh_excess(A, x, lam_min, dps=40):
    """x^T A x / x^T x - lambda_min, evaluated in high precision on the exact float64 values."""
    with mpmath.workdps(dps):
        xs = [mpmath.mpf(float(v)) for v in x]
        num = mpmath.fsum(xs[i] * mpmath.mpf(float(A[i, j])) * xs[j] for i in range(9) for j in range(9))
        return float(num / mpmath.fsum(v * v for v in xs) - mpmath.mpf(lam_min))


def fraction_null_vector(Zt):
    """The exact null vector (rational Gauss-Jordan) of the k x 9 float64 system Zt of rank 8, unit-normalised in float64;
    None when the exact rank is below 8."""
    rows = [[Fraction(float(v)) for v in r] for r in Zt]
    piv_cols, r = [], 0
    for col in range(9):
        p = next((i for i in range(r, len(rows)) if rows[i][col] != 0), None)
        if p is None:
            continue
        rows[r], rows[p] = rows[p], rows[r]
        inv = 1 / rows[r][col]
        rows[r] = [v * inv for v in rows[r]]
        for i in range(len(rows)):
            if i != r and rows[i][col] != 0:
                f = rows[i][col]
                rows[i] = [a - f * b for a, b in zip(rows[i], rows[r])]
        piv_cols.append(col)
        r += 1
    if r != 8:
        return None
    free = next(c for c in range(9) if c not in piv_cols)
    n = [Fraction(0)] * 9
    n[free] = Fraction(1)
    for i, c in enumerate(piv_cols):
        n[c] = -rows[i][free]
    big = max(abs(v) for v in n)
    with mpmath.workdps(40):
        v = [mpmath.mpf(x.numerator) / mpmath.mpf(x.denominator) / (mpmath.mpf(big.numerator) / big.denominator) for x in n]
        nrm = mpmath.sqrt(mpmath.fsum(t * t for t in v))
        return np.array([float(t / nrm) for t in v])


def sin_angle(q, n):
    q = q / np.linalg.norm(q)
    return float(np.linalg.norm(q - np.dot(q, n) * n))


def f_sampson_exact(metric, F, x1, y1, x2, y2):
    F = [Fraction(float(v)) for v in F]
    x1, y1, x2, y2 = (Fraction(float(v)) for v in (x1, y1, x2, y2))
    rxc = F[0] * x2 + F[3] * y2 + F[6]
    ryc = F[1] * x2 + F[4] * y2 + F[7]
    rwc = F[2] * x2 + F[5] * y2 + F[8]
    r = x1 * rxc + y1 * ryc + rwc
    rx = F[0] * x1 + F[1] * y1 + F[2]
    ry = F[3] * x1 + F[4] * y1 + F[5]
    a, b = rxc * rxc + ryc * ryc, rx * rx + ry * ry
    if metric == 1:
        return r * r * (a + b) / (a * b) if a * b != 0 else None
    return r * r / (a + b) if a + b != 0 else None


def h_sampson_exact(h, x1, y1, x2, y2):
    """r^T (J J^T)^-1 r of the reference's HDs, exact (h column-major, image 2 -> image 1)."""
    h = [Fraction(float(v)) for v in h]
    x1, y1, x2, y2 = (Fraction(float(v)) for v in (x1, y1, x2, y2))
    wz = h[2] * x2 + h[5] * y2 + h[8]
    r1 = h[0] * x2 + h[3] * y2 + h[6] - x1 * wz
    r2 = h[1] * x2 + h[4] * y2 + h[7] - y1 * wz
    a, b, c = h[0] - h[2] * x1, h[3] - h[5] * x1, -wz
    d, e = h[1] - h[2] * y1, h[4] - h[5] * y1
    A, D, B = a * a + b * b + c * c, d * d + e * e + c * c, a * d + b * e
    det = A * D - B * B
    if det == 0:
        return None
    return (D * r1 * r1 - 2 * B * r1 * r2 + A * r2 * r2) / det


def f_sampson64(metric, F, x1, y1, x2, y2):
    """[m, n] residuals of the F models [m, 9] in float64 (the reference's operation order, as f_resid)."""
    F = F[:, :, None]
    rxc = F[:, 0] * x2 + F[:, 3] * y2 + F[:, 6]
    ryc = F[:, 1] * x2 + F[:, 4] * y2 + F[:, 7]
    rwc = F[:, 2] * x2 + F[:, 5] * y2 + F[:, 8]
    r = x1 * rxc + y1 * ryc + rwc
    rx = F[:, 0] * x1 + F[:, 1] * y1 + F[:, 2]
    ry = F[:, 3] * x1 + F[:, 4] * y1 + F[:, 5]
    a, b = rxc * rxc + ryc * ryc, rx * rx + ry * ry
    with np.errstate(all="ignore"):
        return r * r * (a + b) / (a * b) if metric == 1 else r * r / (a + b)


def h_sampson64(h, x1, y1, x2, y2):
    h = h[:, :, None]
    wz = h[:, 2] * x2 + h[:, 5] * y2 + h[:, 8]
    r1 = h[:, 0] * x2 + h[:, 3] * y2 + h[:, 6] - x1 * wz
    r2 = h[:, 1] * x2 + h[:, 4] * y2 + h[:, 7] - y1 * wz
    a, b, c = h[:, 0] - h[:, 2] * x1, h[:, 3] - h[:, 5] * x1, -wz
    d, e = h[:, 1] - h[:, 2] * y1, h[:, 4] - h[:, 5] * y1
    A, D, B = a * a + b * b + c * c, d * d + e * e + c * c, a * d + b * e
    with np.errstate(all="ignore"):
        return (D * r1 * r1 - 2 * B * r1 * r2 + A * r2 * r2) / (A * D - B * B)


# ------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------
def orthogonal(rng, first=None):
    M = rng.normal(size=(9, 9))
    if first is not None:
        M[:, 0] = first
    Q, R = np.linalg.qr(M)
    return Q * np.sign(np.diag(R))[None, :]


SPECTRUM_RATIOS = (1e-12, 1e-3, 0.5, 0.9, 0.999, 1 - 1e-9)


def spectrum_cases(seed=5):
    """(name, A, intended eigenvalues ascending) with set spectra: lambda_1 / lambda_2 from SPECTRUM_RATIOS, rank 8,
    rank 7, overall scales 1e-12 .. 1e12; and start-vector cases whose v_min has a (nearly) vanishing last component,
    so that the solver's start vector L^-T e_8 = A^-1 e_8 / |.| (nearly) misses it."""
    rng = np.random.default_rng(seed)
    out = []
    for scale in (1e-12, 1.0, 1e12):
        for ratio in SPECTRUM_RATIOS + (0.0, "rank7"):
            lam2 = 10 ** rng.uniform(-4, -1)
            tail = np.sort(10 ** rng.uniform(np.log10(lam2) + 0.3, 0, 7))
            lam = np.concatenate([[0.0 if ratio == "rank7" else ratio * lam2, 0.0 if ratio == "rank7" else lam2], tail])
            for start in ("random", "orthogonal", "nearly"):
                v = rng.normal(size=9)
                if start != "random":
                    v[8] = 0.0 if start == "orthogonal" else 1e-8 * np.linalg.norm(v)
                Q = orthogonal(rng, v)
                A = (Q * lam[None, :]) @ Q.T
                A = (A + A.T) / 2 * scale
                out.append(("scale=%g ratio=%s start=%s" % (scale, ratio, start), A, lam * scale))
    # entries spanning 12 orders of magnitude (as the normal matrix of un-normalised pixel coordinates)
    for ratio in SPECTRUM_RATIOS:
        lam = np.concatenate([[ratio * 1e-3, 1e-3], np.sort(10 ** rng.uniform(-2, 0, 7))])
        Q = orthogonal(rng)
        Dg = 10.0 ** np.linspace(-3, 3, 9)
        A = Dg[:, None] * ((Q * lam[None, :]) @ Q.T) * Dg[None, :]
        out.append(("graded ratio=%g" % ratio, (A + A.T) / 2, None))
    return out


def dumped_normal_matrices(tmp_path, limit=60):
    """The 9x9 matrices the LO / DEGENSAC / large fits hand to the eigen-solver on seeded benchmark scenes, dumped by the
    host emulation (DG_EIG_DUMP)."""
    path = str(tmp_path / "eig_dump.bin")
    old = os.environ.get("DG_EIG_DUMP")
    os.environ["DG_EIG_DUMP"] = path
    try:
        for s, plane in ((0, 0.0), (1, 0.8)):
            p1, p2, _ = scene_F(800, 0.4, 60 + s, plane)
            emu.find_fundamental(p1, p2, 1.0, 0.999, 1500, seed=s)
        q1, q2, _ = scene_H(800, 300, 61)
        emu.find_homography_raw(q1, q2, 3.0, 0.999, 1500, seed=2)
    finally:
        if old is None:
            del os.environ["DG_EIG_DUMP"]
        else:
            os.environ["DG_EIG_DUMP"] = old
    A = np.fromfile(path, dtype=np.float64).reshape(-1, 9, 9)
    idx = np.random.default_rng(0).permutation(len(A))[:limit]
    return A[np.sort(idx)]


# ------------------------------------------------------------------------------------------------------------------
# oracle self-tests (no GPU)
# ------------------------------------------------------------------------------------------------------------------
def test_fraction_null_vector_matches_numpy_svd():
    rng = np.random.default_rng(1)
    for t in range(20):
        Zt = rng.normal(size=(8, 9)) * 10 ** rng.uniform(-3, 3, 9)[None, :]
        n = fraction_null_vector(Zt)
        v = np.linalg.svd(Zt)[2][-1]
        s = np.linalg.svd(Zt, compute_uv=False)
        assert sin_angle(v, n) < 1e3 * EPS * s[0] / s[-1]
        assert np.linalg.norm(Zt @ n) <= 1e-14 * np.linalg.norm(Zt)
    Zt[3] = Zt[5]
    assert fraction_null_vector(Zt) is None


def test_constructed_spectra_have_the_intended_gaps():
    for name, A, lam in spectrum_cases():
        E, Q = mp_eigh(A)
        nrm = np.abs(E).max()
        assert np.abs(Q.T @ Q - np.eye(9)).max() < 1e-13, name
        if lam is not None:
            assert np.abs(E - lam).max() <= 64 * EPS * nrm, name
            if "start=orthogonal" in name and E[0] > 1e-6 * nrm and E[1] - E[0] > 1e-6 * nrm:
                # (v_min well defined) the start vector's component along v_min is at rounding level
                y = np.linalg.solve(A, np.eye(9)[8])
                assert abs(np.dot(y / np.linalg.norm(y), Q[:, 0])) < 1e-6, name


def test_exact_residual_oracles_agree_with_float64():
    rng = np.random.default_rng(2)
    F = rng.normal(size=(3, 9)); h = rng.normal(size=(3, 9)) * [1, 1, 1e-3, 1, 1, 1e-3, 100, 100, 1]
    pts = rng.uniform(-300, 300, size=(4, 50))
    for metric in (0, 1):
        e64 = f_sampson64(metric, F, *pts)
        for m in range(3):
            for i in range(0, 50, 7):
                ex = f_sampson_exact(metric, F[m], *pts[:, i])
                assert abs(float(ex) - e64[m, i]) <= 1e-12 * abs(float(ex)) + 1e-300
    e64 = h_sampson64(h, *pts)
    for m in range(3):
        for i in range(0, 50, 7):
            assert abs(float(h_sampson_exact(h[m], *pts[:, i])) - e64[m, i]) <= 1e-10 * abs(e64[m, i])
    # the host spelling of the reference residuals (hostemu's f_resid / h_resid) is what the float64 oracle restates
    E = emu.lib()
    E.emu_f_resid.restype = ctypes.c_double
    E.emu_h_resid.restype = ctypes.c_double
    Fi = np.ascontiguousarray(F[0]); hi = np.ascontiguousarray(h[0])
    for i in range(10):
        args = [ctypes.c_double(v) for v in pts[:, i]]
        assert E.emu_f_resid(0, _dp(Fi), *args) == pytest.approx(f_sampson64(0, F[:1], *pts[:, i:i + 1])[0, 0], rel=1e-12)
        assert E.emu_h_resid(0, _dp(hi), *args) == pytest.approx(h_sampson64(h[:1], *pts[:, i:i + 1])[0, 0], rel=1e-9)


# ------------------------------------------------------------------------------------------------------------------
# 1. the 9x9 smallest-eigenvector solver
# ------------------------------------------------------------------------------------------------------------------
C_EIG = 128


def eigvec_error(A, x, E, Q):
    """None when x is a unit eigenvector of the smallest eigenvalue: Rayleigh quotient lambda_min to c eps |A|_F, and
    along v_min to c eps |A|_F / gap where the gap allows it (|A|_F: the scale of the solvers' own tests)."""
    nrm = float(np.sqrt(np.sum(E ** 2)))
    if not (np.all(np.isfinite(x)) and abs(np.linalg.norm(x) - 1.0) < 1e-13):
        return "not a unit vector: %s" % x
    excess = mp_rayleigh_excess(A, x, E[0])
    if not excess <= C_EIG * EPS * nrm:
        return "x^T A x - lambda_min = %.3g |A| (lambda_2 - lambda_1 = %.3g |A|): not the smallest eigenvector" % (
            excess / nrm, (E[1] - E[0]) / nrm)
    gap = E[1] - E[0]
    if gap >= 1e-6 * nrm and not 1.0 - abs(np.dot(x, Q[:, 0])) <= C_EIG * EPS * nrm / gap:
        return "|x . v_min| = %.17g" % abs(np.dot(x, Q[:, 0]))
    return None


@pytest.mark.gpu
def test_smallest_eigvec9_flavours_against_mpmath(tmp_path):
    """Every flavour, called directly and through the dispatch, on benchmark normal matrices and on set spectra.  A flavour
    may decline (false, ws->A intact: the caller moves on); what it returns must be the smallest eigenvector."""
    dev = _dev()
    cases = [("dump %d" % i, A, None) for i, A in enumerate(dumped_normal_matrices(tmp_path))] + spectrum_cases()
    A = np.stack([c[1] for c in cases])
    truth = [mp_eigh(a) for a in A]
    errors, declined = [], {}
    for mode, label in ((dev.EIG_DISPATCH, "dispatch"), (dev.EIG_INV, "inv"), (dev.EIG_REG, "reg"),
                        (dev.EIG_JACOBI, "jacobi")):
        x, Aout, Vout, ok = dev.eig9(A, mode)
        for i, (name, _, _) in enumerate(cases):
            if mode == dev.EIG_JACOBI:        # the dispatch's last resort: argmin of the diagonal, that column of V
                x[i] = Vout[i][:, int(np.argmin(np.diag(Aout[i])))]
            elif not ok[i]:                   # declined: the caller's matrix must be intact for the next flavour
                if not np.array_equal(Aout[i], A[i]):
                    errors.append("%s [%s]: declined but changed ws->A" % (name, label))
                kind = "dump" if name.startswith("dump") else name.split("start=")[-1] if "start=" in name else "graded"
                declined.setdefault(label, {}).setdefault(kind, []).append(name)
                continue
            err = eigvec_error(A[i], x[i], *truth[i])
            if err:
                errors.append("%s [%s]: %s" % (name, label, err))
    print("eigen-solver: %d matrices, declined: %s" % (len(cases), {k: sum(map(len, v.values())) for k, v in declined.items()}))
    assert not errors, "%d wrong results:\n%s" % (len(errors), "\n".join(errors[:20]))
    # the fast flavour itself must not give up where its shifts are meant to work: on the benchmark's matrices (DESIGN.md:
    # no fallback), on a well-separated lambda_min (lambda_1 / lambda_2 <= 1e-3) from any start vector, and on a moderate
    # gap (0.5) from a generic one
    must = lambda n: n.startswith("dump") or "ratio=1e-12 " in n or "ratio=0.001 " in n or "ratio=0.5 start=random" in n  # noqa: E731
    gave_up = [n for names in declined.get("inv", {}).values() for n in names if must(n)]
    assert not gave_up, gave_up


@pytest.mark.gpu
def test_smallest_eigvec9_non_finite_input_returns():
    """NaN / inf entries: every flavour must return (its loops are bounded), the two inverse-iteration flavours must
    decline and leave ws->A as it was."""
    dev = _dev()
    rng = np.random.default_rng(9)
    base = orthogonal(rng) @ np.diag(np.linspace(0.1, 1, 9)) @ orthogonal(rng).T
    mats = []
    for v in (np.nan, np.inf, -np.inf, 1e308):
        M = (base + base.T) / 2
        M[2, 5] = M[5, 2] = v
        mats.append(M)
        M = M.copy()
        M[8, 8] = v
        mats.append(M)
    A = np.stack(mats)
    for mode in (dev.EIG_INV, dev.EIG_REG):
        x, Aout, _, ok = dev.eig9(A, mode)
        assert not ok[:6].any(), mode
        assert np.array_equal(Aout, A, equal_nan=True), mode
    for mode in (dev.EIG_DISPATCH, dev.EIG_JACOBI):
        dev.eig9(A, mode)


# ------------------------------------------------------------------------------------------------------------------
# 2. the wave's 7x9 pair elimination
# ------------------------------------------------------------------------------------------------------------------
def _sample_rows(p1, p2, seed, kbeg, kend):
    E = emu.lib()
    N = p1.shape[0]
    sel = np.zeros(7, dtype=np.int32)
    M = np.zeros((kend - kbeg + 1, 81))
    for k in range(kbeg, kend + 1):
        E.emu_minimal_sample(ctypes.c_uint64(seed), ctypes.c_uint32(k), N, 7, sel.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
        for r, p in enumerate(sel):
            x1, y1, x2, y2 = p1[p, 0], p1[p, 1], p2[p, 0], p2[p, 1]
            M[k - kbeg, 9 * r:9 * r + 9] = (x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0)
    return M


def pairsolve_scenes():
    """(name, p1, p2): benchmark-like scenes at scale 1 and with 1e3 offsets; scenes with duplicated, collinear and
    nearly duplicated correspondences, so that both outcomes of the pivot test occur (and pivots straddle 1e-12)."""
    out = []
    for s in range(2):
        p1, p2, _ = scene_F(300, 0.5, 70 + s)
        out.append(("scene %d" % s, p1, p2))
        out.append(("scene %d offset 1e3" % s, p1 + 1e3, p2 - 1e3))
        out.append(("scene %d normalised" % s, (p1 - 320) / 400, (p2 - 240) / 400))
    rng = np.random.default_rng(3)
    p1, p2, _ = scene_F(12, 1.0, 80)
    d1, d2 = p1.copy(), p2.copy()
    d1[8:], d2[8:] = d1[0], d2[0]                 # four copies of one correspondence
    out.append(("duplicates", d1, d2))
    c1, c2 = p1.copy(), p2.copy()
    t = rng.uniform(0, 1, 12)
    c1[:7] = np.stack([100 + 300 * t[:7], 50 + 200 * t[:7]], 1)   # seven correspondences on a line in both images
    c2[:7] = np.stack([80 + 250 * t[:7], 400 - 100 * t[:7]], 1)
    out.append(("collinear", c1, c2))
    n1, n2 = scene_F(8, 1.0, 81)[:2]
    for e in range(-16, -5):
        a1, a2 = n1.copy(), n2.copy()
        a1[7] = a1[0] + 10.0 ** e * rng.normal(size=2) * 300
        a2[7] = a2[0] + 10.0 ** e * rng.normal(size=2) * 300
        out.append(("near duplicate 1e%d" % e, (a1 - 320) / 400, (a2 - 240) / 400))
    return out


@pytest.mark.gpu
def test_wave_pairsolve_is_nullspace9_bit_for_bit():
    dev = _dev()
    E = emu.lib()
    counts = [0, 0]
    for name, p1, p2 in pairsolve_scenes():
        seed, kbeg = 17, 1
        kend = 700 if p1.shape[0] > 20 else 120
        ns = dev.pairsolve(p1, p2, seed, kbeg, kend)
        M = _sample_rows(p1, p2, seed, kbeg, kend)
        dns, dnf = dev.nullspace9(M)
        for j in range(M.shape[0]):
            m = M[j].copy()
            ref = np.zeros(81)
            nf = E.emu_nullspace9(_dp(m), _dp(ref))
            # the one-thread device routine (the wave's fallback) is the host one bit for bit
            assert dnf[j] == nf and np.array_equal(dns[j, :9 * min(nf, 2)].view(np.uint64),
                                                   ref[:9 * min(nf, 2)].view(np.uint64)), "%s k=%d" % (name, kbeg + j)
            declines = not (nf == 2 and ref[7] == 1.0 and ref[8] == 0.0 and ref[16] == 0.0 and ref[17] == 1.0)
            generic = ns[j, 14]
            assert generic in (0.0, 1.0)
            assert (generic == 0.0) == declines, "%s k=%d: generic=%d, nullspace9 declines=%s" % (
                name, kbeg + j, generic, declines)
            counts[int(generic)] += 1
            if generic:
                got = np.concatenate([ns[j, 0:7], ns[j, 7:14]])
                want = np.concatenate([ref[0:7], ref[9:16]])
                assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), "%s k=%d: %s vs %s" % (
                    name, kbeg + j, got, want)
    print("pair elimination: %d generic, %d non-generic samples" % (counts[1], counts[0]))
    assert counts[0] > 100 and counts[1] > 1000


# ------------------------------------------------------------------------------------------------------------------
# 3. 32-lane null vectors
# ------------------------------------------------------------------------------------------------------------------
def null_cases(seed=4):
    """(name, Z [9 x len row-major, zero padded to 72], len, exact rank deficient?) from scene correspondences."""
    rng = np.random.default_rng(seed)
    p1, p2, _ = scene_F(400, 1.0, 90)
    out = []
    for coords in ("pixels", "normalised", "offset 1e4"):
        a, b = p1, p2
        if coords == "normalised":
            a, b = (p1 - 320) / 400, (p2 - 240) / 400
        elif coords == "offset 1e4":
            a, b = p1 + 1e4, p2 - 1e4
        for t in range(40):
            ln = 8 if t < 25 else 1 + t % 8
            idx = rng.choice(400, ln, replace=False)
            w = rng.uniform(0.1, 1.0, ln) if t % 2 else np.ones(ln)
            cols = [w[i] * np.array([b[k, 0] * a[k, 0], b[k, 0] * a[k, 1], b[k, 0], b[k, 1] * a[k, 0], b[k, 1] * a[k, 1],
                                     b[k, 1], a[k, 0], a[k, 1], 1.0]) for i, k in enumerate(idx)]
            Z = np.zeros(72)
            Z[:9 * ln] = np.stack(cols, 1).ravel()
            out.append(("%s len=%d #%d" % (coords, ln, t), Z, ln, False))
        for t in range(6):
            idx = rng.choice(400, 8, replace=False)
            idx[1 + t % 3] = idx[0]                 # a duplicated correspondence: rank 7
            cols = [np.array([b[k, 0] * a[k, 0], b[k, 0] * a[k, 1], b[k, 0], b[k, 1] * a[k, 0], b[k, 1] * a[k, 1],
                              b[k, 1], a[k, 0], a[k, 1], 1.0]) for k in idx]
            out.append(("%s duplicate #%d" % (coords, t), np.stack(cols, 1).ravel(), 8, False))
    for t in range(4):                              # x1 = 0 on every correspondence: exactly zero pivot column
        b = rng.uniform(0, 600, (8, 2))
        y1 = rng.uniform(0, 600, 8) if t % 2 else np.zeros(8)
        cols = [np.array([0.0, b[k, 0] * y1[k], b[k, 0], 0.0, b[k, 1] * y1[k], b[k, 1], 0.0, y1[k], 1.0]) for k in range(8)]
        out.append(("x1 = 0 #%d" % t, np.stack(cols, 1).ravel(), 8, True))
    return out


@pytest.mark.gpu
def test_warp_null_vectors_against_exact_null_space():
    dev = _dev()
    E = emu.lib()
    cases = null_cases()
    Z = np.stack([c[1] for c in cases]); lens = np.array([c[2] for c in cases])
    res = {mode: dev.null9(Z, lens, mode) for mode in (dev.NULL_REG, dev.NULL_8X9, dev.NULL_HOUSEHOLDER, dev.NULL_DISPATCH)}
    worst = 0.0
    for i, (name, z, ln, deficient) in enumerate(cases):
        Zm = z[:9 * ln].reshape(9, ln)
        zn = np.linalg.norm(Zm)
        # Householder route (all len): the host routine's arithmetic, and orthogonal to the columns
        qh = res[dev.NULL_HOUSEHOLDER][0][i]
        href = np.zeros(9)
        E.emu_left_null(_dp(np.ascontiguousarray(Zm.ravel().copy())), int(ln), _dp(href))
        assert np.array_equal(qh, href), name + ": warp Householder differs from left_null_9xk"
        assert abs(np.linalg.norm(qh) - 1) < 1e-13 and np.linalg.norm(Zm.T @ qh) <= 64 * EPS * zn, name
        qd = res[dev.NULL_DISPATCH][0][i]
        assert abs(np.linalg.norm(qd) - 1) < 1e-13 and np.linalg.norm(Zm.T @ qd) <= 64 * EPS * zn * (
            1 if ln < 8 else 1e3), "%s: |Z^T q| = %.3g |Z|" % (name, np.linalg.norm(Zm.T @ qd) / zn)
        if ln != 8:
            continue
        qr, okr = res[dev.NULL_REG][0][i], res[dev.NULL_REG][1][i]
        q8, ok8 = res[dev.NULL_8X9][0][i], res[dev.NULL_8X9][1][i]
        assert ok8 == okr and (not okr or np.array_equal(q8, qr)), name
        n = fraction_null_vector(Zm.T)
        if deficient:
            assert n is None and not okr, name + ": exactly rank-deficient system accepted"
            continue
        if n is None or "duplicate" in name:
            continue
        s = np.linalg.svd(Zm, compute_uv=False)
        cond = s[0] / s[-1]
        assert okr, name
        assert qr[8] > 0 and abs(np.linalg.norm(qr) - 1) < 1e-13, name
        ang = sin_angle(qr, n)
        worst = max(worst, ang / (EPS * cond))
        assert ang <= 64 * EPS * cond, "%s: angle %.3g, eps cond %.3g" % (name, ang, EPS * cond)
    print("null vectors: %d systems, worst angle / (eps cond) = %.3g" % (len(cases), worst))


# ------------------------------------------------------------------------------------------------------------------
# 4. 3x3 device arithmetic
# ------------------------------------------------------------------------------------------------------------------
def small3_inputs(kind, n=400):
    rng = np.random.default_rng(11)
    out = []
    for t in range(n):
        F = rng.uniform(-0.5, 0.5, (3, 3))
        if kind == "unnormalised":
            sc = np.array([1e-6, 1e-3, 1.0])
            F = F * sc[:, None] * sc[None, :]
        elif kind == "near_rank2":
            U, s, Vt = np.linalg.svd(F)
            s[2] *= 1e-7
            F = U @ np.diag(s) @ Vt
        elif kind == "clustered":
            U, s, Vt = np.linalg.svd(F)
            s[2] = 0.97 * s[1]
            F = U @ np.diag(s) @ Vt
        out.append(F)
    return np.stack(out)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["random", "unnormalised", "near_rank2", "clustered"])
def test_device_rank2_projection_and_svd3_match_numpy(kind):
    """The tolerances of test_small_la.py's host check, on the device spellings (rsqrt)."""
    dev = _dev()
    F = small3_inputs(kind)
    r = dev.small3(F)
    tol = 2e-10 if kind == "clustered" else 5e-12
    for i, f in enumerate(F):
        U, s, Vt = np.linalg.svd(f)
        ref = U @ np.diag([s[0], s[1], 0.0]) @ Vt
        n = np.linalg.norm(ref)
        for key in ("rank2", "rank2_slow", "rank2_inl"):
            assert np.linalg.norm(r[key][i].reshape(3, 3) - ref) / n < tol, (key, i)
        if r["fast_ok"][i]:
            v = r["v"][i]
            assert abs(np.linalg.norm(v) - 1) < 1e-14 and 1 - abs(np.dot(v, Vt[2])) < tol, i
        G, V, sv = r["G"][i].reshape(3, 3), r["V"][i].reshape(3, 3), r["sv"][i]
        assert np.abs(V.T @ V - np.eye(3)).max() < 1e-14, i
        assert np.linalg.norm(f @ V - G) <= 1e-14 * s[0], i
        assert np.abs(np.sort(sv)[::-1] - s).max() <= 1e-14 * s[0], i
    if kind == "clustered":
        assert r["fast_ok"].sum() < len(F)
    else:
        assert r["fast_ok"].sum() > 0.95 * len(F)


def pow2_inv_exponent_host(t):
    if not (t > 1e-290) or not (t < 1e290):
        return 0.0
    return math.ldexp(1.0, 1 - math.frexp(t)[1])


@pytest.mark.gpu
def test_device_pow2_inv_exponent_equals_host_spelling():
    dev = _dev()
    rng = np.random.default_rng(12)
    t = [10.0 ** rng.uniform(-300, 300, 20000), rng.uniform(0.5, 4, 1000)]
    edge = []
    for b in (1e-290, 1e290, 2.0 ** -963, 2.0 ** 963, 1.0, 2.0, 0.5):
        edge += [b, np.nextafter(b, 0), np.nextafter(b, np.inf)]
    edge += [0.0, -0.0, -1.0, 5e-324, 2.2250738585072014e-308, np.inf, -np.inf, np.nan, 1.7976931348623157e308]
    t = np.concatenate(t + [np.array(edge)])
    got = dev.pow2_inv_exponent(t)
    want = np.array([pow2_inv_exponent_host(v) for v in t])
    bad = np.flatnonzero(got.view(np.uint64) != want.view(np.uint64))
    assert bad.size == 0, [(t[i], got[i], want[i]) for i in bad[:5]]


# ------------------------------------------------------------------------------------------------------------------
# 5. FP32 upper bounds on the pair-interleaved tile
# ------------------------------------------------------------------------------------------------------------------
def _rank2(F):
    U, s, Vt = np.linalg.svd(F.reshape(3, 3))
    return (U @ np.diag([s[0], s[1], 0.0]) @ Vt).ravel(), Vt[2], U[:, 2]


def _eight_point(a, b):
    rows = np.stack([b[:, 0] * a[:, 0], b[:, 0] * a[:, 1], b[:, 0], b[:, 1] * a[:, 0], b[:, 1] * a[:, 1], b[:, 1],
                     a[:, 0], a[:, 1], np.ones(len(a))], 1)
    return np.linalg.svd(rows)[2][-1]


def _bisect(fun, target, lo, hi, iters=80):
    """t in [lo, hi] with fun(t) = target (vectorised, fun(lo) <= target <= fun(hi) assumed)."""
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        up = fun(mid) >= target
        hi = np.where(up, mid, hi)
        lo = np.where(up, lo, mid)
    return 0.5 * (lo + hi)


def f_filter_scene(rng, N, scale, offset, th, metric):
    """Correspondences of a scene (scaled, offset) plus correspondences placed at e = w (1 +- 2^-20), 18 th (1 +- 2^-20),
    on the epipolar line and next to the epipoles, for the model F0 fitted to the scene's inliers; models: F0, 8-point fits
    of random inlier samples, perturbations of F0."""
    p1, p2, gt = scene_F(N, 0.5, int(rng.integers(1 << 30)))
    p1 = p1 * scale + offset
    p2 = p2 * scale - 0.37 * offset
    inl = np.flatnonzero(gt)
    F0, e1, e2 = _rank2(_eight_point(p1[inl], p2[inl]))
    w = 9 * th / 4
    targets = np.array([w * (1 - 2 ** -20), w * (1 + 2 ** -20), 18 * th * (1 - 2 ** -20), 18 * th * (1 + 2 ** -20), 0.0])
    k = N // 3
    pick = inl[rng.integers(len(inl), size=k)]
    tg = targets[np.arange(k) % len(targets)]
    x1 = p1[pick].copy()
    l = np.stack([F0[0] * x1[:, 0] + F0[1] * x1[:, 1] + F0[2], F0[3] * x1[:, 0] + F0[4] * x1[:, 1] + F0[5],
                  F0[6] * x1[:, 0] + F0[7] * x1[:, 1] + F0[8]], 1)          # epipolar line of x1 in image 2
    nl = np.hypot(l[:, 0], l[:, 1])
    foot = p2[pick] - ((l[:, 0] * p2[pick, 0] + l[:, 1] * p2[pick, 1] + l[:, 2]) / nl ** 2)[:, None] * l[:, :2]
    nrm = l[:, :2] / nl[:, None]

    def err(t):
        q = foot + t[:, None] * nrm
        return f_sampson64(metric, F0[None, :], x1[:, 0], x1[:, 1], q[:, 0], q[:, 1])[0]
    t = _bisect(err, tg, np.zeros(k), np.full(k, 100.0 * math.sqrt(th) + 1.0))
    q = foot + t[:, None] * nrm
    p1[N - k:], p2[N - k:] = x1, q
    # next to the epipoles (tiny gradient) when they are finite
    if abs(e1[2]) > 1e-12 and abs(e2[2]) > 1e-12:
        for j in range(8):
            d = 10.0 ** -(j % 4 + 1) * scale
            p1[j] = e1[:2] / e1[2] + rng.normal(size=2) * d
            p2[j] = e2[:2] / e2[2] + rng.normal(size=2) * d
    models = [F0]
    for _ in range(20):
        s = rng.choice(inl, 8, replace=False)
        models.append(_rank2(_eight_point(p1[s], p2[s]))[0])
    for rel in (1e-9, 1e-6, 1e-3, 1e-1):
        for _ in range(2):
            models.append(F0 * (1 + rel * rng.normal(size=9)))
    return p1, p2, np.stack(models) * 10.0 ** rng.uniform(-3, 3), w


def h_filter_scene(rng, N, scale, offset, th):
    n_in = N // 2
    p1, p2, gt = scene_H(N, n_in, int(rng.integers(1 << 30)))
    p1 = p1 * scale + offset
    p2 = p2 * scale - 0.37 * offset
    inl = np.flatnonzero(gt)

    def dlt(a, b):       # column-major h with a ~ Hm b  (image 2 -> image 1)
        rows = []
        for (x1, y1), (x2, y2) in zip(a, b):
            rows.append([x2, 0, -x1 * x2, y2, 0, -x1 * y2, 1, 0, -x1])
            rows.append([0, x2, -y1 * x2, 0, y2, -y1 * y2, 0, 1, -y1])
        return np.linalg.svd(np.array(rows))[2][-1]
    h0 = dlt(p1[inl], p2[inl])
    w, far = 9 * th / 4, 18 * th
    targets = np.array([w * (1 - 2 ** -20), w * (1 + 2 ** -20), far * (1 - 2 ** -20), far * (1 + 2 ** -20), 0.0])
    k = N // 3
    pick = inl[rng.integers(len(inl), size=k)]
    tg = targets[np.arange(k) % len(targets)]
    x2 = p2[pick]
    Hm = h0.reshape(3, 3, order="F")
    pr = (Hm @ np.concatenate([x2, np.ones((k, 1))], 1).T).T
    x1c = pr[:, :2] / pr[:, 2:3]
    ang = rng.uniform(0, 2 * np.pi, k)
    dirn = np.stack([np.cos(ang), np.sin(ang)], 1)

    def err(t):
        q = x1c + t[:, None] * dirn
        return h_sampson64(h0[None, :], q[:, 0], q[:, 1], x2[:, 0], x2[:, 1])[0]
    t = _bisect(err, tg, np.zeros(k), np.full(k, 100.0 * math.sqrt(th) + 1.0))
    p1[N - k:], p2[N - k:] = x1c + t[:, None] * dirn, x2
    models = [h0]
    for _ in range(20):
        s = rng.choice(inl, 4, replace=False)
        models.append(dlt(p1[s], p2[s]))
    for rel in (1e-9, 1e-6, 1e-3, 1e-1):
        for _ in range(2):
            models.append(h0 * (1 + rel * rng.normal(size=9)))
    return p1, p2, np.stack(models) * 10.0 ** rng.uniform(-3, 3), w, far


class BoundLedger:
    """Counts the (model, correspondence) checks of g_up >= truncQuad(e_exact) and keeps the smallest slack."""

    def __init__(self):
        self.checks = 0
        self.min_slack = np.inf
        self.rechecked = 0

    def gains(self, what, g, e64, w, exact):
        g = g.astype(np.float64)
        with np.errstate(invalid="ignore"):
            t64 = np.where(e64 < w, 1.0 - e64 / w, 0.0)
            t64 = np.where(np.isnan(e64), 0.0, t64)
        self.checks += g.size
        slack = g - t64
        live = (t64 > 0) & (t64 < 1)
        if live.any():
            self.min_slack = min(self.min_slack, float(slack[live].min()))
        # where float64 cannot settle it, the exact residual does
        doubt = (slack < 1e-9) & ~((g == 0) & (e64 >= w * (1 + 1e-9))) & ~(g >= 1.0)
        for m, i in zip(*np.nonzero(doubt)):
            self.rechecked += 1
            e = exact(m, i)
            assert e is not None, "%s: model %d, correspondence %d has a degenerate exact residual" % (what, m, i)
            tq = 1 - e / Fraction(w) if e < Fraction(w) else Fraction(0)
            assert Fraction(float(g[m, i])) >= tq, "%s: model %d, correspondence %d: g_up %.9g < exact gain %.9g" % (
                what, m, i, g[m, i], float(tq))

    def score(self, what, J, g64sum):
        Jup = J.astype(np.float64) * (1.0 + 2.0 ** -16) + 1e-3
        assert np.all(Jup >= g64sum * (1 + 1e-12)), "%s: J_up %s < J %s" % (what, Jup[Jup < g64sum], g64sum[Jup < g64sum])


def _check_tile(p1, p2, tile, cb):
    """The tile is the pair kernel's: centred single-precision coordinates, pair-interleaved, zero padding slot."""
    N = p1.shape[0]
    cen = np.array([p1[:, 0].mean(), p1[:, 1].mean(), p2[:, 0].mean(), p2[:, 1].mean()])
    assert np.allclose(cb[:4], cen, rtol=1e-12, atol=1e-9 * np.abs(cen).max())
    c = np.stack([p1[:, 0] - cb[0], p1[:, 1] - cb[1], p2[:, 0] - cb[2], p2[:, 1] - cb[3]], 1).astype(np.float32)
    full = np.zeros((tile.shape[0] * 2, 4), dtype=np.float32)
    full[:N] = c
    want = np.stack([full[0::2, 0], full[1::2, 0], full[0::2, 1], full[1::2, 1],
                     full[0::2, 2], full[1::2, 2], full[0::2, 3], full[1::2, 3]], 1)
    assert np.array_equal(tile, want)
    assert np.array_equal(cb[4:], np.abs(c).max(0).astype(np.float64))


FILTER_CONFIGS = [(N, scale, offset) for N in (2001, 1500) for scale, offset in ((1.0, 0.0), (8.0, 1e4), (0.05, -300.0))]


@pytest.mark.gpu
def test_fp32_score_bounds_hold_on_the_device_tile():
    dev = _dev()
    rng = np.random.default_rng(13)
    led = BoundLedger()
    for N, scale, offset in FILTER_CONFIGS:
        for px in (1.0, 0.3):
            th = (px * scale) ** 2
            # F, both metrics
            for metric in (0, 1):
                p1, p2, F, w = f_filter_scene(rng, N, scale, offset, th, metric)
                tile, cb = dev.tile32(p1, p2)
                _check_tile(p1, p2, tile, cb)
                g, J = dev.ffilter(tile, cb, N, metric, w, F)
                if N % 2:
                    assert np.all(g[:, N] == 0), "padding slot scored"
                g = g[:, :N]
                e64 = f_sampson64(metric, F, p1[:, 0], p1[:, 1], p2[:, 0], p2[:, 1])
                what = "F metric %d N %d scale %g offset %g th %g" % (metric, N, scale, offset, th)
                led.gains(what, g, e64, w, lambda m, i: f_sampson_exact(metric, F[m], p1[i, 0], p1[i, 1], p2[i, 0], p2[i, 1]))
                with np.errstate(invalid="ignore"):
                    led.score(what, J, np.where(e64 < w, 1 - e64 / w, 0.0).sum(1))
            # H, Sampson
            p1, p2, h, w, far = h_filter_scene(rng, N, scale, offset, th)
            tile, cb = dev.tile32(p1, p2)
            _check_tile(p1, p2, tile, cb)
            g, J, raw = dev.hfilter(tile, cb, N, w, far, h)
            if N % 2:
                assert np.all(g[:, N] == 0), "padding slot scored"
            g, raw = g[:, :N], raw[:, :N]
            e64 = h_sampson64(h, p1[:, 0], p1[:, 1], p2[:, 0], p2[:, 1])
            what = "H N %d scale %g offset %g th %g" % (N, scale, offset, th)
            exact = lambda m, i: h_sampson_exact(h[m], p1[i, 0], p1[i, 1], p2[i, 0], p2[i, 1])   # noqa: E731
            led.gains(what, g, e64, w, exact)
            with np.errstate(invalid="ignore"):
                led.score(what, J, np.where(e64 < w, 1 - e64 / w, 0.0).sum(1))
            # marked far (raw <= 0, an ordinary number) => exact error >= 18 th
            marked = (raw <= 0) & (raw >= -3e38)
            led.checks += raw.size
            assert marked.sum() > 0.2 * raw.size
            for m, i in zip(*np.nonzero(marked & ~(e64 >= far * (1 + 1e-9)))):
                led.rechecked += 1
                e = exact(m, i)
                assert e is not None and e >= Fraction(far), "%s: model %d, correspondence %d marked far" % (what, m, i)
    print("FP32 bounds: %d checks, smallest slack of a positive gain %.3g, %d settled exactly" % (
        led.checks, led.min_slack, led.rechecked))
    assert led.checks >= 10 ** 6
