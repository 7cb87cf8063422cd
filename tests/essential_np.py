"""numpy restatement of matching.find_essential_ragged -- TEST INFRASTRUCTURE ONLY.

The estimator's contract (include/degensac_b200.h) written out literally:
  * usable rows: mask set and four finite coordinates, listed in row order; fewer than 5: no model;
  * iteration k = 1, 2, ...: Philox minimal sample of 5 list entries (csrc/rng.h), the five-point solver on the
    normalised coordinates K^-1 [x, y, 1] (csrc/five_point.h, restated here operation by operation over numpy arrays of
    samples, so that the two agree to the bit);
  * F = K2^-T E K1^-1 at unit norm, MSAC cost sum min(e^2, th^2) with e^2 the Sampson error in pixels and the inlier
    rule e^2 < th^2, strict improvement only, the N_req stopping rule for samples of 5;
  * local optimisation: up to 3 rounds of Levenberg-Marquardt on the inliers (refine_pose_ragged's arithmetic, from one
    decomposition of E) and re-selection, kept when its MSAC cost is <= the RANSAC model's.

tests/test_essential.py pins the solver to cv2.findEssentialMat and the sampling to the host build of csrc/rng.h."""
import math

import numpy as np

from tests.absolute_pose_np import inv3, philox4x32_10
from tests.pose_refine_np import refine_pair, sampson_sq

MIN_ROWS, LO_MIN_INLIERS, LO_ROUNDS = 5, 6, 3
MAX_SOLUTIONS, ISOLATE_STEPS, REFINE_STEPS, POLISH_STEPS = 10, 128, 100, 3
TIE_REL = 1e-12

_Q = [0, 1, 2, 3, 1, 4, 5, 6, 2, 5, 7, 8, 3, 6, 8, 9]
_C = [0, 2, 4, 5, 2, 3, 8, 9, 4, 8, 10, 11, 5, 9, 11, 12, 3, 1, 6, 7,
      8, 6, 13, 14, 9, 7, 14, 15, 10, 13, 16, 17, 11, 14, 17, 18, 12, 15, 18, 19]


# ------------------------------------------------------------------------------------------------ Philox (csrc/rng.h)
def minimal_sample(seed, k, n, m=5):
    """dg::minimal_sample<m>: m distinct indices in [0, n) in draw order (partial Fisher-Yates over a virtual pool)"""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    key = (seed & 0xFFFFFFFF, seed >> 32)
    r = list(philox4x32_10((0, int(k) & 0xFFFFFFFF, 0, 0), key))
    if m > 4:
        r += list(philox4x32_10((1, int(k) & 0xFFFFFFFF, 0, 0), key))
    pool = {}
    sel = []
    for i in range(m):
        s = (r[i] >> 1) % (n - i)
        top = n - i - 1
        vs, vt = pool.get(s, s), pool.get(top, top)
        pool[s] = vt
        pool[top] = vs
        sel.append(vs)
    return sel


# ------------------------------------------------------------------------------------------------ five_point.h
def _mul11(a, b, s, q):
    for i in range(4):
        for j in range(4):
            m = _Q[4 * i + j]
            q[:, m] = q[:, m] + s * (a[:, i] * b[:, j])


def _mul21(q, l, c):
    for i in range(10):
        for j in range(4):
            m = _C[4 * i + j]
            c[:, m] = c[:, m] + q[:, i] * l[:, j]


def _pmul(a, b, c):
    for i in range(a.shape[1]):
        for j in range(b.shape[1]):
            c[:, i + j] = c[:, i + j] + a[:, i] * b[:, j]


def horner(p, deg, z):
    v = p[..., deg]
    for i in range(deg - 1, -1, -1):
        v = v * z + p[..., i]
    return v


def variations(s, z):
    """sign variations of the packed Sturm sequences s [..., 66] at z [...], zeros skipped"""
    count = np.zeros(z.shape, np.int64)
    last = np.zeros(z.shape, np.int64)
    off = 0
    for k in range(11):
        deg = 10 - k
        v = horner(s[..., off:off + deg + 1], deg, z)
        off += deg + 1
        sg = np.where(v > 0.0, 1, np.where(v < 0.0, -1, 0))
        count += (sg != 0) & (last != 0) & (sg != last)
        last = np.where(sg != 0, sg, last)
    return count


def null_space(x1, x2):
    """fp_null_space over samples: x1, x2 [S,5,3] -> (N [S,4,9], ok [S])"""
    S = len(x1)
    M = np.empty((S, 9, 5))
    for c in range(5):
        for i in range(3):
            for j in range(3):
                M[:, 3 * i + j, c] = x2[:, c, i] * x1[:, c, j]
    V = np.zeros((S, 5, 9))
    beta = np.zeros((S, 5))
    ok = np.ones(S, bool)
    for c in range(5):
        s = np.zeros(S)
        for r in range(c, 9):
            s = s + M[:, r, c] * M[:, r, c]
        ok &= s > 0.0
        nrm = np.sqrt(s)
        alpha = np.where(M[:, c, c] < 0.0, nrm, -nrm)
        V[:, c, c:] = M[:, c:, c]
        V[:, c, c] = V[:, c, c] - alpha
        vv = np.zeros(S)
        for r in range(c, 9):
            vv = vv + V[:, c, r] * V[:, c, r]
        ok &= vv > 0.0
        beta[:, c] = 2.0 / vv
        w = np.zeros((S, 4 - c))
        for r in range(c, 9):
            w = w + V[:, c, r, None] * M[:, r, c + 1:]
        f = beta[:, c, None] * w
        for r in range(c, 9):
            M[:, r, c + 1:] = M[:, r, c + 1:] - f * V[:, c, r, None]
    N = np.empty((S, 4, 9))
    for j in range(4):
        y = np.zeros((S, 9))
        y[:, 5 + j] = 1.0
        for c in range(4, -1, -1):
            w = np.zeros(S)
            for r in range(c, 9):
                w = w + V[:, c, r] * y[:, r]
            f = beta[:, c] * w
            for r in range(c, 9):
                y[:, r] = y[:, r] - f * V[:, c, r]
        N[:, j] = y
    return N, ok


def constraints(N):
    """fp_constraints: C [S,10,20]"""
    S = len(N)
    E = np.transpose(N, (0, 2, 1))                   # [S,9,4]
    C = np.zeros((S, 10, 20))
    cof = np.zeros((3, S, 10))
    for j in range(3):
        j1, j2 = (j + 1) % 3, (j + 2) % 3
        _mul11(E[:, 3 + j1], E[:, 6 + j2], 1.0, cof[j])
        _mul11(E[:, 3 + j2], E[:, 6 + j1], -1.0, cof[j])
    for j in range(3):
        _mul21(cof[j], E[:, j], C[:, 0])
    Q = np.zeros((3, 3, S, 10))
    for i in range(3):
        for j in range(3):
            for k in range(3):
                _mul11(E[:, 3 * i + k], E[:, 3 * j + k], 1.0, Q[i, j])
    tr = (Q[0, 0] + Q[1, 1]) + Q[2, 2]
    for i in range(3):
        for j in range(3):
            row = C[:, 1 + 3 * i + j]
            for k in range(3):
                T = 2.0 * Q[i, k] - tr if i == k else 2.0 * Q[i, k]
                _mul21(T, E[:, 3 * k + j], row)
            C[:, 1 + 3 * i + j] = row
    return C


def eliminate(C):
    """fp_eliminate in place; returns ok [S]"""
    S = len(C)
    ar = np.arange(S)
    ok = np.ones(S, bool)
    for c in range(10):
        p = np.full(S, c)
        best = np.abs(C[:, c, c])
        for r in range(c + 1, 10):
            up = np.abs(C[:, r, c]) > best
            best = np.where(up, np.abs(C[:, r, c]), best)
            p = np.where(up, r, p)
        ok &= best > 0.0
        rc, rp = C[:, c, c:].copy(), C[ar, p, c:].copy()
        C[:, c, c:] = rp
        C[ar, p, c:] = np.where((p == c)[:, None], rp, rc)
        piv = C[:, c, c].copy()
        C[:, c, c:] = C[:, c, c:] / piv[:, None]
        others = [r for r in range(10) if r != c]
        f = C[:, others, c].copy()
        C[:, others, c:] = C[:, others, c:] - f[:, :, None] * C[:, None, c, c:]
    return ok


def _brow(ra, rb):
    px = np.stack([ra[:, 12], ra[:, 11] - rb[:, 12], ra[:, 10] - rb[:, 11], -rb[:, 10]], 1)
    py = np.stack([ra[:, 15], ra[:, 14] - rb[:, 15], ra[:, 13] - rb[:, 14], -rb[:, 13]], 1)
    p1 = np.stack([ra[:, 19], ra[:, 18] - rb[:, 19], ra[:, 17] - rb[:, 18], ra[:, 16] - rb[:, 17], -rb[:, 16]], 1)
    return px, py, p1


def sturm(a):
    """fp_sturm: (s [S,66], ok [S])"""
    S = len(a)
    s = np.zeros((S, 66))
    s[:, :11] = a
    for i in range(10):
        s[:, 11 + i] = float(i + 1) * a[:, i + 1]
    ok = np.ones(S, bool)
    offA, offB = 0, 11
    for d in range(9, 0, -1):
        A, B = s[:, offA:offA + d + 2], s[:, offB:offB + d + 1]
        ok &= B[:, d] != 0.0
        q1 = A[:, d + 1] / B[:, d]
        q0 = (A[:, d] - q1 * B[:, d - 1]) / B[:, d]
        R0 = offB + d + 1
        for i in range(d):
            r = A[:, i] - q0 * B[:, i]
            if i > 0:
                r = r - q1 * B[:, i - 1]
            s[:, R0 + i] = -r
        offA, offB = offB, offB + d + 1
    ok &= s[:, 65] != 0.0
    return s, ok


def residual(C, x, y, z):
    """fp_residual over roots: C [J,10,20] -> (|r|^2 [J], r [J,10], Jac [J,10,3])"""
    xx, yy, zz, xy, xz, yz = x * x, y * y, z * z, x * y, x * z, y * z
    zero, one = np.zeros_like(x), np.ones_like(x)
    m = [xx * x, yy * y, xx * y, x * yy, xx * z, xx, yy * z, yy, xy * z, xy, x * zz, xz, x, y * zz, yz, y, zz * z, zz,
         z, one]
    mx = [3.0 * xx, zero, 2.0 * xy, yy, 2.0 * xz, 2.0 * x, zero, zero, yz, y, zz, z, one, zero, zero, zero, zero, zero,
          zero, zero]
    my = [zero, 3.0 * yy, xx, 2.0 * xy, zero, zero, 2.0 * yz, 2.0 * y, xz, x, zero, zero, zero, zz, z, one, zero, zero,
          zero, zero]
    mz = [zero, zero, zero, zero, xx, zero, yy, zero, xy, zero, 2.0 * xz, x, zero, 2.0 * yz, y, zero, 3.0 * zz, 2.0 * z,
          one, zero]
    r = np.zeros((len(x), 10))
    Jc = np.zeros((len(x), 10, 3))
    rr = np.zeros(len(x))
    for i in range(10):
        v, a, b, c = zero, zero, zero, zero
        for k in range(20):
            v = v + C[:, i, k] * m[k]
            a = a + C[:, i, k] * mx[k]
            b = b + C[:, i, k] * my[k]
            c = c + C[:, i, k] * mz[k]
        r[:, i], Jc[:, i, 0], Jc[:, i, 1], Jc[:, i, 2] = v, a, b, c
        rr = rr + v * v
    return rr, r, Jc


def polish(C, x, y, z):
    """fp_polish over roots"""
    rr, r, Jc = residual(C, x, y, z)
    act = np.ones(len(x), bool)
    for _ in range(POLISH_STEPS):
        H = [np.zeros(len(x)) for _ in range(6)]
        g = [np.zeros(len(x)) for _ in range(3)]
        for i in range(10):
            j0, j1, j2, ri = Jc[:, i, 0], Jc[:, i, 1], Jc[:, i, 2], r[:, i]
            H[0] = H[0] + j0 * j0; H[1] = H[1] + j0 * j1; H[2] = H[2] + j0 * j2
            H[3] = H[3] + j1 * j1; H[4] = H[4] + j1 * j2; H[5] = H[5] + j2 * j2
            g[0] = g[0] + j0 * ri; g[1] = g[1] + j1 * ri; g[2] = g[2] + j2 * ri
        act = act & (H[0] > 0.0)
        l00 = np.sqrt(H[0]); l10 = H[1] / l00; l20 = H[2] / l00
        d1 = H[3] - l10 * l10
        act = act & (d1 > 0.0)
        l11 = np.sqrt(d1); l21 = (H[4] - l20 * l10) / l11
        d2 = (H[5] - l20 * l20) - l21 * l21
        act = act & (d2 > 0.0)
        l22 = np.sqrt(d2)
        y0 = -g[0] / l00; y1 = (-g[1] - l10 * y0) / l11; y2 = ((-g[2] - l20 * y0) - l21 * y1) / l22
        D2 = y2 / l22; D1 = (y1 - l21 * D2) / l11; D0 = ((y0 - l10 * D1) - l20 * D2) / l00
        xn, yn, zn = x + D0, y + D1, z + D2
        rn, r, Jc = residual(C, xn, yn, zn)
        act = act & (rn < rr)
        x, y, z = np.where(act, xn, x), np.where(act, yn, y), np.where(act, zn, z)
        rr = np.where(act, rn, rr)
        if not act.any():
            break
    return x, y, z


def five_point(x1, x2):
    """dg::five_point over samples x1, x2 [S,5,3] (normalised coordinates): a list of S arrays [ns,9] of essential
    matrices at unit Frobenius norm, in the solver's order"""
    x1, x2 = np.asarray(x1, np.float64), np.asarray(x2, np.float64)
    S = len(x1)
    with np.errstate(all="ignore"):
        N, ok = null_space(x1, x2)
        C0 = constraints(N)
        C = C0.copy()
        ok &= eliminate(C)
        Bp = [_brow(C[:, 4 + 2 * r], C[:, 5 + 2 * r]) for r in range(3)]
        (kx, ky, k1), (lx, ly, l1), (mx, my, m1) = Bp
        p = np.zeros((S, 11))
        u, v = np.zeros((S, 8)), np.zeros((S, 8))
        _pmul(ly, m1, u); _pmul(l1, my, v)
        u = u - v
        t = np.zeros((S, 11)); _pmul(kx, u, t)
        p = p + t
        u, v = np.zeros((S, 8)), np.zeros((S, 8))
        _pmul(lx, m1, u); _pmul(l1, mx, v)
        u = u - v
        t = np.zeros((S, 11)); _pmul(ky, u, t)
        p = p - t
        w, v = np.zeros((S, 7)), np.zeros((S, 7))
        _pmul(lx, my, w); _pmul(ly, mx, v)
        w = w - v
        t = np.zeros((S, 11)); _pmul(k1, w, t)
        p = p + t
        ok &= (np.abs(p[:, 10]) > 0.0) & (np.abs(p[:, 10]) < np.inf)
        a = np.empty((S, 11))
        bound = np.zeros(S)
        for m in range(10):
            a[:, m] = p[:, m] / p[:, 10]
            ok &= np.abs(a[:, m]) < np.inf
            bound = np.where(np.abs(a[:, m]) > bound, np.abs(a[:, m]), bound)
        a[:, 10] = 1.0
        bound = 1.0 + bound
        s, sok = sturm(a)
        ok &= sok
        v_lo = variations(s, -bound)
        n_roots = np.where(ok, v_lo - variations(s, bound), 0)
        # every (sample, root index) at once
        si = np.repeat(np.arange(S), np.minimum(n_roots, MAX_SOLUTIONS))
        ji = np.concatenate([np.arange(min(int(n), MAX_SOLUTIONS)) for n in n_roots]) if S else np.zeros(0, np.int64)
        ji = ji.astype(np.int64)
        ss, vl = s[si], v_lo[si]
        lo, hi = -bound[si], bound[si].copy()
        nlo, nhi = np.zeros(len(si), np.int64), n_roots[si].astype(np.int64)
        for _ in range(ISOLATE_STEPS):
            act = ~((nlo == ji) & (nhi == ji + 1))
            if not act.any():
                break
            mid = 0.5 * (lo + hi)
            c = vl - variations(ss, mid)
            up = act & (c > ji)
            dn = act & ~(c > ji)
            hi = np.where(up, mid, hi); nhi = np.where(up, c, nhi)
            lo = np.where(dn, mid, lo); nlo = np.where(dn, c, nlo)
        aa = a[si]
        flo = horner(aa, 10, lo)
        fhi = horner(aa, 10, hi)
        keep = ((flo <= 0.0) & (fhi >= 0.0)) | ((flo >= 0.0) & (fhi <= 0.0))
        for _ in range(REFINE_STEPS):
            mid = 0.5 * (lo + hi)
            fm = horner(aa, 10, mid)
            same = (fm < 0.0) == (flo < 0.0)
            lo = np.where(same, mid, lo); flo = np.where(same, fm, flo)
            hi = np.where(same, hi, mid)
        z = 0.5 * (lo + hi)
        b = np.empty((len(si), 3, 3))
        for r in range(3):
            b[:, r, 0] = horner(Bp[r][0][si], 3, z)
            b[:, r, 1] = horner(Bp[r][1][si], 3, z)
            b[:, r, 2] = horner(Bp[r][2][si], 4, z)
        best = np.zeros((len(si), 3))
        best_n = np.full(len(si), -1.0)
        for r in range(3):
            u, w = b[:, 1 if r == 2 else 0], b[:, 1 if r == 0 else 2]
            cr = np.stack([u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1], u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2],
                           u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]], 1)
            nn = (cr[:, 0] * cr[:, 0] + cr[:, 1] * cr[:, 1]) + cr[:, 2] * cr[:, 2]
            up = nn > best_n
            best_n = np.where(up, nn, best_n)
            best = np.where(up[:, None], cr, best)
        keep &= best[:, 2] != 0.0
        x = best[:, 0] / best[:, 2]
        y = best[:, 1] / best[:, 2]
        x, y, z = polish(C0[si], x, y, z)
        Ns = N[si]
        E = ((x[:, None] * Ns[:, 0] + y[:, None] * Ns[:, 1]) + z[:, None] * Ns[:, 2]) + Ns[:, 3]
        nrm = np.zeros(len(si))
        for e in range(9):
            nrm = nrm + E[:, e] * E[:, e]
        keep &= (nrm > 0.0) & (nrm < np.inf)
        E = E * (1.0 / np.sqrt(nrm))[:, None]
    out = [np.zeros((0, 9)) for _ in range(S)]
    for i in range(S):
        out[i] = E[(si == i) & keep]
    return out


# ------------------------------------------------------------------------------------------------ essential.h
def normalise(Ki, x, y):
    """K^-1 [x, y, 1] per row: [n,3]"""
    Ki = np.asarray(Ki, np.float64).ravel()
    return np.stack([Ki[3 * i] * x + Ki[3 * i + 1] * y + Ki[3 * i + 2] for i in range(3)], -1)


def unit9(M):
    M = np.asarray(M, np.float64).ravel()
    nrm = 0.0
    for i in range(9):
        nrm = nrm + M[i] * M[i]
    inv = 1.0 / math.sqrt(nrm) if nrm > 0.0 else 0.0
    return M * inv


def mul3(A, B):
    """pr_mul3, row-major [9] x [9]"""
    A, B = np.asarray(A, np.float64).ravel(), np.asarray(B, np.float64).ravel()
    return np.array([A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j]
                     for i in range(3) for j in range(3)])


def fundamental(E, A, Bk):
    """es_fundamental: A E Bk at unit norm (A = K2^-T, Bk = K1^-1)"""
    return unit9(mul3(mul3(A, E), Bk))


def fundamentals(Es, A, Bk):
    """fundamental over [H,9] essential matrices, vectorised in the same operation order"""
    Es = np.asarray(Es, np.float64).reshape(-1, 9)
    A, Bk = np.asarray(A, np.float64).ravel(), np.asarray(Bk, np.float64).ravel()
    AE = np.stack([A[3 * i] * Es[:, j] + A[3 * i + 1] * Es[:, 3 + j] + A[3 * i + 2] * Es[:, 6 + j]
                   for i in range(3) for j in range(3)], 1)
    F = np.stack([AE[:, 3 * i] * Bk[j] + AE[:, 3 * i + 1] * Bk[3 + j] + AE[:, 3 * i + 2] * Bk[6 + j]
                  for i in range(3) for j in range(3)], 1)
    nrm = np.zeros(len(F))
    for i in range(9):
        nrm = nrm + F[:, i] * F[:, i]
    with np.errstate(divide="ignore"):
        inv = np.where(nrm > 0.0, 1.0 / np.sqrt(nrm), 0.0)
    return F * inv[:, None]


def msac(F, p1, p2, th2):
    """es_msac per row of F [H,9] (or [9]): terms min(e^2, th^2) [H,n] and inlier flags e^2 < th^2"""
    F = np.asarray(F, np.float64).reshape(-1, 9)
    with np.errstate(all="ignore"):
        e2 = np.stack([sampson_sq(f, p1, p2) for f in F])
    return np.fmin(e2, th2), e2 < th2


def _cross(a, b):
    return np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


def _unit3(v):
    inv = 1.0 / math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    return v * inv


def orthonormalise(R):
    """pr_orthonormalise on R [9]"""
    R = np.array(R, np.float64).ravel()
    R[0:3] = _unit3(R[0:3])
    p = R[0] * R[3] + R[1] * R[4] + R[2] * R[5]
    for i in range(3):
        R[3 + i] = R[3 + i] - p * R[i]
    R[3:6] = _unit3(R[3:6])
    R[6:9] = _cross(R[0:3], R[3:6])
    return R


def skew(v):
    return np.array([0.0, -v[2], v[1], v[2], 0.0, -v[0], -v[1], v[0], 0.0])


def pose(E):
    """es_pose: (R [9], t [3]) with E ~ [t]x R, or None for a rank < 2 E"""
    E = np.asarray(E, np.float64).ravel()
    c = [np.array([E[0], E[3], E[6]]), np.array([E[1], E[4], E[7]]), np.array([E[2], E[5], E[8]])]
    best, t = -1.0, None
    for k in range(3):
        u = _cross(c[1 if k == 2 else 0], c[1 if k == 0 else 2])
        nn = (u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]
        if nn > best:
            best, t = nn, u
    if not (best > 0.0 and best < math.inf):
        return None
    t = _unit3(t)
    cof = np.r_[_cross(E[3:6], E[6:9]), _cross(E[6:9], E[0:3]), _cross(E[0:3], E[3:6])]
    TE = mul3(skew(t), E)
    R = 2.0 * cof - math.sqrt(2.0) * TE
    return orthonormalise(R), t


def essential(R, t):
    """es_essential: [t]x R at unit norm"""
    return unit9(mul3(skew(np.asarray(t, np.float64).ravel()), R))


def required_iters(has_best, inl, n, conf, max_iters, k):
    if not has_best or conf >= 1.0:
        return max_iters
    if inl >= n:
        return k
    w = inl / n
    with np.errstate(divide="ignore"):
        q = np.ceil(np.log(1.0 - conf) / np.log1p(-((((w * w) * w) * w) * w)))
    return int(q) if q < max_iters else max_iters


# ------------------------------------------------------------------------------------------------ RANSAC
def usable(p1, p2, mask=None):
    ok = np.isfinite(p1[:, :2]).all(1) & np.isfinite(p2[:, :2]).all(1)
    if mask is not None:
        ok &= np.asarray(mask).astype(bool)
    return ok


def find_essential(p1, p2, K1, K2, mask=None, px_th=1.0, conf=0.999, max_iters=10000, seed=0, refine_iters=10,
                   chunk=64):
    """One pair.  Returns a dict: E, F [3,3], mask (over the given rows), n_inliers, iters, cost0, cost; near_tie: a
    strict hypothesis other than the best, with other inliers or a model more than 1e-9 away, has a cost within 1e-12
    of the best's, so that summation order may pick either; lo_tie: the same for the LO's acceptance; lo_rounds."""
    p1, p2 = np.asarray(p1, np.float64)[:, :2], np.asarray(p2, np.float64)[:, :2]
    K1, K2 = np.asarray(K1, np.float64), np.asarray(K2, np.float64)
    rows = len(p1)
    lst = np.flatnonzero(usable(p1, p2, mask))
    n = len(lst)
    out = dict(E=np.zeros((3, 3)), F=np.zeros((3, 3)), mask=np.zeros(rows, bool), n_inliers=0, iters=0,
               cost0=np.nan, cost=np.nan, near_tie=False, lo_tie=False, lo_rounds=0)
    if n < MIN_ROWS:
        return out
    a1, a2 = p1[lst], p2[lst]
    th2 = float(px_th) * float(px_th)
    K1i, K2i = inv3(K1), inv3(K2)
    A = K2i.T.copy()
    n1, n2 = normalise(K1i, a1[:, 0], a1[:, 1]), normalise(K2i, a2[:, 0], a2[:, 1])
    best = None                                      # (cost, inliers, E, F)
    seen = []
    k, done = 0, False
    while not done:
        ks = list(range(k + 1, min(k + chunk, max_iters) + 1))
        sels = np.array([minimal_sample(seed, kk, n) for kk in ks])
        sols = five_point(n1[sels], n2[sels])
        for kk, Es in zip(ks, sols):
            k = kk
            if len(Es):
                Fs = fundamentals(Es, A, K1i)
                terms, inl = msac(Fs, a1, a2, th2)
                for s in range(len(Es)):
                    c = float(terms[s].sum())
                    seen.append((c, int(inl[s].sum()), Es[s], Fs[s]))
                    if best is None or c < best[0]:
                        best = seen[-1]
            req = required_iters(best is not None, best[1] if best else 0, n, conf, max_iters, k)
            if not k < req:
                done = True
                break
    out["iters"] = k
    if best is None:
        return out
    out["near_tie"] = any(h is not best and abs(h[0] - best[0]) <= TIE_REL * abs(best[0]) and
                          (h[1] != best[1] or min(np.abs(h[2] - best[2]).max(), np.abs(h[2] + best[2]).max()) > 1e-9)
                          for h in seen)
    cost0, _, E0, F0 = best
    terms, inl = msac(F0, a1, a2, th2)
    inl = inl[0]
    E, F, cost = E0, F0, cost0
    if refine_iters > 0 and inl.sum() >= LO_MIN_INLIERS:
        st = pose(E0)
        if st is not None:
            R, t = st[0].reshape(3, 3), st[1]
            flags = inl
            for rnd in range(LO_ROUNDS):
                r = refine_pair(R, t, K1, K2, a1[flags], a2[flags], refine_iters)
                R, t = r["R"], r["t"]
                El = essential(R, t)
                Fl = fundamental(El, A, K1i)
                terms, new = msac(Fl, a1, a2, th2)
                new = new[0]
                out["lo_rounds"] = rnd + 1
                changed = int((new != flags).sum())
                flags = new
                if changed == 0 or new.sum() < LO_MIN_INLIERS:
                    break
            c = float(terms.sum())
            out["lo_tie"] = abs(c - cost0) <= TIE_REL * abs(cost0)
            if c <= cost0:
                E, F, cost, inl = El, Fl, c, flags
    m = np.zeros(rows, bool)
    m[lst] = inl
    out.update(E=np.asarray(E).reshape(3, 3), F=np.asarray(F).reshape(3, 3), mask=m, n_inliers=int(inl.sum()),
               cost0=cost0, cost=cost)
    return out


def find_essential_ragged(p1, p2, K1, K2, offsets, mask=None, px_th=1.0, conf=0.999, max_iters=10000, seeds=None,
                          refine_iters=10):
    """The ragged call: per pair the dict of find_essential; malformed spans (decreasing, negative, past the rows) get
    no model and iters 0."""
    p1, p2 = np.asarray(p1, np.float64), np.asarray(p2, np.float64)
    offsets = np.asarray(offsets)
    P = len(offsets) - 1
    K1, K2 = np.asarray(K1, np.float64), np.asarray(K2, np.float64)
    seeds = np.broadcast_to(np.asarray(seeds if seeds is not None else 0, dtype=np.uint64), (P,))
    res = []
    for p in range(P):
        b, e = int(offsets[p]), int(offsets[p + 1])
        K1p = K1[p] if K1.ndim == 3 else K1
        K2p = K2[p] if K2.ndim == 3 else K2
        if not (0 <= b <= e <= len(p1)):
            r = find_essential(np.zeros((0, 2)), np.zeros((0, 2)), K1p, K2p)
            r["span"] = None
        else:
            r = find_essential(p1[b:e], p2[b:e], K1p, K2p, None if mask is None else np.asarray(mask)[b:e], px_th,
                               conf, max_iters, int(seeds[p]), refine_iters)
            r["span"] = (b, e)
        res.append(r)
    return res
