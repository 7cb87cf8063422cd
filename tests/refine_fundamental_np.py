"""numpy restatement of matching.refine_fundamental_ragged -- TEST INFRASTRUCTURE ONLY.

Levenberg-Marquardt on the Sampson error of a fundamental matrix over the rank-2 matrices, with the pieces of
csrc/refine_f.h and the schedule of f_refine_ragged_kernel (csrc/frontend.cu) written out once more so that the two
take the same steps:

    F row-major, x2^T F x1 = 0;  r = (p2^T F p1) / sqrt((F p1)_0^2 + (F p1)_1^2 + (F^T p2)_0^2 + (F^T p2)_1^2), so r^2 is
    f_resid_sampson (csrc/fgeom.h)
    T1, T2: centroid to the origin, RMS distance sqrt(2), from the masked rows;  Fn = T2^-T F T1^-1;  F = T2^T Fn T1
    start Fn0 = unit(rank2(T2^-T F_in T1^-1)), rank2 the rank-2 projection of csrc/la.h (enforce_rank2_inl)
    local step d [7]:  Fn <- unit(rank2(Fn + B d)),  B = basis(Fn): an orthonormal basis of the complement of vec(Fn)
    and vec(cof Fn) by two Householder reflections;  residuals in pixels
    schedule: that of tests/pose_refine_np.py with a 7 x 7 solve and at least 8 rows.

tests/test_refine_fundamental.py pins the Jacobian to central differences and the result to
scipy.optimize.least_squares."""
import numpy as np

from tests.pose_refine_np import LAMBDA0, LAMBDA_MAX, LAMBDA_MIN, REL_DECREASE
from tests.refine_homography_np import solve_damped, tinv, tmat, transform  # noqa: F401 (transform: the tests)

MIN_ROWS = 8


def sampson_sq(F, p1, p2):
    """f_resid_sampson per row, in its operation order"""
    F = np.asarray(F, np.float64).ravel()
    x1, y1, x2, y2 = p1[:, 0], p1[:, 1], p2[:, 0], p2[:, 1]
    rxc = F[0] * x2 + F[3] * y2 + F[6]
    ryc = F[1] * x2 + F[4] * y2 + F[7]
    rwc = F[2] * x2 + F[5] * y2 + F[8]
    r = x1 * rxc + y1 * ryc + rwc
    rx = F[0] * x1 + F[1] * y1 + F[2]
    ry = F[3] * x1 + F[4] * y1 + F[5]
    return r * r / (rxc * rxc + ryc * ryc + rx * rx + ry * ry)


def unit(M):
    M = np.asarray(M, np.float64)
    return M / np.sqrt((M * M).sum())


def cofactor(F):
    """the cofactor matrix, row-major 9-vector (cof F = det(F) F^-T)"""
    f = np.asarray(F, np.float64).ravel()
    return np.array([f[4] * f[8] - f[5] * f[7], f[5] * f[6] - f[3] * f[8], f[3] * f[7] - f[4] * f[6],
                     f[2] * f[7] - f[1] * f[8], f[0] * f[8] - f[2] * f[6], f[1] * f[6] - f[0] * f[7],
                     f[1] * f[5] - f[2] * f[4], f[2] * f[3] - f[0] * f[5], f[0] * f[4] - f[1] * f[3]])


def _smallest_right_sv(F):
    """la.h smallest_right_sv3_fast: the dominant eigenvector of K = C^T C by seven squarings, or None"""
    C = cofactor(F).reshape(3, 3)
    K = C.T @ C
    t = np.trace(K)
    if not 1e-290 < t < 1e290:
        return None
    K = K * np.ldexp(1.0, 1 - np.frexp(t)[1])
    M = K.copy()
    for _ in range(7):
        M = M @ M
    col = 0 if (M[0, 0] >= M[1, 1] and M[0, 0] >= M[2, 2]) else (1 if M[1, 1] >= M[2, 2] else 2)
    v = M[:, col].copy()
    n2 = v @ v
    if not 0.0 < n2 < 1e300:
        return None
    v = v / np.sqrt(n2)
    w = K @ v
    mu = w @ v
    r = w - mu * v
    return v if r @ r <= 1e-29 * mu * mu else None


def rank2(F):
    """la.h enforce_rank2 (enforce_rank2_inl): F - (F v) v^T with v the right singular vector of the smallest singular
    value"""
    F = np.asarray(F, np.float64).reshape(3, 3)
    v = _smallest_right_sv(F)
    if v is None:
        v = np.linalg.svd(F)[2][2]
    return (F - np.outer(F @ v, v)).ravel()


def to_pixels(T1, T2, Fn):
    """F = T2^T Fn T1 (row-major 9-vectors)"""
    return (tmat(T2).T @ np.asarray(Fn).reshape(3, 3) @ tmat(T1)).ravel()


def start(T1, T2, F):
    """Fn0 = unit(rank2(T2^-T F T1^-1))"""
    return unit(rank2(tinv(T2).T @ np.asarray(F, np.float64).reshape(3, 3) @ tinv(T1)))


def householder(m):
    """Q [L, L] = I - 2 v v^T / v^T v, v = e_L - s m, s = -sign(m_L-1) (-1 at 0): Q e_L = s m, so the first L - 1
    columns are an orthonormal basis of the complement of the unit vector m"""
    m = np.asarray(m, np.float64)
    s = -1.0 if m[-1] >= 0 else 1.0
    v = -s * m
    v[-1] = 1.0 - s * m[-1]
    return np.eye(len(m)) - 2.0 * np.outer(v, v) / (v @ v)


def basis(Fn):
    """B [9, 7]: the first reflection maps e_9 to +-vec(Fn); inside its 8 columns B1 the second maps e_8 to +-a, the
    coordinates a = B1^T c of the unit cofactor vector c; B = B1 Q2[:, :7]"""
    B1 = householder(Fn)[:, :8]
    c = unit(cofactor(Fn))
    a = unit(B1.T @ c)
    return B1 @ householder(a)[:, :7]


def retract(Fn, d):
    return unit(rank2(np.asarray(Fn) + basis(Fn) @ d))


def linearise(T1, T2, Fn):
    """F [9] and dF [7, 9] in pixels: dF_k = T2^T B_k T1"""
    B = basis(Fn)
    return to_pixels(T1, T2, Fn), np.stack([to_pixels(T1, T2, B[:, k]) for k in range(7)])


def residuals(F, p1, p2):
    """the signed Sampson residual r per row"""
    F = np.asarray(F, np.float64).reshape(3, 3)
    h1, h2 = np.c_[p1[:, :2], np.ones(len(p1))], np.c_[p2[:, :2], np.ones(len(p2))]
    a, b = h1 @ F.T, h2 @ F
    return (h2 * a).sum(1) / np.sqrt(a[:, 0] ** 2 + a[:, 1] ** 2 + b[:, 0] ** 2 + b[:, 1] ** 2)


def jacobian(F, dF, p1, p2):
    """r [n] and J [n, 7] = dr / d(d_k): dc_k / sqrt(s) - r (ds_k / 2) / s"""
    F = np.asarray(F, np.float64).reshape(3, 3)
    h1, h2 = np.c_[p1[:, :2], np.ones(len(p1))], np.c_[p2[:, :2], np.ones(len(p2))]
    a, b = h1 @ F.T, h2 @ F
    s = a[:, 0] ** 2 + a[:, 1] ** 2 + b[:, 0] ** 2 + b[:, 1] ** 2
    r = (h2 * a).sum(1) / np.sqrt(s)
    J = np.empty((len(p1), 7))
    for k in range(7):
        D = dF[k].reshape(3, 3)
        u, v = h1 @ D.T, h2 @ D
        hs = a[:, 0] * u[:, 0] + a[:, 1] * u[:, 1] + b[:, 0] * v[:, 0] + b[:, 1] * v[:, 1]
        J[:, k] = (h2 * u).sum(1) / np.sqrt(s) - r * hs / s
    return r, J


def normal_equations(T1, T2, Fn, p1, p2):
    F, dF = linearise(T1, T2, Fn)
    r, J = jacobian(F, dF, p1, p2)
    return float(sampson_sq(F, p1, p2).sum()), J.T @ J, J.T @ r


def output(T1, T2, Fn, F_in):
    """F = T2^T Fn T1 at unit Frobenius norm, signed so that <F, F_in> >= 0"""
    F = unit(to_pixels(T1, T2, Fn)).reshape(3, 3)
    return -F if (F * np.asarray(F_in).reshape(3, 3)).sum() < 0 else F


def has_model(F):
    F = np.asarray(F, np.float64)
    return bool(F.any() and np.isfinite(F).all())


def refine_pair(F, p1, p2, max_iters=10):
    """One pair over the rows given (already masked).  dict of F (unit norm, rank 2, <F, F_in> >= 0), cost0, cost,
    n_used, iters, accepted and Fn (the final normalised model)."""
    n = len(p1)
    if not has_model(F):
        return dict(F=np.zeros((3, 3)), cost0=np.nan, cost=np.nan, n_used=0, iters=0, accepted=0, Fn=None)
    T1, T2 = transform(p1), transform(p2)
    Fn = start(T1, T2, F)
    C, JJ, Jr = normal_equations(T1, T2, Fn, p1, p2)
    cost0, lam, iters, accepted = C, LAMBDA0, 0, 0
    while n >= MIN_ROWS and iters < max_iters:
        iters += 1
        D = solve_damped(JJ, Jr, lam)
        better = flat = False
        if D is not None:
            Fn2 = retract(Fn, D)
            C2, JJ2, Jr2 = normal_equations(T1, T2, Fn2, p1, p2)
            better, flat = C2 < C, abs(C - C2) < REL_DECREASE * C
        if better:
            Fn, C, JJ, Jr = Fn2, C2, JJ2, Jr2
            lam = max(lam / 10.0, LAMBDA_MIN)
            accepted += 1
        else:
            lam *= 10.0
        if flat or lam > LAMBDA_MAX:
            break
    return dict(F=output(T1, T2, Fn, F), cost0=cost0, cost=C, n_used=n, iters=iters, accepted=accepted, Fn=Fn)


def refine_ragged(F, p1, p2, offsets, mask=None, max_iters=10, px_th=None):
    """The whole batch: dict of F [P,3,3], cost0, cost [P], n_used, iters [P] and, with px_th, inliers [rows] (False
    outside any valid pair) and r2 [rows], the Sampson error behind it (NaN outside)."""
    F = np.asarray(F, np.float64).reshape(-1, 3, 3)
    P, rows = len(F), len(p1)
    out = dict(F=np.zeros((P, 3, 3)), cost0=np.full(P, np.nan), cost=np.full(P, np.nan), n_used=np.zeros(P, np.int64),
               iters=np.zeros(P, np.int64), inliers=np.zeros(rows, bool), r2=np.full(rows, np.nan))
    for p in range(P):
        a, b = int(offsets[p]), int(offsets[p + 1])
        if not 0 <= a <= b <= rows:
            continue
        mk = np.ones(b - a, bool) if mask is None else np.asarray(mask[a:b], bool)
        o = refine_pair(F[p], p1[a:b][mk], p2[a:b][mk], max_iters)
        for k in ("F", "cost0", "cost", "n_used", "iters"):
            out[k][p] = o[k]
        if px_th is not None and o["Fn"] is not None:
            with np.errstate(all="ignore"):
                out["r2"][a:b] = sampson_sq(o["F"], p1[a:b], p2[a:b])
            out["inliers"][a:b] = out["r2"][a:b] <= px_th * px_th
    return out
