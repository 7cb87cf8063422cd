"""numpy restatement of matching.refine_homography_ragged -- TEST INFRASTRUCTURE ONLY.

Levenberg-Marquardt on the engine's Sampson error of a homography, with the pieces of csrc/refine_h.h and the schedule
of h_refine_ragged_kernel (csrc/frontend.cu) written out once more so that the two take the same steps:

    G = H^-1 (image 2 -> image 1), as a 9-vector g column-major (g[i + 3 j] = G_ij), the layout of csrc/hgeom.h
    e = (r1, r2), JJ^T = [[A, B], [B, D]] of h_resid_sampson;  z1 = r1 / sqrt(A),  z2 = (r2 - B / sqrt(A) z1) /
    sqrt(D - B^2 / A),  |z|^2 = the Sampson error
    T1, T2: centroid to the origin, RMS distance sqrt(2), from the masked rows;  M = T1 G T2^-1 / |.|_F
    local step d [8]:  M <- (M + B d) / |M + B d|_F,  B = basis(M) (Householder);  residuals in pixels, G = T1^-1 M T2
    schedule: that of tests/pose_refine_np.py with an 8 x 8 solve and at least 5 rows.

tests/test_refine_homography.py pins the Jacobian to central differences and the result to
scipy.optimize.least_squares."""
import numpy as np

from tests.pose_refine_np import LAMBDA0, LAMBDA_MAX, LAMBDA_MIN, REL_DECREASE

MIN_ROWS = 5


def adjugate(A):
    a = np.asarray(A, np.float64).ravel()
    return np.array([[a[4] * a[8] - a[5] * a[7], a[2] * a[7] - a[1] * a[8], a[1] * a[5] - a[2] * a[4]],
                     [a[5] * a[6] - a[3] * a[8], a[0] * a[8] - a[2] * a[6], a[2] * a[3] - a[0] * a[5]],
                     [a[3] * a[7] - a[4] * a[6], a[1] * a[6] - a[0] * a[7], a[0] * a[4] - a[1] * a[3]]])


def engine_model(H):
    """g [9] = H^-1 column-major, or None when H is all zero, holds a NaN or has no finite inverse"""
    H = np.asarray(H, np.float64).reshape(3, 3)
    if not H.any() or np.isnan(H).any():
        return None
    C = adjugate(H)
    with np.errstate(all="ignore"):
        G = C / (H[0] @ C[:, 0])
    return G.ravel(order="F") if np.isfinite(G).all() else None


def norm_model(H):
    """H / |H|_F with det H > 0"""
    H = np.asarray(H, np.float64).reshape(3, 3)
    H = H / np.sqrt((H * H).sum())
    return -H if np.linalg.det(H) < 0 else H


def public_model(g):
    """the public H (x2 ~ H x1, unit norm, det > 0) of an engine model"""
    return norm_model(adjugate(np.asarray(g).reshape(3, 3, order="F")))


def transform(p):
    """(s, mx, my) of the rows p [n, >=2]: T = [[s, 0, -s mx], [0, s, -s my], [0, 0, 1]]; s = 1 without spread"""
    n = len(p)
    if n == 0:
        return np.array([1.0, 0.0, 0.0])
    mx, my = p[:, 0].sum() / n, p[:, 1].sum() / n
    var = ((p[:, 0] ** 2).sum() + (p[:, 1] ** 2).sum()) / n - mx * mx - my * my
    return np.array([np.sqrt(2.0 / var) if 0.0 < var < np.inf else 1.0, mx, my])


def tmat(T):
    s, mx, my = T
    return np.array([[s, 0.0, -s * mx], [0.0, s, -s * my], [0.0, 0.0, 1.0]])


def tinv(T):
    s, mx, my = T
    return np.array([[1.0 / s, 0.0, mx], [0.0, 1.0 / s, my], [0.0, 0.0, 1.0]])


def to_pixels(T1, T2, M):
    return (tinv(T1) @ np.asarray(M).reshape(3, 3, order="F") @ tmat(T2)).ravel(order="F")


def from_pixels(T1, T2, g):
    M = (tmat(T1) @ np.asarray(g).reshape(3, 3, order="F") @ tinv(T2)).ravel(order="F")
    return M / np.sqrt(M @ M)


def basis(m):
    """B [9, 8]: columns 0..7 of the Householder reflection Q = I - 2 v v^T / v^T v, v = e_9 - s m, s = -sign(m_8)
    (-1 at 0), which maps e_9 to s m: an orthonormal basis of the plane orthogonal to m"""
    m = np.asarray(m, np.float64)
    s = -1.0 if m[8] >= 0 else 1.0
    v = -s * m
    v[8] = 1.0 - s * m[8]
    Q = np.eye(9) - 2.0 * np.outer(v, v) / (v @ v)
    return Q[:, :8]


def step(M, D):
    M2 = np.asarray(M) + basis(M) @ D
    return M2 / np.sqrt(M2 @ M2)


def _terms(g, p1, p2):
    """r1, r2, a, b, c, d, e per row under g (the quantities of h_resid_sampson)"""
    g = np.asarray(g, np.float64)
    x1, y1, x2, y2 = p1[:, 0], p1[:, 1], p2[:, 0], p2[:, 1]
    wz = g[2] * x2 + g[5] * y2 + g[8]
    r1 = g[0] * x2 + g[3] * y2 + g[6] - x1 * wz
    r2 = g[1] * x2 + g[4] * y2 + g[7] - y1 * wz
    return r1, r2, g[0] - g[2] * x1, g[3] - g[5] * x1, -wz, g[1] - g[2] * y1, g[4] - g[5] * y1


def sampson_sq(g, p1, p2):
    """the engine's Sampson error per row, e^T (JJ^T)^-1 e (tests/test_device_leaves.h_sampson64)"""
    r1, r2, a, b, c, d, e = _terms(g, p1, p2)
    A, B, D = a * a + b * b + c * c, a * d + b * e, d * d + e * e + c * c
    return (D * r1 * r1 - 2 * B * r1 * r2 + A * r2 * r2) / (A * D - B * B)


def whitened(g, p1, p2):
    """z [n, 2]"""
    r1, r2, a, b, c, d, e = _terms(g, p1, p2)
    A, B, D = a * a + b * b + c * c, a * d + b * e, d * d + e * e + c * c
    sA = np.sqrt(A)
    be = B / sA
    z1 = r1 / sA
    return np.c_[z1, (r2 - be * z1) / np.sqrt(D - be * be)]


def linearise(T1, T2, M):
    """G [9] and dG [8, 9] in pixels: dG_k = T1^-1 B_k T2"""
    B = basis(M)
    return to_pixels(T1, T2, M), np.stack([to_pixels(T1, T2, B[:, k]) for k in range(8)])


def jacobian(G, dG, p1, p2):
    """z [2n] (z1 of every row, then z2) and J [2n, 8] = dz / d(d_k), by the chain rule through e, A, B, D"""
    r1, r2, a, b, c, d, e = _terms(G, p1, p2)
    A, B, D = a * a + b * b + c * c, a * d + b * e, d * d + e * e + c * c
    sA = np.sqrt(A)
    be = B / sA
    S = D - be * be
    sS = np.sqrt(S)
    z1 = r1 / sA
    z2 = (r2 - be * z1) / sS
    J1, J2 = np.empty((len(p1), 8)), np.empty((len(p1), 8))
    for k in range(8):
        q1, q2, qa, qb, qc, qd, qe = _terms(dG[k], p1, p2)
        dA = 2 * (a * qa + b * qb + c * qc)
        dB = a * qd + d * qa + b * qe + e * qb
        dD = 2 * (d * qd + e * qe + c * qc)
        dz1 = q1 / sA - r1 * dA / (2 * A * sA)
        dbe = dB / sA - B * dA / (2 * A * sA)
        dS = dD - 2 * be * dbe
        J1[:, k] = dz1
        J2[:, k] = (q2 - dbe * z1 - be * dz1) / sS - z2 * dS / (2 * S)
    return np.r_[z1, z2], np.r_[J1, J2]


def normal_equations(T1, T2, M, p1, p2):
    G, dG = linearise(T1, T2, M)
    z, J = jacobian(G, dG, p1, p2)
    return float(sampson_sq(G, p1, p2).sum()), J.T @ J, J.T @ z


def solve_damped(H, g, lam):
    """D of (H + lam diag(H)) D = -g by Cholesky, or None at a non-positive (or NaN) pivot"""
    N = len(g)
    Mx = H + lam * np.diag(np.diag(H))
    L = np.zeros((N, N))
    for j in range(N):
        d = Mx[j, j] - L[j, :j] @ L[j, :j]
        if not d > 0.0:
            return None
        L[j, j] = np.sqrt(d)
        for i in range(j + 1, N):
            L[i, j] = (Mx[i, j] - L[i, :j] @ L[j, :j]) / L[j, j]
    y = np.zeros(N)
    for i in range(N):
        y[i] = (-g[i] - L[i, :i] @ y[:i]) / L[i, i]
    x = np.zeros(N)
    for i in range(N - 1, -1, -1):
        x[i] = (y[i] - L[i + 1:, i] @ x[i + 1:]) / L[i, i]
    return x


def refine_pair(H, p1, p2, max_iters=10):
    """One pair over the rows given (already masked).  dict of H (unit norm, det > 0), cost0, cost, n_used, iters,
    accepted, g (the engine model of the output H) and M (the final normalised model)."""
    g0 = engine_model(H)
    n = len(p1)
    if g0 is None:
        return dict(H=np.zeros((3, 3)), cost0=np.nan, cost=np.nan, n_used=0, iters=0, accepted=0, g=None, M=None)
    T1, T2 = transform(p1), transform(p2)
    M = from_pixels(T1, T2, g0)
    C, JJ, Jz = normal_equations(T1, T2, M, p1, p2)
    cost0, lam, iters, accepted = C, LAMBDA0, 0, 0
    while n >= MIN_ROWS and iters < max_iters:
        iters += 1
        D = solve_damped(JJ, Jz, lam)
        better = flat = False
        if D is not None:
            M2 = step(M, D)
            C2, JJ2, Jz2 = normal_equations(T1, T2, M2, p1, p2)
            better, flat = C2 < C, abs(C - C2) < REL_DECREASE * C
        if better:
            M, C, JJ, Jz = M2, C2, JJ2, Jz2
            lam = max(lam / 10.0, LAMBDA_MIN)
            accepted += 1
        else:
            lam *= 10.0
        if flat or lam > LAMBDA_MAX:
            break
    Hout = public_model(to_pixels(T1, T2, M)) if accepted else norm_model(H)
    return dict(H=Hout, cost0=cost0, cost=C, n_used=n, iters=iters, accepted=accepted, g=engine_model(Hout), M=M)


def refine_ragged(H, p1, p2, offsets, mask=None, max_iters=10, px_th=None):
    """The whole batch: dict of H [P,3,3], cost0, cost [P], n_used, iters [P] and, with px_th, inliers [rows] (False
    outside any valid pair) and r2 [rows], the Sampson error behind it (NaN outside)."""
    H = np.asarray(H, np.float64).reshape(-1, 3, 3)
    P, rows = len(H), len(p1)
    out = dict(H=np.zeros((P, 3, 3)), cost0=np.full(P, np.nan), cost=np.full(P, np.nan), n_used=np.zeros(P, np.int64),
               iters=np.zeros(P, np.int64), inliers=np.zeros(rows, bool), r2=np.full(rows, np.nan))
    for p in range(P):
        a, b = int(offsets[p]), int(offsets[p + 1])
        if not 0 <= a <= b <= rows:
            continue
        mk = np.ones(b - a, bool) if mask is None else np.asarray(mask[a:b], bool)
        o = refine_pair(H[p], p1[a:b][mk], p2[a:b][mk], max_iters)
        for k in ("H", "cost0", "cost", "n_used", "iters"):
            out[k][p] = o[k]
        if px_th is not None and o["g"] is not None:
            with np.errstate(all="ignore"):
                out["r2"][a:b] = sampson_sq(o["g"], p1[a:b], p2[a:b])
            out["inliers"][a:b] = out["r2"][a:b] <= px_th * px_th
    return out
