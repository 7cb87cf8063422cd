"""numpy restatement of matching.refine_pose_ragged -- TEST INFRASTRUCTURE ONLY.

Levenberg-Marquardt on the pixel-domain Sampson residual over the 5-parameter essential manifold, with the schedule of
pose_refine_ragged_kernel (csrc/frontend.cu) written out once more so that the two take the same steps:

    F = K2^-T [t]x R K1^-1,   r_i = (p2^T F p1) / sqrt((F p1)_0^2 + (F p1)_1^2 + (F^T p2)_0^2 + (F^T p2)_1^2)
    local step (w, d):  R <- exp([w]x) R,  t <- (t + B d) / |t + B d|,  B = tangent_basis(t)
    lambda = 1e-3;  per trial step: solve (J^T J + lambda diag(J^T J)) D = -J^T r by Cholesky (a non-positive pivot is a
    rejected step); accept when the trial cost is strictly lower (lambda <- max(lambda / 10, 1e-12)), else lambda <- 10
    lambda; stop after max_iters trial steps, after a trial step (accepted or not) whose cost differs from the current
    one by less than 1e-12 of it, or when lambda > 1e8.

tests/test_pose_refine.py pins the Jacobian to central differences and the result to scipy.optimize.least_squares."""
import numpy as np

LAMBDA0, LAMBDA_MIN, LAMBDA_MAX, REL_DECREASE, MIN_ROWS, ORTHO_TOL = 1e-3, 1e-12, 1e8, 1e-12, 6, 1e-12


def skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def rodrigues(w):
    """exp([w]x) = I + (sin a / a) [w]x + (2 sin^2(a/2) / a^2) [w]x^2, a = |w|"""
    a = np.sqrt(w @ w)
    W = skew(w)
    if a == 0.0:
        c1, c2 = 1.0, 0.5
    else:
        h = np.sin(0.5 * a) / a
        c1, c2 = np.sin(a) / a, 2.0 * h * h
    return np.eye(3) + c1 * W + c2 * (W @ W)


def tangent_basis(t):
    """B [3,2]: orthonormal basis of the plane orthogonal to t, from the coordinate axis of t's smallest |component|
    (the first such axis on ties): b1 = t x e / |t x e|, b2 = t x b1 / |t x b1|"""
    e = np.zeros(3)
    e[int(np.argmin(np.abs(t)))] = 1.0
    b1 = np.cross(t, e)
    b1 = b1 / np.sqrt(b1 @ b1)
    b2 = np.cross(t, b1)
    b2 = b2 / np.sqrt(b2 @ b2)
    return np.c_[b1, b2]


def fundamental(R, t, K1, K2):
    return np.linalg.inv(K2).T @ skew(t) @ R @ np.linalg.inv(K1)


def linearise(R, t, K1, K2):
    """F and the five dF / d(theta_k) at theta = 0: three rotation axes, then the two columns of tangent_basis(t)"""
    A, Bk = np.linalg.inv(K2).T, np.linalg.inv(K1)
    T, B = skew(t), tangent_basis(t)
    dE = [T @ skew(np.eye(3)[k]) @ R for k in range(3)] + [skew(B[:, j]) @ R for j in range(2)]
    return A @ T @ R @ Bk, np.stack([A @ d @ Bk for d in dE])


def _hom(p):
    return np.c_[p[:, :2], np.ones(len(p))]


def sampson_sq(F, p1, p2):
    """r^2 per row, in the operation order of f_resid_sampson (csrc/fgeom.h)"""
    x1, y1, x2, y2 = p1[:, 0], p1[:, 1], p2[:, 0], p2[:, 1]
    F = np.asarray(F, np.float64).ravel()
    rxc = F[0] * x2 + F[3] * y2 + F[6]
    ryc = F[1] * x2 + F[4] * y2 + F[7]
    rwc = F[2] * x2 + F[5] * y2 + F[8]
    r = x1 * rxc + y1 * ryc + rwc
    rx = F[0] * x1 + F[1] * y1 + F[2]
    ry = F[3] * x1 + F[4] * y1 + F[5]
    return r * r / (rxc * rxc + ryc * ryc + rx * rx + ry * ry)


def residuals(F, p1, p2):
    """the signed Sampson residual r per row"""
    h1, h2 = _hom(p1), _hom(p2)
    a, b = h1 @ F.T, h2 @ F                       # rows F p1, F^T p2
    return (h2 * a).sum(1) / np.sqrt(a[:, 0] ** 2 + a[:, 1] ** 2 + b[:, 0] ** 2 + b[:, 1] ** 2)


def jacobian(F, dF, p1, p2):
    """r [n] and J [n,5]: dr/dtheta_k = (p2^T dF_k p1) / sqrt(s) - c (ds/dtheta_k) / (2 s sqrt(s))"""
    h1, h2 = _hom(p1), _hom(p2)
    a, b = h1 @ F.T, h2 @ F
    c = (h2 * a).sum(1)
    s = a[:, 0] ** 2 + a[:, 1] ** 2 + b[:, 0] ** 2 + b[:, 1] ** 2
    rs = np.sqrt(s)
    J = np.empty((len(h1), 5))
    for k in range(5):
        u, v = h1 @ dF[k].T, h2 @ dF[k]
        half_ds = a[:, 0] * u[:, 0] + a[:, 1] * u[:, 1] + b[:, 0] * v[:, 0] + b[:, 1] * v[:, 1]
        J[:, k] = (h2 * u).sum(1) / rs - c * half_ds / (s * rs)
    return c / rs, J


def _normal_equations(R, t, K1, K2, p1, p2):
    F, dF = linearise(R, t, K1, K2)
    r, J = jacobian(F, dF, p1, p2)
    return float(sampson_sq(F, p1, p2).sum()), J.T @ J, J.T @ r


def solve_damped(H, g, lam):
    """D of (H + lam diag(H)) D = -g by Cholesky, or None at a non-positive (or NaN) pivot"""
    M = H + lam * np.diag(np.diag(H))
    L = np.zeros((5, 5))
    for j in range(5):
        d = M[j, j] - L[j, :j] @ L[j, :j]
        if not d > 0.0:
            return None
        L[j, j] = np.sqrt(d)
        for i in range(j + 1, 5):
            L[i, j] = (M[i, j] - L[i, :j] @ L[j, :j]) / L[j, j]
    y = np.zeros(5)
    for i in range(5):
        y[i] = (-g[i] - L[i, :i] @ y[:i]) / L[i, i]
    x = np.zeros(5)
    for i in range(4, -1, -1):
        x[i] = (y[i] - L[i + 1:, i] @ x[i + 1:]) / L[i, i]
    return x


def step(R, t, D):
    t2 = t + tangent_basis(t) @ D[3:]
    return rodrigues(D[:3]) @ R, t2 / np.sqrt(t2 @ t2)


def orthonormalise(R):
    """Gram-Schmidt on the rows, third row their cross product (det +1)"""
    r0 = R[0] / np.sqrt(R[0] @ R[0])
    r1 = R[1] - (r0 @ R[1]) * r0
    r1 = r1 / np.sqrt(r1 @ r1)
    return np.stack([r0, r1, np.cross(r0, r1)])


def unit_frobenius(F):
    n = np.sqrt((F * F).sum())
    return F / n if n > 0 else np.zeros((3, 3))


def refine_pair(R, t, K1, K2, p1, p2, max_iters=10):
    """One pair over the rows given (already masked).  dict of R, t, F (unit Frobenius norm), cost0, cost, n_used,
    iters, accepted (number of accepted steps)."""
    R, t = np.array(R, np.float64).reshape(3, 3), np.array(t, np.float64).ravel()
    n = len(p1)
    if not R.any() or np.isnan(R).any() or np.isnan(t).any():
        return dict(R=np.zeros((3, 3)), t=np.zeros(3), F=np.zeros((3, 3)), cost0=np.nan, cost=np.nan, n_used=0, iters=0,
                    accepted=0)
    C, H, g = _normal_equations(R, t, K1, K2, p1, p2)
    cost0, lam, iters, accepted = C, LAMBDA0, 0, 0
    while n >= MIN_ROWS and iters < max_iters:
        iters += 1
        D = solve_damped(H, g, lam)
        better = flat = False
        if D is not None:
            R2, t2 = step(R, t, D)
            C2, H2, g2 = _normal_equations(R2, t2, K1, K2, p1, p2)
            better, flat = C2 < C, abs(C - C2) < REL_DECREASE * C
        if better:
            R, t, C, H, g = R2, t2, C2, H2, g2
            lam = max(lam / 10.0, LAMBDA_MIN)
            accepted += 1
        else:
            lam *= 10.0
        if flat or lam > LAMBDA_MAX:
            break
    if accepted and np.abs(R @ R.T - np.eye(3)).max() > ORTHO_TOL:
        R = orthonormalise(R)
    return dict(R=R, t=t, F=unit_frobenius(fundamental(R, t, K1, K2)), cost0=cost0, cost=C, n_used=n, iters=iters,
                accepted=accepted)


def refine_ragged(R, t, K1, K2, p1, p2, offsets, mask=None, max_iters=10, px_th=None):
    """The whole batch: dict of R [P,3,3], t [P,3], F [P,3,3], cost0, cost [P], n_used, iters [P] and, with px_th,
    inliers [rows] (False outside any valid pair) and r2 [rows], the squared residual behind it (NaN outside)."""
    R = np.asarray(R, np.float64).reshape(-1, 3, 3)
    P, rows = len(R), len(p1)
    K1 = np.broadcast_to(K1, (P, 3, 3)); K2 = np.broadcast_to(K2, (P, 3, 3))
    out = dict(R=np.zeros((P, 3, 3)), t=np.zeros((P, 3)), F=np.zeros((P, 3, 3)), cost0=np.full(P, np.nan),
               cost=np.full(P, np.nan), n_used=np.zeros(P, np.int64), iters=np.zeros(P, np.int64),
               inliers=np.zeros(rows, bool), r2=np.full(rows, np.nan))
    for p in range(P):
        a, b = int(offsets[p]), int(offsets[p + 1])
        if not 0 <= a <= b <= rows:
            continue
        mk = np.ones(b - a, bool) if mask is None else np.asarray(mask[a:b], bool)
        o = refine_pair(R[p], t[p], K1[p], K2[p], p1[a:b][mk], p2[a:b][mk], max_iters)
        for k in ("R", "t", "F", "cost0", "cost", "n_used", "iters"):
            out[k][p] = o[k]
        if px_th is not None and o["F"].any():
            out["r2"][a:b] = sampson_sq(o["F"], p1[a:b], p2[a:b])
            out["inliers"][a:b] = out["r2"][a:b] <= px_th * px_th
    return out
