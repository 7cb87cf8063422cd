"""numpy restatement of matching.find_absolute_pose_ragged -- TEST INFRASTRUCTURE ONLY.

The estimator's contract (include/degensac_b200.h) written out literally:
  * usable rows: mask set and five finite coordinates, listed in row order; fewer than 4: no model;
  * iteration k = 1, 2, ...: Philox minimal sample of 3 list entries (csrc/rng.h), Lambda Twist P3P on the unit bearings
    normalize(K^-1 [x, y, 1]) (csrc/p3p.h, restated here line by line with Python floats, so the two agree to the bit);
  * MSAC cost sum min(e^2, th^2) (th^2 behind the camera), strict improvement only, the N_req stopping rule;
  * local optimisation: up to 3 rounds of Levenberg-Marquardt on the inliers (the schedule of
    pose_refine_ragged_kernel) and re-selection, kept when its MSAC cost is <= the RANSAC pose's.

tests/test_absolute_pose.py pins P3P to cv2.solveP3P, the Jacobian to central differences, the LM to
scipy.optimize.least_squares and the sampling to the host build of csrc/rng.h."""
import math

import numpy as np

from tests.pose_refine_np import LAMBDA0, LAMBDA_MIN, LAMBDA_MAX, REL_DECREASE, ORTHO_TOL, orthonormalise, rodrigues

MIN_ROWS, LO_ROUNDS = 4, 3
CUBIC_ITERS, NEWTON_ITERS, P3P_ORTHO_TOL, P3P_DEGENERATE = 50, 5, 1e-6, 1e-20
TIE_REL = 1e-12


# ------------------------------------------------------------------------------------------------ Philox (csrc/rng.h)
def philox4x32_10(c, k):
    c0, c1, c2, c3 = c
    k0, k1 = k
    M = 0xFFFFFFFF
    for _ in range(10):
        p0 = 0xD2511F53 * c0
        p1 = 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & M, p1 & M, ((p0 >> 32) ^ c3 ^ k1) & M, p0 & M
        k0 = (k0 + 0x9E3779B9) & M
        k1 = (k1 + 0xBB67AE85) & M
    return c0, c1, c2, c3


def minimal_sample(seed, k, n, m=3):
    """dg::minimal_sample<m>: m distinct indices in [0, n) in draw order (partial Fisher-Yates over a virtual pool)"""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    r = philox4x32_10((0, int(k) & 0xFFFFFFFF, 0, 0), (seed & 0xFFFFFFFF, seed >> 32))
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


# ------------------------------------------------------------------------------------------------ Lambda Twist (p3p.h)
def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _root2(b, c):
    v = b * b - 4.0 * c
    if not v >= 0.0:
        return None
    y = math.sqrt(v)
    q = -0.5 * (b - y) if b < 0.0 else -0.5 * (b + y)
    return q, (c / q if q != 0.0 else 0.0)


def _div(a, b):
    """IEEE a / b (Python raises on a zero divisor)"""
    if b != 0.0:
        return a / b
    if a != a or a == 0.0:
        return math.nan
    return math.copysign(math.inf, a) * math.copysign(1.0, b)


def _sqrt(v):
    return math.sqrt(v) if v >= 0.0 else (math.inf if v == math.inf else math.nan)


def cubic_root(b, c, d):
    if b * b >= 3.0 * c:
        v = _sqrt(b * b - 3.0 * c)
        t1 = _div(-b - v, 3.0)
        k1 = ((t1 + b) * t1 + c) * t1 + d
        if k1 > 0.0:
            r = t1 - _sqrt(_div(-k1, 3.0 * t1 + b))
        else:
            t2 = _div(-b + v, 3.0)
            k2 = ((t2 + b) * t2 + c) * t2 + d
            r = t2 + _sqrt(_div(-k2, 3.0 * t2 + b))
    else:
        r = _div(-b, 3.0)
        if abs((3.0 * r + 2.0 * b) * r + c) < 1e-4:
            r += 1.0
    for i in range(CUBIC_ITERS):
        f = ((r + b) * r + c) * r + d
        if i >= 7 and not abs(f) > 1e-13:
            break
        fp = (3.0 * r + 2.0 * b) * r + c
        r -= _div(f, fp)
    return r


def refine_depths(l, a12, a13, a23, b12, b13, b23):
    l = list(l)
    for _ in range(NEWTON_ITERS):
        l1, l2, l3 = l
        r1 = l1 * l1 + l2 * l2 + b12 * l1 * l2 - a12
        r2 = l1 * l1 + l3 * l3 + b13 * l1 * l3 - a13
        r3 = l2 * l2 + l3 * l3 + b23 * l2 * l3 - a23
        if r1 == 0.0 and r2 == 0.0 and r3 == 0.0:
            break
        p, q = 2.0 * l1 + b12 * l2, 2.0 * l2 + b12 * l1
        r, s = 2.0 * l1 + b13 * l3, 2.0 * l3 + b13 * l1
        u, w = 2.0 * l2 + b23 * l3, 2.0 * l3 + b23 * l2
        det = -(p * s * u) - q * r * w
        if det == 0.0:
            break
        d1 = (-(s * u) * r1 - q * w * r2 + q * s * r3) / det
        d2 = (-(r * w) * r1 + p * w * r2 - p * s * r3) / det
        d3 = (r * u * r1 - p * u * r2 - q * r * r3) / det
        n1, n2, n3 = l1 - d1, l2 - d2, l3 - d3
        if not abs(n1) + abs(n2) + abs(n3) < math.inf:
            break
        l = [n1, n2, n3]
    return l


def eig_rank2(A):
    a00, a01, a02, a11, a12, a22 = A
    b = -a00 - a11 - a22
    c = -(a01 * a01) - a02 * a02 - a12 * a12 + a00 * (a11 + a22) + a11 * a22
    roots = _root2(b, c)
    if roots is None:
        return None
    x1, x2 = roots
    if abs(x1) < abs(x2):
        x1, x2 = x2, x1
    pr0, pr1 = a01 * a12 - a02 * a11, a01 * a02 - a00 * a12
    vs = []
    for e in (x1, x2):
        det = e * e - e * (a00 + a11) + a00 * a11 - a01 * a01
        c1, c2 = _div(e * a02 + pr0, det), _div(e * a12 + pr1, det)
        inv = _div(1.0, _sqrt(c1 * c1 + c2 * c2 + 1.0))
        vs.append([c1 * inv, c2 * inv, inv])
    return vs[0], vs[1], x1, x2


def _finite(v):
    return abs(v) < math.inf


def p3p(y, X):
    """Lambda Twist: the poses (R [3,3], t [3]) with x ~ R X + t of unit bearings y [3][3] and world points X [3][3]"""
    y1, y2, y3 = [list(map(float, v)) for v in y]
    x1, x2, x3 = [list(map(float, v)) for v in X]
    b12, b13, b23 = -2.0 * _dot(y1, y2), -2.0 * _dot(y1, y3), -2.0 * _dot(y2, y3)
    d12 = [x1[i] - x2[i] for i in range(3)]
    d13 = [x1[i] - x3[i] for i in range(3)]
    d23 = [x2[i] - x3[i] for i in range(3)]
    dx = _cross(d12, d13)
    a12, a13, a23 = _dot(d12, d12), _dot(d13, d13), _dot(d23, d23)
    vol = _dot(y1, _cross(y2, y3))
    if not _dot(dx, dx) > P3P_DEGENERATE * a12 * a13 or not vol * vol > P3P_DEGENERATE:
        return []
    c31, c23, c12 = -0.5 * b13, -0.5 * b23, -0.5 * b12
    blob = c12 * c23 * c31 - 1.0
    s31, s23, s12 = 1.0 - c31 * c31, 1.0 - c23 * c23, 1.0 - c12 * c12
    p3 = a13 * (a23 * s31 - a13 * s23)
    p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23 + a23 * (a23 - a12) * s31
    p1 = a23 * (a13 - a23) * s12 - a12 * a12 * s23 - 2.0 * a12 * (blob * a23 + a13 * s23)
    p0 = a12 * (a12 * s23 - a23 * s12)
    if abs(p3) >= abs(p0):
        g = cubic_root(_div(p2, p3), _div(p1, p3), _div(p0, p3))
    else:
        g = _div(1.0, cubic_root(_div(p1, p0), _div(p2, p0), _div(p3, p0)))
    A = (a23 * (1.0 - g), a23 * b12 * 0.5, a23 * b13 * g * -0.5, a23 - a12 + a13 * g, b23 * (a13 * g - a12) * 0.5,
         g * (a13 - a23) - a12)
    eig = eig_rank2(A)
    if eig is None:
        return []
    v1, v2, e1, e2 = eig
    q = _div(-e2, e1)
    sv = math.sqrt(q) if q > 0.0 else 0.0             # sqrt(fmax(0, q))
    L = []
    for s in (sv, -sv):
        w2 = _div(1.0, s * v2[0] - v1[0])
        w0 = (v1[1] - s * v2[1]) * w2
        w1 = (v1[2] - s * v2[2]) * w2
        ia = _div(1.0, (a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12)
        qb = (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13)) * ia
        qc = ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13) * ia
        taus = _root2(qb, qc)
        if taus is None:
            continue
        for tau in taus:
            if not tau > 0.0:
                continue
            d = _div(a23, tau * (b23 + tau) + 1.0)
            if not d > 0.0:
                continue
            l2 = math.sqrt(d)
            l3 = tau * l2
            l1 = w0 * l2 + w1 * l3
            if not l1 > 0.0:
                continue
            L.append([l1, l2, l3])
    Xi = _cross(d13, dx) + _cross(dx, d12) + _cross(d12, d13)
    det = _dot(d12, Xi[:3])
    Xi = [_div(v, det) for v in Xi]
    out = []
    for l0 in L:
        l = refine_depths(l0, a12, a13, a23, b12, b13, b23)
        if not (l[0] > 0.0 and l[1] > 0.0 and l[2] > 0.0):
            continue
        yd1 = [y1[i] * l[0] - y2[i] * l[1] for i in range(3)]
        yd2 = [y1[i] * l[0] - y3[i] * l[2] for i in range(3)]
        yx = _cross(yd1, yd2)
        R = [[yd1[i] * Xi[j] + yd2[i] * Xi[3 + j] + yx[i] * Xi[6 + j] for j in range(3)] for i in range(3)]
        t = [y1[i] * l[0] - (R[i][0] * x1[0] + R[i][1] * x1[1] + R[i][2] * x1[2]) for i in range(3)]
        ok = all(_finite(v) for row in R for v in row) and all(_finite(v) for v in t)
        for i in range(3):
            for j in range(i, 3):
                v = R[i][0] * R[j][0] + R[i][1] * R[j][1] + R[i][2] * R[j][2] - (1.0 if i == j else 0.0)
                ok = ok and abs(v) <= P3P_ORTHO_TOL
        if ok:
            out.append((np.array(R), np.array(t)))
    return out


# ------------------------------------------------------------------------------------------------ absolute_pose.h
def inv3(K):
    """K^-1 by the adjugate, in the operation order of ap_inv3"""
    K = [float(v) for v in np.asarray(K, np.float64).ravel()]
    c0, c1, c2 = [K[0], K[3], K[6]], [K[1], K[4], K[7]], [K[2], K[5], K[8]]
    Ki = _cross(c1, c2) + _cross(c2, c0) + _cross(c0, c1)
    det = c0[0] * Ki[0] + c0[1] * Ki[1] + c0[2] * Ki[2]
    return np.array([v / det for v in Ki]).reshape(3, 3)


def bearing(Ki, x, y):
    b = [Ki[i, 0] * x + Ki[i, 1] * y + Ki[i, 2] for i in range(3)]
    inv = 1.0 / math.sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2])
    return [v * inv for v in b]


def camera(R, t, X):
    """R X + t per row, in the operation order of ap_camera"""
    return np.stack([R[i, 0] * X[:, 0] + R[i, 1] * X[:, 1] + R[i, 2] * X[:, 2] + t[i] for i in range(3)], 1)


def residual(R, t, K, x, X):
    """pixel residuals [n,2] and depths [n] per row (ap_residual)"""
    p = camera(R, t, X)
    q = [K[i, 0] * p[:, 0] + K[i, 1] * p[:, 1] + K[i, 2] * p[:, 2] for i in range(3)]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.stack([q[0] / q[2] - x[:, 0], q[1] / q[2] - x[:, 1]], 1), p[:, 2]


def msac(R, t, K, x, X, th2):
    """per row: the MSAC term min(e^2, th^2) (th^2 behind the camera or for a NaN e^2) and the inlier flag"""
    r, z = residual(R, t, K, x, X)
    e2 = r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]
    front = z > 0.0
    with np.errstate(invalid="ignore"):
        return np.where(front, np.fmin(e2, th2), th2), front & (e2 <= th2)


def jacobian(R, t, K, x, X):
    """r [n,2] and J [n,2,6] by (w, d) at zero for R <- exp([w]x) R, t <- t + d (ap_jacobian)"""
    g = np.stack([R[i, 0] * X[:, 0] + R[i, 1] * X[:, 1] + R[i, 2] * X[:, 2] for i in range(3)], 1)
    p = g + t
    q = [K[i, 0] * p[:, 0] + K[i, 1] * p[:, 1] + K[i, 2] * p[:, 2] for i in range(3)]
    iz = 1.0 / q[2]
    u, v = q[0] * iz, q[1] * iz
    r = np.stack([u - x[:, 0], v - x[:, 1]], 1)
    Du = np.stack([(K[0, j] - u * K[2, j]) * iz for j in range(3)], 1)
    Dv = np.stack([(K[1, j] - v * K[2, j]) * iz for j in range(3)], 1)
    J = np.zeros((len(x), 2, 6))
    for a, D in enumerate((Du, Dv)):
        J[:, a, 0] = D[:, 2] * g[:, 1] - D[:, 1] * g[:, 2]
        J[:, a, 1] = D[:, 0] * g[:, 2] - D[:, 2] * g[:, 0]
        J[:, a, 2] = D[:, 1] * g[:, 0] - D[:, 0] * g[:, 1]
        J[:, a, 3:] = D
    return r, J


def row_sums(R, t, K, x, X):
    """[28] (cost, J^T J upper triangle by rows, J^T r): the sums of ap_row over the rows"""
    r, J = jacobian(R, t, K, x, X)
    H = np.einsum("nai,naj->ij", J, J)
    g = np.einsum("nai,na->i", J, r)
    return np.r_[(r * r).sum(), H[np.triu_indices(6)], g]


def solve_damped(H, g, lam):
    """D of (H + lam diag(H)) D = -g by Cholesky (pr_cholesky_solve), or None at a pivot that is not positive"""
    n = len(g)
    M = H + lam * np.diag(np.diag(H))
    L = np.zeros((n, n))
    for j in range(n):
        d = M[j, j] - L[j, :j] @ L[j, :j]
        if not d > 0.0:
            return None
        L[j, j] = np.sqrt(d)
        for i in range(j + 1, n):
            L[i, j] = (M[i, j] - L[i, :j] @ L[j, :j]) / L[j, j]
    y = np.zeros(n)
    for i in range(n):
        y[i] = (-g[i] - L[i, :i] @ y[:i]) / L[i, i]
    D = np.zeros(n)
    for i in range(n - 1, -1, -1):
        D[i] = (y[i] - L[i + 1:, i] @ D[i + 1:]) / L[i, i]
    return D


def step(R, t, D):
    return rodrigues(D[:3]) @ R, t + D[3:]


def _unpack(s):
    H = np.zeros((6, 6))
    H[np.triu_indices(6)] = s[1:22]
    return H + np.triu(H, 1).T, s[22:]


def lm(R, t, K, x, X, max_iters):
    """Levenberg-Marquardt on sum |r|^2 over the rows given, the schedule of pose_refine_ragged_kernel:
    (R, t, trial steps, accepted steps)"""
    cur = row_sums(R, t, K, x, X)
    lam, it, accepted = LAMBDA0, 0, 0
    while it < max_iters:
        it += 1
        H, g = _unpack(cur)
        D = solve_damped(H, g, lam)
        better = flat = False
        if D is not None:
            R2, t2 = step(R, t, D)
            trial = row_sums(R2, t2, K, x, X)
            better = trial[0] < cur[0]
            flat = abs(cur[0] - trial[0]) < REL_DECREASE * cur[0]
        if better:
            R, t, cur = R2, t2, trial
            lam = max(lam / 10.0, LAMBDA_MIN)
            accepted += 1
            if flat:
                break
        else:
            lam *= 10.0
            if flat or lam > LAMBDA_MAX:
                break
    if accepted and np.abs(R @ R.T - np.eye(3)).max() > ORTHO_TOL:
        R = orthonormalise(R)
    return R, t, it, accepted


def required_iters(has_best, inl, n, conf, max_iters, k):
    if not has_best or conf >= 1.0:
        return max_iters
    if inl >= n:
        return k
    w = inl / n
    with np.errstate(divide="ignore"):
        q = np.ceil(np.log(1.0 - conf) / np.log1p(-(w * w * w)))
    return int(q) if q < max_iters else max_iters


def usable(x, X, mask=None):
    ok = np.isfinite(x).all(1) & np.isfinite(X).all(1)
    if mask is not None:
        ok &= np.asarray(mask).astype(bool)
    return ok


def absolute_pose(x, X, K, mask=None, px_th=2.0, conf=0.999, max_iters=10000, seed=0, refine_iters=10):
    """One pair.  Returns a dict: R, t, mask (over the given rows), n_inliers, iters, cost0, cost; near_tie: a strict
    hypothesis other than the best, with other inliers or a pose more than 1e-9 away, has a cost within 1e-12 of the
    best's, so that summation order may pick either;
    lo_tie: the same for the LO's acceptance; lo_rounds: the LO rounds run."""
    x, X, K = np.asarray(x, np.float64), np.asarray(X, np.float64), np.asarray(K, np.float64)
    rows = len(x)
    lst = np.flatnonzero(usable(x, X, mask))
    n = len(lst)
    out = dict(R=np.zeros((3, 3)), t=np.zeros(3), mask=np.zeros(rows, bool), n_inliers=0, iters=0, cost0=np.nan,
               cost=np.nan, near_tie=False, lo_tie=False, lo_rounds=0)
    if n < MIN_ROWS:
        return out
    xs, Xs = x[lst], X[lst]
    th2 = float(px_th) * float(px_th)
    Ki = inv3(K)
    best = None                                      # (cost, inliers, R, t)
    seen = []
    k = 0
    while True:
        k += 1
        sel = minimal_sample(seed, k, n)
        y = [bearing(Ki, xs[j, 0], xs[j, 1]) for j in sel]
        for R, t in p3p(y, Xs[sel]):
            terms, inl = msac(R, t, K, xs, Xs, th2)
            c = float(terms.sum())
            seen.append((c, int(inl.sum()), R, t))
            if best is None or c < best[0]:
                best = seen[-1]
        req = required_iters(best is not None, best[1] if best else 0, n, conf, max_iters, k)
        if not k < req:
            break
    out["iters"] = k
    if best is None:
        return out
    # another hypothesis within 1e-12 of the best cost, with other inliers or a pose more than 1e-9 away: summation
    # order may pick either
    out["near_tie"] = any(h is not best and abs(h[0] - best[0]) <= TIE_REL * abs(best[0]) and
                          (h[1] != best[1] or np.abs(h[2] - best[2]).max() > 1e-9 or
                           np.abs(h[3] - best[3]).max() > 1e-9 * max(1.0, np.abs(best[3]).max())) for h in seen)
    cost0, _, R0, t0 = best
    terms, inl = msac(R0, t0, K, xs, Xs, th2)
    R, t, cost = R0, t0, cost0
    if refine_iters > 0 and inl.sum() >= MIN_ROWS:
        Rc, tc, flags = R0, t0, inl
        for rnd in range(LO_ROUNDS):
            Rc, tc, _, _ = lm(Rc, tc, K, xs[flags], Xs[flags], refine_iters)
            terms, new = msac(Rc, tc, K, xs, Xs, th2)
            out["lo_rounds"] = rnd + 1
            changed = int((new != flags).sum())
            flags = new
            if changed == 0 or new.sum() < MIN_ROWS:
                break
        c = float(terms.sum())
        out["lo_tie"] = abs(c - cost0) <= TIE_REL * abs(cost0)
        if c <= cost0:
            R, t, cost, inl = Rc, tc, c, flags
        else:
            terms, inl = msac(R0, t0, K, xs, Xs, th2)
    m = np.zeros(rows, bool)
    m[lst] = inl
    out.update(R=R, t=t, mask=m, n_inliers=int(inl.sum()), cost0=cost0, cost=cost)
    return out


def absolute_pose_ragged(x, X, K, offsets, mask=None, px_th=2.0, conf=0.999, max_iters=10000, seeds=None,
                         refine_iters=10):
    """The ragged call: per pair the dict of absolute_pose; malformed spans (decreasing, negative, past the rows) get
    no model and iters 0."""
    x, X = np.asarray(x, np.float64), np.asarray(X, np.float64)
    offsets = np.asarray(offsets)
    P = len(offsets) - 1
    K = np.asarray(K, np.float64)
    seeds = np.broadcast_to(np.asarray(seeds if seeds is not None else 0, dtype=np.uint64), (P,))
    res = []
    for p in range(P):
        b, e = int(offsets[p]), int(offsets[p + 1])
        Kp = K[p] if K.ndim == 3 else K
        if not (0 <= b <= e <= len(x)):
            r = absolute_pose(np.zeros((0, 2)), np.zeros((0, 3)), Kp)
            r["span"] = None
        else:
            r = absolute_pose(x[b:e], X[b:e], Kp, None if mask is None else np.asarray(mask)[b:e], px_th, conf,
                              max_iters, int(seeds[p]), refine_iters)
            r["span"] = (b, e)
        res.append(r)
    return res
