"""numpy restatement of matching.triangulate_tracks_ragged -- TEST INFRASTRUCTURE ONLY.

The estimator's contract (include/degensac_b200.h) written out literally:
  * usable observations: mask set, camera index in range, finite pixel, registered camera (finite R, t and
    det R > 0.5), listed in row order; fewer than 2: no model;
  * world rays C = -R^T t, d = R^T normalize(K^-1 [x, y, 1]) and the two-ray midpoint hypothesis with its angle gate
    (csrc/triangulate.h, restated here line by line with Python floats, so the two agree to the bit);
  * iteration k: the k-th pair in lexicographic order when the track has at most max_iters pairs, else the Philox
    minimal sample of 2 (csrc/rng.h);
  * MSAC cost sum min(e^2, th^2) (th^2 behind a camera), strict improvement only, the N_req stopping rule with w^2;
  * local optimisation: up to 3 rounds of Levenberg-Marquardt over X on the inliers (the schedule of
    pose_refine_ragged_kernel) and re-selection, kept when its MSAC cost is <= the RANSAC point's.

tests/test_triangulate.py pins the hypothesis to the planted points and cv2.triangulatePoints, the Jacobian to central
differences, the LM to scipy.optimize.least_squares and the host build of csrc/triangulate.h to this file."""
import itertools
import math

import numpy as np

from tests.absolute_pose_np import _cross, _dot, bearing, inv3, minimal_sample
from tests.pose_refine_np import LAMBDA0, LAMBDA_MAX, LAMBDA_MIN, REL_DECREASE

MIN_ROWS, LO_ROUNDS = 2, 3
TIE_REL = 1e-12


# ------------------------------------------------------------------------------------------------ triangulate.h
def camera(R, t, K):
    """One row of the camera table as a dict: R, t, K, Ki, C and ok (tr_camera)"""
    R, t, K = (np.asarray(v, np.float64) for v in (R, t, K))
    Rl = [float(v) for v in R.ravel()]
    tl = [float(v) for v in t.ravel()]
    finite = all(abs(v) < math.inf for v in Rl + tl)
    C = [-(Rl[k] * tl[0] + Rl[3 + k] * tl[1] + Rl[6 + k] * tl[2]) for k in range(3)]
    det = _dot(Rl[0:3], _cross(Rl[3:6], Rl[6:9]))
    return dict(R=R.reshape(3, 3), t=t.reshape(3), K=K.reshape(3, 3), Ki=inv3(K), C=C,
                ok=bool(finite and det > 0.5))


def ray(cam, x, y):
    """d = R^T ap_bearing(K^-1, x, y), in the operation order of tr_ray"""
    b = bearing(cam["Ki"], float(x), float(y))
    R = [float(v) for v in cam["R"].ravel()]
    return [R[k] * b[0] + R[3 + k] * b[1] + R[6 + k] * b[2] for k in range(3)]


def midpoint(Ci, di, Cj, dj, cos_max):
    """tr_midpoint: the point [3] or None"""
    b = _dot(di, dj)
    den = 1.0 - b * b
    if b > cos_max or not den > 0.0:
        return None
    w = [Ci[0] - Cj[0], Ci[1] - Cj[1], Ci[2] - Cj[2]]
    pi, pj = _dot(di, w), _dot(dj, w)
    li, lj = (b * pj - pi) / den, (pj - b * pi) / den
    if not li > 0.0 or not lj > 0.0:
        return None
    return [0.5 * ((Ci[k] + li * di[k]) + (Cj[k] + lj * dj[k])) for k in range(3)]


def residual(Rs, ts, Ks, X, x):
    """pixel residuals [n,2] and depths [n] of point X observed at x [n,2] by cameras (Rs [n,3,3], ts [n,3],
    Ks [n,3,3]), in the operation order of ap_camera / ap_residual"""
    p = [Rs[:, i, 0] * X[0] + Rs[:, i, 1] * X[1] + Rs[:, i, 2] * X[2] + ts[:, i] for i in range(3)]
    q = [Ks[:, i, 0] * p[0] + Ks[:, i, 1] * p[1] + Ks[:, i, 2] * p[2] for i in range(3)]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.stack([q[0] / q[2] - x[:, 0], q[1] / q[2] - x[:, 1]], 1), p[2]


def msac(Rs, ts, Ks, X, x, th2):
    """per observation: the MSAC term min(e^2, th^2) (th^2 behind the camera or for a NaN e^2) and the inlier flag"""
    r, z = residual(Rs, ts, Ks, X, x)
    e2 = r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]
    front = z > 0.0
    with np.errstate(invalid="ignore"):
        return np.where(front, np.fmin(e2, th2), th2), front & (e2 <= th2)


def jacobian(Rs, ts, Ks, X, x):
    """r [n,2] and J [n,2,3] by X (tr_jacobian)"""
    p = [Rs[:, i, 0] * X[0] + Rs[:, i, 1] * X[1] + Rs[:, i, 2] * X[2] + ts[:, i] for i in range(3)]
    q = [Ks[:, i, 0] * p[0] + Ks[:, i, 1] * p[1] + Ks[:, i, 2] * p[2] for i in range(3)]
    iz = 1.0 / q[2]
    u, v = q[0] * iz, q[1] * iz
    r = np.stack([u - x[:, 0], v - x[:, 1]], 1)
    Du = np.stack([(Ks[:, 0, j] - u * Ks[:, 2, j]) * iz for j in range(3)], 1)
    Dv = np.stack([(Ks[:, 1, j] - v * Ks[:, 2, j]) * iz for j in range(3)], 1)
    J = np.stack([np.stack([D[:, 0] * Rs[:, 0, m] + D[:, 1] * Rs[:, 1, m] + D[:, 2] * Rs[:, 2, m] for m in range(3)], 1)
                  for D in (Du, Dv)], 1)
    return r, J


def warp_sum(terms):
    """the kernel's order of a sum over the observations: lane l adds terms l, l + 32, ... in turn, then a butterfly
    over the 32 lanes (terms [n] or [n, m])"""
    terms = np.asarray(terms, np.float64)
    acc = np.zeros((32,) + terms.shape[1:])
    for c in range(0, len(terms), 32):
        blk = terms[c:c + 32]
        acc[:len(blk)] = acc[:len(blk)] + blk
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[np.arange(32) ^ o]
    return acc[0]


def row_terms(Rs, ts, Ks, X, x):
    """[n, 10] per observation: what tr_row adds (cost, J^T J upper triangle by rows, J^T r), in its operation order"""
    r, J = jacobian(Rs, ts, Ks, X, x)
    cols = [r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]]
    cols += [J[:, 0, k] * J[:, 0, l] + J[:, 1, k] * J[:, 1, l] for k in range(3) for l in range(k, 3)]
    cols += [J[:, 0, k] * r[:, 0] + J[:, 1, k] * r[:, 1] for k in range(3)]
    return np.stack(cols, 1)


def row_sums(Rs, ts, Ks, X, x):
    """[10] (cost, J^T J upper triangle by rows, J^T r): the sums of tr_row over the observations, in the kernel's
    order"""
    return warp_sum(row_terms(Rs, ts, Ks, X, x))


def solve3(s, lam):
    """pr_cholesky_solve<3> on the sums s [10] (H upper triangle s[1:7], g s[7:10]) in its operation order: D [3] or
    None at a pivot that is not positive"""
    H, g = [float(v) for v in s[1:7]], [float(v) for v in s[7:10]]
    L = [[0.0] * 3 for _ in range(3)]
    m = 0
    for k in range(3):
        for l in range(k, 3):
            L[l][k] = H[m] + lam * H[m] if l == k else H[m]
            m += 1
    for j in range(3):
        d = L[j][j]
        for k in range(j):
            d -= L[j][k] * L[j][k]
        if not d > 0.0:
            return None
        L[j][j] = math.sqrt(d)
        for i in range(j + 1, 3):
            v = L[i][j]
            for k in range(j):
                v -= L[i][k] * L[j][k]
            L[i][j] = v / L[j][j]
    y = [0.0] * 3
    for i in range(3):
        v = -g[i]
        for k in range(i):
            v -= L[i][k] * y[k]
        y[i] = v / L[i][i]
    D = [0.0] * 3
    for i in range(2, -1, -1):
        v = y[i]
        for k in range(i + 1, 3):
            v -= L[k][i] * D[k]
        D[i] = v / L[i][i]
    return np.array(D)


def _unpack(s):
    H = np.zeros((3, 3))
    H[np.triu_indices(3)] = s[1:7]
    return H + np.triu(H, 1).T, s[7:]


def lm(Rs, ts, Ks, X, x, max_iters):
    """Levenberg-Marquardt on sum |r|^2 over X, the schedule of pose_refine_ragged_kernel: (X, trial steps)"""
    X = np.asarray(X, np.float64)
    cur = row_sums(Rs, ts, Ks, X, x)
    lam, it = LAMBDA0, 0
    while it < max_iters:
        it += 1
        D = solve3(cur, lam)
        better = flat = False
        if D is not None:
            X2 = X + D
            trial = row_sums(Rs, ts, Ks, X2, x)
            better = trial[0] < cur[0]
            flat = abs(cur[0] - trial[0]) < REL_DECREASE * cur[0]
        if better:
            X, cur = X2, trial
            lam = max(lam / 10.0, LAMBDA_MIN)
            if flat:
                break
        else:
            lam *= 10.0
            if flat or lam > LAMBDA_MAX:
                break
    return X, it


def required_iters(s, has_best, inl, n, conf, max_iters, k):
    """required_iters<s> of absolute_pose.h"""
    if not has_best or conf >= 1.0:
        return max_iters
    if inl >= n:
        return k
    w = inl / n
    ws = w
    for _ in range(s - 1):
        ws = ws * w
    with np.errstate(divide="ignore"):
        q = np.ceil(np.log(1.0 - conf) / np.log1p(-ws))
    return int(q) if q < max_iters else max_iters


def pairs(n):
    """the enumeration order: (i, j), i < j < n, lexicographic"""
    return list(itertools.combinations(range(n), 2))


def max_angle(X, centres, cams):
    """the largest atan2(|a x b|, a . b), a = X - C_i, b = X - C_j, over pairs from distinct cameras (0 without one)"""
    best = 0.0
    a = np.asarray(X)[None, :] - np.asarray(centres, np.float64).reshape(-1, 3)
    for i in range(len(a)):
        for j in range(i + 1, len(a)):
            if cams[i] == cams[j]:
                continue
            w = np.cross(a[i], a[j])
            best = max(best, math.atan2(math.sqrt(float(w @ w)), float(a[i] @ a[j])))
    return best


def usable(cams, pts, table, mask=None):
    cams = np.asarray(cams)
    inr = (cams >= 0) & (cams < len(table))
    ok = inr & np.isfinite(pts).all(1)
    ok[inr] &= np.array([table[c]["ok"] for c in cams[inr]], bool)
    if mask is not None:
        ok &= np.asarray(mask).astype(bool)
    return ok


def triangulate_track(cams, pts, table, mask=None, px_th=2.0, min_angle=math.radians(1.5), conf=0.999,
                      max_iters=1000, seed=0, refine_iters=10):
    """One track over the camera table (a list of camera()).  Returns a dict: X, mask (over the given rows), n_inliers,
    iters, cost0, cost, angle; near_tie: a hypothesis other than the best, with other inliers or a point more than
    1e-9 away, has a cost within 1e-12 of the best's, so that summation order may pick either; lo_tie: the same for the
    LO's acceptance.  A best point without inliers is still a model: X and cost0 = n th^2 are kept, angle is 0."""
    cams, pts = np.asarray(cams), np.asarray(pts, np.float64)
    rows = len(pts)
    lst = np.flatnonzero(usable(cams, pts, table, mask))
    n = len(lst)
    nan3 = np.full(3, np.nan)
    out = dict(X=nan3, mask=np.zeros(rows, bool), n_inliers=0, iters=0, cost0=np.nan, cost=np.nan, angle=np.nan,
               near_tie=False, lo_tie=False)
    if n < MIN_ROWS:
        return out
    cs, xs = cams[lst], pts[lst]
    Rs = np.stack([table[c]["R"] for c in cs])
    ts = np.stack([table[c]["t"] for c in cs])
    Ks = np.stack([table[c]["K"] for c in cs])
    centres = [table[c]["C"] for c in cs]
    rays = [ray(table[c], x[0], x[1]) for c, x in zip(cs, xs)]
    th2 = float(px_th) * float(px_th)
    cos_max = math.cos(min_angle)
    M = n * (n - 1) // 2
    enum = M <= max_iters
    kmax = M if enum else max_iters
    order = pairs(n) if enum else None
    best, seen = None, []                          # (cost, inliers, X)
    k = 0
    while True:
        k += 1
        i, j = order[k - 1] if enum else minimal_sample(seed, k, n, 2)
        X = None
        if cs[i] != cs[j]:
            X = midpoint(centres[i], rays[i], centres[j], rays[j], cos_max)
        if X is not None:
            terms, inl = msac(Rs, ts, Ks, X, xs, th2)
            seen.append((float(np.add.accumulate(terms)[-1]), int(inl.sum()), np.array(X)))
            if best is None or seen[-1][0] < best[0]:
                best = seen[-1]
        req = required_iters(2, best is not None, best[1] if best else 0, n, conf, kmax, k)
        if not k < req:
            break
    out["iters"] = k
    if best is None:
        return out
    # (two points without inliers both cost exactly n th^2, in any summation order: not a near tie)
    out["near_tie"] = any(h is not best and abs(h[0] - best[0]) <= TIE_REL * abs(best[0]) and h[1] + best[1] > 0 and
                          (h[1] != best[1] or np.abs(h[2] - best[2]).max() > 1e-9 * max(1.0, np.abs(best[2]).max()))
                          for h in seen)
    cost0, _, X0 = best
    terms, inl = msac(Rs, ts, Ks, X0, xs, th2)
    X, cost = X0, cost0
    if refine_iters > 0 and inl.sum() >= MIN_ROWS:
        Xc, flags = X0, inl
        for _ in range(LO_ROUNDS):
            Xc, _ = lm(Rs[flags], ts[flags], Ks[flags], Xc, xs[flags], refine_iters)
            terms, new = msac(Rs, ts, Ks, Xc, xs, th2)
            changed = int((new != flags).sum())
            flags = new
            if changed == 0 or new.sum() < MIN_ROWS:
                break
        c = float(warp_sum(terms))
        out["lo_tie"] = abs(c - cost0) <= TIE_REL * abs(cost0)
        if c <= cost0:
            X, cost, inl = Xc, c, flags
        else:
            terms, inl = msac(Rs, ts, Ks, X0, xs, th2)
    m = np.zeros(rows, bool)
    m[lst] = inl
    sel = np.flatnonzero(inl)
    out.update(X=np.asarray(X, np.float64), mask=m, n_inliers=int(inl.sum()), cost0=cost0, cost=cost,
               angle=max_angle(X, [centres[s] for s in sel], cs[sel]))
    return out


def triangulate_tracks_ragged(cams, pts, R, t, K, offsets, mask=None, px_th=2.0, min_angle=math.radians(1.5),
                              conf=0.999, max_iters=1000, seeds=None, refine_iters=10):
    """The ragged call: per track the dict of triangulate_track; malformed spans (decreasing, negative, past the rows)
    get no model and iters 0."""
    R, t, K = (np.asarray(v, np.float64) for v in (R, t, K))
    table = [camera(R[c], t[c], K[c] if K.ndim == 3 else K) for c in range(len(R))]
    cams, pts = np.asarray(cams), np.asarray(pts, np.float64)
    offsets = np.asarray(offsets)
    T = len(offsets) - 1
    seeds = np.broadcast_to(np.asarray(seeds if seeds is not None else 0, dtype=np.uint64), (T,))
    res = []
    for j in range(T):
        b, e = int(offsets[j]), int(offsets[j + 1])
        if not (0 <= b <= e <= len(pts)):
            r = triangulate_track(np.zeros(0, np.int32), np.zeros((0, 2)), table)
            r["span"] = None
        else:
            r = triangulate_track(cams[b:e], pts[b:e], table, None if mask is None else np.asarray(mask)[b:e], px_th,
                                  min_angle, conf, max_iters, int(seeds[j]), refine_iters)
            r["span"] = (b, e)
        res.append(r)
    return res
