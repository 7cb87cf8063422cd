"""numpy oracle of the global positioning (matching.global_positioning_ragged, csrc/global_positioning.cu) -- TEST
INFRASTRUCTURE ONLY.  The estimator of include/degensac_b200.h written out: the usable observations and used tracks,
the components and anchors, the Philox start, the Huber cost and IRLS weights, and Levenberg-Marquardt whose trial
steps go through the nested Schur complement (scales, then points, then the centres by PCG or a dense solve).  The
per-thread functions of csrc/global_positioning.h are restated with the device's operation order (no FMA), so the host
build matches them to the bit; the sums are taken in numpy's order.  dense_step() solves the full damped normal
equations over (c, X, d) directly, the reference the nested Schur step is checked against."""
import math

import numpy as np

from tests.absolute_pose_np import inv3 as k_inverse
from tests.absolute_pose_np import philox4x32_10
from tests.bundle_adjust_np import inv3
from tests.pose_refine_np import LAMBDA0, LAMBDA_MAX, LAMBDA_MIN, REL_DECREASE

D_MIN = 1e-5
KIND_VIEW, KIND_TRACK = 0, 1


# ------------------------------------------------------------------------------------------------ global_positioning.h
def ray(Ki, R, x, y):
    """gp_ray over rows: normalise(R^T Ki (x, y, 1)), Ki and R [n,3,3]"""
    b = [Ki[:, i, 0] * x + Ki[:, i, 1] * y + Ki[:, i, 2] for i in range(3)]
    v = [R[:, 0, k] * b[0] + R[:, 1, k] * b[1] + R[:, 2, k] * b[2] for k in range(3)]
    inv = 1.0 / np.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    return np.stack([v[0] * inv, v[1] * inv, v[2] * inv], -1)


def start(seed, kind, index, init_scale):
    """gp_start: [3]"""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    o = philox4x32_10((0, int(index) & 0xFFFFFFFF, kind, 0), (seed & 0xFFFFFFFF, seed >> 32))
    return np.array([init_scale * (2.0 * ((float(o[k]) + 0.5) * 2.3283064365386963e-10) - 1.0) for k in range(3)])


def residual(c, X, d, v):
    """gp_residual over rows: (a, r, |r|^2)"""
    a = X - c
    r = d[:, None] * a - v
    return a, r, r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2]


def rho(s, delta):
    if delta > 0.0:
        return np.where(s > delta * delta, 2.0 * delta * np.sqrt(s) - delta * delta, s)
    return np.asarray(s, np.float64)


def weight(s, delta):
    if delta > 0.0:
        with np.errstate(divide="ignore"):
            return np.where(s > delta * delta, delta / np.sqrt(s), 1.0)
    return np.ones_like(s)


def obs_terms(a, r, d, w):
    """gp_obs_terms over rows: (ok, u, n, s, h, ar)"""
    na = np.sqrt(a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1] + a[:, 2] * a[:, 2])
    ok = (na > 0.0) & (na < np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / na
    u = a * inv[:, None]
    h = (w * d)[:, None] * r
    s = w * d * d
    ar = a[:, 0] * r[:, 0] + a[:, 1] * r[:, 1] + a[:, 2] * r[:, 2]
    return ok, u, na, s, h, ar


def m_apply(u, s, f, p):
    """gp_m_apply over rows: s (p - f u (u . p))"""
    up = f * (u[:, 0] * p[:, 0] + u[:, 1] * p[:, 1] + u[:, 2] * p[:, 2])
    return s[:, None] * (p - up[:, None] * u)


def block(S, Q, lam):
    """gp_block: [n,6] upper triangles from S [n] and Q [n,6]"""
    f, g = 1.0 / (1.0 + lam), (1.0 + lam) * S
    diag = np.array([1.0, 0.0, 0.0, 1.0, 0.0, 1.0])
    return np.where(diag > 0, g[:, None], 0.0) - f * Q


def outer6(u, s):
    """s u u^T, upper triangle by rows [n,6], in gp_add_outer's order"""
    return np.stack([s * u[:, k] * u[:, l] for k in range(3) for l in range(k, 3)], -1)


def scale_step(ar, n, d, u, dXc, lam):
    """gp_scale_step over rows"""
    ud = u[:, 0] * dXc[:, 0] + u[:, 1] * dXc[:, 1] + u[:, 2] * dXc[:, 2]
    dd = -(ar + d * n * ud) / ((1.0 + lam) * (n * n))
    t = d + dd
    return np.where(t > D_MIN, t, D_MIN)


def angle(v, a):
    """gp_angle over rows"""
    x0 = v[:, 1] * a[:, 2] - v[:, 2] * a[:, 1]
    x1 = v[:, 2] * a[:, 0] - v[:, 0] * a[:, 2]
    x2 = v[:, 0] * a[:, 1] - v[:, 1] * a[:, 0]
    return np.arctan2(np.sqrt(x0 * x0 + x1 * x1 + x2 * x2), v[:, 0] * a[:, 0] + v[:, 1] * a[:, 1] + v[:, 2] * a[:, 2])


def sym(V6):
    """[n,6] upper triangles -> [n,3,3]"""
    i = [[0, 1, 2], [1, 3, 4], [2, 4, 5]]
    return V6[:, i]


# ------------------------------------------------------------------------------------------------ the problem
def setup(cams, pts, R, K, offsets, mask=None):
    """The usable observations and their rays, the used tracks, the components and the views that move"""
    cams = np.asarray(cams, np.int64)
    pts = np.asarray(pts, np.float64).reshape(-1, 2)
    R = np.asarray(R, np.float64).reshape(-1, 3, 3)
    C, obs = len(R), len(cams)
    K = np.asarray(K, np.float64)
    Ks = np.broadcast_to(K.reshape(-1, 3, 3), (C, 3, 3)) if K.ndim == 2 else K.reshape(C, 3, 3)
    offsets = np.asarray(offsets, np.int64)
    T = len(offsets) - 1
    with np.errstate(invalid="ignore"):
        fin = np.isfinite(R).all(axis=(1, 2))
        Rz = np.where(fin[:, None, None], R, 0.0)
        det = np.einsum("ci,ci->c", Rz[:, 0], np.cross(Rz[:, 1], Rz[:, 2]))
    registered = fin & (det > 0.5)
    Ki = np.stack([k_inverse(Ks[c]) for c in range(C)]) if C else np.zeros((0, 3, 3))
    m = np.ones(obs, bool) if mask is None else np.asarray(mask).astype(bool)
    inr = (cams >= 0) & (cams < C)
    cc = np.where(inr, cams, 0)
    usable = m & inr & np.isfinite(pts).all(1) & registered[cc]
    v = np.full((obs, 3), np.nan)
    if usable.any():
        with np.errstate(invalid="ignore"):
            v[usable] = ray(Ki[cc[usable]], R[cc[usable]], pts[usable, 0], pts[usable, 1])
    used = np.zeros(obs, bool)
    track_of = np.full(obs, -1, np.int64)
    trk_used = np.zeros(T, np.int64)
    parent = list(range(C))

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x
    for j in range(T):
        b, e = int(offsets[j]), int(offsets[j + 1])
        if not (0 <= b <= e <= obs):
            continue
        track_of[b:e] = j
        rows = np.arange(b, e)[usable[b:e]]
        if len(set(cams[rows].tolist())) >= 2:
            used[rows] = True
            trk_used[j] = len(rows)
            for r in rows[1:]:
                x, y = find(int(cams[rows[0]])), find(int(cams[r]))
                if x != y:
                    parent[max(x, y)] = min(x, y)
    active = np.zeros(C, bool)
    active[cams[used]] = True
    comp = np.array([find(c) if active[c] else -1 for c in range(C)], np.int64)
    anchor = active & (comp == np.arange(C))
    key = used & ~anchor[cc]
    return dict(cams=cc, R=R, v=v, used=used, track_of=track_of, trk_used=trk_used, active=active, comp=comp,
                anchor=anchor, key=key, C=C, T=T, obs=obs, moving=active & ~anchor)


def start_state(P, seed, init_scale):
    c = np.full((P["C"], 3), np.nan)
    for i in range(P["C"]):
        if P["active"][i]:
            c[i] = 0.0 if P["anchor"][i] else start(seed, KIND_VIEW, i, init_scale)
    X = np.full((P["T"], 3), np.nan)
    for j in range(P["T"]):
        if P["trk_used"][j]:
            X[j] = start(seed, KIND_TRACK, j, init_scale)
    d = np.where(P["used"], 1.0, np.nan)
    return c, X, d


def obs_cost(P, c, X, d, delta):
    """rho per used observation [n_used], +inf where |a| is 0 or not finite (the trial-point rule)"""
    u = np.flatnonzero(P["used"])
    a, r, s2 = residual(c[P["cams"][u]], X[P["track_of"][u]], d[u], P["v"][u])
    na = np.sqrt(a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1] + a[:, 2] * a[:, 2])
    return np.where((na > 0.0) & (na < np.inf), rho(s2, delta), np.inf)


def total_cost(P, c, X, d, delta):
    return float(np.sum(obs_cost(P, c, X, d, delta)))


def linearise(P, c, X, d, delta):
    """The used observations' linearisation: dict(rows, cam, trk, key, u, n, s, h, ar, w, a, r, d) and ok"""
    u_ = np.flatnonzero(P["used"])
    cam, trk = P["cams"][u_], P["track_of"][u_]
    a, r, s2 = residual(c[cam], X[trk], d[u_], P["v"][u_])
    w = weight(s2, delta)
    with np.errstate(invalid="ignore", divide="ignore"):
        ok, u, n, s, h, ar = obs_terms(a, r, d[u_], w)
    return dict(rows=u_, cam=cam, trk=trk, key=P["key"][u_], u=u, n=n, s=s, h=h, ar=ar, w=w, a=a, r=r,
                d=d[u_]), bool(ok.all())


def _seg(idx, v, n):
    out = np.zeros((n,) + v.shape[1:])
    np.add.at(out, idx, v)
    return out


def points(P, L, lam):
    """(Vi [T,3,3], t [T,3]) or None at a non-positive pivot"""
    f = 1.0 / (1.0 + lam)
    T = P["T"]
    S = _seg(L["trk"], L["s"], T)
    Q = _seg(L["trk"], outer6(L["u"], L["s"]), T)
    uh = np.einsum("ni,ni->n", L["u"], L["h"])
    g = _seg(L["trk"], L["h"], T) - f * _seg(L["trk"], L["u"] * uh[:, None], T)
    Vs = sym(block(S, Q, lam))
    Vi = np.zeros((T, 3, 3))
    for j in np.flatnonzero(P["trk_used"]):
        inv = inv3(Vs[j], 0.0)
        if inv is None:
            return None
        Vi[j] = inv
    return Vi, np.einsum("tij,tj->ti", Vi, g)


def _m(L, f):
    """m_o [n,3,3] = s (I - f u u^T)"""
    return L["s"][:, None, None] * (np.eye(3) - f * L["u"][:, :, None] * L["u"][:, None, :])


def reduced(P, L, lam, Vi, t):
    """(U* [C,3,3], M [C,3,3], b [C,3]) over the views that move (others: U* = 0, M = I, b = 0)"""
    f = 1.0 / (1.0 + lam)
    C = P["C"]
    k = L["key"]
    cam, trk = L["cam"][k], L["trk"][k]
    m = _m(L, f)[k]
    S = _seg(cam, L["s"][k], C)
    Q = _seg(cam, outer6(L["u"][k], L["s"][k]), C)
    U = sym(block(S, Q, lam))
    # W_ij = the sum of m over view i's observations of track j, so that M is S's diagonal block
    pair, gi = np.unique(cam * P["T"] + trk, return_inverse=True)
    Wij = _seg(gi.reshape(-1), m, len(pair))
    gc, gt = pair // P["T"], pair % P["T"]
    mvm = _seg(gc, Wij @ Vi[gt] @ Wij, C)
    uh = np.einsum("ni,ni->n", L["u"][k], L["h"][k])
    e = L["h"][k] - f * uh[:, None] * L["u"][k]
    b = _seg(cam, e - np.einsum("nij,nj->ni", m, t[trk]), C)
    mov = np.zeros(C, bool)
    mov[cam] = True
    U[~mov] = 0.0
    M = np.where(mov[:, None, None], U - mvm, np.eye(3))
    b[~mov] = 0.0
    return U, M, b, mov


def schur_matvec(P, L, lam, Vi, U, p):
    f = 1.0 / (1.0 + lam)
    k = L["key"]
    cam, trk = L["cam"][k], L["trk"][k]
    m = _m(L, f)[k]
    y = np.einsum("tij,tj->ti", Vi, _seg(trk, np.einsum("nij,nj->ni", m, p[cam]), P["T"]))
    return np.einsum("cij,cj->ci", U, p) - _seg(cam, np.einsum("nij,nj->ni", m, y[trk]), P["C"])


def pcg(P, L, lam, Vi, U, M, b, cg_tol, cg_max_iters):
    """(x [C,3], iterations, rejected) by the stopping rules of bundle_adjust_pcg; None when M has no Cholesky factor"""
    try:
        Lc = np.linalg.cholesky(M)
    except np.linalg.LinAlgError:
        return None

    def apply_m(r):
        return np.linalg.solve(M, r[..., None])[..., 0]
    del Lc
    x = np.zeros_like(b)
    bb = float(np.sum(b * b))
    if not bb > 0.0:
        return x, 0, False
    r = b.copy()
    z = apply_m(r)
    p = z.copy()
    rho_ = float(np.sum(r * z))
    it = 0
    while True:
        q = schur_matvec(P, L, lam, Vi, U, p)
        kappa = float(np.sum(p * q))
        it += 1
        if not (kappa > 0.0) or not np.isfinite(kappa):
            return x, it, it == 1
        alpha = rho_ / kappa
        x = x + alpha * p
        r = r - alpha * q
        rr = float(np.sum(r * r))
        if rr <= cg_tol * cg_tol * bb or it >= cg_max_iters:
            return x, it, False
        z = apply_m(r)
        rz = float(np.sum(r * z))
        p = z + (rz / rho_) * p
        rho_ = rz


def dense_reduced(P, L, lam, Vi, U, b, mov):
    """dc [C,3] by a dense solve of S dc = b over the views that move"""
    idx = np.flatnonzero(mov)
    n = len(idx)
    Sd = np.zeros((3 * n, 3 * n))
    for q, c in enumerate(idx):
        e = np.zeros((P["C"], 3))
        for k in range(3):
            e[:] = 0.0
            e[c, k] = 1.0
            Sd[:, 3 * q + k] = schur_matvec(P, L, lam, Vi, U, e)[idx].reshape(-1)
    dc = np.zeros((P["C"], 3))
    if n:
        dc[idx] = np.linalg.solve(Sd, b[idx].reshape(-1)).reshape(n, 3)
    return dc


def back_substitute(P, L, lam, Vi, t, dc):
    """(dX [T,3], dXc [n_used,3]: dX_j - dc_i per used observation)"""
    f = 1.0 / (1.0 + lam)
    k = L["key"]
    m = _m(L, f)[k]
    acc = _seg(L["trk"][k], np.einsum("nij,nj->ni", m, dc[L["cam"][k]]), P["T"])
    dX = np.einsum("tij,tj->ti", Vi, acc) - t
    dcx = np.where(k[:, None], dc[L["cam"]], 0.0)
    return dX, dX[L["trk"]] - dcx


def schur_step(P, L, lam, solver="pcg", cg_tol=1e-6, cg_max_iters=500):
    """The nested Schur step: dict(dc, dX, dd (not projected), cg) or None when the step is rejected"""
    pv = points(P, L, lam)
    if pv is None:
        return None
    Vi, t = pv
    U, M, b, mov = reduced(P, L, lam, Vi, t)
    if solver == "dense":
        dc, cgi = dense_reduced(P, L, lam, Vi, U, b, mov), 0
    else:
        out = pcg(P, L, lam, Vi, U, M, b, cg_tol, cg_max_iters)
        if out is None:
            return None
        dc, cgi, rej = out
        if rej:
            return dict(rejected=True, cg=cgi)
    dX, dXc = back_substitute(P, L, lam, Vi, t, dc)
    ud = np.einsum("ni,ni->n", L["u"], dXc)
    dd = -(L["ar"] + L["d"] * L["n"] * ud) / ((1.0 + lam) * (L["n"] * L["n"]))
    return dict(dc=dc, dX=dX, dXc=dXc, dd=dd, cg=cgi, rejected=False)


def dense_step(P, L, lam):
    """The same step from the full damped normal equations over (c of the views that move, X of the used tracks, d of
    the used observations): J = [-d I, d I, a] per observation, H = J^T W J, H* = H + lam diag H, H* x = -J^T W r"""
    mov = np.flatnonzero(P["moving"])
    trk = np.flatnonzero(P["trk_used"])
    ci = {c: q for q, c in enumerate(mov)}
    ti = {j: q for q, j in enumerate(trk)}
    nu = len(L["rows"])
    n = 3 * len(mov) + 3 * len(trk) + nu
    J = np.zeros((3 * nu, n))
    for o in range(nu):
        d, a = L["d"][o], L["a"][o]
        c = int(L["cam"][o])
        if c in ci:
            J[3 * o:3 * o + 3, 3 * ci[c]:3 * ci[c] + 3] = -d * np.eye(3)
        q = 3 * len(mov) + 3 * ti[int(L["trk"][o])]
        J[3 * o:3 * o + 3, q:q + 3] = d * np.eye(3)
        J[3 * o:3 * o + 3, 3 * len(mov) + 3 * len(trk) + o] = a
    W = np.repeat(L["w"], 3)
    H = J.T @ (W[:, None] * J)
    g = J.T @ (W * L["r"].reshape(-1))
    x = np.linalg.solve(H + lam * np.diag(np.diag(H)), -g)
    dc = np.zeros((P["C"], 3))
    dc[mov] = x[:3 * len(mov)].reshape(-1, 3)
    dX = np.zeros((P["T"], 3))
    dX[trk] = x[3 * len(mov):3 * len(mov) + 3 * len(trk)].reshape(-1, 3)
    return dict(dc=dc, dX=dX, dd=x[3 * len(mov) + 3 * len(trk):])


def global_positioning(cams, pts, R, K, offsets, mask=None, seed=0, init_scale=100.0, loss_scale=0.1, max_iters=100,
                       max_angle=math.radians(2.0), cg_max_iters=500, cg_tol=1e-6, solver="pcg", trace=None):
    """The whole estimator: dict(t, X, component, angle, inliers, cost0, cost, iters, n_used, cg_iters, c, d, start).
    trace: a list that gets (lambda, cost) after each trial step"""
    P = setup(cams, pts, R, K, offsets, mask)
    delta = float(loss_scale)
    c, X, d = start_state(P, seed, init_scale)
    st = (c.copy(), X.copy(), d.copy())
    cost = total_cost(P, c, X, d, delta)
    cost0, lam, iters, cg_total = cost, LAMBDA0, 0, 0
    L, lin_ok = linearise(P, c, X, d, delta)
    while iters < max_iters:
        step = schur_step(P, L, lam, solver, cg_tol, cg_max_iters) if lin_ok else None
        go = step is not None and not step["rejected"]
        if step is not None:
            cg_total += step["cg"]
        c_new = cost
        if go:
            c2, X2, d2 = c.copy(), X.copy(), d.copy()
            mov = P["moving"] & (_seg(L["cam"][L["key"]], np.ones(int(L["key"].sum())), P["C"]) > 0)
            c2[mov] = c[mov] + step["dc"][mov]
            tu = P["trk_used"] > 0
            X2[tu] = X[tu] + step["dX"][tu]
            d2[L["rows"]] = scale_step(L["ar"], L["n"], L["d"], L["u"], step["dXc"], lam)
            c_new = total_cost(P, c2, X2, d2, delta)
        iters += 1
        better = go and c_new < cost
        flat = go and abs(cost - c_new) < REL_DECREASE * cost
        if better:
            c, X, d, cost = c2, X2, d2, c_new
            lam = max(lam / 10.0, LAMBDA_MIN)
            L, lin_ok = linearise(P, c, X, d, delta)
            stop = flat
        else:
            lam *= 10.0
            stop = flat or lam > LAMBDA_MAX
        if trace is not None:
            trace.append((lam, cost))
        if stop:
            break
    t = np.full((P["C"], 3), np.nan)
    a_ = P["active"]
    Rr = P["R"]
    for k in range(3):
        t[a_, k] = -(Rr[a_, k, 0] * c[a_, 0] + Rr[a_, k, 1] * c[a_, 1] + Rr[a_, k, 2] * c[a_, 2])
    ang = np.full(P["obs"], np.nan)
    u = np.flatnonzero(P["used"])
    ang[u] = angle(P["v"][u], X[P["track_of"][u]] - c[P["cams"][u]])
    with np.errstate(invalid="ignore"):
        inl = ang <= max_angle
    return dict(t=t, X=X, component=P["comp"], angle=ang, inliers=inl, cost0=cost0, cost=cost, iters=iters,
                n_used=int(P["used"].sum()), cg_iters=cg_total, c=c, d=d, start=st, P=P)
