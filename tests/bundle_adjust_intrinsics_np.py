"""numpy restatement of matching.bundle_adjust_intrinsics_ragged and matching.undistort_points -- TEST INFRASTRUCTURE
ONLY.

The RADIAL camera model of csrc/camera_radial.h and the estimator of include/degensac_b200.h written out literally:
  * the problem of tests/bundle_adjust_np.py (usable and used observations, optimised tracks, scale gauge, loss), with
    the RADIAL projection and a camera of an invalid group treated as unregistered;
  * the unknowns [free poses (6 each); free groups' intrinsics (5 each)], pinned coordinates (inactive slots and
    groups, the held coordinate, the intrinsics not refined) with identity rows and columns and a zero right-hand side;
  * one trial step by PCG on the matrix-free Schur complement with the SCHUR_JACOBI preconditioner (`pcg_step`), or
    by the full damped normal equations (`dense_step`);
  * the schedule of tests/bundle_adjust_pcg_np.py.

tests/test_bundle_adjust_intrinsics.py pins this file to central differences, to a dense S, to the pose-only oracle and
to scipy.optimize.least_squares, and the kernel to this file."""
import math

import numpy as np

from tests.bundle_adjust_np import expmap, gauge_axis, inv3, registered, rho, step_pose, weight
from tests.pose_refine_np import LAMBDA0, LAMBDA_MAX, LAMBDA_MIN, REL_DECREASE

FOCAL, PRINCIPAL_POINT, DISTORTION = 1, 2, 4
UNDISTORT_ITERS = 50


# ------------------------------------------------------------------------------------------------ camera_radial.h
def valid(k):
    k = np.asarray(k, np.float64)
    return bool(np.isfinite(k).all() and k[0] > 0.0)


def project(Rc, tc, kc, X, x):
    """per observation (Rc [n,3,3], tc [n,3], intrinsics kc [n,5], X [n,3], pixel x [n,2]): r [n,2], J_cam [n,2,6],
    J_X [n,2,3], J_k [n,2,5] and the depth [n] (rad_jacobian)"""
    g = np.einsum("nij,nj->ni", Rc, X)
    p = g + tc
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        iz = 1.0 / p[:, 2]
        u = p[:, :2] * iz[:, None]
        s = (u ** 2).sum(1)
        f, k1, k2 = kc[:, 0], kc[:, 3], kc[:, 4]
        d = 1.0 + s * (k1 + s * k2)
        r = (f * d)[:, None] * u + kc[:, 1:3] - x
        c = 2.0 * f * (k1 + 2.0 * s * k2)
        A = (f * d)[:, None, None] * np.eye(2) + c[:, None, None] * np.einsum("ni,nj->nij", u, u)
        Dp = np.zeros((len(x), 2, 3))
        Dp[:, 0, 0] = Dp[:, 1, 1] = iz
        Dp[:, :, 2] = -u * iz[:, None]
        D = A @ Dp
    Jc = np.zeros((len(x), 2, 6))
    Jc[:, 0, :3], Jc[:, 0, 3:] = np.cross(g, D[:, 0]), D[:, 0]
    Jc[:, 1, :3], Jc[:, 1, 3:] = np.cross(g, D[:, 1]), D[:, 1]
    Jx = D @ Rc
    Jk = np.zeros((len(x), 2, 5))
    Jk[:, :, 0] = d[:, None] * u
    Jk[:, 0, 1] = Jk[:, 1, 2] = 1.0
    Jk[:, :, 3] = (f * s)[:, None] * u
    Jk[:, :, 4] = (f * s * s)[:, None] * u
    return r, Jc, Jx, Jk, p[:, 2]


def max_radius(k1, k2):
    """the first turning point of rho (1 + k1 rho^2 + k2 rho^4), or inf"""
    s = math.inf
    if k2 == 0.0:
        if k1 < 0.0:
            s = -1.0 / (3.0 * k1)
    else:
        disc = 9.0 * k1 * k1 - 20.0 * k2
        if disc >= 0.0:
            q = math.sqrt(disc)
            for v in ((-3.0 * k1 - q) / (10.0 * k2), (-3.0 * k1 + q) / (10.0 * k2)):
                if v > 0.0:
                    s = min(s, v)
    return math.sqrt(s)


def distort(k, u):
    """the raw pixels [n,2] of normalised points u [n,2]"""
    s = (u ** 2).sum(1)
    return (k[0] * (1.0 + s * (k[3] + s * k[4])))[:, None] * u + np.asarray(k[1:3])


def undistort(k, x, y):
    """rad_undistort: the pinhole pixel (f u + c) of the raw pixel (x, y), or (nan, nan)"""
    nan = (math.nan, math.nan)
    if not valid(k) or not (math.isfinite(x) and math.isfinite(y)):
        return nan
    f, cx, cy, k1, k2 = (float(v) for v in k)
    dx, dy = x - cx, y - cy
    rd = math.sqrt(dx * dx + dy * dy) / f
    if rd == 0.0:
        return x, y
    rmax = max_radius(k1, k2)
    lo, hi = 0.0, rmax
    if rmax < math.inf:
        s = rmax * rmax
        if not rd < rmax * (1.0 + s * (k1 + s * k2)):
            return nan
    rho_ = rd if rd < hi else 0.5 * hi
    for _ in range(UNDISTORT_ITERS):
        s = rho_ * rho_
        phi = rho_ * (1.0 + s * (k1 + s * k2)) - rd
        if phi == 0.0:
            break
        if phi > 0.0:
            hi = rho_
        else:
            lo = rho_
        nxt = rho_ - phi / (1.0 + s * (3.0 * k1 + 5.0 * k2 * s))
        if abs(nxt - rho_) <= 1e-15 * rho_:
            rho_ = nxt
            break
        rho_ = nxt if lo < nxt < hi else (0.5 * (lo + hi) if hi < math.inf else 2.0 * rho_)
    s = rho_ * rho_
    if not abs(rho_ * (1.0 + s * (k1 + s * k2)) - rd) <= 1e-14 * rd:
        return nan
    return cx + dx * (rho_ / rd), cy + dy * (rho_ / rd)


def undistort_points(pts, cams, groups, intrinsics):
    out = np.full((len(pts), 2), np.nan)
    C, G = len(groups), len(intrinsics)
    for i, (c, (x, y)) in enumerate(zip(cams, pts)):
        if 0 <= c < C and 0 <= groups[c] < G:
            out[i] = undistort(intrinsics[groups[c]], float(x), float(y))
    return out


# ------------------------------------------------------------------------------------------------ the problem
def setup(cams, pts, R, t, groups, intrinsics, offsets, X, mask=None, free=None, free_groups=None,
          refine=FOCAL | DISTORTION, scale_gauge="auto", loss_scale=None):
    cams, pts, R, t, X = (np.asarray(v) for v in (cams, pts, R, t, X))
    R, t, X, pts = R.astype(np.float64), t.astype(np.float64), X.astype(np.float64), pts.astype(np.float64)
    groups = np.asarray(groups, np.int64)
    k = np.asarray(intrinsics, np.float64)
    C, T, obs, G = len(R), len(offsets) - 1, len(cams), len(k)
    free = list(range(1, C)) if free is None else [int(c) for c in free]
    fgroups = list(range(G)) if free_groups is None else [int(g) for g in free_groups]
    if refine == 0:
        fgroups = []
    held = [c for c in range(C) if c not in free]
    if isinstance(scale_gauge, str):
        gauge = free[0] if len(held) == 1 and free else None
    else:
        gauge = scale_gauge
    sig2 = 0.0 if loss_scale is None else float(loss_scale) ** 2
    gok = np.array([valid(k[g]) for g in range(G)])
    ok = np.array([registered(R[c], t[c]) and 0 <= groups[c] < G and gok[groups[c]] for c in range(C)])
    grp = np.where((groups >= 0) & (groups < G), groups, 0)
    m = np.ones(obs, bool) if mask is None else np.asarray(mask, bool)
    trk = np.zeros(obs, np.int64)
    usable = np.zeros(obs, bool)
    used = np.zeros(obs, bool)
    opt = np.zeros(T, bool)
    for j in range(T):
        b, e = int(offsets[j]), int(offsets[j + 1])
        if not (0 <= b <= e <= obs):
            continue
        trk[b:e] = j
        if not np.isfinite(X[j]).all():
            continue
        cj = cams[b:e]
        u = m[b:e] & (cj >= 0) & (cj < C) & np.isfinite(pts[b:e]).all(1)
        u &= ok[np.clip(cj, 0, C - 1)]
        idx = np.flatnonzero(u) + b
        if len(idx):
            c = cams[idx]
            r, _, Jx, _, z = project(R[c], t[c], k[grp[c]], np.broadcast_to(X[j], (len(idx), 3)), pts[idx])
            front = z > 0.0
            u[idx - b] = front
            idx, r, Jx = idx[front], r[front], Jx[front]
        usable[b:e] = u
        if len(idx) == 0 or len(set(cams[idx].tolist())) < 2:
            continue
        w = weight((r ** 2).sum(1), sig2)
        V = np.einsum("n,nik,nil->kl", w, Jx, Jx)
        if inv3(V, 0.0) is None:
            continue
        opt[j] = True
        used[idx] = True
    slot_of = np.full(C, -1)
    for s, c in enumerate(free):
        slot_of[c] = s
    gslot_of = np.full(G, -1)
    for q, g in enumerate(fgroups):
        gslot_of[g] = q
    cu = np.clip(cams, 0, C - 1)
    active = np.array([bool((used & (slot_of[cu] == s)).any()) for s in range(len(free))], bool)
    gactive = np.array([bool((used & (gslot_of[grp[cu]] == q)).any()) for q in range(len(fgroups))], bool)
    hold = None
    if gauge is not None:
        a = held[0]
        hold = 6 * free.index(gauge) + 3 + gauge_axis(R[gauge], t[gauge], -R[a].T @ t[a])
    nf, ng = len(free), len(fgroups)
    pin = np.r_[~np.repeat(active, 6), np.ones(5 * ng, bool)]
    bits = np.array([refine & FOCAL, refine & PRINCIPAL_POINT, refine & PRINCIPAL_POINT, refine & DISTORTION,
                     refine & DISTORTION], bool)
    for q in range(ng):
        pin[6 * nf + 5 * q:6 * nf + 5 * q + 5] = ~(gactive[q] & bits)
    if hold is not None:
        pin[hold] = True
    return dict(cams=cams, pts=pts, R=R, t=t, k=k, groups=grp, X=X, T=T, C=C, G=G, free=free, fgroups=fgroups,
                slot_of=slot_of, gslot_of=gslot_of, active=active, gactive=gactive, hold=hold, pin=pin, sig2=sig2,
                usable=usable, used=used, opt=opt, trk=trk, offsets=np.asarray(offsets))


def _obs(P, R, t, k, X):
    u = np.flatnonzero(P["used"])
    c = P["cams"][u]
    return u, c, project(R[c], t[c], k[P["groups"][c]], X[P["trk"][u]], P["pts"][u])


def cost(P, R, t, k, X):
    """sum rho(e^2) over the used observations (+inf when one has depth <= 0 or its group f <= 0)"""
    u, c, (r, _, _, _, z) = _obs(P, R, t, k, X)
    if len(u) and not ((z > 0.0) & (k[P["groups"][c], 0] > 0.0)).all():
        return math.inf
    return float(rho((r ** 2).sum(1), P["sig2"]).sum())


def linearise(P, R, t, k, X):
    """the used observations' r, w, J_cam, J_X, J_k, track p, slot s and group slot h; V [T,3,3], g_p [T,3]"""
    u, c, (r, Jc, Jx, Jk, _) = _obs(P, R, t, k, X)
    w = weight((r ** 2).sum(1), P["sig2"])
    p = P["trk"][u]
    V = np.zeros((P["T"], 3, 3))
    gp = np.zeros((P["T"], 3))
    np.add.at(V, p, np.einsum("n,nik,nil->nkl", w, Jx, Jx))
    np.add.at(gp, p, np.einsum("n,nik,ni->nk", w, Jx, r))
    return dict(r=r, w=w, Jc=Jc, Jx=Jx, Jk=Jk, p=p, s=P["slot_of"][c], h=P["gslot_of"][P["groups"][c]], V=V, gp=gp)


def _sizes(P):
    return len(P["free"]), len(P["fgroups"])


def _jv(P, lin, x):
    """J_ext x per observation [n,2]: J_cam x_slot + J_k x_group"""
    nf, ng = _sizes(P)
    xp, xg = x[:6 * nf].reshape(nf, 6), x[6 * nf:].reshape(ng, 5)
    v = np.zeros((len(lin["w"]), 2))
    f = lin["s"] >= 0
    v[f] += np.einsum("nij,nj->ni", lin["Jc"][f], xp[lin["s"][f]])
    f = lin["h"] >= 0
    v[f] += np.einsum("nij,nj->ni", lin["Jk"][f], xg[lin["h"][f]])
    return v


def _jtv(P, lin, v):
    """sum J_ext^T v [N] over the observations"""
    nf, ng = _sizes(P)
    out = np.zeros(6 * nf + 5 * ng)
    f = lin["s"] >= 0
    a = np.zeros((nf, 6))
    np.add.at(a, lin["s"][f], np.einsum("nij,ni->nj", lin["Jc"][f], v[f]))
    f = lin["h"] >= 0
    b = np.zeros((ng, 5))
    np.add.at(b, lin["h"][f], np.einsum("nij,ni->nj", lin["Jk"][f], v[f]))
    out[:6 * nf], out[6 * nf:] = a.reshape(-1), b.reshape(-1)
    return out


def _diag_u(P, lin):
    nf, ng = _sizes(P)
    out = np.zeros(6 * nf + 5 * ng)
    f = lin["s"] >= 0
    a = np.zeros((nf, 6))
    np.add.at(a, lin["s"][f], lin["w"][f, None] * (lin["Jc"][f] ** 2).sum(1))
    f = lin["h"] >= 0
    b = np.zeros((ng, 5))
    np.add.at(b, lin["h"][f], lin["w"][f, None] * (lin["Jk"][f] ** 2).sum(1))
    out[:6 * nf], out[6 * nf:] = a.reshape(-1), b.reshape(-1)
    return out


def point_inverses(P, lin, lam):
    Vi = np.zeros_like(lin["V"])
    for j in np.flatnonzero(P["opt"]):
        v = inv3(lin["V"][j], lam)
        if v is None:
            return None
        Vi[j] = v
    return Vi


def schur_matvec(P, lin, Vi, lam, x):
    """S p, pinned rows and columns of the identity: U* p - sum_p W_p V*_p^-1 W_p^T p"""
    pin = P["pin"]
    xx = np.where(pin, 0.0, x)
    v = _jv(P, lin, xx)
    wv = lin["w"][:, None] * v
    tp = np.zeros((P["T"], 3))
    np.add.at(tp, lin["p"], np.einsum("nij,ni->nj", lin["Jx"], wv))
    y = np.einsum("tml,tl->tm", Vi, tp)
    q = _jtv(P, lin, wv) + lam * _diag_u(P, lin) * xx
    q -= _jtv(P, lin, lin["w"][:, None] * np.einsum("nij,nj->ni", lin["Jx"], y[lin["p"]]))
    q[pin] = x[pin]
    return q


def rhs(P, lin, Vi):
    """b = -(g - sum_p W_p V*_p^-1 g_p), 0 at the pinned coordinates"""
    g = _jtv(P, lin, lin["w"][:, None] * lin["r"])
    vg = np.einsum("tml,tl->tm", Vi, lin["gp"])
    h = _jtv(P, lin, lin["w"][:, None] * np.einsum("nij,nj->ni", lin["Jx"], vg[lin["p"]]))
    b = h - g
    b[P["pin"]] = 0.0
    return b


def _blocks(P):
    """the parameter blocks: (start, size) of every free slot, then every free group"""
    nf, ng = _sizes(P)
    return [(6 * a, 6) for a in range(nf)] + [(6 * nf + 5 * q, 5) for q in range(ng)]


def preconditioner(P, lin, Vi, lam):
    """the Cholesky factors of the SCHUR_JACOBI blocks U*_bb - sum W_b V*^-1 W_b^T (pinned rows and columns of the
    identity), or None at a non-positive pivot"""
    nf, ng = _sizes(P)
    w = lin["w"]
    Wp = np.einsum("n,nik,nil->nkl", w, lin["Jc"], lin["Jx"])
    Wk = np.einsum("n,nik,nil->nkl", w, lin["Jk"], lin["Jx"])
    Vp = Vi[lin["p"]]
    Ma = np.zeros((nf, 6, 6))
    f = lin["s"] >= 0
    np.add.at(Ma, lin["s"][f], np.einsum("n,nik,nil->nkl", w[f], lin["Jc"][f], lin["Jc"][f]))
    Ma = Ma + lam * np.einsum("aii->ai", Ma)[:, :, None] * np.eye(6)
    np.add.at(Ma, lin["s"][f], -np.einsum("nkm,nml,njl->nkj", Wp[f], Vp[f], Wp[f]))
    Mg = np.zeros((ng, 5, 5))
    f = lin["h"] >= 0
    np.add.at(Mg, lin["h"][f], np.einsum("n,nik,nil->nkl", w[f], lin["Jk"][f], lin["Jk"][f]))
    Mg = Mg + lam * np.einsum("aii->ai", Mg)[:, :, None] * np.eye(5)
    np.add.at(Mg, lin["h"][f], -np.einsum("nkm,nml,njl->nkj", Wk[f], Vp[f], Wk[f]))
    Ls = []
    for (o, n), M in zip(_blocks(P), list(Ma) + list(Mg)):
        M = M.copy()
        for kk in np.flatnonzero(P["pin"][o:o + n]):
            M[kk, :] = 0.0
            M[:, kk] = 0.0
            M[kk, kk] = 1.0
        try:
            L = np.linalg.cholesky(M)
        except np.linalg.LinAlgError:
            return None
        if not (np.diag(L) > 0.0).all():
            return None
        Ls.append(L)
    return Ls


def _apply_m(P, Ls, r):
    z = np.zeros_like(r)
    for (o, n), L in zip(_blocks(P), Ls):
        z[o:o + n] = np.linalg.solve(L.T, np.linalg.solve(L, r[o:o + n]))
    return z


def pcg(P, lin, Vi, lam, cg_tol, cg_max_iters):
    """(dx, iterations), dx None when the step is rejected"""
    Ls = preconditioner(P, lin, Vi, lam)
    if Ls is None:
        return None, 0
    b = rhs(P, lin, Vi)
    x = np.zeros_like(b)
    bb = float(b @ b)
    if bb == 0.0:
        return x, 0
    r = b.copy()
    z = _apply_m(P, Ls, r)
    p = z.copy()
    rho_ = float(r @ z)
    k = 0
    while True:
        q = schur_matvec(P, lin, Vi, lam, p)
        kappa = float(p @ q)
        k += 1
        if not (kappa > 0.0) or not np.isfinite(kappa):
            return (None if k == 1 else x), k
        alpha = rho_ / kappa
        x = x + alpha * p
        r = r - alpha * q
        if float(r @ r) <= cg_tol * cg_tol * bb or k >= cg_max_iters:
            return x, k
        z = _apply_m(P, Ls, r)
        rz = float(r @ z)
        p = z + (rz / rho_) * p
        rho_ = rz


def back_substitute(P, lin, Vi, dx):
    acc = np.zeros((P["T"], 3))
    np.add.at(acc, lin["p"], np.einsum("nij,ni->nj", lin["Jx"], lin["w"][:, None] * _jv(P, lin, dx)))
    dX = -np.einsum("pkl,pl->pk", Vi, lin["gp"] + acc)
    dX[~P["opt"]] = 0.0
    return dX


def pcg_step(P, lin, lam, cg_tol, cg_max_iters):
    """((dx, dX) or None when the step is rejected, CG iterations)"""
    Vi = point_inverses(P, lin, lam)
    if Vi is None:
        return None, 0
    dx, k = pcg(P, lin, Vi, lam, cg_tol, cg_max_iters)
    if dx is None:
        return None, k
    return (dx, back_substitute(P, lin, Vi, dx)), k


# ------------------------------------------------------------------------------------------------ dense views
def dense_jacobian(P, lin):
    """J_ext [n,2,N] over [free poses; free groups]"""
    nf, ng = _sizes(P)
    J = np.zeros((len(lin["w"]), 2, 6 * nf + 5 * ng))
    for i in range(len(lin["w"])):
        if lin["s"][i] >= 0:
            J[i, :, 6 * lin["s"][i]:6 * lin["s"][i] + 6] = lin["Jc"][i]
        if lin["h"][i] >= 0:
            J[i, :, 6 * nf + 5 * lin["h"][i]:6 * nf + 5 * lin["h"][i] + 5] = lin["Jk"][i]
    return J


def dense_s(P, lin, lam, absolute=False):
    """S over the kept coordinates (absolute: with |J|, |V*^-1| and the terms added, the scale of its rounding)"""
    J = dense_jacobian(P, lin)
    Jx, w = lin["Jx"], lin["w"]
    Vi = point_inverses(P, lin, lam)
    if absolute:
        J, Jx, Vi = np.abs(J), np.abs(Jx), np.abs(Vi)
    U = np.einsum("n,nik,nil->kl", w, J, J)
    U = U + lam * np.diag(np.diag(U))
    W = np.zeros((P["T"], J.shape[2], 3))
    np.add.at(W, lin["p"], np.einsum("n,nik,nil->nkl", w, J, Jx))
    S = U + (1 if absolute else -1) * np.einsum("tkm,tml,tjl->kj", W, Vi, W)
    keep = ~P["pin"]
    return S[np.ix_(keep, keep)], keep


def dense_step(P, lin, lam):
    """the step from the full damped normal equations [[U*, W], [W^T, V*]], pinned unknowns removed; or None"""
    J = dense_jacobian(P, lin)
    N, T = J.shape[2], P["T"]
    w = lin["w"]
    H = np.zeros((N + 3 * T, N + 3 * T))
    g = np.zeros(N + 3 * T)
    for i in range(len(w)):
        p = lin["p"][i]
        Ji = np.zeros((2, N + 3 * T))
        Ji[:, :N] = J[i]
        Ji[:, N + 3 * p:N + 3 * p + 3] = lin["Jx"][i]
        H += w[i] * Ji.T @ Ji
        g += w[i] * Ji.T @ lin["r"][i]
    H = H + lam * np.diag(np.diag(H))
    keep = np.r_[~P["pin"], np.repeat(P["opt"], 3)]
    d = np.zeros(len(g))
    try:
        d[keep] = np.linalg.solve(H[np.ix_(keep, keep)], -g[keep])
    except np.linalg.LinAlgError:
        return None
    return d[:N], d[N:].reshape(T, 3)


def apply(P, R, t, k, X, dx, dX):
    nf, _ = _sizes(P)
    R2, t2, k2, X2 = R.copy(), t.copy(), k.copy(), X.copy()
    for s, c in enumerate(P["free"]):
        if P["active"][s]:
            R2[c], t2[c] = step_pose(R[c], t[c], dx[6 * s:6 * s + 6])
    for q, g in enumerate(P["fgroups"]):
        if P["gactive"][q]:
            k2[g] = k[g] + dx[6 * nf + 5 * q:6 * nf + 5 * q + 5]
    X2[P["opt"]] = X[P["opt"]] + dX[P["opt"]]
    return R2, t2, k2, X2


def bundle_adjust_intrinsics(cams, pts, R, t, groups, intrinsics, offsets, X, mask=None, free=None, free_groups=None,
                             refine=FOCAL | DISTORTION, scale_gauge="auto", loss_scale=None, max_iters=50, px_th=2.0,
                             cg_max_iters=100, cg_tol=0.1, dense=False, P=None):
    """The whole call: dict(R, t, X, intrinsics, mask, cost0, cost, iters, n_used, cg_iters); dense: every trial step
    from the full normal equations"""
    if P is None:
        P = setup(cams, pts, R, t, groups, intrinsics, offsets, X, mask, free, free_groups, refine, scale_gauge,
                  loss_scale)
    R, t, k, X = P["R"].copy(), P["t"].copy(), P["k"].copy(), P["X"].copy()
    c_cur = c0 = cost(P, R, t, k, X)
    lam, iters, cg_iters = LAMBDA0, 0, 0
    lin = linearise(P, R, t, k, X)
    for _ in range(max_iters):
        iters += 1
        if dense:
            Vi = point_inverses(P, lin, lam)
            step = None if Vi is None else dense_step(P, lin, lam)
        else:
            step, kk = pcg_step(P, lin, lam, cg_tol, cg_max_iters)
            cg_iters += kk
        go = step is not None
        c_new = c_cur
        if go:
            R2, t2, k2, X2 = apply(P, R, t, k, X, *step)
            c_new = cost(P, R2, t2, k2, X2)
        better = go and c_new < c_cur
        flat = go and abs(c_cur - c_new) < REL_DECREASE * c_cur
        if better:
            R, t, k, X, c_cur = R2, t2, k2, X2, c_new
            lam = max(lam / 10.0, LAMBDA_MIN)
            lin = linearise(P, R, t, k, X)
            if flat:
                break
        else:
            lam *= 10.0
            if flat or lam > LAMBDA_MAX:
                break
    out_mask = np.zeros(len(P["cams"]), bool)
    u = np.flatnonzero(P["usable"])
    if len(u):
        c = P["cams"][u]
        r, _, _, _, z = project(R[c], t[c], k[P["groups"][c]], X[P["trk"][u]], P["pts"][u])
        out_mask[u] = (z > 0.0) & ((r ** 2).sum(1) <= px_th * px_th)
    return dict(R=R, t=t, X=X, intrinsics=k, mask=out_mask, cost0=c0, cost=c_cur, iters=iters,
                n_used=int(P["used"].sum()), cg_iters=cg_iters, P=P)


# ------------------------------------------------------------------------------------------------ scipy's view
def residuals(P, v):
    """the pixel residuals at v = (the kept coordinates of [poses; intrinsics], then 3 per optimised track), relative
    to the start"""
    nf, _ = _sizes(P)
    keep = np.flatnonzero(~P["pin"])
    trk = np.flatnonzero(P["opt"])
    dx = np.zeros(len(P["pin"]))
    dx[keep] = v[:len(keep)]
    R, t, k, X = P["R"].copy(), P["t"].copy(), P["k"].copy(), P["X"].copy()
    for s, c in enumerate(P["free"]):
        if P["active"][s]:
            R[c] = expmap(dx[6 * s:6 * s + 3]) @ P["R"][c]
            t[c] = P["t"][c] + dx[6 * s + 3:6 * s + 6]
    for q, g in enumerate(P["fgroups"]):
        k[g] = P["k"][g] + dx[6 * nf + 5 * q:6 * nf + 5 * q + 5]
    X[trk] = P["X"][trk] + v[len(keep):].reshape(-1, 3)
    return _obs(P, R, t, k, X)[2][0].ravel()
