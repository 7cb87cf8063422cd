"""numpy restatement of matching.bundle_adjust_ragged -- TEST INFRASTRUCTURE ONLY.

The estimator's contract (include/degensac_b200.h) written out literally, vectorised over the observations:
  * usable observations: mask set, camera index in range and registered (finite R, t and det R > 0.5), finite pixel,
    finite X of the track, depth > 0 at the start; a track is optimised when its usable observations come from 2
    distinct cameras and V_p at the start has a positive Cholesky factor; a free camera without a used observation is
    held;
  * the scale gauge: translation coordinate argmax |t_g + R_g c_a| of camera g held, a the lowest index outside free;
  * cost sum rho(e^2) (the squared error, or Cauchy sigma^2 log1p(e^2 / sigma^2)), IRLS weights rho'(e^2);
  * one trial step by the Schur complement (`schur_step`) or by the full damped normal equations (`dense_step`);
  * the schedule of the pose refinement and re-orthonormalisation of a trial R above 1e-12.

tests/test_bundle_adjust.py pins this file to scipy.optimize.least_squares, to central differences and to the host
build of csrc/bundle_adjust.h, and the kernel to this file."""
import math

import numpy as np

from tests.pose_refine_np import LAMBDA0, LAMBDA_MAX, LAMBDA_MIN, REL_DECREASE

MAX_FREE = 64
ORTHO_TOL = 1e-12


# ------------------------------------------------------------------------------------------------ bundle_adjust.h
def rho(s, sig2):
    return sig2 * np.log1p(s / sig2) if sig2 > 0.0 else s


def weight(s, sig2):
    return 1.0 / (1.0 + s / sig2) if sig2 > 0.0 else np.ones_like(s)


def project(Rc, tc, Kc, X, x):
    """per observation (camera Rc [n,3,3], tc [n,3], Kc [n,3,3], point X [n,3], pixel x [n,2]): r [n,2], J_cam [n,2,6]
    by (w, d) of R <- exp([w]x) R, t <- t + d, J_X [n,2,3] and the depth [n] (ba_jacobian)"""
    g = np.einsum("nij,nj->ni", Rc, X)
    p = g + tc
    q = np.einsum("nij,nj->ni", Kc, p)
    with np.errstate(divide="ignore", invalid="ignore"):
        iz = 1.0 / q[:, 2]
        u, v = q[:, 0] * iz, q[:, 1] * iz
        r = np.stack([u - x[:, 0], v - x[:, 1]], 1)
        Du = (Kc[:, 0, :] - u[:, None] * Kc[:, 2, :]) * iz[:, None]
        Dv = (Kc[:, 1, :] - v[:, None] * Kc[:, 2, :]) * iz[:, None]
    Jc = np.zeros((len(x), 2, 6))
    Jc[:, 0, :3], Jc[:, 0, 3:] = np.cross(g, Du), Du
    Jc[:, 1, :3], Jc[:, 1, 3:] = np.cross(g, Dv), Dv
    Jx = np.stack([np.einsum("nk,nkm->nm", Du, Rc), np.einsum("nk,nkm->nm", Dv, Rc)], 1)
    return r, Jc, Jx, p[:, 2]


def inv3(V, lam):
    """(V + lam diag V)^-1 of a symmetric 3 x 3 by the pivots of ba_inv3, or None at a pivot that is not positive"""
    A = V + lam * np.diag(np.diag(V))
    l00 = A[0, 0]
    if not l00 > 0.0:
        return None
    l00 = math.sqrt(l00)
    l10, l20 = A[0, 1] / l00, A[0, 2] / l00
    d1 = A[1, 1] - l10 * l10
    if not d1 > 0.0:
        return None
    l11 = math.sqrt(d1)
    l21 = (A[1, 2] - l20 * l10) / l11
    d2 = A[2, 2] - l20 * l20 - l21 * l21
    if not d2 > 0.0:
        return None
    L = np.array([[l00, 0, 0], [l10, l11, 0], [l20, l21, math.sqrt(d2)]])
    M = np.linalg.inv(L)
    return M.T @ M


def gauge_axis(Rg, tg, Ca):
    return int(np.argmax(np.abs(Rg @ Ca + tg)))


def expmap(w):
    a = float(np.linalg.norm(w))
    W = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    if a == 0.0:
        return np.eye(3) + W + 0.5 * W @ W
    return np.eye(3) + math.sin(a) / a * W + 2.0 * (math.sin(0.5 * a) / a) ** 2 * W @ W


def orthonormalise(R):
    R = R.copy()
    R[0] /= np.linalg.norm(R[0])
    R[1] -= (R[0] @ R[1]) * R[0]
    R[1] /= np.linalg.norm(R[1])
    R[2] = np.cross(R[0], R[1])
    return R


def step_pose(R, t, D):
    R2 = expmap(D[:3]) @ R
    if np.abs(R2 @ R2.T - np.eye(3)).max() > ORTHO_TOL:
        R2 = orthonormalise(R2)
    return R2, t + D[3:]


# ------------------------------------------------------------------------------------------------ the problem
def registered(R, t):
    return bool(np.isfinite(R).all() and np.isfinite(t).all() and np.linalg.det(R) > 0.5)


def setup(cams, pts, R, t, K, offsets, X, mask=None, free=None, scale_gauge="auto", loss_scale=None):
    """The problem at the start point: the used observations, the optimised tracks, the active slots and the held
    coordinate"""
    cams, pts, R, t, X = (np.asarray(v) for v in (cams, pts, R, t, X))
    R, t, X, pts = R.astype(np.float64), t.astype(np.float64), X.astype(np.float64), pts.astype(np.float64)
    C, T, obs = len(R), len(offsets) - 1, len(cams)
    K = np.asarray(K, np.float64)
    Ks = np.broadcast_to(K, (C, 3, 3)) if K.ndim == 2 else K
    free = list(range(1, C)) if free is None else [int(c) for c in free]
    held = [c for c in range(C) if c not in free]
    if isinstance(scale_gauge, str):
        gauge = free[0] if len(held) == 1 and free else None
    else:
        gauge = scale_gauge
    sig2 = 0.0 if loss_scale is None else float(loss_scale) ** 2
    ok = np.array([registered(R[c], t[c]) for c in range(C)])
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
            r, _, Jx, z = project(R[c], t[c], Ks[c], np.broadcast_to(X[j], (len(idx), 3)), pts[idx])
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
    active = np.array([bool((used & (slot_of[np.clip(cams, 0, C - 1)] == s)).any()) for s in range(len(free))], bool)
    hold = None
    if gauge is not None:
        a = held[0]
        hold = 6 * free.index(gauge) + 3 + gauge_axis(R[gauge], t[gauge], -R[a].T @ t[a])
    return dict(cams=cams, pts=pts, R=R, t=t, K=Ks, X=X, T=T, C=C, free=free, slot_of=slot_of, active=active,
                hold=hold, sig2=sig2, usable=usable, used=used, opt=opt, trk=trk, offsets=np.asarray(offsets))


def _obs(P, R, t, X):
    u = np.flatnonzero(P["used"])
    c = P["cams"][u]
    return u, c, R[c], t[c], P["K"][c], X[P["trk"][u]], P["pts"][u]


def cost(P, R, t, X):
    """sum rho(e^2) over the used observations (+inf when one has depth <= 0)"""
    u, c, Rc, tc, Kc, Xo, x = _obs(P, R, t, X)
    r, _, _, z = project(Rc, tc, Kc, Xo, x)
    if len(u) and not (z > 0.0).all():
        return math.inf
    return float(rho((r ** 2).sum(1), P["sig2"]).sum())


def linearise(P, R, t, X):
    """the blocks of the normal equations: U [nf,6,6], g_c [nf,6], V [T,3,3], g_p [T,3], W [nf,T,6,3]"""
    nf, T = len(P["free"]), P["T"]
    u, c, Rc, tc, Kc, Xo, x = _obs(P, R, t, X)
    r, Jc, Jx, _ = project(Rc, tc, Kc, Xo, x)
    w = weight((r ** 2).sum(1), P["sig2"])
    p = P["trk"][u]
    s = P["slot_of"][c]
    V = np.zeros((T, 3, 3))
    gp = np.zeros((T, 3))
    np.add.at(V, p, np.einsum("n,nik,nil->nkl", w, Jx, Jx))
    np.add.at(gp, p, np.einsum("n,nik,ni->nk", w, Jx, r))
    U = np.zeros((nf, 6, 6))
    gc = np.zeros((nf, 6))
    W = np.zeros((nf, T, 6, 3))
    f = s >= 0
    np.add.at(U, s[f], np.einsum("n,nik,nil->nkl", w[f], Jc[f], Jc[f]))
    np.add.at(gc, s[f], np.einsum("n,nik,ni->nk", w[f], Jc[f], r[f]))
    np.add.at(W, (s[f], p[f]), np.einsum("n,nik,nil->nkl", w[f], Jc[f], Jx[f]))
    return dict(U=U, gc=gc, V=V, gp=gp, W=W)


def _keep(P):
    """the camera unknowns in the system: active slots without the held coordinate"""
    keep = np.repeat(P["active"], 6)
    if P["hold"] is not None:
        keep[P["hold"]] = False
    return keep


def _damp(A, lam):
    return A + lam * np.einsum("...ii->...i", A)[..., None] * np.eye(A.shape[-1])


def schur_step(P, lin, lam):
    """(dc [nf*6], dX [T,3]) of one damped step by the Schur complement, or None at a non-positive pivot"""
    nf, opt = len(P["free"]), P["opt"]
    Vi = np.zeros_like(lin["V"])
    for j in np.flatnonzero(opt):
        v = inv3(lin["V"][j], lam)
        if v is None:
            return None
        Vi[j] = v
    Ud = _damp(lin["U"], lam)
    Y = np.einsum("apkl,plm->apkm", lin["W"], Vi)
    S = np.einsum("apkm,bplm->akbl", Y, lin["W"]).reshape(6 * nf, 6 * nf)
    S = _blockdiag(Ud) - S
    rhs = -(lin["gc"] - np.einsum("apkm,pm->ak", Y, lin["gp"])).reshape(-1)
    keep = _keep(P)
    dc = np.zeros(6 * nf)
    if keep.any():
        Sk = S[np.ix_(keep, keep)]
        try:
            L = np.linalg.cholesky(Sk)
        except np.linalg.LinAlgError:
            return None
        dc[keep] = np.linalg.solve(L.T, np.linalg.solve(L, rhs[keep]))
    dX = -np.einsum("pkl,pl->pk", Vi, lin["gp"] + np.einsum("apkm,ak->pm", lin["W"], dc.reshape(nf, 6)))
    dX[~opt] = 0.0
    return dc, dX


def _blockdiag(B):
    n = len(B)
    out = np.zeros((6 * n, 6 * n))
    for a in range(n):
        out[6 * a:6 * a + 6, 6 * a:6 * a + 6] = B[a]
    return out


def dense_step(P, lin, lam):
    """the same step from the full damped normal equations [[U*, W], [W^T, V*]] (held unknowns removed)"""
    nf, T, opt = len(P["free"]), P["T"], P["opt"]
    nc = 6 * nf
    H = np.zeros((nc + 3 * T, nc + 3 * T))
    H[:nc, :nc] = _blockdiag(lin["U"])
    for j in range(T):
        H[nc + 3 * j:nc + 3 * j + 3, nc + 3 * j:nc + 3 * j + 3] = lin["V"][j]
    Wm = lin["W"].transpose(0, 2, 1, 3).reshape(nc, 3 * T)
    H[:nc, nc:], H[nc:, :nc] = Wm, Wm.T
    H = H + lam * np.diag(np.diag(H))
    g = np.r_[lin["gc"].reshape(-1), lin["gp"].reshape(-1)]
    keep = np.r_[_keep(P), np.repeat(opt, 3)]
    d = np.zeros(len(g))
    d[keep] = np.linalg.solve(H[np.ix_(keep, keep)], -g[keep])
    return d[:nc], d[nc:].reshape(T, 3)


def apply(P, R, t, X, dc, dX):
    R2, t2, X2 = R.copy(), t.copy(), X.copy()
    for s, c in enumerate(P["free"]):
        if P["active"][s]:
            R2[c], t2[c] = step_pose(R[c], t[c], dc[6 * s:6 * s + 6])
    X2[P["opt"]] = X[P["opt"]] + dX[P["opt"]]
    return R2, t2, X2


def bundle_adjust(cams, pts, R, t, K, offsets, X, mask=None, free=None, scale_gauge="auto", loss_scale=None,
                  max_iters=50, px_th=2.0, P=None):
    """The whole call: dict(R, t, X, mask, cost0, cost, iters, n_used) as bundle_adjust_ragged returns it"""
    if P is None:
        P = setup(cams, pts, R, t, K, offsets, X, mask, free, scale_gauge, loss_scale)
    R, t, X = P["R"].copy(), P["t"].copy(), P["X"].copy()
    c_cur = c0 = cost(P, R, t, X)
    lam, iters = LAMBDA0, 0
    lin = linearise(P, R, t, X)
    for _ in range(max_iters):
        iters += 1
        step = schur_step(P, lin, lam)
        go = step is not None
        c_new = c_cur
        if go:
            R2, t2, X2 = apply(P, R, t, X, *step)
            c_new = cost(P, R2, t2, X2)
        better = go and c_new < c_cur
        flat = go and abs(c_cur - c_new) < REL_DECREASE * c_cur
        if better:
            R, t, X, c_cur = R2, t2, X2, c_new
            lam = max(lam / 10.0, LAMBDA_MIN)
            lin = linearise(P, R, t, X)
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
        r, _, _, z = project(R[c], t[c], P["K"][c], X[P["trk"][u]], P["pts"][u])
        out_mask[u] = (z > 0.0) & ((r ** 2).sum(1) <= px_th * px_th)
    return dict(R=R, t=t, X=X, mask=out_mask, cost0=c0, cost=c_cur, iters=iters, n_used=int(P["used"].sum()), P=P)


# ------------------------------------------------------------------------------------------------ scipy's view
def unknowns(P):
    """the parameter vector's layout: (free slot, coordinate) pairs kept, then the optimised tracks"""
    keep = _keep(P)
    return np.flatnonzero(keep), np.flatnonzero(P["opt"])


def residuals(P, v, per_observation=False):
    """the residual vector at v (the kept camera coordinates, then 3 per optimised track, relative to the start):
    2 pixel residuals per used observation, or with per_observation the error e per observation"""
    cam_idx, trk_idx = unknowns(P)
    dc = np.zeros(6 * len(P["free"]))
    dc[cam_idx] = v[:len(cam_idx)]
    R, t, X = P["R"].copy(), P["t"].copy(), P["X"].copy()
    for s, c in enumerate(P["free"]):
        if P["active"][s]:
            R[c] = expmap(dc[6 * s:6 * s + 3]) @ P["R"][c]
            t[c] = P["t"][c] + dc[6 * s + 3:6 * s + 6]
    X[trk_idx] = P["X"][trk_idx] + v[len(cam_idx):].reshape(-1, 3)
    u, c, Rc, tc, Kc, Xo, x = _obs(P, R, t, X)
    r = project(Rc, tc, Kc, Xo, x)[0]
    return np.sqrt((r ** 2).sum(1)) if per_observation else r.ravel()
