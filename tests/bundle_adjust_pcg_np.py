"""numpy restatement of matching.bundle_adjust_pcg_ragged -- TEST INFRASTRUCTURE ONLY.

The estimator of tests/bundle_adjust_np.py (the problem, the cost, the update and the schedule are imported from
there), with the reduced camera system S dc = b solved by preconditioned conjugate gradients as
include/degensac_b200.h specifies it:
  * S p = U* p - sum_p W_p V*_p^-1 (W_p^T p), computed matrix-free from the linearisation stored per observation (not
    as the dense oracle's [nf, T, 6, 3]), so that it runs at hundreds of cameras;
  * the pinned coordinates (the held one and those of slots without used observations) have identity rows and columns
    and a zero right-hand side;
  * the block-Jacobi preconditioner M_a = U*_a - sum_{i in a} W_i V*^-1 W_i^T, Cholesky-factorised;
  * PCG from x = 0, stopped by |r| <= cg_tol |b|, cg_max_iters, or p . q <= 0 (which rejects the step on the first
    iteration).

tests/test_bundle_adjust_pcg.py pins this file to bundle_adjust_np.py (whose schur_step and bundle_adjust are pinned to
the full normal equations and to scipy), and the kernel to this file."""
import numpy as np

from tests.bundle_adjust_np import apply, cost, inv3, project, setup, weight
from tests.pose_refine_np import LAMBDA0, LAMBDA_MAX, LAMBDA_MIN, REL_DECREASE


def linearise(P, R, t, X):
    """per observation: U [nf,6,6], g_c [nf,6], V [T,3,3], g_p [T,3], and W [n,6,3] with its slot s [n] and track
    p [n] for the used observations of free cameras"""
    nf, T = len(P["free"]), P["T"]
    u = np.flatnonzero(P["used"])
    c = P["cams"][u]
    r, Jc, Jx, _ = project(R[c], t[c], P["K"][c], X[P["trk"][u]], P["pts"][u])
    w = weight((r ** 2).sum(1), P["sig2"])
    p = P["trk"][u]
    s = P["slot_of"][c]
    V = np.zeros((T, 3, 3))
    gp = np.zeros((T, 3))
    np.add.at(V, p, np.einsum("n,nik,nil->nkl", w, Jx, Jx))
    np.add.at(gp, p, np.einsum("n,nik,ni->nk", w, Jx, r))
    f = s >= 0
    U = np.zeros((nf, 6, 6))
    gc = np.zeros((nf, 6))
    np.add.at(U, s[f], np.einsum("n,nik,nil->nkl", w[f], Jc[f], Jc[f]))
    np.add.at(gc, s[f], np.einsum("n,nik,ni->nk", w[f], Jc[f], r[f]))
    W = np.einsum("n,nik,nil->nkl", w[f], Jc[f], Jx[f])
    return dict(U=U, gc=gc, V=V, gp=gp, W=W, s=s[f], p=p[f])


def pinned(P):
    """the camera coordinates held at 0: slots without used observations and the held coordinate"""
    pin = ~np.repeat(P["active"], 6)
    if P["hold"] is not None:
        pin[P["hold"]] = True
    return pin


def point_inverses(P, lin, lam):
    """V*_p^-1 of the optimised tracks (0 for the others), or None at a non-positive pivot"""
    Vi = np.zeros_like(lin["V"])
    for j in np.flatnonzero(P["opt"]):
        v = inv3(lin["V"][j], lam)
        if v is None:
            return None
        Vi[j] = v
    return Vi


def _damp(U, lam):
    return U + lam * np.einsum("aii->ai", U)[:, :, None] * np.eye(6)


def _segment_sum(idx, v, n):
    """sum of the rows v [m, k] by idx [m] into [n, k]"""
    return np.stack([np.bincount(idx, weights=v[:, k], minlength=n) for k in range(v.shape[1])], 1)


def schur_matvec(P, lin, Vi, lam, x):
    """S p with the pinned rows and columns of the identity: one pass over the tracks, then one over the cameras"""
    nf, T = len(P["free"]), P["T"]
    pin = pinned(P)
    xx = np.where(pin, 0.0, x).reshape(nf, 6)
    tp = _segment_sum(lin["p"], np.einsum("nkm,nk->nm", lin["W"], xx[lin["s"]]), T)
    y = np.einsum("tml,tl->tm", Vi, tp)
    q = np.einsum("akl,al->ak", _damp(lin["U"], lam), xx)
    q -= _segment_sum(lin["s"], np.einsum("nkm,nm->nk", lin["W"], y[lin["p"]]), nf).reshape(nf, 6)
    q = q.reshape(-1)
    q[pin] = x[pin]
    return q


def rhs(P, lin, Vi):
    """b = -(g_c - sum_p W_p V*_p^-1 g_p), 0 at the pinned coordinates"""
    nf = len(P["free"])
    h = np.zeros((nf, 6))
    np.add.at(h, lin["s"], np.einsum("nkm,nm->nk", lin["W"], np.einsum("nml,nl->nm", Vi[lin["p"]],
                                                                         lin["gp"][lin["p"]])))
    b = (h - lin["gc"]).reshape(-1)
    b[pinned(P)] = 0.0
    return b


def preconditioner(P, lin, Vi, lam):
    """the Cholesky factors [nf,6,6] of the blocks M_a, pinned rows and columns of the identity, or None at a
    non-positive pivot"""
    nf = len(P["free"])
    M = _damp(lin["U"], lam)
    Y = np.einsum("nkm,nml->nkl", lin["W"], Vi[lin["p"]])
    np.add.at(M, lin["s"], -np.einsum("nkm,nlm->nkl", Y, lin["W"]))
    pin = pinned(P).reshape(nf, 6)
    L = np.zeros_like(M)
    for a in range(nf):
        Ma = M[a].copy()
        for k in np.flatnonzero(pin[a]):
            Ma[k, :] = 0.0
            Ma[:, k] = 0.0
            Ma[k, k] = 1.0
        try:
            L[a] = np.linalg.cholesky(Ma)
        except np.linalg.LinAlgError:
            return None
        if not (np.diag(L[a]) > 0.0).all():
            return None
    return L


def _apply_m(L, r):
    nf = len(L)
    z = np.linalg.solve(L, r.reshape(nf, 6, 1))
    return np.linalg.solve(L.transpose(0, 2, 1), z).reshape(-1)


def pcg(P, lin, Vi, lam, cg_tol, cg_max_iters):
    """(dc, iterations), dc None when the step is rejected"""
    L = preconditioner(P, lin, Vi, lam)
    if L is None:
        return None, 0
    b = rhs(P, lin, Vi)
    x = np.zeros_like(b)
    bb = float(b @ b)
    if bb == 0.0:
        return x, 0
    r = b.copy()
    z = _apply_m(L, r)
    p = z.copy()
    rho = float(r @ z)
    k = 0
    while True:
        q = schur_matvec(P, lin, Vi, lam, p)
        kappa = float(p @ q)
        k += 1
        if not (kappa > 0.0) or not np.isfinite(kappa):
            return (None if k == 1 else x), k
        alpha = rho / kappa
        x = x + alpha * p
        r = r - alpha * q
        if float(r @ r) <= cg_tol * cg_tol * bb or k >= cg_max_iters:
            return x, k
        z = _apply_m(L, r)
        rz = float(r @ z)
        p = z + (rz / rho) * p
        rho = rz


def back_substitute(P, lin, Vi, dc):
    nf = len(P["free"])
    acc = np.zeros((P["T"], 3))
    np.add.at(acc, lin["p"], np.einsum("nkm,nk->nm", lin["W"], dc.reshape(nf, 6)[lin["s"]]))
    dX = -np.einsum("pkl,pl->pk", Vi, lin["gp"] + acc)
    dX[~P["opt"]] = 0.0
    return dX


def pcg_step(P, lin, lam, cg_tol, cg_max_iters):
    """((dc, dX) or None when the step is rejected, CG iterations)"""
    Vi = point_inverses(P, lin, lam)
    if Vi is None:
        return None, 0
    dc, k = pcg(P, lin, Vi, lam, cg_tol, cg_max_iters)
    if dc is None:
        return None, k
    return (dc, back_substitute(P, lin, Vi, dc)), k


def bundle_adjust_pcg(cams, pts, R, t, K, offsets, X, mask=None, free=None, scale_gauge="auto", loss_scale=None,
                      max_iters=50, px_th=2.0, cg_max_iters=100, cg_tol=0.1, P=None):
    """The whole call: dict(R, t, X, mask, cost0, cost, iters, n_used, cg_iters) as bundle_adjust_pcg_ragged returns
    it"""
    if P is None:
        P = setup(cams, pts, R, t, K, offsets, X, mask, free, scale_gauge, loss_scale)
    R, t, X = P["R"].copy(), P["t"].copy(), P["X"].copy()
    c_cur = c0 = cost(P, R, t, X)
    lam, iters, cg_iters = LAMBDA0, 0, 0
    lin = linearise(P, R, t, X)
    for _ in range(max_iters):
        iters += 1
        step, k = pcg_step(P, lin, lam, cg_tol, cg_max_iters)
        cg_iters += k
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
    return dict(R=R, t=t, X=X, mask=out_mask, cost0=c0, cost=c_cur, iters=iters, n_used=int(P["used"].sum()),
                cg_iters=cg_iters, P=P)
