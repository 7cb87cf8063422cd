"""numpy oracle of the view-graph calibration (matching.calibrate_view_graph, csrc/view_graph_calibration.cu): the
estimator of include/degensac_b200.h line for line.  The per-thread functions of csrc/view_graph_calibration.h are
restated per edge; the SVD is numpy's, whose singular vectors may differ from the device's in sign (r2 changes sign
with them, s = r1^2 + r2^2 and the step do not).  The sums of the normal equations and of CG are taken in numpy's
order.

An edge's constants c [12] are alpha [3], beta [3], gamma [3], delta [3]; A_k = alpha_k e^{2 ti} + beta_k, B_k =
gamma_k e^{2 tj} + delta_k."""
import numpy as np
import scipy.sparse as sp

MIN_S2 = 1e-6
LAMBDA0, LAMBDA_MIN, LAMBDA_MAX, REL_DECREASE = 1e-3, 1e-12, 1e8, 1e-12


def K_of(k):
    """the pinhole K of an intrinsics row (f, cx, cy, k1, k2)"""
    return np.array([[k[0], 0.0, k[1]], [0.0, k[0], k[2]], [0.0, 0.0, 1.0]])


def intrinsics_ok(k):
    k = np.asarray(k, dtype=np.float64)
    return bool(np.isfinite(k).all() and k[0] > 0.0)


def constants(F, ki, kj):
    """c [12] of F [3,3] between the start intrinsics ki (view i) and kj (view j), or None (vg_constants)"""
    G = K_of(kj).T @ np.asarray(F, dtype=np.float64).reshape(3, 3) @ K_of(ki)
    n = np.linalg.norm(G)
    if not (np.isfinite(n) and n > 0.0):
        return None
    G = G / n
    _, s, Vt = np.linalg.svd(G)
    s1, s2 = s[0], s[1]
    if not s2 > MIN_S2 * s1:
        return None
    v1, v2 = Vt[0], Vt[1]
    u1, u2 = G @ v1 / s1, G @ v2 / s2
    xy = lambda p, q: p[0] * q[0] + p[1] * q[1]
    return np.array([s1 * s1 * xy(v1, v1), s1 * s2 * xy(v1, v2), s2 * s2 * xy(v2, v2),
                     s1 * s1 * v1[2] * v1[2], s1 * s2 * v1[2] * v2[2], s2 * s2 * v2[2] * v2[2],
                     xy(u2, u2), -xy(u1, u2), xy(u1, u1),
                     u2[2] * u2[2], -u1[2] * u2[2], u1[2] * u1[2]])


def residuals_v(c, ti, tj):
    """residuals over edges: c [P,12], ti, tj [P] -> (r [P,2], J [P,2,2] with columns (ti, tj), s [P])"""
    a, b = np.exp(2.0 * ti)[:, None], np.exp(2.0 * tj)[:, None]
    A, B = c[:, 0:3] * a + c[:, 3:6], c[:, 6:9] * b + c[:, 9:12]
    dA, dB = 2.0 * c[:, 0:3] * a, 2.0 * c[:, 6:9] * b
    P, Q = A[:, 0] * B[:, 2], A[:, 2] * B[:, 0]
    den = P + Q
    qa, qb = 1.0 / np.sqrt(A[:, 0] * A[:, 2]), 1.0 / np.sqrt(B[:, 0] * B[:, 2])
    ra, rb = A[:, 1] * qa, B[:, 1] * qb
    r = np.stack([(P - Q) / den, 0.5 * (ra - rb)], 1)
    id2 = 2.0 / (den * den)
    J = np.empty((len(c), 2, 2))
    J[:, 0, 0] = id2 * (Q * (dA[:, 0] * B[:, 2]) - P * (dA[:, 2] * B[:, 0]))
    J[:, 0, 1] = id2 * (Q * (A[:, 0] * dB[:, 2]) - P * (A[:, 2] * dB[:, 0]))
    J[:, 1, 0] = 0.5 * (dA[:, 1] * qa - 0.5 * ra * (dA[:, 0] / A[:, 0] + dA[:, 2] / A[:, 2]))
    J[:, 1, 1] = -0.5 * (dB[:, 1] * qb - 0.5 * rb * (dB[:, 0] / B[:, 0] + dB[:, 2] / B[:, 2]))
    return r, J, r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]


def residuals(c, ti, tj):
    """(r [2], J [2,2] with columns (ti, tj), s) of one edge (vg_residuals)"""
    r, J, s = residuals_v(np.asarray(c, dtype=np.float64)[None], np.array([ti], dtype=np.float64),
                          np.array([tj], dtype=np.float64))
    return r[0], J[0], float(s[0])


def rho(s, sig2):
    return sig2 * np.log1p(s / sig2) if sig2 > 0.0 else s


def weight(s, sig2):
    return 1.0 / (1.0 + s / sig2) if sig2 > 0.0 else 1.0


def cost_term(s, sig2):
    return rho(s, sig2) if s < np.inf else np.inf


def prepare(pairs, F, groups, intrinsics, mask=None):
    """(used [P] bool, consts [P,12] (NaN where not used), gi [P], gj [P])"""
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    F = np.asarray(F, dtype=np.float64).reshape(-1, 9)
    groups = np.asarray(groups, dtype=np.int64)
    kin = np.asarray(intrinsics, dtype=np.float64).reshape(-1, 5)
    C, G, P = len(groups), len(kin), len(pairs)
    ii, jj = pairs[:, 0], pairs[:, 1]
    inside = (ii != jj) & (ii >= 0) & (jj >= 0) & (ii < C) & (jj < C)
    if mask is not None:
        inside &= np.asarray(mask).astype(bool)
    a = np.where(inside, groups[np.clip(ii, 0, C - 1)], -1)
    b = np.where(inside, groups[np.clip(jj, 0, C - 1)], -1)
    kok = np.isfinite(kin).all(1) & (kin[:, 0] > 0.0)
    ok = inside & np.isfinite(F).all(1) & (a >= 0) & (a < G) & (b >= 0) & (b < G)
    ok[ok] &= kok[a[ok]] & kok[b[ok]]
    consts = np.full((P, 12), np.nan)
    e = np.flatnonzero(ok)
    Ki, Kj = _K_batch(kin[a[e]]), _K_batch(kin[b[e]])
    with np.errstate(all="ignore"):
        Gm = np.einsum("pji,pjk,pkl->pil", Kj, F[e].reshape(-1, 3, 3), Ki)
        n = np.sqrt((Gm * Gm).sum((1, 2)))
        fin = np.isfinite(n) & (n > 0.0)
        Gm = np.where(fin[:, None, None], Gm / np.where(fin, n, 1.0)[:, None, None], np.eye(3))
        _, sv, Vt = np.linalg.svd(Gm)
        s1, s2 = sv[:, 0], sv[:, 1]
        fin &= s2 > MIN_S2 * s1
        v1, v2 = Vt[:, 0], Vt[:, 1]
        u1 = np.einsum("pij,pj->pi", Gm, v1) / s1[:, None]
        u2 = np.einsum("pij,pj->pi", Gm, v2) / s2[:, None]
    xy = lambda p, q: p[:, 0] * q[:, 0] + p[:, 1] * q[:, 1]  # noqa: E731
    c = np.stack([s1 * s1 * xy(v1, v1), s1 * s2 * xy(v1, v2), s2 * s2 * xy(v2, v2),
                  s1 * s1 * v1[:, 2] * v1[:, 2], s1 * s2 * v1[:, 2] * v2[:, 2], s2 * s2 * v2[:, 2] * v2[:, 2],
                  xy(u2, u2), -xy(u1, u2), xy(u1, u1),
                  u2[:, 2] * u2[:, 2], -u1[:, 2] * u2[:, 2], u1[:, 2] * u1[:, 2]], 1)
    ok[e] = fin
    consts[e[fin]] = c[fin]
    gi = np.where(ok, a, -1)
    gj = np.where(ok, b, -1)
    return ok, consts, gi, gj


def _K_batch(k):
    K = np.zeros((len(k), 3, 3))
    K[:, 0, 0] = K[:, 1, 1] = k[:, 0]
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = k[:, 1], k[:, 2], 1.0
    return K


def edge_costs(consts, used, gi, gj, theta, sig2):
    """per-edge (cost term, s) at theta [G]; 0 and NaN for an edge that is not used"""
    P = len(used)
    cost, s = np.zeros(P), np.full(P, np.nan)
    u = np.flatnonzero(used)
    with np.errstate(all="ignore"):
        _, _, se = residuals_v(consts[u], theta[gi[u]], theta[gj[u]])
        s[u] = se
        cost[u] = np.where(se < np.inf, sig2 * np.log1p(se / sig2) if sig2 > 0.0 else se, np.inf)
    return cost, s


def linearise(consts, used, gi, gj, theta, sig2, G):
    """the normal equations at theta: H [G,G] (sparse) = sum J^T w J and g [G] = sum J^T w r over the used edges (an
    edge inside one group contributes one column, the sum of its two)"""
    u = np.flatnonzero(used)
    with np.errstate(all="ignore"):                  # (a point far out gives a non-finite H, which rejects the step)
        r, J, s = residuals_v(consts[u], theta[gi[u]], theta[gj[u]])
    w = 1.0 / (1.0 + s / sig2) if sig2 > 0.0 else np.ones(len(u))
    a, b = gi[u], gj[u]
    one = a == b
    ci = np.where(one[:, None], J[:, :, 0] + J[:, :, 1], J[:, :, 0])
    cj = np.where(one[:, None], 0.0, J[:, :, 1])
    dii, djj, dij = w * (ci * ci).sum(1), w * (cj * cj).sum(1), w * (ci * cj).sum(1)
    rows = np.r_[a, b, a, b]
    cols = np.r_[a, b, b, a]
    vals = np.r_[dii, djj, dij, dij]
    H = sp.coo_matrix((vals, (rows, cols)), shape=(G, G)).tocsr()
    g = np.bincount(a, w * (ci * r).sum(1), minlength=G) + np.bincount(b, w * (cj * r).sum(1), minlength=G)
    return H, g


def pcg(A, m, b, cg_tol, cg_max_iters):
    """Jacobi-preconditioned CG on A x = b, M = diag(m), the device's loop (pcg_run): stops at |r| <= cg_tol |b| or
    after cg_max_iters iterations; (x, iterations, reject) where reject: the first p . q is not positive or finite"""
    x = np.zeros_like(b)
    r = b.copy()
    z = r / m
    bb, rho_ = float(b @ b), float(r @ z)
    p = np.zeros_like(b)
    beta, it = 0.0, 0
    if not bb > 0.0:
        return x, 0, False
    while True:
        p = z + beta * p
        q = A @ p
        kappa = float(p @ q)
        it += 1
        if not (kappa > 0.0 and np.isfinite(kappa)):
            return x, it, it == 1
        alpha = rho_ / kappa
        x = x + alpha * p
        r = r - alpha * q
        z = r / m
        rr, rz = float(r @ r), float(r @ z)
        if rr <= cg_tol * cg_tol * bb or it >= cg_max_iters:
            return x, it, False
        beta = rz / rho_
        rho_ = rz


def damped(H, lam, active):
    """H + lam diag(H) over the active groups, identity rows and columns for the others (sparse); and its Jacobi
    diagonal"""
    H = sp.csr_matrix(H)
    d = H.diagonal().copy()
    keep = sp.diags(active.astype(np.float64))
    A = keep @ (H + lam * sp.diags(d)) @ keep + sp.diags((~active).astype(np.float64))
    m = np.where(active, (1.0 + lam) * d, 1.0)
    return A.tocsr(), m


def calibrate_view_graph(pairs, F, groups, intrinsics, mask=None, loss_scale=1e-2, max_error=1e-2, max_ratio=10.0,
                         max_iters=100, cg_max_iters=500, cg_tol=1e-6):
    """dict(intrinsics [G,5], refined [G], error [P], inliers [P], theta [G], cost0, cost, iters, n_used, cg_iters)"""
    kin = np.asarray(intrinsics, dtype=np.float64).reshape(-1, 5)
    G = len(kin)
    sig2 = loss_scale * loss_scale
    used, consts, gi, gj = prepare(pairs, F, groups, kin, mask)
    active = np.zeros(G, bool)
    active[gi[used]] = True
    active[gj[used]] = True
    theta = np.zeros(G)
    cost = float(edge_costs(consts, used, gi, gj, theta, sig2)[0].sum())
    cost0 = cost
    lam, lin, stop, iters, cg_iters = LAMBDA0, True, False, 0, 0
    H = g = None
    for _ in range(max_iters):
        if stop:
            break
        if lin:
            H, g = linearise(consts, used, gi, gj, theta, sig2, G)
        A, m = damped(H, lam, active)
        b = np.where(active, -g, 0.0)
        bad = not (np.isfinite(m).all() and (m > 0.0).all() and np.isfinite(b).all())
        c_new = cost
        if not bad:
            x, k, rej = pcg(A, m, b, cg_tol, cg_max_iters)
            cg_iters += k
            bad = rej
            if not bad:
                trial = np.where(active, theta + x, theta)
                c_new = float(edge_costs(consts, used, gi, gj, trial, sig2)[0].sum())
        go = not bad
        better = go and c_new < cost
        flat = go and abs(cost - c_new) < REL_DECREASE * cost
        iters += 1
        if better:
            cost, theta, lam, lin = c_new, trial, max(lam / 10.0, LAMBDA_MIN), True
            stop = flat
        else:
            lin = False
            lam *= 10.0
            stop = flat or lam > LAMBDA_MAX
    kout = kin.copy()
    refined = np.zeros(G, bool)
    for q in range(G):
        ratio = np.exp(theta[q])
        refined[q] = active[q] and 1.0 / max_ratio <= ratio <= max_ratio
        if refined[q]:
            kout[q, 0] = kin[q, 0] * ratio
    theta_eff = np.where(refined, theta, 0.0)
    _, s = edge_costs(consts, used, gi, gj, theta_eff, sig2)
    error = np.where(used, np.sqrt(s), np.nan)
    with np.errstate(invalid="ignore"):
        inliers = used & (error <= max_error)
    return dict(intrinsics=kout, refined=refined, error=error, inliers=inliers, theta=theta, cost0=cost0, cost=cost,
                iters=iters, n_used=int(used.sum()), cg_iters=cg_iters, used=used)


# ------------------------------------------------------------------------------------------------ scenes
def look_at(c, target, rng=None, roll=0.0):
    """the world-to-camera R of a camera at c looking at target"""
    z = np.asarray(target, float) - c
    z /= np.linalg.norm(z)
    up = np.array([0.0, 1.0, 0.0])
    x = np.cross(up, z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    if roll:
        cr, sr = np.cos(roll), np.sin(roll)
        R = np.array([[cr, -sr, 0.0], [sr, cr, 0.0], [0.0, 0.0, 1.0]]) @ R
    return R


def fundamental(Ki, Ri, ti, Kj, Rj, tj):
    """F with x_j^T F x_i = 0 for the world-to-camera poses (R, t) of views i and j"""
    R = Rj @ Ri.T
    t = tj - R @ ti
    tx = np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])
    return np.linalg.inv(Kj).T @ tx @ R @ np.linalg.inv(Ki)


def random_views(rng, n, spread=0.6):
    """n views with random, non-degenerate poses: centres scattered around a ring, each looking at a jittered point
    near the origin and rolled, so that no two optical axes meet at one point"""
    Rs, ts = [], []
    for v in range(n):
        a = 2.0 * np.pi * v / n + rng.uniform(-0.2, 0.2)
        c = np.array([4.0 * np.cos(a * spread), rng.uniform(-1.0, 1.0), 4.0 * np.sin(a * spread) - 6.0])
        target = rng.uniform(-0.8, 0.8, 3)
        R = look_at(c, target, roll=rng.uniform(-0.5, 0.5))
        Rs.append(R)
        ts.append(-R @ c)
    return np.array(Rs), np.array(ts)
