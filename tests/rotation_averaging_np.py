"""numpy oracle of the rotation averaging (matching.average_rotations, csrc/rotation_averaging.cu): the estimator of
include/degensac_b200.h line for line, vectorised over edges and views.  The per-thread functions of
csrc/rotation_averaging.h are restated with the device's operation order (no FMA), so the tree start matches the
device to rounding; the sums of the Laplacian and of CG are taken in numpy's order.

Rotations are [..., 3, 3] arrays, row-major as on the device."""
import numpy as np
import scipy.sparse as sp

SMALL, NEAR_PI, L1_FLOOR, MIN_DET, ORTHO_TOL = 1e-4, 1e-3, 1e-3, 0.5, 1e-12


def mul(A, B):
    """A B over [..., 3, 3], each entry a0 b0 + a1 b1 + a2 b2 in that order (pr_mul3)"""
    return (A[..., :, 0, None] * B[..., None, 0, :] + A[..., :, 1, None] * B[..., None, 1, :]) + \
        A[..., :, 2, None] * B[..., None, 2, :]


def mul_tn(A, B):
    """A^T B (ra_mul3_tn)"""
    return mul(np.swapaxes(A, -1, -2), B)


def drift(R):
    """largest |R R^T - I| entry (pr_ortho_drift)"""
    return np.abs(mul(R, np.swapaxes(R, -1, -2)) - np.eye(3)).max(axis=(-2, -1))


def _unit(v):
    return v * (1.0 / np.sqrt(v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1] + v[..., 2] * v[..., 2]))[..., None]


def orthonormalise(R):
    """Gram-Schmidt on the rows, the third their cross product (pr_orthonormalise)"""
    R = R.copy()
    R[..., 0, :] = _unit(R[..., 0, :])
    p = R[..., 0, 0] * R[..., 1, 0] + R[..., 0, 1] * R[..., 1, 1] + R[..., 0, 2] * R[..., 1, 2]
    R[..., 1, :] = _unit(R[..., 1, :] - p[..., None] * R[..., 0, :])
    R[..., 2, :] = np.cross(R[..., 0, :], R[..., 1, :])
    return R


def edge_ok(R):
    """finite with det > 0.5 (ra_edge_ok)"""
    with np.errstate(invalid="ignore"):
        fin = np.isfinite(R).all(axis=(-2, -1))
        Rz = np.where(fin[..., None, None], R, 0.0)
        det = Rz[..., 0, 0] * (Rz[..., 1, 1] * Rz[..., 2, 2] - Rz[..., 1, 2] * Rz[..., 2, 1]) - \
            Rz[..., 0, 1] * (Rz[..., 1, 0] * Rz[..., 2, 2] - Rz[..., 1, 2] * Rz[..., 2, 0]) + \
            Rz[..., 0, 2] * (Rz[..., 1, 0] * Rz[..., 2, 1] - Rz[..., 1, 1] * Rz[..., 2, 0])
    return fin & (det > MIN_DET)


def log_map(dR):
    """(r [..., 3], theta [...]) of ra_log"""
    dR = np.asarray(dR, dtype=np.float64)
    a = np.stack([dR[..., 2, 1] - dR[..., 1, 2], dR[..., 0, 2] - dR[..., 2, 0], dR[..., 1, 0] - dR[..., 0, 1]], -1)
    s = np.sqrt(a[..., 0] * a[..., 0] + a[..., 1] * a[..., 1] + a[..., 2] * a[..., 2])
    c2 = dR[..., 0, 0] + dR[..., 1, 1] + dR[..., 2, 2] - 1.0
    th = np.arctan2(s, c2)
    t2 = th * th
    with np.errstate(divide="ignore", invalid="ignore"):
        f = np.where(th < SMALL, 0.5 * (1.0 + t2 / 6.0 + 7.0 * t2 * t2 / 360.0), th / (2.0 * np.sin(th)))
    r = f[..., None] * a
    far = th > np.pi - NEAR_PI
    if far.any():
        D, A, T, C = dR[far], a[far], th[far], 0.5 * c2[far]
        k = np.where((D[:, 0, 0] >= D[:, 1, 1]) & (D[:, 0, 0] >= D[:, 2, 2]), 0, np.where(D[:, 1, 1] >= D[:, 2, 2], 1, 2))
        idx = np.arange(len(k))
        n = 0.5 * (D[idx, :, k] + D[idx, k, :])
        n[idx, k] -= C
        inv = 1.0 / np.sqrt(n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2])
        sg = np.where(n[:, 0] * A[:, 0] + n[:, 1] * A[:, 1] + n[:, 2] * A[:, 2] < 0.0, -inv, inv)
        r[far] = (T * sg)[:, None] * n
    return r, th


def expmap(w):
    """exp([w]x), Rodrigues"""
    w = np.asarray(w, dtype=np.float64)
    th = np.linalg.norm(w)
    W = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    if th == 0.0:
        return np.eye(3)
    return np.eye(3) + np.sin(th) / th * W + (1 - np.cos(th)) / th ** 2 * W @ W


def weight(phase, th, sig2):
    """ra_weight"""
    if phase == 0:
        return 1.0 / np.where(th > L1_FLOOR, th, L1_FLOOR)
    q = sig2 / (sig2 + th * th)
    return q * q


def gm_cost(th, sig2):
    """sum of rho_GM(theta) = sig2 theta^2 / (sig2 + theta^2)"""
    return float(np.sum(sig2 * th * th / (sig2 + th * th)))


def update(R, w):
    """R exp([w]x) = exp([R w]x) R by ap_step's arithmetic, re-orthonormalised past ORTHO_TOL (ra_update), over
    [..., 3, 3] and [..., 3]"""
    D = R[..., :, 0] * w[..., 0, None] + R[..., :, 1] * w[..., 1, None] + R[..., :, 2] * w[..., 2, None]
    a = np.sqrt(D[..., 0] * D[..., 0] + D[..., 1] * D[..., 1] + D[..., 2] * D[..., 2])
    with np.errstate(divide="ignore", invalid="ignore"):
        h = np.sin(0.5 * a) / a
        c1 = np.where(a != 0.0, np.sin(a) / a, 1.0)
        c2 = np.where(a != 0.0, 2.0 * h * h, 0.5)
    z = np.zeros_like(a)
    W = np.stack([np.stack([z, -D[..., 2], D[..., 1]], -1), np.stack([D[..., 2], z, -D[..., 0]], -1),
                  np.stack([-D[..., 1], D[..., 0], z], -1)], -2)
    E = np.eye(3) + c1[..., None, None] * W + c2[..., None, None] * mul(W, W)
    R2 = mul(E, R)
    bad = drift(R2) > ORTHO_TOL
    if np.any(bad):
        R2[bad] = orthonormalise(R2[bad])
    return R2


# ------------------------------------------------------------------------------------------------ graph
def prepare(pairs, R_rel, mask=None, weights=None):
    """(valid [P] bool, the prepared R_e [P,3,3], weights [P] int64) of step 1"""
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    Re = np.asarray(R_rel, dtype=np.float64).reshape(-1, 3, 3).copy()
    P = len(pairs)
    w = np.zeros(P, np.int64) if weights is None else np.asarray(weights, dtype=np.int64)
    m = np.ones(P, bool) if mask is None else np.asarray(mask).astype(bool)
    valid = (pairs[:, 0] != pairs[:, 1]) & m & (w >= 0) & edge_ok(Re)
    fix = valid & (drift(np.where(valid[:, None, None], Re, 0.0)) > ORTHO_TOL)
    if fix.any():
        Re[fix] = orthonormalise(Re[fix])
    return valid, Re, w


def _find(parent, x):
    while parent[x] != x:
        parent[x] = parent[parent[x]]
        x = parent[x]
    return x


def spanning_forest(pairs, valid, w, n_views):
    """(in_tree [P] bool, component [n_views]: the smallest view of each component or -1) by Kruskal's algorithm under
    the strict order of step 3 (which gives the same unique forest as the device's Boruvka rounds)"""
    pairs = np.asarray(pairs, dtype=np.int64)
    idx = np.flatnonzero(valid)
    order = idx[np.lexsort((idx, -w[idx]))]
    parent = list(range(n_views))
    in_tree = np.zeros(len(pairs), bool)
    for e in order:
        a, b = _find(parent, pairs[e, 0]), _find(parent, pairs[e, 1])
        if a != b:
            if a > b:
                a, b = b, a
            parent[b] = a
            in_tree[e] = True
    comp = np.array([_find(parent, v) for v in range(n_views)], dtype=np.int64)
    deg = np.zeros(n_views, np.int64)
    np.add.at(deg, pairs[valid, 0], 1)
    np.add.at(deg, pairs[valid, 1], 1)
    comp[deg == 0] = -1
    return in_tree, comp


def tree_start(pairs, Re, in_tree, comp, n_views):
    """(R [n_views,3,3], level [n_views]) of step 3: I at each root, then level by level down the forest"""
    pairs = np.asarray(pairs, dtype=np.int64)
    R = np.full((n_views, 3, 3), np.nan)
    level = np.full(n_views, -1, np.int64)
    roots = np.flatnonzero(comp == np.arange(n_views))
    R[roots] = np.eye(3)
    level[roots] = 0
    te = np.flatnonzero(in_tree)
    i, j = pairs[te, 0], pairs[te, 1]
    d = 0
    while True:
        down_j = (level[i] == d) & (level[j] < 0)          # child j: R_j = R_e R_i
        down_i = (level[j] == d) & (level[i] < 0)          # child i: R_i = R_e^T R_j
        if not (down_j.any() or down_i.any()):
            break
        cj, ci = te[down_j], te[down_i]
        R[pairs[cj, 1]] = mul(Re[cj], R[pairs[cj, 0]])
        R[pairs[ci, 0]] = mul_tn(Re[ci], R[pairs[ci, 1]])
        level[pairs[cj, 1]] = d + 1
        level[pairs[ci, 0]] = d + 1
        d += 1
    return R, level


def residuals(pairs, Re, R, valid):
    """(r [P,3], theta [P]) of step 4 over the valid edges (0 elsewhere)"""
    pairs = np.asarray(pairs, dtype=np.int64)
    r = np.zeros((len(pairs), 3))
    th = np.zeros(len(pairs))
    v = np.flatnonzero(valid)
    if len(v):
        dR = mul_tn(R[pairs[v, 1]], mul(Re[v], R[pairs[v, 0]]))
        r[v], th[v] = log_map(dR)
    return r, th


def laplacian(pairs, we, valid, pinned, n_views):
    """(the pinned Laplacian as a sparse [n, n] matrix, its diagonal) of step 5, per coordinate"""
    pairs = np.asarray(pairs, dtype=np.int64)
    v = np.flatnonzero(valid)
    i, j, w = pairs[v, 0], pairs[v, 1], we[v]
    d = np.zeros(n_views)
    np.add.at(d, i, w)
    np.add.at(d, j, w)
    A = sp.coo_matrix((np.r_[w, w], (np.r_[i, j], np.r_[j, i])), shape=(n_views, n_views)).tocsr()
    keep = sp.diags((~pinned).astype(np.float64))
    d = np.where(pinned, 1.0, d)
    S = sp.diags(d) - keep @ A @ keep
    return S.tocsr(), d


def rhs(pairs, r, we, valid, pinned, n_views):
    """b [n, 3] of step 5: + w r at view j, - w r at view i, 0 at pinned views"""
    pairs = np.asarray(pairs, dtype=np.int64)
    v = np.flatnonzero(valid)
    b = np.zeros((n_views, 3))
    np.add.at(b, pairs[v, 1], we[v, None] * r[v])
    np.add.at(b, pairs[v, 0], -we[v, None] * r[v])
    b[pinned] = 0.0
    return b


def pcg(S, d, b, cg_tol, cg_max_iters):
    """(x [n, 3], iterations, rejected) by step 7's Jacobi-preconditioned CG on S (x) I_3"""
    x = np.zeros_like(b)
    bb = float(np.sum(b * b))
    if not bb > 0.0:
        return x, 0, False
    r = b.copy()
    z = r / d[:, None]
    p = z.copy()
    rho = float(np.sum(r * z))
    it = 0
    while True:
        q = S @ p
        kappa = float(np.sum(p * q))
        it += 1
        if not (kappa > 0.0) or not np.isfinite(kappa):
            return x, it, it == 1
        alpha = rho / kappa
        x = x + alpha * p
        r = r - alpha * q
        rr = float(np.sum(r * r))
        if rr <= cg_tol * cg_tol * bb or it >= cg_max_iters:
            return x, it, False
        z = r / d[:, None]
        rz = float(np.sum(r * z))
        p = z + (rz / rho) * p
        rho = rz


def average_rotations(pairs, R_rel, n_views, mask=None, weights=None, sigma=np.radians(5.0), l1_iters=5,
                      max_iters=100, step_tol=1e-6, cg_max_iters=500, cg_tol=1e-6, trace=None):
    """The whole estimator: dict(R, component, residual, iters, cg_iters, start, in_tree).  trace: a list that gets
    the rotations after each iteration"""
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    valid, Re, w = prepare(pairs, R_rel, mask, weights)
    in_tree, comp = spanning_forest(pairs, valid, w, n_views)
    R, _ = tree_start(pairs, Re, in_tree, comp, n_views)
    start = R.copy()
    pinned = (comp == np.arange(n_views)) | (comp < 0)     # roots and views without an edge
    sig2 = sigma * sigma
    iters, cg_total = [0, 0], 0
    for phase, limit in ((0, l1_iters), (1, max_iters)):
        while iters[phase] < limit:
            r, th = residuals(pairs, Re, R, valid)
            we = np.where(valid, weight(phase, th, sig2), 0.0)
            S, d = laplacian(pairs, we, valid, pinned, n_views)
            b = rhs(pairs, r, we, valid, pinned, n_views)
            x, k, reject = pcg(S, d, b, cg_tol, cg_max_iters)
            cg_total += k
            iters[phase] += 1
            if reject:
                break
            move = ~pinned
            x[~move] = 0.0
            R[move] = update(R[move], x[move])
            if trace is not None:
                trace.append(R.copy())
            if np.sqrt((x * x).sum(1)).max() <= step_tol:
                break
    _, th = residuals(pairs, Re, R, valid)
    return dict(R=R, component=comp, residual=np.where(valid, th, np.nan), iters=np.array(iters),
                cg_iters=cg_total, start=start, in_tree=in_tree)
