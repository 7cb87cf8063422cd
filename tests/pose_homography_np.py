"""numpy restatement of matching.pose_from_homography_ragged -- TEST INFRASTRUCTURE ONLY.

Per pair: Hn = K2^-1 H K1 divided by its middle singular value and negated when det(Hn) < 0.  When
max |Hn^T Hn - I| < 1e-3 the pair is a pure rotation: one candidate, R = U V^T (the rotation nearest to Hn), t = 0.
Otherwise the four decompositions Hn = R + t' n^T, |n| = 1, of Malis & Vargas ("Deeper understanding of the homography
decomposition for vision-based control", INRIA RR-6303, 2007, section 4: the analytical method), in the order
(Ra, t'a, na), (Ra, -t'a, -na), (Rb, t'b, nb), (Rb, -t'b, -nb).  The vote, the ranking and the rows are those of
matching.pose_from_homography_ragged; the rows reuse tests.pose_ragged_np.rows_under_pose."""
import numpy as np

from tests.pose_ragged_np import rays, rows_under_pose

ROTATION_TOL = 1e-3


def _sign(x):
    return 1.0 if x >= 0 else -1.0


def normalised(H, K1, K2):
    """Hn = K2^-1 H K1 / sigma_2(.), with det(Hn) > 0"""
    Hn = np.linalg.solve(K2, H @ K1)
    Hn = Hn / np.linalg.svd(Hn, compute_uv=False)[1]
    return -Hn if np.linalg.det(Hn) < 0 else Hn


def nearest_rotation(Hn):
    U, _, Vt = np.linalg.svd(Hn)
    return U @ Vt


def decompose(Hn):
    """the four (R, t', n) of Hn = R + t' n^T (Hn normalised as above, not a rotation)"""
    S = Hn.T @ Hn - np.eye(3)
    # opposites of the principal minors of S, and of the off-diagonal ones
    m11 = S[1, 2] ** 2 - S[1, 1] * S[2, 2]
    m22 = S[0, 2] ** 2 - S[0, 0] * S[2, 2]
    m33 = S[0, 1] ** 2 - S[0, 0] * S[1, 1]
    m12 = S[1, 2] * S[0, 2] - S[0, 1] * S[2, 2]
    m13 = S[1, 1] * S[0, 2] - S[0, 1] * S[1, 2]
    m23 = S[0, 1] * S[0, 2] - S[0, 0] * S[1, 2]
    r11, r22, r33 = (np.sqrt(max(m, 0.0)) for m in (m11, m22, m33))
    d = np.abs(np.diag(S))
    i = 0 if d[0] >= d[1] and d[0] >= d[2] else (1 if d[1] >= d[2] else 2)
    if i == 0:
        e = _sign(m23)
        na = np.array([S[0, 0], S[0, 1] + r33, S[0, 2] + e * r22])
        nb = np.array([S[0, 0], S[0, 1] - r33, S[0, 2] - e * r22])
    elif i == 1:
        e = _sign(m13)
        na = np.array([S[0, 1] + r33, S[1, 1], S[1, 2] - e * r11])
        nb = np.array([S[0, 1] - r33, S[1, 1], S[1, 2] + e * r11])
    else:
        e = _sign(m12)
        na = np.array([S[0, 2] + e * r22, S[1, 2] + r11, S[2, 2]])
        nb = np.array([S[0, 2] - e * r22, S[1, 2] - r11, S[2, 2]])
    na, nb = na / np.linalg.norm(na), nb / np.linalg.norm(nb)
    tr = np.trace(S)
    nu = 2.0 * np.sqrt(max(1.0 + tr - m11 - m22 - m33, 0.0))
    rho = np.sqrt(2.0 + tr + nu)
    te = np.sqrt(max(2.0 + tr - nu, 0.0))
    es = _sign(S[i, i])
    ta_s = 0.5 * te * (es * rho * nb - te * na)          # t' in camera 1's frame (R^T t')
    tb_s = 0.5 * te * (es * rho * na - te * nb)
    Ra = Hn @ (np.eye(3) - (2.0 / nu) * np.outer(ta_s, na))
    Rb = Hn @ (np.eye(3) - (2.0 / nu) * np.outer(tb_s, nb))
    ta, tb = Ra @ ta_s, Rb @ tb_s
    return [(Ra, ta, na), (Ra, -ta, -na), (Rb, tb, nb), (Rb, -tb, -nb)]


def candidates(H, K1, K2):
    """(rotation_only, list of (R, t', n)): one (R, 0, NaN) for a rotation, else the four decompositions"""
    Hn = normalised(np.asarray(H, np.float64).reshape(3, 3), K1, K2)
    S = Hn.T @ Hn - np.eye(3)
    if np.abs(S).max() < ROTATION_TOL:
        return True, [(nearest_rotation(Hn), np.zeros(3), np.full(3, np.nan))]
    return False, decompose(Hn)


def votes(rotation_only, cands, K1, K2, p1, p2, mask=None):
    """per candidate, the rows with mask != 0 that it puts in front of both cameras (x1 . R^T x2 > 0 for a rotation)"""
    m = np.ones(len(p1), bool) if mask is None else np.asarray(mask, bool)
    out = []
    for R, t, _ in cands:
        if rotation_only:
            x1, x2 = rays(K1, p1), rays(K2, p2)
            out.append(int((m & ((x1 * (x2 @ R)).sum(1) > 0)).sum()))
        else:
            out.append(int(rows_under_pose(R, t / np.linalg.norm(t), K1, K2, p1, p2, m)[1].sum()))
    return out


def ranking(v):
    """candidate 0: the most votes; candidate 1: the most among the rest; ties to the earlier candidate"""
    first = int(np.argmax(v))
    rest = [c for c in range(len(v)) if c != first]
    return [first] + ([max(rest, key=lambda c: (v[c], -c))] if rest else [])


def pose_h_ragged(H, K1, K2, p1, p2, offsets, mask=None):
    """The whole batch: dict of R [P,2,3,3], t [P,2,3], plane [P,2,4], good [P,2], rotation_only [P], points [rows,3],
    in_front [rows], angle [rows], median_angle [P], l1 / l2 [rows].  H [P,9] or [P,3,3]; K [3,3] or [P,3,3]."""
    H = np.asarray(H, np.float64).reshape(-1, 3, 3)
    P, rows = len(H), len(p1)
    K1 = np.broadcast_to(K1, (P, 3, 3)); K2 = np.broadcast_to(K2, (P, 3, 3))
    out = dict(R=np.zeros((P, 2, 3, 3)), t=np.zeros((P, 2, 3)), plane=np.full((P, 2, 4), np.nan),
               good=np.zeros((P, 2), np.int64), rotation_only=np.zeros(P, bool),
               points=np.full((rows, 3), np.nan), in_front=np.zeros(rows, bool), angle=np.full(rows, np.nan),
               median_angle=np.full(P, np.nan), l1=np.full(rows, np.nan), l2=np.full(rows, np.nan))
    for p in range(P):
        a, b = int(offsets[p]), int(offsets[p + 1])
        if not 0 <= a <= b <= rows:
            a = b = 0
        if not H[p].any() or np.isnan(H[p]).any():
            continue
        mk = None if mask is None else np.asarray(mask[a:b], bool)
        rot, cands = candidates(H[p], K1[p], K2[p])
        v = votes(rot, cands, K1[p], K2[p], p1[a:b], p2[a:b], mk)
        out["rotation_only"][p] = rot
        for slot, c in enumerate(ranking(v)):
            R, t, n = cands[c]
            tn = np.linalg.norm(t)
            out["R"][p, slot] = R
            out["good"][p, slot] = v[c]
            if not rot:
                out["t"][p, slot] = t / tn
                out["plane"][p, slot] = np.r_[n, 1.0 / tn]
        if b == a:
            continue
        R0, t0 = out["R"][p, 0], out["t"][p, 0]
        pts, front, ang, l1, l2 = rows_under_pose(R0, t0, K1[p], K2[p], p1[a:b], p2[a:b], mk)
        if rot:
            m = np.ones(b - a, bool) if mk is None else mk
            x1, x2 = rays(K1[p], p1[a:b]), rays(K2[p], p2[a:b])
            front = m & ((x1 * (x2 @ R0)).sum(1) > 0)
            pts = np.full_like(pts, np.nan)
        out["points"][a:b], out["in_front"][a:b], out["angle"][a:b] = pts, front, ang
        out["l1"][a:b], out["l2"][a:b] = l1, l2
        if front.any():
            out["median_angle"][p] = np.median(ang[front])
    return out
