"""numpy restatement of matching.pose_from_fundamental_ragged -- TEST INFRASTRUCTURE ONLY.

Pose per pair from oracle.frontend_np.pose_from_fundamental; per row, under that pose, the least-squares depths of
l1 R x1 + t = l2 x2, the midpoint 0.5 (l1 x1 + R^T (l2 x2 - t)), in_front = mask & l1 > 0 & l2 > 0 and the parallax
angle atan2(|x1 x R^T x2|, x1 . R^T x2); the per-pair median by np.median.  tests/test_pose_ragged.py pins it to
planted two-view geometry."""
import numpy as np

from oracle.frontend_np import pose_from_fundamental


def rays(K, p):
    return np.linalg.solve(K, np.c_[p[:, :2], np.ones(len(p))].T).T


def rows_under_pose(R, t, K1, K2, p1, p2, mask=None):
    """points [n,3], in_front [n], angle [n] and the depths l1, l2 [n] of the rows under (R, t)"""
    x1, x2 = rays(K1, p1), rays(K2, p2)
    a1 = x1 @ R.T
    aa = (a1 * a1).sum(1); bb = (x2 * x2).sum(1); ab = (a1 * x2).sum(1); at = a1 @ t; bt = x2 @ t
    det = aa * bb - ab * ab
    l1 = (-at * bb + ab * bt) / det
    l2 = (aa * bt - ab * at) / det
    y = x2 @ R                                        # rows of R^T x2
    points = 0.5 * (l1[:, None] * x1 + (l2[:, None] * x2 - t) @ R)
    angle = np.arctan2(np.linalg.norm(np.cross(x1, y), axis=1), (x1 * y).sum(1))
    m = np.ones(len(p1), bool) if mask is None else np.asarray(mask, bool)
    return points, m & (l1 > 0) & (l2 > 0), angle, l1, l2


def pose_ragged(F, K1, K2, p1, p2, offsets, mask=None):
    """The whole batch: dict of R [P,3,3], t [P,3], good [P], points [rows,3], in_front [rows], angle [rows],
    median_angle [P], l1 / l2 [rows] (NaN outside a valid non-degenerate pair).  F [P,9] or [P,3,3]; K [3,3] or
    [P,3,3]."""
    F = np.asarray(F, np.float64).reshape(-1, 3, 3)
    P, rows = len(F), len(p1)
    K1 = np.broadcast_to(K1, (P, 3, 3)); K2 = np.broadcast_to(K2, (P, 3, 3))
    out = dict(R=np.zeros((P, 3, 3)), t=np.zeros((P, 3)), good=np.zeros(P, np.int64),
               points=np.full((rows, 3), np.nan), in_front=np.zeros(rows, bool), angle=np.full(rows, np.nan),
               median_angle=np.full(P, np.nan), l1=np.full(rows, np.nan), l2=np.full(rows, np.nan))
    for p in range(P):
        a, b = int(offsets[p]), int(offsets[p + 1])
        if not 0 <= a <= b <= rows:
            a = b = 0
        if not F[p].any() or np.isnan(F[p]).any():
            continue
        mk = None if mask is None else np.asarray(mask[a:b], bool)
        R, t, good = pose_from_fundamental(F[p], K1[p], K2[p], p1[a:b, :2], p2[a:b, :2], mk)
        out["R"][p], out["t"][p], out["good"][p] = R, t, good
        if b == a:
            continue
        pts, front, ang, l1, l2 = rows_under_pose(R, t, K1[p], K2[p], p1[a:b], p2[a:b], mk)
        out["points"][a:b], out["in_front"][a:b], out["angle"][a:b] = pts, front, ang
        out["l1"][a:b], out["l2"][a:b] = l1, l2
        if front.any():
            out["median_angle"][p] = np.median(ang[front])
    return out
