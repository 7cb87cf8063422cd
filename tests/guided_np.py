"""numpy restatement of guided matching (match_descriptors_guided) -- TEST INFRASTRUCTURE ONLY.

The dense distance matrix, +inf outside the gate, stable 2-NN, the matcher's ratio rule and mutual check.  The gates
are the header's expressions in float64, in the same operation order (numpy rounds every operation and fuses none),
so they are bit for bit what the kernel evaluates."""
import numpy as np

DBL_MIN = np.finfo(np.float64).tiny


def f_sampson(F, xq, yq, xt, yt):
    """dg::f_resid_sampson(F, xq, yq, xt, yt) (csrc/fgeom.h) elementwise, F [9] row-major with x_t^T F x_q = 0"""
    F = [np.float64(v) for v in np.asarray(F, np.float64).reshape(9)]
    with np.errstate(all="ignore"):
        rxc = F[0] * xt + F[3] * yt + F[6]
        ryc = F[1] * xt + F[4] * yt + F[7]
        rwc = F[2] * xt + F[5] * yt + F[8]
        r = xq * rxc + yq * ryc + rwc
        rx = F[0] * xq + F[1] * yq + F[2]
        ry = F[3] * xq + F[4] * yq + F[5]
        return r * r / (rxc * rxc + ryc * ryc + rx * rx + ry * ry)


def f_pretest_rejects(num, den, th):
    """the kernel's division-free pre-test of the F gate on the numerator r*r and the denominator of f_sampson"""
    with np.errstate(all="ignore"):
        t = th * den
        return (t >= DBL_MIN) & (num > 2.0 * t)


def h_transfer_sq(H, xq, yq, xt, yt):
    """squared distance of (xt, yt) from the transfer of (xq, yq) by H (x_t ~ H x_q, row-major)"""
    H = [np.float64(v) for v in np.asarray(H, np.float64).reshape(9)]
    with np.errstate(all="ignore"):
        w = H[6] * xq + H[7] * yq + H[8]
        px = (H[0] * xq + H[1] * yq + H[2]) / w
        py = (H[3] * xq + H[4] * yq + H[5]) / w
        dx = xt - px
        dy = yt - py
        return dx * dx + dy * dy


def gate(model, guide, kq, kt, px_th):
    """[n1, n2] bool: train j is a candidate of query i (kq [n1,>=2], kt [n2,>=2] keypoints)"""
    th = np.float64(px_th) * np.float64(px_th)
    xq, yq = kq[:, 0:1].astype(np.float64), kq[:, 1:2].astype(np.float64)
    xt, yt = kt[None, :, 0].astype(np.float64), kt[None, :, 1].astype(np.float64)
    e = (f_sampson if guide == "F" else h_transfer_sq)(model, xq, yq, xt, yt)
    with np.errstate(invalid="ignore"):
        return e <= th


def distances(d1, d2, hamming=False):
    """float64 [n1, n2]: Hamming distances of uint8 rows, or squared L2 of float32 rows summed in float64 (the kernel's
    FP32 value exactly when every partial sum is exact in FP32, e.g. for descriptors on a coarse dyadic grid)"""
    if hamming:
        d1 = np.asarray(d1, np.uint8); d2 = np.asarray(d2, np.uint8)
        out = np.empty((len(d1), len(d2)), np.float64)
        for i in range(0, len(d1), 64):
            out[i:i + 64] = np.bitwise_count(d1[i:i + 64, None, :] ^ d2[None, :, :]).sum(2, dtype=np.int64)
        return out
    a = np.asarray(d1, np.float32).astype(np.float64); b = np.asarray(d2, np.float32).astype(np.float64)
    if grid_exact(a) and grid_exact(b):   # |a|^2 + |b|^2 - 2 a.b is then exact in float64 too
        return ((a * a).sum(1)[:, None] + (b * b).sum(1)[None, :]) - 2.0 * (a @ b.T)
    out = np.empty((len(a), len(b)), np.float64)
    for i in range(len(a)):
        out[i] = ((b - a[i]) ** 2).sum(1)
    return out


def grid_exact(a):
    """values on the grid of 1/8 with magnitude < 8: products and sums of up to 256 of them are exact in float64"""
    return bool(np.all(np.abs(a) < 8) and np.all(a * 8 == np.round(a * 8)))


def select(dist, admit, ratio=0.9, mutual=False, hamming=False):
    """2-NN among the admitted candidates, ratio test and mutual check of the matcher: returns (queries, trains)"""
    n1, n2 = dist.shape
    if n1 < 1 or n2 < 2:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    Dm = np.where(admit, dist, np.inf)
    rows = np.arange(n1)
    nn = np.argmin(Dm, 1)                      # the first of the smallest: ties to the lowest train index
    b1 = Dm[rows, nn]
    rest = Dm.copy()
    rest[rows, nn] = np.inf
    b2 = rest.min(1)                           # second smallest of the multiset (a tie at the minimum gives b2 == b1)
    has = admit.any(1)
    if hamming:
        with np.errstate(invalid="ignore"):
            ok = b1 < float(ratio) * b2
    else:
        r32 = np.float32(ratio)
        r2 = np.float32(r32 * r32)
        with np.errstate(invalid="ignore", over="ignore"):
            ok = b1.astype(np.float32) < r2 * b2.astype(np.float32)
    ok &= has
    if mutual:
        ok &= np.argmin(Dm, 0)[nn] == rows
    q = np.nonzero(ok)[0]
    return q, nn[q]


def match_descriptors_guided(d1, d2, kq, kt, model, guide, px_th, ratio=0.9, mutual=False, hamming=False, dist=None):
    """one pair of guided matching: (queries, trains) in ascending query order"""
    if dist is None:
        dist = distances(d1, d2, hamming)
    return select(dist, gate(model, guide, np.asarray(kq), np.asarray(kt), px_th), ratio, mutual, hamming)
