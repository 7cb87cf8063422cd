"""matching.triangulate_tracks_ragged: two-ray midpoint MSAC-RANSAC with local optimisation on ragged batches of tracks
across registered views.  CPU: the numpy oracle (tests/triangulate_np.py) against the planted points,
cv2.triangulatePoints, central differences, scipy's LM and planted tracks with outliers; the host build of the
kernel's pieces against the oracle; special cases; the argument checks.  GPU: the kernel against the oracle, batch
independence, edge cases and a three-view pipeline without a host synchronisation."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

from pydegensac_b200.scenes import _K, _rot
from tests import absolute_pose_np as ap
from tests import triangulate_np as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")
K2 = _K.copy(); K2[0, 0] *= 1.1; K2[1, 1] *= 1.07; K2[0, 2] += 7.0
MIN_ANGLE = math.radians(1.5)


def rig(C, seed, unregistered=()):
    """C cameras along a line (centres 0.4 units apart with some jitter, small rotations, looking along +z), world to
    camera: R [C,3,3], t [C,3], K [C,3,3] (alternately _K and K2, focal jittered); the cameras listed in
    `unregistered` get R = t = 0"""
    rng = np.random.default_rng(seed)
    R = np.stack([_rot("y", rng.uniform(-0.1, 0.1)) @ _rot("x", rng.uniform(-0.05, 0.05)) for _ in range(C)])
    centres = np.c_[0.4 * np.arange(C) - 0.2 * C, rng.uniform(-0.2, 0.2, C), rng.uniform(-0.2, 0.2, C)]
    t = -np.einsum("cij,cj->ci", R, centres)
    K = np.stack([(_K if c % 2 == 0 else K2).copy() for c in range(C)])
    K[:, 0, 0] *= 1.0 + 0.05 * rng.uniform(-1, 1, C)
    for c in unregistered:
        R[c], t[c] = 0.0, 0.0
    return R, t, K


def project(R, t, K, X):
    p = K @ (R @ X + t)
    return p[:2] / p[2]


def track(R, t, K, cams, X, noise, outlier, rng):
    """the pixels of X in cameras `cams` with Gaussian noise; observations flagged in `outlier` at random pixels"""
    x = np.array([project(R[c], t[c], K[c], X) for c in cams]).reshape(-1, 2)
    x += noise * rng.normal(size=x.shape)
    x[outlier] = np.c_[rng.uniform(0, 640, outlier.sum()), rng.uniform(0, 480, outlier.sum())]
    return x


def _centre(R, t):
    return -R.T @ t


def _point(R, t, cams, rng):
    cx = float(np.mean([_centre(R[c], t[c])[0] for c in cams])) if len(cams) else 0.0
    return np.array([rng.uniform(-3, 3) + cx, rng.uniform(-2, 2), rng.uniform(4, 12)])


def _table(R, t, K):
    return [o.camera(R[c], t[c], K[c]) for c in range(len(R))]


# ------------------------------------------------------------------------------------------------ oracle (CPU)
def test_oracle_midpoint_recovers_planted_points_and_agrees_with_cv2():
    import cv2
    R, t, K = rig(12, 0)
    tab = _table(R, t, K)
    rng = np.random.default_rng(1)
    worst = worst_cv2 = 0.0
    for _ in range(500):
        ci, cj = rng.choice(12, 2, replace=False)
        X = _point(R, t, [ci, cj], rng)
        xi, xj = project(R[ci], t[ci], K[ci], X), project(R[cj], t[cj], K[cj], X)
        Y = o.midpoint(tab[ci]["C"], o.ray(tab[ci], *xi), tab[cj]["C"], o.ray(tab[cj], *xj), 1.0)
        assert Y is not None
        worst = max(worst, np.abs(np.array(Y) - X).max() / np.abs(X).max())
        P1 = K[ci] @ np.c_[R[ci], t[ci]]
        P2 = K[cj] @ np.c_[R[cj], t[cj]]
        h = cv2.triangulatePoints(P1, P2, xi.reshape(2, 1), xj.reshape(2, 1)).ravel()
        worst_cv2 = max(worst_cv2, np.abs(np.array(Y) - h[:3] / h[3]).max() / np.abs(X).max())
    print("noise-free midpoint: worst relative error %.2e to the planted point, %.2e to cv2.triangulatePoints"
          % (worst, worst_cv2))
    assert worst <= 1e-9 and worst_cv2 <= 1e-9


def test_oracle_jacobian_against_central_differences():
    R, t, K = rig(6, 2)
    rng = np.random.default_rng(3)
    cams = np.arange(6)
    X = _point(R, t, cams, rng)
    x = track(R, t, K, cams, X, 1.0, np.zeros(6, bool), rng)
    r, J = o.jacobian(R, t, K, X, x)
    h = 1e-6
    for k in range(3):
        D = np.zeros(3)
        D[k] = h
        num = (o.residual(R, t, K, X + D, x)[0] - o.residual(R, t, K, X - D, x)[0]) / (2 * h)
        assert np.abs(num - J[:, :, k]).max() <= 1e-6 * max(1.0, np.abs(J[:, :, k]).max())
    assert np.abs(r - o.residual(R, t, K, X, x)[0]).max() <= 1e-12 * np.abs(x).max()


@pytest.mark.parametrize("n", [2, 5, 40])
def test_oracle_lm_reaches_the_optimum_of_scipy(n):
    from scipy.optimize import least_squares
    R, t, K = rig(max(n, 2), 4 + n)
    rng = np.random.default_rng(n)
    cams = np.arange(n)
    X = _point(R, t, cams, rng)
    x = track(R, t, K, cams, X, 0.7, np.zeros(n, bool), rng)
    X0 = X + np.array([0.05, -0.03, 0.1])
    Xo, it = o.lm(R, t, K, X0, x, 50)
    s = least_squares(lambda v: o.residual(R, t, K, v, x)[0].ravel(), X0, method="lm", xtol=1e-15, ftol=1e-15,
                      gtol=1e-15)
    c_o = float((o.residual(R, t, K, Xo, x)[0] ** 2).sum())
    assert abs(c_o - 2 * s.cost) <= 1e-9 * max(c_o, 1e-12)
    assert np.abs(Xo - s.x).max() <= 1e-6 * np.abs(X).max()


def test_oracle_rejects_outliers_and_lo_lowers_the_error():
    R, t, K = rig(20, 5)
    tab = _table(R, t, K)
    rng = np.random.default_rng(6)
    before, after, missed = [], [], 0
    for i in range(300):
        L = int(rng.integers(3, 15))
        cams = np.sort(rng.choice(20, L, replace=False))
        X = _point(R, t, cams, rng)
        out = rng.uniform(size=L) < 0.2
        out[:2] = False                                # at least two true observations
        x = track(R, t, K, cams, X, 0.5, out, rng)
        raw = o.triangulate_track(cams, x, tab, seed=i, refine_iters=0)
        res = o.triangulate_track(cams, x, tab, seed=i, refine_iters=10)
        assert res["iters"] == raw["iters"] and res["cost0"] == raw["cost0"] and res["cost"] <= res["cost0"]
        assert res["n_inliers"] == res["mask"].sum()
        missed += int((res["mask"] & out).sum())
        assert res["angle"] > 0.0
        before.append(np.linalg.norm(raw["X"] - X))
        after.append(np.linalg.norm(res["X"] - X))
    before, after = np.array(before), np.array(after)
    print("3D error over 300 tracks: RANSAC median %.3e, after LO %.3e; outlier observations kept %d"
          % (np.median(before), np.median(after), missed))
    assert np.median(after) < np.median(before)
    assert missed <= 3


def test_oracle_special_cases():
    R, t, K = rig(4, 7, unregistered=(3,))
    tab = _table(R, t, K)
    rng = np.random.default_rng(8)
    X = _point(R, t, [0, 1, 2], rng)
    x = track(R, t, K, [0, 1, 2], X, 0.0, np.zeros(3, bool), rng)
    none = lambda r: r["n_inliers"] == 0 and np.isnan(r["X"]).all() and np.isnan(r["cost"]) and np.isnan(r["angle"])
    # all observations from one camera: no hypothesis, every pair still counts
    r = o.triangulate_track([1, 1, 1], x, tab)
    assert none(r) and r["iters"] == 3
    # parallel rays (the same pixel seen by two cameras of one orientation): the gate rejects them
    Rp, tp, Kp = rig(2, 9)
    Rp[1] = Rp[0]
    tp[1] = -Rp[1] @ (_centre(Rp[0], tp[0]) + np.array([0.5, 0.0, 0.0]))
    Kp[1] = Kp[0]
    tabp = _table(Rp, tp, Kp)
    px = np.array([[320.0, 240.0], [320.0, 240.0]])
    assert none(o.triangulate_track([0, 1], px, tabp))
    assert o.midpoint(tabp[0]["C"], o.ray(tabp[0], 320, 240), tabp[1]["C"], o.ray(tabp[1], 320, 240), 1.0) is None
    # a point behind both cameras (rays that meet only behind them): no hypothesis
    Xb = np.array([X[0], X[1], -X[2]])
    xb = np.array([project(R[c], t[c], K[c], Xb) for c in (0, 1)])
    assert none(o.triangulate_track([0, 1], xb, tab))
    # unregistered camera, camera index out of range, non-finite pixel: not usable
    assert not tab[3]["ok"] and all(tab[c]["ok"] for c in range(3))
    xs = np.r_[x, x[:1], x[:1], [[np.nan, 1.0]]]
    cams = [0, 1, 2, 3, 7, 1]
    r = o.triangulate_track(cams, xs, tab)
    assert r["n_inliers"] == 3 and list(np.flatnonzero(r["mask"])) == [0, 1, 2]
    assert o.usable(cams, xs, tab).tolist() == [True, True, True, False, False, False]
    assert none(o.triangulate_track([0, -1], x[:2], tab))
    # a short track tries every pair, in order; conf = 1 runs them all
    assert o.triangulate_track([0, 1, 2], x, tab, conf=1.0)["iters"] == 3
    assert o.triangulate_track([0, 1, 2], x, tab)["iters"] == 1            # w = 1 after the first pair


# ------------------------------------------------------------------------------------------------ host build (CPU)
def _host(tmp_path):
    so = os.path.join(str(tmp_path), "libtriangulate_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-o", so, os.path.join(ROOT, "tests", "triangulate_host.cpp")])
    return ctypes.CDLL(so)


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def _ip(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))


def _host_table(L, R, t, K):
    tab = np.zeros((len(R), 34))
    for c in range(len(R)):
        L.trh_camera(_dp(np.ascontiguousarray(R[c]).ravel().copy()), _dp(np.ascontiguousarray(t[c]).copy()),
                     _dp(np.ascontiguousarray(K[c]).ravel().copy()), _dp(tab[c]))
    return tab


def test_host_build_equals_the_oracle(tmp_path):
    L = _host(tmp_path)
    R, t, K = rig(10, 11, unregistered=(9,))
    R[8, 0, 0] = np.inf                                # a camera with a non-finite pose
    tab = _host_table(L, R, t, K)
    otab = _table(R, t, K)
    for c in range(10):
        assert np.array_equal(tab[c, 0:9], R[c].ravel()) and np.array_equal(tab[c, 12:21], K[c].ravel())
        assert np.array_equal(tab[c, 21:30], otab[c]["Ki"].ravel()) and tab[c, 30:33].tolist() == otab[c]["C"]
        assert tab[c, 33] == (1.0 if otab[c]["ok"] else 0.0)
    assert tab[8, 33] == 0.0 and tab[9, 33] == 0.0 and (tab[:8, 33] == 1.0).all()
    # rays, hypotheses and the gate, bit for bit, over noisy pixels and several gates
    rng = np.random.default_rng(12)
    d, Y = np.zeros(3), np.zeros(3)
    counts = [0, 0]
    for _ in range(3000):
        ci, cj = rng.choice(8, 2, replace=False)
        X = _point(R, t, [ci, cj], rng)
        xi = project(R[ci], t[ci], K[ci], X) + rng.normal(size=2)
        xj = project(R[cj], t[cj], K[cj], X) + rng.normal(size=2)
        if rng.uniform() < 0.1:
            X[2] = -X[2]
            xj = project(R[cj], t[cj], K[cj], X)
        rays = []
        for c, x in ((ci, xi), (cj, xj)):
            L.trh_ray(_dp(tab[c]), ctypes.c_double(x[0]), ctypes.c_double(x[1]), _dp(d))
            assert d.tolist() == o.ray(otab[c], *x)
            rays.append(d.copy())
        cos_max = math.cos(float(rng.choice([0.0, 0.02, 0.05, 0.2])))
        ok = L.trh_midpoint(_dp(tab[ci, 30:33].copy()), _dp(rays[0]), _dp(tab[cj, 30:33].copy()), _dp(rays[1]),
                            ctypes.c_double(cos_max), _dp(Y))
        ref = o.midpoint(otab[ci]["C"], rays[0].tolist(), otab[cj]["C"], rays[1].tolist(), cos_max)
        assert bool(ok) == (ref is not None)
        if ok:
            assert Y.tolist() == ref
        counts[bool(ok)] += 1
    assert min(counts) >= 100                          # both outcomes of the gate are exercised
    # score rows, Jacobian rows and the LM sums
    cams = rng.integers(0, 8, 400).astype(np.int32)
    X = np.array([0.3, -0.2, 7.0])
    pts = np.stack([project(R[c], t[c], K[c], X) for c in cams]) + rng.normal(size=(400, 2))
    pts[:30] = rng.uniform(0, 640, (30, 2))
    term, inl = np.zeros(400), np.zeros(400, np.int32)
    Rs, ts, Ks = R[cams], t[cams], K[cams]
    L.trh_msac(_dp(tab), _ip(cams), _dp(pts), 400, _dp(X), ctypes.c_double(4.0), _dp(term), _ip(inl))
    ot, oi = o.msac(Rs, ts, Ks, X, pts, 4.0)
    assert np.abs(term - ot).max() <= 1e-12 * 4.0 and np.array_equal(inl.astype(bool), oi)
    Xb = np.array([0.3, -0.2, -7.0])                   # behind every camera: th^2 and no inlier
    L.trh_msac(_dp(tab), _ip(cams), _dp(pts), 400, _dp(Xb), ctypes.c_double(4.0), _dp(term), _ip(inl))
    assert (term == 4.0).all() and not inl.any()
    r, J = np.zeros(800), np.zeros(2400)
    L.trh_jacobian(_dp(tab), _ip(cams), _dp(pts), 400, _dp(X), _dp(r), _dp(J))
    orr, oJ = o.jacobian(Rs, ts, Ks, X, pts)
    assert np.abs(r - orr.ravel()).max() <= 1e-12 * max(1.0, np.abs(orr).max())
    assert np.abs(J - oJ.ravel()).max() <= 1e-12 * np.abs(oJ).max()
    sums = np.zeros(10)
    L.trh_sums(_dp(tab), _ip(cams), _dp(pts), 400, _dp(X), _dp(sums))
    os_ = o.row_sums(Rs, ts, Ks, X, pts)
    assert np.abs(sums - os_).max() <= 1e-12 * np.abs(os_).max()
    # the damped 3 x 3 solve
    H, g = o._unpack(os_)
    D = np.zeros(3)
    for lam in (0.0, 1e-3, 10.0):
        assert L.trh_solve(_dp(os_[1:7].copy()), _dp(os_[7:].copy()), ctypes.c_double(lam), _dp(D)) == 1
        assert np.abs(D - ap.solve_damped(H, g, lam)).max() <= 1e-10 * np.abs(D).max()
        assert D.tolist() == o.solve3(os_, lam).tolist()       # the oracle's restatement, bit for bit
    assert L.trh_solve(_dp(np.zeros(6)), _dp(np.ones(3)), ctypes.c_double(1e-3), _dp(D)) == 0
    # the enumeration order, one step at a time and in strides
    i, j = np.zeros(1, np.int32), np.zeros(1, np.int32)
    for n in (2, 3, 4, 7, 45):
        order = o.pairs(n)
        for s in (1, 5, 32):
            i[0], j[0] = 0, 1
            for k in range(s, len(order), s):
                L.trh_pair_advance(n, s, _ip(i), _ip(j))
                assert (int(i[0]), int(j[0])) == order[k], (n, s, k)
            L.trh_pair_advance(n, len(order), _ip(i), _ip(j))
            assert int(i[0]) == n - 1                  # past the last pair
    # the stopping rule of sizes 2 and 3; size 3 is ap_required_iters
    for args in ((0, 0, 10, 0.99, 500, 3), (1, 5, 10, 1.0, 500, 3), (1, 10, 10, 0.99, 500, 4), (1, 0, 10, 0.99, 500, 2),
                 (1, 7, 10, 0.999, 500, 9), (1, 30, 1000, 0.999, 10000, 9), (1, 300, 1000, 0.5, 10000, 1),
                 (1, 2, 3, 0.999, 3, 1), (1, 9, 10, 0.999, 45, 1)):
        cargs = (*args[:3], ctypes.c_double(args[3]), *args[4:])
        for s in (2, 3):
            assert L.trh_required_iters(s, *cargs) == o.required_iters(s, *args), (s, args)
        assert L.trh_ap_required_iters(*cargs) == ap.required_iters(*args) == o.required_iters(3, *args)
    # minimal_sample<2> of rng.h
    sel = np.zeros(2, np.int32)
    for seed in (0, 1, 12345, 2 ** 40 + 17, 2 ** 64 - 1):
        for n in (2, 3, 17, 1000, 99991):
            for k in (1, 2, 3, 100, 65537):
                L.trh_sample(ctypes.c_ulonglong(seed), ctypes.c_uint(k), n, _ip(sel))
                assert list(sel) == ap.minimal_sample(seed, k, n, 2), (seed, n, k)
                assert sel[0] != sel[1] and sel.min() >= 0 and sel.max() < n


# ------------------------------------------------------------------------------------------------ arguments (CPU)
def test_entry_point_rejects_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["cams", "pts", "R", "t", "K", "offsets", "mask", "seeds", "X", "mask_out", "n_inliers", "iters", "cost0",
             "cost", "angle"]

    def call(n_cams=4, n_tracks=3, obs=10, px_th=2.0, min_angle=0.02, conf=0.99, max_iters=100, refine_iters=10,
             **null):
        b = {k: (None if null.get(k) else fake) for k in names}
        return L.dgb200_triangulate_tracks_ragged_dev(
            b["cams"], b["pts"], b["R"], b["t"], b["K"], 0, n_cams, b["offsets"], n_tracks, obs, b["mask"],
            ctypes.c_double(px_th), ctypes.c_double(min_angle), ctypes.c_double(conf), max_iters, refine_iters,
            b["seeds"], b["X"], b["mask_out"], b["n_inliers"], b["iters"], b["cost0"], b["cost"], b["angle"], None)

    for k in names:
        if k != "mask":
            assert call(**{k: True}) == -1, k
            assert L.dgb200_triangulate_last_error().decode() != ""
    for kw in (dict(n_tracks=0), dict(n_tracks=-1), dict(obs=-1), dict(n_cams=0), dict(max_iters=0),
               dict(refine_iters=-1)):
        assert call(**kw) == -1, kw
    for px_th in (0.0, -1.0, float("nan"), float("inf")):
        assert call(px_th=px_th) == -1
        assert "px_th" in L.dgb200_triangulate_last_error().decode()
    for a in (-1e-9, math.pi, 4.0, float("nan")):
        assert call(min_angle=a) == -1
        assert "min_angle" in L.dgb200_triangulate_last_error().decode()
    for conf in (0.0, -0.5, 1.0000001, float("nan")):
        assert call(conf=conf) == -1


def test_python_argument_errors():
    import torch
    from pydegensac_b200.matching import triangulate_tracks_ragged as tt
    f64, i32 = torch.float64, torch.int32
    good = dict(cams=torch.zeros(10, dtype=i32), pts=torch.zeros((10, 2), dtype=f64),
                R=torch.eye(3, dtype=f64).repeat(4, 1, 1), t=torch.zeros((4, 3), dtype=f64), K=torch.eye(3, dtype=f64),
                offsets=torch.tensor([0, 4, 10], dtype=i32))
    bad = [
        dict(cams=np.zeros(10, np.int32)), dict(cams=torch.zeros(10, dtype=torch.int64)), dict(cams=torch.zeros(9, dtype=i32)),
        dict(pts=torch.zeros((10, 3), dtype=f64)), dict(pts=torch.zeros((10, 2), dtype=torch.int64)),
        dict(R=torch.eye(3, dtype=f64)), dict(R=torch.zeros((0, 3, 3), dtype=f64)), dict(t=torch.zeros((3, 3), dtype=f64)),
        dict(K=torch.eye(3, dtype=f64).repeat(3, 1, 1)), dict(K=torch.eye(4, dtype=f64)),
        dict(K=torch.eye(3, dtype=torch.int64)), dict(offsets=torch.tensor([0, 4, 10])),
        dict(offsets=torch.tensor([0], dtype=i32)), dict(mask=torch.ones(9, dtype=torch.bool)),
        dict(mask=torch.ones(10, dtype=torch.int32)), dict(mask=np.ones(10, bool)), dict(px_th=0.0),
        dict(px_th=float("nan")), dict(min_angle=-0.1), dict(min_angle=math.pi), dict(conf=0.0), dict(conf=1.5),
        dict(max_iters=0), dict(refine_iters=-1),
        dict(),                                    # well-formed, but on the host
    ]
    for kw in bad:
        args = dict(good)
        args.update(kw)
        with pytest.raises(ValueError):
            tt(**args)
    with pytest.raises(ValueError, match="^t must be"):
        tt(**dict(good, t=torch.zeros((3, 3), dtype=f64)))


# ------------------------------------------------------------------------------------------------ GPU
def _dev(*xs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0") for a in xs]


def _np(res):
    return {k: getattr(res, k).cpu().numpy() for k in res._fields}


def _ragged_batch(T, seed, C=24):
    """T tracks over a rig of C cameras (two unregistered) with per-camera K: lengths 0-60 and a few of several
    hundred, 0-40 % outlier observations, some repeated cameras, mask holes, non-finite pixels and camera indices out of
    range.  Returns (cams, pts, R, t, K, offsets, mask, seeds, planted points)."""
    rng = np.random.default_rng(seed)
    R, t, K = rig(C, seed, unregistered=(5, 17))
    cs, xs, ms, truth = [], [], [], []
    for j in range(T):
        n = int(rng.integers(300, 700)) if j % 500 == 7 else int(rng.choice([0, 1, 2, 3, 4, 6, 10, 20, 45, 46, 60])
                                                                  if j % 3 == 0 else rng.integers(2, 12))
        cams = rng.integers(0, C, n) if j % 4 == 0 else (int(rng.integers(0, C)) + np.arange(n)) % C
        X = _point(R, t, cams, rng)
        out = rng.uniform(size=n) < float(rng.choice([0.0, 0.1, 0.2, 0.4]))
        x = track(R, t, K, np.where(np.isin(cams, (5, 17)), 0, cams), X, float(rng.uniform(0.1, 1.0)), out, rng)
        m = rng.uniform(size=n) > 0.1
        if n > 4 and j % 5 == 1:
            x[1, 0] = np.nan
            cams[2] = C + 3 if j % 2 else -1
        cs.append(cams.astype(np.int32)); xs.append(x); ms.append(m); truth.append(X)
    off = np.zeros(T + 1, np.int32)
    off[1:] = np.cumsum([len(a) for a in cs])
    seeds = rng.integers(0, 2 ** 62, T).astype(np.int64)
    return (np.concatenate(cs), np.concatenate(xs), R, t, K, off, np.concatenate(ms), seeds, np.array(truth))


def _run(cams, pts, R, t, K, off, mask, seeds, **kw):
    from pydegensac_b200.matching import triangulate_tracks_ragged
    d = _dev(cams, pts, R, t, K, off, mask, seeds)
    return _np(triangulate_tracks_ragged(*d[:7], seeds=d[7], **kw))


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


@pytest.mark.gpu
def test_kernel_against_the_oracle():
    T = 3000
    cams, pts, R, t, K, off, mask, seeds, _ = _ragged_batch(T, 1)
    kw = dict(px_th=2.0, min_angle=MIN_ANGLE, conf=0.999, max_iters=1000, refine_iters=10)
    g = _run(cams, pts, R, t, K, off, mask, seeds, **kw)
    ref = o.triangulate_tracks_ragged(cams, pts, R, t, K, off, mask, seeds=seeds.astype(np.uint64), **kw)
    ties = 0
    worst = dict(X=0.0, cost0=0.0, cost=0.0, angle=0.0)
    philox = enumerated = 0
    for j, r in enumerate(ref):
        b, e = off[j], off[j + 1]
        if r["near_tie"] or r["lo_tie"]:
            ties += 1
            continue
        assert g["iters"][j] == r["iters"], j
        assert g["n_inliers"][j] == r["n_inliers"], j
        assert np.array_equal(g["mask"][b:e], r["mask"]), j
        if np.isnan(r["cost0"]):
            assert np.isnan(g["X"][j]).all() and np.isnan(g["cost0"][j]) and np.isnan(g["angle"][j]), j
            continue
        n = int(o.usable(cams[b:e], pts[b:e], _table(R, t, K), mask[b:e]).sum())
        philox += n * (n - 1) // 2 > 1000
        enumerated += n * (n - 1) // 2 <= 1000
        for k in worst:
            d = _rel(g[k][j], np.asarray(r[k]))
            worst[k] = max(worst[k], d)
            assert d <= 1e-9, (j, k, d)
        assert g["cost"][j] <= g["cost0"][j]
    n_model = int((g["n_inliers"] > 0).sum())
    print("tracks %d (with a model %d; enumerated %d, sampled %d), near ties %d; worst relative difference %s; "
          "iters mean %.1f max %d" % (T, n_model, enumerated, philox, ties,
                                      {k: "%.2e" % v for k, v in worst.items()}, g["iters"].mean(), g["iters"].max()))
    assert ties <= 15 and n_model >= 2000 and philox >= 30


@pytest.mark.gpu
def test_same_bytes_alone_in_a_batch_permuted_and_on_a_rerun():
    cams, pts, R, t, K, off, mask, seeds, _ = _ragged_batch(400, 2)
    full = _run(cams, pts, R, t, K, off, mask, seeds)
    again = _run(cams, pts, R, t, K, off, mask, seeds)
    for k in full:
        assert full[k].tobytes() == again[k].tobytes(), k
    perm = np.random.default_rng(0).permutation(400)
    pc, px, pm, poff = [], [], [], [0]
    for j in perm:
        b, e = off[j], off[j + 1]
        pc.append(cams[b:e]); px.append(pts[b:e]); pm.append(mask[b:e]); poff.append(poff[-1] + e - b)
    pres = _run(np.concatenate(pc), np.concatenate(px), R, t, K, np.array(poff, np.int32), np.concatenate(pm),
                seeds[perm])
    scalar = ("X", "n_inliers", "iters", "cost0", "cost", "angle")
    for i, j in enumerate(perm):
        for k in scalar:
            assert full[k][j].tobytes() == pres[k][i].tobytes(), (k, j)
        assert full["mask"][off[j]:off[j + 1]].tobytes() == pres["mask"][poff[i]:poff[i + 1]].tobytes()
    for j in (1, 7, 33, 250):
        b, e = off[j], off[j + 1]
        alone = _run(cams[b:e], pts[b:e], R, t, K, np.array([0, e - b], np.int32), mask[b:e], seeds[j:j + 1])
        for k in scalar:
            assert full[k][j].tobytes() == alone[k][0].tobytes(), (k, j)
        assert full["mask"][b:e].tobytes() == alone["mask"].tobytes()


@pytest.mark.gpu
def test_edge_cases():
    import torch
    from pydegensac_b200.matching import triangulate_tracks_ragged
    R, t, K = rig(8, 3)
    rng = np.random.default_rng(4)
    cams = np.arange(8, dtype=np.int32)
    X = _point(R, t, cams, rng)
    out = np.zeros(8, bool); out[[2, 5]] = True
    x = track(R, t, K, cams, X, 0.5, out, rng)
    one = np.array([0, 8], np.int32)
    ones = np.ones(8, bool)
    # refine_iters = 0: the RANSAC point itself
    z = _run(cams, x, R, t, K, one, ones, np.array([5]), refine_iters=0)
    r0 = o.triangulate_track(cams, x, _table(R, t, K), seed=5, refine_iters=0)
    assert z["cost"][0] == z["cost0"][0] and z["iters"][0] == r0["iters"] and z["n_inliers"][0] == r0["n_inliers"]
    assert _rel(z["X"][0], r0["X"]) <= 1e-9
    full = _run(cams, x, R, t, K, one, ones, np.array([5]))
    assert full["cost0"][0] == z["cost0"][0] and full["cost"][0] <= full["cost0"][0]
    # conf = 1: K_max iterations, all 28 pairs when they are no more than max_iters, else max_iters
    assert _run(cams, x, R, t, K, one, ones, np.array([5]), conf=1.0)["iters"][0] == 28
    assert _run(cams, x, R, t, K, one, ones, np.array([5]), conf=1.0, max_iters=13)["iters"][0] == 13
    # malformed offsets: no model, no row read or written (tracks 1, 2 and 4; track 4 passes the 8 rows)
    d = _dev(cams, x, R, t, K)
    bad = torch.tensor([0, 4, -1, 4, 8, 12], dtype=torch.int32, device="cuda:0")
    res = _np(triangulate_tracks_ragged(*d, bad, seeds=torch.arange(5, device="cuda:0")))
    for j in (1, 2, 4):
        assert res["iters"][j] == 0 and res["n_inliers"][j] == 0 and np.isnan(res["X"][j]).all()
        assert np.isnan(res["cost"][j]) and np.isnan(res["angle"][j])
    ref = o.triangulate_tracks_ragged(cams, x, R, t, K, [0, 4, 8], seeds=np.array([0, 3], np.uint64))
    for j, jj in ((0, 0), (1, 3)):
        assert res["iters"][jj] == ref[j]["iters"] and res["n_inliers"][jj] == ref[j]["n_inliers"]


def _planted_points(n_pts, n_hold, seed):
    """the planted points of tests.test_refine_fundamental._multiview_two_cameras (its first three draws)"""
    rng = np.random.default_rng(seed)
    m = n_pts + n_hold
    return np.c_[rng.uniform(-4, 4, m), rng.uniform(-4, 4, m), rng.uniform(2, 12, m)][:n_pts]


@pytest.mark.gpu
def test_pipeline_register_a_third_view_then_triangulate_three_view_tracks_without_sync():
    """matching (0, 1) and (2, 0) -> F RANSAC -> pose from F -> pose refinement -> triangulation of the pair ->
    P3P registration of view 2 -> 3-slot tracks keyed by view 0's keypoints -> triangulate_tracks_ragged, with no host
    synchronisation from the descriptors to the points"""
    import torch
    from scipy.spatial import cKDTree
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import (find_absolute_pose_ragged, match_descriptors_batch,
                                          pose_from_fundamental_ragged, refine_pose_ragged, triangulate_tracks_ragged)
    from tests.test_refine_fundamental import _multiview_two_cameras
    dev = torch.device("cuda:0")
    kps, descs, Rs, ts, Ks, _ = _multiview_two_cameras(3, 900, 300, 0, 64, 21)
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    K0, K1, Kv2 = (torch.from_numpy(k).to(dev) for k in Ks)
    n0 = len(kps[0])
    seeds = torch.tensor([3], dtype=torch.int64, device=dev)
    f64 = torch.float64
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m = match_descriptors_batch(dt, [(0, 1)], kt, ratio=0.9, mutual=True)
        F, mask = pdg.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                                 n_max=m.n_max)
        pose = pose_from_fundamental_ragged(F, K0, K1, m.pts1, m.pts2, m.offsets, mask)
        fine = refine_pose_ragged(pose.R, pose.t, K0, K1, m.pts1, m.pts2, m.offsets, pose.in_front, px_th=1.0)
        tri = pose_from_fundamental_ragged(fine.F, K0, K1, m.pts1, m.pts2, m.offsets, fine.inliers)
        live = torch.arange(m.idx1.shape[0], device=dev) < m.offsets[1]
        slot = torch.where(live, m.idx1, n0)
        P0 = torch.full((n0 + 1, 3), float("nan"), dtype=f64, device=dev).index_put_((slot,), tri.points)
        V0 = torch.zeros(n0 + 1, dtype=torch.bool, device=dev).index_put_((slot,), tri.in_front & live)
        m2 = match_descriptors_batch(dt, [(2, 0)], kt, ratio=0.9, mutual=True)
        live2 = torch.arange(m2.idx2.shape[0], device=dev) < m2.offsets[1]
        src = torch.where(live2, m2.idx2, n0)
        view = find_absolute_pose_ragged(m2.pts1, P0.index_select(0, src), Kv2, m2.offsets,
                                         V0.index_select(0, src) & live2, px_th=2.0, seeds=seeds + 1)
        # 3-slot tracks keyed by view 0's keypoints: slot 0 the keypoint, slot 1 its match in view 1, slot 2 in view 2
        pts = torch.zeros((n0 + 1, 3, 2), dtype=f64, device=dev)
        obs = torch.zeros((n0 + 1, 3), dtype=torch.bool, device=dev)
        pts[:n0, 0] = kt[0].to(f64)
        obs[:n0, 0] = True
        pts[:, 1].index_put_((slot,), m.pts2.to(f64))
        obs[:, 1].index_put_((slot,), live)
        pts[:, 2].index_put_((src,), m2.pts1.to(f64))
        obs[:, 2].index_put_((src,), live2)
        R = torch.stack([torch.eye(3, dtype=f64, device=dev), fine.R[0], view.R[0]])
        t = torch.stack([torch.zeros(3, dtype=f64, device=dev), fine.t[0], view.t[0]])
        K = torch.stack([K0, K1, Kv2])
        cams = torch.arange(3, dtype=torch.int32, device=dev).repeat(n0)
        offsets = torch.arange(0, 3 * n0 + 1, 3, dtype=torch.int32, device=dev)
        tr = triangulate_tracks_ragged(cams, pts[:n0].reshape(-1, 2), R, t, K, offsets, obs[:n0].reshape(-1),
                                       px_th=2.0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    # the planted point of each view-0 keypoint: the one that projects within 0.5 px of it; camera 0's frame is the
    # world frame of the scene (R0 = I, t0 = 0), and the two-view geometry has the first pair's baseline as unit
    Xw = _planted_points(900, 0, 21)
    proj = Xw @ Ks[0].T
    d, idx = cKDTree(proj[:, :2] / proj[:, 2:]).query(kps[0])
    planted = d < 0.5
    base = np.linalg.norm(ts[1] - Rs[1] @ Rs[0].T @ ts[0])
    truth = Xw[idx] / base
    r = _np(tr)
    n_in = r["n_inliers"]
    ok = (n_in >= 2) & planted
    err = np.linalg.norm(r["X"] - truth, axis=1)
    three = ok & (n_in == 3)
    vals = V0[:n0].cpu().numpy() & three
    e2 = np.linalg.norm(P0[:n0].cpu().numpy()[vals] - truth[vals], axis=1)
    e3 = err[vals]
    print("tracks %d: %d triangulated (%d with 3 inliers); median 3D error %.3e baselines; on %d tracks with a two-view "
          "point: three-view median %.3e, two-view median %.3e" % (n0, int((n_in >= 2).sum()), int(three.sum()),
                                                                    np.median(err[ok]), int(vals.sum()), np.median(e3),
                                                                    np.median(e2)))
    assert int((n_in >= 2).sum()) >= 600 and int(three.sum()) >= 400
    assert np.median(err[ok]) <= 2e-2
    assert np.median(e3) <= np.median(e2)
    assert (r["angle"][n_in >= 2] > 0).all()
