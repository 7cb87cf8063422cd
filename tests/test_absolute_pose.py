"""matching.find_absolute_pose_ragged: P3P MSAC-RANSAC with local optimisation on ragged batches of 2D-3D
correspondences.  CPU: the numpy oracle (tests/absolute_pose_np.py) against cv2.solveP3P, central differences, scipy's
LM and planted scenes; the host build of the kernel's pieces against the oracle; the argument checks.  GPU: the kernel
against the oracle, batch independence, edge cases and a three-view pipeline without a host synchronisation."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from pydegensac_b200.scenes import _K
from tests import absolute_pose_np as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")
K2 = _K.copy(); K2[0, 0] *= 1.1; K2[1, 1] *= 1.07; K2[0, 2] += 7.0


def _random_rotation(rng):
    q = rng.normal(size=4)
    a, b, c, d = q / np.linalg.norm(q)
    return np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])


def _rot_error(Ra, Rb):
    return float(np.arccos(np.clip((np.trace(Ra @ Rb.T) - 1.0) / 2.0, -1.0, 1.0)))


def scene(n, inlier_ratio, seed, noise=0.5, K=_K):
    """n 2D-3D rows of one view: points 2-10 units in front of a camera with a random pose (R, t), x ~ K (R X + t);
    the first round(n * inlier_ratio) rows observed with Gaussian pixel noise, the rest at uniform random pixels.
    Returns (x [n,2], X [n,3], R, t, is_inlier [n])."""
    rng = np.random.default_rng(seed)
    R, t = _random_rotation(rng), rng.uniform(-1.0, 1.0, 3)
    z = rng.uniform(2.0, 10.0, n)
    u = np.c_[rng.uniform(0, 640, n), rng.uniform(0, 480, n)]
    P = (np.c_[u, np.ones(n)] @ np.linalg.inv(K).T) * z[:, None]    # camera frame
    X = (P - t) @ R                                                  # R X + t = P
    x = u + noise * rng.normal(size=(n, 2))
    n_in = int(round(n * inlier_ratio))
    x[n_in:] = np.c_[rng.uniform(0, 640, n - n_in), rng.uniform(0, 480, n - n_in)]
    return x, X, R, t, np.arange(n) < n_in


def _bearings(K, x):
    Ki = o.inv3(K)
    return np.array([o.bearing(Ki, *p) for p in x])


# ------------------------------------------------------------------------------------------------ oracle (CPU)
def _triples(count, seed):
    rng = np.random.default_rng(seed)
    for _ in range(count):
        R, t = _random_rotation(rng), rng.uniform(-1.0, 1.0, 3)
        P = np.c_[rng.uniform(-2, 2, (3, 2)), rng.uniform(3, 8, 3)]
        X = (P - t) @ R
        x = P @ _K.T
        yield R, t, X, x[:, :2] / x[:, 2:]


def test_oracle_p3p_against_cv2_solveP3P():
    """The planted pose is among the oracle's solutions, and so is every cv2 solution that reprojects its three points
    with positive depths (Lambda Twist, by design, returns no pose that puts a point behind the camera; cv2 returns
    such poses too, since they reproject as well)."""
    import cv2
    worst_planted = worst_cv2 = 0.0
    matched = behind = 0
    for R, t, X, x in _triples(2000, 0):
        sols = o.p3p(_bearings(_K, x), X)
        assert all(np.isfinite(Ro).all() and np.isfinite(to).all() for Ro, to in sols)
        err = [max(np.abs(Ro - R).max(), np.abs(to - t).max()) for Ro, to in sols]
        worst_planted = max(worst_planted, min(err))
        for flag in (cv2.SOLVEPNP_P3P, cv2.SOLVEPNP_AP3P):
            _, rv, tv = cv2.solveP3P(X.reshape(3, 1, 3), x.reshape(3, 1, 2), _K, None, flags=flag)
            for r_, t_ in zip(rv, tv):
                Rc, tc = cv2.Rodrigues(r_)[0], t_.ravel()
                pc = X @ Rc.T + tc
                pr = pc @ _K.T
                if np.abs(pr[:, :2] / pr[:, 2:] - x).max() > 1e-6:
                    continue
                if (pc[:, 2] <= 0).any():
                    behind += 1
                    continue
                m = min(max(np.abs(Ro - Rc).max(), np.abs(to - tc).max()) for Ro, to in sols)
                worst_cv2 = max(worst_cv2, m)
                matched += 1
    print("planted pose: worst %.3e; %d cv2 solutions matched (worst %.3e), %d with a point behind the camera"
          % (worst_planted, matched, worst_cv2, behind))
    assert worst_planted <= 1e-8
    assert matched >= 4000 and worst_cv2 <= 1e-8


def test_oracle_jacobian_against_central_differences():
    x, X, R, t, _ = scene(50, 1.0, 3, noise=1.0, K=K2)
    r, J = o.jacobian(R, t, K2, x, X)
    h = 1e-6
    for k in range(6):
        D = np.zeros(6)
        D[k] = h
        rp, _ = o.residual(*o.step(R, t, D), K2, x, X)
        rm, _ = o.residual(*o.step(R, t, -D), K2, x, X)
        num = (rp - rm) / (2 * h)
        assert np.abs(num - J[:, :, k]).max() <= 1e-6 * max(1.0, np.abs(J[:, :, k]).max())
    r0, _ = o.residual(R, t, K2, x, X)
    assert np.abs(r - r0).max() <= 1e-12 * np.abs(x).max()       # (q0 / q2 there, q0 * (1 / q2) here)


@pytest.mark.parametrize("n", [10, 300, 3000])
def test_oracle_lm_reaches_the_optimum_of_scipy(n):
    from scipy.optimize import least_squares
    x, X, R, t, _ = scene(n, 1.0, 11 + n, noise=0.7)
    R0 = o.rodrigues(np.array([0.01, -0.02, 0.015])) @ R
    t0 = t + np.array([0.02, -0.01, 0.03])
    Ro, to, it, acc = o.lm(R0, t0, _K, x, X, 50)
    assert acc >= 1

    def fun(v):
        Rv, tv = o.step(R0, t0, v)
        return o.residual(Rv, tv, _K, x, X)[0].ravel()
    s = least_squares(fun, np.zeros(6), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    Rs, ts = o.step(R0, t0, s.x)
    c_o = float((o.residual(Ro, to, _K, x, X)[0] ** 2).sum())
    assert abs(c_o - 2 * s.cost) <= 1e-9 * c_o
    # the schedule stops when a step moves the cost by less than 1e-12 of it: the pose to about the square root
    assert _rot_error(Ro, Rs) <= 1e-6 and np.abs(to - ts).max() <= 1e-6


def test_oracle_recovers_planted_poses_and_lo_helps():
    """Planted scenes over rows, inlier ratio, noise and K: the pose after the local optimisation is never worse than
    the RANSAC's in the median and within fixed bounds; cv2.solvePnPRansac on the same scenes is reported beside."""
    import cv2
    cases = [(n, w, s, K) for n in (8, 60, 400, 3000) for w in (0.15, 0.5, 0.9) for s in (0.0, 0.5, 1.0)
             for K in (_K, K2) if not (n == 8 and w < 0.5)]
    before, after, cv = [], [], []
    for i, (n, w, sigma, K) in enumerate(cases):
        x, X, R, t, gt = scene(n, w, 100 + i, noise=sigma, K=K)
        raw = o.absolute_pose(x, X, K, px_th=max(2.0, 4 * sigma), seed=i, refine_iters=0)
        res = o.absolute_pose(x, X, K, px_th=max(2.0, 4 * sigma), seed=i, refine_iters=10)
        assert res["iters"] == raw["iters"] and res["cost0"] == raw["cost0"]
        assert res["cost"] <= res["cost0"]
        assert res["n_inliers"] == res["mask"].sum()
        e = [max(_rot_error(r["R"], R), np.abs(r["t"] - t).max() / 6.0) for r in (raw, res)]
        before.append(e[0]); after.append(e[1])
        ok, rv, tv, _ = cv2.solvePnPRansac(X, x, K, None, reprojectionError=max(2.0, 4 * sigma), confidence=0.999,
                                           iterationsCount=10000)
        cv.append(max(_rot_error(cv2.Rodrigues(rv)[0], R), np.abs(tv.ravel() - t).max() / 6.0) if ok else np.inf)
    before, after, cv = map(np.array, (before, after, cv))
    print("pose error (max of rotation rad and translation / 6 units) over %d scenes: RANSAC median %.3e worst %.3e; "
          "after LO median %.3e worst %.3e; cv2.solvePnPRansac median %.3e worst %.3e"
          % (len(cases), np.median(before), before.max(), np.median(after), after.max(), np.median(cv), cv.max()))
    assert np.median(after) <= np.median(before)
    assert after.max() <= 0.05


def test_oracle_stopping_rule_and_special_cases():
    assert o.required_iters(False, 0, 10, 0.99, 500, 3) == 500
    assert o.required_iters(True, 5, 10, 1.0, 500, 3) == 500
    assert o.required_iters(True, 10, 10, 0.99, 500, 3) == 3
    assert o.required_iters(True, 5, 10, 0.99, 500, 3) == int(np.ceil(np.log(0.01) / np.log1p(-0.125)))
    assert o.required_iters(True, 0, 10, 0.99, 500, 3) == 500
    x, X, R, t, _ = scene(3, 1.0, 1)
    assert o.absolute_pose(x, X, _K)["cost"] != o.absolute_pose(x, X, _K)["cost"]   # n < 4: NaN
    x, X, R, t, _ = scene(200, 1.0, 2, noise=0.0)
    res = o.absolute_pose(x, X, _K, conf=0.999)
    assert res["iters"] == 1 and res["n_inliers"] == 200       # w = 1 after the first iteration
    assert o.absolute_pose(x, X, _K, conf=1.0, max_iters=37)["iters"] == 37


# ------------------------------------------------------------------------------------------------ host build (CPU)
def _host(tmp_path):
    so = os.path.join(str(tmp_path), "libabsolute_pose_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-o", so, os.path.join(ROOT, "tests", "absolute_pose_host.cpp")])
    return ctypes.CDLL(so)


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def _host_p3p(L, y, X):
    R, t = np.zeros(36), np.zeros(12)
    n = L.aph_p3p(_dp(np.ascontiguousarray(y, np.float64).ravel()), _dp(np.ascontiguousarray(X, np.float64).ravel()),
                  _dp(R), _dp(t))
    return [(R[9 * s:9 * s + 9].reshape(3, 3), t[3 * s:3 * s + 3]) for s in range(n)]


def test_host_build_equals_the_oracle(tmp_path):
    L = _host(tmp_path)
    # P3P: the same solutions, in the same order (both are +, -, *, /, sqrt in one order: the bits agree)
    for R, t, X, x in _triples(500, 7):
        y = _bearings(_K, x)
        hs, os_ = _host_p3p(L, y, X), o.p3p(y, X)
        assert len(hs) == len(os_) >= 1
        for (Rh, th), (Ro, to) in zip(hs, os_):
            assert np.abs(Rh - Ro).max() <= 1e-12 and np.abs(th - to).max() <= 1e-12 * max(1.0, np.abs(to).max())
    # degenerate triples: no pose, never a NaN
    rng = np.random.default_rng(3)
    for _ in range(200):
        R, t, X, x = next(_triples(1, int(rng.integers(1 << 30))))
        y = _bearings(_K, x)
        d = rng.normal(size=3)
        for Xd, yd in ((np.array([X[0], X[0] + d, X[0] + 2.5 * d]), y),      # collinear points
                       (np.array([X[0], X[0], X[2]]), y),                     # coincident points
                       (X, np.array([y[0], y[0], y[2]]))):                    # coincident bearings
            assert _host_p3p(L, yd, Xd) == [] and o.p3p(yd, Xd) == []
    # bearings, the MSAC rows, the Jacobian rows and the LM sums
    x, X, R, t, _ = scene(300, 0.6, 5, noise=0.8, K=K2)
    X[:5] = (np.c_[x[:5], np.ones(5)] @ np.linalg.inv(K2).T) * -3.0 - t @ R    # some rows behind the camera
    X[:5] = X[:5] @ R
    P = np.r_[R.ravel(), t]
    Ki = np.zeros(9)
    L.aph_inv3(_dp(K2.ravel().copy()), _dp(Ki))
    assert np.array_equal(Ki.reshape(3, 3), o.inv3(K2))
    b = np.zeros(3)
    L.aph_bearing(_dp(Ki), ctypes.c_double(x[7, 0]), ctypes.c_double(x[7, 1]), _dp(b))
    assert np.array_equal(b, o.bearing(o.inv3(K2), x[7, 0], x[7, 1]))
    xc, Xc = np.ascontiguousarray(x), np.ascontiguousarray(X)
    term, inl = np.zeros(300), np.zeros(300, np.int32)
    L.aph_msac(_dp(P), _dp(K2.ravel().copy()), _dp(xc), _dp(Xc), 300, ctypes.c_double(4.0), _dp(term),
               inl.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
    ot, oi = o.msac(R, t, K2, x, X, 4.0)
    assert np.abs(term - ot).max() <= 1e-12 * 4.0 and np.array_equal(inl.astype(bool), oi)
    assert (~oi[:5]).all() and (ot[:5] == 4.0).all()
    r, J = np.zeros(600), np.zeros(3600)
    L.aph_jacobian(_dp(P), _dp(K2.ravel().copy()), _dp(xc), _dp(Xc), 300, _dp(r), _dp(J))
    orr, oJ = o.jacobian(R, t, K2, x, X)
    assert np.abs(r - orr.ravel()).max() <= 1e-12 * max(1.0, np.abs(orr).max())
    assert np.abs(J - oJ.ravel()).max() <= 1e-12 * np.abs(oJ).max()
    sums = np.zeros(28)
    L.aph_sums(_dp(P), _dp(K2.ravel().copy()), _dp(xc[5:]), _dp(np.ascontiguousarray(Xc[5:])), 295, _dp(sums))
    os_ = o.row_sums(R, t, K2, x[5:], X[5:])
    assert np.abs(sums - os_).max() <= 1e-12 * np.abs(os_).max()
    # the damped solve and the step
    H, g = o._unpack(os_)
    D = np.zeros(6)
    assert L.aph_solve(_dp(os_[1:22].copy()), _dp(os_[22:].copy()), ctypes.c_double(1e-3), _dp(D)) == 1
    assert np.abs(D - o.solve_damped(H, g, 1e-3)).max() <= 1e-10 * np.abs(D).max()
    P2 = np.zeros(12)
    Dq = np.array([0.01, -0.02, 0.005, 0.1, 0.2, -0.3])
    L.aph_step(_dp(P), _dp(Dq), _dp(P2))
    R2, t2 = o.step(R, t, Dq)
    assert np.abs(P2 - np.r_[R2.ravel(), t2]).max() <= 1e-14
    for args in ((0, 0, 10, 0.99, 500, 3), (1, 5, 10, 1.0, 500, 3), (1, 10, 10, 0.99, 500, 4), (1, 0, 10, 0.99, 500, 2),
                 (1, 7, 10, 0.999, 500, 9), (1, 30, 1000, 0.999, 10000, 9), (1, 300, 1000, 0.5, 10000, 1)):
        assert L.aph_required_iters(*args[:3], ctypes.c_double(args[3]), *args[4:]) == o.required_iters(*args)


def test_philox_sampling_of_the_oracle_equals_rng_h(tmp_path):
    L = _host(tmp_path)
    sel = np.zeros(3, np.int32)
    for seed in (0, 1, 12345, 2 ** 40 + 17, 2 ** 64 - 1):
        for n in (3, 4, 5, 17, 1000, 99991):
            for k in (1, 2, 3, 100, 65537):
                L.aph_sample(ctypes.c_ulonglong(seed), ctypes.c_uint(k), n, sel.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
                assert list(sel) == o.minimal_sample(seed, k, n), (seed, n, k)
                assert len(set(sel)) == 3 and sel.min() >= 0 and sel.max() < n


# ------------------------------------------------------------------------------------------------ arguments (CPU)
def test_entry_point_rejects_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["x", "X", "K", "offsets", "mask", "seeds", "R", "t", "mask_out", "n_inliers", "iters", "cost0", "cost"]

    def call(n_pairs=3, rows=10, px_th=2.0, conf=0.99, max_iters=100, refine_iters=10, **null):
        b = {k: (None if null.get(k) else fake) for k in names}
        return L.dgb200_find_absolute_pose_ragged_dev(
            b["x"], b["X"], b["K"], 0, b["offsets"], n_pairs, rows, b["mask"], ctypes.c_double(px_th),
            ctypes.c_double(conf), max_iters, refine_iters, b["seeds"], b["R"], b["t"], b["mask_out"], b["n_inliers"],
            b["iters"], b["cost0"], b["cost"], None)

    for k in names:
        if k != "mask":
            assert call(**{k: True}) == -1, k
            assert L.dgb200_absolute_pose_last_error().decode() != ""
    for n_pairs in (0, -1):
        assert call(n_pairs=n_pairs) == -1
    assert call(rows=-1) == -1
    for px_th in (0.0, -1.0, float("nan"), float("inf")):
        assert call(px_th=px_th) == -1
        assert "px_th" in L.dgb200_absolute_pose_last_error().decode()
    for conf in (0.0, -0.5, 1.0000001, float("nan")):
        assert call(conf=conf) == -1
    assert call(max_iters=0) == -1
    assert call(refine_iters=-1) == -1


def test_python_argument_errors():
    import torch
    from pydegensac_b200.matching import find_absolute_pose_ragged as fap
    f64 = torch.float64
    x, X = torch.zeros((10, 2), dtype=f64), torch.zeros((10, 3), dtype=f64)
    K = torch.eye(3, dtype=f64)
    off = torch.tensor([0, 4, 10], dtype=torch.int32)
    bad = [
        dict(pts2d=np.zeros((10, 2))), dict(pts2d=torch.zeros((10, 3), dtype=f64)), dict(pts2d=torch.zeros(10, dtype=f64)),
        dict(pts2d=torch.zeros((10, 2), dtype=torch.int64)), dict(pts3d=torch.zeros((9, 3), dtype=f64)),
        dict(pts3d=torch.zeros((10, 2), dtype=f64)), dict(K=torch.eye(4, dtype=f64)), dict(K=torch.zeros((3, 3, 3))),
        dict(K=torch.eye(3, dtype=torch.int64)), dict(offsets=torch.tensor([0, 4, 10])),
        dict(offsets=torch.tensor([0], dtype=torch.int32)), dict(offsets=torch.tensor([[0, 4, 10]], dtype=torch.int32)),
        dict(mask=torch.ones(9, dtype=torch.bool)), dict(mask=torch.ones(10, dtype=torch.int32)),
        dict(mask=np.ones(10, bool)), dict(px_th=0.0), dict(px_th=-1.0), dict(px_th=float("nan")),
        dict(conf=0.0), dict(conf=1.5), dict(max_iters=0), dict(refine_iters=-1),
        dict(),                                    # well-formed, but on the host
    ]
    for kw in bad:
        args = dict(pts2d=x, pts3d=X, K=K, offsets=off)
        args.update(kw)
        with pytest.raises(ValueError):
            fap(**args)
    with pytest.raises(ValueError, match="^pts3d must be"):
        fap(x, torch.zeros((10, 2), dtype=f64), K, off)


# ------------------------------------------------------------------------------------------------ GPU
def _dev(*xs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0") for a in xs]


def _np(res):
    return {k: getattr(res, k).cpu().numpy() for k in res._fields}


def _ragged_batch(P, seed):
    """P pairs of planted scenes with per-pair K, empty and tiny pairs, mask holes and non-finite rows: (x, X, K [P],
    offsets, mask, seeds, planted (R, t) per pair)"""
    rng = np.random.default_rng(seed)
    xs, Xs, Ks, ms, truth = [], [], [], [], []
    for p in range(P):
        n = int(rng.choice([0, 2, 3, 4, 5, 9, 30]) if p % 16 == 0 else rng.integers(8, 1500))
        w = float(rng.choice([0.3, 0.5, 0.7, 0.9]) if p % 5 else 0.2)
        K = _K.copy() if p % 3 else K2.copy()
        K[0, 0] *= 1.0 + 0.2 * rng.uniform(-1, 1)
        K[0, 1] = 0.0 if p % 7 else 0.5
        x, X, R, t, _ = scene(n, w, seed * 1000 + p, noise=float(rng.uniform(0.1, 1.0)), K=K)
        m = rng.uniform(size=n) > 0.1
        if n > 10 and p % 4 == 1:
            x[3, 0] = np.nan
            X[5, 2] = np.inf
        xs.append(x); Xs.append(X); Ks.append(K); ms.append(m); truth.append((R, t))
    off = np.zeros(P + 1, np.int32)
    off[1:] = np.cumsum([len(a) for a in xs])
    seeds = rng.integers(0, 2 ** 62, P).astype(np.int64)
    return (np.concatenate(xs) if off[-1] else np.zeros((0, 2)), np.concatenate(Xs) if off[-1] else np.zeros((0, 3)),
            np.stack(Ks), off, np.concatenate(ms), seeds, truth)


def _run(x, X, K, off, mask, seeds, **kw):
    from pydegensac_b200.matching import find_absolute_pose_ragged
    dx, dX, dK, doff, dm, ds = _dev(x, X, K, off, mask, seeds)
    return _np(find_absolute_pose_ragged(dx, dX, dK, doff, dm, seeds=ds, **kw))


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


@pytest.mark.gpu
def test_kernel_against_the_oracle():
    P = 272
    x, X, K, off, mask, seeds, truth = _ragged_batch(P, 1)
    g = _run(x, X, K, off, mask, seeds, px_th=2.0, conf=0.999, max_iters=5000, refine_iters=10)
    ref = o.absolute_pose_ragged(x, X, K, off, mask, 2.0, 0.999, 5000, seeds.astype(np.uint64), 10)
    ties = 0
    worst = dict(R=0.0, t=0.0, cost0=0.0, cost=0.0)
    for p, r in enumerate(ref):
        b, e = off[p], off[p + 1]
        assert g["iters"][p] == r["iters"], p
        assert g["n_inliers"][p] == r["n_inliers"], p
        if r["near_tie"]:
            # so far only pairs of a few rows whose best pose explains just its own sample, as every sample's does
            assert r["n_inliers"] <= 3, p
            ties += 1
            continue
        assert np.array_equal(g["mask"][b:e], r["mask"]), p
        if r["n_inliers"] == 0 and np.isnan(r["cost0"]):
            assert np.isnan(g["cost0"][p]) and np.isnan(g["cost"][p]) and not g["R"][p].any()
            continue
        for k, ref_v in (("R", r["R"]), ("t", r["t"]), ("cost0", r["cost0"]), ("cost", r["cost"])):
            d = _rel(g[k][p], np.asarray(ref_v))
            worst[k] = max(worst[k], d)
            assert d <= 1e-9, (p, k, d)
        assert g["cost"][p] <= g["cost0"][p]
    n_model = int((g["n_inliers"] > 0).sum())
    print("pairs %d (with a model %d), near ties %d; worst relative difference %s; iters mean %.1f max %d"
          % (P, n_model, ties, {k: "%.2e" % v for k, v in worst.items()}, g["iters"].mean(), g["iters"].max()))
    assert ties <= 5 and n_model >= 200


@pytest.mark.gpu
def test_same_bytes_alone_in_a_batch_permuted_and_on_a_rerun():
    x, X, K, off, mask, seeds, _ = _ragged_batch(48, 2)
    full = _run(x, X, K, off, mask, seeds)
    again = _run(x, X, K, off, mask, seeds)
    for k in full:
        assert full[k].tobytes() == again[k].tobytes(), k
    perm = np.random.default_rng(0).permutation(48)
    px, pX, pm, poff = [], [], [], [0]
    for p in perm:
        b, e = off[p], off[p + 1]
        px.append(x[b:e]); pX.append(X[b:e]); pm.append(mask[b:e]); poff.append(poff[-1] + e - b)
    pres = _run(np.concatenate(px), np.concatenate(pX), K[perm], np.array(poff, np.int32), np.concatenate(pm),
                seeds[perm])
    for i, p in enumerate(perm):
        for k in ("R", "t", "n_inliers", "iters", "cost0", "cost"):
            assert full[k][p].tobytes() == pres[k][i].tobytes(), (k, p)
        assert full["mask"][off[p]:off[p + 1]].tobytes() == pres["mask"][poff[i]:poff[i + 1]].tobytes()
    for p in (1, 17, 33):
        b, e = off[p], off[p + 1]
        alone = _run(x[b:e], X[b:e], K[p:p + 1], np.array([0, e - b], np.int32), mask[b:e], seeds[p:p + 1])
        for k in ("R", "t", "n_inliers", "iters", "cost0", "cost"):
            assert full[k][p].tobytes() == alone[k][0].tobytes(), (k, p)
        assert full["mask"][b:e].tobytes() == alone["mask"].tobytes()


@pytest.mark.gpu
def test_edge_cases():
    import torch
    from pydegensac_b200.matching import find_absolute_pose_ragged
    x, X, R, t, _ = scene(300, 0.6, 9, noise=0.5)
    cases = {}
    cases["n3"] = (x[:3], X[:3])
    cases["behind"] = (x[:50], (-(X[:50] @ R.T + t) - t) @ R)          # every point mirrored behind the camera
    cases["collinear"] = (x[:40], X[0] + np.linspace(-2, 2, 40)[:, None] * np.array([1.0, 0.0, 0.0]))
    xn, Xn = x[:60].copy(), X[:60].copy()
    xn[::2, 1] = np.nan
    Xn[1::4, 0] = -np.inf
    cases["nonfinite"] = (xn, Xn)
    cases["good"] = (x, X)
    names = list(cases)
    xs = np.concatenate([cases[k][0] for k in names])
    Xs = np.concatenate([cases[k][1] for k in names])
    off = np.zeros(len(names) + 1, np.int32)
    off[1:] = np.cumsum([len(cases[k][0]) for k in names])
    seeds = np.arange(len(names), dtype=np.int64) + 5
    g = _run(xs, Xs, _K, off, np.ones(len(xs), bool), seeds)
    ref = o.absolute_pose_ragged(xs, Xs, _K, off, None, 2.0, 0.999, 10000, seeds.astype(np.uint64), 10)
    for i, k in enumerate(names):
        assert g["iters"][i] == ref[i]["iters"], k
        assert g["n_inliers"][i] == ref[i]["n_inliers"], k
        assert np.isfinite(g["R"][i]).all() and np.isfinite(g["t"][i]).all(), k
    i = names.index("n3")
    assert g["iters"][i] == 0 and np.isnan(g["cost"][i]) and not g["R"][i].any()
    i = names.index("collinear")
    assert g["n_inliers"][i] == 0 and np.isnan(g["cost0"][i]) and g["iters"][i] == 10000
    i = names.index("behind")
    assert g["n_inliers"][i] <= 5          # a sample's own three points may fit a pose; nothing else does
    i = names.index("nonfinite")
    b = off[i]
    assert not g["mask"][b:b + 60][::2].any() and not g["mask"][b + 1:b + 60:4].any()
    assert g["n_inliers"][names.index("good")] >= 150
    # refine_iters = 0: the RANSAC pose itself; conf = 1: max_iters iterations
    z = _run(x, X, _K, np.array([0, 300], np.int32), np.ones(300, bool), seeds[:1], refine_iters=0)
    r0 = o.absolute_pose(x, X, _K, seed=5, refine_iters=0)
    assert z["cost"][0] == z["cost0"][0] and z["iters"][0] == r0["iters"] and z["n_inliers"][0] == r0["n_inliers"]
    assert _rel(z["R"][0], r0["R"]) <= 1e-9
    c = _run(x, X, _K, np.array([0, 300], np.int32), np.ones(300, bool), seeds[:1], conf=1.0, max_iters=77)
    assert c["iters"][0] == 77
    # malformed offsets: no model, no row read or written (pairs 1, 2 and 4; pair 4 passes the 300 rows)
    dx, dX, dK = _dev(x, X, _K)
    bad = torch.tensor([0, 150, -1, 150, 300, 400], dtype=torch.int32, device="cuda:0")
    mo = torch.full((300,), 7, dtype=torch.uint8, device="cuda:0")
    dm = torch.ones(300, dtype=torch.bool, device="cuda:0")
    r = _np(find_absolute_pose_ragged(dx, dX, dK, bad, dm, seeds=torch.arange(5, device="cuda:0")))
    for p in (1, 2, 4):
        assert r["iters"][p] == 0 and r["n_inliers"][p] == 0 and np.isnan(r["cost"][p]) and not r["R"][p].any()
    assert r["n_inliers"][0] > 50 and r["n_inliers"][3] > 20        # (rows 180 .. 299 of the scene are outliers)
    whole = _run(x, X, _K, np.array([0, 150, 300], np.int32), np.ones(300, bool), np.array([0, 3], np.int64))
    for k in ("R", "t", "n_inliers", "iters", "cost"):
        assert whole[k][0].tobytes() == r[k][0].tobytes() and whole[k][1].tobytes() == r[k][3].tobytes(), k
    del mo


def _three_views(n_pts, n_clutter, D, seed):
    """tests.test_refine_fundamental._multiview_two_cameras with three views: views 0 and 2 by _K, view 1 by K2"""
    from tests.test_refine_fundamental import _multiview_two_cameras
    return _multiview_two_cameras(3, n_pts, n_clutter, 0, D, seed)


@pytest.mark.gpu
def test_pipeline_two_view_initialisation_then_register_a_third_view_without_sync():
    """matching (0, 1) and (2, 0) -> F RANSAC -> pose from F -> pose refinement -> re-triangulation from the refined
    calibrated F -> scatter of the points onto view 0's keypoints and gather through the (2, 0) matches ->
    find_absolute_pose_ragged, with no host synchronisation from the descriptors to the pose of view 2"""
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import (find_absolute_pose_ragged, match_descriptors_batch,
                                          pose_from_fundamental_ragged, refine_pose_ragged)
    dev = torch.device("cuda:0")
    kps, descs, Rs, ts, Ks, _ = _three_views(900, 300, 64, 21)
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    K0, K1, Kv2 = (torch.from_numpy(k).to(dev) for k in Ks)
    n0 = len(kps[0])
    seeds = torch.tensor([3], dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m = match_descriptors_batch(dt, [(0, 1)], kt, ratio=0.9, mutual=True)
        F, mask = pdg.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                                 n_max=m.n_max)
        pose = pose_from_fundamental_ragged(F, K0, K1, m.pts1, m.pts2, m.offsets, mask)
        fine = refine_pose_ragged(pose.R, pose.t, K0, K1, m.pts1, m.pts2, m.offsets, pose.in_front, px_th=1.0)
        tri = pose_from_fundamental_ragged(fine.F, K0, K1, m.pts1, m.pts2, m.offsets, fine.inliers)
        # view 0's keypoints get the first pair's points (slot n0 absorbs the rows past the pair's matches)
        live = torch.arange(m.idx1.shape[0], device=dev) < m.offsets[1]
        slot = torch.where(live, m.idx1, n0)
        P0 = torch.full((n0 + 1, 3), float("nan"), dtype=torch.float64, device=dev)
        V0 = torch.zeros(n0 + 1, dtype=torch.bool, device=dev)
        P0.index_put_((slot,), tri.points)
        V0.index_put_((slot,), tri.in_front & live)
        m2 = match_descriptors_batch(dt, [(2, 0)], kt, ratio=0.9, mutual=True)
        live2 = torch.arange(m2.idx2.shape[0], device=dev) < m2.offsets[1]
        src = torch.where(live2, m2.idx2, n0)
        view = find_absolute_pose_ragged(m2.pts1, P0.index_select(0, src), Kv2, m2.offsets,
                                         V0.index_select(0, src) & live2, px_th=2.0, seeds=seeds + 1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    # the planted pose of view 2 in camera 0's frame, translation in units of the first pair's baseline
    R20 = Rs[2] @ Rs[0].T
    t20 = ts[2] - R20 @ ts[0]
    R10 = Rs[1] @ Rs[0].T
    base = np.linalg.norm(ts[1] - R10 @ ts[0])
    R, t = view.R[0].cpu().numpy(), view.t[0].cpu().numpy()
    er, et = _rot_error(R, R20), float(np.linalg.norm(t - t20 / base))
    print("view 2 registered on %d of %d usable rows in %d iterations: rotation error %.3e rad, translation error "
          "%.3e baselines; MSAC cost %.2f -> %.2f"
          % (int(view.n_inliers[0]), int((V0.index_select(0, src) & live2).sum()), int(view.iters[0]), er, et,
             float(view.cost0[0]), float(view.cost[0])))
    assert int(view.n_inliers[0]) >= 300
    assert float(view.cost[0]) <= float(view.cost0[0])
    assert er <= 5e-3 and et <= 2e-2
