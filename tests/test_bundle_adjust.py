"""matching.bundle_adjust_ragged: Levenberg-Marquardt over free cameras and tracks jointly, with the Schur complement.
CPU: the numpy oracle (tests/bundle_adjust_np.py) against scipy.optimize.least_squares, its Schur step against the
full damped normal equations, its Jacobians against central differences, the scale gauge on a planted scene, the host
build of csrc/bundle_adjust.h against the oracle, special cases and the argument checks.  GPU: the kernel against the
oracle, determinism and pass-through, edge cases and a pipeline from matching to bundle adjustment without a host
synchronisation."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

from tests import bundle_adjust_np as o
from tests.test_triangulate import _point, rig, track

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")


def scene(C, T, seed, noise=0.5, outliers=0.0, lmax=12, perturb=1.0):
    """T tracks of 2 .. min(lmax, C) distinct cameras of a rig of C cameras (tests.test_triangulate.rig, mixed K), the
    planted (R, t, X) and a perturbed start: camera 0 at its planted pose, the others rotated by ~2e-3 rad and moved
    by ~1e-2, the points moved by ~2e-2 (times `perturb`).  Returns cams, pts, K, offsets, planted (R, t, X), start
    (R, t, X)."""
    rng = np.random.default_rng(seed)
    R, t, K = rig(C, seed)
    cs, xs, Xs = [], [], []
    for _ in range(T):
        L = int(rng.integers(2, min(lmax, C) + 1))
        cams = np.sort(rng.choice(C, L, replace=False))
        X = _point(R, t, cams, rng)
        out = rng.uniform(size=L) < outliers
        cs.append(cams.astype(np.int32)); xs.append(track(R, t, K, cams, X, noise, out, rng)); Xs.append(X)
    off = np.zeros(T + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in cs])
    X = np.array(Xs)
    R0, t0 = R.copy(), t.copy()
    for c in range(1, C):
        R0[c] = o.expmap(perturb * 2e-3 * rng.normal(size=3)) @ R[c]
        t0[c] = t[c] + perturb * 1e-2 * rng.normal(size=3)
    X0 = X + perturb * 2e-2 * rng.normal(size=X.shape)
    return np.concatenate(cs), np.concatenate(xs), K, off, (R, t, X), (R0, t0, X0)


def _rot_err(Ra, Rb):
    return float(np.arccos(np.clip((np.trace(Ra @ Rb.T) - 1) / 2, -1, 1)))


# ------------------------------------------------------------------------------------------------ oracle (CPU)
@pytest.mark.parametrize("C", [3, 5, 8])
@pytest.mark.parametrize("loss_scale", [None, 1.0])
def test_oracle_reaches_the_optimum_of_scipy(C, loss_scale):
    from scipy.optimize import least_squares
    cams, pts, K, off, _, (R0, t0, X0) = scene(C, 30, 10 + C)
    res = o.bundle_adjust(cams, pts, R0, t0, K, off, X0, loss_scale=loss_scale, max_iters=200)
    P = res["P"]
    n = sum(len(u) for u in o.unknowns(P)[:1]) + 3 * int(P["opt"].sum())
    if loss_scale is None:
        s = least_squares(lambda v: o.residuals(P, v), np.zeros(n), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15,
                          max_nfev=20000)
    else:
        # scipy's trust region with the Cauchy loss converges too slowly from the start to settle to 1e-8 here, so it
        # starts from the oracle's optimum, which it must not be able to lower
        from scipy.spatial.transform import Rotation
        cam_idx, trk_idx = o.unknowns(P)
        dc = np.zeros(6 * len(P["free"]))
        for q, c in enumerate(P["free"]):
            dc[6 * q:6 * q + 3] = Rotation.from_matrix(res["R"][c] @ R0[c].T).as_rotvec()
            dc[6 * q + 3:6 * q + 6] = res["t"][c] - t0[c]
        v0 = np.r_[dc[cam_idx], (res["X"][trk_idx] - X0[trk_idx]).ravel()]
        assert abs(0.5 * o.rho(o.residuals(P, v0, per_observation=True) ** 2, 1.0).sum() * 2 - res["cost"]) \
            <= 1e-10 * res["cost"]
        s = least_squares(lambda v: o.residuals(P, v, per_observation=True), v0, method="trf",
                          loss="cauchy", f_scale=loss_scale, xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=100)
    print("C %d loss %s: oracle cost %.12e after %d steps, scipy %.12e" % (C, loss_scale, res["cost"], res["iters"],
                                                                          2 * s.cost))
    assert res["cost"] <= res["cost0"]
    assert abs(res["cost"] - 2 * s.cost) <= 1e-8 * 2 * s.cost


def test_schur_step_equals_the_dense_solve():
    cams, pts, K, off, _, (R0, t0, X0) = scene(6, 40, 3, outliers=0.1)
    P = o.setup(cams, pts, R0, t0, K, off, X0, loss_scale=2.0)
    assert P["hold"] is not None
    lin = o.linearise(P, P["R"], P["t"], P["X"])
    for lam in (0.0, 1e-3, 1.0, 100.0):
        dc, dX = o.schur_step(P, lin, lam)
        ec, eX = o.dense_step(P, lin, lam)
        assert np.abs(dc - ec).max() <= 1e-9 * np.abs(ec).max(), lam
        assert np.abs(dX - eX).max() <= 1e-9 * np.abs(eX).max(), lam
        assert dc[P["hold"]] == 0.0


def test_jacobians_against_central_differences():
    R, t, K = rig(6, 2)
    rng = np.random.default_rng(3)
    cams = np.arange(6)
    X = _point(R, t, cams, rng)
    x = track(R, t, K, cams, X, 1.0, np.zeros(6, bool), rng)
    Xn = np.broadcast_to(X, (6, 3))
    r, Jc, Jx, _ = o.project(R, t, K, Xn, x)
    h = 1e-6
    for k in range(6):
        D = np.zeros(6)
        D[k] = h
        up = [o.step_pose(R[c], t[c], D) for c in cams]
        dn = [o.step_pose(R[c], t[c], -D) for c in cams]
        rp = o.project(np.array([u[0] for u in up]), np.array([u[1] for u in up]), K, Xn, x)[0]
        rm = o.project(np.array([u[0] for u in dn]), np.array([u[1] for u in dn]), K, Xn, x)[0]
        num = (rp - rm) / (2 * h)
        assert np.abs(num - Jc[:, :, k]).max() <= 1e-6 * max(1.0, np.abs(Jc[:, :, k]).max()), k
    for k in range(3):
        D = np.zeros(3)
        D[k] = h
        num = (o.project(R, t, K, Xn + D, x)[0] - o.project(R, t, K, Xn - D, x)[0]) / (2 * h)
        assert np.abs(num - Jx[:, :, k]).max() <= 1e-6 * max(1.0, np.abs(Jx[:, :, k]).max()), k


def _gauge_scene(C, T, seed):
    """noise-free planted scene whose start keeps camera 0 and the held coordinate of camera 1 at the planted values"""
    cams, pts, K, off, (R, t, X), (R0, t0, X0) = scene(C, T, seed, noise=0.0)
    a = o.gauge_axis(R0[1], t0[1], -R0[0].T @ t0[0])
    t0[1, a] = t[1, a]
    assert o.gauge_axis(R0[1], t0[1], -R0[0].T @ t0[0]) == a
    return cams, pts, K, off, (R, t, X), (R0, t0, X0), a


def test_gauge_recovers_the_planted_scene():
    cams, pts, K, off, (R, t, X), (R0, t0, X0), a = _gauge_scene(5, 60, 21)
    res = o.bundle_adjust(cams, pts, R0, t0, K, off, X0, free=[1, 2, 3, 4], scale_gauge=1, max_iters=100)
    print("planted scene: cost %.3e -> %.3e in %d steps" % (res["cost0"], res["cost"], res["iters"]))
    assert np.abs(res["R"] - R).max() <= 1e-8 and np.abs(res["t"] - t).max() <= 1e-8
    assert np.abs(res["X"] - X).max() <= 1e-8 * np.abs(X).max()
    assert res["t"][1, a].tobytes() == t0[1, a].tobytes()
    assert res["R"][0].tobytes() == R0[0].tobytes() and res["t"][0].tobytes() == t0[0].tobytes()
    # without the scale hold the same problem has a scale direction: the step still exists (damping) but the scale
    # drifts freely, so it only reaches the planted scene up to scale
    free = o.bundle_adjust(cams, pts, R0, t0, K, off, X0, free=[1, 2, 3, 4], scale_gauge=None, max_iters=100)
    assert free["cost"] <= free["cost0"]


# ------------------------------------------------------------------------------------------------ host build (CPU)
def _host(tmp_path):
    so = os.path.join(str(tmp_path), "libbundle_adjust_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-o", so, os.path.join(ROOT, "tests", "bundle_adjust_host.cpp")])
    return ctypes.CDLL(so)


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def test_host_build_equals_the_oracle(tmp_path):
    L = _host(tmp_path)
    R, t, K = rig(8, 11)
    rng = np.random.default_rng(12)
    n = 500
    c = rng.integers(0, 8, n)
    X = np.array([_point(R, t, [k], rng) for k in c])
    x = np.array([track(R, t, K, [k], Xk, 1.0, np.zeros(1, bool), rng)[0] for k, Xk in zip(c, X)])
    x[:40] = rng.uniform(0, 640, (40, 2))
    P = np.ascontiguousarray(np.c_[R[c].reshape(n, 9), t[c]])
    Kc = np.ascontiguousarray(K[c].reshape(n, 9))
    r, Jc, Jx = np.zeros(2 * n), np.zeros(12 * n), np.zeros(6 * n)
    L.bah_jacobian(_dp(P), _dp(Kc), _dp(np.ascontiguousarray(X)), _dp(np.ascontiguousarray(x)), n, _dp(r), _dp(Jc),
                   _dp(Jx))
    orr, oJc, oJx, _ = o.project(R[c], t[c], K[c], X, x)
    assert np.abs(r - orr.ravel()).max() <= 1e-12 * np.abs(orr).max()
    assert np.abs(Jc - oJc.ravel()).max() <= 1e-12 * np.abs(oJc).max()
    assert np.abs(Jx - oJx.ravel()).max() <= 1e-12 * np.abs(oJx).max()
    # the losses and weights
    s = np.ascontiguousarray((orr ** 2).sum(1))
    rh, w = np.zeros(n), np.zeros(n)
    for sig in (0.0, 0.5, 3.0):
        L.bah_loss(_dp(s), n, ctypes.c_double(sig * sig), _dp(rh), _dp(w))
        assert np.abs(rh - o.rho(s, sig * sig)).max() <= 1e-13 * max(1.0, np.abs(rh).max())
        assert np.abs(w - o.weight(s, sig * sig)).max() <= 1e-15
    # V, g of a track, its damped inverse, the Schur rows and the cross blocks
    V, g = np.zeros(6), np.zeros(3)
    wt = o.weight(s, 4.0)
    L.bah_point_terms(_dp(Jx), _dp(r), _dp(np.ascontiguousarray(wt)), n, _dp(V), _dp(g))
    oV = np.einsum("n,nik,nil->kl", wt, oJx, oJx)
    assert np.abs(V - oV[np.triu_indices(3)]).max() <= 1e-12 * np.abs(oV).max()
    assert np.abs(g - np.einsum("n,nik,ni->k", wt, oJx, orr)).max() <= 1e-11 * np.abs(g).max()
    Vi, W, Y = np.zeros(6), np.zeros(18), np.zeros(18)
    for lam in (0.0, 1e-3, 10.0):
        assert L.bah_inv3(_dp(V), ctypes.c_double(lam), _dp(Vi)) == 1
        ref = o.inv3(oV, lam)
        assert np.abs(Vi - ref[np.triu_indices(3)]).max() <= 1e-12 * np.abs(ref).max()
        assert np.abs(ref @ (oV + lam * np.diag(np.diag(oV))) - np.eye(3)).max() <= 1e-10
        L.bah_cross_block(_dp(Jc[:12].copy()), _dp(Jx[:6].copy()), ctypes.c_double(wt[0]), _dp(W))
        oW = wt[0] * oJc[0].T @ oJx[0]
        assert np.abs(W - oW.ravel()).max() <= 1e-12 * np.abs(oW).max()
        L.bah_schur_row(_dp(W), _dp(Vi), _dp(Y))
        assert np.abs(Y - (oW @ ref).ravel()).max() <= 1e-10 * np.abs(oW @ ref).max()
    assert L.bah_inv3(_dp(np.zeros(6)), ctypes.c_double(1e-3), _dp(Vi)) == 0
    assert L.bah_inv3(_dp(np.array([1.0, 2.0, 0.0, 1.0, 0.0, 1.0])), ctypes.c_double(0.0), _dp(Vi)) == 0
    # the gauge axis, ties to the lower axis
    for v, a in (([0.1, -3.0, 2.0], 1), ([2.0, 2.0, -2.0], 0), ([0.0, 1.0, -1.0], 1), ([0.0, 0.0, 0.5], 2)):
        Pg = np.r_[np.eye(3).ravel(), np.array(v)]
        assert L.bah_gauge_axis(_dp(Pg), _dp(np.zeros(3))) == a == o.gauge_axis(np.eye(3), np.array(v), np.zeros(3))
    for k in range(20):
        Pg = np.ascontiguousarray(np.r_[R[k % 8].ravel(), t[k % 8]])
        Ca = -R[0].T @ t[0] + rng.normal(size=3)
        assert L.bah_gauge_axis(_dp(Pg), _dp(np.ascontiguousarray(Ca))) == o.gauge_axis(R[k % 8], t[k % 8], Ca)


# ------------------------------------------------------------------------------------------------ special cases (CPU)
def test_oracle_special_cases():
    cams, pts, K, off, _, (R0, t0, X0) = scene(5, 40, 31)
    # an unregistered camera in free: held, passed through, its observations unused
    Ru, tu = R0.copy(), t0.copy()
    Ru[3], tu[3] = 0.0, 0.0
    r = o.bundle_adjust(cams, pts, Ru, tu, K, off, X0)
    P = r["P"]
    assert not P["active"][P["free"].index(3)] and not P["used"][cams == 3].any() and not r["mask"][cams == 3].any()
    assert r["R"][3].tobytes() == Ru[3].tobytes() and r["t"][3].tobytes() == tu[3].tobytes()
    assert r["cost"] < r["cost0"]
    # a one-camera track and an observation behind its camera at the start
    c1 = np.r_[cams, [2, 2]].astype(np.int32)
    p1 = np.r_[pts, pts[:2]]
    X1 = np.r_[X0, [[0.1, 0.2, 6.0]]]
    off1 = np.r_[off, off[-1] + 2].astype(np.int32)
    Xb = X1.copy()
    j = 5
    b, e = off1[j], off1[j + 1]
    Ci = -R0[cams[b]].T @ t0[cams[b]]
    Xb[j] = Ci - 2.0 * (X1[j] - Ci)                      # behind camera cams[b], maybe ahead of the others
    r = o.bundle_adjust(c1, p1, R0, t0, K, off1, Xb)
    P = r["P"]
    assert not P["opt"][-1] and r["X"][-1].tobytes() == X1[-1].tobytes() and not P["used"][-2:].any()
    assert not P["usable"][b]
    # free empty: structure only, every camera bit-identical
    r = o.bundle_adjust(cams, pts, R0, t0, K, off, X0, free=[])
    assert r["R"].tobytes() == R0.tobytes() and r["t"].tobytes() == t0.tobytes() and r["cost"] < r["cost0"]
    # max_iters = 0: the input comes back, cost == cost0
    r = o.bundle_adjust(cams, pts, R0, t0, K, off, X0, max_iters=0)
    assert r["iters"] == 0 and r["cost"] == r["cost0"] and r["X"].tobytes() == X0.tobytes()


# ------------------------------------------------------------------------------------------------ arguments (CPU)
def test_entry_point_rejects_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["cams", "pts", "R", "t", "K", "offsets", "X", "mask", "R_out", "t_out", "X_out", "mask_out", "cost0",
             "cost", "iters", "n_used"]

    def call(n_cams=4, n_tracks=3, obs=10, free=(1, 2, 3), gauge=1, loss_scale=0.0, max_iters=10, px_th=2.0,
             n_free=None, **null):
        b = {k: (None if null.get(k) else fake) for k in names}
        hf = (ctypes.c_int32 * max(len(free), 1))(*free)
        return L.dgb200_bundle_adjust_ragged_dev(
            b["cams"], b["pts"], b["R"], b["t"], b["K"], 0, n_cams, b["offsets"], n_tracks, obs, b["X"], b["mask"], hf,
            len(free) if n_free is None else n_free, gauge, ctypes.c_double(loss_scale), max_iters,
            ctypes.c_double(px_th), b["R_out"], b["t_out"], b["X_out"], b["mask_out"], b["cost0"], b["cost"],
            b["iters"], b["n_used"], None)

    for k in names:
        if k != "mask":
            assert call(**{k: True}) == -1, k
            assert L.dgb200_bundle_adjust_last_error().decode() != ""
    for kw in (dict(n_tracks=0), dict(obs=-1), dict(n_cams=0), dict(n_free=-1), dict(n_free=65),
               dict(free=(1, 1)), dict(free=(1, 4)), dict(free=(-1, 2)), dict(gauge=0), dict(gauge=-2),
               dict(free=(0, 1, 2, 3), gauge=1), dict(max_iters=-1)):
        assert call(**kw) == -1, kw
    assert "repeated" in (call(free=(2, 2)) == -1 and L.dgb200_bundle_adjust_last_error().decode())
    for s in (-1.0, float("nan"), float("inf")):
        assert call(loss_scale=s) == -1
        assert "loss_scale" in L.dgb200_bundle_adjust_last_error().decode()
    for px_th in (0.0, -1.0, float("nan"), float("inf")):
        assert call(px_th=px_th) == -1
        assert "px_th" in L.dgb200_bundle_adjust_last_error().decode()


def test_python_argument_errors():
    import torch
    from pydegensac_b200.matching import bundle_adjust_ragged as ba
    f64, i32 = torch.float64, torch.int32
    good = dict(cams=torch.zeros(10, dtype=i32), pts=torch.zeros((10, 2), dtype=f64),
                R=torch.eye(3, dtype=f64).repeat(4, 1, 1), t=torch.zeros((4, 3), dtype=f64), K=torch.eye(3, dtype=f64),
                offsets=torch.tensor([0, 4, 10], dtype=i32), X=torch.zeros((2, 3), dtype=f64))
    bad = [
        dict(cams=np.zeros(10, np.int32)), dict(cams=torch.zeros(10, dtype=torch.int64)),
        dict(pts=torch.zeros((10, 3), dtype=f64)), dict(R=torch.eye(3, dtype=f64)), dict(t=torch.zeros((3, 3), dtype=f64)),
        dict(K=torch.eye(3, dtype=f64).repeat(3, 1, 1)), dict(offsets=torch.tensor([0, 4, 10])),
        dict(X=torch.zeros((3, 3), dtype=f64)), dict(X=torch.zeros((2, 3), dtype=torch.int64)),
        dict(mask=torch.ones(9, dtype=torch.bool)), dict(mask=torch.ones(10, dtype=torch.int32)),
        dict(free=[1, 1]), dict(free=[4]), dict(free=[-1]), dict(free=list(range(65))),
        dict(free=torch.tensor([1]).cuda() if torch.cuda.is_available() else "x"),
        dict(scale_gauge=0), dict(scale_gauge="first"), dict(free=[0, 1, 2, 3], scale_gauge=1),
        dict(loss_scale=0.0), dict(loss_scale=-1.0), dict(loss_scale=float("nan")), dict(loss_scale=float("inf")),
        dict(max_iters=-1), dict(px_th=0.0), dict(px_th=float("nan")),
        dict(),                                    # well-formed, but on the host
    ]
    for kw in bad:
        args = dict(good)
        args.update(kw)
        with pytest.raises(ValueError):
            ba(**args)
    big = dict(good, R=torch.eye(3, dtype=f64).repeat(66, 1, 1), t=torch.zeros((66, 3), dtype=f64))
    with pytest.raises(ValueError, match="explicit free"):
        ba(**big)


# ------------------------------------------------------------------------------------------------ GPU
def _dev(*xs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0") for a in xs]


def _np(res):
    return {k: getattr(res, k).cpu().numpy() for k in res._fields}


def _run(cams, pts, R, t, K, off, X, mask=None, **kw):
    from pydegensac_b200.matching import bundle_adjust_ragged
    d = _dev(cams, pts, R, t, K, off, X)
    m = _dev(mask)[0] if mask is not None else None
    return _np(bundle_adjust_ragged(*d, mask=m, **kw))


@pytest.mark.gpu
@pytest.mark.parametrize("loss_scale", [None, 1.0])
def test_kernel_against_the_oracle(loss_scale):
    cams, pts, K, off, (R, t, X), (R0, t0, X0) = scene(12, 2000, 41, noise=0.5, outliers=0.1)
    kw = dict(free=list(range(1, 12)), scale_gauge=1, loss_scale=loss_scale, max_iters=50, px_th=2.0)
    g = _run(cams, pts, R0, t0, K, off, X0, **kw)
    ref = o.bundle_adjust(cams, pts, R0, t0, K, off, X0, **kw)
    dR = np.abs(g["R"] - ref["R"]).max()
    dt = np.abs(g["t"] - ref["t"]).max()
    dXj = np.abs(g["X"] - ref["X"]).max(1) / np.abs(ref["X"]).max()
    dX = float(np.percentile(dXj, 99))
    dc = abs(g["cost"][0] - ref["cost"]) / ref["cost"]
    print("loss %s: cost %.6e -> %.6e (oracle %.6e) in %d steps (oracle %d), n_used %d; |dR| %.2e |dt| %.2e "
          "|dX|/|X| 99th percentile %.2e, worst %.2e; rotation error %.2e -> %.2e rad" % (loss_scale, g["cost0"][0], g["cost"][0], ref["cost"],
                                                              g["iters"][0], ref["iters"], g["n_used"][0], dR, dt, dX, dXj.max(),
                                                              max(_rot_err(R0[c], R[c]) for c in range(12)),
                                                              max(_rot_err(g["R"][c], R[c]) for c in range(12))))
    assert abs(g["cost0"][0] - ref["cost0"]) <= 1e-12 * ref["cost0"]
    assert g["n_used"][0] == ref["n_used"] and g["iters"][0] == ref["iters"]
    # with the Cauchy loss a track whose outlier is down-weighted is barely constrained along its ray, and IRLS creeps
    # along that flat valley (relative cost changes of ~4e-8 per step at the end): reordered sums move such a point by
    # far more than the rest, so the points are compared at their 99th percentile
    assert dc <= 1e-9 and dR <= 1e-8 and dt <= 1e-8 and dX <= 1e-8
    assert g["cost"][0] <= g["cost0"][0]
    assert (g["mask"] == ref["mask"]).mean() >= 0.999


@pytest.mark.gpu
def test_same_bytes_on_a_rerun_and_pass_through():
    cams, pts, K, off, _, (R0, t0, X0) = scene(10, 800, 42, outliers=0.1)
    # a one-camera track and a track with a non-finite point: not optimised
    cams = np.r_[cams, [3, 3, 1, 2]].astype(np.int32)
    pts = np.r_[pts, pts[:4]]
    X0 = np.r_[X0, [[0.0, 0.0, 5.0], [np.nan, 0.0, 5.0]]]
    off = np.r_[off, off[-1] + 2, off[-1] + 4].astype(np.int32)
    kw = dict(free=[2, 4, 5, 6, 7, 8], scale_gauge=4, loss_scale=1.5, max_iters=30)
    a = _run(cams, pts, R0, t0, K, off, X0, **kw)
    b = _run(cams, pts, R0, t0, K, off, X0, **kw)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    for c in (0, 1, 3, 9):
        assert a["R"][c].tobytes() == R0[c].tobytes() and a["t"][c].tobytes() == t0[c].tobytes()
    assert a["X"][-2:].tobytes() == X0[-2:].tobytes()
    assert a["cost"][0] < a["cost0"][0] and a["iters"][0] >= 1


@pytest.mark.gpu
def test_edge_cases():
    # 64 free cameras
    cams, pts, K, off, _, (R0, t0, X0) = scene(65, 1500, 43, lmax=8)
    kw = dict(free=list(range(1, 65)), max_iters=20)
    g = _run(cams, pts, R0, t0, K, off, X0, **kw)
    ref = o.bundle_adjust(cams, pts, R0, t0, K, off, X0, **kw)
    print("64 free cameras: cost %.6e -> %.6e (oracle %.6e), %d steps (oracle %d)"
          % (g["cost0"][0], g["cost"][0], ref["cost"], g["iters"][0], ref["iters"]))
    assert abs(g["cost"][0] - ref["cost"]) <= 1e-8 * ref["cost"] and g["cost"][0] < g["cost0"][0]
    assert g["R"][0].tobytes() == R0[0].tobytes()
    # no usable observation at all: everything passes through
    cams, pts, K, off, _, (R0, t0, X0) = scene(6, 50, 44)
    z = _run(cams, pts, R0, t0, K, off, X0, mask=np.zeros(len(cams), bool))
    assert z["n_used"][0] == 0 and z["cost0"][0] == 0.0 and z["cost"][0] == 0.0 and not z["mask"].any()
    assert z["R"].tobytes() == R0.tobytes() and z["t"].tobytes() == t0.tobytes() and z["X"].tobytes() == X0.tobytes()
    # every camera held: structure only
    s = _run(cams, pts, R0, t0, K, off, X0, free=[])
    ref = o.bundle_adjust(cams, pts, R0, t0, K, off, X0, free=[])
    assert s["R"].tobytes() == R0.tobytes() and s["t"].tobytes() == t0.tobytes()
    assert abs(s["cost"][0] - ref["cost"]) <= 1e-9 * ref["cost"] and s["iters"][0] == ref["iters"]
    # max_iters = 0
    m0 = _run(cams, pts, R0, t0, K, off, X0, max_iters=0)
    assert m0["iters"][0] == 0 and m0["cost"][0] == m0["cost0"][0] and m0["X"].tobytes() == X0.tobytes()


@pytest.mark.gpu
def test_pipeline_register_triangulate_then_bundle_adjust_without_sync():
    """two-view initialisation (matching, F RANSAC, pose, refinement), P3P registration of view 2, triangulation of
    3-view tracks, then bundle adjustment of views 1 and 2 with view 0 held, without a host synchronisation"""
    import torch
    from scipy.spatial import cKDTree
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import (bundle_adjust_ragged, find_absolute_pose_ragged, match_descriptors_batch,
                                          pose_from_fundamental_ragged, refine_pose_ragged, triangulate_tracks_ragged)
    from tests.test_refine_fundamental import _multiview_two_cameras
    from tests.test_triangulate import _planted_points
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
        flat = pts[:n0].reshape(-1, 2)
        tr = triangulate_tracks_ragged(cams, flat, R, t, K, offsets, obs[:n0].reshape(-1), px_th=2.0)
        ba = bundle_adjust_ragged(cams, flat, R, t, K, offsets, tr.X, mask=tr.mask, free=[1, 2], scale_gauge=1,
                                  loss_scale=1.0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    Xw = _planted_points(900, 0, 21)
    proj = Xw @ Ks[0].T
    d, idx = cKDTree(proj[:, :2] / proj[:, 2:]).query(kps[0])
    planted = d < 0.5
    base = np.linalg.norm(ts[1] - Rs[1] @ Rs[0].T @ ts[0])
    truth = Xw[idx] / base
    n_in = tr.n_inliers.cpu().numpy()
    ok = (n_in >= 2) & planted
    Rt = [Rs[c] @ Rs[0].T for c in (1, 2)]
    rot0 = sum(_rot_err(R[c].cpu().numpy(), Rt[c - 1]) for c in (1, 2))
    rot1 = sum(_rot_err(ba.R[c].cpu().numpy(), Rt[c - 1]) for c in (1, 2))
    e0 = np.median(np.linalg.norm(tr.X.cpu().numpy()[ok] - truth[ok], axis=1))
    # the planted points are in baseline units (|t_1| = 1, as the pose refinement returns it); the scale gauge holds one
    # coordinate of t_1, so the adjusted scene is brought back to a unit baseline before it is compared
    unit = 1.0 / np.linalg.norm(ba.t[1].cpu().numpy())
    e1 = np.median(np.linalg.norm(unit * ba.X.cpu().numpy()[ok] - truth[ok], axis=1))
    c0, c1 = float(ba.cost0[0]), float(ba.cost[0])
    print("bundle adjustment of views 1, 2 over %d observations in %d steps: cost %.4f -> %.4f; rotation error "
          "%.3e -> %.3e rad; median 3D error %.3e -> %.3e baselines" % (int(ba.n_used[0]), int(ba.iters[0]), c0, c1,
                                                                        rot0, rot1, e0, e1))
    assert c1 <= c0 and int(ba.n_used[0]) >= 1500
    # three observations per point and poses already within ~4e-5 rad: the point error is the pixel noise's, which
    # joint refinement of the cameras cannot remove, so it may only stay level
    assert rot1 < rot0 and e1 <= 1.02 * e0
