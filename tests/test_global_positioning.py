"""matching.global_positioning_ragged: the views' centres and the tracks' points from the views' rotations, by
Levenberg-Marquardt on BATA's direction error with a nested Schur complement and PCG over the centres.
CPU: the oracle (tests/global_positioning_np.py) -- its Jacobian by central differences, its nested Schur step against
the full damped normal equations, its PCG against the dense reduced solve, its squared-loss optimum against scipy, its
Huber fixed point as a stationary point, planted recovery -- the host build of csrc/global_positioning.h, and the
argument checks of the Python wrapper and the C entry point.  GPU: the kernels against the oracle on scenes with several
components, unregistered views, masked rows, one-camera tracks, the padded layout, tracks that see a view twice and
outliers; determinism; the example pipeline from descriptors to bundle adjustment without a host read."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from tests import global_positioning_np as gp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")
TIGHT = 1e-13
K0 = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])


def scene(n_views, n_pts, seed, noise_px=0.5, vis=0.6, baseline=0.3):
    """n_views views along the x axis (baseline apart, a few degrees of rotation each) looking at n_pts points 4 to 6
    ahead; each point seen by each view with probability vis (at least 2 views).  Returns (cams, pts, R, offsets,
    centres, X) in the ragged track layout"""
    rng = np.random.default_rng(seed)
    R = Rotation.from_rotvec(np.radians(3.0) * rng.normal(size=(n_views, 3))).as_matrix()
    Cw = np.c_[baseline * np.arange(n_views), 0.05 * rng.normal(size=(n_views, 2))]
    X = np.c_[rng.uniform(-1.0, baseline * n_views + 1.0, n_pts), rng.uniform(-1.0, 1.0, n_pts),
              rng.uniform(4.0, 6.0, n_pts)]
    cams, pts, offsets = [], [], [0]
    for j in range(n_pts):
        seen = np.flatnonzero(rng.random(n_views) < vis)
        if len(seen) < 2:
            seen = np.sort(rng.choice(n_views, 2, replace=False))
        for v in seen:
            p = K0 @ (R[v] @ (X[j] - Cw[v]))
            cams.append(v)
            pts.append(p[:2] / p[2] + noise_px * rng.normal(size=2))
        offsets.append(len(cams))
    return (np.array(cams, np.int32), np.array(pts), R, np.array(offsets, np.int32), Cw, X)


def twice_in_a_view(cams, pts, offsets, every=5, seed=0):
    """The scene with the first observation of every `every`-th track repeated right after it, 0.3 px away: tracks that
    see one view twice (user-supplied ragged input may; build_tracks_ragged never emits them)"""
    rng = np.random.default_rng(seed)
    c2, p2, o2 = [], [], [0]
    for j in range(len(offsets) - 1):
        b, e = int(offsets[j]), int(offsets[j + 1])
        rows = list(range(b, e))
        c2 += [cams[r] for r in rows]
        p2 += [pts[r] for r in rows]
        if j % every == 0:
            c2.insert(len(c2) - len(rows) + 1, cams[b])
            p2.insert(len(p2) - len(rows) + 1, pts[b] + 0.3 * rng.normal(size=2))
        o2.append(len(c2))
    return np.array(c2, np.int32), np.array(p2), np.array(o2, np.int32)


def align(est, ref):
    """The similarity s Q est + t closest to ref (Umeyama), applied to est"""
    me, mr = est.mean(0), ref.mean(0)
    A, B = est - me, ref - mr
    U, S, Vt = np.linalg.svd(B.T @ A)
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    Q = U @ D @ Vt
    s = np.trace(np.diag(S) @ D) / np.sum(A * A)
    return (s * (Q @ A.T)).T + mr


def centres_of(R, t):
    return -np.einsum("cji,cj->ci", R, t)


# ------------------------------------------------------------------------------------------------ oracle (CPU)
def test_jacobian_by_central_differences():
    rng = np.random.default_rng(1)
    c, X, v = rng.normal(size=3), rng.normal(size=3) + 3.0, rng.normal(size=3)
    v /= np.linalg.norm(v)
    d = 0.7

    def r(z):
        return gp.residual(z[None, :3], z[None, 3:6], np.array([z[6]]), v[None])[1][0]
    z = np.r_[c, X, d]
    J = np.c_[-d * np.eye(3), d * np.eye(3), (X - c)[:, None]]
    h = 1e-6
    Jn = np.stack([(r(z + h * e) - r(z - h * e)) / (2 * h) for e in np.eye(7)], 1)
    assert np.abs(J - Jn).max() <= 1e-8


def _lin(seed=2, n_views=6, n_pts=40, loss=0.1, mask=None):
    cams, pts, R, off, Cw, Xw = scene(n_views, n_pts, seed)
    P = gp.setup(cams, pts, R, K0, off, mask)
    c, X, d = gp.start_state(P, 5, 3.0)
    rng = np.random.default_rng(seed)
    d = np.where(P["used"], rng.uniform(0.2, 2.0, len(d)), np.nan)
    L, ok = gp.linearise(P, c, X, d, loss)
    assert ok
    return P, L


def test_nested_schur_step_equals_the_dense_normal_equations():
    for loss in (0.0, 0.1):
        P, L = _lin(loss=loss)
        # (the undamped system is singular along each component's free scale, so lambda stays away from 0)
        for lam in (1e-3, 1.0, 1e3):
            ref = gp.dense_step(P, L, lam)
            got = gp.schur_step(P, L, lam, solver="dense")
            scale = max(1.0, np.abs(ref["dc"]).max(), np.abs(ref["dX"]).max(), np.abs(ref["dd"]).max())
            assert np.abs(got["dc"] - ref["dc"]).max() <= 1e-10 * scale, (loss, lam)
            tu = P["trk_used"] > 0
            assert np.abs(got["dX"][tu] - ref["dX"][tu]).max() <= 1e-10 * scale, (loss, lam)
            assert np.abs(got["dd"] - ref["dd"]).max() <= 1e-10 * scale, (loss, lam)


def test_pcg_step_equals_the_dense_reduced_solve():
    P, L = _lin(3, 10, 80)
    for lam in (1e-6, 1e-3, 10.0):
        ref = gp.schur_step(P, L, lam, solver="dense")
        got = gp.schur_step(P, L, lam, solver="pcg", cg_tol=1e-14, cg_max_iters=500)
        scale = max(1.0, np.abs(ref["dc"]).max())
        assert not got["rejected"] and got["cg"] < 500
        assert np.abs(got["dc"] - ref["dc"]).max() <= 1e-9 * scale, lam


def test_preconditioner_is_the_diagonal_block_of_s():
    """M_i is S's exact diagonal block, also for tracks that see one view twice"""
    cams, pts, R, off, Cw, Xw = scene(8, 60, 21)
    cams, pts, off = twice_in_a_view(cams, pts, off)
    P = gp.setup(cams, pts, R, K0, off)
    c, X, d = gp.start_state(P, 5, 3.0)
    L, ok = gp.linearise(P, c, X, d, 0.1)
    assert ok
    for lam in (1e-6, 1e-3, 1.0):
        Vi, t = gp.points(P, L, lam)
        U, M, b, mov = gp.reduced(P, L, lam, Vi, t)
        for i in np.flatnonzero(mov):
            Sii = np.zeros((3, 3))
            for k in range(3):
                e = np.zeros((P["C"], 3))
                e[i, k] = 1.0
                Sii[:, k] = gp.schur_matvec(P, L, lam, Vi, U, e)[i]
            assert np.abs(M[i] - Sii).max() <= 1e-12 * np.abs(Sii).max(), (lam, i)
        np.linalg.cholesky(M)


def test_squared_loss_cost_at_or_below_scipy():
    from scipy.optimize import least_squares
    cams, pts, R, off, Cw, Xw = scene(6, 40, 4)
    out = gp.global_positioning(cams, pts, R, K0, off, loss_scale=0.0, seed=3, cg_tol=TIGHT, max_iters=200)
    P = out["P"]
    c0, X0, d0 = out["start"]
    mov, tu, u = np.flatnonzero(P["moving"]), np.flatnonzero(P["trk_used"]), np.flatnonzero(P["used"])
    nc, nt = 3 * len(mov), 3 * len(tu)

    def unpack(z):
        c, X, d = c0.copy(), X0.copy(), d0.copy()
        c[mov] = z[:nc].reshape(-1, 3)
        X[tu] = z[nc:nc + nt].reshape(-1, 3)
        d[u] = z[nc + nt:]
        return c, X, d

    def res(z):
        c, X, d = unpack(z)
        return gp.residual(c[P["cams"][u]], X[P["track_of"][u]], d[u], P["v"][u])[1].reshape(-1)
    z0 = np.r_[c0[mov].reshape(-1), X0[tu].reshape(-1), d0[u]]
    lo = np.r_[np.full(nc + nt, -np.inf), np.full(len(u), gp.D_MIN)]
    sol = least_squares(res, z0, bounds=(lo, np.inf), method="trf", x_scale="jac", xtol=1e-15, ftol=1e-15,
                        gtol=1e-15, max_nfev=20000)
    ref = float(np.sum(sol.fun ** 2))
    print("squared loss: oracle %.6e in %d steps, scipy %.6e" % (out["cost"], out["iters"], ref))
    assert out["cost"] <= ref * (1.0 + 1e-6) + 1e-15


def test_huber_fixed_point_is_stationary():
    cams, pts, R, off, Cw, Xw = scene(6, 40, 5)
    rng = np.random.default_rng(5)
    bad = rng.random(len(cams)) < 0.03
    pts = pts.copy()
    pts[bad] = rng.uniform(0, 640, (int(bad.sum()), 2))
    out = gp.global_positioning(cams, pts, R, K0, off, seed=1, cg_tol=TIGHT, max_iters=400)
    assert out["iters"] < 400
    P, c, X, d = out["P"], out["c"], out["X"], out["d"]
    mov, tu, u = np.flatnonzero(P["moving"]), np.flatnonzero(P["trk_used"]), np.flatnonzero(P["used"])

    def f(c, X, d):
        return gp.total_cost(P, c, X, d, 0.1)
    h = 1e-7
    g = []
    for arr, idx in ((c, mov), (X, tu)):
        for i in idx:
            for k in range(3):
                a1, a2 = arr.copy(), arr.copy()
                a1[i, k] += h
                a2[i, k] -= h
                args1 = (a1, X, d) if arr is c else (c, a1, d)
                args2 = (a2, X, d) if arr is c else (c, a2, d)
                g.append((f(*args1) - f(*args2)) / (2 * h))
    for o in u:
        d1, d2 = d.copy(), d.copy()
        d1[o] += h
        d2[o] = max(d[o] - h, 0.0)
        gd = (f(c, X, d1) - f(c, X, d2)) / (d1[o] - d2[o])
        g.append(min(gd, 0.0) if d[o] <= gp.D_MIN * (1 + 1e-12) else gd)
    g = np.abs(np.array(g))
    print("largest projected gradient component at the fixed point: %.3e (cost %.4e)" % (g.max(), out["cost"]))
    assert g.max() <= 1e-5


def test_planted_recovery_oracle():
    cams, pts, R, off, Cw, Xw = scene(10, 150, 6, noise_px=0.5)
    out = gp.global_positioning(cams, pts, R, K0, off, seed=0)
    Ce = centres_of(R, out["t"])
    err = np.linalg.norm(align(Ce, Cw) - Cw, axis=1)
    print("10 views: centre errors after alignment: largest %.2e (baseline 0.3), %d steps, CG %d"
          % (err.max(), out["iters"], out["cg_iters"]))
    # measured with this seed: largest error 3.5e-3 in 10 trial steps; 0.5 px noise at f = 500 is 1e-3 rad
    assert err.max() < 0.01 and out["iters"] < 60
    assert (out["component"] == 0).all() and out["inliers"].mean() > 0.95


# ------------------------------------------------------------------------------------------------ host build (CPU)
def test_host_build_matches_the_oracle(tmp_path):
    so = os.path.join(str(tmp_path), "libglobal_positioning_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-o", so, os.path.join(ROOT, "tests", "global_positioning_host.cpp")])
    L = ctypes.CDLL(so)
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))  # noqa: E731
    rng = np.random.default_rng(8)
    n = 400
    R = np.ascontiguousarray(Rotation.random(n, random_state=rng).as_matrix())
    K = np.ascontiguousarray(np.broadcast_to(K0, (n, 3, 3)) * rng.uniform(0.5, 2.0, (n, 1, 1)))
    K[:, 2, 2] = 1.0
    xy = np.ascontiguousarray(rng.uniform(-100, 800, (n, 2)))
    v = np.zeros((n, 3))
    L.gph_ray(n, dp(R), dp(K), dp(xy), dp(v))
    Ki = np.stack([gp.k_inverse(K[i]) for i in range(n)])
    assert np.array_equal(v, gp.ray(Ki, R, xy[:, 0], xy[:, 1]))
    idx = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    for kind in (0, 1):
        s = np.zeros((n, 3))
        L.gph_start(n, ctypes.c_ulonglong(0x123456789ABCDEF), kind, idx.ctypes.data_as(ctypes.POINTER(ctypes.c_uint)),
                    ctypes.c_double(100.0), dp(s))
        ref = np.stack([gp.start(0x123456789ABCDEF, kind, int(i), 100.0) for i in idx])
        assert np.array_equal(s, ref)
        assert np.abs(s).max() < 100.0
    c, X = rng.normal(size=(n, 3)), rng.normal(size=(n, 3))
    X[:5] = c[:5]                                     # |a| = 0: the linearisation is refused
    d = rng.uniform(1e-5, 3.0, n)
    for delta in (0.0, 0.1):
        outs = {k: np.zeros((n, 3)) for k in ("a", "r", "u", "h")}
        outs.update({k: np.zeros(n) for k in ("s2", "rho", "w", "nrm", "s", "ar")})
        ok = np.zeros(n, np.intc)
        L.gph_terms(n, dp(c), dp(X), dp(d), dp(v), ctypes.c_double(delta), dp(outs["a"]), dp(outs["r"]),
                    dp(outs["s2"]), dp(outs["rho"]), dp(outs["w"]), ok.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                    dp(outs["u"]), dp(outs["nrm"]), dp(outs["s"]), dp(outs["h"]), dp(outs["ar"]))
        a, r, s2 = gp.residual(c, X, d, v)
        assert np.array_equal(outs["a"], a) and np.array_equal(outs["r"], r) and np.array_equal(outs["s2"], s2)
        assert np.array_equal(outs["rho"], gp.rho(s2, delta)) and np.array_equal(outs["w"], gp.weight(s2, delta))
        with np.errstate(invalid="ignore", divide="ignore"):
            okr, u, nr, s, h, ar = gp.obs_terms(a, r, d, outs["w"])
        assert np.array_equal(ok.astype(bool), okr) and (~okr[:5]).all() and okr[5:].all()
        for k, ref in (("u", u), ("nrm", nr), ("s", s), ("h", h), ("ar", ar)):
            assert np.array_equal(outs[k][okr], ref[okr]), k
    u = outs["u"][5:]
    m = n - 5
    p = rng.normal(size=(m, 3))
    for lam in (1e-12, 1e-3, 10.0):
        out, blk, dn, th = np.zeros((m, 3)), np.zeros((m, 6)), np.zeros(m), np.zeros(m)
        su, sa, sn, sd = (np.ascontiguousarray(x[5:]) for x in (outs["s"], outs["ar"], outs["nrm"], d))
        uc = np.ascontiguousarray(u)
        L.gph_blocks(m, dp(uc), dp(su), ctypes.c_double(lam), dp(p), dp(sa), dp(sn), dp(sd), dp(out), dp(blk), dp(dn),
                     dp(th))
        assert np.array_equal(out, gp.m_apply(uc, su, 1.0 / (1.0 + lam), p))
        assert np.array_equal(blk, gp.block(su, gp.outer6(uc, su), lam))
        assert np.array_equal(dn, gp.scale_step(sa, sn, sd, uc, p, lam))
        assert np.abs(th - gp.angle(uc, p)).max() <= 1e-15     # (atan2: glibc's and numpy's differ in the last bit)


# ------------------------------------------------------------------------------------------------ arguments (CPU)
def test_python_messages():
    torch = pytest.importorskip("torch")
    from pydegensac_b200.matching import global_positioning_ragged
    f64, i32 = torch.float64, torch.int32
    good = dict(cams=torch.zeros(4, dtype=i32), pts=torch.zeros((4, 2), dtype=f64),
                R=torch.eye(3, dtype=f64).repeat(2, 1, 1), K=torch.eye(3, dtype=f64),
                offsets=torch.tensor([0, 2, 4], dtype=i32))
    host = "cams, pts, R, K, offsets and mask must be CUDA tensors on one device"
    cases = [
        ({"cams": [0, 0, 0, 0]}, "cams must be a torch tensor"),
        ({"offsets": torch.tensor([0], dtype=i32)}, "offsets must be [T+1] with T >= 1, not [1]"),
        ({"offsets": torch.tensor([0, 4])}, "offsets must be int32, not torch.int64"),
        ({"cams": torch.zeros(4)}, "cams must be int32, not torch.float32"),
        ({"pts": torch.zeros((4, 3), dtype=f64)}, "pts must be [obs,2], not [4, 3]"),
        ({"cams": torch.zeros(3, dtype=i32)}, "cams must be [obs] = [4], not [3]"),
        ({"R": torch.eye(3, dtype=f64)}, "R must be [C,3,3] with C >= 1, not [3, 3]"),
        ({"K": torch.eye(3, dtype=f64).repeat(3, 1, 1)}, "K must be [3,3] or [C,3,3] with C = 2, not [3, 3, 3]"),
        ({"pts": torch.zeros((4, 2), dtype=i32)}, "pts must be a floating tensor, not torch.int32"),
        ({"mask": torch.ones(3, dtype=torch.bool)}, "mask must be [obs] = [4], not [3]"),
        ({"seed": -1}, "seed must lie in [0, 2^64), not -1"),
        ({"init_scale": -1.0}, "init_scale must be a non-negative finite number, not -1.0"),
        ({"init_scale": float("inf")}, "init_scale must be a non-negative finite number, not inf"),
        ({"loss_scale": float("nan")}, "loss_scale must be a non-negative finite number, not nan"),
        ({"loss_scale": -0.1}, "loss_scale must be a non-negative finite number, not -0.1"),
        ({"max_angle": float("inf")}, "max_angle must be a non-negative finite number, not inf"),
        ({"max_iters": -1}, "max_iters must not be negative, not -1"),
        ({"cg_max_iters": 0}, "cg_max_iters must be at least 1, not 0"),
        ({"cg_tol": -1e-6}, "cg_tol must be a non-negative finite number, not -1e-06"),
        ({"cg_tol": float("nan")}, "cg_tol must be a non-negative finite number, not nan"),
        ({"init_scale": 0.0, "loss_scale": 0.0, "max_angle": 0.0, "max_iters": 0, "cg_tol": 0.0}, host),
        ({}, host),
    ]
    for kw, msg in cases:
        with pytest.raises(ValueError) as e:
            global_positioning_ragged(**dict(good, **kw))
        assert str(e.value) == msg, kw


def test_c_entry_point_refuses_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["cams", "pts", "R", "K", "offsets", "t", "X", "component", "angle", "inliers", "cost0", "cost", "iters",
             "n_used", "cg_iters"]

    def call(n_cams=2, n_tracks=2, obs=4, init_scale=100.0, loss_scale=0.1, max_iters=100, max_angle=0.03,
             cg_max_iters=500, cg_tol=1e-6, null=()):
        b = {k: (None if k in null else fake) for k in names}
        return L.dgb200_global_positioning_ragged_dev(
            b["cams"], b["pts"], b["R"], b["K"], 0, n_cams, b["offsets"], n_tracks, obs, None, 7,
            ctypes.c_double(init_scale), ctypes.c_double(loss_scale), max_iters, ctypes.c_double(max_angle),
            cg_max_iters, ctypes.c_double(cg_tol), b["t"], b["X"], b["component"], b["angle"], b["inliers"],
            b["cost0"], b["cost"], b["iters"], b["n_used"], b["cg_iters"], None)

    sizes = "need n_tracks >= 1, obs >= 0 and n_cams >= 1"
    nnf = "must be a non-negative finite number"
    cases = [(dict(null={k}), "null buffer") for k in ("R", "K", "offsets", "t", "X", "component", "cost0", "cost",
                                                       "iters", "n_used", "cg_iters")]
    cases += [(dict(null={k}), "null observation buffer") for k in ("cams", "pts", "angle", "inliers")]
    cases += [
        (dict(n_tracks=0), sizes), (dict(obs=-1), sizes), (dict(n_cams=0), sizes),
        (dict(loss_scale=-1.0), "loss_scale must be a positive number (or 0 for the trivial loss)"),
        (dict(loss_scale=float("inf")), "loss_scale must be a positive number (or 0 for the trivial loss)"),
        (dict(loss_scale=float("nan")), "loss_scale must be a positive number (or 0 for the trivial loss)"),
        (dict(max_iters=-1), "max_iters must not be negative"),
        (dict(init_scale=-1.0), "init_scale " + nnf), (dict(init_scale=float("nan")), "init_scale " + nnf),
        (dict(max_angle=-0.1), "max_angle " + nnf), (dict(max_angle=float("inf")), "max_angle " + nnf),
        (dict(cg_max_iters=0), "cg_max_iters must be at least 1"),
        (dict(cg_tol=float("nan")), "cg_tol " + nnf), (dict(cg_tol=-1.0), "cg_tol " + nnf),
        (dict(null={"cams"}, obs=0, n_tracks=0), sizes),
    ]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert L.dgb200_global_positioning_last_error().decode() == msg, kw


# ------------------------------------------------------------------------------------------------ GPU
def _scenes():
    """(name, cams, pts, R, offsets, mask) over every kind of input the estimator distinguishes"""
    out = []
    c, p, R, o, _, _ = scene(8, 60, 10)
    out.append(("one component", c, p, R, o, None))
    c1, p1, R1, o1, _, _ = scene(6, 40, 11)
    c2, p2, R2, o2, _, _ = scene(5, 30, 12)
    # views 0 and 1 see nothing; then two components; view 13 is unregistered (NaN rotation)
    cams = np.r_[c1 + 2, c2 + 8].astype(np.int32)
    pts = np.r_[p1, p2]
    offs = np.r_[o1, o2[1:] + o1[-1]].astype(np.int32)
    Rall = np.r_[np.tile(np.eye(3), (2, 1, 1)), R1, R2, np.full((1, 3, 3), np.nan)]
    rng = np.random.default_rng(13)
    mask = rng.random(len(cams)) > 0.1
    # one-camera tracks and a track on the unregistered view
    extra_c = np.array([3, 3, 9, 13, 13, 4], np.int32)
    extra_p = rng.uniform(0, 640, (6, 2))
    cams = np.r_[cams, extra_c].astype(np.int32)
    pts = np.r_[pts, extra_p]
    mask = np.r_[mask, np.ones(6, bool)]
    offs = np.r_[offs, offs[-1] + 2, offs[-1] + 3, offs[-1] + 6].astype(np.int32)
    out.append(("components, unregistered views, masked rows, one-camera tracks", cams, pts, Rall, offs, mask))
    # the padded layout of build_tracks_ragged: empty tracks past T, rows with cams = -1 and pts = NaN past the last
    c, p, R, o, _, _ = scene(7, 50, 14)
    cams = np.r_[c, np.full(9, -1)].astype(np.int32)
    pts = np.r_[p, np.full((9, 2), np.nan)]
    offs = np.r_[o, np.full(5, o[-1])].astype(np.int32)
    out.append(("padded layout", cams, pts, R, offs, None))
    # tracks that see one view twice
    c, p, R, o, _, _ = scene(8, 60, 16)
    c, p, o = twice_in_a_view(c, p, o)
    out.append(("a view twice in a track", c, p, R, o, None))
    # rows with outliers, a Huber problem
    c, p, R, o, _, _ = scene(9, 80, 15)
    p = p.copy()
    bad = rng.random(len(c)) < 0.05
    p[bad] = rng.uniform(0, 640, (int(bad.sum()), 2))
    out.append(("outliers", c, p, R, o, None))
    return out


def _run(cams, pts, R, offsets, mask=None, K=K0, **kw):
    import torch
    from pydegensac_b200.matching import global_positioning_ragged
    dev = torch.device("cuda:0")
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    out = global_positioning_ragged(T(cams), T(pts), T(R), T(K), T(offsets), mask=T(mask) if mask is not None else None,
                                    **kw)
    return {k: getattr(out, k).cpu().numpy() for k in out._fields}


def unscaled(t, X, R, P):
    """t and X with each component's scale taken out: divided by the RMS distance of the component's centres from its
    anchor (a track belongs to the component of its views)"""
    comp = P["comp"]
    C = centres_of(R, np.nan_to_num(t))
    t2, X2 = t.copy(), X.copy()
    trk_comp = np.full(P["T"], -1)
    u = np.flatnonzero(P["used"])
    trk_comp[P["track_of"][u]] = comp[P["cams"][u]]
    for a in set(comp[comp >= 0].tolist()):
        s = np.sqrt(np.mean(np.sum(C[comp == a] ** 2, axis=1)))
        t2[comp == a] /= s
        X2[trk_comp == a] /= s
    return t2, X2


def _close(a, b, tol):
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.nan_to_num(np.abs(a - b)).max() <= tol


@pytest.mark.gpu
def test_full_call_equals_the_oracle():
    for name, c, p, R, o, m in _scenes():
        g = _run(c, p, R, o, m, seed=3, cg_tol=TIGHT)
        r = gp.global_positioning(c, p, R, K0, o, m, seed=3, cg_tol=TIGHT)
        sc = max(1.0, np.nanmax(np.abs(r["X"])))
        print("%s: %d steps (oracle %d), CG %d (oracle %d), cost %.6e (oracle %.6e), largest |dt| %.2e, |dX| %.2e"
              % (name, g["iters"][0], r["iters"], g["cg_iters"][0], r["cg_iters"], g["cost"][0], r["cost"],
                 np.nanmax(np.abs(g["t"] - r["t"])), np.nanmax(np.abs(g["X"] - r["X"]))))
        assert g["iters"][0] == r["iters"], name
        # Each component's scale is free and held by the damping alone, so the rounding of the device's and numpy's
        # sums moves t and X along it (by up to 4e-6 of the scene with outliers, whose scales sit at d_min).  t and X
        # are compared with that scale taken out: each component's divided by the RMS distance of its centres from
        # its anchor, in each result.
        gt, gX = unscaled(g["t"], g["X"], R, r["P"])
        rt, rX = unscaled(r["t"], r["X"], R, r["P"])
        sc = max(1.0, np.nanmax(np.abs(rX)))
        print("  without the scale: largest |dt| %.2e, |dX| %.2e" % (np.nanmax(np.abs(gt - rt)),
                                                                     np.nanmax(np.abs(gX - rX))))
        assert _close(gt, rt, 1e-9 * sc), name
        assert _close(gX, rX, 1e-9 * sc), name
        assert _close(g["angle"], r["angle"], 1e-9), name
        assert (g["component"] == r["component"]).all(), name
        assert (g["inliers"] == r["inliers"]).all(), name
        assert g["n_used"][0] == r["n_used"], name
        assert abs(g["cost0"][0] - r["cost0"]) <= 1e-12 * r["cost0"], name
        assert g["cost"][0] <= g["cost0"][0], name


@pytest.mark.gpu
def test_same_bytes_on_a_rerun_and_unused_outputs():
    name, c, p, R, o, m = _scenes()[1]
    a = _run(c, p, R, o, m, seed=9)
    b = _run(c, p, R, o, m, seed=9)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    r = gp.global_positioning(c, p, R, K0, o, m, seed=9, max_iters=0)
    P = r["P"]
    assert (a["component"][:2] == -1).all() and a["component"][13] == -1 and np.isnan(a["t"][[0, 1, 13]]).all()
    assert set(a["component"][P["active"]].tolist()) == {2, 8}
    assert (a["t"][[2, 8]] == 0.0).all()                               # the anchors sit at the origin
    T = len(o) - 1
    unused = np.flatnonzero(P["trk_used"][:T] == 0)
    assert {T - 3, T - 2, T - 1} <= set(unused.tolist()) and np.isnan(a["X"][unused]).all()   # + masked-out tracks
    assert (np.isnan(a["angle"]) == ~P["used"]).all() and not a["inliers"][~P["used"]].any()


@pytest.mark.gpu
def test_planted_recovery_device():
    cams, pts, R, off, Cw, Xw = scene(10, 150, 6, noise_px=0.5)
    g = _run(cams, pts, R, off, seed=0)
    err = np.linalg.norm(align(centres_of(R, g["t"]), Cw) - Cw, axis=1)
    print("device: largest centre error %.2e after alignment, %d steps, CG %d" % (err.max(), g["iters"][0],
                                                                                   g["cg_iters"][0]))
    assert err.max() < 0.01


@pytest.mark.gpu
def test_example_pipeline_without_a_host_read():
    """examples/gpu_pipeline.py: descriptors to matching, F RANSAC, pose, refinement, rotation averaging, tracks,
    positioning, triangulation on its inliers and bundle adjustment, with no host read; errors measured after BA"""
    import sys
    import torch
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import gpu_pipeline
    from pydegensac_b200.scenes import _K
    dev = torch.device("cuda:0")
    K = torch.from_numpy(_K).to(dev)
    scene = gpu_pipeline.path_scene(dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = gpu_pipeline.global_reconstruction_run(dev, K, scene)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    c0, c1, r1 = gpu_pipeline.report_global_reconstruction(scene, out)
    # measured on an H100: largest centre error 1.6e-2 positioned and 1.4e-3 after BA (the views are 0.3 apart), largest
    # rotation error 0.013 deg after BA; positioning took 49 trial steps
    assert c0 < 0.05 and c1 < 0.005 and c1 < c0 and r1 < 0.05
