"""Refinement of the relative pose on the inliers (matching.refine_pose_ragged, dgb200_refine_pose_ragged_dev):
Levenberg-Marquardt on the Sampson error over ragged batches.  The numpy oracle tests/pose_refine_np.py is pinned to
central differences, to scipy.optimize.least_squares and to planted poses; the kernel is pinned to the oracle."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from pydegensac_b200.scenes import _K, _rot
from tests import pose_refine_np as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")
K2 = _K.copy(); K2[0, 0] *= 1.1; K2[1, 1] *= 1.07; K2[0, 2] += 7.0


def _angle(u, v):
    return float(np.arctan2(np.linalg.norm(np.cross(u, v)), u @ v))


def _rot_angle(Ra, Rb):
    return float(np.arccos(np.clip((np.trace(Ra @ Rb.T) - 1) / 2, -1, 1)))


def _scene(n, seed, noise=0.0, K2=K2):
    """Two views of n random 3-D points with a planted pose (x2 ~ R x1 + t, |t| = 1), camera 1 calibrated by _K and
    camera 2 by K2, Gaussian pixel noise in both images: p1, p2, R, t."""
    rng = np.random.default_rng(seed)
    R = _rot("z", rng.uniform(-0.1, 0.1)) @ _rot("y", rng.uniform(-0.3, 0.3)) @ _rot("x", rng.uniform(-0.1, 0.1))
    t = np.array([rng.uniform(0.5, 1.5), rng.uniform(-0.3, 0.3), rng.uniform(-0.4, 0.4)])
    t /= np.linalg.norm(t)
    X = np.c_[rng.uniform(-3, 3, n), rng.uniform(-3, 3, n), rng.uniform(3, 10, n)]
    x1 = X @ _K.T
    x2 = (X @ R.T + t) @ K2.T
    p1 = x1[:, :2] / x1[:, 2:3] + noise * rng.normal(size=(n, 2))
    p2 = x2[:, :2] / x2[:, 2:3] + noise * rng.normal(size=(n, 2))
    return p1, p2, R, t


def _off_by(R, t, degrees, seed):
    """(R, t) turned by `degrees` about seeded random axes"""
    rng = np.random.default_rng(seed)
    a, b = rng.normal(size=3), rng.normal(size=3)
    w = np.radians(degrees)
    return o.rodrigues(w * a / np.linalg.norm(a)) @ R, o.rodrigues(w * b / np.linalg.norm(b)) @ t


# ------------------------------------------------------------------------------------------------ CPU
def test_oracle_jacobian_against_central_differences():
    for seed in range(6):
        p1, p2, R, t = _scene(40, seed, noise=0.5)
        R0, t0 = _off_by(R, t, 3.0, seed)
        F, dF = o.linearise(R0, t0, _K, K2)
        r, J = o.jacobian(F, dF, p1, p2)
        assert np.abs(r - o.residuals(F, p1, p2)).max() <= 1e-12 * np.abs(r).max()
        assert np.abs(r * r - o.sampson_sq(F, p1, p2)).max() <= 1e-12 * (r * r).max()
        h = 1e-6
        Jn = np.empty_like(J)
        for k in range(5):
            D = np.zeros(5); D[k] = h
            Fa, Fb = o.fundamental(*o.step(R0, t0, D), _K, K2), o.fundamental(*o.step(R0, t0, -D), _K, K2)
            Jn[:, k] = (o.residuals(Fa, p1, p2) - o.residuals(Fb, p1, p2)) / (2 * h)
        assert np.abs(J - Jn).max() <= 1e-6 * np.abs(J).max(), (seed, np.abs(J - Jn).max() / np.abs(J).max())


@pytest.mark.parametrize("n", [50, 400, 3000])
def test_oracle_reaches_the_optimum_of_an_independent_optimiser(n):
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    p1, p2, R, t = _scene(n, 10 + n, noise=0.5)
    R0, t0 = _off_by(R, t, 1.0, n)
    got = o.refine_pair(R0, t0, _K, K2, p1, p2, max_iters=100)
    assert got["cost"] < got["cost0"] and got["iters"] < 100          # stopped on the decrease test, not the cap

    def pose(x):                                   # rotation vector about R0, t in spherical angles
        th, ph = x[3], x[4]
        return Rotation.from_rotvec(x[:3]).as_matrix() @ R0, np.array([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph),
                                                                      np.cos(th)])

    x0 = np.r_[0, 0, 0, np.arccos(t0[2]), np.arctan2(t0[1], t0[0])]
    assert np.allclose(pose(x0)[1], t0, atol=1e-14)
    sol = least_squares(lambda x: o.residuals(o.fundamental(*pose(x), _K, K2), p1, p2), x0, method="lm", xtol=1e-15,
                        ftol=1e-15, gtol=1e-15)
    Rs, ts = pose(sol.x)
    assert _rot_angle(got["R"], Rs) <= 1e-7 and _angle(got["t"], ts) <= 1e-7, (_rot_angle(got["R"], Rs), _angle(got["t"], ts))
    assert abs(got["cost"] - 2 * sol.cost) <= 1e-9 * got["cost"]
    assert abs(got["cost"] - o.sampson_sq(got["F"], p1, p2).sum()) <= 1e-9 * got["cost"]


@pytest.mark.parametrize("degrees", [2.0, 5.0])
def test_oracle_recovers_a_planted_pose(degrees):
    for seed in range(4):
        p1, p2, R, t = _scene(300, 20 + seed)
        R0, t0 = _off_by(R, t, degrees, seed)
        got = o.refine_pair(R0, t0, _K, K2, p1, p2, max_iters=20)
        assert np.abs(got["R"] - R).max() <= 1e-9 and np.abs(got["t"] - t).max() <= 1e-9, (seed, got["iters"])
        assert got["cost"] <= 1e-15 * got["cost0"]
        Fp = o.unit_frobenius(o.fundamental(R, t, _K, K2))
        assert np.abs(got["F"] - Fp).max() <= 1e-9


def _host_pieces(tmp_path):
    so = os.path.join(str(tmp_path), "libpose_refine_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-o", so, os.path.join(ROOT, "tests", "pose_refine_host.cpp")])
    return ctypes.CDLL(so)


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def test_kernel_pieces_built_for_the_host_equal_the_oracle(tmp_path):
    """csrc/pose_refine.h (residual, Jacobian, normal equations, damped solve, step) compiled with g++"""
    H = _host_pieces(tmp_path)
    c = np.zeros(6)
    H.prh_constants(_dp(c))
    assert list(c) == [o.LAMBDA0, o.LAMBDA_MIN, o.LAMBDA_MAX, o.REL_DECREASE, o.MIN_ROWS, o.ORTHO_TOL]
    A, Bk = np.ascontiguousarray(np.linalg.inv(K2).T), np.linalg.inv(_K)
    for seed, t_axis in enumerate([None, 0, 1, 2]):
        p1, p2, R, t = _scene(500, 40 + seed, noise=0.5)
        if t_axis is not None:                     # each choice of the tangent basis' coordinate axis
            t = np.full(3, 0.6); t[t_axis] = 0.1; t /= np.linalg.norm(t)
        R0, t0 = _off_by(R, t, 1.0, seed)
        F, dF, sums = np.zeros(9), np.zeros(45), np.zeros(21)
        H.prh_pass(_dp(np.ascontiguousarray(R0)), _dp(t0), _dp(A), _dp(Bk), _dp(p1), _dp(p2), len(p1), _dp(F), _dp(dF),
                   _dp(sums))
        Fo, dFo = o.linearise(R0, t0, _K, K2)
        assert np.abs(F - Fo.ravel()).max() <= 1e-12 * np.abs(Fo).max()
        assert np.abs(dF - dFo.ravel()).max() <= 1e-12 * np.abs(dFo).max()
        C, Ho, go = o._normal_equations(R0, t0, _K, K2, p1, p2)
        iu = np.triu_indices(5)
        assert abs(sums[0] - C) <= 1e-12 * C
        assert np.abs(sums[1:16] - Ho[iu]).max() <= 1e-11 * np.abs(Ho).max()
        assert np.abs(sums[16:] - go).max() <= 1e-11 * np.abs(go).max() + 1e-9 * np.sqrt(np.diag(Ho).max() * C)
        for lam in (1e-3, 1.0, 1e6):
            D, Do = np.zeros(5), o.solve_damped(Ho, go, lam)
            assert H.prh_solve(_dp(np.ascontiguousarray(Ho[iu])), _dp(go), ctypes.c_double(lam), _dp(D)) == 1
            assert np.abs(D - Do).max() <= 1e-10 * np.abs(Do).max()
        R2, t2 = np.zeros(9), np.zeros(3)
        H.prh_step(_dp(np.ascontiguousarray(R0)), _dp(t0), _dp(Do), _dp(R2), _dp(t2))
        Ro, to = o.step(R0, t0, Do)
        assert np.abs(R2 - Ro.ravel()).max() <= 1e-14 and np.abs(t2 - to).max() <= 1e-14
        Rd = np.ascontiguousarray(R0 + 1e-6 * np.arange(9).reshape(3, 3))
        want = o.orthonormalise(Rd)
        H.prh_orthonormalise.restype = ctypes.c_double
        assert H.prh_orthonormalise(_dp(Rd)) > 1e-7          # the drift it found
        assert np.abs(Rd - want).max() <= 1e-15 and np.abs(Rd @ Rd.T - np.eye(3)).max() <= 1e-15
    # a matrix that is not positive definite is refused, as the oracle refuses it
    Hbad = np.diag([1.0, 1.0, 0.0, 1.0, 1.0])
    assert o.solve_damped(Hbad, np.ones(5), 1e-3) is None
    assert H.prh_solve(_dp(np.ascontiguousarray(Hbad[np.triu_indices(5)])), _dp(np.ones(5)), ctypes.c_double(1e-3),
                       _dp(np.zeros(5))) == 0


def test_refine_entry_point_rejects_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["R", "t", "K1", "K2", "x1y1", "x2y2", "offsets", "mask", "R_out", "t_out", "F_out", "cost0", "cost",
             "n_used", "iters", "inliers"]
    optional = ("mask", "cost0", "n_used", "iters", "inliers")

    def call(n_pairs=3, rows=10, dim=2, max_iters=10, px_th=1.0, **null):
        b = {k: (None if null.get(k) else fake) for k in names}
        return L.dgb200_refine_pose_ragged_dev(b["R"], b["t"], b["K1"], b["K2"], 0, b["x1y1"], b["x2y2"], b["offsets"],
                                               n_pairs, rows, dim, b["mask"], max_iters, ctypes.c_double(px_th),
                                               b["R_out"], b["t_out"], b["F_out"], b["cost0"], b["cost"], b["n_used"],
                                               b["iters"], b["inliers"], None)

    for k in names:
        if k not in optional:
            assert call(**{k: True}) == -1, k
            assert L.dgb200_frontend_last_error().decode() != ""
    for n_pairs in (0, -1):
        assert call(n_pairs=n_pairs) == -1
    assert call(rows=-1) == -1
    for dim in (1, 0, -2):
        assert call(dim=dim) == -1
    assert call(max_iters=-1) == -1
    for px_th in (-1.0, float("nan")):
        assert call(px_th=px_th) == -1
        assert "px_th" in L.dgb200_frontend_last_error().decode()


def test_refine_python_argument_errors():
    import torch
    from pydegensac_b200.matching import refine_pose_ragged as rpr
    f64 = torch.float64
    R = torch.eye(3, dtype=f64).repeat(2, 1, 1)
    t = torch.ones((2, 3), dtype=f64)
    K = torch.eye(3, dtype=f64)
    p = torch.zeros((10, 2), dtype=f64)
    off = torch.tensor([0, 4, 10], dtype=torch.int32)
    bad = [
        dict(R=torch.zeros((2, 8))), dict(R=torch.zeros((0, 9))), dict(R=torch.zeros(9)), dict(R=np.zeros((2, 9))),
        dict(R=torch.zeros((2, 9), dtype=torch.int64)),
        dict(t=torch.ones((3, 3), dtype=f64)), dict(t=torch.ones(6, dtype=f64)), dict(t=torch.ones((2, 3), dtype=torch.int32)),
        dict(pts1=torch.zeros(10, 1, dtype=f64)), dict(pts2=torch.zeros((9, 2), dtype=f64)),
        dict(pts1=torch.zeros(10, dtype=f64)), dict(pts1=torch.zeros((10, 2), dtype=torch.int64)),
        dict(K1=torch.eye(4, dtype=f64)), dict(K2=torch.zeros((3, 3, 3), dtype=f64)), dict(K1=torch.eye(3, dtype=torch.int32)),
        dict(offsets=torch.tensor([0, 10], dtype=torch.int32)), dict(offsets=torch.tensor([0, 4, 10])),
        dict(offsets=torch.tensor([[0, 4, 10]], dtype=torch.int32)),
        dict(mask=torch.ones(9, dtype=torch.bool)), dict(mask=torch.ones(10, dtype=torch.int32)),
        dict(mask=np.ones(10, bool)),
        dict(max_iters=-1), dict(px_th=-0.5), dict(px_th=float("nan")),
        dict(),                                    # well-formed, but on the host
    ]
    for kw in bad:
        args = dict(R=R, t=t, K1=K, K2=K, pts1=p, pts2=p, offsets=off, mask=None)
        args.update(kw)
        with pytest.raises(ValueError):
            rpr(**args)
    if torch.cuda.is_available():
        dev = torch.device("cuda:0")
        with pytest.raises(ValueError, match="device"):
            rpr(R.to(dev), t.to(dev), K, K.to(dev), p.to(dev), p.to(dev), off.to(dev))


# ------------------------------------------------------------------------------------------------ GPU
LENGTHS = [0, 1, 5, 6, 33, 400, 2048, 4097, 20000]


def _batch(lengths, seed, noise=0.5, degrees=0.5, K2=K2):
    """a ragged batch of noisy planted scenes (pair p: seed + p) and, as the start, each planted pose turned by
    `degrees`: p1, p2, R0 [P,3,3], t0 [P,3], offsets, planted R, planted t"""
    ps1, ps2, R0s, t0s, Rs, ts = [], [], [], [], [], []
    for i, n in enumerate(lengths):
        p1, p2, R, t = _scene(max(n, 8), seed + i, noise=noise, K2=K2)
        R0, t0 = _off_by(R, t, degrees, seed + i)
        ps1.append(p1[:n]); ps2.append(p2[:n]); R0s.append(R0); t0s.append(t0); Rs.append(R); ts.append(t)
    off = np.r_[0, np.cumsum(lengths)].astype(np.int32)
    return np.concatenate(ps1), np.concatenate(ps2), np.stack(R0s), np.stack(t0s), off, np.stack(Rs), np.stack(ts)


def _holes(rows, seed):
    mask = np.random.default_rng(seed).random(rows) < 0.8
    mask[::7] = False
    return mask


def _dev(*xs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0") for x in xs]


def _np(res):
    return {k: v.cpu().numpy() for k, v in res._asdict().items() if v is not None}


def _same_bytes(a, b):
    return all(a[k].tobytes() == b[k].tobytes() for k in a) and a.keys() == b.keys()


@pytest.mark.gpu
@pytest.mark.parametrize("per_pair_K", [False, True])
def test_refined_batch_against_oracle(per_pair_K):
    from pydegensac_b200.matching import refine_pose_ragged
    p1, p2, R0, t0, off, _, _ = _batch(LENGTHS, 100)
    mask = _holes(len(p1), 1)
    mask[off[3]:off[4]] = True                       # the 6-row pair keeps its 6 rows: the fewest that are refined
    P = len(LENGTHS)
    if per_pair_K:
        K1 = np.stack([_K * np.array([[1 + 0.01 * p], [1 + 0.01 * p], [1]]) for p in range(P)])
        K2s = np.stack([K2 * np.array([[1 - 0.01 * p], [1 - 0.01 * p], [1]]) for p in range(P)])
    else:
        K1, K2s = _K, K2
    d1, d2, dR, dt, doff, dm, dK1, dK2 = _dev(p1, p2, R0, t0, off, mask, K1, K2s)
    # one trial step: the arithmetic of a step, to rounding
    g1 = _np(refine_pose_ragged(dR, dt, dK1, dK2, d1, d2, doff, dm, max_iters=1))
    w1 = o.refine_ragged(R0, t0, K1, K2s, p1, p2, off, mask, max_iters=1)
    assert np.array_equal(g1["iters"], w1["iters"]) and np.array_equal(g1["iters"], [0, 0, 0] + [1] * (P - 3))
    for k in ("R", "t", "F"):
        assert np.abs(g1[k] - w1[k]).max() <= 1e-11, (k, np.abs(g1[k] - w1[k]).max())
    for k in ("cost0", "cost"):
        assert np.abs(g1[k] - w1[k]).max() <= 1e-9 * np.abs(w1[k]).max(), k
    assert (g1["cost"][3:] < g1["cost0"][3:]).all()
    # the whole refinement.  At the minimum the cost is flat to 1e-12 of itself and the last trial step, of the order
    # of 1e-9 in the pose, moves it by rounding only: the kernel may take it where the oracle does not, so the poses
    # agree to that step and the costs to rounding.
    g = _np(refine_pose_ragged(dR, dt, dK1, dK2, d1, d2, doff, dm, max_iters=10))
    w = o.refine_ragged(R0, t0, K1, K2s, p1, p2, off, mask, max_iters=10)
    assert np.array_equal(g["n_used"], w["n_used"])
    assert (g["n_used"][:3] < 6).all() and (g["iters"][:3] == 0).all() and (g["iters"][3:] > 0).all()
    differ = [p for p in range(P) if g["iters"][p] != w["iters"][p]]
    print("pairs whose trial-step count differs from the oracle's (an accept / reject tie):", differ)
    assert (np.abs(g["iters"] - w["iters"]) <= 1).all()
    for p in range(P):
        for k in ("R", "t", "F"):
            assert np.abs(g[k][p] - w[k][p]).max() <= 1e-7, (p, k, np.abs(g[k][p] - w[k][p]).max())
        for k in ("cost0", "cost"):
            assert abs(g[k][p] - w[k][p]) <= 1e-9 * abs(w[k][p]), (p, k, g[k][p], w[k][p])
    # invariants of every pair
    Kb1, Kb2 = np.broadcast_to(K1, (P, 3, 3)), np.broadcast_to(K2s, (P, 3, 3))
    for p in range(P):
        R, t, F = g["R"][p], g["t"][p], g["F"][p]
        assert g["cost"][p] <= g["cost0"][p]
        assert np.abs(R @ R.T - np.eye(3)).max() <= 1e-12 and abs(np.linalg.det(R) - 1) <= 1e-12
        assert abs(np.linalg.norm(t) - 1) <= 1e-12 and abs(np.linalg.norm(F) - 1) <= 1e-12
        assert np.abs(F - o.unit_frobenius(o.fundamental(R, t, Kb1[p], Kb2[p]))).max() <= 1e-12
    # pairs of 400 rows and more are well determined: the refinement moves them towards the planted pose
    assert (g["cost"][5:] < 0.9 * g["cost0"][5:]).all()


@pytest.mark.gpu
def test_batch_independence_determinism_and_in_place():
    import torch
    from pydegensac_b200 import _cabi
    from pydegensac_b200.matching import refine_pose_ragged
    p1, p2, R0, t0, off, _, _ = _batch(LENGTHS, 200)
    mask = _holes(len(p1), 2)
    d1, d2, dR, dt, doff, dm, dK1, dK2 = _dev(p1, p2, R0, t0, off, mask, _K, K2)
    g = _np(refine_pose_ragged(dR, dt, dK1, dK2, d1, d2, doff, dm, px_th=1.0))
    assert _same_bytes(g, _np(refine_pose_ragged(dR, dt, dK1, dK2, d1, d2, doff, dm, px_th=1.0)))
    for p in range(len(LENGTHS)):
        a, b = int(off[p]), int(off[p + 1])
        one = _np(refine_pose_ragged(dR[p:p + 1], dt[p:p + 1], dK1, dK2, d1[a:b], d2[a:b],
                                     torch.tensor([0, b - a], dtype=torch.int32, device="cuda:0"), dm[a:b], px_th=1.0))
        for k in ("R", "t", "F", "cost0", "cost", "n_used", "iters"):
            assert one[k][0].tobytes() == g[k][p].tobytes(), (p, k)
        assert np.array_equal(one["inliers"], g["inliers"][a:b]), p
    # in place through the C entry point: R_out = R, t_out = t
    Ri, ti = dR.clone(), dt.clone()
    P, rows = len(LENGTHS), len(p1)
    Fo = torch.empty((P, 9), dtype=torch.float64, device="cuda:0")
    cost = torch.empty(P, dtype=torch.float64, device="cuda:0")
    vp = ctypes.c_void_p
    rc = _cabi.lib().dgb200_refine_pose_ragged_dev(
        vp(Ri.data_ptr()), vp(ti.data_ptr()), vp(dK1.data_ptr()), vp(dK2.data_ptr()), 0, vp(d1.data_ptr()),
        vp(d2.data_ptr()), vp(doff.data_ptr()), P, rows, 2, vp(dm.view(torch.uint8).data_ptr()), 10, ctypes.c_double(0.0),
        vp(Ri.data_ptr()), vp(ti.data_ptr()), vp(Fo.data_ptr()), None, vp(cost.data_ptr()), None, None, None,
        vp(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    assert Ri.cpu().numpy().tobytes() == g["R"].tobytes() and ti.cpu().numpy().tobytes() == g["t"].tobytes()
    assert Fo.cpu().numpy().tobytes() == g["F"].tobytes() and cost.cpu().numpy().tobytes() == g["cost"].tobytes()


@pytest.mark.gpu
def test_inlier_rows_are_the_sampson_rule_of_the_refined_F():
    from pydegensac_b200.matching import refine_pose_ragged
    lengths = [300, 0, 2500, 40]
    p1, p2, R0, t0, off, _, _ = _batch(lengths, 300, noise=1.0)
    rng = np.random.default_rng(3)
    out = rng.random(len(p1)) < 0.3                  # gross outliers, masked out of the fit
    p2[out] = rng.uniform(0, 640, (int(out.sum()), 2))
    d1, d2, dR, dt, doff, dm, dK1, dK2 = _dev(p1, p2, R0, t0, off, ~out, _K, K2)
    th = 1.5
    g = _np(refine_pose_ragged(dR, dt, dK1, dK2, d1, d2, doff, dm, px_th=th))
    assert g["inliers"].dtype == np.bool_ and g["inliers"].shape == (len(p1),)
    for p in range(len(lengths)):
        a, b = off[p], off[p + 1]
        r2 = o.sampson_sq(g["F"][p], p1[a:b], p2[a:b])
        clear = np.abs(r2 - th * th) >= 1e-9 * th * th
        assert np.array_equal(g["inliers"][a:b][clear], (r2 <= th * th)[clear]), p
    # written for the rows outside the mask too: some outliers fall inside the band, most inliers of the fit are inliers
    assert g["inliers"][out].any() and not g["inliers"][out].all()
    assert g["inliers"][~out].mean() > 0.5
    assert refine_pose_ragged(dR, dt, dK1, dK2, d1, d2, doff, dm).inliers is None


@pytest.mark.gpu
def test_pairs_that_are_not_refined_and_malformed_offsets():
    import torch
    from pydegensac_b200 import _cabi
    from pydegensac_b200.matching import refine_pose_ragged
    lengths = [300, 200, 150, 250, 0, 120]
    p1, p2, R0, t0, off, _, _ = _batch(lengths, 400)
    R0[1] = 0.0
    t0[2, 1] = np.nan
    mask = np.ones(len(p1), bool)
    mask[off[3] + 5:off[4]] = False                  # pair 3: five rows used
    d1, d2, dR, dt, doff, dm, dK1, dK2 = _dev(p1, p2, R0, t0, off, mask, _K, K2)
    g = _np(refine_pose_ragged(dR, dt, dK1, dK2, d1, d2, doff, dm, px_th=1.0))
    for p in (1, 2):                                 # no model
        a, b = off[p], off[p + 1]
        assert not g["R"][p].any() and not g["t"][p].any() and not g["F"][p].any()
        assert np.isnan(g["cost0"][p]) and np.isnan(g["cost"][p]) and g["n_used"][p] == 0 and g["iters"][p] == 0
        assert not g["inliers"][a:b].any()
    for p in (3, 4):                                 # fewer than 6 rows used: the pose passes through
        a, b = off[p], off[p + 1]
        assert np.array_equal(g["R"][p], R0[p]) and np.array_equal(g["t"][p], t0[p]) and g["iters"][p] == 0
        assert g["n_used"][p] == min(5, b - a) and g["cost0"][p] == g["cost"][p]
        assert np.abs(g["F"][p] - o.unit_frobenius(o.fundamental(R0[p], t0[p], _K, K2))).max() <= 1e-12
        m = mask[a:b]
        assert abs(g["cost"][p] - o.sampson_sq(g["F"][p], p1[a:b][m], p2[a:b][m]).sum()) <= 1e-9 * max(g["cost"][p], 1e-300)
    assert g["iters"][0] > 0 and g["iters"][5] > 0 and g["cost"][0] < g["cost0"][0]
    # malformed device offsets: negative, decreasing or past the rows make empty pairs whose rows stay untouched
    rows_n = len(p1)
    bad_off, = _dev(np.array([0, 300, -5, 300 + 200 + 150, rows_n + 10], dtype=np.int32))
    P = 4
    f64 = torch.float64
    out = dict(R=torch.full((P, 9), 7.0, dtype=f64, device="cuda:0"), t=torch.full((P, 3), 7.0, dtype=f64, device="cuda:0"),
               F=torch.full((P, 9), 7.0, dtype=f64, device="cuda:0"), cost0=torch.full((P,), 7.0, dtype=f64, device="cuda:0"),
               cost=torch.full((P,), 7.0, dtype=f64, device="cuda:0"),
               n_used=torch.full((P,), 7, dtype=torch.int32, device="cuda:0"),
               iters=torch.full((P,), 7, dtype=torch.int32, device="cuda:0"),
               inliers=torch.full((rows_n,), 7, dtype=torch.uint8, device="cuda:0"))
    Rb, tb = dR[[0, 3, 3, 3]].contiguous(), dt[[0, 3, 3, 3]].contiguous()
    vp = ctypes.c_void_p
    rc = _cabi.lib().dgb200_refine_pose_ragged_dev(
        vp(Rb.data_ptr()), vp(tb.data_ptr()), vp(dK1.data_ptr()), vp(dK2.data_ptr()), 0, vp(d1.data_ptr()),
        vp(d2.data_ptr()), vp(bad_off.data_ptr()), P, rows_n, 2, vp(dm.view(torch.uint8).data_ptr()), 10,
        ctypes.c_double(1.0), *[vp(out[k].data_ptr()) for k in ("R", "t", "F", "cost0", "cost", "n_used", "iters",
                                                                 "inliers")],
        vp(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    q = {k: v.cpu().numpy() for k, v in out.items()}
    assert q["R"][0].tobytes() == g["R"][0].tobytes() and q["cost"][0] == g["cost"][0] and q["iters"][0] == g["iters"][0]
    assert not q["R"][1:].any() and not q["t"][1:].any() and not q["F"][1:].any()
    assert np.isnan(q["cost0"][1:]).all() and np.isnan(q["cost"][1:]).all()
    assert not q["n_used"][1:].any() and not q["iters"][1:].any()
    assert np.array_equal(q["inliers"][:300], g["inliers"][:300].view(np.uint8)) and (q["inliers"][300:] == 7).all()


@pytest.mark.gpu
def test_drifted_rotation_is_made_orthonormal_after_an_accepted_step():
    from pydegensac_b200.matching import refine_pose_ragged
    p1, p2, R0, t0, off, _, _ = _batch([500, 500], 500)
    R0[1] = R0[1] + 1e-7 * np.arange(9).reshape(3, 3)
    d1, d2, dR, dt, doff, dK1, dK2 = _dev(p1, p2, R0, t0, off, _K, K2)
    g = _np(refine_pose_ragged(dR, dt, dK1, dK2, d1, d2, doff))
    w = o.refine_ragged(R0, t0, _K, K2, p1, p2, off)
    for p in range(2):
        R = g["R"][p]
        assert g["iters"][p] > 0 and np.abs(R @ R.T - np.eye(3)).max() <= 1e-12 and abs(np.linalg.det(R) - 1) <= 1e-12
        assert np.abs(R - w["R"][p]).max() <= 1e-7 and np.abs(g["t"][p] - w["t"][p]).max() <= 1e-7


@pytest.mark.gpu
def test_pose_from_the_refined_F_is_the_refined_pose():
    from pydegensac_b200.matching import pose_from_fundamental_ragged, refine_pose_ragged
    lengths = [400, 2048, 33, 900]
    p1, p2, R0, t0, off, _, _ = _batch(lengths, 600)
    d1, d2, dR, dt, doff, dK1, dK2 = _dev(p1, p2, R0, t0, off, _K, K2)
    fine = refine_pose_ragged(dR, dt, dK1, dK2, d1, d2, doff)
    pose = pose_from_fundamental_ragged(fine.F, dK1, dK2, d1, d2, doff)
    assert (pose.R - fine.R).abs().max().item() <= 1e-9 and (pose.t - fine.t).abs().max().item() <= 1e-9


@pytest.mark.gpu
def test_pipeline_match_ransac_pose_refine_without_sync():
    """The no-sync pipeline of test_pose_ragged.test_pipeline_match_ransac_pose_without_sync with the refinement as
    its last step: the refined poses are closer to the planted ones than the poses from the uncalibrated F, whose test
    can ask for 1e-2 only."""
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import match_descriptors_batch, pose_from_fundamental_ragged, refine_pose_ragged
    from tests.test_pose_ragged import _multiview_pose
    dev = torch.device("cuda:0")
    kps, descs, Rs, ts = _multiview_pose(4, 800, 400, 64, 5)
    pairs = np.array([(i, j) for i in range(4) for j in range(4) if i != j], dtype=np.int32)
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    seeds = torch.arange(len(pairs), dtype=torch.int64, device=dev) + 100
    K = torch.from_numpy(_K).to(dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m = match_descriptors_batch(dt, pairs, kt, ratio=0.9, mutual=True)
        F, mask = pdg.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                                 n_max=m.n_max)
        pose = pose_from_fundamental_ragged(F, K, K, m.pts1, m.pts2, m.offsets, mask)
        fine = refine_pose_ragged(pose.R, pose.t, K, K, m.pts1, m.pts2, m.offsets, pose.in_front, px_th=0.5)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    err = {"R": ([], []), "t": ([], [])}
    for p, (i, j) in enumerate(pairs):
        R = Rs[j] @ Rs[i].T
        t = ts[j] - R @ ts[i]
        t = t / np.linalg.norm(t)
        for k, res in enumerate((pose, fine)):
            err["R"][k].append(_rot_angle(res.R[p].cpu().numpy(), R))
            err["t"][k].append(_angle(res.t[p].cpu().numpy(), t))
    for name, (before, after) in err.items():
        before, after = np.array(before), np.array(after)
        print("%s error, rad: median %.3e -> %.3e, worst %.3e -> %.3e" % (name, np.median(before), np.median(after),
                                                                         before.max(), after.max()))
        # The refined pose is the least-squares estimate and sits at the noise floor (0.1 px over 800 matches); a pose
        # from the uncalibrated F scatters more widely about the planted one and now and then lands inside that floor,
        # so a single pair may get worse by part of it.  What holds: every pair reaches the floor, the worst pair and
        # the median improve.
        assert (after < (1e-4 if name == "R" else 1e-3)).all(), (name, after)
        assert after.max() < before.max(), (name, before, after)
        assert np.median(after) <= 0.5 * np.median(before), (name, np.median(before), np.median(after))
    assert (fine.cost <= fine.cost0).all().item() and (fine.n_used == pose.good).all().item()
    assert (fine.inliers.sum() >= 0.9 * mask.sum()).item()
