"""Refinement of fundamental matrices on their inliers (matching.refine_fundamental_ragged,
dgb200_refine_fundamental_ragged_dev): Levenberg-Marquardt on the Sampson error over the rank-2 matrices, for ragged
batches.  The numpy oracle tests/refine_fundamental_np.py is pinned to central differences, to the engine's Sampson
formula, to scipy.optimize.least_squares and to planted scenes; the kernel is pinned to the oracle.  The scenes use
different intrinsics in the two views, so that F is not an essential matrix in disguise."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from pydegensac_b200.scenes import _K, _rot
from tests import refine_fundamental_np as o
from tests.test_pose_refine import K2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")


def _fundamental(R, t, K1=_K, K2=K2):
    """K2^-T [t]x R K1^-1 at unit norm (x2^T F x1 = 0)"""
    tx = np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])
    F = np.linalg.inv(K2).T @ tx @ R @ np.linalg.inv(K1)
    return F / np.linalg.norm(F)


def _scene(n, seed, noise=0.0, n_hold=300, plane=False):
    """Two views (camera 1 by _K, camera 2 by K2) of n random 3-D points with a planted pose and Gaussian pixel noise in
    both images, and n_hold noise-free held-out views of further points of the scene: p1, p2, the planted F, q1, q2.
    plane: the n points lie on one plane (F is then poorly determined by them); the held-out points do not."""
    rng = np.random.default_rng(seed)
    R = _rot("z", rng.uniform(-0.1, 0.1)) @ _rot("y", rng.uniform(-0.3, 0.3)) @ _rot("x", rng.uniform(-0.1, 0.1))
    t = np.array([rng.uniform(0.5, 1.5), rng.uniform(-0.3, 0.3), rng.uniform(-0.4, 0.4)])
    t /= np.linalg.norm(t)
    m = n + n_hold
    X = np.c_[rng.uniform(-3, 3, m), rng.uniform(-3, 3, m), rng.uniform(3, 10, m)]
    if plane:
        X[:n, 2] = 6.0 + 0.3 * X[:n, 0] - 0.2 * X[:n, 1]
    x1 = X @ _K.T
    x2 = (X @ R.T + t) @ K2.T
    h1, h2 = x1[:, :2] / x1[:, 2:3], x2[:, :2] / x2[:, 2:3]
    p1 = h1[:n] + noise * rng.normal(size=(n, 2))
    p2 = h2[:n] + noise * rng.normal(size=(n, 2))
    return p1, p2, _fundamental(R, t), h1[n:], h2[n:]


def _perturbed(F, seed, size=1.0):
    """F moved by a few pixels over both images (size 1: about 1-5 px): A2^T F A1 with A1, A2 affine maps near the
    identity, so the result has rank 2"""
    rng = np.random.default_rng(seed)
    A = []
    for _ in range(2):
        e = size * rng.uniform(-1, 1, 5)
        A.append(np.array([[1 + 5e-3 * e[0], 5e-3 * e[1], 2.0 * e[2]], [5e-3 * e[3], 1 - 5e-3 * e[0], 2.0 * e[4]],
                           [0.0, 0.0, 1.0]]))
    return A[1].T @ F @ A[0]


def geometry_error(F, q1, q2):
    """the mean Sampson distance (px) of noise-free held-out correspondences of the planted scene under F"""
    return float(np.sqrt(o.sampson_sq(F, q1, q2)).mean())


# ------------------------------------------------------------------------------------------------ CPU
def test_oracle_jacobian_basis_and_residual_formula():
    for seed in range(6):
        p1, p2, F, _, _ = _scene(40, seed, noise=0.5)
        F0 = _perturbed(F, seed)
        if seed % 2:
            F0 = F0 + 1e-3 * np.abs(F0).max() * np.random.default_rng(seed).normal(size=(3, 3))   # full rank
        T1, T2 = o.transform(p1), o.transform(p2)
        Fn = o.start(T1, T2, F0)
        assert abs(np.linalg.det(Fn.reshape(3, 3))) <= 1e-15 and abs(Fn @ Fn - 1) <= 1e-15
        B = o.basis(Fn)
        c = o.unit(o.cofactor(Fn))
        assert np.abs(B.T @ B - np.eye(7)).max() <= 1e-15
        assert np.abs(Fn @ B).max() <= 1e-15 and np.abs(c @ B).max() <= 1e-15
        F, dF = o.linearise(T1, T2, Fn)
        r, J = o.jacobian(F, dF, p1, p2)
        # the engine's Sampson formula (fgeom.h) against the textbook one and the residual's square
        Fm = F.reshape(3, 3)
        h1, h2 = np.c_[p1, np.ones(len(p1))], np.c_[p2, np.ones(len(p2))]
        a, b = h1 @ Fm.T, h2 @ Fm
        want = (h2 * a).sum(1) ** 2 / (a[:, 0] ** 2 + a[:, 1] ** 2 + b[:, 0] ** 2 + b[:, 1] ** 2)
        r2 = o.sampson_sq(F, p1, p2)
        assert np.abs(r2 - want).max() <= 1e-12 * want.max() and np.abs(r * r - r2).max() <= 1e-12 * r2.max()
        h = 1e-6
        Jn = np.empty_like(J)
        for k in range(7):
            D = np.zeros(7); D[k] = h
            ra = o.residuals(o.to_pixels(T1, T2, o.retract(Fn, D)), p1, p2)
            rb = o.residuals(o.to_pixels(T1, T2, o.retract(Fn, -D)), p1, p2)
            Jn[:, k] = (ra - rb) / (2 * h)
        assert np.abs(J - Jn).max() <= 1e-6 * np.abs(J).max(), (seed, np.abs(J - Jn).max() / np.abs(J).max())


@pytest.mark.parametrize("n", [50, 400, 3000])
def test_oracle_reaches_the_optimum_of_an_independent_optimiser(n):
    from scipy.optimize import least_squares
    p1, p2, F, q1, q2 = _scene(n, 10 + n, noise=0.5)
    F0 = _perturbed(F, n, size=2.0)
    got = o.refine_pair(F0, p1, p2, max_iters=100)
    assert got["cost"] < got["cost0"] and got["iters"] < 100          # stopped on the decrease test, not the cap
    T1, T2 = o.transform(p1), o.transform(p2)
    Fn0 = o.start(T1, T2, F0)

    def res(d):
        return o.residuals(o.to_pixels(T1, T2, o.retract(Fn0, d)), p1, p2)

    sol = least_squares(res, np.zeros(7), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    assert abs(got["cost"] - 2 * sol.cost) <= 1e-9 * got["cost"], (got["cost"], 2 * sol.cost)
    Fs = o.output(T1, T2, o.retract(Fn0, sol.x), F0)
    assert np.abs(got["F"] - Fs).max() <= 1e-6, np.abs(got["F"] - Fs).max()
    assert abs(got["cost"] - o.sampson_sq(got["F"], p1, p2).sum()) <= 1e-9 * got["cost"]


def test_oracle_recovers_a_planted_fundamental_matrix():
    for seed in range(4):
        p1, p2, F, _, _ = _scene(300, 20 + seed)
        got = o.refine_pair(_perturbed(F, seed), p1, p2, max_iters=30)
        assert got["cost"] <= 1e-15 * got["cost0"] and got["cost"] <= 1e-18, (seed, got["cost"], got["iters"])
        err = min(np.abs(got["F"] - F).max(), np.abs(got["F"] + F).max())
        assert err <= 1e-9, (seed, err)


@pytest.mark.parametrize("noise", [0.3, 0.5])
def test_oracle_moves_a_noisy_start_towards_the_planted_geometry(noise):
    before, after = [], []
    for seed in range(6):
        p1, p2, F, q1, q2 = _scene(500, 30 + seed, noise=noise)
        F0 = _perturbed(F, seed)
        got = o.refine_pair(F0, p1, p2)
        assert got["cost"] < got["cost0"]
        before.append(geometry_error(F0, q1, q2)); after.append(geometry_error(got["F"], q1, q2))
    before, after = np.array(before), np.array(after)
    # 500 rows at this noise leave a few hundredths of a pixel over the held-out points (0.013 - 0.061 px in oracle
    # runs, at most 0.067 of the start); the start (0.6 - 3.7 px) falls to that floor
    assert (after < 0.1 * before).all() and (after < 0.1).all(), (before, after)


def _host_pieces(tmp_path):
    so = os.path.join(str(tmp_path), "librefine_f_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-o", so, os.path.join(ROOT, "tests", "refine_fundamental_host.cpp")])
    return ctypes.CDLL(so)


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def test_kernel_pieces_built_for_the_host_equal_the_oracle(tmp_path):
    """csrc/refine_f.h (transforms, start point, basis, linearisation, row sums, damped 7 x 7 solve, retraction,
    output F) with g++"""
    L = _host_pieces(tmp_path)
    c = np.zeros(6)
    L.rfh_constants(_dp(c))
    assert list(c) == [o.LAMBDA0, o.LAMBDA_MIN, o.LAMBDA_MAX, o.REL_DECREASE, o.MIN_ROWS, 36]
    iu = np.triu_indices(7)
    for seed in range(4):
        p1, p2, F, _, _ = _scene(500, 40 + seed, noise=0.5)
        F0 = _perturbed(F, seed) * (-1) ** seed                       # both signs
        if seed >= 2:
            F0 = F0 + 1e-3 * np.abs(F0).max() * np.random.default_rng(seed).normal(size=(3, 3))   # full rank
        F0 = np.ascontiguousarray(F0.ravel())
        T, Fn, Fl, dF, sums = (np.zeros(k) for k in (6, 9, 9, 63, 36))
        assert L.rfh_pass(_dp(F0), _dp(p1), _dp(p2), len(p1), _dp(T), _dp(Fn), _dp(Fl), _dp(dF), _dp(sums)) == 1
        T1, T2 = o.transform(p1), o.transform(p2)
        assert np.abs(T - np.r_[T1, T2]).max() <= 1e-12 * np.abs(T).max()
        Fno = o.start(T1, T2, F0)
        assert np.abs(Fn - Fno).max() <= 1e-12
        r2 = F0.copy()
        L.rfh_rank2(_dp(r2))
        assert np.abs(r2 - o.rank2(F0)).max() <= 1e-14 * np.abs(F0).max()
        B = np.zeros(63)
        L.rfh_basis(_dp(Fn), _dp(B))
        assert np.abs(B.reshape(7, 9).T - o.basis(Fn)).max() <= 1e-12
        Fo, dFo = o.linearise(T1, T2, Fno)
        assert np.abs(Fl - Fo).max() <= 1e-12 * np.abs(Fo).max()
        assert np.abs(dF - dFo.ravel()).max() <= 1e-12 * np.abs(dFo).max()
        C, JJ, Jr = o.normal_equations(T1, T2, Fno, p1, p2)
        assert abs(sums[0] - C) <= 1e-12 * C
        assert np.abs(sums[1:29] - JJ[iu]).max() <= 1e-11 * np.abs(JJ).max()
        assert np.abs(sums[29:] - Jr).max() <= 1e-11 * np.abs(Jr).max() + 1e-9 * np.sqrt(np.diag(JJ).max() * C)
        for lam in (1e-3, 1.0, 1e6):
            D, Do = np.zeros(7), o.solve_damped(JJ, Jr, lam)
            assert L.rfh_solve(_dp(np.ascontiguousarray(JJ[iu])), _dp(Jr), ctypes.c_double(lam), _dp(D)) == 1
            assert np.abs(D - Do).max() <= 1e-10 * np.abs(Do).max()
        Fn2 = np.zeros(9)
        L.rfh_retract(_dp(Fn), _dp(Do), _dp(Fn2))
        assert np.abs(Fn2 - o.retract(Fn, Do)).max() <= 1e-14
        Fout = np.zeros(9)
        L.rfh_output(_dp(T), _dp(Fn2), _dp(F0), _dp(Fout))
        want = o.output(T1, T2, o.retract(Fn, Do), F0)
        assert np.abs(Fout - want.ravel()).max() <= 1e-12 and Fout @ F0 >= 0
    # no model: all zero, a NaN, an infinity
    for bad in (np.zeros(9), np.r_[np.ones(8), np.nan], np.r_[np.ones(8), np.inf]):
        assert not o.has_model(bad)
        assert L.rfh_pass(_dp(bad), _dp(p1), _dp(p2), 10, *(_dp(np.zeros(k)) for k in (6, 9, 9, 63, 36))) == 0
    # a matrix that is not positive definite is refused, as the oracle refuses it
    bad = np.diag([1.0, 1.0, 1.0, 0.0, 1.0, 1.0, 1.0])
    assert o.solve_damped(bad, np.ones(7), 1e-3) is None
    assert L.rfh_solve(_dp(np.ascontiguousarray(bad[iu])), _dp(np.ones(7)), ctypes.c_double(1e-3), _dp(np.zeros(7))) == 0


def test_refine_entry_point_rejects_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["F", "x1y1", "x2y2", "offsets", "mask", "F_out", "cost0", "cost", "n_used", "iters", "inliers"]
    optional = ("mask", "cost0", "n_used", "iters", "inliers")

    def call(n_pairs=3, rows=10, dim=2, max_iters=10, px_th=1.0, **null):
        b = {k: (None if null.get(k) else fake) for k in names}
        return L.dgb200_refine_fundamental_ragged_dev(b["F"], b["x1y1"], b["x2y2"], b["offsets"], n_pairs, rows, dim,
                                                      b["mask"], max_iters, ctypes.c_double(px_th), b["F_out"],
                                                      b["cost0"], b["cost"], b["n_used"], b["iters"], b["inliers"], None)

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
    from pydegensac_b200.matching import refine_fundamental_ragged as rfr
    f64 = torch.float64
    F = torch.eye(3, dtype=f64).repeat(2, 1, 1)
    p = torch.zeros((10, 2), dtype=f64)
    off = torch.tensor([0, 4, 10], dtype=torch.int32)
    bad = [
        dict(F=torch.zeros((2, 8))), dict(F=torch.zeros((0, 9))), dict(F=torch.zeros(9)), dict(F=np.zeros((2, 9))),
        dict(F=torch.zeros((2, 9), dtype=torch.int64)), dict(F=torch.zeros((2, 3, 4), dtype=f64)),
        dict(pts1=torch.zeros(10, 1, dtype=f64)), dict(pts2=torch.zeros((9, 2), dtype=f64)),
        dict(pts1=torch.zeros(10, dtype=f64)), dict(pts1=torch.zeros((10, 2), dtype=torch.int64)),
        dict(offsets=torch.tensor([0, 10], dtype=torch.int32)), dict(offsets=torch.tensor([0, 4, 10])),
        dict(offsets=torch.tensor([[0, 4, 10]], dtype=torch.int32)),
        dict(mask=torch.ones(9, dtype=torch.bool)), dict(mask=torch.ones(10, dtype=torch.int32)),
        dict(mask=np.ones(10, bool)),
        dict(max_iters=-1), dict(px_th=-0.5), dict(px_th=float("nan")),
        dict(),                                    # well-formed, but on the host
    ]
    for kw in bad:
        args = dict(F=F, pts1=p, pts2=p, offsets=off, mask=None)
        args.update(kw)
        with pytest.raises(ValueError):
            rfr(**args)
    with pytest.raises(ValueError, match="^F must be"):
        rfr(torch.zeros((2, 8)), p, p, off)
    if torch.cuda.is_available():
        dev = torch.device("cuda:0")
        with pytest.raises(ValueError, match="device"):
            rfr(F, p.to(dev), p.to(dev), off)


# ------------------------------------------------------------------------------------------------ GPU
LENGTHS = [0, 1, 7, 8, 33, 400, 2048, 3000, 9000]
N_FEW = 3                                          # the pairs of 0, 1 and 7 rows: fewer than 8, not refined


def _batch(lengths, seed, noise=0.5, size=1.0):
    """a ragged batch of noisy planted scenes (pair p: seed + p) and, as the start, each planted F perturbed:
    p1, p2, F0 [P,3,3], offsets, planted F [P,3,3], held-out views (q1, q2) per pair"""
    ps1, ps2, F0s, Fs, hold = [], [], [], [], []
    for i, n in enumerate(lengths):
        p1, p2, F, q1, q2 = _scene(max(n, 8), seed + i, noise=noise)
        ps1.append(p1[:n]); ps2.append(p2[:n]); F0s.append(_perturbed(F, seed + i, size)); Fs.append(F)
        hold.append((q1, q2))
    off = np.r_[0, np.cumsum(lengths)].astype(np.int32)
    return np.concatenate(ps1), np.concatenate(ps2), np.stack(F0s), off, np.stack(Fs), hold


def _holes(rows, seed):
    mask = np.random.default_rng(seed).random(rows) < 0.8
    mask[::7] = False
    return mask


def _dev(*xs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0") for x in xs]


def _np(res):
    return {k: v.cpu().numpy() for k, v in res._asdict().items() if v is not None}


def _check_outputs(g, F0):
    """what every refined pair satisfies: unit norm, <F_out, F_in> >= 0, rank 2, cost <= cost0"""
    for p in range(len(F0)):
        Fq = g["F"][p]
        sv = np.linalg.svd(Fq, compute_uv=False)
        assert abs(np.linalg.norm(Fq) - 1) <= 1e-12 and (Fq * F0[p]).sum() >= 0 and sv[2] <= 1e-12 * sv[0], p
        assert g["cost"][p] <= g["cost0"][p], p


@pytest.mark.gpu
@pytest.mark.parametrize("masked", [False, True])
def test_refined_batch_against_oracle(masked):
    from pydegensac_b200.matching import refine_fundamental_ragged
    p1, p2, F0, off, Fp, hold = _batch(LENGTHS, 100)
    mask = None
    if masked:
        mask = _holes(len(p1), 1)
        mask[off[3]:off[4]] = True                   # the 8-row pair keeps its 8 rows: the fewest that are refined
    P = len(LENGTHS)
    d1, d2, dF = _dev(p1, p2, F0)
    doff, = _dev(off)
    dm = _dev(mask)[0] if masked else None
    # one trial step: the arithmetic of a step, to rounding
    g1 = _np(refine_fundamental_ragged(dF, d1, d2, doff, dm, max_iters=1))
    w1 = o.refine_ragged(F0, p1, p2, off, mask, max_iters=1)
    assert np.array_equal(g1["iters"], w1["iters"]) and np.array_equal(g1["iters"], [0] * N_FEW + [1] * (P - N_FEW))
    print("largest |F - F_oracle| after one trial step: %.3e" % np.abs(g1["F"] - w1["F"]).max())
    assert np.abs(g1["F"] - w1["F"]).max() <= 1e-11
    for k in ("cost0", "cost"):
        assert np.all(np.abs(g1[k] - w1[k]) <= 1e-9 * np.abs(w1[k])), k
    assert (g1["cost"][N_FEW:] < g1["cost0"][N_FEW:]).all()
    # the whole refinement
    g = _np(refine_fundamental_ragged(dF, d1, d2, doff, dm, max_iters=10))
    w = o.refine_ragged(F0, p1, p2, off, mask, max_iters=10)
    assert np.array_equal(g["n_used"], w["n_used"])
    assert (g["n_used"][:N_FEW] < 8).all() and (g["iters"][:N_FEW] == 0).all() and (g["iters"][N_FEW:] > 0).all()
    print("trial steps per pair:", list(g["iters"]), " oracle:", list(w["iters"]))
    assert np.array_equal(g["iters"], w["iters"])
    print("largest |F - F_oracle| after ten trial steps: %.3e" % np.abs(g["F"] - w["F"]).max())
    assert np.abs(g["F"] - w["F"]).max() <= 1e-10
    for k in ("cost0", "cost"):
        assert np.all(np.abs(g[k] - w[k]) <= 1e-9 * np.abs(w[k])), k
    _check_outputs(g, F0)
    for p in range(N_FEW):                           # not refined: the start point, mapped back to pixels
        assert np.abs(g["F"][p] - w["F"][p]).max() <= 1e-14 and g["cost"][p] == g["cost0"][p]
    # pairs of 400 rows and more are well determined: the refinement moves them towards the planted geometry
    for p in range(5, P):
        q1, q2 = hold[p]
        assert geometry_error(g["F"][p], q1, q2) < 0.5 * geometry_error(F0[p], q1, q2), p


@pytest.mark.gpu
def test_batch_independence_determinism_and_in_place():
    import torch
    from pydegensac_b200 import _cabi
    from pydegensac_b200.matching import refine_fundamental_ragged
    p1, p2, F0, off, _, _ = _batch(LENGTHS, 200)
    mask = _holes(len(p1), 2)
    d1, d2, dF, doff, dm = _dev(p1, p2, F0, off, mask)
    g = _np(refine_fundamental_ragged(dF, d1, d2, doff, dm, px_th=1.0))
    again = _np(refine_fundamental_ragged(dF, d1, d2, doff, dm, px_th=1.0))
    assert all(g[k].tobytes() == again[k].tobytes() for k in g)
    for p in range(len(LENGTHS)):
        a, b = int(off[p]), int(off[p + 1])
        one = _np(refine_fundamental_ragged(dF[p:p + 1], d1[a:b], d2[a:b],
                                            torch.tensor([0, b - a], dtype=torch.int32, device="cuda:0"), dm[a:b],
                                            px_th=1.0))
        for k in ("F", "cost0", "cost", "n_used", "iters"):
            assert one[k][0].tobytes() == g[k][p].tobytes(), (p, k)
        assert np.array_equal(one["inliers"], g["inliers"][a:b]), p
    # mask=None means every row
    ones = torch.ones(len(p1), dtype=torch.bool, device="cuda:0")
    every, none = (_np(refine_fundamental_ragged(dF, d1, d2, doff, m, px_th=1.0)) for m in (ones, None))
    assert all(every[k].tobytes() == none[k].tobytes() for k in every)
    # in place through the C entry point: F_out = F
    Fi = dF.clone()
    P, rows = len(LENGTHS), len(p1)
    cost = torch.empty(P, dtype=torch.float64, device="cuda:0")
    vp = ctypes.c_void_p
    rc = _cabi.lib().dgb200_refine_fundamental_ragged_dev(
        vp(Fi.data_ptr()), vp(d1.data_ptr()), vp(d2.data_ptr()), vp(doff.data_ptr()), P, rows, 2,
        vp(dm.view(torch.uint8).data_ptr()), 10, ctypes.c_double(0.0), vp(Fi.data_ptr()), None, vp(cost.data_ptr()),
        None, None, None, vp(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    assert Fi.cpu().numpy().tobytes() == g["F"].tobytes() and cost.cpu().numpy().tobytes() == g["cost"].tobytes()


@pytest.mark.gpu
def test_inlier_rows_are_the_sampson_rule_of_the_refined_F():
    from pydegensac_b200.matching import refine_fundamental_ragged
    lengths = [300, 0, 2500, 40]
    p1, p2, F0, off, _, _ = _batch(lengths, 300, noise=1.0)
    rng = np.random.default_rng(3)
    out = rng.random(len(p1)) < 0.3                  # outliers 0 to 4 px off, masked out of the fit
    p2[out] += rng.uniform(-4, 4, (int(out.sum()), 2))
    d1, d2, dF, doff, dm = _dev(p1, p2, F0, off, ~out)
    th = 1.5
    g = _np(refine_fundamental_ragged(dF, d1, d2, doff, dm, px_th=th))
    assert g["inliers"].dtype == np.bool_ and g["inliers"].shape == (len(p1),)
    for p in range(len(lengths)):
        a, b = off[p], off[p + 1]
        r2 = o.sampson_sq(g["F"][p], p1[a:b], p2[a:b])
        clear = np.abs(r2 - th * th) >= 1e-9 * th * th
        assert np.array_equal(g["inliers"][a:b][clear], (r2 <= th * th)[clear]), p
    # written for the rows outside the mask too: some outliers fall inside the band, most inliers of the fit are inliers
    assert g["inliers"][out].any() and not g["inliers"][out].all()
    assert g["inliers"][~out].mean() > 0.5
    assert refine_fundamental_ragged(dF, d1, d2, doff, dm).inliers is None


@pytest.mark.gpu
def test_pairs_that_are_not_refined_and_malformed_offsets():
    import torch
    from pydegensac_b200 import _cabi
    from pydegensac_b200.matching import refine_fundamental_ragged
    lengths = [300, 200, 150, 250, 0, 120, 180]
    p1, p2, F0, off, _, _ = _batch(lengths, 400)
    F0[1] = 0.0
    F0[2, 1, 2] = np.nan
    F0[6, 0, 0] = np.inf
    mask = np.ones(len(p1), bool)
    mask[off[3] + 7:off[4]] = False                  # pair 3: seven rows used
    d1, d2, dF, doff, dm = _dev(p1, p2, F0, off, mask)
    g = _np(refine_fundamental_ragged(dF, d1, d2, doff, dm, px_th=1.0))
    for p in (1, 2, 6):                              # no model
        a, b = off[p], off[p + 1]
        assert not g["F"][p].any(), p
        assert np.isnan(g["cost0"][p]) and np.isnan(g["cost"][p]) and g["n_used"][p] == 0 and g["iters"][p] == 0
        assert not g["inliers"][a:b].any()
    for p in (3, 4):                                 # fewer than 8 rows used: the start point passes through
        a, b = off[p], off[p + 1]
        m = mask[a:b]
        want = o.refine_pair(F0[p], p1[a:b][m], p2[a:b][m])
        assert np.abs(g["F"][p] - want["F"]).max() <= 1e-14 and g["iters"][p] == 0
        assert g["n_used"][p] == min(7, b - a) and g["cost0"][p] == g["cost"][p]
        assert abs(g["cost"][p] - want["cost"]) <= 1e-9 * max(want["cost"], 1e-300)
    assert g["iters"][0] > 0 and g["iters"][5] > 0 and g["cost"][0] < g["cost0"][0]
    # max_iters = 0: every pair passes through, cost0 = cost
    z = _np(refine_fundamental_ragged(dF, d1, d2, doff, dm, max_iters=0))
    for p in (0, 5):
        assert np.abs(z["F"][p] - F0[p] / np.linalg.norm(F0[p])).max() <= 1e-12 and z["iters"][p] == 0
        assert z["cost0"][p] == z["cost"][p] == g["cost0"][p]
    # malformed device offsets: negative, decreasing or past the rows make empty pairs whose rows stay untouched
    rows_n = len(p1)
    bad_off, = _dev(np.array([0, 300, -5, 300 + 200 + 150, rows_n + 10], dtype=np.int32))
    P = 4
    f64 = torch.float64
    out = dict(F=torch.full((P, 9), 7.0, dtype=f64, device="cuda:0"),
               cost0=torch.full((P,), 7.0, dtype=f64, device="cuda:0"),
               cost=torch.full((P,), 7.0, dtype=f64, device="cuda:0"),
               n_used=torch.full((P,), 7, dtype=torch.int32, device="cuda:0"),
               iters=torch.full((P,), 7, dtype=torch.int32, device="cuda:0"),
               inliers=torch.full((rows_n,), 7, dtype=torch.uint8, device="cuda:0"))
    Fb = dF[[0, 5, 5, 5]].contiguous()
    vp = ctypes.c_void_p
    rc = _cabi.lib().dgb200_refine_fundamental_ragged_dev(
        vp(Fb.data_ptr()), vp(d1.data_ptr()), vp(d2.data_ptr()), vp(bad_off.data_ptr()), P, rows_n, 2,
        vp(dm.view(torch.uint8).data_ptr()), 10, ctypes.c_double(1.0),
        *[vp(out[k].data_ptr()) for k in ("F", "cost0", "cost", "n_used", "iters", "inliers")],
        vp(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    q = {k: v.cpu().numpy() for k, v in out.items()}
    assert q["F"][0].tobytes() == g["F"][0].tobytes() and q["cost"][0] == g["cost"][0] and q["iters"][0] == g["iters"][0]
    assert not q["F"][1:].any()
    assert np.isnan(q["cost0"][1:]).all() and np.isnan(q["cost"][1:]).all()
    assert not q["n_used"][1:].any() and not q["iters"][1:].any()
    assert np.array_equal(q["inliers"][:300], g["inliers"][:300].view(np.uint8)) and (q["inliers"][300:] == 7).all()
    # rows = 0: every pair is empty, its start point passes through with zero cost
    empty = torch.zeros((0, 2), dtype=f64, device="cuda:0")
    e = _np(refine_fundamental_ragged(dF[[0, 5]], empty, empty, torch.zeros(3, dtype=torch.int32, device="cuda:0"),
                                      px_th=1.0))
    assert e["inliers"].shape == (0,) and (e["n_used"] == 0).all() and (e["iters"] == 0).all()
    assert (e["cost0"] == 0).all() and (e["cost"] == 0).all()
    for i, p in enumerate((0, 5)):
        assert np.abs(e["F"][i] - F0[p] / np.linalg.norm(F0[p])).max() <= 1e-12


@pytest.mark.gpu
def test_dominant_plane_scene_stays_finite_and_never_raises_the_cost():
    """F of a planar scene is undetermined in a family of directions: J^T J is near singular there, the steps must not
    produce NaN or a higher cost"""
    from pydegensac_b200.matching import refine_fundamental_ragged
    ps1, ps2, F0s, lengths = [], [], [], [600, 2000, 150]
    for i, n in enumerate(lengths):
        p1, p2, F, _, _ = _scene(n, 500 + i, noise=0.3, plane=True)
        k = n // 20                                  # 5 % of the rows off the plane
        p1b, p2b, _, _, _ = _scene(k, 500 + i, noise=0.3)
        ps1.append(np.r_[p1, p1b]); ps2.append(np.r_[p2, p2b]); F0s.append(_perturbed(F, i))
    off = np.r_[0, np.cumsum([len(p) for p in ps1])].astype(np.int32)
    d1, d2, dF, doff = _dev(np.concatenate(ps1), np.concatenate(ps2), np.stack(F0s), off)
    g = _np(refine_fundamental_ragged(dF, d1, d2, doff, px_th=1.0))
    assert all(np.isfinite(g[k]).all() for k in ("F", "cost0", "cost"))
    assert (g["iters"] > 0).all()
    _check_outputs(g, np.stack(F0s))


def _multiview_two_cameras(n_img, n_pts, n_clutter, n_hold, D, seed):
    """tests.test_pose_ragged._multiview_pose with two cameras: even views by _K, odd views by K2.  Besides the
    keypoints and descriptors, per view the planted (R, t), its K and the noise-free views of n_hold further points."""
    rng = np.random.default_rng(seed)
    m = n_pts + n_hold
    X = np.c_[rng.uniform(-4, 4, m), rng.uniform(-4, 4, m), rng.uniform(2, 12, m)]
    code = rng.normal(size=(n_pts, D)).astype(np.float32)
    Rs, ts, Ks, kps, descs, held = [], [], [], [], [], []
    for i in range(n_img):
        R = _rot("y", 0.08 * i) @ _rot("x", 0.02 * i)
        t = np.array([0.6 * i, 0.05 * i, 0.1 * i])
        K = _K if i % 2 == 0 else K2
        x = (K @ (R @ X.T + t[:, None])).T
        x = x[:, :2] / x[:, 2:3]
        held.append(x[n_pts:])
        x = x[:n_pts] + 0.1 * rng.normal(size=(n_pts, 2))
        kp = np.r_[x, rng.uniform(0, 640, (n_clutter, 2))]
        d = np.r_[code + 0.15 * rng.normal(size=code.shape).astype(np.float32),
                  rng.normal(size=(n_clutter, D)).astype(np.float32)]
        perm = rng.permutation(n_pts + n_clutter)
        kps.append(kp[perm]); descs.append(d[perm]); Rs.append(R); ts.append(t); Ks.append(K)
    return kps, descs, Rs, ts, Ks, held


def _angle(u, v):
    return float(np.arctan2(np.linalg.norm(np.cross(u, v)), u @ v))


@pytest.mark.gpu
def test_pipeline_match_ransac_refine_guided_match_and_pose_without_sync():
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import (match_descriptors_batch, match_descriptors_guided,
                                          pose_from_fundamental_ragged, refine_fundamental_ragged)
    dev = torch.device("cuda:0")
    kps, descs, Rs, ts, Ks, held = _multiview_two_cameras(4, 800, 400, 300, 64, 5)
    pairs = np.array([(i, j) for i in range(4) for j in range(4) if i != j], dtype=np.int32)
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    seeds = torch.arange(len(pairs), dtype=torch.int64, device=dev) + 100
    K1 = torch.from_numpy(np.stack([Ks[i] for i, _ in pairs])).to(dev)
    K2p = torch.from_numpy(np.stack([Ks[j] for _, j in pairs])).to(dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m = match_descriptors_batch(dt, pairs, kt, ratio=0.9, mutual=True)
        F, mask = pdg.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                                 n_max=m.n_max)
        fine = refine_fundamental_ragged(F, m.pts1, m.pts2, m.offsets, mask, px_th=0.5)
        g = match_descriptors_guided(dt, pairs, kt, fine.F, 0.5, guide="F")
        pose0 = pose_from_fundamental_ragged(F, K1, K2p, m.pts1, m.pts2, m.offsets, mask)
        pose1 = pose_from_fundamental_ragged(fine.F, K1, K2p, m.pts1, m.pts2, m.offsets, fine.inliers)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    f, Fr = _np(fine), F.cpu().numpy().reshape(-1, 3, 3)
    off, mk = m.offsets.cpu().numpy(), mask.cpu().numpy()
    assert (f["cost"] <= f["cost0"]).all() and (f["iters"] > 0).all()
    for p in range(len(pairs)):
        assert f["n_used"][p] == mk[off[p]:off[p + 1]].sum()
    _check_outputs(f, Fr)
    # with max_iters = 0 the RANSAC's F comes back at unit norm
    z = _np(refine_fundamental_ragged(F, m.pts1, m.pts2, m.offsets, mask, max_iters=0))
    assert np.abs(z["F"] - Fr / np.linalg.norm(Fr, axis=(1, 2))[:, None, None]).max() <= 1e-12
    err = {"F": ([], []), "R": ([], []), "t": ([], [])}
    for p, (i, j) in enumerate(pairs):
        R = Rs[j] @ Rs[i].T
        t = ts[j] - R @ ts[i]
        for k, (Fq, pose) in enumerate(((Fr[p], pose0), (f["F"][p], pose1))):
            err["F"][k].append(geometry_error(Fq, held[i], held[j]))
            err["R"][k].append(float(np.arccos(np.clip((np.trace(pose.R[p].cpu().numpy() @ R.T) - 1) / 2, -1, 1))))
            err["t"][k].append(_angle(pose.t[p].cpu().numpy(), t / np.linalg.norm(t)))
    med = {}
    for name, (before, after) in err.items():
        before, after = np.array(before), np.array(after)
        med[name] = (np.median(before), np.median(after))
        print("%s error (%s): median %.4e -> %.4e (%.2fx), worst %.4e -> %.4e"
              % (name, "px, held-out Sampson distance" if name == "F" else "rad", np.median(before), np.median(after),
                 np.median(before) / np.median(after), before.max(), after.max()))
    assert med["F"][1] < med["F"][0]
    # the pose error of a pair is the larger of its rotation and translation-direction errors
    pe0 = np.maximum(err["R"][0], err["t"][0])
    pe1 = np.maximum(err["R"][1], err["t"][1])
    print("pose error (rad): median %.4e -> %.4e" % (np.median(pe0), np.median(pe1)))
    assert np.median(pe1) <= np.median(pe0)
    # the refined F guides the re-match: its band keeps the matches of the first pass
    goff = g.offsets.cpu().numpy()
    assert (np.diff(goff) >= np.diff(off) // 2).all()
