"""Refinement of homographies on their inliers (matching.refine_homography_ragged, dgb200_refine_homography_ragged_dev):
Levenberg-Marquardt on the engine's Sampson error over ragged batches.  The numpy oracle tests/refine_homography_np.py is
pinned to central differences, to the engine's Sampson formula, to scipy.optimize.least_squares and to planted planar
scenes; the kernel is pinned to the oracle."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from pydegensac_b200.scenes import _K
from tests import refine_homography_np as o
from tests.test_pose_homography import K2_OTHER, _plane_scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")
GRID = np.stack(np.meshgrid(np.linspace(0, 640, 9), np.linspace(0, 480, 7)), -1).reshape(-1, 2)


def _scene(n, seed, noise=0.0):
    """n points of a planted plane seen by two cameras, pixel noise in image 1: p1, p2 and the planted H (x2 ~ H x1)"""
    p1, p2, _, _, _, _, H = _plane_scene(n, seed, noise=noise, K2=K2_OTHER)
    return p1, p2, H


def _perturbed(H, seed, size=1.0):
    """H moved by a few pixels over the image (size 1: about 1-3 px): A H with A near the identity"""
    rng = np.random.default_rng(seed)
    e = size * rng.uniform(-1, 1, 6)
    A = np.array([[1 + 5e-3 * e[0], 5e-3 * e[1], 2.0 * e[2]], [5e-3 * e[3], 1 - 5e-3 * e[0], 2.0 * e[4]],
                  [1e-5 * e[5], -1e-5 * e[5], 1.0]])
    return A @ H


def transfer_error(H, Hp, pts=GRID):
    """mean distance between the transfers of pts by H and by Hp (px)"""
    h = np.c_[pts, np.ones(len(pts))]
    a, b = h @ np.asarray(H).reshape(3, 3).T, h @ np.asarray(Hp).reshape(3, 3).T
    return float(np.linalg.norm(a[:, :2] / a[:, 2:] - b[:, :2] / b[:, 2:], axis=1).mean())


# ------------------------------------------------------------------------------------------------ CPU
def test_oracle_jacobian_against_central_differences_and_the_engine_formula():
    for seed in range(6):
        p1, p2, H = _scene(40, seed, noise=0.5)
        g0 = o.engine_model(_perturbed(H, seed))
        T1, T2 = o.transform(p1), o.transform(p2)
        M = o.from_pixels(T1, T2, g0)
        assert np.abs(o.basis(M).T @ o.basis(M) - np.eye(8)).max() <= 1e-15 and np.abs(M @ o.basis(M)).max() <= 1e-15
        G, dG = o.linearise(T1, T2, M)
        z, J = o.jacobian(G, dG, p1, p2)
        r2 = o.sampson_sq(G, p1, p2)
        zz = (o.whitened(G, p1, p2) ** 2).sum(1)
        assert np.abs(zz - r2).max() <= 1e-12 * r2.max() and np.abs(z[:40] ** 2 + z[40:] ** 2 - r2).max() <= 1e-12 * r2.max()
        h = 1e-6
        Jn = np.empty_like(J)
        for k in range(8):
            D = np.zeros(8); D[k] = h
            za = o.whitened(o.to_pixels(T1, T2, o.step(M, D)), p1, p2)
            zb = o.whitened(o.to_pixels(T1, T2, o.step(M, -D)), p1, p2)
            Jn[:, k] = np.r_[za[:, 0] - zb[:, 0], za[:, 1] - zb[:, 1]] / (2 * h)
        assert np.abs(J - Jn).max() <= 1e-6 * np.abs(J).max(), (seed, np.abs(J - Jn).max() / np.abs(J).max())


@pytest.mark.parametrize("n", [50, 400, 3000])
def test_oracle_reaches_the_optimum_of_an_independent_optimiser(n):
    from scipy.optimize import least_squares
    p1, p2, H = _scene(n, 10 + n, noise=0.5)
    H0 = _perturbed(H, n)
    got = o.refine_pair(H0, p1, p2, max_iters=100)
    assert got["cost"] < got["cost0"] and got["iters"] < 100          # stopped on the decrease test, not the cap
    T1, T2 = o.transform(p1), o.transform(p2)
    M0 = o.from_pixels(T1, T2, o.engine_model(H0))

    def res(d):
        return o.whitened(o.to_pixels(T1, T2, o.step(M0, d)), p1, p2).ravel()

    sol = least_squares(res, np.zeros(8), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    assert abs(got["cost"] - 2 * sol.cost) <= 1e-9 * got["cost"], (got["cost"], 2 * sol.cost)
    Hs = o.public_model(o.to_pixels(T1, T2, o.step(M0, sol.x)))
    assert transfer_error(got["H"], Hs) <= 1e-6, transfer_error(got["H"], Hs)
    assert abs(got["cost"] - o.sampson_sq(got["g"], p1, p2).sum()) <= 1e-9 * got["cost"]


def test_oracle_recovers_a_planted_homography():
    for seed in range(4):
        p1, p2, H = _scene(300, 20 + seed)
        got = o.refine_pair(_perturbed(H, seed), p1, p2, max_iters=30)
        assert got["cost"] <= 1e-15 * got["cost0"] and got["cost"] <= 1e-18, (seed, got["cost"], got["iters"])
        assert np.abs(got["H"] - o.norm_model(H)).max() <= 1e-9, (seed, np.abs(got["H"] - o.norm_model(H)).max())


@pytest.mark.parametrize("noise", [0.3, 0.5])
def test_oracle_moves_a_noisy_start_towards_the_planted_homography(noise):
    before, after = [], []
    for seed in range(6):
        p1, p2, H = _scene(500, 30 + seed, noise=noise)
        H0 = _perturbed(H, seed)
        got = o.refine_pair(H0, p1, p2)
        assert got["cost"] < got["cost0"]
        before.append(transfer_error(H0, H)); after.append(transfer_error(got["H"], H))
    before, after = np.array(before), np.array(after)
    # 500 rows at this noise leave about 0.1 px of error over the image: the start (1.5 - 3.5 px) falls to that floor
    assert (after < 0.1 * before).all(), (before, after)


def _host_pieces(tmp_path):
    so = os.path.join(str(tmp_path), "librefine_h_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-o", so, os.path.join(ROOT, "tests", "refine_homography_host.cpp")])
    return ctypes.CDLL(so)


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def test_kernel_pieces_built_for_the_host_equal_the_oracle(tmp_path):
    """csrc/refine_h.h (transforms, basis, linearisation, row sums, damped 8 x 8 solve, step, output H) with g++"""
    L = _host_pieces(tmp_path)
    c = np.zeros(6)
    L.rhh_constants(_dp(c))
    assert list(c) == [o.LAMBDA0, o.LAMBDA_MIN, o.LAMBDA_MAX, o.REL_DECREASE, o.MIN_ROWS, 45]
    iu = np.triu_indices(8)
    for seed in range(4):
        p1, p2, H = _scene(500, 40 + seed, noise=0.5)
        H0 = np.ascontiguousarray(_perturbed(H, seed) * (-1) ** seed)   # both signs of H
        g, T, M, G, dG, sums = (np.zeros(k) for k in (9, 6, 9, 9, 72, 45))
        assert L.rhh_pass(_dp(H0), _dp(p1), _dp(p2), len(p1), _dp(g), _dp(T), _dp(M), _dp(G), _dp(dG), _dp(sums)) == 1
        go = o.engine_model(H0)
        T1, T2 = o.transform(p1), o.transform(p2)
        assert np.abs(g - go).max() <= 1e-14 * np.abs(go).max()
        assert np.abs(T - np.r_[T1, T2]).max() <= 1e-12 * np.abs(T).max()
        Mo = o.from_pixels(T1, T2, go)
        assert np.abs(M - Mo).max() <= 1e-12
        Go, dGo = o.linearise(T1, T2, Mo)
        assert np.abs(G - Go).max() <= 1e-12 * np.abs(Go).max()
        assert np.abs(dG - dGo.ravel()).max() <= 1e-12 * np.abs(dGo).max()
        C, JJ, Jz = o.normal_equations(T1, T2, Mo, p1, p2)
        assert abs(sums[0] - C) <= 1e-12 * C
        assert np.abs(sums[1:37] - JJ[iu]).max() <= 1e-11 * np.abs(JJ).max()
        assert np.abs(sums[37:] - Jz).max() <= 1e-11 * np.abs(Jz).max() + 1e-9 * np.sqrt(np.diag(JJ).max() * C)
        for lam in (1e-3, 1.0, 1e6):
            D, Do = np.zeros(8), o.solve_damped(JJ, Jz, lam)
            assert L.rhh_solve(_dp(np.ascontiguousarray(JJ[iu])), _dp(Jz), ctypes.c_double(lam), _dp(D)) == 1
            assert np.abs(D - Do).max() <= 1e-10 * np.abs(Do).max()
        M2 = np.zeros(9)
        L.rhh_step(_dp(M), _dp(Do), _dp(M2))
        assert np.abs(M2 - o.step(M, Do)).max() <= 1e-15
        Ho = np.zeros(9)
        L.rhh_public(_dp(T), _dp(M2), _dp(Ho))
        want = o.public_model(o.to_pixels(T1, T2, o.step(M, Do)))
        assert np.abs(Ho - want.ravel()).max() <= 1e-12 and np.linalg.det(Ho.reshape(3, 3)) > 0
    # no model: all zero, a NaN, singular
    for bad in (np.zeros(9), np.r_[np.ones(8), np.nan], np.array([1.0, 2, 3, 2, 4, 6, 0, 1, 1])):
        assert o.engine_model(bad) is None
        assert L.rhh_pass(_dp(bad), _dp(p1), _dp(p2), 10, *(_dp(np.zeros(k)) for k in (9, 6, 9, 9, 72, 45))) == 0
    # a matrix that is not positive definite is refused, as the oracle refuses it
    bad = np.diag([1.0, 1.0, 1.0, 0.0, 1.0, 1.0, 1.0, 1.0])
    assert o.solve_damped(bad, np.ones(8), 1e-3) is None
    assert L.rhh_solve(_dp(np.ascontiguousarray(bad[iu])), _dp(np.ones(8)), ctypes.c_double(1e-3), _dp(np.zeros(8))) == 0


def test_refine_entry_point_rejects_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["H", "x1y1", "x2y2", "offsets", "mask", "H_out", "cost0", "cost", "n_used", "iters", "inliers"]
    optional = ("mask", "cost0", "n_used", "iters", "inliers")

    def call(n_pairs=3, rows=10, dim=2, max_iters=10, px_th=1.0, **null):
        b = {k: (None if null.get(k) else fake) for k in names}
        return L.dgb200_refine_homography_ragged_dev(b["H"], b["x1y1"], b["x2y2"], b["offsets"], n_pairs, rows, dim,
                                                     b["mask"], max_iters, ctypes.c_double(px_th), b["H_out"],
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
    from pydegensac_b200.matching import refine_homography_ragged as rhr
    f64 = torch.float64
    H = torch.eye(3, dtype=f64).repeat(2, 1, 1)
    p = torch.zeros((10, 2), dtype=f64)
    off = torch.tensor([0, 4, 10], dtype=torch.int32)
    bad = [
        dict(H=torch.zeros((2, 8))), dict(H=torch.zeros((0, 9))), dict(H=torch.zeros(9)), dict(H=np.zeros((2, 9))),
        dict(H=torch.zeros((2, 9), dtype=torch.int64)), dict(H=torch.zeros((2, 3, 4), dtype=f64)),
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
        args = dict(H=H, pts1=p, pts2=p, offsets=off, mask=None)
        args.update(kw)
        with pytest.raises(ValueError):
            rhr(**args)
    if torch.cuda.is_available():
        dev = torch.device("cuda:0")
        with pytest.raises(ValueError, match="device"):
            rhr(H, p.to(dev), p.to(dev), off.to(dev))


# ------------------------------------------------------------------------------------------------ GPU
LENGTHS = [0, 1, 4, 5, 33, 400, 2048, 4097, 20000]


def _batch(lengths, seed, noise=0.5, size=1.0):
    """a ragged batch of noisy planted planar scenes (pair p: seed + p) and, as the start, each planted H perturbed:
    p1, p2, H0 [P,3,3], offsets, planted H [P,3,3]"""
    ps1, ps2, H0s, Hs = [], [], [], []
    for i, n in enumerate(lengths):
        p1, p2, H = _scene(max(n, 8), seed + i, noise=noise)
        ps1.append(p1[:n]); ps2.append(p2[:n]); H0s.append(_perturbed(H, seed + i, size)); Hs.append(H)
    off = np.r_[0, np.cumsum(lengths)].astype(np.int32)
    return np.concatenate(ps1), np.concatenate(ps2), np.stack(H0s), off, np.stack(Hs)


def _holes(rows, seed):
    mask = np.random.default_rng(seed).random(rows) < 0.8
    mask[::7] = False
    return mask


def _dev(*xs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0") for x in xs]


def _np(res):
    return {k: v.cpu().numpy() for k, v in res._asdict().items() if v is not None}


@pytest.mark.gpu
@pytest.mark.parametrize("masked", [False, True])
def test_refined_batch_against_oracle(masked):
    from pydegensac_b200.matching import refine_homography_ragged
    p1, p2, H0, off, Hp = _batch(LENGTHS, 100)
    mask = None
    if masked:
        mask = _holes(len(p1), 1)
        mask[off[3]:off[4]] = True                   # the 5-row pair keeps its 5 rows: the fewest that are refined
    P = len(LENGTHS)
    d1, d2, dH = _dev(p1, p2, H0)
    doff, = _dev(off)
    dm = _dev(mask)[0] if masked else None
    # one trial step: the arithmetic of a step, to rounding
    g1 = _np(refine_homography_ragged(dH, d1, d2, doff, dm, max_iters=1))
    w1 = o.refine_ragged(H0, p1, p2, off, mask, max_iters=1)
    assert np.array_equal(g1["iters"], w1["iters"]) and np.array_equal(g1["iters"], [0, 0, 0] + [1] * (P - 3))
    assert np.abs(g1["H"] - w1["H"]).max() <= 1e-11, np.abs(g1["H"] - w1["H"]).max()
    for k in ("cost0", "cost"):
        assert np.all(np.abs(g1[k] - w1[k]) <= 1e-9 * np.abs(w1[k])), k
    assert (g1["cost"][3:] < g1["cost0"][3:]).all()
    # the whole refinement
    g = _np(refine_homography_ragged(dH, d1, d2, doff, dm, max_iters=10))
    w = o.refine_ragged(H0, p1, p2, off, mask, max_iters=10)
    assert np.array_equal(g["n_used"], w["n_used"])
    assert (g["n_used"][:3] < 5).all() and (g["iters"][:3] == 0).all() and (g["iters"][3:] > 0).all()
    differ = [p for p in range(P) if g["iters"][p] != w["iters"][p]]
    print("pairs whose trial-step count differs from the oracle's (an accept / reject tie):", differ)
    assert (np.abs(g["iters"] - w["iters"]) <= 1).all()
    print("largest |H - H_oracle| after ten trial steps: %.3e" % np.abs(g["H"] - w["H"]).max())
    for p in range(P):
        assert np.abs(g["H"][p] - w["H"][p]).max() <= 1e-7, (p, np.abs(g["H"][p] - w["H"][p]).max())
        for k in ("cost0", "cost"):
            assert abs(g[k][p] - w[k][p]) <= 1e-9 * abs(w[k][p]), (p, k, g[k][p], w[k][p])
    for p in range(P):
        Hq = g["H"][p]
        assert g["cost"][p] <= g["cost0"][p]
        assert abs(np.linalg.norm(Hq) - 1) <= 1e-12 and np.linalg.det(Hq) > 0
    for p in range(3):                               # not refined: the input H, normalised
        assert np.abs(g["H"][p] - o.norm_model(H0[p])).max() <= 1e-15 and g["cost"][p] == g["cost0"][p]
    # pairs of 400 rows and more are well determined: the refinement moves them towards the planted H
    for p in range(5, P):
        assert transfer_error(g["H"][p], Hp[p]) < 0.5 * transfer_error(H0[p], Hp[p]), p


@pytest.mark.gpu
def test_batch_independence_determinism_and_in_place():
    import torch
    from pydegensac_b200 import _cabi
    from pydegensac_b200.matching import refine_homography_ragged
    p1, p2, H0, off, _ = _batch(LENGTHS, 200)
    mask = _holes(len(p1), 2)
    d1, d2, dH, doff, dm = _dev(p1, p2, H0, off, mask)
    g = _np(refine_homography_ragged(dH, d1, d2, doff, dm, px_th=1.0))
    again = _np(refine_homography_ragged(dH, d1, d2, doff, dm, px_th=1.0))
    assert all(g[k].tobytes() == again[k].tobytes() for k in g)
    for p in range(len(LENGTHS)):
        a, b = int(off[p]), int(off[p + 1])
        one = _np(refine_homography_ragged(dH[p:p + 1], d1[a:b], d2[a:b],
                                           torch.tensor([0, b - a], dtype=torch.int32, device="cuda:0"), dm[a:b],
                                           px_th=1.0))
        for k in ("H", "cost0", "cost", "n_used", "iters"):
            assert one[k][0].tobytes() == g[k][p].tobytes(), (p, k)
        assert np.array_equal(one["inliers"], g["inliers"][a:b]), p
    # in place through the C entry point: H_out = H
    Hi = dH.clone()
    P, rows = len(LENGTHS), len(p1)
    cost = torch.empty(P, dtype=torch.float64, device="cuda:0")
    vp = ctypes.c_void_p
    rc = _cabi.lib().dgb200_refine_homography_ragged_dev(
        vp(Hi.data_ptr()), vp(d1.data_ptr()), vp(d2.data_ptr()), vp(doff.data_ptr()), P, rows, 2,
        vp(dm.view(torch.uint8).data_ptr()), 10, ctypes.c_double(0.0), vp(Hi.data_ptr()), None, vp(cost.data_ptr()),
        None, None, None, vp(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    assert Hi.cpu().numpy().tobytes() == g["H"].tobytes() and cost.cpu().numpy().tobytes() == g["cost"].tobytes()


@pytest.mark.gpu
def test_inlier_rows_are_the_sampson_rule_of_the_refined_H():
    from pydegensac_b200.matching import refine_homography_ragged
    lengths = [300, 0, 2500, 40]
    p1, p2, H0, off, _ = _batch(lengths, 300, noise=1.0)
    rng = np.random.default_rng(3)
    out = rng.random(len(p1)) < 0.3                  # outliers 0 to 4 px off, masked out of the fit
    p2[out] += rng.uniform(-4, 4, (int(out.sum()), 2))
    d1, d2, dH, doff, dm = _dev(p1, p2, H0, off, ~out)
    th = 1.5
    g = _np(refine_homography_ragged(dH, d1, d2, doff, dm, px_th=th))
    assert g["inliers"].dtype == np.bool_ and g["inliers"].shape == (len(p1),)
    for p in range(len(lengths)):
        a, b = off[p], off[p + 1]
        r2 = o.sampson_sq(o.engine_model(g["H"][p]), p1[a:b], p2[a:b])
        clear = np.abs(r2 - th * th) >= 1e-9 * th * th
        assert np.array_equal(g["inliers"][a:b][clear], (r2 <= th * th)[clear]), p
    # written for the rows outside the mask too: some outliers fall inside the disc, most inliers of the fit are inliers
    assert g["inliers"][out].any() and not g["inliers"][out].all()
    assert g["inliers"][~out].mean() > 0.5
    assert refine_homography_ragged(dH, d1, d2, doff, dm).inliers is None


@pytest.mark.gpu
def test_pairs_that_are_not_refined_and_malformed_offsets():
    import torch
    from pydegensac_b200 import _cabi
    from pydegensac_b200.matching import refine_homography_ragged
    lengths = [300, 200, 150, 250, 0, 120, 180]
    p1, p2, H0, off, _ = _batch(lengths, 400)
    H0[1] = 0.0
    H0[2, 1, 2] = np.nan
    H0[6] = np.array([[1.0, 2.0, 3.0], [2.0, 4.0, 6.0], [0.0, 1.0, 1.0]])   # singular
    mask = np.ones(len(p1), bool)
    mask[off[3] + 4:off[4]] = False                  # pair 3: four rows used
    d1, d2, dH, doff, dm = _dev(p1, p2, H0, off, mask)
    g = _np(refine_homography_ragged(dH, d1, d2, doff, dm, px_th=1.0))
    for p in (1, 2, 6):                              # no model
        a, b = off[p], off[p + 1]
        assert not g["H"][p].any(), p
        assert np.isnan(g["cost0"][p]) and np.isnan(g["cost"][p]) and g["n_used"][p] == 0 and g["iters"][p] == 0
        assert not g["inliers"][a:b].any()
    for p in (3, 4):                                 # fewer than 5 rows used: H passes through
        a, b = off[p], off[p + 1]
        assert np.abs(g["H"][p] - o.norm_model(H0[p])).max() <= 1e-15 and g["iters"][p] == 0
        assert g["n_used"][p] == min(4, b - a) and g["cost0"][p] == g["cost"][p]
        m = mask[a:b]
        want = o.sampson_sq(o.engine_model(H0[p]), p1[a:b][m], p2[a:b][m]).sum()
        assert abs(g["cost"][p] - want) <= 1e-9 * max(want, 1e-300)
    assert g["iters"][0] > 0 and g["iters"][5] > 0 and g["cost"][0] < g["cost0"][0]
    # max_iters = 0: every pair passes through, cost0 = cost
    z = _np(refine_homography_ragged(dH, d1, d2, doff, dm, max_iters=0))
    for p in (0, 5):
        assert np.abs(z["H"][p] - o.norm_model(H0[p])).max() <= 1e-15 and z["iters"][p] == 0
        assert z["cost0"][p] == z["cost"][p] == g["cost0"][p]
    # malformed device offsets: negative, decreasing or past the rows make empty pairs whose rows stay untouched
    rows_n = len(p1)
    bad_off, = _dev(np.array([0, 300, -5, 300 + 200 + 150, rows_n + 10], dtype=np.int32))
    P = 4
    f64 = torch.float64
    out = dict(H=torch.full((P, 9), 7.0, dtype=f64, device="cuda:0"),
               cost0=torch.full((P,), 7.0, dtype=f64, device="cuda:0"),
               cost=torch.full((P,), 7.0, dtype=f64, device="cuda:0"),
               n_used=torch.full((P,), 7, dtype=torch.int32, device="cuda:0"),
               iters=torch.full((P,), 7, dtype=torch.int32, device="cuda:0"),
               inliers=torch.full((rows_n,), 7, dtype=torch.uint8, device="cuda:0"))
    Hb = dH[[0, 5, 5, 5]].contiguous()
    vp = ctypes.c_void_p
    rc = _cabi.lib().dgb200_refine_homography_ragged_dev(
        vp(Hb.data_ptr()), vp(d1.data_ptr()), vp(d2.data_ptr()), vp(bad_off.data_ptr()), P, rows_n, 2,
        vp(dm.view(torch.uint8).data_ptr()), 10, ctypes.c_double(1.0),
        *[vp(out[k].data_ptr()) for k in ("H", "cost0", "cost", "n_used", "iters", "inliers")],
        vp(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    q = {k: v.cpu().numpy() for k, v in out.items()}
    assert q["H"][0].tobytes() == g["H"][0].tobytes() and q["cost"][0] == g["cost"][0] and q["iters"][0] == g["iters"][0]
    assert not q["H"][1:].any()
    assert np.isnan(q["cost0"][1:]).all() and np.isnan(q["cost"][1:]).all()
    assert not q["n_used"][1:].any() and not q["iters"][1:].any()
    assert np.array_equal(q["inliers"][:300], g["inliers"][:300].view(np.uint8)) and (q["inliers"][300:] == 7).all()


def _planted_pair_H(Rs, ts, i, j):
    """x_j ~ H x_i for the plane of test_pose_homography._multiview_plane (n^T X = 7 in the world frame)"""
    from pydegensac_b200.scenes import _K as K
    nw = np.array([0.15, -0.1, 1.0]); nw /= np.linalg.norm(nw)
    A = [K @ (R + np.outer(t, nw) / 7.0) for R, t in zip(Rs, ts)]
    return A[j] @ np.linalg.inv(A[i])


@pytest.mark.gpu
def test_pipeline_match_ransac_refine_pose_and_guided_match_without_sync():
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import (match_descriptors_batch, match_descriptors_guided,
                                          pose_from_homography_ragged, refine_homography_ragged)
    from tests.test_pose_homography import _multiview_plane
    dev = torch.device("cuda:0")
    kps, descs, Rs, ts = _multiview_plane(4, 800, 400, 64, 5)
    pairs = np.array([(i, j) for i in range(4) for j in range(4) if i != j], dtype=np.int32)
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    seeds = torch.arange(len(pairs), dtype=torch.int64, device=dev) + 100
    K = torch.from_numpy(_K).to(dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m = match_descriptors_batch(dt, pairs, kt, ratio=0.9, mutual=True)
        H, mask = pdg.findHomographyBatch(m.pts1, m.pts2, 2.0, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                          n_max=m.n_max)
        fine = refine_homography_ragged(H, m.pts1, m.pts2, m.offsets, mask, px_th=2.0)
        pose = pose_from_homography_ragged(fine.H, K, K, m.pts1, m.pts2, m.offsets, fine.inliers)
        g = match_descriptors_guided(dt, pairs, kt, fine.H, 2.0, guide="H")
    finally:
        torch.cuda.set_sync_debug_mode(0)
    f, Hn = _np(fine), H.cpu().numpy()
    before, after = [], []
    for p, (i, j) in enumerate(pairs):
        Hp = _planted_pair_H(Rs, ts, i, j)
        before.append(transfer_error(Hn[p], Hp)); after.append(transfer_error(f["H"][p], Hp))
    before, after = np.array(before), np.array(after)
    print("transfer error to the planted H, px: median %.4f -> %.4f (%.2fx), worst %.4f -> %.4f"
          % (np.median(before), np.median(after), np.median(before) / np.median(after), before.max(), after.max()))
    assert (f["cost"] <= f["cost0"]).all() and (f["iters"] > 0).all()
    off = m.offsets.cpu().numpy()
    mk = mask.cpu().numpy()
    for p in range(len(pairs)):
        assert f["n_used"][p] == mk[off[p]:off[p + 1]].sum()
    assert np.median(after) < np.median(before)
    # the refined H feeds pose from H and guided matching
    hp = _np(pose)
    assert not hp["rotation_only"].any() and (hp["good"][:, 0] > 0).all()
    goff = g.offsets.cpu().numpy()
    assert (np.diff(goff) >= np.diff(off) // 2).all()
