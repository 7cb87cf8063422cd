"""matching.find_essential_ragged: five-point MSAC-RANSAC with local optimisation on ragged batches of calibrated
correspondences.  CPU: the numpy oracle (tests/essential_np.py) against cv2.findEssentialMat and planted scenes; the
host build of the kernel's pieces against the oracle; the argument checks.  GPU: the kernel against the oracle, batch
independence, edge cases and a matcher-to-refined-pose pipeline without a host synchronisation."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from pydegensac_b200.scenes import _K
from tests import essential_np as o
from tests.test_absolute_pose import _random_rotation, _rot_error

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")
K2 = _K.copy(); K2[0, 0] *= 1.1; K2[1, 1] *= 1.07; K2[0, 2] += 7.0


def _skew(t):
    return np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])


def _unit(E):
    return E / np.linalg.norm(E)


def _sign_dist(A, B):
    A, B = np.asarray(A).ravel(), np.asarray(B).ravel()
    return min(np.abs(A - B).max(), np.abs(A + B).max())


def scene(n, inlier_ratio, seed, noise=0.5, K1=_K, K2=_K, planar=False):
    """n correspondences of one calibrated pair: points 3-10 units in front of camera 1 (identity pose), camera 2 at a
    random (R, t), |t| = 1, x2 ~ K2 (R X + t); the first round(n * inlier_ratio) rows with Gaussian pixel noise, the
    rest at uniform random pixels in image 2.  planar: every point on one plane.  Returns (x1, x2, R, t, is_inlier)."""
    rng = np.random.default_rng(seed)
    R = _small_rotation(rng) if planar else _random_rotation(rng)
    t = rng.normal(size=3)
    t /= np.linalg.norm(t)
    u = np.c_[rng.uniform(0, 640, n), rng.uniform(0, 480, n)]
    ray = np.c_[u, np.ones(n)] @ np.linalg.inv(K1).T
    if planar:
        nrm = np.array([0.2, -0.1, 1.0]) + 0.2 * rng.normal(size=3)
        z = 6.0 / (ray @ nrm)
    else:
        z = rng.uniform(3.0, 10.0, n)
    X = ray * z[:, None]
    Y = X @ R.T + t
    q = Y @ K2.T
    x2 = q[:, :2] / q[:, 2:] + noise * rng.normal(size=(n, 2))
    x1 = u + noise * rng.normal(size=(n, 2))
    n_in = int(round(n * inlier_ratio))
    x2[n_in:] = np.c_[rng.uniform(0, 640, n - n_in), rng.uniform(0, 480, n - n_in)]
    return x1, x2, R, t, np.arange(n) < n_in


def _small_rotation(rng):
    w = 0.3 * rng.normal(size=3)
    a = np.linalg.norm(w)
    W = _skew(w / a)
    return np.eye(3) + np.sin(a) * W + (1 - np.cos(a)) * W @ W


def _samples(count, seed, planar):
    """five normalised correspondences of random poses, general or on one plane, and the planted E"""
    rng = np.random.default_rng(seed)
    x1s, x2s, Es = [], [], []
    for _ in range(count):
        R = _random_rotation(rng)
        t = rng.normal(size=3)
        t /= np.linalg.norm(t)
        if planar:
            xy = rng.uniform(-1, 1, (5, 2))
            P = np.c_[xy, 5.0 + xy @ rng.uniform(-0.5, 0.5, 2)]
        else:
            P = np.c_[rng.uniform(-1, 1, (5, 2)), rng.uniform(3, 8, 5)]
        Q = P @ R.T + t
        x1s.append(P / P[:, 2:]); x2s.append(Q / Q[:, 2:]); Es.append(_unit(_skew(t) @ R))
    return np.array(x1s), np.array(x2s), Es


def _constraint_residual(E):
    E = np.asarray(E).reshape(3, 3)
    return max(abs(np.linalg.det(E)), np.abs(2 * E @ E.T @ E - np.trace(E @ E.T) * E).max())


# ------------------------------------------------------------------------------------------------ oracle (CPU)
@pytest.mark.parametrize("planar", [False, True])
def test_oracle_five_point_against_cv2_findEssentialMat(planar):
    """cv2.findEssentialMat on exactly five correspondences returns every solution stacked [3k,3].  The oracle finds
    each of cv2's up to sign (and in at most 1 % of the samples a further near-double pair of real roots that cv2's
    eigenvalue solver returns as complex).  In all but 1 % of the samples every solution satisfies both constraints
    within 1e-10 and the planted E is among them within 1e-9; the rest hold a near-double root, which the Gauss-Newton
    polish approaches only linearly.  A match within 1e-8 is required for every cv2 solution that itself meets the constraints within 1e-12.  cv2
    does not polish its roots: the others (most of them on planar samples) can miss the constraints by 1e-3 where the
    oracle's meet them within 1e-10."""
    import cv2
    x1, x2, Es = _samples(600, 11 if planar else 12, planar)
    sols = o.five_point(x1, x2)
    worst = dict(planted=0.0, cv2=0.0, constraint=0.0)
    loose = extra = missed = 0
    for s in range(len(Es)):
        Ec = cv2.findEssentialMat(x1[s, :, :2].copy(), x2[s, :, :2].copy(), np.eye(3))[0].reshape(-1, 3, 3)
        assert len(sols[s]) >= len(Ec), s
        extra += len(sols[s]) > len(Ec)
        if len(sols[s]) > len(Ec):
            Ec = []                        # cv2 keeps the real part of the pair it found complex: nothing to match
        planted = min([_sign_dist(e, Es[s]) for e in sols[s]] + [np.inf])
        if planted <= 1e-9:
            worst["planted"] = max(worst["planted"], planted)
        c = max([_constraint_residual(e) for e in sols[s]] + [0.0])
        if planted > 1e-9 or c > 1e-10:
            missed += 1
        else:
            worst["constraint"] = max(worst["constraint"], c)
        for e in Ec:
            e = _unit(e)
            d = min(_sign_dist(e, f) for f in sols[s])
            if _constraint_residual(e) > 1e-12:
                loose += 1                 # cv2's own root is off: its distance says nothing
            else:
                assert d <= 1e-8 or c > 1e-10, (s, d)
                worst["cv2"] = max(worst["cv2"], d)
    print("%s: worst %s; %d of cv2's solutions off the constraints; %d samples with more real roots than cv2's; a solution off "
          "the constraints or the planted E in %d samples" % ("planar" if planar else "general", worst, loose, extra, missed))
    assert loose <= 0.5 * sum(len(s) for s in sols) and extra <= 0.01 * len(sols) and missed <= 0.01 * len(sols)


def _pair(n, w, seed, **kw):
    x1, x2, R, t, _ = scene(n, w, seed, **kw)
    return x1, x2, R, t


def _pose_errors(E, R, t):
    """rotation and translation-direction errors of the best decomposition of E against the planted (R, t)"""
    U, _, Vt = np.linalg.svd(np.asarray(E).reshape(3, 3))
    W = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    best = (np.inf, np.inf)
    for Wx in (W, W.T):
        Rc = U @ Wx @ Vt
        Rc *= np.sign(np.linalg.det(Rc))
        tc = U[:, 2]
        et = min(np.arccos(np.clip(abs(tc @ t), -1.0, 1.0)), np.pi)
        er = _rot_error(Rc, R)
        if er < best[0]:
            best = (er, et)
    return best


def test_oracle_recovers_planted_poses_and_lo_helps():
    lower = 0
    for i, (w, n) in enumerate([(0.3, 400), (0.3, 250), (0.7, 600), (0.7, 1500)]):
        x1, x2, R, t = _pair(n, w, 30 + i, K1=_K, K2=K2)
        r = o.find_essential(x1, x2, _K, K2, px_th=1.0, seed=i)
        er, et = _pose_errors(r["E"], R, t)
        assert r["n_inliers"] >= 0.8 * w * n, (w, r["n_inliers"])
        assert er <= 5e-3 and et <= 3e-2, (w, er, et)
        assert r["cost"] <= r["cost0"]
        lower += r["cost"] < r["cost0"]
        assert np.allclose(r["F"], _unit(np.linalg.inv(K2).T @ r["E"] @ np.linalg.inv(_K)), atol=1e-12) or \
            np.allclose(r["F"], -_unit(np.linalg.inv(K2).T @ r["E"] @ np.linalg.inv(_K)), atol=1e-12)
    assert lower >= 3


def test_oracle_stopping_rule_and_special_cases():
    x1, x2, _, _ = _pair(200, 0.5, 5)
    r = o.find_essential(x1, x2, _K, _K, conf=1.0, max_iters=23)
    assert r["iters"] == 23
    x1, x2, _, _ = _pair(60, 1.0, 6, noise=0.0)                      # w = 1: the first model explains every row
    r = o.find_essential(x1, x2, _K, _K, px_th=1.0)
    assert r["iters"] == 1 and r["n_inliers"] == 60
    r = o.find_essential(x1[:4], x2[:4], _K, _K)
    assert r["iters"] == 0 and r["n_inliers"] == 0 and np.isnan(r["cost0"]) and not r["E"].any()
    assert o.required_iters(False, 0, 10, 0.99, 500, 3) == 500
    assert o.required_iters(True, 10, 10, 0.99, 500, 4) == 4
    assert o.required_iters(True, 3, 10, 0.99, 10 ** 6, 1) == int(np.ceil(np.log(0.01) / np.log1p(-0.3 ** 5)))


# ------------------------------------------------------------------------------------------------ host build (CPU)
def _host(tmp_path):
    so = os.path.join(str(tmp_path), "libessential_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-o", so, os.path.join(ROOT, "tests", "essential_host.cpp")])
    return ctypes.CDLL(so)


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def test_host_build_equals_the_oracle(tmp_path):
    L = _host(tmp_path)
    # the solver: the same solutions, in the same order, to the bit (both are +, -, *, /, sqrt in one order)
    for planar in (False, True):
        x1, x2, _ = _samples(300, 40 + planar, planar)
        sols = o.five_point(x1, x2)
        for s in range(len(x1)):
            Es = np.zeros(90)
            ns = L.esh_five_point(_dp(np.ascontiguousarray(x1[s])), _dp(np.ascontiguousarray(x2[s])), _dp(Es))
            assert ns == len(sols[s]) and np.array_equal(Es[:9 * ns].reshape(ns, 9), sols[s]), s
    # degenerate samples: the same count, never a NaN; no solution from a zero constraint matrix
    x1, x2, _ = _samples(50, 3, False)
    for s in range(50):
        for a, b in ((np.r_[x1[s, :4], x1[s, :1]], np.r_[x2[s, :4], x2[s, :1]]),      # a repeated correspondence
                     (np.zeros((5, 3)), x2[s])):
            Es = np.zeros(90)
            ns = L.esh_five_point(_dp(np.ascontiguousarray(a)), _dp(np.ascontiguousarray(b)), _dp(Es))
            assert ns == len(o.five_point(a[None], b[None])[0]) and np.isfinite(Es).all()
            assert ns == 0 or a.any()
    # the per-row pieces
    x1, x2, R, t = _pair(300, 0.6, 5, K1=_K, K2=K2)
    K1i, K2i = o.inv3(_K), o.inv3(K2)
    A = K2i.T.copy()
    n = np.zeros(3)
    L.esh_normalise(_dp(K1i.ravel().copy()), ctypes.c_double(x1[7, 0]), ctypes.c_double(x1[7, 1]), _dp(n))
    assert np.array_equal(n, o.normalise(K1i, x1[7:8, 0], x1[7:8, 1])[0])
    E = _unit(_skew(t) @ R).ravel()
    F = np.zeros(9)
    L.esh_fundamental(_dp(E), _dp(A.ravel().copy()), _dp(K1i.ravel().copy()), _dp(F))
    assert np.array_equal(F, o.fundamental(E, A, K1i)) and np.array_equal(F, o.fundamentals(E[None], A, K1i)[0])
    term, inl = np.zeros(300), np.zeros(300, np.int32)
    x1[3, 0] = np.nan
    L.esh_msac(_dp(F), _dp(np.ascontiguousarray(x1)), _dp(np.ascontiguousarray(x2)), 300, ctypes.c_double(1.0),
               _dp(term), inl.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
    ot, oi = o.msac(F, x1, x2, 1.0)
    assert np.array_equal(term, ot[0]) and np.array_equal(inl.astype(bool), oi[0])
    assert term[3] == 1.0 and not inl[3]
    Rh, th = np.zeros(9), np.zeros(3)
    assert L.esh_pose(_dp(E), _dp(Rh), _dp(th)) == 1
    Ro, to = o.pose(E)
    assert np.array_equal(Rh, Ro) and np.array_equal(th, to)
    assert _sign_dist(o.essential(Ro, to), E) <= 1e-14 and abs(np.linalg.det(Ro.reshape(3, 3)) - 1.0) <= 1e-14
    Eh = np.zeros(9)
    L.esh_essential(_dp(R.ravel().copy()), _dp(t.copy()), _dp(Eh))
    assert np.array_equal(Eh, o.essential(R, t))
    assert L.esh_pose(_dp(np.zeros(9)), _dp(Rh), _dp(th)) == 0 and o.pose(np.zeros(9)) is None
    for args in ((0, 0, 10, 0.99, 500, 3), (1, 5, 10, 1.0, 500, 3), (1, 10, 10, 0.99, 500, 4), (1, 0, 10, 0.99, 500, 2),
                 (1, 7, 10, 0.999, 500, 9), (1, 300, 1000, 0.999, 10000, 9), (1, 700, 1000, 0.5, 10000, 1)):
        assert L.esh_required_iters(*args[:3], ctypes.c_double(args[3]), *args[4:]) == o.required_iters(*args)


def test_philox_sampling_of_the_oracle_equals_rng_h(tmp_path):
    L = _host(tmp_path)
    sel = np.zeros(5, np.int32)
    for seed in (0, 1, 12345, 2 ** 40 + 17, 2 ** 64 - 1):
        for n in (5, 6, 17, 1000, 99991):
            for k in (1, 2, 3, 100, 65537):
                L.esh_sample(ctypes.c_ulonglong(seed), ctypes.c_uint(k), n, sel.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
                assert list(sel) == o.minimal_sample(seed, k, n), (seed, n, k)
                assert len(set(sel)) == 5 and sel.min() >= 0 and sel.max() < n


# ------------------------------------------------------------------------------------------------ arguments (CPU)
def test_entry_point_rejects_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["x1", "x2", "K1", "K2", "offsets", "mask", "seeds", "E", "F", "mask_out", "n_inliers", "iters", "cost0",
             "cost"]

    def call(n_pairs=3, rows=10, px_th=1.0, conf=0.99, max_iters=100, refine_iters=10, **null):
        b = {k: (None if null.get(k) else fake) for k in names}
        return L.dgb200_find_essential_ragged_dev(
            b["x1"], b["x2"], b["K1"], b["K2"], 0, b["offsets"], n_pairs, rows, b["mask"], ctypes.c_double(px_th),
            ctypes.c_double(conf), max_iters, refine_iters, b["seeds"], b["E"], b["F"], b["mask_out"], b["n_inliers"],
            b["iters"], b["cost0"], b["cost"], None)

    for k in names:
        if k != "mask":
            assert call(**{k: True}) == -1, k
            assert L.dgb200_essential_last_error().decode() != ""
    for n_pairs in (0, -1):
        assert call(n_pairs=n_pairs) == -1
    assert call(rows=-1) == -1
    for px_th in (0.0, -1.0, float("nan"), float("inf")):
        assert call(px_th=px_th) == -1
        assert "px_th" in L.dgb200_essential_last_error().decode()
    for conf in (0.0, -0.5, 1.0000001, float("nan")):
        assert call(conf=conf) == -1
    assert call(max_iters=0) == -1
    assert call(refine_iters=-1) == -1


def test_python_argument_errors():
    import torch
    from pydegensac_b200.matching import find_essential_ragged as fe
    f64 = torch.float64
    p = torch.zeros((10, 2), dtype=f64)
    K = torch.eye(3, dtype=f64)
    off = torch.tensor([0, 4, 10], dtype=torch.int32)
    bad = [
        dict(pts1=np.zeros((10, 2))), dict(pts1=torch.zeros((10, 3), dtype=f64)), dict(pts1=torch.zeros(10, dtype=f64)),
        dict(pts1=torch.zeros((10, 2), dtype=torch.int64), pts2=torch.zeros((10, 2), dtype=torch.int64)),
        dict(pts2=torch.zeros((9, 2), dtype=f64)), dict(K1=torch.eye(4, dtype=f64)), dict(K2=torch.zeros((3, 3, 3))),
        dict(K1=torch.eye(3, dtype=torch.int64)), dict(offsets=torch.tensor([0, 4, 10])),
        dict(offsets=torch.tensor([0], dtype=torch.int32)), dict(offsets=torch.tensor([[0, 4, 10]], dtype=torch.int32)),
        dict(mask=torch.ones(9, dtype=torch.bool)), dict(mask=torch.ones(10, dtype=torch.int32)),
        dict(mask=np.ones(10, bool)), dict(px_th=0.0), dict(px_th=-1.0), dict(px_th=float("nan")),
        dict(conf=0.0), dict(conf=1.5), dict(max_iters=0), dict(refine_iters=-1),
        dict(),                                    # well-formed, but on the host
    ]
    for kw in bad:
        args = dict(pts1=p, pts2=p, K1=K, K2=K, offsets=off)
        args.update(kw)
        with pytest.raises(ValueError):
            fe(**args)
    with pytest.raises(ValueError, match="^pts1 and pts2 must be"):
        fe(p, torch.zeros((10, 3), dtype=f64), K, K, off)


# ------------------------------------------------------------------------------------------------ GPU
def _dev(*xs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0") for a in xs]


def _np(res):
    return {k: getattr(res, k).cpu().numpy() for k in res._fields}


def _ragged_batch(P, seed, big=True):
    """P pairs of planted scenes with per-pair K1 != K2, empty and tiny pairs, a pair of 20000 rows, mask holes and
    non-finite rows: (x1, x2, K1 [P], K2 [P], offsets, mask, seeds, planted (R, t) per pair)"""
    rng = np.random.default_rng(seed)
    x1s, x2s, K1s, K2s, ms, truth = [], [], [], [], [], []
    for p in range(P):
        if p == 3 and big:
            n, w = 20000, 0.7
        elif p % 8 == 0:
            n, w = int(rng.choice([0, 3, 4, 5, 6, 9, 30])), 0.9
        else:
            n, w = int(rng.integers(20, 1200)), float(rng.choice([0.35, 0.5, 0.7, 0.9]))
        Ka = _K.copy(); Ka[0, 0] *= 1.0 + 0.2 * rng.uniform(-1, 1)
        Kb = K2.copy() if p % 3 else _K.copy()
        Kb[1, 1] *= 1.0 + 0.1 * rng.uniform(-1, 1)
        x1, x2, R, t, _ = scene(n, w, seed * 1000 + p, noise=float(rng.uniform(0.1, 0.8)), K1=Ka, K2=Kb,
                                planar=p % 11 == 5)
        m = rng.uniform(size=n) > 0.1
        if n > 10 and p % 4 == 1:
            x1[3, 0] = np.nan
            x2[5, 1] = np.inf
        x1s.append(x1); x2s.append(x2); K1s.append(Ka); K2s.append(Kb); ms.append(m); truth.append((R, t))
    off = np.zeros(P + 1, np.int32)
    off[1:] = np.cumsum([len(a) for a in x1s])
    seeds = rng.integers(0, 2 ** 62, P).astype(np.int64)
    return (np.concatenate(x1s), np.concatenate(x2s), np.stack(K1s), np.stack(K2s), off, np.concatenate(ms), seeds,
            truth)


def _run(x1, x2, K1, K2, off, mask, seeds, **kw):
    from pydegensac_b200.matching import find_essential_ragged
    d1, d2, dK1, dK2, doff, dm, ds = _dev(x1, x2, K1, K2, off, mask, seeds)
    return _np(find_essential_ragged(d1, d2, dK1, dK2, doff, dm, seeds=ds, **kw))


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


@pytest.mark.gpu
def test_kernel_against_the_oracle():
    P = 48
    x1, x2, K1, K2_, off, mask, seeds, truth = _ragged_batch(P, 1)
    g = _run(x1, x2, K1, K2_, off, mask, seeds, px_th=1.0, conf=0.999, max_iters=5000, refine_iters=10)
    ref = o.find_essential_ragged(x1, x2, K1, K2_, off, mask, 1.0, 0.999, 5000, seeds.astype(np.uint64), 10)
    ties = 0
    worst = dict(E=0.0, F=0.0, cost0=0.0, cost=0.0)
    for p, r in enumerate(ref):
        b, e = off[p], off[p + 1]
        assert g["iters"][p] == r["iters"], p
        if r["near_tie"] or r["lo_tie"]:
            ties += 1
            continue
        assert g["n_inliers"][p] == r["n_inliers"], p
        assert np.array_equal(g["mask"][b:e], r["mask"]), p
        if r["n_inliers"] == 0 and np.isnan(r["cost0"]):
            assert np.isnan(g["cost0"][p]) and np.isnan(g["cost"][p]) and not g["E"][p].any() and not g["F"][p].any()
            continue
        for k in ("E", "F"):
            # the RANSAC model is the solver's, to rounding; after the LO, the oracle's numpy LM (inverses and products
            # of another rounding) may stop one flat step from the kernel's: 1e-7 on E and F, 1e-8 on the cost
            d = _sign_dist(g[k][p], r[k])
            worst[k] = max(worst[k], d)
            assert d <= (1e-9 if r["cost"] == r["cost0"] else 1e-7), (p, k, d)
        for k in ("cost0", "cost"):
            d = abs(g[k][p] - r[k]) / max(1.0, abs(r[k]))
            worst[k] = max(worst[k], d)
            assert d <= (1e-9 if k == "cost0" or r["cost"] == r["cost0"] else 1e-8), (p, k, d)
        assert g["cost"][p] <= g["cost0"][p]
    n_model = int((g["n_inliers"] > 0).sum())
    print("pairs %d (with a model %d), near ties %d; worst difference %s; iters mean %.1f max %d"
          % (P, n_model, ties, {k: "%.2e" % v for k, v in worst.items()}, g["iters"].mean(), g["iters"].max()))
    assert ties <= 3 and n_model >= 38


@pytest.mark.gpu
def test_same_bytes_alone_in_a_batch_permuted_and_on_a_rerun():
    x1, x2, K1, K2_, off, mask, seeds, _ = _ragged_batch(24, 2, big=False)
    full = _run(x1, x2, K1, K2_, off, mask, seeds)
    again = _run(x1, x2, K1, K2_, off, mask, seeds)
    for k in full:
        assert full[k].tobytes() == again[k].tobytes(), k
    perm = np.random.default_rng(0).permutation(24)
    p1, p2, pm, poff = [], [], [], [0]
    for p in perm:
        b, e = off[p], off[p + 1]
        p1.append(x1[b:e]); p2.append(x2[b:e]); pm.append(mask[b:e]); poff.append(poff[-1] + e - b)
    pres = _run(np.concatenate(p1), np.concatenate(p2), K1[perm], K2_[perm], np.array(poff, np.int32),
                np.concatenate(pm), seeds[perm])
    for i, p in enumerate(perm):
        for k in ("E", "F", "n_inliers", "iters", "cost0", "cost"):
            assert full[k][p].tobytes() == pres[k][i].tobytes(), (k, p)
        assert full["mask"][off[p]:off[p + 1]].tobytes() == pres["mask"][poff[i]:poff[i + 1]].tobytes()
    for p in (1, 9, 17):
        b, e = off[p], off[p + 1]
        alone = _run(x1[b:e], x2[b:e], K1[p:p + 1], K2_[p:p + 1], np.array([0, e - b], np.int32), mask[b:e],
                     seeds[p:p + 1])
        for k in ("E", "F", "n_inliers", "iters", "cost0", "cost"):
            assert full[k][p].tobytes() == alone[k][0].tobytes(), (k, p)
        assert full["mask"][b:e].tobytes() == alone["mask"].tobytes()


@pytest.mark.gpu
def test_edge_cases():
    import torch
    from pydegensac_b200.matching import find_essential_ragged
    x1, x2, R, t, _ = scene(300, 0.6, 9, noise=0.5)
    rng = np.random.default_rng(4)
    cases = {}
    cases["n4"] = (x1[:4], x2[:4])
    y1, y2 = x1[:60].copy(), x2[:60].copy()
    y1[::2, 1] = np.nan
    y2[1::4, 0] = -np.inf
    cases["nonfinite"] = (y1, y2)
    cases["outliers"] = (rng.uniform(0, 640, (200, 2)), rng.uniform(0, 480, (200, 2)))
    px1, px2, pR, pt, _ = scene(400, 1.0, 10, noise=0.3, planar=True)
    cases["planar"] = (px1, px2)
    cases["good"] = (x1, x2)
    names = list(cases)
    a1 = np.concatenate([cases[k][0] for k in names])
    a2 = np.concatenate([cases[k][1] for k in names])
    off = np.zeros(len(names) + 1, np.int32)
    off[1:] = np.cumsum([len(cases[k][0]) for k in names])
    seeds = np.arange(len(names), dtype=np.int64) + 5
    g = _run(a1, a2, _K, _K, off, np.ones(len(a1), bool), seeds)
    ref = o.find_essential_ragged(a1, a2, _K, _K, off, None, 1.0, 0.999, 10000, seeds.astype(np.uint64), 10)
    for i, k in enumerate(names):
        assert g["iters"][i] == ref[i]["iters"], k
        assert g["n_inliers"][i] == ref[i]["n_inliers"], k
        assert np.isfinite(g["E"][i]).all() and np.isfinite(g["F"][i]).all(), k
    i = names.index("n4")
    assert g["iters"][i] == 0 and np.isnan(g["cost"][i]) and not g["E"][i].any()
    i = names.index("nonfinite")
    b = off[i]
    assert not g["mask"][b:b + 60][::2].any() and not g["mask"][b + 1:b + 60:4].any()
    i = names.index("outliers")
    assert g["n_inliers"][i] <= 40          # random pixels: a few rows lie near any epipolar geometry
    # a plane seen from two views fixes its homography, which two (R, t, n) explain: the planted pose or its twin
    i = names.index("planar")
    E = g["E"][i]
    Hn = _planar_homography(px1, px2)
    import cv2
    _, Rs, ts, _ = cv2.decomposeHomographyMat(_K @ Hn @ np.linalg.inv(_K), _K)
    twins = [_unit(_skew(tc.ravel()) @ Rc) for Rc, tc in zip(Rs, ts)]
    d_twin = min(_sign_dist(E, c) for c in twins)
    d_planted = _sign_dist(E, _unit(_skew(pt) @ pR))
    print("planar: %d inliers, E %.2e from the planted E, %.2e from the nearest decomposition of H"
          % (g["n_inliers"][i], d_planted, d_twin))
    assert g["n_inliers"][i] >= 360 and d_twin <= 1e-2
    assert min(_sign_dist(c, _unit(_skew(pt) @ pR)) for c in twins) <= 1e-2
    assert g["n_inliers"][names.index("good")] >= 160
    # refine_iters = 0: the RANSAC model itself; conf = 1: max_iters iterations
    z = _run(x1, x2, _K, _K, np.array([0, 300], np.int32), np.ones(300, bool), seeds[:1], refine_iters=0)
    r0 = o.find_essential(x1, x2, _K, _K, seed=5, refine_iters=0)
    assert z["cost"][0] == z["cost0"][0] and z["iters"][0] == r0["iters"] and z["n_inliers"][0] == r0["n_inliers"]
    assert _sign_dist(z["E"][0], r0["E"]) <= 1e-9
    c = _run(x1, x2, _K, _K, np.array([0, 300], np.int32), np.ones(300, bool), seeds[:1], conf=1.0, max_iters=77)
    assert c["iters"][0] == 77
    # rows = 0: every pair without a model
    e0 = _run(np.zeros((0, 2)), np.zeros((0, 2)), _K, _K, np.zeros(3, np.int32), np.zeros(0, bool), seeds[:2])
    assert (e0["iters"] == 0).all() and (e0["n_inliers"] == 0).all() and np.isnan(e0["cost"]).all()
    # malformed offsets: no model, no row read or written (pairs 1, 2 and 4; pair 4 passes the 300 rows)
    d1, d2, dK = _dev(x1, x2, _K)
    bad = torch.tensor([0, 150, -1, 150, 300, 400], dtype=torch.int32, device="cuda:0")
    dm = torch.ones(300, dtype=torch.bool, device="cuda:0")
    r = _np(find_essential_ragged(d1, d2, dK, dK, bad, dm, seeds=torch.arange(5, device="cuda:0")))
    for p in (1, 2, 4):
        assert r["iters"][p] == 0 and r["n_inliers"][p] == 0 and np.isnan(r["cost"][p]) and not r["E"][p].any()
    whole = _run(x1, x2, _K, _K, np.array([0, 150, 300], np.int32), np.ones(300, bool), np.array([0, 3], np.int64))
    for k in ("E", "F", "n_inliers", "iters", "cost"):
        assert whole[k][0].tobytes() == r[k][0].tobytes() and whole[k][1].tobytes() == r[k][3].tobytes(), k


def _planar_homography(x1, x2):
    """the homography x2 ~ H x1 of a planar pair by cv2's least squares on all rows, in normalised coordinates"""
    import cv2
    H = cv2.findHomography(x1, x2, 0)[0]
    return np.linalg.inv(_K) @ H @ _K


@pytest.mark.gpu
def test_pipeline_matching_essential_pose_refinement_without_sync():
    """match_descriptors_batch -> find_essential_ragged -> pose_from_fundamental_ragged(F) -> refine_pose_ragged with no
    host synchronisation, against the planted relative pose"""
    import torch
    from tests.test_refine_fundamental import _multiview_two_cameras
    from pydegensac_b200.matching import (find_essential_ragged, match_descriptors_batch, pose_from_fundamental_ragged,
                                          refine_pose_ragged)
    dev = torch.device("cuda:0")
    kps, descs, Rs, ts, Ks, _ = _multiview_two_cameras(2, 900, 300, 0, 64, 23)
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    K0, K1 = (torch.from_numpy(k).to(dev) for k in Ks[:2])
    seeds = torch.tensor([3], dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m = match_descriptors_batch(dt, [(0, 1)], kt, ratio=0.9, mutual=True)
        ess = find_essential_ragged(m.pts1, m.pts2, K0, K1, m.offsets, px_th=1.0, seeds=seeds)
        pose = pose_from_fundamental_ragged(ess.F, K0, K1, m.pts1, m.pts2, m.offsets, ess.mask)
        fine = refine_pose_ragged(pose.R, pose.t, K0, K1, m.pts1, m.pts2, m.offsets, pose.in_front, px_th=1.0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    R10 = Rs[1] @ Rs[0].T
    t10 = ts[1] - R10 @ ts[0]
    t10 /= np.linalg.norm(t10)
    out = []
    for R, t in ((pose.R[0], pose.t[0]), (fine.R[0], fine.t[0])):
        R, t = R.cpu().numpy(), t.cpu().numpy()
        out.append((_rot_error(R, R10), float(np.arccos(np.clip(t @ t10 / np.linalg.norm(t), -1.0, 1.0)))))
    print("essential: %d inliers in %d iterations, MSAC cost %.2f -> %.2f; pose error (rad) %s -> refined %s"
          % (int(ess.n_inliers[0]), int(ess.iters[0]), float(ess.cost0[0]), float(ess.cost[0]), out[0], out[1]))
    assert int(ess.n_inliers[0]) >= 500
    assert float(ess.cost[0]) <= float(ess.cost0[0])
    assert int(pose.good[0]) >= 500
    for er, et in out:
        assert er <= 5e-3 and et <= 2e-2
