"""matching.calibrate_view_graph: each camera group's focal length from the pairs' fundamental matrices, robust
Levenberg-Marquardt on the Kruppa residuals with a Jacobi-preconditioned CG step over the groups.
CPU: the oracle (tests/view_graph_calibration_np.py) -- zero residuals at the planted intrinsics, invariance to the
scale of F and to swapping an edge's views, its Jacobian, its CG, its fixed point against scipy, planted recovery and
outlier edges -- the host build of csrc/view_graph_calibration.h, and the argument checks of the Python wrapper and the
C entry point.  GPU: the kernels against the oracle on many graphs, determinism, edge cases, one group over 2 10^5
edges, F from the device RANSAC and the example pipeline without a host read."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
from scipy.optimize import least_squares

from tests import view_graph_calibration_np as vg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")


def planted(n, groups, seed, pairs=None, pp_off=0.0, start_scale=None):
    """n views with random poses, the camera group of each view (groups [n]), each group's true intrinsics and the
    noise-free F of every pair (all pairs when pairs is None).  Returns (pairs, F, k_true [G,5], k_start [G,5]): the
    start is the truth with f scaled by start_scale (default: 768 / 800)"""
    rng = np.random.default_rng(seed)
    groups = np.asarray(groups, np.int32)
    G = int(groups.max()) + 1
    R, t = vg.random_views(rng, n)
    f = rng.uniform(600.0, 1000.0, G)
    pp = np.c_[320.0 + pp_off * rng.uniform(-1, 1, G), 240.0 + pp_off * rng.uniform(-1, 1, G)]
    k_true = np.c_[f, pp, np.zeros((G, 2))]
    K = [vg.K_of(k) for k in k_true]
    if pairs is None:
        pairs = np.array([(i, j) for i in range(n) for j in range(i + 1, n)], np.int32)
    F = np.array([vg.fundamental(K[groups[i]], R[i], t[i], K[groups[j]], R[j], t[j]) for i, j in pairs])
    k_start = k_true.copy()
    k_start[:, 0] *= (768.0 / 800.0) if start_scale is None else start_scale
    return np.asarray(pairs, np.int32), F, k_true, k_start


def noisy(F, rng, sigma=1e-3, f=800.0):
    """F with noise of relative size sigma on the entries of D F D, D = diag(f, f, 1) (close to the essential matrix,
    where every entry counts), projected back to rank 2"""
    D = np.diag([f, f, 1.0])
    out = []
    for M in F:
        E = D @ M @ D
        E = E / np.linalg.norm(E) + sigma * rng.normal(size=(3, 3)) / 3.0
        U, s, Vt = np.linalg.svd(E)
        out.append(np.linalg.inv(D) @ U @ np.diag([s[0], s[1], 0.0]) @ Vt @ np.linalg.inv(D))
    return np.array(out).reshape(-1, 3, 3)


GROUPINGS = {"a group per view": np.arange(8), "one group": np.zeros(8, np.int32),
             "mixed groups": np.array([0, 0, 1, 1, 1, 2, 3, 3])}


# ------------------------------------------------------------------------------------------------ oracle (CPU)
@pytest.mark.parametrize("case", ["different groups", "same group", "principal points off centre", "random poses"])
def test_residuals_vanish_at_the_planted_intrinsics(case):
    groups = {"different groups": np.arange(6), "same group": np.zeros(6, np.int32),
              "principal points off centre": np.arange(6), "random poses": np.array([0, 1, 0, 1, 2, 2])}[case]
    for seed in range(5):
        pairs, F, k_true, _ = planted(6, groups, 10 + seed, pp_off=60.0 if case != "same group" else 0.0)
        used, c, gi, gj = vg.prepare(pairs, F, groups, k_true)
        assert used.all()
        for e in range(len(pairs)):
            r, _, _ = vg.residuals(c[e], 0.0, 0.0)
            assert np.abs(r).max() <= 1e-12, (case, seed, e)


def test_error_and_cost_do_not_change_with_the_scale_of_F_or_a_swap():
    rng = np.random.default_rng(3)
    groups = np.array([0, 1, 2, 0, 1, 2])
    pairs, F, _, k0 = planted(6, groups, 3)
    F = noisy(F, rng, 3e-3)
    base = vg.calibrate_view_graph(pairs, F, groups, k0, max_iters=0)
    for scale in (-3.0, 0.25, 7.0):
        o = vg.calibrate_view_graph(pairs, scale * F, groups, k0, max_iters=0)
        assert np.abs(o["error"] - base["error"]).max() <= 1e-12 and abs(o["cost0"] - base["cost0"]) <= 1e-14
    swap = np.arange(len(pairs)) % 2 == 0
    p2, F2 = pairs.copy(), F.copy()
    p2[swap] = pairs[swap][:, ::-1]
    F2[swap] = np.swapaxes(F[swap], 1, 2)
    o = vg.calibrate_view_graph(p2, F2, groups, k0, max_iters=0)
    assert np.abs(o["error"] - base["error"]).max() <= 1e-12
    # and after the solve
    a = vg.calibrate_view_graph(pairs, F, groups, k0)
    b = vg.calibrate_view_graph(p2, -2.0 * F2, groups, k0)
    assert np.abs(a["theta"] - b["theta"]).max() <= 1e-9 and abs(a["cost"] - b["cost"]) <= 1e-12


def test_jacobian_by_central_differences():
    rng = np.random.default_rng(4)
    pairs, F, _, k0 = planted(6, np.arange(6), 4)
    used, c, _, _ = vg.prepare(pairs, noisy(F, rng), np.arange(6), k0)
    h = 1e-6
    for e in range(len(pairs)):
        ti, tj = rng.uniform(-0.5, 0.5, 2)
        _, J, _ = vg.residuals(c[e], ti, tj)
        Jn = np.stack([(vg.residuals(c[e], ti + h, tj)[0] - vg.residuals(c[e], ti - h, tj)[0]) / (2 * h),
                       (vg.residuals(c[e], ti, tj + h)[0] - vg.residuals(c[e], ti, tj - h)[0]) / (2 * h)], 1)
        assert np.abs(J - Jn).max() <= 1e-8 * max(1.0, np.abs(J).max()), e


def test_oracle_pcg_equals_a_dense_solve():
    rng = np.random.default_rng(5)
    groups = GROUPINGS["mixed groups"]
    pairs, F, _, k0 = planted(8, groups, 5)
    used, c, gi, gj = vg.prepare(pairs, noisy(F, rng), groups, k0)
    G = 4
    theta = rng.uniform(-0.1, 0.1, G)
    H, g = vg.linearise(c, used, gi, gj, theta, 1e-4, G)
    active = np.ones(G, bool)
    for lam in (1e-3, 1.0):
        A, m = vg.damped(H, lam, active)
        x, k, rej = vg.pcg(A, m, -g, 1e-14, 500)
        ref = np.linalg.solve(A.toarray(), -g)
        assert not rej and np.abs(x - ref).max() <= 1e-10 * np.abs(ref).max()
    # a group without an edge is an identity row
    active[2] = False
    A, m = vg.damped(H, 1e-3, active)
    b = np.where(active, -g, 0.0)
    x, _, _ = vg.pcg(A, m, b, 1e-14, 500)
    assert x[2] == 0.0


@pytest.mark.parametrize("loss_scale", [0.0, 1e-2])
def test_final_cost_equals_scipy(loss_scale):
    rng = np.random.default_rng(6)
    groups = np.array([0, 1, 2, 0, 1, 2])
    pairs, F, _, k0 = planted(6, groups, 6)
    F = noisy(F, rng, 1e-2)
    o = vg.calibrate_view_graph(pairs, F, groups, k0, loss_scale=loss_scale, cg_tol=1e-12)
    used, c, gi, gj = vg.prepare(pairs, F, groups, k0)

    if loss_scale == 0.0:
        def fun(th):
            return np.concatenate([vg.residuals(c[e], th[gi[e]], th[gj[e]])[0] for e in range(len(pairs))])
        ref = least_squares(fun, np.zeros(3), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
        ref_cost = 2.0 * ref.cost
    else:
        # one residual per edge, sqrt(s_e), so that scipy's per-residual loss is the per-edge Cauchy loss
        def fun(th):
            return np.array([np.sqrt(vg.residuals(c[e], th[gi[e]], th[gj[e]])[2]) for e in range(len(pairs))])
        ref = least_squares(fun, np.zeros(3), loss="cauchy", f_scale=loss_scale, xtol=1e-15, ftol=1e-15, gtol=1e-15)
        ref_cost = 2.0 * ref.cost
    assert abs(o["cost"] - ref_cost) <= 1e-9 * ref_cost, (o["cost"], ref_cost)
    assert np.abs(o["theta"] - ref.x).max() <= 1e-5


@pytest.mark.parametrize("grouping", list(GROUPINGS))
def test_planted_recovery(grouping):
    groups = GROUPINGS[grouping]
    pairs, F, k_true, k0 = planted(8, groups, 7)
    o = vg.calibrate_view_graph(pairs, F, groups, k0, cg_tol=1e-10)
    assert o["refined"].all() and o["inliers"].all() and o["n_used"] == len(pairs)
    assert np.abs(o["intrinsics"][:, 0] / k_true[:, 0] - 1.0).max() <= 1e-8, grouping
    assert (o["intrinsics"][:, 1:] == k0[:, 1:]).all()


def test_random_F_edges_are_not_inliers():
    rng = np.random.default_rng(8)
    n = 12
    groups = np.zeros(n, np.int32)
    pairs, F, k_true, k0 = planted(n, groups, 8)
    F = noisy(F, rng, 1e-4)
    bad = rng.random(len(pairs)) < 0.1
    bad[0] = True
    F[bad] = noisy(rng.normal(size=(int(bad.sum()), 3, 3)), rng, 0.0)
    o = vg.calibrate_view_graph(pairs, F, groups, k0)
    rel = abs(o["intrinsics"][0, 0] / k_true[0, 0] - 1.0)
    print("f error %.2e, bad edges' errors >= %.3f, good edges' <= %.4f" % (rel, np.nanmin(o["error"][bad]),
                                                                             np.nanmax(o["error"][~bad])))
    assert not o["inliers"][bad].any()
    assert o["inliers"][~bad].mean() >= 0.95
    assert rel <= 1e-3


# ------------------------------------------------------------------------------------------------ host build (CPU)
def test_host_build_matches_the_oracle(tmp_path):
    so = os.path.join(str(tmp_path), "libview_graph_calibration_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-o", so, os.path.join(ROOT, "tests", "view_graph_calibration_host.cpp")])
    L = ctypes.CDLL(so)
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))  # noqa: E731
    ip = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))  # noqa: E731
    rng = np.random.default_rng(9)
    groups = np.array([0, 1, 2, 0, 1, 2, 3, 3])
    pairs, F, _, k0 = planted(8, groups, 9)
    F = np.ascontiguousarray(noisy(F, rng, 1e-2))
    n = len(pairs)
    ki = np.ascontiguousarray(k0[groups[pairs[:, 0]]])
    kj = np.ascontiguousarray(k0[groups[pairs[:, 1]]])
    c, ok = np.zeros((n, 12)), np.zeros(n, np.intc)
    L.vgh_constants(n, dp(F), dp(ki), dp(kj), dp(c), ip(ok))
    assert ok.all()
    ref = np.array([vg.constants(F[e], ki[e], kj[e]) for e in range(n)])
    # index 1 (A1, B1) changes sign with the singular vectors' signs
    sg = np.sign(c[:, 1] * ref[:, 1])
    ref[:, [1, 4, 7, 10]] *= sg[:, None]
    assert np.abs(c - ref).max() <= 1e-12
    ti, tj = rng.uniform(-0.5, 0.5, n), rng.uniform(-0.5, 0.5, n)
    r, J, s = np.zeros((n, 2)), np.zeros((n, 4)), np.zeros(n)
    L.vgh_residuals(n, dp(c), dp(ti), dp(tj), dp(r), dp(J), dp(s))
    for e in range(n):
        rr, JJ, ss = vg.residuals(c[e], ti[e], tj[e])
        assert np.abs(r[e] - rr).max() <= 1e-15 and np.abs(J[e] - JJ.reshape(-1)).max() <= 1e-14
        assert abs(s[e] - ss) <= 1e-16
    rho, w = np.zeros(n), np.zeros(n)
    for sig2 in (0.0, 1e-4):
        L.vgh_loss(n, dp(s), ctypes.c_double(sig2), dp(rho), dp(w))
        assert np.allclose(rho, [vg.rho(x, sig2) for x in s], rtol=1e-15, atol=0)
        assert np.allclose(w, [vg.weight(x, sig2) for x in s], rtol=1e-15, atol=0)
    # validity: self-pair, out-of-range view and group, masked, non-finite F; intrinsics; rank-1 F
    ij = np.ascontiguousarray(np.array([[0, 1], [2, 2], [0, 8], [0, 1], [0, 1], [0, 1], [0, 1]], np.intc))
    gg = np.ascontiguousarray(np.array([[0, 1], [0, 0], [0, 1], [0, 4], [-1, 0], [0, 1], [0, 1]], np.intc))
    mk = np.ascontiguousarray(np.array([1, 1, 1, 1, 1, 0, 1], np.intc))
    FF = np.ascontiguousarray(np.repeat(F[:1], 7, 0))
    FF[6, 1, 1] = np.nan
    out = np.zeros(7, np.intc)
    L.vgh_edge_ok(7, ip(ij), 8, ip(gg), 4, ip(mk), dp(FF), ip(out))
    assert out.tolist() == [1, 0, 0, 0, 0, 0, 0]
    kk = np.ascontiguousarray(np.array([k0[0], [0.0, 320, 240, 0, 0], [800, np.nan, 240, 0, 0], [-5, 1, 1, 0, 0]]))
    out = np.zeros(4, np.intc)
    L.vgh_intrinsics_ok(4, dp(kk), ip(out))
    assert out.tolist() == [1, 0, 0, 0] == [int(vg.intrinsics_ok(k)) for k in kk]
    r1 = np.ascontiguousarray(np.outer([1.0, 2, 3], [0.5, -1, 2]).reshape(1, 9))
    L.vgh_constants(1, dp(r1), dp(ki), dp(kj), dp(c), ip(ok))
    assert ok[0] == 0 and vg.constants(r1.reshape(3, 3), ki[0], kj[0]) is None
    # write-back: inside, outside and at the ratio, without an edge, NaN
    th = np.array([0.1, np.log(11.0), -np.log(10.0), 0.2, np.nan])
    he = np.array([1, 1, 1, 0, 1], np.intc)
    kin = np.ascontiguousarray(np.repeat(k0[:1], 5, 0))
    ko, ref_out = np.zeros((5, 5)), np.zeros(5, np.intc)
    L.vgh_write_back(5, dp(kin), dp(th), ip(he), ctypes.c_double(10.0), dp(ko), ip(ref_out))
    assert ref_out.tolist() == [1, 0, int(np.exp(th[2]) >= 0.1), 0, 0]
    assert ko[0, 0] == kin[0, 0] * np.exp(0.1) and (ko[1] == kin[1]).all() and (ko[3] == kin[3]).all()


# ------------------------------------------------------------------------------------------------ arguments (CPU)
def test_python_messages():
    torch = pytest.importorskip("torch")
    from pydegensac_b200.matching import calibrate_view_graph
    f64, i32 = torch.float64, torch.int32
    k = torch.tensor([[768.0, 320, 240, 0, 0]], dtype=f64)
    good = dict(pairs=[[0, 1], [1, 2]], F=torch.eye(3, dtype=f64).repeat(2, 1, 1), groups=torch.zeros(3, dtype=i32),
                intrinsics=k)
    host = "F, groups, intrinsics and mask must be CUDA tensors on one device"
    cases = [
        ({"F": np.eye(3)}, "F must be a torch tensor"),
        ({"groups": [0, 0, 0]}, "groups must be a torch tensor"),
        ({"groups": torch.zeros(3, dtype=torch.int64)}, "groups must be int32, not torch.int64"),
        ({"groups": torch.zeros((3, 1), dtype=i32)}, "groups must be [C] with C >= 1, not [3, 1]"),
        ({"intrinsics": torch.zeros((1, 4), dtype=f64)}, "intrinsics must be [G,5] with G >= 1, not [1, 4]"),
        ({"intrinsics": torch.zeros((0, 5), dtype=f64)}, "intrinsics must be [G,5] with G >= 1, not [0, 5]"),
        ({"pairs": [[0, 3]]}, "pairs: image index out of range"),
        ({"pairs": [[-1, 0]]}, "pairs: image index out of range"),
        ({"pairs": np.zeros((0, 2))}, "pairs must be a non-empty [P,2] array of (query image, train image)"),
        ({"F": torch.eye(3, dtype=f64).repeat(2, 1)}, "F must be [P,3,3] or [P,9] with P >= 1, not [6, 3]"),
        ({"F": torch.eye(3, dtype=f64).repeat(3, 1, 1)}, "F must hold one matrix per pair (2), not 3"),
        ({"F": torch.zeros((2, 9), dtype=i32)}, "F must be a floating tensor, not torch.int32"),
        ({"intrinsics": torch.zeros((1, 5), dtype=i32)}, "intrinsics must be a floating tensor, not torch.int32"),
        ({"mask": torch.ones(3, dtype=torch.bool)}, "mask must be [P] = [2], not [3]"),
        ({"mask": torch.ones(2, dtype=i32)}, "mask must be bool or uint8, not torch.int32"),
        ({"loss_scale": -1.0}, "loss_scale must be a non-negative finite number, not -1.0"),
        ({"loss_scale": float("nan")}, "loss_scale must be a non-negative finite number, not nan"),
        ({"max_error": float("inf")}, "max_error must be a non-negative finite number, not inf"),
        ({"cg_tol": -1e-6}, "cg_tol must be a non-negative finite number, not -1e-06"),
        ({"max_ratio": 0.5}, "max_ratio must be a finite number >= 1, not 0.5"),
        ({"max_ratio": float("nan")}, "max_ratio must be a finite number >= 1, not nan"),
        ({"max_iters": -1}, "max_iters must not be negative, not -1"),
        ({"cg_max_iters": 0}, "cg_max_iters must be at least 1, not 0"),
        ({"loss_scale": 0.0, "max_iters": 0, "max_ratio": 1.0, "cg_tol": 0.0}, host),
        ({"F": torch.eye(3, dtype=torch.float32).repeat(2, 1, 1).view(2, 9)}, host),
        ({}, host),
    ]
    for kw, msg in cases:
        with pytest.raises(ValueError) as e:
            calibrate_view_graph(**dict(good, **kw))
        assert str(e.value) == msg, kw


def test_c_entry_point_refuses_malformed_input_before_any_call():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["F", "groups", "intrinsics", "k_out", "refined", "error", "inliers", "cost0", "cost", "iters", "n_used",
             "cg_iters"]

    def call(pairs=((0, 1), (1, 2)), n_pairs=None, n_views=3, n_groups=1, loss_scale=0.01, max_error=0.01,
             max_ratio=10.0, max_iters=100, cg_max_iters=500, cg_tol=1e-6, null=()):
        b = {k: (None if k in null else fake) for k in names}
        flat = [v for p in pairs for v in p]
        hp = (ctypes.c_int32 * max(len(flat), 1))(*flat)
        d = ctypes.c_double
        return L.dgb200_calibrate_view_graph_dev(
            None if "pairs" in null else hp, len(pairs) if n_pairs is None else n_pairs, n_views, b["F"], None,
            b["groups"], b["intrinsics"], n_groups, d(loss_scale), d(max_error), d(max_ratio), max_iters, cg_max_iters,
            d(cg_tol), b["k_out"], b["refined"], b["error"], b["inliers"], b["cost0"], b["cost"], b["iters"],
            b["n_used"], b["cg_iters"], None)

    sizes = "need n_views >= 1, n_pairs >= 1 and n_groups >= 1"
    cases = [(dict(null={k}), "null buffer") for k in names]
    cases += [
        (dict(n_views=0), sizes), (dict(n_pairs=0), sizes), (dict(n_groups=0), sizes),
        (dict(null={"pairs"}), "null pair table"),
        (dict(pairs=((0, 3),)), "pair view index out of range"), (dict(pairs=((-1, 1),)), "pair view index out of range"),
        (dict(loss_scale=-1.0), "loss_scale must be a non-negative finite number"),
        (dict(loss_scale=float("inf")), "loss_scale must be a non-negative finite number"),
        (dict(max_error=float("nan")), "max_error must be a non-negative finite number"),
        (dict(max_ratio=0.99), "max_ratio must be a finite number >= 1"),
        (dict(max_ratio=float("inf")), "max_ratio must be a finite number >= 1"),
        (dict(max_iters=-1), "max_iters must not be negative"),
        (dict(cg_max_iters=0), "cg_max_iters must be at least 1"),
        (dict(cg_tol=float("nan")), "cg_tol must be a non-negative finite number"),
    ]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert L.dgb200_view_graph_calibration_last_error().decode() == msg, kw


# ------------------------------------------------------------------------------------------------ GPU
def _run(pairs, F, groups, kin, mask=None, **kw):
    import torch
    from pydegensac_b200.matching import calibrate_view_graph
    dev = torch.device("cuda:0")
    m = torch.from_numpy(np.asarray(mask)).to(dev) if mask is not None else None
    out = calibrate_view_graph(pairs, torch.from_numpy(np.ascontiguousarray(F)).to(dev),
                               torch.from_numpy(np.asarray(groups, np.int32)).to(dev),
                               torch.from_numpy(np.ascontiguousarray(kin)).to(dev), mask=m, **kw)
    return {k: getattr(out, k).cpu().numpy() for k in out._fields}


def _graphs():
    """(name, pairs, F, groups, k_start, mask) over random graphs and groupings, with noisy F and a few random ones"""
    out = []
    for seed in range(12):
        rng = np.random.default_rng(100 + seed)
        n = int(rng.integers(5, 14))
        G = int(rng.integers(1, n + 1))
        groups = np.r_[np.arange(G), rng.integers(0, G, n - G)].astype(np.int32)
        rng.shuffle(groups)
        allp = np.array([(i, j) for i in range(n) for j in range(i + 1, n)], np.int32)
        keep = rng.random(len(allp)) < 0.6
        keep[:1] = True
        pairs, F, _, k0 = planted(n, groups, 100 + seed, pairs=allp[keep], pp_off=20.0,
                                  start_scale=rng.uniform(0.8, 1.2))
        F = noisy(F, rng, 3e-3)
        bad = rng.random(len(pairs)) < 0.1
        F[bad] = noisy(rng.normal(size=(int(bad.sum()), 3, 3)), rng, 0.0)
        rev = rng.random(len(pairs)) < 0.5
        pairs[rev] = pairs[rev][:, ::-1]
        F[rev] = np.swapaxes(F[rev], 1, 2)
        mask = rng.random(len(pairs)) > 0.05 if seed % 3 == 0 else None
        out.append(("graph %d (%d views, %d groups, %d pairs)" % (seed, n, G, len(pairs)), pairs, F, groups, k0, mask))
    return out


@pytest.mark.gpu
def test_kernels_equal_the_oracle():
    for name, p, F, gr, k0, m in _graphs():
        for ls in (0.0, 1e-2):
            g = _run(p, F, gr, k0, m, loss_scale=ls)
            o = vg.calibrate_view_graph(p, F, gr, k0, m, loss_scale=ls)
            th = np.log(g["intrinsics"][:, 0] / k0[:, 0])
            tho = np.where(o["refined"], o["theta"], 0.0)
            print("%s, loss %g: steps %d (oracle %d), CG %d (oracle %d), largest |d theta| %.2e"
                  % (name, ls, g["iters"][0], o["iters"], g["cg_iters"][0], o["cg_iters"], np.abs(th - tho).max()))
            assert g["n_used"][0] == o["n_used"], name
            assert (g["refined"] == o["refined"]).all(), name
            assert (g["inliers"] == o["inliers"]).all(), name
            assert np.abs(th - tho).max() <= 1e-10, name
            assert abs(g["cost"][0] - o["cost"]) <= 1e-10 * max(o["cost"], 1e-300) + 1e-300, name
            assert abs(g["cost0"][0] - o["cost0"]) <= 1e-12 * o["cost0"], name
            assert np.array_equal(np.isnan(g["error"]), np.isnan(o["error"])), name
            assert np.nan_to_num(np.abs(g["error"] - o["error"])).max() <= 1e-9, name


@pytest.mark.gpu
def test_same_bytes_on_a_rerun():
    name, p, F, gr, k0, m = _graphs()[4]
    a = _run(p, F, gr, k0, m)
    b = _run(p, F, gr, k0, m)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


@pytest.mark.gpu
def test_edge_cases():
    rng = np.random.default_rng(12)
    groups = np.array([0, 0, 1, 1, 2, 2, 3], np.int32)       # group 3's only view has no pair; group 4 no view
    pairs, F, k_true, k0 = planted(6, groups[:6], 12)
    k0 = np.r_[k0, [[700.0, 300.0, 200.0, 0.01, -0.02], [650.0, 310.0, 230.0, 0.0, 0.0]]]
    F = noisy(F, rng, 1e-4)
    F[0, 1, 2] = np.nan                                       # NaN F
    F[1] = 0.0                                                # zero F
    F[2] = np.outer([1.0, 2.0, 3.0], [0.5, -1.0, 2.0])        # rank 1
    mask = np.ones(len(pairs), bool)
    mask[3] = False                                           # masked
    g = _run(pairs, F, groups, k0, mask)
    o = vg.calibrate_view_graph(pairs, F, groups, k0, mask)
    assert np.isnan(g["error"][:4]).all() and not g["inliers"][:4].any()
    assert g["n_used"][0] == len(pairs) - 4 == o["n_used"]
    assert not g["refined"][3:].any() and g["refined"][:3].all()
    assert g["intrinsics"][3:].tobytes() == k0[3:].tobytes()
    assert (g["intrinsics"][:3, 1:] == k0[:3, 1:]).all()
    # max_iters = 0: the start
    z = _run(pairs, F, groups, k0, mask, max_iters=0)
    assert z["cost0"][0] == z["cost"][0] and z["iters"][0] == 0 and z["cg_iters"][0] == 0
    assert z["intrinsics"].tobytes() == k0.tobytes()
    assert abs(z["cost0"][0] - o["cost0"]) <= 1e-12 * o["cost0"]
    # a group index outside [0, G): the edges of that view are not used
    bad_groups = groups.copy()
    bad_groups[0] = 9
    b = _run(pairs, F, bad_groups, k0, mask)
    ob = vg.calibrate_view_graph(pairs, F, bad_groups, k0, mask)
    assert b["n_used"][0] == ob["n_used"] and (b["inliers"] == ob["inliers"]).all()


@pytest.mark.gpu
def test_one_group_over_two_hundred_thousand_edges():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from view_graph_calibration_rate import synth
    pairs, F, groups, k0, f_true = synth(10000, 200000, 1, 0)
    g = _run(pairs, F, groups, k0)
    o = vg.calibrate_view_graph(pairs, F, groups, k0)
    th = np.log(g["intrinsics"][:, 0] / k0[:, 0])
    print("one group, %d edges: steps %d (oracle %d), CG %d, f %.4f (true %.1f), |d theta| %.2e"
          % (len(pairs), g["iters"][0], o["iters"], g["cg_iters"][0], g["intrinsics"][0, 0], f_true[0],
             abs(th[0] - o["theta"][0])))
    assert g["n_used"][0] == o["n_used"] and (g["inliers"] == o["inliers"]).all()
    assert abs(th[0] - o["theta"][0]) <= 1e-10
    assert abs(g["intrinsics"][0, 0] / f_true[0] - 1.0) <= 1e-3


@pytest.mark.gpu
def test_path_scene_focal_length_from_the_device_ransac():
    import sys
    import torch
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import gpu_pipeline
    import pydegensac_b200 as pydegensac
    from pydegensac_b200.matching import calibrate_view_graph, match_descriptors_batch
    dev = torch.device("cuda:0")
    _, Rs, _, kps, descs, pairs = gpu_pipeline.path_scene(dev)
    m = match_descriptors_batch(descs, pairs, kps, ratio=0.9, mutual=True)
    seeds = torch.arange(len(pairs), dtype=torch.int64, device=dev)
    F, _ = pydegensac.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                                 n_max=m.n_max)
    groups = torch.zeros(len(Rs), dtype=torch.int32, device=dev)
    k0 = torch.tensor([[768.0, 320.0, 240.0, 0.0, 0.0]], dtype=torch.float64, device=dev)
    cal = calibrate_view_graph(pairs, F, groups, k0)
    f = float(cal.intrinsics[0, 0])
    o = vg.calibrate_view_graph(pairs, F.cpu().numpy(), np.zeros(len(Rs), np.int32), k0.cpu().numpy())
    print("path scene: f %.3f (oracle %.3f), error %.3f %%, %d of %d pairs inliers, %d steps"
          % (f, o["intrinsics"][0, 0], 100 * abs(f / 800.0 - 1), int(cal.inliers.sum()), len(pairs),
             int(cal.iters[0])))
    assert abs(f / 800.0 - 1.0) <= F_BOUND
    assert abs(f - o["intrinsics"][0, 0]) <= 1e-8 * f


@pytest.mark.gpu
def test_example_uncalibrated_stage_without_a_host_read():
    import sys
    import torch
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import gpu_pipeline
    dev = torch.device("cuda:0")
    scene = gpu_pipeline.path_scene(dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = gpu_pipeline.uncalibrated_reconstruction_run(dev, scene)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    e_cal, e_ba, c_max, r_max = gpu_pipeline.report_uncalibrated_reconstruction(scene, out)
    assert e_cal <= F_BOUND and e_ba <= F_BOUND
    assert c_max < 0.05 and r_max < 0.5


# The relative focal error of the path scene's calibration from the device RANSAC's F (start 768, planted 800): 0.44 %
# on an H100, 0.08 % after the bundle adjustment of the example's stage
F_BOUND = 0.01
