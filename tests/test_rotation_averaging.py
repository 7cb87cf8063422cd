"""matching.average_rotations: a world rotation for every view from the relative rotations of its pairs, a maximum-
spanning-forest start and robust IRLS, each step a Jacobi-preconditioned CG solve of the weighted graph Laplacian.
CPU: the oracle (tests/rotation_averaging_np.py) against scipy -- its spanning forest and components, its log map, its
CG -- the linearisation by finite differences, the IRLS fixed point as a stationary point of the Geman-McClure cost,
planted recovery, relabelling, the host build of csrc/rotation_averaging.h, and the argument checks of the Python
wrapper and the C entry point.  GPU: the kernels against the oracle on many graphs, determinism, planted recovery, the
example pipeline without a host read and a 10^4-view graph."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from tests import rotation_averaging_np as ra

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")
TIGHT = 1e-14


def rand_rot(rng, n):
    return Rotation.random(n, random_state=rng).as_matrix()


def rot_exp(w):
    return Rotation.from_rotvec(np.atleast_2d(w)).as_matrix()


def angle(A, B):
    """the angle of A B^T, [...]"""
    return np.linalg.norm(Rotation.from_matrix(A @ np.swapaxes(B, -1, -2)).as_rotvec(), axis=-1)


def planted(n, extra, seed, noise_deg=1.0, outliers=0.0, chain=True, weights=True):
    """n views with random rotations; a path (v, v + 1) when chain, plus `extra` random pairs; R_e = exp(noise)
    R_j R_i^T with noise of noise_deg degrees per axis, a share `outliers` of the random pairs replaced by random
    rotations; distinct random weights, the outliers' below the others' (a wrong pose has little support).  Returns
    (pairs, R_rel, weights, R_true)"""
    rng = np.random.default_rng(seed)
    R = rand_rot(rng, n)
    pairs = [(v, v + 1) for v in range(n - 1)] if chain else []
    while len(pairs) < (n - 1 if chain else 0) + extra:
        i, j = (int(x) for x in rng.choice(n, 2, replace=False))
        pairs.append((i, j))
    pairs = np.array(pairs, dtype=np.int32).reshape(-1, 2)
    P = len(pairs)
    Re = np.einsum("pij,pkj->pik", R[pairs[:, 1]], R[pairs[:, 0]])
    Re = rot_exp(np.radians(noise_deg) * rng.normal(size=(P, 3))) @ Re
    bad = rng.random(P) < outliers
    bad[: n - 1 if chain else 0] = False
    Re[bad] = rand_rot(rng, int(bad.sum()))
    w = rng.permutation(P).astype(np.int32) + 10 + np.where(bad, 0, P).astype(np.int32) if weights else None
    return pairs, Re, w, R


def gauge_errors(Rest, Rtrue, ref=0):
    """the angle between each estimated and planted rotation after aligning the gauge at view `ref` (R_v -> R_v G)"""
    G = Rest[ref].T @ Rtrue[ref]
    return angle(Rest @ G, Rtrue)


# ------------------------------------------------------------------------------------------------ oracle (CPU)
def test_oracle_tree_is_the_maximum_spanning_forest():
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components, minimum_spanning_tree
    rng = np.random.default_rng(1)
    for trial in range(20):
        n = int(rng.integers(5, 60))
        # distinct undirected edges over a few components
        cand = {(int(a), int(b)) for a, b in rng.integers(0, n, (3 * n, 2)) if a != b and (a // 13) == (b // 13)}
        pairs = np.array(sorted({(min(a, b), max(a, b)) for a, b in cand}), dtype=np.int64)
        rev = rng.random(len(pairs)) < 0.5
        pairs[rev] = pairs[rev][:, ::-1]
        w = rng.permutation(len(pairs)).astype(np.int64)
        valid = np.ones(len(pairs), bool)
        in_tree, comp = ra.spanning_forest(pairs, valid, w, n)
        G = coo_matrix((-(w + 1.0), (pairs.min(1), pairs.max(1))), shape=(n, n)).tocsr()
        T = minimum_spanning_tree(G).tocoo()
        ref = {(int(a), int(b)) for a, b in zip(T.row, T.col)}
        got = {(int(min(a, b)), int(max(a, b))) for a, b in pairs[in_tree]}
        assert got == ref, trial
        k, lab = connected_components(G, directed=False)
        deg = np.bincount(pairs.reshape(-1), minlength=n)
        for c in range(k):
            members = np.flatnonzero(lab == c)
            expect = members.min() if deg[members].sum() else -1
            assert (comp[members] == expect).all(), trial


def test_log_map_against_scipy():
    rng = np.random.default_rng(2)
    R = rand_rot(rng, 4000)
    th_ref = np.linalg.norm(Rotation.from_matrix(R).as_rotvec(), axis=1)
    away = th_ref < math.pi - 1e-2
    r, th = ra.log_map(R)
    assert np.abs(r[away] - Rotation.from_matrix(R[away]).as_rotvec()).max() <= 1e-12
    # every branch: small, ordinary, near pi and pi itself
    axes = rng.normal(size=(200, 3))
    axes /= np.linalg.norm(axes, axis=1)[:, None]
    for t in (0.0, 1e-9, 1e-5, 0.99e-4, 1.01e-4, 0.5, 3.0, math.pi - 2e-3, math.pi - 5e-4, math.pi - 1e-7,
              math.pi - 1e-12):
        Rt = rot_exp(t * axes)
        r, th = ra.log_map(Rt)
        assert np.isfinite(r).all() and np.isfinite(th).all(), t
        ref = Rotation.from_matrix(Rt).as_rotvec()
        tol = 1e-12 if t < math.pi - 1e-3 else 1e-9
        assert np.abs(r - ref).max() <= tol, t
    # theta = pi: the axis up to its sign
    Rp = rot_exp(math.pi * axes)
    r, th = ra.log_map(Rp)
    assert np.abs(th - math.pi).max() <= 1e-12
    assert np.abs(np.abs(np.einsum("ni,ni->n", r / math.pi, axes)) - 1.0).max() <= 1e-12


def test_linearisation_by_finite_differences():
    rng = np.random.default_rng(3)
    Ri, Rj = rand_rot(rng, 2)
    Re = Rj @ Ri.T
    wi, wj = rng.normal(size=3), rng.normal(size=3)
    errs = []
    for h in (1e-2, 1e-3, 1e-4):
        dR = (Rj @ ra.expmap(h * wj)).T @ Re @ Ri @ ra.expmap(h * wi)
        r, _ = ra.log_map(dR[None])
        errs.append(np.linalg.norm(r[0] - h * (wi - wj)))
    # second order: each tenfold smaller h cuts the error a hundredfold
    assert 50 <= errs[0] / errs[1] <= 200 and 50 <= errs[1] / errs[2] <= 200, errs


def test_oracle_cg_equals_spsolve():
    from scipy.sparse.linalg import spsolve
    pairs, Re, w, R = planted(60, 150, 4)
    n = 60
    valid = np.ones(len(pairs), bool)
    rng = np.random.default_rng(4)
    we = rng.uniform(0.1, 3.0, len(pairs))
    pinned = np.zeros(n, bool)
    pinned[0] = True
    S, d = ra.laplacian(pairs, we, valid, pinned, n)
    b = rng.normal(size=(n, 3))
    b[pinned] = 0.0
    x, k, rej = ra.pcg(S, d, b, TIGHT, 500)
    ref = np.stack([spsolve(S.tocsc(), b[:, c]) for c in range(3)], 1)
    assert not rej and k < 500
    assert np.abs(x - ref).max() <= 1e-10 * np.abs(ref).max()


def _gm_total(pairs, Re, R, valid, sig2):
    _, th = ra.residuals(pairs, Re, R, valid)
    return ra.gm_cost(th[valid], sig2)


def test_fixed_point_is_stationary_for_the_geman_mcclure_cost():
    pairs, Re, w, _ = planted(30, 60, 5, outliers=0.2)
    sigma = math.radians(5.0)
    out = ra.average_rotations(pairs, Re, 30, weights=w, sigma=sigma, step_tol=1e-13, max_iters=2000, cg_tol=TIGHT)
    assert out["iters"][1] < 2000
    valid = np.ones(len(pairs), bool)
    sig2 = sigma * sigma
    h = 1e-6

    def grad(R):
        g = np.zeros((30, 3))
        for v in range(1, 30):
            for k in range(3):
                e = np.zeros(3)
                e[k] = h
                Rp, Rm = R.copy(), R.copy()
                Rp[v] = R[v] @ ra.expmap(e)
                Rm[v] = R[v] @ ra.expmap(-e)
                g[v, k] = (_gm_total(pairs, Re, Rp, valid, sig2) - _gm_total(pairs, Re, Rm, valid, sig2)) / (2 * h)
        return g
    g1 = np.abs(grad(out["R"])).max()
    g0 = np.abs(grad(out["start"])).max()
    print("largest gradient component: %.3e at the start, %.3e at the fixed point" % (g0, g1))
    assert g1 <= 1e-6 * g0 and g1 <= 1e-7


def test_planted_recovery_oracle():
    pairs, Re, w, R = planted(200, 800, 6, outliers=0.2)
    out = ra.average_rotations(pairs, Re, 200, weights=w)
    e0 = np.degrees(gauge_errors(out["start"], R))
    e1 = np.degrees(gauge_errors(out["R"], R))
    print("200 views: median error %.3f -> %.3f deg, largest %.3f -> %.3f deg, iterations %s, CG %d"
          % (np.median(e0), np.median(e1), e0.max(), e1.max(), out["iters"], out["cg_iters"]))
    # measured with this seed: median 7.68 -> 0.78 deg, largest 14.1 -> 1.94 deg, with 1 deg of edge noise per axis
    # (1.6 deg in angle on average)
    assert np.median(e1) < 1.0 and e1.max() < 2.5
    assert np.median(e1) < np.median(e0) and e1.max() < e0.max()
    assert (out["component"] == 0).all() and out["iters"][0] == 5


def test_relabelling_changes_nothing():
    pairs, Re, w, _ = planted(40, 100, 7, outliers=0.2)
    base = ra.average_rotations(pairs, Re, 40, weights=w)
    rng = np.random.default_rng(7)
    perm = rng.permutation(len(pairs))
    rev = rng.random(len(pairs)) < 0.5
    p2, R2 = pairs[perm].copy(), Re[perm].copy()
    p2[rev[perm]] = p2[rev[perm]][:, ::-1]
    R2[rev[perm]] = np.swapaxes(R2[rev[perm]], 1, 2)
    got = ra.average_rotations(p2, R2, 40, weights=w[perm])
    assert (got["iters"] == base["iters"]).all()
    assert np.abs(got["R"] - base["R"]).max() <= 1e-12
    assert np.abs(got["residual"] - base["residual"][perm]).max() <= 1e-12


# ------------------------------------------------------------------------------------------------ host build (CPU)
def test_host_build_matches_the_oracle(tmp_path):
    so = os.path.join(str(tmp_path), "librotation_averaging_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-o", so, os.path.join(ROOT, "tests", "rotation_averaging_host.cpp")])
    L = ctypes.CDLL(so)
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))  # noqa: E731
    ip = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))  # noqa: E731
    rng = np.random.default_rng(8)
    n = 500
    A, B, C = rand_rot(rng, n), rand_rot(rng, n), rand_rot(rng, n)
    # every branch of the log map among the inputs
    axes = rng.normal(size=(n, 3))
    axes /= np.linalg.norm(axes, axis=1)[:, None]
    t = np.r_[np.zeros(20), rng.uniform(0, 1e-4, 80), rng.uniform(0, math.pi, 300), math.pi - rng.uniform(0, 1e-3, 80),
              np.full(20, math.pi)]
    D = np.ascontiguousarray(rot_exp(t[:, None] * axes))
    r, th = np.zeros((n, 3)), np.zeros(n)
    L.rah_log(n, dp(D), dp(r), dp(th))
    rr, tt = ra.log_map(D)
    assert np.abs(r - rr).max() <= 1e-15 * math.pi and np.abs(th - tt).max() <= 1e-15
    dR = np.zeros((n, 3, 3))
    L.rah_relative(n, dp(A), dp(B), dp(C), dp(dR))
    assert np.abs(dR - ra.mul_tn(B, ra.mul(C, A))).max() <= 1e-15
    cj = (rng.random(n) < 0.5).astype(np.intc)
    Rc = np.zeros((n, 3, 3))
    L.rah_compose(n, dp(A), dp(B), ip(cj), dp(Rc))
    assert np.abs(Rc - np.where(cj[:, None, None] == 1, ra.mul(A, B), ra.mul_tn(A, B))).max() <= 1e-15
    for phase in (0, 1):
        w = np.zeros(n)
        L.rah_weight(n, phase, dp(th), ctypes.c_double(0.01), dp(w))
        assert np.abs(w - ra.weight(phase, th, 0.01)).max() <= 1e-15 * np.abs(w).max()
    om = np.ascontiguousarray(rng.normal(size=(n, 3)) * np.r_[0.0, 1e-9, 1e-3, 0.3, 2.0].repeat(n // 5)[:, None])
    R2 = np.zeros((n, 3, 3))
    L.rah_update(n, dp(A), dp(om), dp(R2))
    assert np.abs(R2 - ra.update(A, om)).max() <= 1e-15
    # preparation: drifting, failed (R = 0), mirrored and non-finite rotations
    P = np.ascontiguousarray(np.r_[A[:40] + 1e-9 * rng.normal(size=(40, 3, 3)), np.zeros((5, 3, 3)), -A[40:45],
                                   np.full((5, 3, 3), np.nan), A[45:50]])
    ok = np.zeros(len(P), np.intc)
    Q = P.copy()
    L.rah_prepare(len(P), dp(Q), ip(ok))
    okr = ra.edge_ok(P)
    assert (ok.astype(bool) == okr).all() and okr.sum() == 45
    ref = ra.orthonormalise(P[okr])
    keep = ra.drift(P[okr]) <= ra.ORTHO_TOL
    ref[keep] = P[okr][keep]
    assert np.abs(Q[okr] - ref).max() <= 1e-15


# ------------------------------------------------------------------------------------------------ arguments (CPU)
def test_python_messages():
    torch = pytest.importorskip("torch")
    from pydegensac_b200.matching import average_rotations
    f64, i32 = torch.float64, torch.int32
    good = dict(pairs=[[0, 1], [1, 2]], R_rel=torch.eye(3, dtype=f64).repeat(2, 1, 1), n_views=3)
    host = "R_rel and mask must be CUDA tensors on one device"
    cases = [
        ({"n_views": 0}, "n_views must be at least 1, not 0"),
        ({"pairs": [[0, 3]]}, "pairs: image index out of range"),
        ({"pairs": np.zeros((0, 2))}, "pairs must be a non-empty [P,2] array of (query image, train image)"),
        ({"R_rel": np.eye(3)}, "R_rel must be a torch tensor"),
        ({"R_rel": torch.eye(3, dtype=f64).repeat(2, 1)}, "R_rel must be [P,3,3] or [P,9] with P >= 1, not [6, 3]"),
        ({"R_rel": torch.eye(3, dtype=f64).repeat(3, 1, 1)}, "R_rel must hold one rotation per pair (2), not 3"),
        ({"R_rel": torch.zeros((2, 9), dtype=i32)}, "R_rel must be a floating tensor, not torch.int32"),
        ({"mask": torch.ones(3, dtype=torch.bool)}, "mask must be [P] = [2], not [3]"),
        ({"mask": torch.ones(2, dtype=i32)}, "mask must be bool or uint8, not torch.int32"),
        ({"weights": [1, 2]}, "weights must be a torch tensor"),
        ({"weights": torch.ones(3, dtype=i32)}, "weights must be [P] = [2], not [3]"),
        ({"weights": torch.ones(2, dtype=torch.int64)}, "weights must be int32, not torch.int64"),
        ({"sigma": 0.0}, "sigma must be a positive number, not 0.0"),
        ({"sigma": float("inf")}, "sigma must be a positive number, not inf"),
        ({"l1_iters": -1}, "l1_iters must not be negative, not -1"),
        ({"max_iters": -2}, "max_iters must not be negative, not -2"),
        ({"step_tol": -1e-6}, "step_tol must be a non-negative finite number, not -1e-06"),
        ({"step_tol": float("nan")}, "step_tol must be a non-negative finite number, not nan"),
        ({"cg_max_iters": 0}, "cg_max_iters must be at least 1, not 0"),
        ({"cg_tol": float("inf")}, "cg_tol must be a non-negative finite number, not inf"),
        ({"weights": torch.ones(2, dtype=i32)}, "R_rel, weights and mask must be CUDA tensors on one device"),
        ({"l1_iters": 0, "max_iters": 0, "step_tol": 0.0, "cg_tol": 0.0}, host),
        ({"R_rel": torch.eye(3, dtype=torch.float32).repeat(2, 1, 1).view(2, 9)}, host),
        ({}, host),
    ]
    for kw, msg in cases:
        with pytest.raises(ValueError) as e:
            average_rotations(**dict(good, **kw))
        assert str(e.value) == msg, kw


def test_c_entry_point_refuses_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["R_rel", "R_out", "component", "residual", "iters", "cg_iters"]

    def call(pairs=((0, 1), (1, 2)), n_pairs=None, n_views=3, sigma=0.1, l1_iters=5, max_iters=100, step_tol=1e-6,
             cg_max_iters=500, cg_tol=1e-6, null=()):
        b = {k: (None if k in null else fake) for k in names}
        flat = [v for p in pairs for v in p]
        hp = (ctypes.c_int32 * max(len(flat), 1))(*flat)
        return L.dgb200_average_rotations_dev(
            None if "pairs" in null else hp, len(pairs) if n_pairs is None else n_pairs, n_views, b["R_rel"], None,
            None, ctypes.c_double(sigma), l1_iters, max_iters, ctypes.c_double(step_tol), cg_max_iters,
            ctypes.c_double(cg_tol), b["R_out"], b["component"], b["residual"], b["iters"], b["cg_iters"], None)

    sizes = "need n_views >= 1 and n_pairs >= 1"
    cases = [(dict(null={k}), "null buffer") for k in names]
    cases += [
        (dict(n_views=0), sizes), (dict(n_pairs=0), sizes), (dict(null={"pairs"}), "null pair table"),
        (dict(pairs=((0, 3),)), "pair view index out of range"), (dict(pairs=((-1, 1),)), "pair view index out of range"),
        (dict(sigma=0.0), "sigma must be a positive finite number"),
        (dict(sigma=float("nan")), "sigma must be a positive finite number"),
        (dict(sigma=float("inf")), "sigma must be a positive finite number"),
        (dict(l1_iters=-1), "l1_iters and max_iters must not be negative"),
        (dict(max_iters=-1), "l1_iters and max_iters must not be negative"),
        (dict(step_tol=-1.0), "step_tol must be a non-negative finite number"),
        (dict(step_tol=float("inf")), "step_tol must be a non-negative finite number"),
        (dict(cg_max_iters=0), "cg_max_iters must be at least 1"),
        (dict(cg_tol=float("nan")), "cg_tol must be a non-negative finite number"),
        (dict(cg_tol=-1.0, cg_max_iters=0), "cg_max_iters must be at least 1"),
    ]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert L.dgb200_rotation_averaging_last_error().decode() == msg, kw


# ------------------------------------------------------------------------------------------------ GPU
def _graphs():
    """(name, pairs, R_rel, n_views, mask, weights) over every kind of input the estimator distinguishes"""
    out = []
    p, R, w, _ = planted(25, 0, 10)
    out.append(("chain", p, R, 25, None, w))
    p, R, w, _ = planted(12, 0, 11, chain=False)
    p = np.array([(i, j) for i in range(12) for j in range(12) if i < j], np.int32)
    Rt = rand_rot(np.random.default_rng(11), 12)
    R = rot_exp(np.radians(2.0) * np.random.default_rng(12).normal(size=(len(p), 3))) @ \
        np.einsum("pij,pkj->pik", Rt[p[:, 1]], Rt[p[:, 0]])
    out.append(("dense", p, R, 12, None, None))
    p1, R1, w1, _ = planted(15, 20, 13, outliers=0.2)
    p2, R2, w2, _ = planted(10, 10, 14, outliers=0.2)
    out.append(("components and isolated views", np.r_[p1 + 3, p2 + 21].astype(np.int32), np.r_[R1, R2], 35, None,
                np.r_[w1, w2]))
    p, R, w, _ = planted(20, 40, 15, outliers=0.1)
    R = R.copy()
    m = np.ones(len(p), bool)
    m[3] = False                      # masked
    R[5, 0, 0] = np.nan               # not finite
    R[7] = 0.0                        # a failed pose (det 0)
    R[9] = -R[9]                      # det -1
    w = w.copy()
    w[11] = -1                        # negative weight
    p = p.copy()
    p[13] = (4, 4)                    # self-pair
    R[15] += 1e-7                     # drifts: re-orthonormalised
    out.append(("dropped edges", p, R, 20, m, w))
    p, R, w, _ = planted(15, 20, 16, outliers=0.1)
    dup = np.r_[p, p[:6], p[6:12, ::-1]].astype(np.int32)
    Rd = np.r_[R, R[:6], np.swapaxes(R[6:12], 1, 2)]
    wd = np.r_[w, w[:6], w[6:12]]     # ties, broken by the edge index
    out.append(("duplicate and reversed edges", dup, Rd, 15, None, wd))
    return out


def _run(pairs, R_rel, n_views, mask=None, weights=None, **kw):
    import torch
    from pydegensac_b200.matching import average_rotations
    dev = torch.device("cuda:0")
    m = torch.from_numpy(np.asarray(mask)).to(dev) if mask is not None else None
    w = torch.from_numpy(np.asarray(weights, np.int32)).to(dev) if weights is not None else None
    out = average_rotations(pairs, torch.from_numpy(np.ascontiguousarray(R_rel)).to(dev), n_views, mask=m, weights=w,
                            **kw)
    return {k: getattr(out, k).cpu().numpy() for k in out._fields}


def _close(a, b, tol):
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.nan_to_num(np.abs(a - b)).max() <= tol


@pytest.mark.gpu
def test_start_equals_the_oracle_tree():
    for name, p, R, n, m, w in _graphs():
        g = _run(p, R, n, m, w, l1_iters=0, max_iters=0)
        o = ra.average_rotations(p, R, n, m, w, l1_iters=0, max_iters=0)
        assert _close(g["R"], o["R"], 1e-14), name
        assert (g["component"] == o["component"]).all(), name
        assert _close(g["residual"], o["residual"], 1e-14), name
        assert (g["iters"] == 0).all() and g["cg_iters"][0] == 0, name


@pytest.mark.gpu
def test_full_call_equals_the_oracle():
    for name, p, R, n, m, w in _graphs():
        g = _run(p, R, n, m, w, cg_tol=TIGHT)
        o = ra.average_rotations(p, R, n, m, w, cg_tol=TIGHT)
        print("%s: iterations %s (oracle %s), CG %d (oracle %d), largest |dR| %.2e"
              % (name, g["iters"], o["iters"], g["cg_iters"][0], o["cg_iters"], np.nanmax(np.abs(g["R"] - o["R"]))))
        assert (g["iters"] == o["iters"]).all(), name
        assert _close(g["R"], o["R"], 1e-9), name
        assert _close(g["residual"], o["residual"], 1e-9), name
        assert (g["component"] == o["component"]).all(), name


@pytest.mark.gpu
def test_same_bytes_on_a_rerun():
    name, p, R, n, m, w = _graphs()[2]
    a = _run(p, R, n, m, w)
    b = _run(p, R, n, m, w)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    assert (a["component"][:3] == -1).all() and np.isnan(a["R"][:3]).all()


@pytest.mark.gpu
def test_planted_recovery_device():
    pairs, Re, w, R = planted(200, 800, 6, outliers=0.2)
    g = _run(pairs, Re, 200, weights=w)
    o = ra.average_rotations(pairs, Re, 200, weights=w)
    e1 = np.degrees(gauge_errors(g["R"], R))
    print("device: median error %.3f deg, largest %.3f deg, iterations %s (oracle %s)"
          % (np.median(e1), e1.max(), g["iters"], o["iters"]))
    assert (g["iters"] == o["iters"]).all() and np.abs(g["R"] - o["R"]).max() <= 1e-9
    assert np.median(e1) < 1.0 and e1.max() < 2.5


@pytest.mark.gpu
def test_example_pipeline_without_a_host_read():
    import sys
    import torch
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import gpu_pipeline
    from pydegensac_b200.scenes import _K
    dev = torch.device("cuda:0")
    K = torch.from_numpy(_K).to(dev)
    scene = gpu_pipeline.view_graph_scene(dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = gpu_pipeline.view_graph_rotations(dev, K, scene)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    e0, e1 = gpu_pipeline.report_view_graph(scene, out)
    assert e1 < 0.5 and e1 < e0


@pytest.mark.gpu
def test_ten_thousand_views_match_the_oracle():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from rotation_averaging_rate import synth
    pairs, Re, w, R = synth(10000, 200000, 0)
    g = _run(pairs, Re, 10000, weights=w)
    o = ra.average_rotations(pairs, Re, 10000, weights=w)
    d = np.abs(g["R"] - o["R"]).max()
    print("10^4 views: iterations %s (oracle %s), CG %d (oracle %d), largest |dR| %.2e"
          % (g["iters"], o["iters"], g["cg_iters"][0], o["cg_iters"], d))
    assert (g["component"] == 0).all()
    assert d <= 1e-8
