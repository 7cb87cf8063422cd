"""matching.bundle_adjust_pcg_ragged: Levenberg-Marquardt over any number of cameras, the reduced camera system solved
by preconditioned conjugate gradients on the implicit Schur complement.
CPU: the oracle (tests/bundle_adjust_pcg_np.py) against the dense oracle (tests/bundle_adjust_np.py) -- its matrix-free
S p, its step at a tight tolerance and its whole call -- its two tolerances on a 150-camera scene, the host build of
the new per-thread functions, and the argument checks of the Python wrapper and the C entry point.  GPU: the kernel
against the oracle and against bundle_adjust_ragged, beyond the dense limit, determinism and pass-through, edge cases
and a pipeline without a host synchronisation."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import bundle_adjust_np as o
from tests import bundle_adjust_pcg_np as q
from tests.test_bundle_adjust import _rot_err, scene
from tests.test_triangulate import _point, rig, track

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")
TIGHT = 1e-14


def _dense_s(P, lin, lam, absolute=False):
    """S of bundle_adjust_np.schur_step, restricted to the kept coordinates (absolute: with |V*^-1| and the two terms
    added, for the scale of the rounding error of S p)"""
    nf = len(P["free"])
    Vi = np.zeros_like(lin["V"])
    for j in np.flatnonzero(P["opt"]):
        Vi[j] = o.inv3(lin["V"][j], lam)
    if absolute:
        Vi = np.abs(Vi)
    Y = np.einsum("apkl,plm->apkm", lin["W"], Vi)
    S = o._blockdiag(o._damp(lin["U"], lam)) + (1 if absolute else -1) * np.einsum(
        "apkm,bplm->akbl", Y, lin["W"]).reshape(6 * nf, 6 * nf)
    keep = o._keep(P)
    return S[np.ix_(keep, keep)], keep


def _schur_problem():
    cams, pts, K, off, _, (R0, t0, X0) = scene(6, 40, 3, outliers=0.1)
    # camera 4 sees no used observation: its slot is inactive
    m = cams != 4
    return dict(cams=cams, pts=pts, R=R0, t=t0, K=K, offsets=off, X=X0, mask=m, loss_scale=2.0)


# ------------------------------------------------------------------------------------------------ oracle (CPU)
@pytest.mark.parametrize("lam", [0.0, 1e-3, 1.0, 100.0])
def test_matrix_free_product_equals_the_dense_schur_complement(lam):
    a = _schur_problem()
    P = o.setup(**a)
    assert P["hold"] is not None and not P["active"].all()
    dense = o.linearise(P, P["R"], P["t"], P["X"])
    lin = q.linearise(P, P["R"], P["t"], P["X"])
    Vi = q.point_inverses(P, lin, lam)
    S, keep = _dense_s(P, dense, lam)
    Sa = _dense_s(P, dict(dense, U=np.abs(dense["U"]), W=np.abs(dense["W"])), lam, absolute=True)[0]
    rng = np.random.default_rng(5)
    for _ in range(3):
        p = rng.normal(size=6 * len(P["free"]))
        p[~keep] = 0.0
        got = q.schur_matvec(P, lin, Vi, lam, p)
        ref = S @ p[keep]
        # relative to the terms summed in S p, |U*| |p| + |W| |V*^-1| |W^T| |p|: at lambda = 0 the product is far
        # smaller than they are
        assert np.abs(got[keep] - ref).max() <= 1e-12 * (Sa @ np.abs(p[keep])).max(), lam
        assert (got[~keep] == 0.0).all()


def test_tight_pcg_step_equals_the_schur_step():
    a = _schur_problem()
    P = o.setup(**a)
    dense = o.linearise(P, P["R"], P["t"], P["X"])
    lin = q.linearise(P, P["R"], P["t"], P["X"])
    nf = len(P["free"])
    for lam in (0.0, 1e-3, 1.0, 100.0):
        (dc, dX), k = q.pcg_step(P, lin, lam, TIGHT, 6 * nf)
        ec, eX = o.schur_step(P, dense, lam)
        # undamped, S is nearly singular along the scale that the gauge barely holds: both solves lose digits there
        tol = 1e-9 if lam > 0.0 else 1e-8
        assert np.abs(dc - ec).max() <= tol * np.abs(ec).max(), lam
        assert np.abs(dX - eX).max() <= tol * np.abs(eX).max(), lam
        assert dc[P["hold"]] == 0.0 and 1 <= k <= 6 * nf


@pytest.mark.parametrize("loss_scale", [None, 1.0])
def test_tight_whole_call_equals_the_dense_oracle(loss_scale):
    cams, pts, K, off, _, (R0, t0, X0) = scene(8, 60, 18)
    kw = dict(free=list(range(1, 8)), scale_gauge=1, loss_scale=loss_scale, max_iters=50)
    ref = o.bundle_adjust(cams, pts, R0, t0, K, off, X0, **kw)
    got = q.bundle_adjust_pcg(cams, pts, R0, t0, K, off, X0, cg_tol=TIGHT, cg_max_iters=6 * 7, **kw)
    assert got["iters"] == ref["iters"]
    assert abs(got["cost"] - ref["cost"]) <= 1e-10 * ref["cost"]
    for k in ("R", "t", "X"):
        assert np.abs(got[k] - ref[k]).max() <= 1e-8 * max(1.0, np.abs(ref[k]).max()), k
    assert (got["mask"] == ref["mask"]).all() and got["n_used"] == ref["n_used"]


def test_default_tolerance_reaches_the_tight_optimum_at_150_cameras():
    # tracks over random sets of up to 12 of the 150 cameras.  (Over runs of consecutive cameras along the line, the
    # scene's bending is so weakly held that inexact steps at cg_tol 0.1 approach the optimum linearly and do not
    # meet the 1e-12 stopping rule within 60 steps, while exact steps do in 10: see the PR's measurements.)
    cams, pts, K, off, _, (R0, t0, X0) = scene(150, 1500, 7, lmax=12)
    P = o.setup(cams, pts, R0, t0, K, off, X0)
    kw = dict(max_iters=200, P=P)
    loose = q.bundle_adjust_pcg(cams, pts, R0, t0, K, off, X0, **kw)
    tight = q.bundle_adjust_pcg(cams, pts, R0, t0, K, off, X0, cg_tol=TIGHT, cg_max_iters=6 * 149, **kw)
    print("150 cameras: cost %.10e (cg_tol 0.1, %d steps, %d CG) vs %.10e (tight, %d steps, %d CG)"
          % (loose["cost"], loose["iters"], loose["cg_iters"], tight["cost"], tight["iters"], tight["cg_iters"]))
    assert loose["iters"] < 200 and tight["iters"] < 200
    assert abs(loose["cost"] - tight["cost"]) <= 1e-8 * tight["cost"]
    assert loose["cost"] < loose["cost0"]


# ------------------------------------------------------------------------------------------------ host build (CPU)
def test_host_build_of_the_preconditioner_cholesky(tmp_path):
    so = os.path.join(str(tmp_path), "libbundle_adjust_pcg_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-o", so, os.path.join(ROOT, "tests", "bundle_adjust_pcg_host.cpp")])
    L = ctypes.CDLL(so)
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))  # noqa: E731
    rng = np.random.default_rng(9)
    iu = np.triu_indices(6)
    il = np.tril_indices(6)
    for _ in range(50):
        B = rng.normal(size=(6, 6))
        A = B @ B.T + 0.1 * np.eye(6)
        up = np.ascontiguousarray(A[iu])
        Lp = np.zeros(21)
        b = rng.normal(size=6)
        x = np.zeros(6)
        assert L.pcgh_solve(dp(up), dp(Lp), dp(b), dp(x)) == 1
        ref = np.linalg.cholesky(A)
        assert np.abs(Lp - ref[il]).max() <= 1e-12 * np.abs(ref).max()
        assert np.abs(x - np.linalg.solve(A, b)).max() <= 1e-10 * np.abs(np.linalg.solve(A, b)).max()
    A = np.eye(6)
    A[3, 3] = -1.0
    assert L.pcgh_solve(dp(np.ascontiguousarray(A[iu])), dp(np.zeros(21)), dp(np.ones(6)), dp(np.zeros(6))) == 0


# ------------------------------------------------------------------------------------------------ arguments (CPU)
def _raises(fn, args, message):
    with pytest.raises(ValueError) as e:
        fn(**args)
    assert str(e.value) == message


def test_python_messages():
    torch = pytest.importorskip("torch")
    from pydegensac_b200.matching import bundle_adjust_pcg_ragged
    f64, i32 = torch.float64, torch.int32
    good = dict(cams=torch.zeros(10, dtype=i32), pts=torch.zeros((10, 2), dtype=f64),
                R=torch.eye(3, dtype=f64).repeat(4, 1, 1), t=torch.zeros((4, 3), dtype=f64), K=torch.eye(3, dtype=f64),
                offsets=torch.tensor([0, 4, 10], dtype=i32), X=torch.zeros((2, 3), dtype=f64))
    host = "cams, pts, R, t, K, offsets, X and mask must be CUDA tensors on one device"
    cases = [
        ({"cams": np.zeros(10, np.int32)}, "cams must be a torch tensor"),
        ({"offsets": torch.tensor([0, 4, 10])}, "offsets must be int32, not torch.int64"),
        ({"X": torch.zeros((3, 3), dtype=f64)}, "X must be [T,3] = [2,3], not [3, 3]"),
        ({"mask": torch.ones(9, dtype=torch.bool)}, "mask must be [obs] = [10], not [9]"),
        ({"free": [1, 1]}, "free holds a camera twice"),
        ({"free": [4]}, "free holds a camera index outside [0, 4)"),
        ({"free": "x"}, "free must be a host sequence of camera indices"),
        ({"scale_gauge": 0}, "scale_gauge 0 is not one of the free cameras"),
        ({"scale_gauge": "first"}, "scale_gauge must be 'auto', None or a camera of free, not 'first'"),
        ({"free": [0, 1, 2, 3], "scale_gauge": 1}, "scale_gauge needs a held camera: every camera is free"),
        ({"loss_scale": 0.0}, "loss_scale must be a positive number or None, not 0.0"),
        ({"max_iters": -1}, "max_iters must not be negative, not -1"),
        ({"px_th": 0.0}, "px_th must be a positive number, not 0.0"),
        ({"cg_max_iters": 0}, "cg_max_iters must be at least 1, not 0"),
        ({"cg_max_iters": 0, "px_th": 0.0}, "px_th must be a positive number, not 0.0"),
        ({"cg_tol": -0.1}, "cg_tol must be a non-negative finite number, not -0.1"),
        ({"cg_tol": float("nan")}, "cg_tol must be a non-negative finite number, not nan"),
        ({"cg_tol": float("inf")}, "cg_tol must be a non-negative finite number, not inf"),
        ({"cg_tol": -1.0, "cg_max_iters": 0}, "cg_max_iters must be at least 1, not 0"),
        # no camera limit: 65 free cameras, or free=None over 66 cameras, pass the checks
        ({"R": torch.eye(3, dtype=f64).repeat(66, 1, 1), "t": torch.zeros((66, 3), dtype=f64)}, host),
        ({"R": torch.eye(3, dtype=f64).repeat(66, 1, 1), "t": torch.zeros((66, 3), dtype=f64),
          "free": list(range(65))}, host),
        ({"cg_tol": 0.0, "cg_max_iters": 1}, host),
        ({}, host),
    ]
    for kw, msg in cases:
        _raises(bundle_adjust_pcg_ragged, dict(good, **kw), msg)


def test_c_entry_point_refuses_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["cams", "pts", "R", "t", "K", "offsets", "X", "mask", "R_out", "t_out", "X_out", "mask_out", "cost0",
             "cost", "iters", "n_used", "cg_iters"]

    def call(n_cams=4, n_tracks=3, obs=10, free=(1, 2, 3), gauge=1, loss_scale=0.0, max_iters=10, px_th=2.0,
             cg_max_iters=10, cg_tol=0.1, n_free=None, null=()):
        b = {k: (None if k in null else fake) for k in names}
        hf = (ctypes.c_int32 * max(len(free), 1))(*free)
        return L.dgb200_bundle_adjust_pcg_ragged_dev(
            b["cams"], b["pts"], b["R"], b["t"], b["K"], 0, n_cams, b["offsets"], n_tracks, obs, b["X"], b["mask"],
            None if null == "free" else hf, len(free) if n_free is None else n_free, gauge,
            ctypes.c_double(loss_scale), max_iters, ctypes.c_double(px_th), cg_max_iters, ctypes.c_double(cg_tol),
            b["R_out"], b["t_out"], b["X_out"], b["mask_out"], b["cost0"], b["cost"], b["iters"], b["n_used"],
            b["cg_iters"], None)

    sizes = "need n_tracks >= 1, obs >= 0 and n_cams >= 1"
    cases = [(dict(null={k}), "null buffer") for k in names if k not in ("cams", "pts", "mask", "mask_out")]
    cases += [(dict(null={k}), "null observation buffer") for k in ("cams", "pts", "mask_out")]
    cases += [
        (dict(null={"cams"}, obs=0, n_tracks=0), sizes),
        (dict(n_tracks=0), sizes), (dict(obs=-1), sizes), (dict(n_cams=0), sizes),
        (dict(n_free=-1), "n_free must lie in [0, n_cams]"), (dict(n_free=5), "n_free must lie in [0, n_cams]"),
        (dict(null="free"), "null free-camera list"),
        (dict(free=(1, 1)), "free camera index repeated"), (dict(free=(1, 4)), "free camera index out of range"),
        (dict(free=(-1, 2)), "free camera index out of range"), (dict(free=(2, 5, 2)), "free camera index out of range"),
        (dict(gauge=0), "scale_gauge must be one of the free cameras"),
        (dict(gauge=-2), "scale_gauge must be a free camera or -1"),
        (dict(free=(0, 1, 2, 3), gauge=1), "scale_gauge needs a held camera"),
        (dict(loss_scale=-1.0), "loss_scale must be a positive number (or 0 for the trivial loss)"),
        (dict(loss_scale=float("nan")), "loss_scale must be a positive number (or 0 for the trivial loss)"),
        (dict(loss_scale=float("inf")), "loss_scale must be a positive number (or 0 for the trivial loss)"),
        (dict(max_iters=-1), "max_iters must not be negative"),
        (dict(px_th=0.0), "px_th must be a positive number"), (dict(px_th=float("nan")), "px_th must be a positive number"),
        (dict(cg_max_iters=0), "cg_max_iters must be at least 1"),
        (dict(cg_max_iters=0, px_th=0.0), "px_th must be a positive number"),
        (dict(cg_tol=-1.0), "cg_tol must be a non-negative finite number"),
        (dict(cg_tol=float("nan")), "cg_tol must be a non-negative finite number"),
        (dict(cg_tol=float("inf")), "cg_tol must be a non-negative finite number"),
        (dict(cg_tol=float("inf"), cg_max_iters=0), "cg_max_iters must be at least 1"),
    ]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert L.dgb200_bundle_adjust_pcg_last_error().decode() == msg, kw
    # 64 free cameras of 65 and all 70 of 70 without a gauge are no longer refused for their number: a refusal
    # further on (the null output) shows they passed
    assert call(n_cams=70, free=tuple(range(70)), gauge=-1, null={"cost"}) == -1
    assert L.dgb200_bundle_adjust_pcg_last_error().decode() == "null buffer"


# ------------------------------------------------------------------------------------------------ GPU
def _dev(*xs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0") for a in xs]


def _np(res):
    return {k: getattr(res, k).cpu().numpy() for k in res._fields}


def _run(cams, pts, R, t, K, off, X, mask=None, dense=False, **kw):
    from pydegensac_b200.matching import bundle_adjust_pcg_ragged, bundle_adjust_ragged
    d = _dev(cams, pts, R, t, K, off, X)
    m = _dev(mask)[0] if mask is not None else None
    return _np((bundle_adjust_ragged if dense else bundle_adjust_pcg_ragged)(*d, mask=m, **kw))


@pytest.mark.gpu
@pytest.mark.parametrize("loss_scale", [None, 1.0])
def test_kernel_against_the_oracle_and_the_dense_entry(loss_scale):
    cams, pts, K, off, (R, t, X), (R0, t0, X0) = scene(12, 2000, 41, noise=0.5, outliers=0.1)
    kw = dict(free=list(range(1, 12)), scale_gauge=1, loss_scale=loss_scale, max_iters=50, px_th=2.0)
    g = _run(cams, pts, R0, t0, K, off, X0, **kw)
    ref = q.bundle_adjust_pcg(cams, pts, R0, t0, K, off, X0, **kw)
    dc = abs(g["cost"][0] - ref["cost"]) / ref["cost"]
    print("loss %s: cost %.9e -> %.9e (oracle %.9e), %d steps (oracle %d), %d CG (oracle %d)"
          % (loss_scale, g["cost0"][0], g["cost"][0], ref["cost"], g["iters"][0], ref["iters"], g["cg_iters"][0],
             ref["cg_iters"]))
    assert abs(g["cost0"][0] - ref["cost0"]) <= 1e-12 * ref["cost0"] and g["n_used"][0] == ref["n_used"]
    assert dc <= 1e-9 and np.abs(g["R"] - ref["R"]).max() <= 1e-8 and np.abs(g["t"] - ref["t"]).max() <= 1e-8
    assert g["cost"][0] <= g["cost0"][0]
    # at a tight tolerance the step is the exact LM step: the dense entry point's result
    tight = _run(cams, pts, R0, t0, K, off, X0, cg_tol=1e-12, cg_max_iters=66, **kw)
    dense = _run(cams, pts, R0, t0, K, off, X0, dense=True, **kw)
    print("tight: cost %.12e in %d steps, dense %.12e in %d" % (tight["cost"][0], tight["iters"][0], dense["cost"][0],
                                                                dense["iters"][0]))
    assert abs(tight["cost"][0] - dense["cost"][0]) <= 1e-9 * dense["cost"][0]
    assert np.abs(tight["R"] - dense["R"]).max() <= 1e-8 and np.abs(tight["t"] - dense["t"]).max() <= 1e-8


def window_scene(C, T, seed, window=12, lmax=8):
    """T tracks of 2 .. lmax cameras drawn from a window of `window` consecutive cameras of a rig of C cameras along a
    line (local covisibility), the planted (R, t, X) and a start perturbed as tests.test_bundle_adjust.scene does"""
    rng = np.random.default_rng(seed)
    R, t, K = rig(C, seed)
    cs, xs, Xs = [], [], []
    for _ in range(T):
        L = int(rng.integers(2, lmax + 1))
        a = int(rng.integers(0, C - window + 1))
        cams = np.sort(rng.choice(np.arange(a, a + window), L, replace=False))
        X = _point(R, t, cams, rng)
        cs.append(cams.astype(np.int32)); xs.append(track(R, t, K, cams, X, 0.5, np.zeros(L, bool), rng))
        Xs.append(X)
    off = np.zeros(T + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in cs])
    X = np.array(Xs)
    R0, t0 = R.copy(), t.copy()
    for c in range(1, C):
        R0[c] = o.expmap(2e-3 * rng.normal(size=3)) @ R[c]
        t0[c] = t[c] + 1e-2 * rng.normal(size=3)
    return np.concatenate(cs), np.concatenate(xs), K, off, (R, t, X), (R0, t0, X + 2e-2 * rng.normal(size=X.shape))


@pytest.mark.gpu
def test_beyond_the_dense_limit():
    # 300 free cameras along a line, local tracks.  The same fixed number of trial steps on both sides: along a line
    # the inexact steps approach the optimum linearly, so the 1e-12 stopping rule is not what this test waits for
    cams, pts, K, off, (R, t, X), (R0, t0, X0) = window_scene(301, 30000, 8)
    kw = dict(max_iters=20)
    g = _run(cams, pts, R0, t0, K, off, X0, **kw)
    ref = q.bundle_adjust_pcg(cams, pts, R0, t0, K, off, X0, **kw)
    e0 = max(_rot_err(R0[c], R[c]) for c in range(301))
    e1 = max(_rot_err(g["R"][c], R[c]) for c in range(301))
    print("300 free cameras, %d observations: cost %.9e -> %.9e (oracle %.9e), %d steps (oracle %d), %d CG (oracle "
          "%d); rotation error %.2e -> %.2e rad" % (len(cams), g["cost0"][0], g["cost"][0], ref["cost"], g["iters"][0],
                                                    ref["iters"], g["cg_iters"][0], ref["cg_iters"], e0, e1))
    assert g["iters"][0] == ref["iters"]
    assert abs(g["cost"][0] - ref["cost"]) <= 1e-8 * ref["cost"]
    assert g["cost"][0] <= g["cost0"][0] and e1 * 2 <= e0


@pytest.mark.gpu
def test_same_bytes_on_a_rerun_pass_through_and_aliased_outputs():
    import torch
    from pydegensac_b200.matching import bundle_adjust_pcg_ragged
    cams, pts, K, off, _, (R0, t0, X0) = scene(10, 800, 42, outliers=0.1)
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
    assert a["cost"][0] < a["cost0"][0] and a["iters"][0] >= 1 and a["cg_iters"][0] >= 1
    # outputs that alias the inputs (R, t, X written over R0, t0, X0): the same result
    from pydegensac_b200 import _cabi
    from pydegensac_b200.matching import _call
    cm, x, Rd, td, Kd, od, Xd = _dev(cams, pts, R0, t0, K, off, X0)
    dev = Rd.device
    mo = torch.empty(len(cams), dtype=torch.uint8, device=dev)
    s1 = [torch.empty(1, dtype=torch.float64, device=dev) for _ in range(2)]
    s2 = [torch.empty(1, dtype=torch.int32, device=dev) for _ in range(3)]
    hf = np.array(kw["free"], np.int32)
    L = _cabi.lib()
    _call(L.dgb200_bundle_adjust_pcg_ragged_dev, L.dgb200_bundle_adjust_pcg_last_error, dev, cm, x, Rd, td, Kd, 1, 10,
          od, len(off) - 1, len(cams), Xd, None, hf.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), len(hf), 4, 1.5, 30,
          2.0, 100, 0.1, Rd, td, Xd, mo, s1[0], s1[1], s2[0], s2[1], s2[2])
    for k, v in (("R", Rd), ("t", td), ("X", Xd), ("cost", s1[1]), ("cg_iters", s2[2])):
        assert v.cpu().numpy().tobytes() == a[k].tobytes(), k


@pytest.mark.gpu
def test_edge_cases():
    from pydegensac_b200.matching import build_tracks_ragged, bundle_adjust_pcg_ragged, trim_tracks  # noqa: F401
    cams, pts, K, off, _, (R0, t0, X0) = scene(6, 60, 44)
    # no free camera: structure only
    s = _run(cams, pts, R0, t0, K, off, X0, free=[])
    ref = q.bundle_adjust_pcg(cams, pts, R0, t0, K, off, X0, free=[])
    assert s["R"].tobytes() == R0.tobytes() and s["t"].tobytes() == t0.tobytes() and s["cg_iters"][0] == 0
    assert abs(s["cost"][0] - ref["cost"]) <= 1e-9 * ref["cost"] and s["iters"][0] == ref["iters"]
    # every camera free, no gauge
    e = _run(cams, pts, R0, t0, K, off, X0, free=list(range(6)), scale_gauge=None, max_iters=20)
    ref = q.bundle_adjust_pcg(cams, pts, R0, t0, K, off, X0, free=list(range(6)), scale_gauge=None, max_iters=20)
    assert abs(e["cost"][0] - ref["cost"]) <= 1e-9 * ref["cost"] and e["cost"][0] <= e["cost0"][0]
    # an unregistered camera in free, and malformed offsets: held, passed through, not optimised
    Ru, tu = R0.copy(), t0.copy()
    Ru[3], tu[3] = 0.0, 0.0
    bad = off.copy()
    bad[5] = bad[4] - 1
    u = _run(cams, pts, Ru, tu, K, bad, X0)
    ref = q.bundle_adjust_pcg(cams, pts, Ru, tu, K, bad, X0)
    assert u["R"][3].tobytes() == Ru[3].tobytes() and u["t"][3].tobytes() == tu[3].tobytes()
    assert u["X"][4].tobytes() == X0[4].tobytes() and not u["mask"][cams == 3].any()
    assert abs(u["cost"][0] - ref["cost"]) <= 1e-9 * ref["cost"]
    # max_iters = 0
    m0 = _run(cams, pts, R0, t0, K, off, X0, max_iters=0)
    assert m0["iters"][0] == 0 and m0["cost"][0] == m0["cost0"][0] and m0["X"].tobytes() == X0.tobytes()
    # the capacity-padded layout of build_tracks_ragged: empty tracks past the last one leave X unchanged
    T = len(off) - 1
    pad = np.r_[off, np.full(7, off[-1])].astype(np.int32)
    Xp = np.r_[X0, np.full((7, 3), np.nan)]
    p = _run(cams, pts, R0, t0, K, pad, Xp)
    assert np.array_equal(p["X"][T:], Xp[T:], equal_nan=True)
    assert abs(p["cost"][0] - q.bundle_adjust_pcg(cams, pts, R0, t0, K, off, X0)["cost"]) <= 1e-9 * p["cost"][0]


@pytest.mark.gpu
def test_pipeline_from_tracks_to_global_adjustment_without_sync():
    """ragged F RANSAC of synthetic matches, build_tracks_ragged, triangulate_tracks_ragged and the new entry point under
    torch.cuda.set_sync_debug_mode("error")"""
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import build_tracks_ragged, bundle_adjust_pcg_ragged, triangulate_tracks_ragged
    dev = torch.device("cuda:0")
    C, N = 8, 400
    rng = np.random.default_rng(3)
    R, t, K = rig(C, 3)
    Xw = np.array([_point(R, t, np.arange(C), rng) for _ in range(N)])
    kps = []
    for c in range(C):
        qq = (Xw @ R[c].T + t[c]) @ K[c].T
        kps.append(qq[:, :2] / qq[:, 2:] + 0.3 * rng.normal(size=(N, 2)))
    pairs = [(c, c + 1) for c in range(C - 1)] + [(c, c + 2) for c in range(C - 2)]
    idx = np.arange(N, dtype=np.int32)
    f64 = torch.float64
    p1 = torch.from_numpy(np.concatenate([kps[a] for a, _ in pairs])).to(dev)
    p2 = torch.from_numpy(np.concatenate([kps[b] for _, b in pairs])).to(dev)
    offsets = torch.arange(0, N * len(pairs) + 1, N, dtype=torch.int32, device=dev)
    i1 = torch.from_numpy(np.tile(idx, len(pairs))).to(dev)
    seeds = torch.arange(len(pairs), dtype=torch.int64, device=dev)
    kp_all = [torch.from_numpy(k).to(dev) for k in kps]
    Rd, td, Kd = (torch.from_numpy(a).to(dev) for a in (R, t, K))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        F, mask = pdg.findFundamentalMatrixBatch(p1, p2, 1.0, 0.999, 2000, seeds=seeds, offsets=offsets, n_max=N)
        ts = build_tracks_ragged([N] * C, pairs, i1, i1, offsets, mask, kps=kp_all)
        tr = triangulate_tracks_ragged(ts.cams, ts.pts, Rd, td, Kd, ts.offsets, px_th=2.0)
        Rp = Rd.clone()
        ba = bundle_adjust_pcg_ragged(ts.cams, ts.pts, Rp, td, Kd, ts.offsets, tr.X, mask=tr.mask, loss_scale=1.0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    print("pipeline: %d tracks, cost %.4f -> %.4f in %d steps, %d CG" % (int(ts.stats[0]), float(ba.cost0[0]),
                                                                      float(ba.cost[0]), int(ba.iters[0]),
                                                                      int(ba.cg_iters[0])))
    assert int(ts.stats[0]) >= 200 and float(ba.cost[0]) <= float(ba.cost0[0]) and int(ba.n_used[0]) > 1000
