"""matching.bundle_adjust_intrinsics_ragged and matching.undistort_points: bundle adjustment that also refines the
RADIAL intrinsics (f, cx, cy, k1, k2) of camera groups, and the undistortion through them.
CPU: the host build of csrc/camera_radial.h against central differences and the oracle
(tests/bundle_adjust_intrinsics_np.py); the oracle's matrix-free S p, tight PCG step and whole call against dense
forms, against the pose-only oracle and against scipy; the argument checks of both Python wrappers and both C entry
points; the new kernels' register report.  GPU: the kernel against the oracle, recovery of f and k1, agreement with
bundle_adjust_pcg_ragged, beyond 64 cameras, determinism and pass-through, the undistortion kernel, and a pipeline
without a host synchronisation."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from tests import bundle_adjust_intrinsics_np as q
from tests import bundle_adjust_np as o
from tests import bundle_adjust_pcg_np as pq
from tests.test_triangulate import _point, rig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")
TIGHT = 1e-14
FD = q.FOCAL | q.DISTORTION
ALL = q.FOCAL | q.PRINCIPAL_POINT | q.DISTORTION


def rscene(C, T, seed, groups=None, k=None, noise=0.5, lmax=12, f_err=0.0, perturb=1.0, zero_k=True):
    """T tracks of 2 .. min(lmax, C) cameras of tests.test_triangulate.rig's poses, observed through the RADIAL model
    with intrinsics k [G,5] by group (groups [C]); the planted (R, t, k, X) and a start with poses and points perturbed
    as tests.test_bundle_adjust.scene does, f scaled by 1 + f_err and (zero_k) k1 = k2 = 0.  Returns cams, pts, groups,
    offsets, planted (R, t, k, X), start (R, t, k, X)."""
    rng = np.random.default_rng(seed)
    R, t, _ = rig(C, seed)
    groups = np.zeros(C, np.int32) if groups is None else np.asarray(groups, np.int32)
    G = int(groups.max()) + 1
    if k is None:
        k = np.tile([520.0, 320.0, 240.0, -0.08, 0.01], (G, 1))
        k[:, 0] *= 1.0 + 0.05 * rng.uniform(-1, 1, G)
    k = np.asarray(k, np.float64)
    cs, xs, Xs = [], [], []
    for _ in range(T):
        L = int(rng.integers(2, min(lmax, C) + 1))
        cams = np.sort(rng.choice(C, L, replace=False))
        X = _point(R, t, cams, rng)
        p = np.einsum("cij,j->ci", R[cams], X) + t[cams]
        u = p[:, :2] / p[:, 2:]
        x = np.array([q.distort(k[groups[c]], u[i:i + 1])[0] for i, c in enumerate(cams)])
        cs.append(cams.astype(np.int32)); xs.append(x + noise * rng.normal(size=x.shape)); Xs.append(X)
    off = np.zeros(T + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in cs])
    X = np.array(Xs)
    R0, t0 = R.copy(), t.copy()
    for c in range(1, C):
        R0[c] = o.expmap(perturb * 2e-3 * rng.normal(size=3)) @ R[c]
        t0[c] = t[c] + perturb * 1e-2 * rng.normal(size=3)
    k0 = k.copy()
    k0[:, 0] *= 1.0 + f_err
    if zero_k:
        k0[:, 3:] = 0.0
    X0 = X + perturb * 2e-2 * rng.normal(size=X.shape)
    return np.concatenate(cs), np.concatenate(xs), groups, off, (R, t, k, X), (R0, t0, k0, X0)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("radh") / "libbundle_adjust_intrinsics_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-o", so, os.path.join(ROOT, "tests", "bundle_adjust_intrinsics_host.cpp")])
    L = ctypes.CDLL(so)
    L.radh_sq_error.restype = ctypes.c_double
    L.radh_sq_error.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_double] * 2 + [ctypes.c_void_p]
    L.radh_jacobian.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_double] * 2 + [ctypes.c_void_p] * 4
    L.radh_undistort.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    L.radh_max_radius.restype = ctypes.c_double
    L.radh_max_radius.argtypes = [ctypes.c_double, ctypes.c_double]
    return L


def _p(a):
    return a.ctypes.data


# ------------------------------------------------------------------------------------------------ host build (CPU)
def test_host_jacobians_match_central_differences(host):
    rng = np.random.default_rng(1)
    worst = 0.0
    for trial in range(40):
        R = o.expmap(0.3 * rng.normal(size=3))
        t = rng.normal(size=3)
        k = np.array([500.0 * (1 + 0.2 * rng.uniform()), 320 + 10 * rng.normal(), 240 + 10 * rng.normal(),
                      0.2 * (1 if trial % 2 else -1), 0.05 * rng.normal()])
        # points up to the image corner (|u| ~ 0.8)
        u = rng.uniform(-0.65, 0.65, 2) if trial % 4 else np.array([0.62, -0.47])
        z = rng.uniform(2, 10)
        X = R.T @ (np.r_[u * z, z] - t)
        x, y = 300.0, 200.0
        P = np.r_[R.reshape(-1), t]
        r, Jc, Jx, Jk = np.zeros(2), np.zeros(12), np.zeros(6), np.zeros(10)
        host.radh_jacobian(_p(P), _p(k), _p(X), x, y, _p(r), _p(Jc), _p(Jx), _p(Jk))
        ref = q.project(R[None], t[None], k[None], X[None], np.array([[x, y]]))
        assert np.abs(r - ref[0][0]).max() <= 1e-9 * np.abs(r).max()

        def res(P2, k2, X2):
            out = np.zeros(2)
            fr = ctypes.c_int()
            host.radh_sq_error(_p(P2), _p(k2), _p(X2), x, y, ctypes.byref(fr))
            r2, Jc2, Jx2, Jk2 = np.zeros(2), np.zeros(12), np.zeros(6), np.zeros(10)
            host.radh_jacobian(_p(P2), _p(k2), _p(X2), x, y, _p(r2), _p(Jc2), _p(Jx2), _p(Jk2))
            out[:] = r2
            return out

        num = np.zeros((2, 14))
        for i in range(6):
            h = 1e-6
            D = np.zeros(6)
            D[i] = h
            Pp = np.r_[(o.expmap(D[:3]) @ R).reshape(-1), t + D[3:]]
            D[i] = -h
            Pm = np.r_[(o.expmap(D[:3]) @ R).reshape(-1), t + D[3:]]
            num[:, i] = (res(Pp, k, X) - res(Pm, k, X)) / (2 * h)
        for i in range(3):
            h = 1e-6 * max(1.0, abs(X[i]))
            e = np.zeros(3)
            e[i] = h
            num[:, 6 + i] = (res(P, k, X + e) - res(P, k, X - e)) / (2 * h)
        for i in range(5):
            h = 1e-2 * max(1.0, abs(k[i]))        # the residual is linear in each intrinsic parameter
            e = np.zeros(5)
            e[i] = h
            num[:, 9 + i] = (res(P, k + e, X) - res(P, k - e, X)) / (2 * h)
        ana = np.c_[Jc.reshape(2, 6), Jx.reshape(2, 3), Jk.reshape(2, 5)]
        # each column against its own scale
        err = np.abs(ana - num).max(0) / np.maximum(np.abs(ana).max(0), 1e-300)
        worst = max(worst, float(err.max()))
        assert (err <= 1e-7).all(), (trial, err)
        assert np.abs(ana - np.c_[ref[1][0], ref[2][0], ref[3][0]]).max() <= 1e-12 * np.abs(ana).max()
    print("worst relative difference to central differences: %.2e" % worst)


def test_host_undistortion_inverts_the_distortion(host):
    rng = np.random.default_rng(2)
    for k1, k2 in ((-0.08, 0.01), (-0.2, 0.0), (0.2, 0.05), (-0.3, 0.02), (0.1, -0.02), (0.0, 0.0)):
        k = np.array([520.0, 320.0, 240.0, k1, k2])
        rmax = q.max_radius(k1, k2)
        assert abs(host.radh_max_radius(k1, k2) - rmax) <= 1e-15 * max(1.0, rmax) or rmax == host.radh_max_radius(k1, k2)
        top = min(0.999 * rmax, 1.5)
        rho = np.r_[rng.uniform(0, top, 400), top, 1e-9, 0.0]
        ang = rng.uniform(0, 2 * np.pi, len(rho))
        u = np.c_[rho * np.cos(ang), rho * np.sin(ang)]
        raw = q.distort(k, u)
        out = np.zeros_like(raw)
        assert host.radh_undistort(_p(k), _p(np.ascontiguousarray(raw)), len(raw), _p(out)) == len(raw)
        assert np.abs(out - (k[0] * u + k[1:3])).max() <= 1e-9, (k1, k2)
        ref = np.array([q.undistort(k, *xy) for xy in raw])
        assert np.abs(out - ref).max() <= 1e-12 * k[0]
        if rmax < np.inf:
            # past the turning point: NaN
            s = rmax * rmax
            rd = rmax * (1 + s * (k1 + s * k2))
            far = np.array([[k[1] + k[0] * rd * 1.001, k[2]], [k[1], k[2] - k[0] * rd * 1.5]])
            got = np.zeros_like(far)
            assert host.radh_undistort(_p(k), _p(far), 2, _p(got)) == 0
            assert np.isnan(got).all() and all(np.isnan(q.undistort(k, *xy)).all() for xy in far)
    bad = np.array([0.0, 320.0, 240.0, 0.0, 0.0])
    got = np.zeros(2)
    assert host.radh_undistort(_p(bad), _p(np.array([1.0, 2.0])), 1, _p(got)) == 0 and np.isnan(got).all()


# ------------------------------------------------------------------------------------------------ oracle (CPU)
def _schur_problem():
    # two groups; camera 4 (group 0) sees no used observation; camera 0 held with group 1 whose other cameras are held
    # too (group 1 = cameras 0 and 5, camera 5 held): group 1 is constrained by held cameras only; group 2 is held
    groups = np.array([1, 0, 0, 0, 0, 1, 2], np.int32)
    cams, pts, g, off, _, (R0, t0, k0, X0) = rscene(7, 50, 3, groups=groups, f_err=0.03, zero_k=False)
    m = cams != 4
    return dict(cams=cams, pts=pts, R=R0, t=t0, groups=g, intrinsics=k0, offsets=off, X=X0, mask=m,
                free=[1, 2, 3, 4, 6], free_groups=[0, 1], refine=FD, loss_scale=2.0, scale_gauge=1)


@pytest.mark.parametrize("lam", [0.0, 1e-3, 1.0, 100.0])
def test_matrix_free_product_equals_the_dense_schur_complement(lam):
    a = _schur_problem()
    P = q.setup(**a)
    assert P["hold"] is not None and not P["active"].all() and P["gactive"].all()
    lin = q.linearise(P, P["R"], P["t"], P["k"], P["X"])
    Vi = q.point_inverses(P, lin, lam)
    S, keep = q.dense_s(P, lin, lam)
    Sa = q.dense_s(P, lin, lam, absolute=True)[0]
    # f, k1 and k2 of both free groups are kept, cx and cy pinned
    assert (keep[6 * len(P["free"]):].reshape(2, 5) == [True, False, False, True, True]).all()
    rng = np.random.default_rng(5)
    for _ in range(3):
        p = rng.normal(size=len(keep))
        p[~keep] = 0.0
        got = q.schur_matvec(P, lin, Vi, lam, p)
        ref = S @ p[keep]
        assert np.abs(got[keep] - ref).max() <= 1e-12 * (Sa @ np.abs(p[keep])).max(), lam
        assert (got[~keep] == 0.0).all()


def test_tight_pcg_step_and_whole_call_equal_the_dense_lm():
    a = _schur_problem()
    P = q.setup(**a)
    lin = q.linearise(P, P["R"], P["t"], P["k"], P["X"])
    n = int((~P["pin"]).sum())
    for lam in (1e-3, 1.0, 100.0):
        (dx, dX), kk = q.pcg_step(P, lin, lam, TIGHT, 2 * n)
        ex, eX = q.dense_step(P, lin, lam)
        assert np.abs(dx - ex).max() <= 1e-9 * np.abs(ex).max(), lam
        assert np.abs(dX - eX).max() <= 1e-9 * np.abs(eX).max(), lam
        assert (dx[P["pin"]] == 0.0).all() and 1 <= kk <= 2 * n
    kw = {k: v for k, v in a.items()}
    got = q.bundle_adjust_intrinsics(cg_tol=TIGHT, cg_max_iters=2 * n, max_iters=30, **kw)
    ref = q.bundle_adjust_intrinsics(dense=True, max_iters=30, **kw)
    assert got["iters"] == ref["iters"] and got["cost"] < got["cost0"]
    assert abs(got["cost"] - ref["cost"]) <= 1e-10 * ref["cost"]
    for key in ("R", "t", "X", "intrinsics"):
        assert np.abs(got[key] - ref[key]).max() <= 1e-8 * max(1.0, np.abs(ref[key]).max()), key
    assert (got["mask"] == ref["mask"]).all()


def test_reduces_to_the_pose_only_oracle():
    cams, pts, g, off, _, (R0, t0, k0, X0) = rscene(8, 60, 4, groups=np.arange(8) % 3, f_err=0.02)
    K = np.zeros((8, 3, 3))
    for c in range(8):
        f, cx, cy = k0[g[c], :3]
        K[c] = [[f, 0, cx], [0, f, cy], [0, 0, 1]]
    kw = dict(free=list(range(1, 8)), scale_gauge=1, loss_scale=1.0, max_iters=30)
    got = q.bundle_adjust_intrinsics(cams, pts, R0, t0, g, k0, off, X0, refine=0, **kw)
    ref = pq.bundle_adjust_pcg(cams, pts, R0, t0, K, off, X0, **kw)
    assert got["iters"] == ref["iters"] and got["cg_iters"] == ref["cg_iters"] and got["n_used"] == ref["n_used"]
    assert abs(got["cost"] - ref["cost"]) <= 1e-12 * ref["cost"] and abs(got["cost0"] - ref["cost0"]) <= 1e-12 * ref["cost0"]
    for key in ("R", "t", "X"):
        assert np.abs(got[key] - ref[key]).max() <= 1e-12 * max(1.0, np.abs(ref[key]).max()), key
    assert (got["mask"] == ref["mask"]).all() and got["intrinsics"].tobytes() == k0.tobytes()


def test_oracle_matches_scipy():
    from scipy.optimize import least_squares
    cams, pts, g, off, (R, t, k, X), (R0, t0, k0, X0) = rscene(5, 60, 6, groups=[0, 0, 0, 1, 1], noise=0.3,
                                                                f_err=0.02)
    kw = dict(free=[1, 2, 3, 4], scale_gauge=1, refine=ALL, max_iters=200)
    got = q.bundle_adjust_intrinsics(cams, pts, R0, t0, g, k0, off, X0, cg_tol=1e-12, cg_max_iters=200, **kw)
    P = got["P"]
    n = int((~P["pin"]).sum()) + 3 * int(P["opt"].sum())
    sol = least_squares(lambda v: q.residuals(P, v), np.zeros(n), method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15,
                        max_nfev=20000)
    c_sp = 2.0 * sol.cost
    print("cost %.12e (oracle, %d steps) vs %.12e (scipy)" % (got["cost"], got["iters"], c_sp))
    nf = len(P["free"])
    keep = np.flatnonzero(~P["pin"])
    dk = np.zeros(len(P["pin"]))
    dk[keep] = sol.x[:len(keep)]
    f_sp = k0[:, 0] + dk[6 * nf::5]
    assert abs(got["cost"] - c_sp) <= 1e-9 * c_sp
    assert np.abs(got["intrinsics"][:, 0] - f_sp).max() <= 1e-6 * f_sp.max()


# ------------------------------------------------------------------------------------------------ arguments (CPU)
def _raises(fn, args, message):
    with pytest.raises(ValueError) as e:
        fn(**args)
    assert str(e.value) == message


def test_python_messages():
    torch = pytest.importorskip("torch")
    from pydegensac_b200.matching import bundle_adjust_intrinsics_ragged, undistort_points
    f64, i32 = torch.float64, torch.int32
    good = dict(cams=torch.zeros(10, dtype=i32), pts=torch.zeros((10, 2), dtype=f64),
                R=torch.eye(3, dtype=f64).repeat(4, 1, 1), t=torch.zeros((4, 3), dtype=f64),
                groups=torch.zeros(4, dtype=i32), intrinsics=torch.tensor([[500.0, 320, 240, 0, 0]], dtype=f64),
                offsets=torch.tensor([0, 4, 10], dtype=i32), X=torch.zeros((2, 3), dtype=f64))
    host = "cams, pts, R, t, groups, intrinsics, offsets, X and mask must be CUDA tensors on one device"
    cases = [
        ({"cams": np.zeros(10, np.int32)}, "cams must be a torch tensor"),
        ({"groups": [0, 0, 0, 0]}, "groups must be a torch tensor"),
        ({"offsets": torch.tensor([0, 4, 10])}, "offsets must be int32, not torch.int64"),
        ({"offsets": torch.tensor([0], dtype=i32)}, "offsets must be [T+1] with T >= 1, not [1]"),
        ({"cams": torch.zeros(10, dtype=torch.int64)}, "cams must be int32, not torch.int64"),
        ({"pts": torch.zeros((10, 3), dtype=f64)}, "pts must be [obs,2], not [10, 3]"),
        ({"cams": torch.zeros(9, dtype=i32)}, "cams must be [obs] = [10], not [9]"),
        ({"R": torch.zeros((4, 3), dtype=f64)}, "R must be [C,3,3] with C >= 1, not [4, 3]"),
        ({"t": torch.zeros((3, 3), dtype=f64)}, "t must be [C,3] = [4,3], not [3, 3]"),
        ({"groups": torch.zeros(4, dtype=torch.int64)}, "groups must be int32, not torch.int64"),
        ({"groups": torch.zeros(3, dtype=i32)}, "groups must be [C] = [4], not [3]"),
        ({"intrinsics": torch.zeros((1, 4), dtype=f64)}, "intrinsics must be [G,5] with G >= 1, not [1, 4]"),
        ({"intrinsics": torch.zeros((0, 5), dtype=f64)}, "intrinsics must be [G,5] with G >= 1, not [0, 5]"),
        ({"X": torch.zeros((3, 3), dtype=f64)}, "X must be [T,3] = [2,3], not [3, 3]"),
        ({"intrinsics": torch.zeros((1, 5), dtype=i32)}, "intrinsics must be a floating tensor, not torch.int32"),
        ({"mask": torch.ones(9, dtype=torch.bool)}, "mask must be [obs] = [10], not [9]"),
        ({"free": [1, 1]}, "free holds a camera twice"),
        ({"free": [4]}, "free holds a camera index outside [0, 4)"),
        ({"scale_gauge": 0}, "scale_gauge 0 is not one of the free cameras"),
        ({"free_groups": "x"}, "free_groups must be a host sequence of group indices"),
        ({"free_groups": [0, 0]}, "free_groups holds a group twice"),
        ({"free_groups": [1]}, "free_groups holds a group index outside [0, 1)"),
        ({"free_groups": [-1]}, "free_groups holds a group index outside [0, 1)"),
        ({"loss_scale": 0.0}, "loss_scale must be a positive number or None, not 0.0"),
        ({"max_iters": -1}, "max_iters must not be negative, not -1"),
        ({"px_th": 0.0}, "px_th must be a positive number, not 0.0"),
        ({"cg_max_iters": 0}, "cg_max_iters must be at least 1, not 0"),
        ({"cg_tol": float("nan")}, "cg_tol must be a non-negative finite number, not nan"),
        ({"free_groups": [], "refine_focal": False, "refine_distortion": False}, host),
        ({"R": torch.eye(3, dtype=f64).repeat(70, 1, 1), "t": torch.zeros((70, 3), dtype=f64),
          "groups": torch.zeros(70, dtype=i32)}, host),
        ({}, host),
    ]
    for kw, msg in cases:
        _raises(bundle_adjust_intrinsics_ragged, dict(good, **kw), msg)
    ugood = dict(pts=good["pts"], cams=good["cams"], groups=good["groups"], intrinsics=good["intrinsics"])
    uhost = "pts, cams, groups, intrinsics and mask must be CUDA tensors on one device"
    ucases = [
        ({"pts": np.zeros((10, 2))}, "pts must be a torch tensor"),
        ({"pts": torch.zeros((10, 3), dtype=f64)}, "pts must be [obs,2], not [10, 3]"),
        ({"cams": torch.zeros(10, dtype=torch.int64)}, "cams must be int32, not torch.int64"),
        ({"cams": torch.zeros(9, dtype=i32)}, "cams must be [obs] = [10], not [9]"),
        ({"groups": torch.zeros(4, dtype=torch.int64)}, "groups must be int32, not torch.int64"),
        ({"groups": torch.zeros((2, 2), dtype=i32)}, "groups must be [C] with C >= 1, not [2, 2]"),
        ({"intrinsics": torch.zeros(5, dtype=f64)}, "intrinsics must be [G,5] with G >= 1, not [5]"),
        ({"pts": torch.zeros((10, 2), dtype=i32)}, "pts must be a floating tensor, not torch.int32"),
        ({}, uhost),
    ]
    for kw, msg in ucases:
        _raises(undistort_points, dict(ugood, **kw), msg)


def _lib():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    return _cabi.lib()


def test_c_entry_points_refuse_malformed_input_before_any_launch():
    L = _lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["cams", "pts", "R", "t", "groups", "intr", "offsets", "X", "mask", "R_out", "t_out", "X_out", "intr_out",
             "mask_out", "cost0", "cost", "iters", "n_used", "cg_iters"]

    def call(n_cams=4, n_groups=2, n_tracks=3, obs=10, free=(1, 2, 3), fgroups=(0, 1), refine=5, gauge=1,
             loss_scale=0.0, max_iters=10, px_th=2.0, cg_max_iters=10, cg_tol=0.1, n_free=None, n_fg=None, null=()):
        b = {k: (None if isinstance(null, set) and k in null else fake) for k in names}
        hf = (ctypes.c_int32 * max(len(free), 1))(*free)
        hg = (ctypes.c_int32 * max(len(fgroups), 1))(*fgroups)
        return L.dgb200_bundle_adjust_intrinsics_ragged_dev(
            b["cams"], b["pts"], b["R"], b["t"], b["groups"], b["intr"], n_groups, n_cams, b["offsets"], n_tracks, obs,
            b["X"], b["mask"], None if null == "free" else hf, len(free) if n_free is None else n_free,
            None if null == "fgroups" else hg, len(fgroups) if n_fg is None else n_fg, refine, gauge,
            ctypes.c_double(loss_scale), max_iters, ctypes.c_double(px_th), cg_max_iters, ctypes.c_double(cg_tol),
            b["R_out"], b["t_out"], b["X_out"], b["intr_out"], b["mask_out"], b["cost0"], b["cost"], b["iters"],
            b["n_used"], b["cg_iters"], None)

    sizes = "need n_tracks >= 1, obs >= 0 and n_cams >= 1"
    cases = [(dict(null={k}), "null buffer") for k in names if k not in ("cams", "pts", "mask", "mask_out")]
    cases += [(dict(null={k}), "null observation buffer") for k in ("cams", "pts", "mask_out")]
    cases += [
        (dict(null={"cams"}, obs=0, n_tracks=0), sizes),
        (dict(n_tracks=0), sizes), (dict(obs=-1), sizes), (dict(n_cams=0), sizes),
        (dict(n_free=-1), "n_free must lie in [0, n_cams]"), (dict(n_free=5), "n_free must lie in [0, n_cams]"),
        (dict(null="free"), "null free-camera list"),
        (dict(free=(1, 1)), "free camera index repeated"), (dict(free=(1, 4)), "free camera index out of range"),
        (dict(gauge=0), "scale_gauge must be one of the free cameras"),
        (dict(gauge=-2), "scale_gauge must be a free camera or -1"),
        (dict(free=(0, 1, 2, 3), gauge=1), "scale_gauge needs a held camera"),
        (dict(loss_scale=-1.0), "loss_scale must be a positive number (or 0 for the trivial loss)"),
        (dict(max_iters=-1), "max_iters must not be negative"),
        (dict(px_th=0.0), "px_th must be a positive number"),
        (dict(cg_max_iters=0), "cg_max_iters must be at least 1"),
        (dict(cg_tol=float("nan")), "cg_tol must be a non-negative finite number"),
        (dict(n_groups=0, n_fg=0), "need n_groups >= 1"),
        (dict(n_fg=-1), "n_free_groups must lie in [0, n_groups]"),
        (dict(n_fg=3), "n_free_groups must lie in [0, n_groups]"),
        (dict(null="fgroups"), "null free-group list"),
        (dict(fgroups=(0, 2)), "free group index out of range"), (dict(fgroups=(-1,)), "free group index out of range"),
        (dict(fgroups=(1, 1)), "free group index repeated"),
        (dict(refine=8), "refine must be a set of DGB200_REFINE_* bits"),
        (dict(refine=-1), "refine must be a set of DGB200_REFINE_* bits"),
        (dict(refine=8, cg_max_iters=0), "cg_max_iters must be at least 1"),
        (dict(fgroups=(0, 2), null={"cost"}), "null buffer"),
    ]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert L.dgb200_bundle_adjust_intrinsics_last_error().decode() == msg, kw

    def ucall(rows=10, n_cams=4, n_groups=2, null=()):
        b = {k: (None if k in null else fake) for k in ("pts", "cams", "groups", "intr", "out")}
        return L.dgb200_undistort_points_dev(b["pts"], b["cams"], rows, b["groups"], n_cams, b["intr"], n_groups,
                                             b["out"], None)

    ucases = [(dict(null={"groups"}), "null buffer"), (dict(null={"intr"}), "null buffer")]
    ucases += [(dict(null={k}), "null row buffer") for k in ("pts", "cams", "out")]
    ucases += [(dict(rows=-1), "need rows >= 0, n_cams >= 1 and n_groups >= 1"),
               (dict(n_cams=0), "need rows >= 0, n_cams >= 1 and n_groups >= 1"),
               (dict(n_groups=0), "need rows >= 0, n_cams >= 1 and n_groups >= 1")]
    for kw, msg in ucases:
        assert ucall(**kw) == -1, kw
        assert L.dgb200_undistort_last_error().decode() == msg, kw
    assert ucall(rows=0, null={"pts", "cams", "out"}) == 0     # nothing to do, nothing launched


def test_new_kernels_do_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "pydegensac_b200", "csrc", "bundle_adjust_intrinsics.cu")
    out = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false",
                          "-cubin", "-Xptxas", "-v", "-o", str(tmp_path / "bai.cubin"), src],
                         capture_output=True, text=True, check=True).stderr
    rows = re.findall(r"Function properties for (\S+)\n\s*ptxas\s+info\s*:?\s*(\d+) bytes stack frame, (\d+) bytes spill "
                      r"stores, (\d+) bytes spill loads", out)
    if not rows:   # older ptxas: the numbers on the line after
        rows = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                          r"(\d+) bytes spill loads", out)
    names = [r[0] for r in rows if "_kernel" in r[0]]
    assert len(names) >= 18, out[-2000:]
    for name, stack, st, ld in rows:
        assert int(st) == 0 and int(ld) == 0, (name, st, ld)


# ------------------------------------------------------------------------------------------------ GPU
def _dev(*xs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0") for a in xs]


def _np(res):
    return {k: getattr(res, k).cpu().numpy() for k in res._fields}


def _run(cams, pts, R, t, g, k, off, X, mask=None, refine=FD, **kw):
    from pydegensac_b200.matching import bundle_adjust_intrinsics_ragged
    d = _dev(cams, pts, R, t, g, k, off, X)
    m = _dev(mask)[0] if mask is not None else None
    return _np(bundle_adjust_intrinsics_ragged(*d, mask=m, refine_focal=bool(refine & q.FOCAL),
                                               refine_principal_point=bool(refine & q.PRINCIPAL_POINT),
                                               refine_distortion=bool(refine & q.DISTORTION), **kw))


def _close(g, ref, tol=1e-9):
    for key in ("R", "t", "X", "intrinsics"):
        scale = max(1.0, np.abs(ref[key]).max())
        assert np.abs(g[key] - ref[key]).max() <= tol * scale, (key, np.abs(g[key] - ref[key]).max())


@pytest.mark.gpu
@pytest.mark.parametrize("loss_scale", [None, 1.0])
def test_kernel_against_the_oracle(loss_scale):
    groups = np.array([0, 0, 1, 1, 0, 1, 0, 1, 1, 0], np.int32)
    cams, pts, g, off, _, (R0, t0, k0, X0) = rscene(10, 600, 41, groups=groups, f_err=0.04)
    kw = dict(free=list(range(1, 10)), scale_gauge=1, loss_scale=loss_scale, max_iters=50, px_th=2.0, refine=ALL)
    # at a tight CG tolerance every trial step is the exact LM step, so the two summation orders follow one path: the
    # same trial steps, and the result within 1e-9
    tight = dict(cg_tol=1e-10, cg_max_iters=200)
    got = _run(cams, pts, R0, t0, g, k0, off, X0, **kw, **tight)
    ref = q.bundle_adjust_intrinsics(cams, pts, R0, t0, g, k0, off, X0, **kw, **tight)
    print("loss %s, tight: cost %.9e -> %.12e (oracle %.12e), %d steps (oracle %d), %d CG (oracle %d); f %s (oracle %s)"
          % (loss_scale, got["cost0"][0], got["cost"][0], ref["cost"], got["iters"][0], ref["iters"],
             got["cg_iters"][0], ref["cg_iters"], got["intrinsics"][:, 0], ref["intrinsics"][:, 0]))
    assert got["iters"][0] == ref["iters"] and got["n_used"][0] == ref["n_used"]
    assert (got["mask"] == ref["mask"]).all()
    assert abs(got["cost0"][0] - ref["cost0"]) <= 1e-12 * ref["cost0"]
    assert abs(got["cost"][0] - ref["cost"]) <= 1e-9 * ref["cost"]
    _close(got, ref)
    # at the default tolerance the inexact steps depend on where CG stops, which rounding can move by an iteration, so
    # the paths differ; both reach the same optimum
    got = _run(cams, pts, R0, t0, g, k0, off, X0, **kw)
    ref = q.bundle_adjust_intrinsics(cams, pts, R0, t0, g, k0, off, X0, **kw)
    print("loss %s, cg_tol 0.1: cost %.12e (oracle %.12e), %d steps (oracle %d), %d CG (oracle %d)"
          % (loss_scale, got["cost"][0], ref["cost"], got["iters"][0], ref["iters"], got["cg_iters"][0],
             ref["cg_iters"]))
    assert abs(got["cost"][0] - ref["cost"]) <= 1e-9 * ref["cost"] and got["cost"][0] < got["cost0"][0]
    _close(got, ref, 1e-7)


# Recovery thresholds, fixed from the oracle's result on the same scene (seed 11, 0.3 px noise per coordinate): it
# reaches |f - 520| / 520 = 4.4e-4, |k1 + 0.08| = 6.5e-5 and a residual RMS per coordinate of 0.265 px; the bounds
# leave a factor of about 5 on f and k1, and the RMS must come back to the noise level.
F_REL_TOL, K1_TOL, RMS_MAX = 2e-3, 3e-4, 0.3


def _recovery_scene():
    k = np.array([[520.0, 320.0, 240.0, -0.08, 0.01]])
    return rscene(40, 1500, 11, k=k, noise=0.3, f_err=0.05)


def test_oracle_recovers_focal_and_distortion():
    cams, pts, g, off, _, (R0, t0, k0, X0) = _recovery_scene()
    ref = q.bundle_adjust_intrinsics(cams, pts, R0, t0, g, k0, off, X0, max_iters=100)
    rms = np.sqrt(ref["cost"] / (2 * ref["n_used"]))
    f_err, k1_err = abs(ref["intrinsics"][0, 0] - 520.0) / 520.0, abs(ref["intrinsics"][0, 3] + 0.08)
    print("oracle: f %.6f (rel err %.2e), k1 %.6f (err %.2e), k2 %.6f, rms %.4f px, %d steps"
          % (ref["intrinsics"][0, 0], f_err, ref["intrinsics"][0, 3], k1_err, ref["intrinsics"][0, 4], rms,
             ref["iters"]))
    assert f_err <= F_REL_TOL and k1_err <= K1_TOL and rms <= RMS_MAX


@pytest.mark.gpu
def test_kernel_recovers_focal_and_distortion():
    cams, pts, g, off, _, (R0, t0, k0, X0) = _recovery_scene()
    got = _run(cams, pts, R0, t0, g, k0, off, X0, max_iters=100)
    rms0 = np.sqrt(got["cost0"][0] / (2 * got["n_used"][0]))
    rms = np.sqrt(got["cost"][0] / (2 * got["n_used"][0]))
    f_err, k1_err = abs(got["intrinsics"][0, 0] - 520.0) / 520.0, abs(got["intrinsics"][0, 3] + 0.08)
    print("kernel: f %.6f (rel err %.2e), k1 %.6f (err %.2e), rms %.3f -> %.4f px, %d steps, %d CG"
          % (got["intrinsics"][0, 0], f_err, got["intrinsics"][0, 3], k1_err, rms0, rms, got["iters"][0],
             got["cg_iters"][0]))
    assert f_err <= F_REL_TOL and k1_err <= K1_TOL and rms <= RMS_MAX


@pytest.mark.gpu
def test_agrees_with_the_pose_only_solver():
    from pydegensac_b200.matching import bundle_adjust_pcg_ragged
    cams, pts, g, off, _, (R0, t0, k0, X0) = rscene(12, 1500, 42, groups=np.arange(12) % 4, f_err=0.02)
    K = np.array([[[k0[gc, 0], 0, k0[gc, 1]], [0, k0[gc, 0], k0[gc, 2]], [0, 0, 1]] for gc in g])
    kw = dict(free=list(range(1, 12)), scale_gauge=1, loss_scale=1.0, max_iters=30)
    got = _run(cams, pts, R0, t0, g, k0, off, X0, refine=0, **kw)
    d = _dev(cams, pts, R0, t0, K, off, X0)
    ref = _np(bundle_adjust_pcg_ragged(*d, **kw))
    assert got["iters"][0] == ref["iters"][0] and got["cg_iters"][0] == ref["cg_iters"][0]
    assert abs(got["cost"][0] - ref["cost"][0]) <= 1e-9 * ref["cost"][0] and (got["mask"] == ref["mask"]).all()
    for key in ("R", "t", "X"):
        assert np.abs(got[key] - ref[key]).max() <= 1e-9 * max(1.0, np.abs(ref[key]).max()), key
    assert got["intrinsics"].tobytes() == k0.tobytes()


@pytest.mark.gpu
def test_beyond_the_dense_limit_with_a_group_per_camera():
    C = 80
    cams, pts, g, off, _, (R0, t0, k0, X0) = rscene(C, 8000, 8, groups=np.arange(C), f_err=0.01, zero_k=False,
                                                    lmax=10)
    kw = dict(max_iters=15, refine=FD)
    got = _run(cams, pts, R0, t0, g, k0, off, X0, **kw)
    ref = q.bundle_adjust_intrinsics(cams, pts, R0, t0, g, k0, off, X0, **kw)
    print("%d cameras, %d groups, %d observations: cost %.9e -> %.9e (oracle %.9e), %d steps (oracle %d), %d CG "
          "(oracle %d)" % (C, C, len(cams), got["cost0"][0], got["cost"][0], ref["cost"], got["iters"][0],
                           ref["iters"], got["cg_iters"][0], ref["cg_iters"]))
    # a focal length and two distortion terms per camera are weakly held, and the inexact steps amplify the rounding
    # differences of the two summation orders along them: the costs agree, the trajectories only roughly
    assert abs(got["cost"][0] - ref["cost"]) <= 1e-6 * ref["cost"] and got["cost"][0] < 0.1 * got["cost0"][0]
    df = np.abs(got["intrinsics"] - ref["intrinsics"]).max(0)
    print("largest differences to the oracle (f, cx, cy, k1, k2): %s" % df)
    assert df[0] <= 0.05 and (df[1:3] == 0).all()


@pytest.mark.gpu
def test_same_bytes_on_a_rerun_pass_through_and_aliased_outputs():
    import torch
    groups = np.array([0, 1, 1, 2, 0, 1, 3, 3, 0, 1], np.int32)
    cams, pts, g, off, _, (R0, t0, k0, X0) = rscene(10, 500, 43, groups=groups, f_err=0.03)
    k0 = np.r_[k0, [[np.nan, 0, 0, 0, 0]]]
    g = g.copy()
    g[9] = 4                                        # camera 9: a group whose intrinsics are not finite
    cams = np.r_[cams, [3, 3]].astype(np.int32)
    pts = np.r_[pts, pts[:2]]
    X0 = np.r_[X0, [[0.0, 0.0, 5.0]]]
    off = np.r_[off, off[-1] + 2].astype(np.int32)
    kw = dict(free=[2, 4, 5, 6, 7], free_groups=[0, 1, 4], scale_gauge=4, loss_scale=1.5, max_iters=30)
    a = _run(cams, pts, R0, t0, g, k0, off, X0, **kw)
    b = _run(cams, pts, R0, t0, g, k0, off, X0, **kw)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    for c in (0, 1, 3, 8, 9):
        assert a["R"][c].tobytes() == R0[c].tobytes() and a["t"][c].tobytes() == t0[c].tobytes()
    for gg in (2, 3, 4):                            # held groups and the invalid free group pass through
        assert a["intrinsics"][gg].tobytes() == k0[gg].tobytes()
    assert a["X"][-1].tobytes() == X0[-1].tobytes() and not a["mask"][cams == 9].any()
    assert a["cost"][0] < a["cost0"][0] and a["intrinsics"][0, 0] != k0[0, 0]
    ref = q.bundle_adjust_intrinsics(cams, pts, R0, t0, g, k0, off, X0, **kw)
    assert abs(a["cost"][0] - ref["cost"]) <= 1e-9 * ref["cost"] and a["iters"][0] == ref["iters"]
    # outputs that alias the inputs (R, t, X, intrinsics written over R0, t0, X0, k0)
    from pydegensac_b200 import _cabi
    from pydegensac_b200.matching import _call
    cm, x, Rd, td, gd, kd, od, Xd = _dev(cams, pts, R0, t0, g, k0, off, X0)
    dev = Rd.device
    mo = torch.empty(len(cams), dtype=torch.uint8, device=dev)
    s1 = [torch.empty(1, dtype=torch.float64, device=dev) for _ in range(2)]
    s2 = [torch.empty(1, dtype=torch.int32, device=dev) for _ in range(3)]
    hf = np.array(kw["free"], np.int32)
    hg = np.array(kw["free_groups"], np.int32)
    L = _cabi.lib()
    ip = ctypes.POINTER(ctypes.c_int32)
    _call(L.dgb200_bundle_adjust_intrinsics_ragged_dev, L.dgb200_bundle_adjust_intrinsics_last_error, dev, cm, x, Rd,
          td, gd, kd, len(k0), 10, od, len(off) - 1, len(cams), Xd, None, hf.ctypes.data_as(ip), len(hf),
          hg.ctypes.data_as(ip), len(hg), FD, 4, 1.5, 30, 2.0, 100, 0.1, Rd, td, Xd, kd, mo, s1[0], s1[1], s2[0], s2[1],
          s2[2])
    for k, v in (("R", Rd), ("t", td), ("X", Xd), ("intrinsics", kd), ("cost", s1[1]), ("cg_iters", s2[2])):
        assert v.cpu().numpy().tobytes() == a[k].tobytes(), k


@pytest.mark.gpu
def test_undistortion_kernel_matches_the_host_oracle():
    from pydegensac_b200.matching import undistort_points
    rng = np.random.default_rng(7)
    k = np.array([[520.0, 320.0, 240.0, -0.08, 0.01], [480.0, 300.0, 250.0, -0.3, 0.02], [500.0, 320, 240, 0.1, 0.0],
                  [0.0, 320, 240, 0, 0]])
    groups = np.array([0, 1, 2, 3, 7], np.int32)
    n = 4000
    cams = rng.integers(-1, 6, n).astype(np.int32)
    pts = np.c_[rng.uniform(-400, 1000, n), rng.uniform(-300, 800, n)]
    pts[:5] = np.nan
    got = undistort_points(*_dev(pts, cams, groups, k)).cpu().numpy()
    ref = q.undistort_points(pts, cams, groups, k)
    assert (np.isnan(got) == np.isnan(ref)).all()
    ok = ~np.isnan(ref)
    assert np.abs(got[ok] - ref[ok]).max() <= 1e-9
    print("undistorted %d of %d rows" % (ok[:, 0].sum(), n))
    assert ok[:, 0].sum() > n // 4 and np.isnan(got[cams == 3]).all() and np.isnan(got[(cams < 0) | (cams > 4)]).all()


@pytest.mark.gpu
def test_pipeline_from_ransac_to_self_calibration_without_sync():
    """ragged F RANSAC of distorted synthetic matches, build_tracks_ragged, undistort_points, triangulate_tracks_ragged
    and bundle_adjust_intrinsics_ragged under torch.cuda.set_sync_debug_mode("error")"""
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import (build_tracks_ragged, bundle_adjust_intrinsics_ragged,
                                          triangulate_tracks_ragged, undistort_points)
    dev = torch.device("cuda:0")
    C, N = 8, 400
    rng = np.random.default_rng(3)
    R, t, _ = rig(C, 3)
    k_true = np.array([[520.0, 320.0, 240.0, -0.08, 0.01]])
    Xw = np.array([_point(R, t, np.arange(C), rng) for _ in range(N)])
    kps = []
    for c in range(C):
        p = Xw @ R[c].T + t[c]
        kps.append(q.distort(k_true[0], p[:, :2] / p[:, 2:]) + 0.3 * rng.normal(size=(N, 2)))
    pairs = [(c, c + 1) for c in range(C - 1)] + [(c, c + 2) for c in range(C - 2)]
    idx = np.arange(N, dtype=np.int32)
    p1 = torch.from_numpy(np.concatenate([kps[a] for a, _ in pairs])).to(dev)
    p2 = torch.from_numpy(np.concatenate([kps[b] for _, b in pairs])).to(dev)
    offsets = torch.arange(0, N * len(pairs) + 1, N, dtype=torch.int32, device=dev)
    i1 = torch.from_numpy(np.tile(idx, len(pairs))).to(dev)
    seeds = torch.arange(len(pairs), dtype=torch.int64, device=dev)
    kp_all = [torch.from_numpy(kk).to(dev) for kk in kps]
    k0 = k_true.copy()
    k0[0, 0] *= 1.03
    k0[0, 3:] = 0.0
    Rd, td, kd = (torch.from_numpy(a).to(dev) for a in (R, t, k0))
    groups = torch.zeros(C, dtype=torch.int32, device=dev)
    # K = f basis[0] + cx basis[1] + cy basis[2] + basis[3], formed on the device from the group's intrinsics
    basis = torch.zeros((4, 3, 3), dtype=torch.float64, device=dev)
    basis[0, 0, 0] = basis[0, 1, 1] = basis[1, 0, 2] = basis[2, 1, 2] = basis[3, 2, 2] = 1.0
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        F, mask = pdg.findFundamentalMatrixBatch(p1, p2, 1.0, 0.999, 2000, seeds=seeds, offsets=offsets, n_max=N)
        ts = build_tracks_ragged([N] * C, pairs, i1, i1, offsets, mask, kps=kp_all)
        und = undistort_points(ts.pts, ts.cams, groups, kd)
        K = kd[0, 0] * basis[0] + kd[0, 1] * basis[1] + kd[0, 2] * basis[2] + basis[3]
        tr = triangulate_tracks_ragged(ts.cams, und, Rd, td, K, ts.offsets, px_th=8.0)
        ba = bundle_adjust_intrinsics_ragged(ts.cams, ts.pts, Rd, td, groups, kd, ts.offsets, tr.X, mask=tr.mask,
                                             loss_scale=1.0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    kr = ba.intrinsics.cpu().numpy()[0]
    print("pipeline: %d tracks, cost %.4f -> %.4f in %d steps, %d CG; f %.3f k1 %.4f" % (
        int(ts.stats[0]), float(ba.cost0[0]), float(ba.cost[0]), int(ba.iters[0]), int(ba.cg_iters[0]), kr[0], kr[3]))
    assert int(ts.stats[0]) >= 200 and float(ba.cost[0]) < float(ba.cost0[0]) and int(ba.n_used[0]) > 1000
    assert abs(kr[0] - 520.0) < abs(k0[0, 0] - 520.0)
