"""Pose from F over ragged batches (matching.pose_from_fundamental_ragged, dgb200_pose_from_fundamental_ragged_dev):
R, t and good of the dense pose kernel per pair, triangulated points, cheirality flags and parallax angles per row, and
the exact per-pair median parallax."""
import ctypes
import os

import numpy as np
import pytest

from pydegensac_b200.scenes import _K, _rot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")


def _skew(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])


def _scene(n, seed, n_behind=0, noise=0.0, K2=_K):
    """Two views of random 3-D points with a KNOWN pose (x2 ~ R x1 + t), camera 1 calibrated by _K and camera 2 by K2:
    pixels p1, p2, R, unit t, |t|, the points X in camera 1's frame, and F.  The last n_behind points lie in front of
    camera 1 but behind camera 2."""
    rng = np.random.default_rng(seed)
    R = _rot("z", 0.03) @ _rot("y", -0.2) @ _rot("x", 0.05)
    t = np.array([1.0, 0.1, 0.2])
    X = np.c_[rng.uniform(-2, 2, n), rng.uniform(-2, 2, n), rng.uniform(4, 10, n)]
    if n_behind:
        Y = np.c_[rng.uniform(-40, 40, 4000), rng.uniform(-2, 2, 4000), rng.uniform(-3, -0.5, 4000)]
        Xb = (Y - t) @ R                              # rows of R^T (Y - t): camera 1's frame
        Xb = Xb[Xb[:, 2] > 0.5][:n_behind]
        assert len(Xb) == n_behind
        X = np.r_[X, Xb]
    x1 = X @ _K.T
    x2 = (X @ R.T + t) @ K2.T
    p1 = x1[:, :2] / x1[:, 2:3] + noise * rng.normal(size=(len(X), 2))
    p2 = x2[:, :2] / x2[:, 2:3]
    nt = np.linalg.norm(t)
    return p1, p2, R, t / nt, nt, X, np.linalg.inv(K2).T @ _skew(t) @ R @ np.linalg.inv(_K)


# ------------------------------------------------------------------------------------------------ CPU
def test_oracle_pinned_to_planted_geometry():
    from oracle.frontend_np import pose_from_fundamental
    from tests.pose_ragged_np import pose_ragged
    lengths = [300, 0, 120, 57]
    scenes = [_scene(max(n - 6, 1), s, n_behind=6) if n else None for s, n in enumerate(lengths)]
    p1 = np.concatenate([s[0] for s in scenes if s]); p2 = np.concatenate([s[1] for s in scenes if s])
    F = np.stack([s[6] if s else np.eye(3) for s in scenes])
    off = np.r_[0, np.cumsum(lengths)]
    o = pose_ragged(F, _K, _K, p1, p2, off)
    for p, s in enumerate(scenes):
        a, b = off[p], off[p + 1]
        if s is None:
            assert o["good"][p] == 0 and np.isnan(o["median_angle"][p])
            continue
        _, _, R, t, nt, X, Fp = s
        Rd, td, gd = pose_from_fundamental(Fp, _K, _K, p1[a:b], p2[a:b])
        assert np.array_equal(o["R"][p], Rd) and np.array_equal(o["t"][p], td) and o["good"][p] == gd
        assert np.allclose(Rd, R, atol=1e-9) and np.allclose(td, t, atol=1e-9)
        front = o["in_front"][a:b]
        assert not front[-6:].any() and front[:-6].all() and gd == b - a - 6
        want = X / nt
        assert np.all(np.linalg.norm(o["points"][a:b] - want, axis=1) <= 1e-9 * np.linalg.norm(want, axis=1))
        # ray of camera 2 in camera 1's frame: K2^-1 [p2; 1] has z > 0, so it points away from a point behind camera 2
        c2 = (X + R.T @ (t * nt)) * np.sign((X @ R.T + t * nt)[:, 2:3])
        ang = np.arctan2(np.linalg.norm(np.cross(X, c2), axis=1), (X * c2).sum(1))
        assert np.abs(o["angle"][a:b] - ang).max() <= 1e-12
        assert abs(o["median_angle"][p] - np.median(ang[:-6])) <= 1e-12


def test_ragged_pose_entry_point_rejects_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["F", "K1", "K2", "x1y1", "x2y2", "offsets", "mask", "R", "t", "good", "points", "in_front", "angle",
             "median"]

    def call(n_pairs=3, rows=10, dim=2, **null):
        b = {k: (None if null.get(k) else fake) for k in names}
        return L.dgb200_pose_from_fundamental_ragged_dev(b["F"], b["K1"], b["K2"], 0, b["x1y1"], b["x2y2"], b["offsets"],
                                                         n_pairs, rows, dim, b["mask"], b["R"], b["t"], b["good"],
                                                         b["points"], b["in_front"], b["angle"], b["median"], None)

    for k in names:
        if k not in ("mask", "good"):              # the two optional buffers
            assert call(**{k: True}) == -1, k
    for n_pairs in (0, -1):
        assert call(n_pairs=n_pairs) == -1
    assert call(rows=-1) == -1
    for dim in (1, 0, -2):
        assert call(dim=dim) == -1


def test_ragged_pose_python_argument_errors():
    import torch
    from pydegensac_b200.matching import pose_from_fundamental_ragged as prp
    F = torch.zeros((2, 3, 3), dtype=torch.float64)
    K = torch.eye(3, dtype=torch.float64)
    p = torch.zeros((10, 2), dtype=torch.float64)
    off = torch.tensor([0, 4, 10], dtype=torch.int32)
    bad = [
        dict(F=torch.zeros((2, 8))), dict(F=torch.zeros((0, 9))), dict(F=torch.zeros(9)), dict(F=np.zeros((2, 9))),
        dict(pts1=torch.zeros(10, 1, dtype=torch.float64)), dict(pts2=torch.zeros((9, 2), dtype=torch.float64)),
        dict(pts1=torch.zeros(10, dtype=torch.float64)), dict(pts1=torch.zeros((10, 2), dtype=torch.int64)),
        dict(K1=torch.eye(4, dtype=torch.float64)), dict(K2=torch.zeros((3, 3, 3), dtype=torch.float64)),
        dict(K1=torch.eye(3, dtype=torch.int32)),
        dict(offsets=torch.tensor([0, 10], dtype=torch.int32)), dict(offsets=torch.tensor([0, 4, 10])),
        dict(offsets=torch.tensor([[0, 4, 10]], dtype=torch.int32)),
        dict(mask=torch.ones(9, dtype=torch.bool)), dict(mask=torch.ones(10, dtype=torch.int32)),
        dict(mask=np.ones(10, bool)),
        dict(),                                    # well-formed, but on the host
    ]
    for kw in bad:
        args = dict(F=F, K1=K, K2=K, pts1=p, pts2=p, offsets=off, mask=None)
        args.update(kw)
        with pytest.raises(ValueError):
            prp(**args)
    if torch.cuda.is_available():
        dev = torch.device("cuda:0")
        with pytest.raises(ValueError, match="device"):
            prp(F.to(dev), K, K.to(dev), p.to(dev), p.to(dev), off.to(dev))


# ------------------------------------------------------------------------------------------------ GPU
def _batch(lengths, seed, noise=0.3, K2=_K):
    """a ragged batch of noisy planted scenes (pair p: seed + p), with F of the planted pose"""
    ps1, ps2, Fs = [], [], []
    for i, n in enumerate(lengths):
        p1, p2, _, _, _, _, F = _scene(max(n, 8), seed + i, noise=noise, K2=K2)
        ps1.append(p1[:n]); ps2.append(p2[:n]); Fs.append(F)
    off = np.r_[0, np.cumsum(lengths)].astype(np.int32)
    return np.concatenate(ps1), np.concatenate(ps2), np.stack(Fs), off


def _dev(*xs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0") for x in xs]


def _np(pose):
    return {k: v.cpu().numpy() for k, v in pose._asdict().items()}


LENGTHS = [0, 1, 7, 33, 400, 2048, 4097, 20000]


@pytest.mark.gpu
def test_ragged_equals_dense_per_pair():
    import torch
    from pydegensac_b200.matching import pose_from_fundamental, pose_from_fundamental_ragged
    p1, p2, F, off = _batch(LENGTHS, 100)
    mask = np.ones(len(p1), bool); mask[::5] = False; mask[3::11] = False
    d1, d2, dF, doff, dm, dK = _dev(p1, p2, F, off, mask, _K)
    pose = pose_from_fundamental_ragged(dF, dK, dK, d1, d2, doff, dm)
    for p, n in enumerate(LENGTHS):
        a, b = int(off[p]), int(off[p + 1])
        if n == 0:
            assert int(pose.good[p]) == 0 and torch.isnan(pose.median_angle[p])
            continue
        R, t, good = pose_from_fundamental(dF[p:p + 1], dK, dK, d1[a:b][None], d2[a:b][None], dm[a:b][None])
        assert torch.equal(pose.R[p], R[0]) and torch.equal(pose.t[p], t[0]) and torch.equal(pose.good[p], good[0]), p
    # per-pair K, given as [P,3,3]: the same poses
    Ks = torch.stack([dK] * len(LENGTHS))
    g, g2 = _np(pose), _np(pose_from_fundamental_ragged(dF, Ks, Ks, d1, d2, doff, dm))
    for k in g:
        assert np.array_equal(g2[k], g[k], equal_nan=g[k].dtype.kind == "f"), k


@pytest.mark.gpu
def test_rows_against_oracle():
    from pydegensac_b200.matching import pose_from_fundamental_ragged
    from tests.pose_ragged_np import pose_ragged, rows_under_pose
    K2 = _K.copy(); K2[0, 0] *= 1.1; K2[0, 2] += 7.0
    p1, p2, F, off = _batch(LENGTHS, 200, noise=0.5, K2=K2)
    mask = np.ones(len(p1), bool); mask[1::4] = False
    d1, d2, dF, doff, dm, dK1, dK2 = _dev(p1, p2, F, off, mask, _K, K2)
    g = _np(pose_from_fundamental_ragged(dF, dK1, dK2, d1, d2, doff, dm))
    o = pose_ragged(F, _K, K2, p1, p2, off, mask)
    assert np.abs(g["R"] - o["R"]).max() <= 1e-9, np.abs(g["R"] - o["R"]).max()
    assert np.abs(g["t"] - o["t"]).max() <= 1e-9, np.abs(g["t"] - o["t"]).max()
    assert np.array_equal(g["good"], o["good"]), (g["good"], o["good"])
    for p in range(len(LENGTHS)):
        a, b = off[p], off[p + 1]
        if a == b:
            continue
        # per row under the GPU's own pose, so that the comparison is of the row arithmetic
        pts, front, ang, l1, l2 = rows_under_pose(g["R"][p], g["t"][p], _K, K2, p1[a:b], p2[a:b], mask[a:b])
        err = np.linalg.norm(g["points"][a:b] - pts, axis=1) / np.linalg.norm(pts, axis=1)
        assert err.max() <= 1e-9, (p, err.max())
        err = np.abs(g["angle"][a:b] - ang) / np.abs(ang)
        assert err.max() <= 1e-9, (p, err.max())
        scale = max(1.0, np.median(np.abs(np.r_[l1, l2])))
        near = (np.abs(l1) < 1e-9 * scale) | (np.abs(l2) < 1e-9 * scale)
        assert np.array_equal(g["in_front"][a:b][~near], front[~near]), p
        assert g["good"][p] == g["in_front"][a:b].sum()
        assert np.all((g["angle"][a:b] >= 0) & (g["angle"][a:b] <= np.pi))


@pytest.mark.gpu
def test_median_is_exact():
    from pydegensac_b200.matching import pose_from_fundamental_ragged
    rng = np.random.default_rng(7)
    # odd / even counts, duplicated rows (many equal angles), a 20000-row pair, a pair with no row in front
    l1, l2, Fs, masks = [], [], [], []
    specs = [(101, "all"), (100, "all"), (2, "all"), (1, "all"), (20000, "all"), (19999, "all"), (3000, "holes"),
             (50, "dup"), (51, "dup"), (40, "none"), (64, "dup2")]
    for i, (n, kind) in enumerate(specs):
        p1, p2, _, _, _, _, F = _scene(max(n, 8), 300 + i, noise=0.3)
        p1, p2 = p1[:n], p2[:n]
        m = np.ones(n, bool)
        if kind == "holes":
            m[rng.random(n) < 0.3] = False
        elif kind == "dup":                          # 5 distinct rows, each repeated
            idx = np.arange(n) % 5
            p1, p2 = p1[idx], p2[idx]
        elif kind == "dup2":                         # two distinct rows: the middle pair straddles them
            idx = (np.arange(n) >= n // 2).astype(int)
            p1, p2 = p1[idx], p2[idx]
        elif kind == "none":
            m[:] = False
        l1.append(p1); l2.append(p2); Fs.append(F); masks.append(m)
    off = np.r_[0, np.cumsum([len(x) for x in l1])].astype(np.int32)
    d1, d2, dF, doff, dm, dK = _dev(np.concatenate(l1), np.concatenate(l2), np.stack(Fs), off, np.concatenate(masks), _K)
    g = _np(pose_from_fundamental_ragged(dF, dK, dK, d1, d2, doff, dm))
    counts = set()
    for p in range(len(specs)):
        a, b = off[p], off[p + 1]
        front = g["in_front"][a:b]
        counts.add(int(front.sum()) % 2 if front.any() else -1)
        if not front.any():
            assert np.isnan(g["median_angle"][p])
            continue
        want = np.median(g["angle"][a:b][front])
        assert np.float64(g["median_angle"][p]).tobytes() == np.float64(want).tobytes(), (p, specs[p])
    assert counts == {0, 1, -1}


@pytest.mark.gpu
def test_degenerate_pairs_and_offsets():
    import torch
    from pydegensac_b200 import _cabi
    from pydegensac_b200.matching import pose_from_fundamental_ragged
    lengths = [300, 200, 150, 250, 0, 120]
    p1, p2, F, off = _batch(lengths, 400)
    F[1] = 0.0
    F[2, 1, 2] = np.nan
    d1, d2, dF, doff, dK = _dev(p1, p2, F, off, _K)
    g = _np(pose_from_fundamental_ragged(dF, dK, dK, d1, d2, doff))
    clean = [0, 3, 5]
    ref = _np(pose_from_fundamental_ragged(dF[clean], dK, dK, *(_dev(
        np.concatenate([p1[off[i]:off[i + 1]] for i in clean]), np.concatenate([p2[off[i]:off[i + 1]] for i in clean]))),
        torch.tensor(np.r_[0, np.cumsum([lengths[i] for i in clean])], dtype=torch.int32, device="cuda:0")))
    rows = np.concatenate([np.arange(off[i], off[i + 1]) for i in clean])
    for k in ("R", "t", "good", "median_angle"):
        assert np.array_equal(g[k][clean], ref[k]), k
    for k in ("points", "in_front", "angle"):
        assert np.array_equal(g[k][rows], ref[k]), k
    for p in (1, 2):
        a, b = off[p], off[p + 1]
        assert not g["R"][p].any() and not g["t"][p].any() and g["good"][p] == 0 and np.isnan(g["median_angle"][p])
        assert np.isnan(g["points"][a:b]).all() and np.isnan(g["angle"][a:b]).all() and not g["in_front"][a:b].any()
    assert g["good"][4] == 0 and np.isnan(g["median_angle"][4])
    # malformed device offsets: negative, decreasing or past the rows make empty pairs whose rows stay untouched
    rows_n = len(p1)
    bad_off = np.array([0, 300, -5, 300 + 200 + 150, rows_n + 10], dtype=np.int32)
    P = 4
    d_off, = _dev(bad_off)
    out = dict(R=torch.full((P, 9), 7.0, dtype=torch.float64, device="cuda:0"),
               t=torch.full((P, 3), 7.0, dtype=torch.float64, device="cuda:0"),
               good=torch.full((P,), 7, dtype=torch.int32, device="cuda:0"),
               points=torch.full((rows_n, 3), 7.0, dtype=torch.float64, device="cuda:0"),
               in_front=torch.full((rows_n,), 7, dtype=torch.uint8, device="cuda:0"),
               angle=torch.full((rows_n,), 7.0, dtype=torch.float64, device="cuda:0"),
               median=torch.full((P,), 7.0, dtype=torch.float64, device="cuda:0"))
    Fb = dF[[0, 3, 3, 3]].contiguous()
    vp = ctypes.c_void_p
    rc = _cabi.lib().dgb200_pose_from_fundamental_ragged_dev(
        vp(Fb.data_ptr()), vp(dK.data_ptr()), vp(dK.data_ptr()), 0, vp(d1.data_ptr()), vp(d2.data_ptr()),
        vp(d_off.data_ptr()), P, rows_n, 2, None, *[vp(out[k].data_ptr()) for k in ("R", "t", "good", "points",
                                                                                     "in_front", "angle", "median")],
        vp(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    o = {k: v.cpu().numpy() for k, v in out.items()}
    assert np.array_equal(o["good"], [g["good"][0], 0, 0, 0])
    assert np.array_equal(o["R"][0], g["R"][0].ravel()) and np.isnan(o["median"][1:]).all()
    assert np.array_equal(o["points"][:300], g["points"][:300]) and np.array_equal(o["angle"][:300], g["angle"][:300])
    assert (o["points"][300:] == 7.0).all() and (o["in_front"][300:] == 7).all() and (o["angle"][300:] == 7.0).all()


def _multiview_pose(n_img, n_pts, n_clutter, D, seed):
    """n_img views of one set of 3-D points (keypoints, descriptors: shared code + noise per point) with the planted
    pose (R_i, t_i) of every view: x_i ~ R_i X + t_i.  The points span a wide field and a 6:1 depth range, so that the
    F found by the RANSAC fixes the direction of t well (a narrow field leaves its forward component loose)."""
    rng = np.random.default_rng(seed)
    X = np.c_[rng.uniform(-4, 4, n_pts), rng.uniform(-4, 4, n_pts), rng.uniform(2, 12, n_pts)]
    code = rng.normal(size=(n_pts, D)).astype(np.float32)
    Rs, ts, kps, descs = [], [], [], []
    for i in range(n_img):
        R = _rot("y", 0.08 * i) @ _rot("x", 0.02 * i)
        t = np.array([0.6 * i, 0.05 * i, 0.1 * i])
        x = (_K @ (R @ X.T + t[:, None])).T
        x = x[:, :2] / x[:, 2:3] + 0.1 * rng.normal(size=(n_pts, 2))
        kp = np.r_[x, rng.uniform(0, 640, (n_clutter, 2))]
        d = np.r_[code + 0.15 * rng.normal(size=code.shape).astype(np.float32),
                  rng.normal(size=(n_clutter, D)).astype(np.float32)]
        perm = rng.permutation(n_pts + n_clutter)
        kps.append(kp[perm]); descs.append(d[perm]); Rs.append(R); ts.append(t)
    return kps, descs, Rs, ts


@pytest.mark.gpu
def test_pipeline_match_ransac_pose_without_sync():
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import match_descriptors_batch, pose_from_fundamental_ragged
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
    finally:
        torch.cuda.set_sync_debug_mode(0)
    g = _np(pose)
    off = m.offsets.cpu().numpy()
    for p, (i, j) in enumerate(pairs):
        R = Rs[j] @ Rs[i].T
        t = ts[j] - R @ ts[i]
        t = t / np.linalg.norm(t)
        dR = g["R"][p] @ R.T
        assert np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)) < 1e-2, p
        assert np.linalg.norm(g["t"][p] - t) < 1e-2, p
        a, b = off[p], off[p + 1]
        assert g["good"][p] == g["in_front"][a:b].sum() > 0.5 * mask[a:b].sum().item()
        assert g["median_angle"][p] > 0
