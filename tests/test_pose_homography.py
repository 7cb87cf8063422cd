"""Pose and scene plane from homographies over ragged batches (matching.pose_from_homography_ragged,
dgb200_pose_from_homography_ragged_dev): the numpy oracle pinned to cv2.decomposeHomographyMat and to planted planar
scenes; argument refusals; and on the GPU agreement with the oracle, the exact median, degenerate pairs, independence
of the batch, and the no-sync pipeline match -> ragged H -> pose -> refinement."""
import ctypes
import os

import numpy as np
import pytest

from pydegensac_b200.scenes import _K, _rot
from tests import pose_homography_np as PH
from tests.pose_ragged_np import rows_under_pose

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")
K2_OTHER = np.array([[560.0, 0.0, 330.0], [0.0, 540.0, 235.0], [0.0, 0.0, 1.0]])


def _pose(rng, min_turn=0.0):
    turn = rng.choice([-1.0, 1.0]) * rng.uniform(min_turn, 0.3)
    R = _rot("z", rng.uniform(-0.1, 0.1)) @ _rot("y", turn) @ _rot("x", rng.uniform(-0.1, 0.1))
    T = np.array([rng.uniform(0.5, 1.5), rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3)])
    return R, T


def _plane_scene(n, seed, n_behind=0, noise=0.0, K2=_K):
    """Two views of n points on a plane n^T X = d (camera 1's frame) with a KNOWN pose x2 ~ R x1 + T: pixels p1, p2,
    R, unit t, the plane (n, d) in baseline units, the points X / |T| and the pixel homography H (x2 ~ H x1).  The last
    n_behind points lie on the plane in front of camera 1 but behind camera 2."""
    rng = np.random.default_rng(seed)
    R, T = _pose(rng, 0.2 if n_behind else 0.0)     # a turn of 0.2 rad or more puts part of the plane behind camera 2
    tilt = 0.05 if n_behind else 0.3                 # along x: keeps that part of the plane in front of camera 1
    nrm = np.array([rng.uniform(-tilt, tilt), rng.uniform(-0.3, 0.3), 1.0])
    nrm /= np.linalg.norm(nrm)
    d = rng.uniform(4.0, 8.0)

    def on_plane(xy):
        return np.c_[xy, (d - xy @ nrm[:2]) / nrm[2]]
    X = on_plane(np.c_[rng.uniform(-2, 2, n), rng.uniform(-2, 2, n)])
    if n_behind:
        Y = on_plane(np.c_[rng.uniform(-200, 200, 8000), rng.uniform(-2, 2, 8000)])
        Y = Y[(Y[:, 2] > 0.5) & ((Y @ R.T + T)[:, 2] < -0.5)][:n_behind]
        assert len(Y) == n_behind
        X = np.r_[X, Y]
    x1 = X @ _K.T
    x2 = (X @ R.T + T) @ K2.T
    p1 = x1[:, :2] / x1[:, 2:3] + noise * rng.normal(size=(len(X), 2))
    p2 = x2[:, :2] / x2[:, 2:3]
    H = K2 @ (R + np.outer(T, nrm) / d) @ np.linalg.inv(_K)
    nt = np.linalg.norm(T)
    return p1, p2, R, T / nt, np.r_[nrm, d / nt], X / nt, H


def _rotation_scene(n, seed, wobble=0.0, noise=0.0, K2=_K):
    """Two views from one centre: pixels p1, p2, R and H = K2 R (I + E) K1^-1, E symmetric with |E_ij| <= wobble (so
    max |Hn^T Hn - I| is about 2 wobble).  Every point is in front of both cameras."""
    rng = np.random.default_rng(seed)
    R = _rot("y", rng.uniform(-0.4, 0.4)) @ _rot("x", rng.uniform(-0.1, 0.1))
    X = np.c_[rng.uniform(-2, 2, n), rng.uniform(-2, 2, n), rng.uniform(3, 10, n)]
    x1 = X @ _K.T
    x2 = (X @ R.T) @ K2.T
    p1 = x1[:, :2] / x1[:, 2:3] + noise * rng.normal(size=(n, 2))
    p2 = x2[:, :2] / x2[:, 2:3]
    E = rng.uniform(-wobble, wobble, (3, 3))
    E = (E + E.T) / 2
    return p1, p2, R, K2 @ R @ (np.eye(3) + E) @ np.linalg.inv(_K)


def _rot_err(A, B):
    return np.arccos(np.clip((np.trace(A @ B.T) - 1) / 2, -1, 1))


# ------------------------------------------------------------------------------------------------ CPU
def test_oracle_candidates_equal_cv2_in_order():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(1)
    worst = 0.0
    for s in range(200):
        R, T = _pose(rng)
        nrm = rng.normal(size=3)
        nrm[2] = abs(nrm[2]) + 0.5
        nrm /= np.linalg.norm(nrm)
        K2 = K2_OTHER if s % 2 else _K
        H = K2 @ (R + np.outer(T, nrm) / rng.uniform(2, 10)) @ np.linalg.inv(_K)
        H *= (-1) ** (s // 2) * rng.uniform(0.01, 100)             # positive and negative scales
        rot, cands = PH.candidates(H, _K, K2)
        assert not rot
        k, Rs, ts, ns = cv2.decomposeHomographyMat(PH.normalised(H, _K, K2), np.eye(3))
        assert k == 4
        for (Ro, to, no), Rc, tc, nc in zip(cands, Rs, ts, ns):
            worst = max(worst, np.abs(Ro - Rc).max(), np.abs(to - tc.ravel()).max(), np.abs(no - nc.ravel()).max())
            assert abs(np.linalg.det(Ro) - 1) < 1e-12
            assert np.abs(Ro + np.outer(to, no) - PH.normalised(H, _K, K2)).max() < 1e-12
    assert worst <= 1e-9, worst


def test_oracle_rotation_rule_against_cv2():
    cv2 = pytest.importorskip("cv2")
    for s in range(40):
        K2 = K2_OTHER if s % 2 else _K
        wobble = 2.5e-4 if s < 20 else 2e-3       # max |S| about 5e-4 (a rotation) or 4e-3 (not one)
        _, _, R, H = _rotation_scene(10, s, wobble=wobble, K2=K2)
        H = H * (-1) ** (s // 2) * 3.0             # -H too: the sign rule gives det R = +1
        Hn = PH.normalised(H, _K, K2)
        smax = np.abs(Hn.T @ Hn - np.eye(3)).max()
        rot, cands = PH.candidates(H, _K, K2)
        k, Rs, ts, _ = cv2.decomposeHomographyMat(Hn, np.eye(3))
        assert rot == (s < 20) and (smax < 7e-4 if rot else smax > 1.5e-3), (s, smax)
        assert k == (1 if rot else 4)
        if rot:
            Rr = cands[0][0]
            assert abs(np.linalg.det(Rr) - 1) < 1e-12 and np.abs(Rr.T @ Rr - np.eye(3)).max() < 1e-12
            assert np.abs(Rr - Rs[0]).max() <= 2e-3 and not ts[0].any()
            assert _rot_err(Rr, R) < 2e-3


def test_oracle_planted_planar_scenes():
    lengths = [300, 0, 120, 57, 200, 80]
    scenes = [_plane_scene(n - 6, 10 + s, n_behind=6, K2=K2_OTHER) if n else None for s, n in enumerate(lengths)]
    p1 = np.concatenate([s[0] for s in scenes if s]); p2 = np.concatenate([s[1] for s in scenes if s])
    H = np.stack([s[6] if s else np.eye(3) for s in scenes])
    off = np.r_[0, np.cumsum(lengths)]
    o = PH.pose_h_ragged(H, _K, K2_OTHER, p1, p2, off)
    separated = 0
    for p, s in enumerate(scenes):
        a, b = off[p], off[p + 1]
        if s is None:
            assert not o["good"][p].any() and np.isnan(o["median_angle"][p])
            continue
        _, _, R, t, plane, X, _ = s
        assert not o["rotation_only"][p]
        hit = [c for c in range(2) if _rot_err(o["R"][p, c], R) < 1e-9 and np.abs(o["t"][p, c] - t).max() < 1e-9
               and np.abs(o["plane"][p, c] - plane).max() < 1e-9]
        assert len(hit) == 1, p
        if o["good"][p, 0] > o["good"][p, 1]:
            assert hit == [0], p
            separated += 1
        for c in range(2):                          # every candidate's points lie on its own plane
            pts = rows_under_pose(o["R"][p, c], o["t"][p, c], _K, K2_OTHER, p1[a:b], p2[a:b])[0]
            n_c, d_c = o["plane"][p, c, :3], o["plane"][p, c, 3]
            assert d_c > 0 and abs(np.linalg.norm(n_c) - 1) < 1e-12
            assert np.all(np.abs(pts @ n_c - d_c) <= 1e-9 * np.maximum(d_c, np.linalg.norm(pts, axis=1))), (p, c)
        if hit == [0]:
            front = o["in_front"][a:b]
            assert not front[-6:].any() and front[:-6].all() and o["good"][p, 0] == b - a - 6
            # (the six far points behind camera 2 triangulate at grazing angles: their in_front is what is checked)
            err = np.linalg.norm(o["points"][a:b] - X, axis=1)[:-6]
            assert np.all(err <= 1e-9 * np.linalg.norm(X[:-6], axis=1))
        else:
            assert o["good"][p, 1] == b - a - 6
    assert separated >= 1


def test_homography_pose_entry_point_rejects_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    names = ["H", "K1", "K2", "x1y1", "x2y2", "offsets", "mask", "R", "t", "plane", "good", "rotation_only", "points",
             "in_front", "angle", "median"]

    def call(n_pairs=3, rows=10, dim=2, **null):
        b = {k: (None if null.get(k) else fake) for k in names}
        return L.dgb200_pose_from_homography_ragged_dev(b["H"], b["K1"], b["K2"], 0, b["x1y1"], b["x2y2"], b["offsets"],
                                                        n_pairs, rows, dim, b["mask"], b["R"], b["t"], b["plane"],
                                                        b["good"], b["rotation_only"], b["points"], b["in_front"],
                                                        b["angle"], b["median"], None)

    for k in names:
        if k not in ("mask", "good"):              # the two optional buffers
            assert call(**{k: True}) == -1, k
    for n_pairs in (0, -1):
        assert call(n_pairs=n_pairs) == -1
    assert call(rows=-1) == -1
    for dim in (1, 0, -2):
        assert call(dim=dim) == -1


def test_homography_pose_python_argument_errors():
    import torch
    from pydegensac_b200.matching import pose_from_homography_ragged as phr
    H = torch.zeros((2, 3, 3), dtype=torch.float64)
    K = torch.eye(3, dtype=torch.float64)
    p = torch.zeros((10, 2), dtype=torch.float64)
    off = torch.tensor([0, 4, 10], dtype=torch.int32)
    bad = [
        dict(H=torch.zeros((2, 8))), dict(H=torch.zeros((0, 9))), dict(H=torch.zeros(9)), dict(H=np.zeros((2, 9))),
        dict(H=torch.zeros((2, 9), dtype=torch.int64)),
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
        args = dict(H=H, K1=K, K2=K, pts1=p, pts2=p, offsets=off, mask=None)
        args.update(kw)
        with pytest.raises(ValueError):
            phr(**args)
    if torch.cuda.is_available():
        dev = torch.device("cuda:0")
        with pytest.raises(ValueError, match="device"):
            phr(H.to(dev), K, K.to(dev), p.to(dev), p.to(dev), off.to(dev))


# ------------------------------------------------------------------------------------------------ GPU
LENGTHS = [0, 1, 7, 33, 400, 2048, 4097, 20000]


def _batch(lengths, seed, noise=0.3, K2=_K, rotation_every=3):
    """A ragged batch of noisy planar scenes with every rotation_every-th pair a pure rotation (a wobble of 2e-4, inside
    the rule, on every other one); H the planted homography."""
    ps1, ps2, Hs = [], [], []
    for i, n in enumerate(lengths):
        if i % rotation_every == 1:
            p1, p2, _, H = _rotation_scene(max(n, 8), seed + i, wobble=2e-4 * (i % 2), noise=noise, K2=K2)
        else:
            p1, p2, _, _, _, _, H = _plane_scene(max(n, 8), seed + i, noise=noise, K2=K2)
        ps1.append(p1[:n]); ps2.append(p2[:n]); Hs.append(H)
    off = np.r_[0, np.cumsum(lengths)].astype(np.int32)
    return np.concatenate(ps1), np.concatenate(ps2), np.stack(Hs), off


def _dev(*xs):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0") for x in xs]


def _np(pose):
    return {k: v.cpu().numpy() for k, v in pose._asdict().items() if v is not None}


def _same_bytes(g, h):
    for k in g:
        assert g[k].tobytes() == h[k].tobytes(), k


@pytest.mark.gpu
@pytest.mark.parametrize("per_pair_K", [False, True])
def test_against_oracle(per_pair_K):
    import torch
    from pydegensac_b200.matching import pose_from_homography_ragged
    p1, p2, H, off = _batch(LENGTHS, 500, noise=0.5, K2=K2_OTHER)
    H[2] *= -3.0                                     # a negative scale
    mask = np.ones(len(p1), bool); mask[1::4] = False
    P = len(LENGTHS)
    if per_pair_K:
        K1 = np.stack([_K * [[1 + 1e-5 * p], [1], [1]] for p in range(P)])   # small: rotations stay rotations
        K1[:, 2] = [0, 0, 1]
        K2 = np.stack([K2_OTHER] * P)
    else:
        K1, K2 = _K, K2_OTHER
    d1, d2, dH, doff, dm, dK1, dK2 = _dev(p1, p2, H, off, mask, K1, K2)
    g = _np(pose_from_homography_ragged(dH, dK1, dK2, d1, d2, doff, dm))
    o = PH.pose_h_ragged(H, K1, K2, p1, p2, off, mask)
    assert np.array_equal(g["rotation_only"], o["rotation_only"])
    assert g["rotation_only"].any() and not g["rotation_only"].all()
    assert np.array_equal(g["good"], o["good"]), (g["good"], o["good"])
    for k in ("R", "t", "plane"):
        assert np.array_equal(np.isnan(g[k]), np.isnan(o[k])), k
        err = np.nan_to_num(np.abs(g[k] - o[k]))
        assert err.max() <= 1e-9, (k, err.max())
    K1s, K2s = np.broadcast_to(K1, (P, 3, 3)), np.broadcast_to(K2, (P, 3, 3))
    for p in range(P):
        a, b = off[p], off[p + 1]
        if a == b:
            assert not g["good"][p].any() and np.isnan(g["median_angle"][p])
            continue
        R0, t0 = g["R"][p, 0], g["t"][p, 0]
        pts, front, ang, l1, l2 = rows_under_pose(R0, t0, K1s[p], K2s[p], p1[a:b], p2[a:b], mask[a:b])
        err = np.abs(g["angle"][a:b] - ang) / np.abs(ang)
        assert err.max() <= 1e-9, (p, err.max())
        if g["rotation_only"][p]:
            assert np.isnan(g["points"][a:b]).all()
            assert np.array_equal(g["in_front"][a:b], o["in_front"][a:b]), p
        else:
            err = np.linalg.norm(g["points"][a:b] - pts, axis=1) / np.linalg.norm(pts, axis=1)
            assert err.max() <= 1e-9, (p, err.max())
            scale = max(1.0, np.median(np.abs(np.r_[l1, l2])))
            near = (np.abs(l1) < 1e-9 * scale) | (np.abs(l2) < 1e-9 * scale)
            assert np.array_equal(g["in_front"][a:b][~near], front[~near]), p
        assert g["good"][p, 0] == g["in_front"][a:b].sum()
        assert np.all((g["angle"][a:b] >= 0) & (g["angle"][a:b] <= np.pi))
    if per_pair_K:                                   # per-pair K given as [P,3,3] equal to a shared one: same bytes
        dK = torch.from_numpy(_K).to("cuda:0")
        shared = _np(pose_from_homography_ragged(dH, dK, dK2[0], d1, d2, doff, dm))
        stacked = _np(pose_from_homography_ragged(dH, torch.stack([dK] * P), dK2, d1, d2, doff, dm))
        _same_bytes(shared, stacked)


@pytest.mark.gpu
def test_median_is_exact():
    from pydegensac_b200.matching import pose_from_homography_ragged
    rng = np.random.default_rng(7)
    l1, l2, Hs, masks = [], [], [], []
    specs = [(101, "all"), (100, "all"), (2, "all"), (1, "all"), (20000, "all"), (19999, "all"), (3000, "holes"),
             (50, "dup"), (51, "dup"), (40, "none"), (64, "dup2"), (1000, "rot"), (999, "rot")]
    for i, (n, kind) in enumerate(specs):
        if kind == "rot":
            p1, p2, _, H = _rotation_scene(n, 300 + i, noise=0.3)
        else:
            p1, p2, _, _, _, _, H = _plane_scene(max(n, 8), 300 + i, noise=0.3)
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
        l1.append(p1); l2.append(p2); Hs.append(H); masks.append(m)
    off = np.r_[0, np.cumsum([len(x) for x in l1])].astype(np.int32)
    d1, d2, dH, doff, dm, dK = _dev(np.concatenate(l1), np.concatenate(l2), np.stack(Hs), off, np.concatenate(masks), _K)
    g = _np(pose_from_homography_ragged(dH, dK, dK, d1, d2, doff, dm))
    assert g["rotation_only"][-2:].all() and not g["rotation_only"][:-2].any()
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
    from pydegensac_b200.matching import pose_from_homography_ragged
    lengths = [300, 200, 150, 250, 0, 120]
    p1, p2, H, off = _batch(lengths, 400)
    H[1] = 0.0
    H[2, 1, 2] = np.nan
    d1, d2, dH, doff, dK = _dev(p1, p2, H, off, _K)
    g = _np(pose_from_homography_ragged(dH, dK, dK, d1, d2, doff))
    for p in (1, 2):
        a, b = off[p], off[p + 1]
        assert not g["R"][p].any() and not g["t"][p].any() and np.isnan(g["plane"][p]).all()
        assert not g["good"][p].any() and not g["rotation_only"][p] and np.isnan(g["median_angle"][p])
        assert np.isnan(g["points"][a:b]).all() and np.isnan(g["angle"][a:b]).all() and not g["in_front"][a:b].any()
    assert not g["good"][4].any() and np.isnan(g["median_angle"][4])      # a model but no row
    # malformed device offsets: negative, decreasing or past the rows make empty pairs whose rows stay untouched
    rows_n = len(p1)
    bad_off = np.array([0, 300, -5, 300 + 200 + 150, rows_n + 10], dtype=np.int32)
    P = 4
    d_off, = _dev(bad_off)
    f64, dev = torch.float64, "cuda:0"
    out = dict(R=torch.full((P, 18), 7.0, dtype=f64, device=dev), t=torch.full((P, 6), 7.0, dtype=f64, device=dev),
               plane=torch.full((P, 8), 7.0, dtype=f64, device=dev),
               good=torch.full((P, 2), 7, dtype=torch.int32, device=dev),
               rotation_only=torch.full((P,), 7, dtype=torch.uint8, device=dev),
               points=torch.full((rows_n, 3), 7.0, dtype=f64, device=dev),
               in_front=torch.full((rows_n,), 7, dtype=torch.uint8, device=dev),
               angle=torch.full((rows_n,), 7.0, dtype=f64, device=dev),
               median=torch.full((P,), 7.0, dtype=f64, device=dev))
    Hb = dH[[0, 3, 3, 3]].contiguous()
    vp = ctypes.c_void_p
    rc = _cabi.lib().dgb200_pose_from_homography_ragged_dev(
        vp(Hb.data_ptr()), vp(dK.data_ptr()), vp(dK.data_ptr()), 0, vp(d1.data_ptr()), vp(d2.data_ptr()),
        vp(d_off.data_ptr()), P, rows_n, 2, None,
        *[vp(out[k].data_ptr()) for k in ("R", "t", "plane", "good", "rotation_only", "points", "in_front", "angle",
                                          "median")],
        vp(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    o = {k: v.cpu().numpy() for k, v in out.items()}
    assert np.array_equal(o["good"][0], g["good"][0]) and not o["good"][1:, 0].any()
    assert np.array_equal(o["R"][0], g["R"][0].ravel()) and np.isnan(o["median"][1:]).all()
    assert np.array_equal(o["points"][:300], g["points"][:300]) and np.array_equal(o["angle"][:300], g["angle"][:300])
    assert (o["points"][300:] == 7.0).all() and (o["in_front"][300:] == 7).all() and (o["angle"][300:] == 7.0).all()


@pytest.mark.gpu
def test_pair_alone_in_batch_and_rerun_give_the_same_bytes():
    import torch
    from pydegensac_b200.matching import pose_from_homography_ragged
    lengths = [900, 30, 2500, 0, 400, 1200]
    p1, p2, H, off = _batch(lengths, 600, rotation_every=2)
    mask = np.ones(len(p1), bool); mask[2::7] = False
    d1, d2, dH, doff, dm, dK = _dev(p1, p2, H, off, mask, _K)
    g = _np(pose_from_homography_ragged(dH, dK, dK, d1, d2, doff, dm))
    _same_bytes(g, _np(pose_from_homography_ragged(dH, dK, dK, d1, d2, doff, dm)))
    for p in range(len(lengths)):
        a, b = int(off[p]), int(off[p + 1])
        one = _np(pose_from_homography_ragged(dH[p:p + 1], dK, dK, d1[a:b], d2[a:b],
                                              torch.tensor([0, b - a], dtype=torch.int32, device="cuda:0"), dm[a:b]))
        for k in ("R", "t", "plane", "good", "rotation_only", "median_angle"):
            assert one[k][0].tobytes() == g[k][p].tobytes(), (p, k)
        for k in ("points", "in_front", "angle"):
            assert one[k].tobytes() == g[k][a:b].tobytes(), (p, k)


def _multiview_plane(n_img, n_pts, n_clutter, D, seed):
    """n_img views of points on one tilted plane (keypoints, descriptors: shared code + noise per point) with the
    planted pose (R_i, t_i) of every view: x_i ~ R_i X + t_i."""
    rng = np.random.default_rng(seed)
    nw = np.array([0.15, -0.1, 1.0]); nw /= np.linalg.norm(nw)
    xy = np.c_[rng.uniform(-4, 4, n_pts), rng.uniform(-3, 3, n_pts)]
    X = np.c_[xy, (7.0 - xy @ nw[:2]) / nw[2]]
    code = rng.normal(size=(n_pts, D)).astype(np.float32)
    Rs, ts, kps, descs = [], [], [], []
    for i in range(n_img):
        R = _rot("y", 0.08 * i) @ _rot("x", 0.03 * i)
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
def test_pipeline_match_ransac_pose_refine_without_sync():
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import match_descriptors_batch, pose_from_homography_ragged, refine_pose_ragged
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
        pose = pose_from_homography_ragged(H, K, K, m.pts1, m.pts2, m.offsets, mask)
        fine = refine_pose_ragged(pose.R[:, 0], pose.t[:, 0], K, K, m.pts1, m.pts2, m.offsets, pose.in_front)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    g, f = _np(pose), _np(fine)
    off = m.offsets.cpu().numpy()
    for p, (i, j) in enumerate(pairs):
        R = Rs[j] @ Rs[i].T
        t = ts[j] - R @ ts[i]
        t = t / np.linalg.norm(t)
        assert not g["rotation_only"][p]
        errs = [_rot_err(g["R"][p, c], R) + np.linalg.norm(g["t"][p, c] - t) for c in range(2)]
        assert min(errs) < 2e-2, (p, errs)
        a, b = off[p], off[p + 1]
        assert g["good"][p, 0] == g["in_front"][a:b].sum() > 0.5 * mask[a:b].sum().item()
        assert g["median_angle"][p] > 0 and (g["plane"][p, :, 3] > 0).all()
        assert f["cost"][p] <= f["cost0"][p]
