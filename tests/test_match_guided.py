"""Guided matching (match_descriptors_guided and its C entry points): the numpy oracle pinned to the engine's host
build, to the unguided oracle and to cv2; argument checks; a repeated-texture scene on which the gate brings true
matches back; and on the GPU exact agreement of the batched guided matcher with the oracle, threshold boundaries, an
open gate against the unguided matcher, and the pipeline unguided -> ragged F / H -> guided."""
import ctypes
import os

import numpy as np
import pytest

from pydegensac_b200.scenes import _K, _rot
from tests import guided_np as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")


def _q(x):
    """float32 values on a grid of 1/8: every squared L2 distance of such rows (|values| < 8, D <= 256) is exact in
    FP32 in any summation order, so the float64 oracle equals the kernel's FP32 distances bit for bit"""
    return (np.clip(np.round(np.asarray(x) * 8), -60, 60) / 8).astype(np.float32)


def scene(n_img, n_pts, n_clutter, D, seed, planar=False, n_alike=4, binary=False):
    """Repeated texture seen from n_img views.  The n_pts points come in groups of n_alike look-alikes: one texture
    code per group, a small point-specific change, and noise per view; every point's true match thus has n_alike - 1
    distractors elsewhere in the image.  Clutter: random descriptors at random places.  planar: the points lie on a
    plane and the views are related by homographies.  binary: uint8 codes of D bytes (bits flipped per point and view)
    in place of float32 rows.
    Returns keypoints, descriptors, where (row of point k in view i) and model(i, j): the planted F (x_j^T F x_i = 0)
    or H (x_j ~ H x_i)."""
    rng = np.random.default_rng(seed)
    n_grp = -(-n_pts // n_alike)
    grp = np.arange(n_pts) // n_alike
    if binary:
        base = rng.integers(0, 256, (n_grp, D), dtype=np.uint8)[grp]
        point = _flip(base, 0.02, rng)
    else:
        point = rng.normal(size=(n_grp, D))[grp] + 0.1 * rng.normal(size=(n_pts, D))
    if planar:
        x0 = np.c_[rng.uniform(20, 620, n_pts), rng.uniform(20, 460, n_pts)]
        Hs = []
        for i in range(n_img):
            H = np.eye(3) + np.r_[rng.normal(0, 0.05, 6), rng.normal(0, 1e-4, 2), 0].reshape(3, 3)
            H[:2, 2] = rng.normal(0, 20, 2)
            Hs.append(H if i else np.eye(3))
    else:
        X = np.c_[rng.uniform(-2, 2, n_pts), rng.uniform(-1.5, 1.5, n_pts), rng.uniform(5, 10, n_pts)]
        Rs = [_rot("y", 0.08 * i) @ _rot("x", 0.02 * i) for i in range(n_img)]
        ts = [np.array([0.6 * i, 0.05 * i, 0.1 * i]) for i in range(n_img)]
    kps, descs, where = [], [], []
    for i in range(n_img):
        if planar:
            h = np.c_[x0, np.ones(n_pts)] @ Hs[i].T
        else:
            h = (_K @ (Rs[i] @ X.T + ts[i][:, None])).T
        x = h[:, :2] / h[:, 2:3] + 0.1 * rng.normal(size=(n_pts, 2))
        kp = np.r_[x, np.c_[rng.uniform(0, 640, n_clutter), rng.uniform(0, 480, n_clutter)]]
        if binary:
            d = np.r_[_flip(point, 0.06, rng), rng.integers(0, 256, (n_clutter, D), dtype=np.uint8)]
        else:
            d = _q(np.r_[point + 0.4 * rng.normal(size=point.shape), rng.normal(size=(n_clutter, D))])
        perm = rng.permutation(n_pts + n_clutter)
        kps.append(kp[perm]); descs.append(d[perm])
        inv = np.empty_like(perm); inv[perm] = np.arange(len(perm))
        where.append(inv[:n_pts])
    Ki = np.linalg.inv(_K)

    def model(i, j):
        if planar:
            return Hs[j] @ np.linalg.inv(Hs[i])
        R = Rs[j] @ Rs[i].T
        t = ts[j] - R @ ts[i]
        tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
        return Ki.T @ tx @ R @ Ki
    return kps, descs, where, model


def _flip(codes, p, rng):
    bits = np.unpackbits(codes, axis=1)
    return np.packbits(bits ^ (rng.random(bits.shape) < p), axis=1)


def _true_count(q, t, wq, wt):
    planted = dict(zip(wq.tolist(), wt.tolist()))
    return sum(planted.get(a) == b for a, b in zip(q.tolist(), t.tolist()))


# ------------------------------------------------------------------------------------------------ CPU
def test_f_gate_is_the_engines_sampson_residual_bit_for_bit():
    from tests.hostemu import emu
    L = emu.lib()
    L.emu_f_resid.restype = ctypes.c_double
    L.emu_f_resid.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_double)] + [ctypes.c_double] * 4
    rng = np.random.default_rng(11)
    kps, _, where, model = scene(2, 200, 0, 8, 4)
    F = model(0, 1)
    n = 100000
    xq = rng.uniform(0, 640, n); yq = rng.uniform(0, 480, n)
    xt = rng.uniform(0, 640, n); yt = rng.uniform(0, 480, n)
    # half of the train points on (or within a fraction of a pixel of) the query's epipolar line
    near = np.arange(n) < n // 2
    l = np.c_[xq, yq, np.ones(n)] @ F.T
    xt[near] = rng.uniform(0, 640, near.sum())
    yt[near] = -(l[near, 0] * xt[near] + l[near, 2]) / l[near, 1] + rng.normal(0, 0.5, near.sum())
    for Fm in (F, rng.normal(size=(3, 3))):
        e = G.f_sampson(Fm, xq, yq, xt, yt)
        fp = Fm.reshape(9).ctypes.data_as(ctypes.POINTER(ctypes.c_double))
        ref = np.array([L.emu_f_resid(0, fp, a, b, c, d) for a, b, c, d in zip(xq, yq, xt, yt)])
        assert np.array_equal(e.view(np.int64), ref.view(np.int64))
    assert np.sum(G.f_sampson(F, xq, yq, xt, yt)[near] <= 1.0) > n // 8


def test_f_pretest_never_rejects_an_exact_accept():
    rng = np.random.default_rng(12)
    n = 1 << 20
    th = np.exp(rng.uniform(np.log(1e-6), np.log(1e6), n))
    th[:1000] = np.float64(np.finfo(np.float64).tiny) * rng.uniform(0.1, 4, 1000)   # subnormal and near-subnormal
    th[1000:2000] = 0.0
    den = np.exp(rng.uniform(np.log(1e-12), np.log(1e12), n))
    # numerators within a few ulps of th * den, so that the quotient lands within a few ulps of th
    num = th * den * (1 + rng.integers(-6, 7, n) * 2.0 ** -52)
    num[::7] = np.nextafter(num[::7], np.inf)
    with np.errstate(all="ignore"):
        q = num / den
        exact = q <= th
    rej = G.f_pretest_rejects(num, den, th)
    assert not np.any(rej & exact)
    with np.errstate(all="ignore"):
        assert np.sum(np.abs(q / th - 1) < 1e-14) > n // 2      # most cases sit at the boundary
    # clear misses are rejected without the division
    assert np.all(G.f_pretest_rejects(4 * th[2000:] * den[2000:], den[2000:], th[2000:]))
    # NaN falls through
    assert not G.f_pretest_rejects(np.nan, 1.0, 1.0) and not G.f_pretest_rejects(1.0, np.nan, 1.0)


def test_open_gate_oracle_equals_unguided_oracle():
    from oracle.frontend_np import match_descriptors as match_np
    from tests.test_match_hamming import match_binary_np
    rng = np.random.default_rng(13)
    kps, descs, _, model = scene(2, 300, 100, 32, 5)
    for ratio in (0.5, 0.75):        # ratios whose square rounds alike in FP32 and FP64
        for mutual in (False, True):
            q, t, _ = match_np(descs[0], descs[1], ratio, mutual)
            gq, gt = G.match_descriptors_guided(descs[0], descs[1], kps[0], kps[1], np.eye(3), "H", 1e6, ratio, mutual)
            assert np.array_equal(q, gq) and np.array_equal(t, gt)
    b1, b2 = (rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in (200, 300))
    k1, k2 = rng.uniform(0, 640, (200, 2)), rng.uniform(0, 640, (300, 2))
    for mutual in (False, True):
        q, t, _ = match_binary_np(b1, b2, 0.9, mutual)
        gq, gt = G.match_descriptors_guided(b1, b2, k1, k2, model(0, 1), "F", 1e12, 0.9, mutual, hamming=True)
        assert np.array_equal(q, gq) and np.array_equal(t, gt)


@pytest.mark.parametrize("B", [32, 61])
def test_hamming_guided_oracle_agrees_with_cv2_masked_knn(B):
    cv2 = pytest.importorskip("cv2")
    from tests.test_match_hamming import _planted, _tie_heavy
    rng = np.random.default_rng(B + 1)
    bf = cv2.BFMatcher(cv2.NORM_HAMMING)
    k1, k2 = rng.uniform(0, 640, (300, 2)), rng.uniform(0, 640, (400, 2))
    H = np.array([[1.0, 0.02, 5], [-0.01, 1.0, -3], [0, 0, 1]])
    for d1, d2 in (_planted([300, 400], B, rng), _tie_heavy([300, 400], B, rng)):
        dist = G.distances(d1, d2, hamming=True)
        for px_th in (20.0, 60.0):
            admit = G.gate(H, "H", k1, k2, px_th)
            c = admit.sum(1)
            assert c.max() >= 2 and (px_th > 20 or (np.any(c == 1) and np.any(c == 0)))   # 0, 1 and 2+ candidates
            knn = bf.knnMatch(d1, d2, k=2, mask=admit.astype(np.uint8))
            for ratio in (0.8, 0.9):
                want = set()
                for ms in knn:
                    if len(ms) == 1 or (len(ms) == 2 and ms[0].distance < ratio * ms[1].distance):
                        want.add((ms[0].queryIdx, ms[0].trainIdx))
                q, t = G.select(dist, admit, ratio, hamming=True)
                assert set(zip(q.tolist(), t.tolist())) == want


def test_guided_entry_points_reject_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    i32 = ctypes.POINTER(ctypes.c_int32)
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host
    good_off, good_pairs = [0, 10, 30, 30], [[0, 1], [2, 0], [1, 2]]

    def call(binary, off=good_off, pairs=good_pairs, D=8, cap=1 << 20, models=fake, guide=0, px_th=1.0, kp=fake,
             kp_dim=2, x1y1=None):
        off = np.ascontiguousarray(off, dtype=np.int32)
        pairs = np.ascontiguousarray(pairs, dtype=np.int32)
        fn = L.dgb200_match_binary_descriptors_guided_batch_dev if binary else L.dgb200_match_descriptors_guided_batch_dev
        r = ctypes.c_double(0.9) if binary else ctypes.c_float(0.9)
        return fn(fake, off.ctypes.data_as(i32), len(off) - 1, D, pairs.ctypes.data_as(i32), len(pairs), models, guide,
                  ctypes.c_double(px_th), r, 1, kp, kp_dim, fake, fake, x1y1, x1y1, 2, cap, fake, fake, None)

    for binary in (False, True):
        assert call(binary, models=None) == -1                     # no models
        assert call(binary, kp=None) == -1                         # no keypoints, though no coordinates are gathered
        assert call(binary, kp_dim=1) == -1
        for guide in (-1, 2, 7):
            assert call(binary, guide=guide) == -1
        for px_th in (-1.0, -1e-300, float("nan"), float("-inf")):
            assert call(binary, px_th=px_th) == -1
        # the batch matcher's own cases
        for D in ((0, 6, 68) if binary else (0, 6, 260)):
            assert call(binary, D=D) == -1
        assert call(binary, pairs=[[0, 3]]) == -1                  # train image index out of range
        assert call(binary, pairs=[[-1, 0]]) == -1                 # query image index out of range
        assert call(binary, off=[0, 10, 5, 30]) == -1              # decreasing offsets
        assert call(binary, off=[1, 10, 20, 30]) == -1             # offsets not starting at 0
        assert call(binary, pairs=np.zeros((0, 2))) == -1          # no pairs
        assert call(binary, cap=10 + 0 + 20 - 1) == -1             # capacity below the sum of query counts
        assert call(binary, x1y1=fake, kp_dim=1) == -1             # gathered columns beyond the keypoint rows


def test_guided_python_argument_errors():
    import torch
    from pydegensac_b200.matching import match_descriptors_guided
    d = [torch.zeros((10, 8)), torch.zeros((10, 8))]
    k = [torch.zeros((10, 2)), torch.zeros((10, 2))]
    F = np.zeros((1, 3, 3))
    for guide in ("E", "f", None):
        with pytest.raises(ValueError, match="guide"):
            match_descriptors_guided(d, [[0, 1]], k, F, 1.0, guide=guide)
    for px_th in (-1.0, float("nan")):
        with pytest.raises(ValueError, match="px_th"):
            match_descriptors_guided(d, [[0, 1]], k, F, px_th)
    for M in (np.zeros((2, 3, 3)), np.zeros((1, 8)), np.zeros((3, 3)), torch.zeros((2, 9), dtype=torch.float64)):
        with pytest.raises(ValueError, match="models"):
            match_descriptors_guided(d, [[0, 1]], k, M, 1.0)
    with pytest.raises(ValueError, match="keypoints"):
        match_descriptors_guided(d, [[0, 1]], None, F, 1.0)
    with pytest.raises(ValueError, match="norm"):
        match_descriptors_guided(d, [[0, 1]], k, F, 1.0, norm="l1")


@pytest.mark.parametrize("planar", [False, True])
def test_repeated_texture_scene_guided_oracle_recovers_true_matches(planar):
    kps, descs, where, model = scene(3, 800, 300, 64, 3, planar=planar)
    guide, px_th = ("H", 3.0) if planar else ("F", 1.0)
    for i, j in ((0, 1), (1, 2), (2, 0)):
        dist = G.distances(descs[i], descs[j])
        qu, tu = G.select(dist, np.ones(dist.shape, bool), 0.9)
        qg, tg = G.match_descriptors_guided(descs[i], descs[j], kps[i], kps[j], model(i, j), guide, px_th, 0.9, dist=dist)
        n_true = len(where[i])
        tu_n, tg_n = _true_count(qu, tu, where[i], where[j]), _true_count(qg, tg, where[i], where[j])
        assert tu_n < n_true / 2, "the plain ratio test should lose most true matches to look-alikes"
        assert tg_n >= 2 * tu_n and tg_n >= 0.9 * len(qg), (tu_n, tg_n, len(qg))


# ------------------------------------------------------------------------------------------------ GPU
def _models(guide, P, rng, planted):
    """per pair: planted, random, all-zero (no model: zero matches) and NaN (zero matches), cycling"""
    out = []
    for p in range(P):
        kind = p % 4
        if kind == 0:
            M = planted
        elif kind == 1:
            M = rng.normal(size=(3, 3)) if guide == "F" else np.eye(3) + rng.normal(0, 0.02, (3, 3)) * [[1, 1, 300],
                                                                                                         [1, 1, 300],
                                                                                                         [1e-4, 1e-4, 0]]
        elif kind == 2:
            M = np.zeros((3, 3))
        else:
            M = planted.copy(); M[1, 2] = np.nan
        out.append(M)
    return np.stack(out)


def _check(m, descs, kps, pairs, models, guide, px_th, ratio, mutual, hamming, dists):
    off = m.offsets.cpu().numpy()
    i1, i2 = m.idx1.cpu().numpy(), m.idx2.cpu().numpy()
    x1, x2 = m.pts1.cpu().numpy(), m.pts2.cpu().numpy()
    assert off[0] == 0 and np.all(np.diff(off) >= 0)
    for p, (qi, ti) in enumerate(pairs):
        a, b = int(off[p]), int(off[p + 1])
        key = (int(qi), int(ti))
        if key not in dists:
            dists[key] = G.distances(descs[qi], descs[ti], hamming)
        q, t = G.select(dists[key], G.gate(models[p], guide, kps[qi], kps[ti], px_th), ratio, mutual, hamming)
        assert np.array_equal(i1[a:b], q) and np.array_equal(i2[a:b], t), "pair %d (%d,%d)" % (p, qi, ti)
        w = x1.shape[1]
        assert np.array_equal(x1[a:b], kps[qi][q, :w]) and np.array_equal(x2[a:b], kps[ti][t, :w])
        if not np.all(np.isfinite(models[p])) or not models[p].any():
            assert a == b


_SIZES = [0, 1, 2, 33, 700, 2000, 3000]
_PAIRS = np.array([[4, 5], [5, 4], [6, 5], [5, 6], [3, 6], [6, 3], [4, 4], [0, 5], [5, 0], [1, 4], [4, 1], [2, 3],
                   [3, 2], [6, 6], [5, 5], [4, 6]], dtype=np.int32)


def _gpu_images(sizes, D, rng, kp_dim, binary):
    if binary:
        descs = [rng.integers(0, 256, (n, D), dtype=np.uint8) for n in sizes]
        for i in range(1, len(sizes)):
            k = min(sizes[i - 1], sizes[i]) // 2
            descs[i][:k] = _flip(descs[i - 1][:k], 0.1, rng)
    else:
        descs = [_q(rng.normal(size=(n, D))) for n in sizes]
        for i in range(1, len(sizes)):
            k = min(sizes[i - 1], sizes[i]) // 2
            descs[i][:k] = _q(descs[i - 1][:k] + 0.3 * rng.normal(size=(k, D)))
    kps = [np.c_[rng.uniform(0, 640, (n, 1)), rng.uniform(0, 480, (n, 1)), rng.normal(size=(n, kp_dim - 2))]
           for n in sizes]
    return descs, kps


@pytest.mark.gpu
@pytest.mark.parametrize("norm,D", [("l2", 8), ("l2", 64), ("l2", 128), ("l2", 256), ("hamming", 1), ("hamming", 32),
                                    ("hamming", 61), ("hamming", 64)])
def test_guided_batch_equals_oracle(norm, D):
    import torch
    from pydegensac_b200.matching import match_descriptors_guided, _match_bank, _banks
    from pydegensac_b200 import _cabi
    dev = torch.device("cuda:0")
    hamming = norm == "hamming"
    rng = np.random.default_rng(200 + D + 7 * hamming)
    kp_dim = 6 if D in (64, 61) else 2
    descs, kps = _gpu_images(_SIZES, D, rng, kp_dim, hamming)
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    _, _, _, planted_F = scene(2, 10, 0, 8, 1)
    planted = {"F": planted_F(0, 1), "H": np.array([[1.01, 0.02, 4.0], [-0.01, 0.99, -3.0], [1e-5, -2e-5, 1.0]])}
    dists = {}
    for guide in ("F", "H"):
        models = _models(guide, len(_PAIRS), rng, planted[guide])
        for px_th in (0.0, 0.5, 4.0):
            for mutual in ((False, True) if px_th == 4.0 else (px_th == 0.5,)):
                Mt = torch.from_numpy(models).to(dev) if px_th else models     # CUDA tensor in place, or uploaded
                m = match_descriptors_guided(dt, _PAIRS, kt, Mt, px_th, guide, 0.9, mutual, norm)
                assert m.n_max == max(_SIZES[q] for q, _ in _PAIRS)
                _check(m, descs, kps, _PAIRS, models, guide, px_th, 0.9, mutual, hamming, dists)
        # a bank 4 bytes past a 16-byte boundary: cooperative loads instead of bulk copies
        bank, counts, kbank = _banks(dt, kt, hamming)
        storage = torch.empty(bank.numel() + 1, dtype=bank.dtype, device=dev)
        ub = storage[1:].view(bank.shape)
        ub.copy_(bank)
        assert ub.data_ptr() % 16 != 0
        m = _match_bank(ub, counts, _PAIRS, kbank, 0.9, True, hamming, guide=_cabi.GUIDE_F if guide == "F" else
                        _cabi.GUIDE_H, models=torch.from_numpy(models).to(dev).view(-1, 9), px_th=4.0)
        _check(m, descs, kps, _PAIRS, models, guide, 4.0, 0.9, True, hamming, dists)


@pytest.mark.gpu
@pytest.mark.parametrize("guide", ["F", "H"])
def test_guided_threshold_boundary(guide):
    """px_th = sqrt(e) for residuals e of chosen candidates: th lands within an ulp of e, on either side"""
    import torch
    from pydegensac_b200.matching import match_descriptors_guided
    dev = torch.device("cuda:0")
    kps, descs, where, model = scene(2, 600, 200, 32, 9, planar=guide == "H")
    M = model(0, 1)
    e_fn = G.f_sampson if guide == "F" else G.h_transfer_sq
    q_pts, t_pts = kps[0][where[0]], kps[1][where[1]]
    e = e_fn(M, q_pts[:, 0], q_pts[:, 1], t_pts[:, 0], t_pts[:, 1])
    rng = np.random.default_rng(3)
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dist = G.distances(descs[0], descs[1])
    for k in rng.choice(len(e), 12, replace=False):
        px_th = float(np.sqrt(e[k]))
        th = px_th * px_th
        m = match_descriptors_guided(dt, [[0, 1]], kt, M[None], px_th, guide, 0.9, False)
        q, t = G.select(dist, G.gate(M, guide, kps[0], kps[1], px_th), 0.9)
        assert np.array_equal(m.idx1.cpu().numpy()[:len(q)], q) and int(m.offsets[1]) == len(q)
        assert np.array_equal(m.idx2.cpu().numpy()[:len(q)], t)
        # the point itself sits on the boundary: admitted exactly when th >= e
        assert bool(G.gate(M, guide, q_pts[k:k + 1], t_pts[k:k + 1], px_th)[0, 0]) == (th >= e[k])


@pytest.mark.gpu
@pytest.mark.parametrize("norm", ["l2", "hamming"])
def test_open_gate_equals_unguided_batch(norm):
    import torch
    from pydegensac_b200.matching import match_descriptors_batch, match_descriptors_guided
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(31)
    descs, kps = _gpu_images(_SIZES, 32 if norm == "hamming" else 64, rng, 2, norm == "hamming")
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    P = len(_PAIRS)
    Fr = rng.normal(size=(P, 3, 3))
    for mutual in (False, True):
        u = match_descriptors_batch(dt, _PAIRS, kt, 0.9, mutual, norm)
        for models, guide, px_th in ((np.broadcast_to(np.eye(3), (P, 3, 3)), "H", 1e6), (Fr, "F", 1e12)):
            g = match_descriptors_guided(dt, _PAIRS, kt, models, px_th, guide, 0.9, mutual, norm)
            assert torch.equal(u.offsets, g.offsets)
            n = int(u.offsets[-1])
            for a, b in ((u.idx1, g.idx1), (u.idx2, g.idx2), (u.pts1, g.pts1), (u.pts2, g.pts2)):
                assert torch.equal(a[:n], b[:n])


@pytest.mark.gpu
@pytest.mark.parametrize("planar", [False, True])
def test_pipeline_unguided_then_ragged_model_then_guided(planar):
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import match_descriptors_batch, match_descriptors_guided
    dev = torch.device("cuda:0")
    kps, descs, where, _ = scene(4, 800, 300, 64, 21, planar=planar)
    pairs = np.array([(i, j) for i in range(4) for j in range(4) if i != j], dtype=np.int32)
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    seeds = np.arange(len(pairs), dtype=np.uint64) + 5
    m = match_descriptors_batch(dt, pairs, kt, ratio=0.9)
    if planar:
        M, _ = pdg.findHomographyBatch(m.pts1, m.pts2, 2.0, 0.999, 10000, seeds=seeds, offsets=m.offsets, n_max=m.n_max)
        guide, px_th = "H", 3.0
    else:
        M, _ = pdg.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                              n_max=m.n_max)
        guide, px_th = "F", 1.0
    g = match_descriptors_guided(dt, pairs, kt, M, px_th, guide, 0.9)
    Mh = M.cpu().numpy()
    off, i1, i2 = m.offsets.cpu().numpy(), m.idx1.cpu().numpy(), m.idx2.cpu().numpy()
    goff, g1, g2 = g.offsets.cpu().numpy(), g.idx1.cpu().numpy(), g.idx2.cpu().numpy()
    for p, (qi, ti) in enumerate(pairs):
        q, t = G.match_descriptors_guided(descs[qi], descs[ti], kps[qi], kps[ti], Mh[p], guide, px_th, 0.9)
        assert np.array_equal(g1[goff[p]:goff[p + 1]], q) and np.array_equal(g2[goff[p]:goff[p + 1]], t)
        tu = _true_count(i1[off[p]:off[p + 1]], i2[off[p]:off[p + 1]], where[qi], where[ti])
        tg = _true_count(q, t, where[qi], where[ti])
        assert tu < len(where[qi]) / 2
        assert tg >= 2 * tu and tg >= 0.9 * len(q), "pair %d: unguided %d true, guided %d true of %d" % (p, tu, tg, len(q))
