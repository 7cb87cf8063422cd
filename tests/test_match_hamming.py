"""Binary descriptors matched by Hamming distance (match_descriptors / match_descriptors_batch with norm="hamming"):
a numpy oracle pinned to cv2.BFMatcher(cv2.NORM_HAMMING), argument checks, and on the GPU exact agreement of the
single and batched matchers with that oracle, and the batched matcher feeding the device-ragged F."""
import ctypes
import os

import numpy as np
import pytest

from pydegensac_b200.scenes import _K, _rot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")


def match_binary_np(d1, d2, ratio=0.9, mutual=False):
    """The matcher's contract in numpy: Hamming distances of uint8 rows, nearest train by stable argsort (ties to the
    lowest train index), d2 the second-smallest distance of the multiset, accepted when float64(d1) < ratio * float64(d2),
    mutual: the query is the train's nearest query (argmin: ties to the lowest query index).
    Returns the accepted queries, their trains and the distance matrix."""
    d1 = np.asarray(d1, np.uint8); d2 = np.asarray(d2, np.uint8)
    dist = np.empty((len(d1), len(d2)), np.int64)
    for i in range(0, len(d1), 64):
        dist[i:i + 64] = np.bitwise_count(d1[i:i + 64, None, :] ^ d2[None, :, :]).sum(2, dtype=np.int64)
    q, t = _select(dist, ratio, mutual)
    return q, t, dist


def _select(dist, ratio, mutual):
    """ratio test (+ mutual check) of match_binary_np on its distance matrix"""
    order = np.argsort(dist, 1, kind="stable")[:, :2]
    rows = np.arange(len(dist))
    nn, b1, b2 = order[:, 0], dist[rows, order[:, 0]], dist[rows, order[:, 1]]
    ok = b1.astype(np.float64) < float(ratio) * b2.astype(np.float64)
    if mutual:
        ok &= np.argmin(dist, 0)[nn] == rows
    q = np.nonzero(ok)[0]
    return q, nn[q]


def _flip(codes, p, rng):
    """codes with every bit flipped independently with probability p"""
    bits = np.unpackbits(codes, axis=1)
    return np.packbits(bits ^ (rng.random(bits.shape) < p), axis=1)


def _planted(sizes, B, rng, p=0.1):
    """random binary descriptors; the first half of each image repeats its predecessor's codes with bits flipped"""
    descs = [rng.integers(0, 256, (n, B), dtype=np.uint8) for n in sizes]
    for i in range(1, len(sizes)):
        k = min(sizes[i - 1], sizes[i]) // 2
        descs[i][:k] = _flip(descs[i - 1][:k], p, rng)
    return descs


def _tie_heavy(sizes, B, rng):
    """rows drawn from five codes (one all-zero), a third of them with one bit flipped: many exact duplicates and many
    tied distances"""
    codes = rng.integers(0, 256, (5, B), dtype=np.uint8)
    codes[0] = 0
    out = []
    for n in sizes:
        d = codes[rng.integers(0, 5, n)].copy()
        for r in np.nonzero(rng.random(n) < 1 / 3)[0]:
            b = rng.integers(0, 8 * B)
            d[r, b // 8] ^= np.uint8(1 << (b % 8))
        out.append(d)
    return out


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("B", [32, 61, 64])
def test_binary_oracle_agrees_with_cv2(B):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(B)
    bf = cv2.BFMatcher(cv2.NORM_HAMMING)
    planted, ties = _planted([300, 400], B, rng), _tie_heavy([300, 400], B, rng)
    s = np.sort(match_binary_np(*ties)[2], 1)
    assert np.sum(s[:, 0] == s[:, 1]) > 50          # ties at the minimum, which no ratio <= 1 accepts
    for d1, d2 in (planted, ties):
        knn = bf.knnMatch(d1, d2, k=2)
        for ratio in (0.8, 0.9):
            # the reference example's ratio test, on cv2's distances
            want = {(m.queryIdx, m.trainIdx) for m, n in knn if m.distance < ratio * n.distance}
            q, t, dist = match_binary_np(d1, d2, ratio)
            assert set(zip(q.tolist(), t.tolist())) == want
            s = np.sort(dist, 1)
            assert [(m.distance, n.distance) for m, n in knn] == list(zip(s[:, 0].tolist(), s[:, 1].tolist()))


def test_binary_entry_points_reject_malformed_input_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    i32 = ctypes.POINTER(ctypes.c_int32)
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host

    def single(n1, n2, W, count=fake):
        return L.dgb200_match_binary_descriptors_dev(fake, n1, fake, n2, W, ctypes.c_double(0.9), 1, None, None, 0, fake,
                                                     fake, None, None, 0, max(n1, 1), count, fake, None)

    def batch(off, pairs, W, cap=1 << 20):
        off = np.ascontiguousarray(off, dtype=np.int32)
        pairs = np.ascontiguousarray(pairs, dtype=np.int32)
        return L.dgb200_match_binary_descriptors_batch_dev(fake, off.ctypes.data_as(i32), len(off) - 1, W,
                                                           pairs.ctypes.data_as(i32), len(pairs), ctypes.c_double(0.9), 1,
                                                           None, 0, fake, fake, None, None, 0, cap, fake, fake, None)

    for W in (0, 2, 6, 68):                                   # n_words not a multiple of 4 in [4, 64]
        assert single(100, 100, W) == -1
    assert single(0, 100, 8) == -1                            # no query
    assert single(100, 1, 8) == -1                            # fewer than 2 train descriptors
    assert single(100, 100, 8, count=None) == -1              # null count
    good_off, good_pairs = [0, 10, 30, 30], [[0, 1], [2, 0], [1, 2]]
    for W in (0, 2, 6, 68):
        assert batch(good_off, good_pairs, W) == -1
    assert batch(good_off, [[0, 3]], 8) == -1                 # train image index out of range
    assert batch(good_off, [[-1, 0]], 8) == -1                # query image index out of range
    assert batch([0, 10, 5, 30], good_pairs, 8) == -1         # decreasing offsets
    assert batch([1, 10, 20, 30], good_pairs, 8) == -1        # offsets not starting at 0
    assert batch(good_off, np.zeros((0, 2)), 8) == -1         # no pairs
    assert batch(good_off, good_pairs, 8, cap=10 + 0 + 20 - 1) == -1   # capacity below the sum of query counts


def test_hamming_argument_errors():
    import torch
    from pydegensac_b200.matching import match_descriptors, match_descriptors_batch
    u8 = torch.zeros((10, 32), dtype=torch.uint8)
    with pytest.raises(ValueError, match="uint8"):
        match_descriptors(u8.float(), u8.float(), norm="hamming")
    with pytest.raises(ValueError, match="uint8"):
        match_descriptors_batch([u8, u8.to(torch.int16)], [[0, 1]], norm="hamming")
    for B in (0, 257):
        d = torch.zeros((10, B), dtype=torch.uint8)
        with pytest.raises(ValueError, match="1 to 256 bytes"):
            match_descriptors(d, d, norm="hamming")
        with pytest.raises(ValueError, match="1 to 256 bytes"):
            match_descriptors_batch([d, d], [[0, 1]], norm="hamming")
    with pytest.raises(ValueError, match="same length"):
        match_descriptors_batch([u8, torch.zeros((10, 61), dtype=torch.uint8)], [[0, 1]], norm="hamming")
    with pytest.raises(ValueError, match="same length"):
        match_descriptors(u8, torch.zeros((10, 61), dtype=torch.uint8), norm="hamming")
    for norm in ("L2", "hamming2", None):
        with pytest.raises(ValueError, match="norm"):
            match_descriptors(u8, u8, norm=norm)
        with pytest.raises(ValueError, match="norm"):
            match_descriptors_batch([u8, u8], [[0, 1]], norm=norm)


# ------------------------------------------------------------------------------------------------ GPU
def _check_against_oracle(m, descs, kps, pairs, mutual, dists):
    """every pair's segment of the batch, and a single call per pair, equal the oracle exactly"""
    import torch
    from pydegensac_b200.matching import match_descriptors
    off = m.offsets.cpu().numpy()
    i1b, i2b, x1b, x2b = (t.cpu().numpy() for t in (m.idx1, m.idx2, m.pts1, m.pts2))
    assert off[0] == 0 and np.all(np.diff(off) >= 0)
    dev = m.idx1.device
    for p, (qi, ti) in enumerate(pairs):
        a, b = int(off[p]), int(off[p + 1])
        n1, n2 = len(descs[qi]), len(descs[ti])
        if n1 < 1 or n2 < 2:
            assert a == b, "degenerate pair %d has matches" % p
            continue
        if (qi, ti) not in dists:
            dists[qi, ti] = match_binary_np(descs[qi], descs[ti])[2]
        q, t = _select(dists[qi, ti], 0.9, mutual)
        assert np.array_equal(i1b[a:b], q) and np.array_equal(i2b[a:b], t), "pair %d (%d,%d)" % (p, qi, ti)
        assert np.array_equal(x1b[a:b], kps[qi][q]) and np.array_equal(x2b[a:b], kps[ti][t])
        s1, s2, y1, y2 = match_descriptors(torch.from_numpy(descs[qi]).to(dev), torch.from_numpy(descs[ti]).to(dev),
                                           torch.from_numpy(kps[qi]).to(dev), torch.from_numpy(kps[ti]).to(dev), 0.9,
                                           mutual, norm="hamming")
        assert torch.equal(s1, m.idx1[a:b]) and torch.equal(s2, m.idx2[a:b]), "single call, pair %d" % p
        assert torch.equal(y1, m.pts1[a:b]) and torch.equal(y2, m.pts2[a:b])


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 8, 32, 61, 64, 256])
def test_hamming_single_and_batch_equal_oracle(B):
    import torch
    from pydegensac_b200.matching import match_descriptors_batch, _match_bank, _binary_words
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(100 + B)
    # query counts off multiples of 32, train counts off multiples of 64; a featureless and a one-descriptor image
    sizes = [0, 1, 45, 333, 700, 1029]
    pairs = np.array([[2, 3], [3, 2], [4, 5], [5, 4], [3, 5], [5, 3], [0, 3], [3, 0], [1, 4], [4, 1], [3, 3], [2, 1],
                      [1, 2], [0, 0]], dtype=np.int32)
    for descs in (_planted(sizes, B, rng), _tie_heavy(sizes, B, rng)):
        kps = [rng.uniform(0, 640, (n, 6 if B == 61 else 2)) for n in sizes]
        dt = [torch.from_numpy(d).to(dev) for d in descs]
        kt = [torch.from_numpy(k).to(dev) for k in kps]
        dists = {}
        for mutual in (False, True):
            m = match_descriptors_batch(dt, pairs, kt, ratio=0.9, mutual=mutual, norm="hamming")
            assert m.n_max == max(sizes[q] for q, _ in pairs)
            _check_against_oracle(m, descs, kps, pairs, mutual, dists)
        # a bank whose base is 4 bytes past a 16-byte boundary: cooperative loads instead of bulk copies
        words = _binary_words(dt)
        storage = torch.empty(words.numel() + 1, dtype=torch.int32, device=dev)
        bank = storage[1:].view(words.shape)
        bank.copy_(words)
        assert bank.data_ptr() % 16 != 0
        m = _match_bank(bank, sizes, pairs, torch.cat(kt, 0), 0.9, True, hamming=True)
        _check_against_oracle(m, descs, kps, pairs, True, dists)


def _binary_multiview(n_img, n_pts, n_clutter, B, seed):
    """n_img views of one set of 3-D points: keypoints, binary descriptors (a shared code per point, each bit flipped
    with probability 0.1 per view; clutter random), and the row of every point in every view"""
    rng = np.random.default_rng(seed)
    X = np.c_[rng.uniform(-2, 2, n_pts), rng.uniform(-2, 2, n_pts), rng.uniform(5, 10, n_pts)]
    code = rng.integers(0, 256, (n_pts, B), dtype=np.uint8)
    kps, descs, where = [], [], []
    for i in range(n_img):
        R = _rot("y", 0.08 * i) @ _rot("x", 0.02 * i)
        t = np.array([0.6 * i, 0.05 * i, 0.1 * i])
        x = (_K @ (R @ X.T + t[:, None])).T
        x = x[:, :2] / x[:, 2:3] + 0.1 * rng.normal(size=(n_pts, 2))
        kp = np.r_[x, rng.uniform(0, 640, (n_clutter, 2))]
        d = np.r_[_flip(code, 0.1, rng), rng.integers(0, 256, (n_clutter, B), dtype=np.uint8)]
        perm = rng.permutation(n_pts + n_clutter)
        kps.append(kp[perm]); descs.append(d[perm])
        inv = np.empty_like(perm); inv[perm] = np.arange(len(perm))
        where.append(inv[:n_pts])
    return kps, descs, where


@pytest.mark.gpu
def test_pipeline_hamming_batch_then_ragged_F():
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import match_descriptors, match_descriptors_batch
    dev = torch.device("cuda:0")
    kps, descs, where = _binary_multiview(4, 800, 400, 32, 7)
    pairs = np.array([(i, j) for i in range(4) for j in range(4) if i != j], dtype=np.int32)
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    seeds = np.arange(len(pairs), dtype=np.uint64) + 100
    m = match_descriptors_batch(dt, pairs, kt, ratio=0.9, mutual=True, norm="hamming")
    F, mask = pdg.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                             n_max=m.n_max)
    off = m.offsets.cpu().numpy()
    F, mask, i1, i2 = F.cpu().numpy(), mask.cpu().numpy(), m.idx1.cpu().numpy(), m.idx2.cpu().numpy()
    for p, (qi, ti) in enumerate(pairs):
        a, b = off[p], off[p + 1]
        planted = set(zip(where[qi].tolist(), where[ti].tolist()))
        found = {(q, t) for q, t, ok in zip(i1[a:b].tolist(), i2[a:b].tolist(), mask[a:b]) if ok}
        assert len(planted & found) >= 0.7 * len(planted), "pair %d: recall %d / %d" % (p, len(planted & found), len(planted))
        assert F[p].any()
        # one pair at a time: match, then verify
        s1, s2, x1, x2 = match_descriptors(dt[qi], dt[ti], kt[qi], kt[ti], 0.9, True, norm="hamming")
        assert np.array_equal(s1.cpu().numpy(), i1[a:b]) and np.array_equal(s2.cpu().numpy(), i2[a:b])
        Fs, ms = pdg.findFundamentalMatrixBatch(x1[None], x2[None], 0.5, 0.999, 10000, seeds=seeds[p:p + 1])
        assert np.array_equal(Fs[0].cpu().numpy(), F[p]) and np.array_equal(ms[0].cpu().numpy(), mask[a:b])
