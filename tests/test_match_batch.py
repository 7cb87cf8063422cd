"""Batched descriptor matcher (one launch for many image pairs, ragged output) and the device-ragged RANSAC entry points
that consume its output without a host read."""
import ctypes
import os

import numpy as np
import pytest

from pydegensac_b200.scenes import scene_F, scene_H, scene_F_laf, _K, _rot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")


# ------------------------------------------------------------------------------------------------ CPU
def test_batch_layout_against_direct_computation():
    from pydegensac_b200.matching import batch_layout
    rng = np.random.default_rng(0)
    counts = [0, 1, 2, 31, 32, 33, 700, 4000]
    pairs = rng.integers(0, len(counts), size=(40, 2))
    pairs[:3] = [[0, 5], [5, 1], [1, 0]]
    lay = batch_layout(counts, pairs)
    tile = row = col = 0
    n_max = 0
    for p, (qi, ti) in enumerate(pairs):
        assert lay.tile_prefix[p] == tile and lay.row_prefix[p] == row and lay.col_prefix[p] == col
        n1, n2 = counts[qi], counts[ti]
        if n1 >= 1 and n2 >= 2:
            tile += -(-n1 // 32)
        row += n1
        col += n2
        n_max = max(n_max, n1)
    assert lay.tile_prefix[-1] == tile and lay.row_prefix[-1] == row and lay.col_prefix[-1] == col
    assert lay.capacity == row and lay.n_max == n_max
    with pytest.raises(ValueError):
        batch_layout(counts, [[0, len(counts)]])
    with pytest.raises(ValueError):
        batch_layout(counts, [[-1, 0]])


def test_batch_matcher_rejects_malformed_metadata_before_any_launch():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    i32 = ctypes.POINTER(ctypes.c_int32)
    fake = ctypes.c_void_p(256)     # never dereferenced: every case is refused on the host

    def call(off, pairs, D, cap=1 << 20):
        off = np.ascontiguousarray(off, dtype=np.int32)
        pairs = np.ascontiguousarray(pairs, dtype=np.int32)
        return L.dgb200_match_descriptors_batch_dev(fake, off.ctypes.data_as(i32), len(off) - 1, D,
                                                    pairs.ctypes.data_as(i32), len(pairs), ctypes.c_float(0.9), 0,
                                                    None, 0, fake, fake, None, None, 0, cap, fake, fake, None)

    good_off, good_pairs = [0, 10, 30, 30], [[0, 1], [2, 0], [1, 2]]
    assert L.dgb200_match_batch_workspace_bytes(np.array(good_off, np.int32).ctypes.data_as(i32), 3,
                                                np.array(good_pairs, np.int32).ctypes.data_as(i32), 3) > 0
    assert call(good_off, [[0, 3]], 64) == -1                 # train image index out of range
    assert call(good_off, [[-1, 0]], 64) == -1                # query image index out of range
    assert call([0, 10, 5, 30], good_pairs, 64) == -1         # decreasing offsets
    for D in (0, 6, 260):                                     # D not a multiple of 4 in [4, 256]
        assert call(good_off, good_pairs, D) == -1
    assert call(good_off, good_pairs, 64, cap=10 + 0 + 20 - 1) == -1   # capacity below the sum of query counts
    assert L.dgb200_match_batch_workspace_bytes(np.array([0, 10, 5], np.int32).ctypes.data_as(i32), 2,
                                                np.array([[0, 1]], np.int32).ctypes.data_as(i32), 1) == 0


# ------------------------------------------------------------------------------------------------ GPU
def _images(sizes, D, rng, kp_dim=2):
    descs = [rng.normal(size=(n, D)).astype(np.float32) for n in sizes]
    kps = [rng.uniform(0, 640, (n, kp_dim)) for n in sizes]
    # planted matches between neighbouring images: shared codes plus noise
    for i in range(1, len(sizes)):
        k = min(sizes[i - 1], sizes[i]) // 2
        descs[i][:k] = descs[i - 1][:k] + 0.15 * rng.normal(size=(k, D)).astype(np.float32)
    return descs, kps


def _segments_equal_single_calls(m, descs_t, kps_t, pairs, mutual):
    import torch
    from pydegensac_b200.matching import match_descriptors
    off = m.offsets.cpu().numpy()
    P = len(pairs)
    assert off[0] == 0 and np.all(np.diff(off) >= 0) and off[P] <= m.idx1.shape[0]
    for p, (qi, ti) in enumerate(pairs):
        a, b = int(off[p]), int(off[p + 1])
        n1, n2 = descs_t[qi].shape[0], descs_t[ti].shape[0]
        if n1 < 1 or n2 < 2:
            assert a == b, "degenerate pair %d has matches" % p
            continue
        i1, i2, x1, x2 = match_descriptors(descs_t[qi], descs_t[ti], kps_t[qi], kps_t[ti], 0.9, mutual)
        assert torch.equal(m.idx1[a:b], i1) and torch.equal(m.idx2[a:b], i2), "pair %d (%d,%d)" % (p, qi, ti)
        assert torch.equal(m.pts1[a:b], x1) and torch.equal(m.pts2[a:b], x2)


@pytest.mark.gpu
def test_batch_matcher_equals_single_calls_bit_for_bit():
    import torch
    from pydegensac_b200.matching import match_descriptors_batch, _match_bank
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(1)
    sizes = [0, 1, 33, 700, 1500, 2000, 3000]
    pairs = np.array([[3, 4], [4, 3], [5, 6], [6, 5], [2, 6], [6, 2], [0, 3], [3, 0], [1, 4], [4, 1], [3, 3], [4, 6],
                      [5, 4], [2, 1], [1, 2], [0, 0]], dtype=np.int32)
    for D in (8, 64, 128, 256):
        descs, kps = _images(sizes, D, rng, kp_dim=6 if D == 64 else 2)
        descs_t = [torch.from_numpy(d).to(dev) for d in descs]
        kps_t = [torch.from_numpy(k).to(dev) for k in kps]
        for mutual in (False, True):
            m = match_descriptors_batch(descs_t, pairs, kps_t, ratio=0.9, mutual=mutual)
            assert m.n_max == max(sizes[q] for q, _ in pairs)
            assert m.idx1.shape[0] == sum(sizes[q] for q, _ in pairs)
            _segments_equal_single_calls(m, descs_t, kps_t, pairs, mutual)
    # a bank whose base is 4 bytes past a 16-byte boundary: cooperative loads instead of bulk copies, same results
    storage = torch.empty(sum(sizes) * D + 1, dtype=torch.float32, device=dev)
    bank = storage[1:].view(sum(sizes), D)
    bank.copy_(torch.cat(descs_t, 0))
    assert bank.data_ptr() % 16 != 0
    m = _match_bank(bank, sizes, pairs, torch.cat(kps_t, 0), 0.9, True)
    _segments_equal_single_calls(m, descs_t, kps_t, pairs, True)


@pytest.mark.gpu
def test_batch_matcher_against_bruteforce_oracle():
    import torch
    from pydegensac_b200.matching import match_descriptors_batch
    from oracle.frontend_np import match_descriptors as match_np
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(2)
    sizes = [900, 1200, 700]
    descs, kps = _images(sizes, 128, rng)
    pairs = [[0, 1], [1, 2], [2, 0]]
    for mutual in (False, True):
        m = match_descriptors_batch([torch.from_numpy(d).to(dev) for d in descs], pairs,
                                    [torch.from_numpy(k).to(dev) for k in kps], 0.9, mutual)
        off = m.offsets.cpu().numpy()
        for p, (qi, ti) in enumerate(pairs):
            q_ref, t_ref, dist = match_np(descs[qi], descs[ti], 0.9, mutual)
            i1 = m.idx1[off[p]:off[p + 1]].cpu().numpy()
            i2 = m.idx2[off[p]:off[p + 1]].cpu().numpy()
            s = np.sort(dist, 1)
            margin = np.abs(s[:, 0] - np.float32(0.81) * s[:, 1]) < 1e-4 * s[:, 1]
            a = set(zip(q_ref.tolist(), t_ref.tolist())); b = set(zip(i1.tolist(), i2.tolist()))
            for (q, t) in a ^ b:
                assert margin[q], "match (%d,%d) differs away from the ratio threshold" % (q, t)
            assert np.all(np.diff(i1) > 0)
            assert np.array_equal(m.pts1[off[p]:off[p + 1]].cpu().numpy(), kps[qi][i1])
            assert np.array_equal(m.pts2[off[p]:off[p + 1]].cpu().numpy(), kps[ti][i2])


def _ragged_case(kind, lengths, seed, laf=False):
    l1, l2 = [], []
    for i, n in enumerate(lengths):
        if laf:
            a, b, _ = scene_F_laf(max(n, 8), 0.5, seed + i)
        elif kind == 0:
            a, b, _ = scene_F(max(n, 8), 0.5, seed + i)
        else:
            a, b, _ = scene_H(max(n, 8), max(n, 8) // 2, seed + i)
        l1.append(a[:n]); l2.append(b[:n])
    return l1, l2


def _check_ragged(kind, lengths, n_max, seed, metric, laf=False):
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200 import _cabi, tensor_api
    from pydegensac_b200.utils import error_type_dict_fundamental, error_type_dict_homography
    dev = torch.device("cuda:0")
    l1, l2 = _ragged_case(kind, lengths, seed, laf)
    dim = l1[0].shape[1]
    off = np.zeros(len(lengths) + 1, dtype=np.int32)
    off[1:] = np.cumsum(lengths)
    p1 = torch.from_numpy(np.concatenate(l1).reshape(-1, dim)).to(dev)
    p2 = torch.from_numpy(np.concatenate(l2).reshape(-1, dim)).to(dev)
    d_off = torch.from_numpy(off).to(dev)
    seeds = np.arange(len(lengths), dtype=np.uint64) * 7 + 3
    min_n = 8 if kind == 0 else 4
    run = [i for i, n in enumerate(lengths) if min_n <= n <= n_max]
    lafc = 3.0 if laf else -1.0
    if kind == 0:
        M, mask, st = pdg.findFundamentalMatrixBatch(p1, p2, 1.0, 0.999, 3000, metric, seeds=seeds, return_stats=True,
                                                     offsets=d_off, n_max=n_max, laf_consistensy_coef=lafc)
        Mh, mh, sh = pdg.findFundamentalMatrixBatch([l1[i] for i in run], [l2[i] for i in run], 1.0, 0.999, 3000, metric,
                                                    seeds=seeds[run], return_stats=True, laf_consistensy_coef=lafc)
    else:
        M, mask, st = pdg.findHomographyBatch(p1, p2, 3.0, 0.999, 3000, metric, seeds=seeds, return_stats=True,
                                              offsets=d_off, n_max=n_max, laf_consistensy_coef=lafc)
        Mh, mh, sh = pdg.findHomographyBatch([l1[i] for i in run], [l2[i] for i in run], 3.0, 0.999, 3000, metric,
                                             seeds=seeds[run], return_stats=True, laf_consistensy_coef=lafc)
        # the raw core output is bit-equal; the OpenCV-convention inversion runs in different libraries
        et = error_type_dict_homography[metric]
        Hraw, _, _ = tensor_api._launch_ragged(1, p1, p2, d_off, n_max, 3.0, 0.999, 3000, et, True, lafc, False,
                                               torch.from_numpy(seeds.view(np.int64)).to(dev), False)
        Hraw_h, _, _ = _cabi.homography_ragged([l1[i] for i in run], [l2[i] for i in run], 3.0, 0.999, 3000, et, True,
                                               max(lafc, 0), seeds[run])
        assert np.array_equal(Hraw.cpu().numpy()[run], Hraw_h)
    assert M.is_cuda and mask.dtype == torch.bool and mask.shape[0] == off[-1]
    M, mask, st = M.cpu().numpy(), mask.cpu().numpy(), st.cpu().numpy()
    for k, i in enumerate(run):
        seg = mask[off[i]:off[i + 1]]
        assert np.array_equal(seg, mh[k]) and np.array_equal(st[i], sh[k]), "pair %d" % i
        if kind == 0:
            assert np.array_equal(M[i], Mh[k])
        else:
            assert np.allclose(M[i], Mh[k], rtol=1e-12, atol=1e-12)
        if lengths[i] >= 50:
            assert seg.sum() > 0
    for i in set(range(len(lengths))) - set(run):
        assert not M[i].any() and not st[i].any() and not mask[off[i]:off[i + 1]].any(), "skipped pair %d" % i


@pytest.mark.gpu
def test_ragged_device_F_equals_host_ragged():
    lengths = [300, 0, 3, 7, 500, 8, 150, 0]
    for metric in ("sampson", "symm_epipolar"):
        _check_ragged(0, lengths, max(lengths), 11, metric)
    # a pair longer than n_max is skipped like a short one; its neighbours are unaffected
    _check_ragged(0, [300, 520, 200], 400, 21, "sampson")
    _check_ragged(0, [200, 5, 400, 120], 400, 31, "sampson", laf=True)     # [N,6] rows with the LAF check


@pytest.mark.gpu
def test_ragged_device_H_equals_host_ragged():
    lengths = [200, 0, 3, 4, 400, 7, 90]
    for metric in ("sampson", "symm_sq_max"):
        _check_ragged(1, lengths, max(lengths), 41, metric)
    _check_ragged(1, [300, 520, 200], 400, 51, "sampson")


@pytest.mark.gpu
def test_ragged_offsets_argument_errors():
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import match_descriptors_batch
    dev = torch.device("cuda:0")
    p = torch.zeros((20, 2), dtype=torch.float64, device=dev)
    off = torch.tensor([0, 20], dtype=torch.int32, device=dev)
    with pytest.raises(ValueError):
        pdg.findFundamentalMatrixBatch(p, p, offsets=off, n_max=20, final_lsq=True)
    with pytest.raises(ValueError):
        pdg.findFundamentalMatrixBatch(p, p, offsets=off)                     # n_max missing
    with pytest.raises(ValueError):
        pdg.findHomographyBatch(p.cpu().numpy(), p.cpu().numpy(), offsets=off, n_max=20)
    with pytest.raises(ValueError):
        match_descriptors_batch([torch.zeros((4, 8), device=dev)], torch.zeros((1, 2), dtype=torch.int32, device=dev))


def _multiview(n_img, n_pts, n_clutter, D, seed):
    """n_img views of one set of 3-D points: keypoints, descriptors (shared code + noise per point), the planted
    correspondence of every point, and the true F of every ordered pair of views."""
    rng = np.random.default_rng(seed)
    X = np.c_[rng.uniform(-2, 2, n_pts), rng.uniform(-2, 2, n_pts), rng.uniform(5, 10, n_pts)]
    code = rng.normal(size=(n_pts, D)).astype(np.float32)
    Rs, ts, kps, descs, where = [], [], [], [], []
    for i in range(n_img):
        R = _rot("y", 0.08 * i) @ _rot("x", 0.02 * i)
        t = np.array([0.6 * i, 0.05 * i, 0.1 * i])
        x = (_K @ (R @ X.T + t[:, None])).T
        x = x[:, :2] / x[:, 2:3] + 0.1 * rng.normal(size=(n_pts, 2))
        kp = np.r_[x, rng.uniform(0, 640, (n_clutter, 2))]
        d = np.r_[code + 0.15 * rng.normal(size=code.shape).astype(np.float32),
                  rng.normal(size=(n_clutter, D)).astype(np.float32)]
        perm = rng.permutation(n_pts + n_clutter)
        kps.append(kp[perm]); descs.append(d[perm])
        inv = np.empty_like(perm); inv[perm] = np.arange(len(perm))
        where.append(inv[:n_pts])          # row of point k in image i
        Rs.append(R); ts.append(t)
    Ki = np.linalg.inv(_K)

    def F(i, j):   # x_j^T F x_i = 0
        R = Rs[j] @ Rs[i].T
        t = ts[j] - R @ ts[i]
        tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
        return Ki.T @ tx @ R @ Ki
    return kps, descs, where, F


@pytest.mark.gpu
def test_pipeline_match_batch_then_ragged_F():
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import match_descriptors, match_descriptors_batch
    dev = torch.device("cuda:0")
    kps, descs, where, Ftrue = _multiview(4, 800, 400, 64, 5)
    pairs = np.array([(i, j) for i in range(4) for j in range(4) if i != j], dtype=np.int32)
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    seeds = np.arange(len(pairs), dtype=np.uint64) + 100
    m = match_descriptors_batch(dt, pairs, kt, ratio=0.9, mutual=True)
    F, mask = pdg.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                             n_max=m.n_max)
    off = m.offsets.cpu().numpy()
    F, mask, i1, i2 = F.cpu().numpy(), mask.cpu().numpy(), m.idx1.cpu().numpy(), m.idx2.cpu().numpy()
    for p, (qi, ti) in enumerate(pairs):
        a, b = off[p], off[p + 1]
        planted = set(zip(where[qi].tolist(), where[ti].tolist()))
        found = {(q, t) for q, t, ok in zip(i1[a:b].tolist(), i2[a:b].tolist(), mask[a:b]) if ok}
        assert len(planted & found) >= 0.7 * len(planted), "pair %d: recall %d / %d" % (p, len(planted & found), len(planted))
        # the planted correspondences satisfy the true F; the found model does on them too
        x1p, x2p = kps[qi][where[qi]], kps[ti][where[ti]]
        h1, h2 = np.c_[x1p, np.ones(len(x1p))], np.c_[x2p, np.ones(len(x2p))]
        Ft = Ftrue(qi, ti)
        l2 = h1 @ Ft.T
        assert np.median(np.abs(np.sum(h2 * l2, 1)) / np.hypot(l2[:, 0], l2[:, 1])) < 0.5
        assert F[p].any()
        # one pair at a time: match, then verify
        s1, s2, x1, x2 = match_descriptors(dt[qi], dt[ti], kt[qi], kt[ti], 0.9, True)
        Fs, ms = pdg.findFundamentalMatrixBatch(x1[None], x2[None], 0.5, 0.999, 10000, seeds=seeds[p:p + 1])
        assert np.array_equal(Fs[0].cpu().numpy(), F[p]) and np.array_equal(ms[0].cpu().numpy(), mask[a:b])
