"""matching.build_tracks_ragged: tracks from verified pairwise matches, the connected components of the keypoint graph in
the ragged track layout.  CPU: the numpy oracle (tests/tracks_np.py) against an independent pure-Python union-find;
the host build of csrc/tracks.h's lock-free union-find from several threads against the oracle; the argument checks
of the Python wrapper and of the C entry point.  GPU: every output byte for byte against the oracle, invariance under
reordering of the matches, a large graph, and a pipeline from descriptors to bundle adjustment without a host
synchronisation."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from tests import tracks_np as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pydegensac_b200", "libdegensac_b200.so")


# ------------------------------------------------------------------------------------------------ random graphs
def graph(seed, I, n_max=30, n_points=25, junk=0.04, long_track=False, chain=False, malformed=True, self_pairs=True):
    """A random match graph: per image a keypoint count (some images empty), planted points seen in random images at
    random keypoints (two points may share a keypoint: conflicts), a pair table with repeated pairs and self-pairs, and
    per pair the rows of the points both images see plus junk rows (random and out-of-range indices).  long_track: one
    point seen by every image at its own keypoint, linked image to image (a track longer than 32 when I > 32); chain:
    keypoint k of image i joined to keypoints k and k + 1 of image i + 1 (a giant conflicting component).
    Returns dict(counts, pairs, rows: per pair [r,2] (idx1, idx2), firm: the first pair of the long track and the
    chain, whose rows layout() never masks or breaks); layout() lays it out."""
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, n_max + 1, I)
    counts[rng.random(I) < 0.15] = 0
    if long_track or chain:
        counts = np.maximum(counts, 3)
    seen = []                                          # per point: {image: keypoint}
    perm = [rng.permutation(c) for c in counts]      # point m takes keypoint perm[i][m % counts[i]] of image i
    for m in range(n_points):
        imgs = [i for i in rng.permutation(I)[:rng.integers(1, min(I, 8) + 1)] if counts[i] > 0]
        seen.append({int(i): int(perm[i][m % counts[i]]) for i in imgs})
    P = max(1, int(rng.integers(I, 3 * I + 2)))
    pairs, rows = [], []
    for _ in range(P):
        q, t = (int(v) for v in rng.integers(0, I, 2))
        if not self_pairs and q == t and I > 1:
            t = (q + 1) % I
        r = [(s[q], s[t]) for s in seen if q in s and t in s and q != t and rng.random() < 0.8]
        for _ in range(rng.integers(0, 4)):             # junk: out-of-range rows, and a few random ones
            a, b = int(rng.integers(0, counts[q] + 1)), int(rng.integers(0, counts[t] + 1))
            if rng.random() < junk:
                r.append((a, b))
            else:
                r.append((a, -1 - b) if rng.random() < 0.5 else (counts[q] + a, b))
        if q == t and counts[q] > 1 and rng.random() < 0.25:
            r.append((0, 1))                          # a self-pair row joins two keypoints of one image: conflict
        pairs.append((q, t))
        rows.append(np.array(r, np.int64).reshape(-1, 2)[rng.permutation(len(r))])
    firm = len(pairs)
    if long_track:
        k = [int(rng.integers(0, counts[i])) for i in range(I)]
        used = {(i, k[i]) for i in range(I)}
        for s in seen:                                 # the long track's keypoints see nothing else
            for i in list(s):
                if (i, s[i]) in used:
                    del s[i]
        rows = [np.array([(a, b) for a, b in r if (q, a) not in used and (t, b) not in used], np.int64).reshape(-1, 2)
                for (q, t), r in zip(pairs, rows)]
        for i in range(I - 1):
            pairs.append((i, i + 1))
            rows.append(np.array([[k[i], k[i + 1]]], np.int64))
    if chain:
        for i in range(I - 1):
            n = int(min(counts[i], counts[i + 1]))
            r = [(j, j) for j in range(n)] + [(j + 1, j) for j in range(n - 1)]
            pairs.append((i, i + 1))
            rows.append(np.array(r, np.int64))
    return dict(counts=counts, pairs=np.array(pairs, np.int64), rows=rows, malformed=malformed, seed=seed, firm=firm)


def layout(g, order=None, flip=None, row_perm_seed=None, mask_p=0.85):
    """The ragged layout of graph g: idx1, idx2, offsets, mask (rows past offsets[P] are junk); pairs in `order`,
    the pairs in `flip` swapped with their idx1 / idx2, rows within a pair permuted by row_perm_seed.  The mask of a
    row is a function of the row's content, so reordering keeps the edge set; with g["malformed"] some offsets are
    broken (in the original order only)."""
    rng = np.random.default_rng(row_perm_seed)
    P = len(g["pairs"])
    order = np.arange(P) if order is None else np.asarray(order)
    flip = set() if flip is None else set(flip)
    pairs, i1, i2, counts = [], [], [], [0]
    for p in order:
        q, t = g["pairs"][p]
        r = g["rows"][p]
        if row_perm_seed is not None:
            r = r[rng.permutation(len(r))]
        if p in flip:
            q, t, r = t, q, r[:, ::-1]
        pairs.append((q, t))
        i1.append(r[:, 0]); i2.append(r[:, 1]); counts.append(len(r))
    i1 = np.concatenate(i1 + [np.array([7, -5, 10 ** 6])])   # junk rows past offsets[P]
    i2 = np.concatenate(i2 + [np.array([3, 2, 1])])
    offsets = np.cumsum(counts).astype(np.int64)
    # the mask: a hash of the (unordered) row and its pair, so every layout masks the same edges
    h = lambda a, b, q, t: ((min((q, a), (t, b)) + max((q, a), (t, b))).__hash__() * 2654435761) % 100
    mask = np.ones(len(i1), bool)
    pos = 0
    for p, (q, t), c in zip(order, pairs, counts[1:]):
        for r in range(pos, pos + c):
            mask[r] = p >= g["firm"] or h(int(i1[r]), int(i2[r]), int(q), int(t)) < 100 * mask_p
        pos += c
    if g["malformed"] and g["firm"] > 3 and list(order) == list(range(P)):
        bad = np.random.default_rng(g["seed"] + 7).choice(np.arange(1, g["firm"]), 3, replace=False)
        offsets[bad[0]] = -1                          # negative
        offsets[bad[1]] = len(i1) + 4                 # past rows
        offsets[bad[2]] = max(offsets[bad[2] - 1] - 1, 0) if bad[2] > 0 else 0   # may decrease
    return np.array(pairs, np.int64), i1.astype(np.int64), i2.astype(np.int64), offsets.astype(np.int32), mask


def py_tracks(counts, pairs, idx1, idx2, offsets, mask, min_length):
    """Pure-Python restatement, independent of the oracle: a union-find by dict, row by row, then the rules"""
    base, s = [], 0
    for c in counts:
        base.append(s)
        s += int(c)
    N = s
    up = {}

    def find(x):
        while up.get(x, x) != x:
            x = up[x]
        return x
    rows = len(idx1)
    for p, (q, t) in enumerate(pairs):
        b, e = int(offsets[p]), int(offsets[p + 1])
        if not (0 <= b <= e <= rows):
            continue
        for r in range(b, e):
            i, j = int(idx1[r]), int(idx2[r])
            if mask is not None and not mask[r]:
                continue
            if 0 <= i < counts[q] and 0 <= j < counts[t]:
                x, y = find(base[q] + i), find(base[t] + j)
                if x != y:
                    up[max(x, y)] = min(x, y)
    comps = {}
    for g in range(N):
        comps.setdefault(find(g), []).append(g)
    img = [i for i, c in enumerate(counts) for _ in range(int(c))]
    tracks, n_conf, n_conf_nodes = [], 0, 0
    for root in sorted(comps):
        nodes = sorted(comps[root])
        if len(nodes) < 2:
            continue
        if len({img[g] for g in nodes}) != len(nodes):
            n_conf += 1
            n_conf_nodes += len(nodes)
        elif len(nodes) >= min_length:
            tracks.append(nodes)
    T_cap = N // min_length
    off, cams, kp, track_of = [0], [], [], [-1] * N
    for j, nodes in enumerate(tracks):
        for g in nodes:
            cams.append(img[g]); kp.append(g - base[img[g]]); track_of[g] = j
        off.append(len(cams))
    n_obs = len(cams)
    return dict(offsets=off + [n_obs] * (T_cap + 1 - len(off)), cams=cams + [-1] * (N - n_obs),
                kp=kp + [-1] * (N - n_obs), track_of=track_of, stats=[len(tracks), n_obs, n_conf, n_conf_nodes])


CASES = [  # (seed, I, options)
    (0, 1, {}), (1, 2, {}), (2, 5, {}), (3, 12, {}), (4, 40, {"long_track": True}), (5, 30, {"chain": True}),
    (6, 60, {"long_track": True, "n_max": 5}), (7, 8, {"n_points": 40, "n_max": 12}), (8, 200, {"n_points": 2000}),
    (9, 3, {"n_max": 2}),
]


# ------------------------------------------------------------------------------------------------ oracle (CPU)
@pytest.mark.parametrize("min_length", [2, 3, 5])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_oracle_equals_pure_python_union_find(case, min_length):
    seed, I, kw = CASES[case]
    g = graph(seed, I, **kw)
    pairs, i1, i2, off, mask = layout(g)
    ref = o.build_tracks(g["counts"], pairs, i1, i2, off, mask, min_length=min_length)
    py = py_tracks(g["counts"], pairs, i1, i2, off, mask, min_length)
    for k in ("offsets", "cams", "kp", "track_of", "stats"):
        assert np.array_equal(ref[k], np.array(py[k], np.int32)), k


def test_oracle_graphs_cover_the_special_cases():
    """the generator makes what the device tests rely on: conflicts of both kinds, a track longer than 32, malformed
    pairs, masked, self-pair and out-of-range rows, empty images"""
    g = graph(4, 40, long_track=True)
    pairs, i1, i2, off, mask = layout(g)
    r = o.build_tracks(g["counts"], pairs, i1, i2, off, mask)
    assert (np.diff(r["offsets"][:r["stats"][0] + 1]) == 40).any()
    g = graph(5, 30, chain=True)
    pairs, i1, i2, off, mask = layout(g)
    r = o.build_tracks(g["counts"], pairs, i1, i2, off, mask)
    assert r["stats"][3] > 30 and r["stats"][2] >= 1       # the chain: more nodes than images
    rows = len(i1)
    assert any(not 0 <= off[p] <= off[p + 1] <= rows for p in range(len(pairs)))
    assert (~mask).any() and (pairs[:, 0] == pairs[:, 1]).any()
    img = pairs[np.clip(np.searchsorted(off[1:], np.arange(rows), side="right"), 0, len(pairs) - 1)]
    assert ((i1 < 0) | (i1 >= g["counts"][img[:, 0]]) | (i2 < 0) | (i2 >= g["counts"][img[:, 1]])).any()
    g8 = graph(8, 200, n_points=2000)
    r8 = o.build_tracks(g8["counts"], *layout(g8))
    assert r8["stats"][2] >= 2 and r8["stats"][3] <= 200 * r8["stats"][2]  # conflicts no larger than I
    assert (g8["counts"] == 0).any()
    assert ((i1 < 0) | (i1 >= g["counts"][pairs[np.searchsorted(off[1:], np.arange(rows), side="right").clip(
        0, len(pairs) - 1), 0]])).any()


# ------------------------------------------------------------------------------------------------ host build (CPU)
def _host(tmp_path):
    so = os.path.join(str(tmp_path), "libtracks_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++20", "-pthread", "-Wno-unknown-pragmas", "-o", so,
                           os.path.join(ROOT, "tests", "tracks_host.cpp")])
    return ctypes.CDLL(so)


def _ip(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))


def test_host_union_find_from_threads_equals_oracle(tmp_path):
    L = _host(tmp_path)
    rng = np.random.default_rng(11)
    for case in range(len(CASES)):
        seed, I, kw = CASES[case]
        g = graph(seed, I, **kw)
        pairs, i1, i2, off, mask = layout(g)
        a, b = o.edges(g["counts"], pairs, i1, i2, off, mask)
        N = int(g["counts"].sum())
        want = o.component_roots(N, a, b)
        for threads in (1, 2, 4, 8):
            for _ in range(3):
                perm = rng.permutation(len(a))
                ea, eb = a[perm], b[perm]
                sw = rng.random(len(a)) < 0.5         # either direction
                ea, eb = np.where(sw, eb, ea).astype(np.int32), np.where(sw, ea, eb).astype(np.int32)
                roots = np.empty(N, np.int32)
                L.tkh_roots(N, _ip(ea), _ip(eb), len(ea), threads, _ip(roots))
                assert np.array_equal(roots, want), (case, threads)
    # a dense random graph, many threads racing on few roots
    N = 3000
    a = rng.integers(0, N, 40000).astype(np.int32)
    b = rng.integers(0, N, 40000).astype(np.int32)
    want = o.component_roots(N, a.astype(np.int64), b.astype(np.int64))
    for _ in range(5):
        roots = np.empty(N, np.int32)
        L.tkh_roots(N, _ip(a), _ip(b), len(a), 16, _ip(roots))
        assert np.array_equal(roots, want)


def test_host_image_lookup(tmp_path):
    L = _host(tmp_path)
    for counts in ([0, 3, 0, 0, 2, 5, 0], [4], [0, 0, 1], [1, 0]):
        off = o.img_offsets(counts).astype(np.int32)
        N = int(off[-1])
        out = np.empty(max(N, 1), np.int32)
        L.tkh_images(_ip(off), len(counts), N, _ip(out))
        assert np.array_equal(out[:N], np.repeat(np.arange(len(counts)), counts))


# ------------------------------------------------------------------------------------------------ argument checks
def _raises(fn, kw, message):
    with pytest.raises(ValueError) as e:
        fn(**kw)
    assert str(e.value) == message


def test_python_argument_messages():
    torch = pytest.importorskip("torch")
    from pydegensac_b200.matching import build_tracks_ragged
    i32 = torch.int32
    base = dict(counts=[3, 4], pairs=[[0, 1]], idx1=torch.zeros(5, dtype=i32), idx2=torch.zeros(5, dtype=i32),
                offsets=torch.tensor([0, 5], dtype=i32))
    dev_msg = "idx1, idx2, offsets and mask must be CUDA tensors on one device"
    cases = [
        (dict(counts=[]), "counts must be a non-empty host sequence of integer keypoint counts"),
        (dict(counts=[[3, 4]]), "counts must be a non-empty host sequence of integer keypoint counts"),
        (dict(counts=[3.0, 4.0]), "counts must be a non-empty host sequence of integer keypoint counts"),
        (dict(counts=[3, -1]), "counts must not be negative"),
        (dict(counts=[2 ** 30, 2 ** 30]), "counts sum to 2147483648 keypoints, more than 2^31 - 1"),
        (dict(pairs=[0, 1]), "pairs must be a non-empty [P,2] array of (query image, train image)"),
        (dict(pairs=np.zeros((0, 2))), "pairs must be a non-empty [P,2] array of (query image, train image)"),
        (dict(pairs=[[0, 2]]), "pairs: image index out of range"),
        (dict(pairs=[[-1, 1]]), "pairs: image index out of range"),
        (dict(idx1=np.zeros(5, np.int32)), "idx1 must be a torch tensor"),
        (dict(idx2=None), "idx2 must be a torch tensor"),
        (dict(offsets=[0, 5]), "offsets must be a torch tensor"),
        (dict(mask=np.ones(5, bool)), "mask must be a torch tensor"),
        (dict(idx1=torch.zeros((5, 1), dtype=i32)), "idx1 must be [rows], not [5, 1]"),
        (dict(idx2=torch.zeros(4, dtype=i32)), "idx2 must be [rows] = [5], not [4]"),
        (dict(idx1=torch.zeros(5)), "idx1 must be int32 or int64, not torch.float32"),
        (dict(idx2=torch.zeros(5, dtype=torch.int16)), "idx2 must be int32 or int64, not torch.int16"),
        (dict(offsets=torch.tensor([0, 2, 5], dtype=i32)), "offsets must be [P+1] = [2], not [3]"),
        (dict(offsets=torch.tensor([0, 5])), "offsets must be int32, not torch.int64"),
        (dict(mask=torch.ones(4, dtype=torch.bool)), "mask must be [rows] = [5], not [4]"),
        (dict(mask=torch.ones(5, dtype=i32)), "mask must be bool or uint8, not torch.int32"),
        (dict(min_length=1), "min_length must be at least 2, not 1"),
        (dict(), dev_msg),
        (dict(idx1=torch.zeros(5, dtype=torch.int64), mask=torch.ones(5, dtype=torch.uint8)), dev_msg),
    ]
    for kw, msg in cases:
        _raises(build_tracks_ragged, dict(base, **kw), msg)
    if torch.cuda.is_available():
        c = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in base.items()}
        _raises(build_tracks_ragged, dict(c, counts=torch.tensor([3, 4]).cuda()),
                "counts must be a host sequence: reading a CUDA tensor would synchronise")
        _raises(build_tracks_ragged, dict(c, pairs=torch.tensor([[0, 1]]).cuda()),
                "pairs must be a host array: reading a CUDA tensor would synchronise")
        _raises(build_tracks_ragged, dict(c, kps=[torch.zeros((3, 2)).cuda()]),
                "kps must hold one keypoint tensor per image (2)")
        _raises(build_tracks_ragged, dict(c, kps=[torch.zeros((3, 2)).cuda(), torch.zeros((5, 2)).cuda()]),
                "keypoint tensors must be [n_i, k] with k >= 2 and n_i = counts[i]")
        _raises(build_tracks_ragged, dict(c, kps=[torch.zeros((3, 2)).cuda(), torch.zeros((4, 1)).cuda()]),
                "keypoint tensors must be [n_i, k] with k >= 2 and n_i = counts[i]")
        _raises(build_tracks_ragged, dict(c, kps=[torch.zeros((3, 2)).cuda(), torch.zeros((4, 2))]),
                "kps must be on the device of idx1")
        _raises(build_tracks_ragged, dict(c, kps=[torch.zeros((3, 2)).cuda(), torch.zeros((4, 2), dtype=i32).cuda()]),
                "kps must be a floating tensor, not torch.int32")


FAKE = ctypes.c_void_p(256)      # never dereferenced: every case is refused on the host


def test_c_entry_point_refusals():
    if not os.path.exists(LIB):
        pytest.skip("libdegensac_b200.so not built")
    from pydegensac_b200 import _cabi
    L = _cabi.lib()
    names = ["idx1", "idx2", "offsets", "mask", "kp", "off_out", "cams", "kp_out", "pts", "track_of", "stats"]

    def call(img_off=(0, 3, 7), n_images=2, pairs=(0, 1), n_pairs=1, rows=5, min_length=2, null=(), host_null=()):
        b = {k: (None if k in null else FAKE) for k in names}
        io = np.array(img_off, np.int32)
        pr = np.array(pairs, np.int32)
        return L.dgb200_build_tracks_ragged_dev(
            None if "img_off" in host_null else _ip(io), n_images, None if "pairs" in host_null else _ip(pr), n_pairs,
            b["idx1"], b["idx2"], b["offsets"], rows, b["mask"], b["kp"], min_length, b["off_out"], b["cams"],
            b["kp_out"], b["pts"], b["track_of"], b["stats"], None)

    sizes = "need n_images >= 1, n_pairs >= 1 and rows >= 0"
    offs = "img_offsets must start at 0 and must not decrease"
    kpb = "d_kp and d_pts_out must both be given (with keypoints) or both be null"
    cases = [
        (dict(host_null={"img_off"}), "null buffer"), (dict(host_null={"pairs"}), "null buffer"),
        (dict(null={"offsets"}), "null buffer"), (dict(null={"off_out"}), "null buffer"),
        (dict(null={"stats"}, n_images=0), "null buffer"),
        (dict(n_images=0), sizes), (dict(n_images=-1), sizes), (dict(n_pairs=0), sizes), (dict(rows=-1), sizes),
        (dict(null={"idx1"}), "null row buffer"), (dict(null={"idx2"}), "null row buffer"),
        (dict(min_length=1), "min_length must be at least 2"), (dict(min_length=-3), "min_length must be at least 2"),
        (dict(img_off=(1, 3, 7)), offs), (dict(img_off=(0, 3, 2)), offs), (dict(img_off=(0, -1, 7)), offs),
        (dict(null={"cams"}), "null keypoint buffer"), (dict(null={"kp_out"}), "null keypoint buffer"),
        (dict(null={"track_of"}), "null keypoint buffer"),
        (dict(null={"kp"}), kpb), (dict(null={"pts"}), kpb), (dict(img_off=(0, 0, 0), null={"cams"}), kpb),
        (dict(pairs=(0, 2)), "pairs: image index out of range"), (dict(pairs=(-1, 0)), "pairs: image index out of range"),
        (dict(pairs=(0, 1, 1, 2), n_pairs=2), "pairs: image index out of range"),
        (dict(min_length=1, rows=-1), sizes), (dict(null={"idx1"}, min_length=1), "null row buffer"),
    ]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert L.dgb200_tracks_last_error().decode() == msg, kw
    # with no row, no keypoint: the row and keypoint buffers may be null (refused here only by the pair index)
    assert call(img_off=(0, 0, 0), rows=0, null={"idx1", "idx2", "cams", "kp_out", "track_of", "kp", "pts"},
                pairs=(0, 5)) == -1
    assert L.dgb200_tracks_last_error().decode() == "pairs: image index out of range"


# ------------------------------------------------------------------------------------------------ GPU
def _run(g_layout, counts, kp=None, min_length=2, idx64=False, mask_u8=False, no_mask=False):
    import torch
    from pydegensac_b200.matching import build_tracks_ragged
    pairs, i1, i2, off, mask = g_layout
    dev = torch.device("cuda:0")
    dt = torch.int64 if idx64 else torch.int32
    m = None if no_mask else torch.from_numpy(mask).to(dev)
    if m is not None and mask_u8:
        m = m.to(torch.uint8)
    kps = None
    if kp is not None:
        base = o.img_offsets(counts)
        kps = [torch.from_numpy(kp[base[i]:base[i + 1]]).to(dev) for i in range(len(counts))]
    i1c = np.clip(i1, -2 ** 31, 2 ** 31 - 1) if not idx64 else i1
    i2c = np.clip(i2, -2 ** 31, 2 ** 31 - 1) if not idx64 else i2
    ts = build_tracks_ragged(list(counts), pairs, torch.from_numpy(i1c).to(dev, dt), torch.from_numpy(i2c).to(dev, dt),
                             torch.from_numpy(off).to(dev), m, kps=kps, min_length=min_length)
    return {k: (None if v is None else v.cpu().numpy()) for k, v in ts._asdict().items()}


def _same(got, ref):
    for k in ("offsets", "cams", "kp", "track_of", "stats"):
        assert got[k].dtype == np.int32 and np.array_equal(got[k], ref[k]), k
    if ref["pts"] is None:
        assert got["pts"] is None
    else:
        assert got["pts"].shape == ref["pts"].shape
        assert np.array_equal(got["pts"].view(np.uint64), ref["pts"].view(np.uint64))


def _kp(counts, seed):
    N = int(np.sum(counts))
    return np.random.default_rng(seed).uniform(-10, 650, (N, 2))


@pytest.mark.gpu
@pytest.mark.parametrize("min_length", [2, 3, 4])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_gpu_equals_oracle(case, min_length):
    seed, I, kw = CASES[case]
    g = graph(seed, I, **kw)
    lay = layout(g)
    kp = _kp(g["counts"], seed) if case % 2 == 0 else None
    ref = o.build_tracks(g["counts"], *lay, kp=kp, min_length=min_length)
    got = _run(lay, g["counts"], kp, min_length, idx64=case % 3 == 0, mask_u8=case % 4 == 1)
    _same(got, ref)
    if kw.get("long_track"):
        assert (np.diff(got["offsets"][:got["stats"][0] + 1]) == I).any()
    # without a mask every row of a well-formed pair counts
    ref = o.build_tracks(g["counts"], *lay[:4], None, kp=kp, min_length=min_length)
    _same(_run(lay, g["counts"], kp, min_length, no_mask=True), ref)


@pytest.mark.gpu
def test_gpu_same_bytes_under_reordering():
    for seed, I, kw in CASES[2:]:
        g = graph(seed, I, malformed=False, **kw)
        kp = _kp(g["counts"], seed)
        first = _run(layout(g), g["counts"], kp)
        ref = o.build_tracks(g["counts"], *layout(g), kp=kp)
        _same(first, ref)
        _same(_run(layout(g), g["counts"], kp), ref)                       # a rerun
        P = len(g["pairs"])
        rng = np.random.default_rng(seed + 100)
        order = rng.permutation(P)
        _same(_run(layout(g, order=order), g["counts"], kp), ref)          # pairs permuted
        _same(_run(layout(g, row_perm_seed=seed), g["counts"], kp), ref)   # rows permuted within pairs
        flip = rng.choice(P, P // 2, replace=False)
        _same(_run(layout(g, flip=flip), g["counts"], kp), ref)            # pair directions swapped
        _same(_run(layout(g, order=order, flip=flip, row_perm_seed=seed + 1), g["counts"], kp), ref)


@pytest.mark.gpu
def test_gpu_edge_cases():
    # no keypoint at all; one image with only a self-pair; every row masked; all pairs malformed
    lay = (np.array([[0, 1]]), np.array([0, 1]), np.array([1, 0]), np.array([0, 2], np.int32), np.ones(2, bool))
    _same(_run(lay, [0, 0]), o.build_tracks([0, 0], *lay))
    _same(_run(lay, [0, 0], kp=np.zeros((0, 2))), o.build_tracks([0, 0], *lay, kp=np.zeros((0, 2))))
    lay = (np.array([[0, 0]]), np.array([0, 1, 2]), np.array([1, 2, 2]), np.array([0, 3], np.int32), np.ones(3, bool))
    r = _run(lay, [4])
    _same(r, o.build_tracks([4], *lay))
    assert list(r["stats"]) == [0, 0, 1, 3] and (r["track_of"] == -1).all()
    lay = (np.array([[0, 1]]), np.array([0, 1]), np.array([1, 0]), np.array([0, 2], np.int32), np.zeros(2, bool))
    r = _run(lay, [2, 2])
    assert list(r["stats"]) == [0, 0, 0, 0] and list(r["offsets"]) == [0, 0, 0]
    lay = (np.array([[0, 1], [1, 0]]), np.array([0, 1]), np.array([1, 0]), np.array([-1, 2, 1], np.int32),
           np.ones(2, bool))
    _same(_run(lay, [2, 2]), o.build_tracks([2, 2], *lay))
    # rows past offsets[P] are never read: with rows = 0 past the end, a huge junk tail changes nothing
    lay = (np.array([[0, 1]]), np.r_[0, np.full(1000, 1)], np.r_[1, np.full(1000, 0)], np.array([0, 1], np.int32),
           np.ones(1001, bool))
    r = _run(lay, [2, 2])
    assert list(r["stats"]) == [1, 2, 0, 0] and list(r["cams"]) == [0, 1, -1, -1] and list(r["kp"]) == [0, 1, -1, -1]


@pytest.mark.gpu
def test_gpu_large_graph_equals_oracle():
    """about 4e6 keypoints: 500 images of 8000, each paired with its next 8, 400 verified rows per pair from planted
    points plus 20 junk rows; one call against the oracle, byte for byte"""
    rng = np.random.default_rng(3)
    I, n, P_nb = 500, 8000, 8
    counts = np.full(I, n)
    counts[rng.choice(I, 5, replace=False)] = 0
    # planted points: point m is seen by images m_0 .. m_0 + span at random keypoints (collisions make conflicts)
    pairs, i1, i2 = [], [], []
    kp_of = {}
    for i in range(I):
        for d in range(1, P_nb + 1):
            j = (i + d) % I
            pairs.append((i, j))
            if counts[i] == 0 or counts[j] == 0:
                i1.append(np.zeros(0, np.int64)); i2.append(np.zeros(0, np.int64))
                continue
            a = rng.integers(0, n, 420)
            b = (a * 7 + d * 13 + i) % n                 # a structured map: chains of keypoints across images
            b[400:] = rng.integers(-5, n + 5, 20)
            i1.append(a); i2.append(b)
    counts_rows = [len(x) for x in i1]
    off = np.r_[0, np.cumsum(counts_rows)].astype(np.int32)
    i1, i2 = np.concatenate(i1), np.concatenate(i2)
    mask = rng.random(len(i1)) < 0.9
    lay = (np.array(pairs), i1, i2, off, mask)
    kp = _kp(counts, 4)
    ref = o.build_tracks(counts, *lay, kp=kp, min_length=3)
    got = _run(lay, counts, kp, min_length=3)
    print("N %d, stats %s" % (counts.sum(), list(got["stats"])))
    assert got["stats"][0] > 1000
    _same(got, ref)


def _planted_ids(kps, Rs, ts, Ks, n_pts, seed):
    """the planted point of every keypoint of tests.test_refine_fundamental._multiview_two_cameras (-1 for clutter):
    the point that projects within 0.5 px of it"""
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(seed)
    X = np.c_[rng.uniform(-4, 4, n_pts), rng.uniform(-4, 4, n_pts), rng.uniform(2, 12, n_pts)]
    ids = []
    for kp, R, t, K in zip(kps, Rs, ts, Ks):
        x = (K @ (R @ X.T + t[:, None])).T
        d, idx = cKDTree(x[:, :2] / x[:, 2:3]).query(kp)
        ids.append(np.where(d < 0.5, idx, -1))
    return X, ids


@pytest.mark.gpu
def test_pipeline_match_verify_build_triangulate_adjust_register_without_sync():
    """all pairs of 5 views -> match_descriptors_batch -> ragged F RANSAC -> build_tracks_ragged ->
    triangulate_tracks_ragged on the padded layout with the planted poses -> bundle_adjust_ragged, with no host
    synchronisation; then a sixth view registered by P3P through a track_of lookup"""
    import torch
    import pydegensac_b200 as pdg
    from pydegensac_b200.matching import (build_tracks_ragged, bundle_adjust_ragged, find_absolute_pose_ragged,
                                          match_descriptors_batch, triangulate_tracks_ragged, trim_tracks)
    from tests.test_refine_fundamental import _multiview_two_cameras
    dev = torch.device("cuda:0")
    V, n_pts, seed = 5, 700, 31
    kps, descs, Rs, ts, Ks, _ = _multiview_two_cameras(V + 1, n_pts, 250, 0, 64, seed)
    keep = np.random.default_rng(seed).random(len(kps[0])) < 0.6     # view 0 misses 40 % of the scene
    kps[0], descs[0] = kps[0][keep], descs[0][keep]
    X_true, ids = _planted_ids(kps, Rs, ts, Ks, n_pts, seed)
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    pairs = np.array([(i, j) for i in range(V) for j in range(i + 1, V)], np.int32)
    f64 = torch.float64
    R = torch.from_numpy(np.stack(Rs[:V])).to(dev)
    t = torch.from_numpy(np.stack(ts[:V])).to(dev)
    K = torch.from_numpy(np.stack(Ks[:V])).to(dev)
    K5 = torch.from_numpy(Ks[V]).to(dev)
    seeds = torch.arange(len(pairs), dtype=torch.int64, device=dev) + 7
    counts = [len(k) for k in kps[:V]]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m = match_descriptors_batch(dt[:V], pairs, kt[:V], ratio=0.9, mutual=True)
        F, mask = pdg.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                                 n_max=m.n_max)
        tks = build_tracks_ragged(counts, pairs, m.idx1, m.idx2, m.offsets, mask, kps=kt[:V])
        tr = triangulate_tracks_ragged(tks.cams, tks.pts, R, t, K, tks.offsets, px_th=2.0)
        ba = bundle_adjust_ragged(tks.cams, tks.pts, R, t, K, tks.offsets, tr.X, mask=tr.mask, free=[1, 2, 3, 4],
                                  max_iters=10)
        # the held-out view: its matches to view 0 see the tracks through track_of
        m5 = match_descriptors_batch([dt[V], dt[0]], [(0, 1)], [kt[V], kt[0]], ratio=0.9, mutual=True)
        live = torch.arange(m5.idx2.shape[0], device=dev) < m5.offsets[1]
        trk = tks.track_of.index_select(0, torch.where(live, m5.idx2, 0))
        ok = live & (trk >= 0)
        j = trk.clamp(min=0)
        X5 = tr.X.index_select(0, j)
        ok = ok & (tr.n_inliers.index_select(0, j) >= 2) & torch.isfinite(X5).all(1)
        view = find_absolute_pose_ragged(m5.pts1, X5, K5, m5.offsets, ok, px_th=2.0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    s = tks.stats.cpu().numpy()
    T, n_obs = int(s[0]), int(s[1])
    ex = trim_tracks(tks)
    off, cams, kp = ex.offsets.cpu().numpy(), ex.cams.cpu().numpy(), ex.kp.cpu().numpy()
    assert len(off) == T + 1 and off[-1] == n_obs and len(cams) == n_obs
    # tracks against the planted points
    pid = np.array([ids[c][k] for c, k in zip(cams, kp)])
    pure = np.array([(pid[off[j]] >= 0) and (pid[off[j]:off[j + 1]] == pid[off[j]]).all() for j in range(T)])
    lens = np.diff(off)
    print("tracks %d (%d observations, length %s), pure %.4f, conflicting components %d (%d keypoints)"
          % (T, n_obs, np.bincount(lens).tolist(), pure.mean(), s[2], s[3]))
    assert T >= 300 and pure.mean() >= 0.95 and lens.max() >= 4
    assert (cams[off[:-1]] > 0).any()                  # tracks that view 0 does not see
    # the whole padded layout, as the device output it is: empty tracks get no model and keep their X
    Xt, Xb = tr.X.cpu().numpy(), ba.X.cpu().numpy()
    assert np.isnan(Xt[T:]).all() and np.array_equal(Xb[T:].view(np.uint64), Xt[T:].view(np.uint64))
    assert (tr.n_inliers.cpu().numpy()[T:] == 0).all()
    good = tr.n_inliers.cpu().numpy()[:T] >= 2
    err = np.linalg.norm(Xt[:T][good & pure] - X_true[pid[off[:-1]][good & pure]], axis=1)
    print("triangulated %d, median 3D error %.3e; bundle adjustment cost %.2f -> %.2f in %d steps"
          % (good.sum(), np.median(err), float(ba.cost0[0]), float(ba.cost[0]), int(ba.iters[0])))
    assert np.median(err) < 0.05 and float(ba.cost[0]) <= float(ba.cost0[0])
    # the held-out view, registered through track_of
    Rv = view.R[0].cpu().numpy()
    rot = np.arccos(np.clip((np.trace(Rv @ Rs[V].T) - 1) / 2, -1, 1))
    cen = np.linalg.norm(-Rv.T @ view.t[0].cpu().numpy() + Rs[V].T @ ts[V])
    print("held-out view: %d inliers, rotation error %.2e rad, centre error %.2e" % (int(view.n_inliers[0]), rot, cen))
    assert int(view.n_inliers[0]) >= 100 and rot < 5e-3 and cen < 5e-2
