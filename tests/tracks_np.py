"""numpy oracle of dgb200_build_tracks_ragged_dev (include/degensac_b200.h): the edges of the verified matches, the
connected components by scipy.sparse.csgraph, the conflict and length rules, and the capacity-sized output in the
kernel's order, byte for byte."""
import numpy as np


def img_offsets(counts):
    off = np.zeros(len(counts) + 1, dtype=np.int64)
    off[1:] = np.cumsum(np.asarray(counts, dtype=np.int64))
    return off


def edges(counts, pairs, idx1, idx2, offsets, mask=None):
    """the edge list (a, b) of node ids: per well-formed pair, the rows with mask set and both indices in range"""
    counts = np.asarray(counts, dtype=np.int64)
    off = img_offsets(counts)
    idx1, idx2 = np.asarray(idx1, dtype=np.int64), np.asarray(idx2, dtype=np.int64)
    offsets = np.asarray(offsets, dtype=np.int64)
    rows = len(idx1)
    A, B = [], []
    for p, (q, t) in enumerate(np.asarray(pairs, dtype=np.int64).reshape(-1, 2)):
        b, e = offsets[p], offsets[p + 1]
        if not 0 <= b <= e <= rows:
            continue
        i, j = idx1[b:e], idx2[b:e]
        keep = (i >= 0) & (i < counts[q]) & (j >= 0) & (j < counts[t])
        if mask is not None:
            keep &= np.asarray(mask[b:e]) != 0
        A.append(off[q] + i[keep])
        B.append(off[t] + j[keep])
    if not A:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(A), np.concatenate(B)


def component_roots(n, a, b):
    """the smallest node of every node's connected component (scipy's connected_components, relabelled)"""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    if n == 0:
        return np.zeros(0, np.int64)
    g = sp.coo_matrix((np.ones(len(a), np.int8), (a, b)), shape=(n, n)).tocsr()
    _, lab = connected_components(g, directed=False)
    _, first = np.unique(lab, return_index=True)      # nodes ascend, so the first of a label is its smallest node
    return first[lab].astype(np.int64)


def tracks_from_roots(counts, roots, min_length=2, kp=None):
    """the six outputs from the roots of the components: offsets [T_cap+1], cams [N], kp [N], pts [N,2] (None without
    kp, a float64 [N,2] of every node's pixel), track_of [N], stats [4]"""
    counts = np.asarray(counts, dtype=np.int64)
    I, N = len(counts), int(counts.sum())
    off = img_offsets(counts)
    img = np.repeat(np.arange(I), counts)
    node = np.arange(N)
    size = np.bincount(roots, minlength=N) if N else np.zeros(0, np.int64)
    # conflicting: a component (of two or more nodes) with two nodes of one image
    key = roots * I + img
    ks = np.sort(key)
    dup_keys = ks[1:][ks[1:] == ks[:-1]]
    conflict = np.zeros(N, bool)
    conflict[np.unique(dup_keys // I)] = True
    is_root = roots == node
    conflicting_roots = is_root & conflict
    live_root = is_root & (size >= 2) & ~conflict & (size >= min_length)
    track_of_root = np.full(N, -1, np.int64)
    track_of_root[live_root] = np.arange(int(live_root.sum()))
    track_of = track_of_root[roots] if N else np.zeros(0, np.int64)
    sel = np.nonzero(track_of >= 0)[0]
    order = sel[np.lexsort((sel, track_of[sel]))]      # by track, then by node
    T, n_obs = int(live_root.sum()), len(order)
    T_cap = N // min_length
    offsets = np.full(T_cap + 1, n_obs, np.int32)
    offsets[:T + 1] = np.r_[0, np.cumsum(size[live_root])]
    cams = np.full(N, -1, np.int32)
    kpo = np.full(N, -1, np.int32)
    cams[:n_obs] = img[order]
    kpo[:n_obs] = order - off[img[order]]
    pts = None
    if kp is not None:
        pts = np.full((N, 2), np.nan)
        pts[:n_obs] = np.asarray(kp, dtype=np.float64).reshape(N, 2)[order]
    stats = np.array([T, n_obs, int(conflicting_roots.sum()), int(size[conflicting_roots].sum())], np.int32)
    return dict(offsets=offsets, cams=cams, kp=kpo, pts=pts, track_of=track_of.astype(np.int32), stats=stats)


def build_tracks(counts, pairs, idx1, idx2, offsets, mask=None, kp=None, min_length=2):
    """the oracle of the whole entry point; kp: the [N,2] pixels of the nodes, or None"""
    a, b = edges(counts, pairs, idx1, idx2, offsets, mask)
    roots = component_roots(int(np.sum(counts)), a, b)
    return tracks_from_roots(counts, roots, min_length, kp)
