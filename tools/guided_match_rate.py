#!/usr/bin/env python
"""Rate of guided matching against the unguided batched matcher, on one GPU.

    python tools/guided_match_rate.py [--out FILE]

Workload: the one of tools/match_batch_rate.py -- I = 64 synthetic images of n = 4000 descriptors (60 % views of one
set of 3-D points, 40 % clutter), P = 512 pairs (image i against images i+1 .. i+8, mod 64) -- with float32 D = 128
and ORB-like 32-byte binary descriptors.  Per descriptor type, timed alternating on the same inputs:
  unguided   match_descriptors_batch (ratio 0.9)
  guided_F   match_descriptors_guided(guide="F", px_th=1) with the F of each pair found by findFundamentalMatrixBatch
             on the unguided matches (found once, untimed)
  guided_H   on a planar variant of the scene (the points on one plane), guide="H" at px_th=4 with the H of each pair
             found by findHomographyBatch on the unguided matches
Reported per path: ms per call, pairs/s, tentative matches and true matches (the planted correspondences), and for the
guided paths the share of (32-query x 4-train) groups that the gate leaves to compute -- counted on the host from the
geometry, over the first 16 pairs -- which is the share of distance work the kernel cannot skip.  The card's name,
power limit and clocks are read in the same run.  Prints one JSON line.
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import pydegensac_b200 as pdg  # noqa: E402
from pydegensac_b200.matching import match_descriptors_batch, match_descriptors_guided  # noqa: E402
from pydegensac_b200.scenes import _K, _rot  # noqa: E402
from tests import guided_np as G  # noqa: E402
from match_batch_rate import card, emit, flip_bits, med  # noqa: E402


def synth(n_img, n, D, binary, planar, seed=0, n_true_frac=0.6):
    """match_batch_rate.synth_images, also returning the row of every planted point in every view; planar: the
    points at depth 7 on one fronto-parallel plane (the views then are related by homographies)"""
    rng = np.random.default_rng(seed)
    n_true = int(n * n_true_frac)
    X = np.c_[rng.uniform(-2, 2, n_true), rng.uniform(-2, 2, n_true),
              np.full(n_true, 7.0) if planar else rng.uniform(5, 10, n_true)]
    code = rng.integers(0, 256, (n_true, D), dtype=np.uint8) if binary else rng.normal(size=(n_true, D)).astype(np.float32)
    kps, descs, where = [], [], []
    for i in range(n_img):
        R = _rot("y", 0.01 * i) @ _rot("x", 0.003 * i)
        t = np.array([0.05 * i, 0.01 * i, 0.0])
        x = (_K @ (R @ X.T + t[:, None])).T
        kp = np.r_[x[:, :2] / x[:, 2:3] + 0.1 * rng.normal(size=(n_true, 2)), rng.uniform(0, 640, (n - n_true, 2))]
        if binary:
            d = np.r_[flip_bits(code, 0.1, rng), rng.integers(0, 256, (n - n_true, D), dtype=np.uint8)]
        else:
            d = np.r_[code + 0.2 * rng.normal(size=code.shape).astype(np.float32),
                      rng.normal(size=(n - n_true, D)).astype(np.float32)]
        perm = rng.permutation(n)
        kps.append(kp[perm]); descs.append(d[perm])
        inv = np.empty_like(perm); inv[perm] = np.arange(n)
        where.append(inv[:n_true])
    return kps, descs, where


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def true_matches(m, pairs, where):
    off, i1, i2 = m.offsets.cpu().numpy(), m.idx1.cpu().numpy(), m.idx2.cpu().numpy()
    tot = 0
    for p, (q, t) in enumerate(pairs):
        planted = dict(zip(where[q].tolist(), where[t].tolist()))
        tot += sum(planted.get(a) == b for a, b in zip(i1[off[p]:off[p + 1]].tolist(), i2[off[p]:off[p + 1]].tolist()))
    return int(off[-1]), int(tot)


def group_share(kps, pairs, models, guide, px_th, n_pairs=16):
    """share of (32-query x 4-train) groups with at least one admitted (query, train) over the first n_pairs pairs"""
    live = total = 0
    for p in range(n_pairs):
        q, t = pairs[p]
        adm = G.gate(models[p], guide, kps[q], kps[t], px_th)
        n1, n2 = adm.shape
        a = np.zeros((-(-n1 // 32) * 32, -(-n2 // 4) * 4), bool)
        a[:n1, :n2] = adm
        g = a.reshape(a.shape[0] // 32, 32, a.shape[1] // 4, 4).any(axis=(1, 3))
        live += int(g.sum()); total += g.size
    return live / total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--n", type=int, default=4000)
    ap.add_argument("--neighbours", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    pairs = np.array([(i, (i + k) % args.images) for i in range(args.images) for k in range(1, args.neighbours + 1)],
                     dtype=np.int32)
    P = len(pairs)
    seeds = np.arange(P, dtype=np.uint64)
    res = {"workload": "%d images x %d descriptors, %d pairs (each image vs its %d successors), ratio 0.9; guided F at "
                       "px_th 1, guided H at px_th 4 on a planar variant" % (args.images, args.n, P, args.neighbours),
           "card": card(), "rounds": args.rounds}
    for name, D, binary in (("l2_D128", 128, False), ("orb_32B", 32, True)):
        norm = "hamming" if binary else "l2"
        r = {}
        paths = {}
        scenes = {}
        for planar in (False, True):
            kps, descs, where = synth(args.images, args.n, D, binary, planar)
            dt = [torch.from_numpy(d).to(dev) for d in descs]
            kt = [torch.from_numpy(k).to(dev) for k in kps]
            m = match_descriptors_batch(dt, pairs, kt, 0.9, False, norm)
            if planar:
                M, _ = pdg.findHomographyBatch(m.pts1, m.pts2, 2.0, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                               n_max=m.n_max)
                guide, px_th, key = "H", 4.0, "guided_H"
            else:
                M, _ = pdg.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds,
                                                      offsets=m.offsets, n_max=m.n_max)
                guide, px_th, key = "F", 1.0, "guided_F"
                paths["unguided"] = (lambda dt=dt, kt=kt: match_descriptors_batch(dt, pairs, kt, 0.9, False, norm))
                scenes["unguided"] = where
            paths[key] = (lambda dt=dt, kt=kt, M=M, guide=guide, px_th=px_th:
                          match_descriptors_guided(dt, pairs, kt, M, px_th, guide, 0.9, False, norm))
            scenes[key] = where
            r[key] = {"px_th": px_th, "gate_group_share_first16": group_share(kps, pairs, M.cpu().numpy(), guide, px_th)}
            if planar:
                r[key]["unguided_on_planar"] = dict(zip(("tentative", "true"), true_matches(m, pairs, where)))
        for fn in paths.values():      # warm-up
            timed(fn)
        t = {k: [] for k in paths}
        outs = {}
        for _ in range(args.rounds):
            for k, fn in paths.items():
                s, outs[k] = timed(fn)
                t[k].append(s)
        for k in paths:
            tent, tru = true_matches(outs[k], pairs, scenes[k])
            r.setdefault(k, {}).update({"ms": 1e3 * med(t[k]), "pairs_per_s": P / med(t[k]), "all_s": t[k],
                                        "tentative": tent, "true": tru})
        res[name] = r
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
