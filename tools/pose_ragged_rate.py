#!/usr/bin/env python
"""Rate of pose_from_fundamental_ragged on one GPU, against a loop of dense calls and against the ragged F RANSAC.

    python tools/pose_ragged_rate.py [--pairs 512] [--rounds 5] [--out FILE]

Workload: P = 512 synthetic two-view pairs of 500 to 3000 correspondences each (uniform, seeded), 70 % of them views of
random 3-D points with 0.3 px noise and 30 % random pixels; the mask given to the pose step is the planted inlier flag
(about 70 % of the rows), F the planted one.  Timed with CUDA events after one warm-up call of each path, alternating
the paths in every round:
  ragged   one pose_from_fundamental_ragged call over the whole batch (R, t, good, points, in_front, angle, median)
  loop     a Python loop of pose_from_fundamental calls, one per pair, on views of the same rows (R, t, good only)
  ransac   findFundamentalMatrixBatch(..., offsets=, n_max=) on the same batch (px_th 1, conf 0.999, 10000 iterations),
           the step before pose in the pipeline, for the share pose takes
Also checked in the same run: the ragged R, t, good equal the loop's bit for bit.  The card's name, power limit and
clocks are read before and after.  Prints one JSON line.
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import pydegensac_b200 as pdg  # noqa: E402
from pydegensac_b200.matching import pose_from_fundamental, pose_from_fundamental_ragged  # noqa: E402
from pydegensac_b200.scenes import _K, _rot  # noqa: E402
from match_batch_rate import card, emit, med  # noqa: E402


def synth(P, lo, hi, inlier_frac, seed=0):
    rng = np.random.default_rng(seed)
    Ki = np.linalg.inv(_K)
    ps1, ps2, ms, Fs, lengths = [], [], [], [], []
    for p in range(P):
        n = int(rng.integers(lo, hi + 1))
        R = _rot("y", rng.uniform(-0.3, 0.3)) @ _rot("x", rng.uniform(-0.1, 0.1))
        t = np.array([rng.uniform(0.5, 1.5), rng.uniform(-0.2, 0.2), rng.uniform(-0.3, 0.3)])
        X = np.c_[rng.uniform(-2, 2, n), rng.uniform(-2, 2, n), rng.uniform(4, 10, n)]
        x1 = X @ _K.T
        x2 = (X @ R.T + t) @ _K.T
        p1 = x1[:, :2] / x1[:, 2:3] + 0.3 * rng.normal(size=(n, 2))
        p2 = x2[:, :2] / x2[:, 2:3] + 0.3 * rng.normal(size=(n, 2))
        inl = rng.random(n) < inlier_frac
        p2[~inl] = rng.uniform(0, 640, (int((~inl).sum()), 2))
        tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
        ps1.append(p1); ps2.append(p2); ms.append(inl); Fs.append(Ki.T @ tx @ R @ Ki); lengths.append(n)
    off = np.r_[0, np.cumsum(lengths)].astype(np.int32)
    return np.concatenate(ps1), np.concatenate(ps2), np.concatenate(ms), np.stack(Fs), off


def event_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    r = fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--min-rows", type=int, default=500)
    ap.add_argument("--max-rows", type=int, default=3000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    p1, p2, mask, F, off = synth(args.pairs, args.min_rows, args.max_rows, 0.7)
    P = args.pairs
    d1, d2, dm, dF, doff, dK = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (p1, p2, mask, F, off, _K))
    seeds = torch.arange(P, dtype=torch.int64, device=dev)
    n_max = int(np.diff(off).max())
    res = {"workload": "%d pairs, %d to %d rows each (%d in all), %.1f %% masked inliers; F planted; RANSAC px_th 1, "
                       "conf 0.999, 10000 iterations" % (P, args.min_rows, args.max_rows, int(off[-1]),
                                                         100.0 * mask.mean()),
           "card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call"}

    def ragged():
        return pose_from_fundamental_ragged(dF, dK, dK, d1, d2, doff, dm)

    def loop():
        out = []
        for p in range(P):
            a, b = int(off[p]), int(off[p + 1])
            out.append(pose_from_fundamental(dF[p:p + 1], dK, dK, d1[a:b][None], d2[a:b][None], dm[a:b][None]))
        return out

    def ransac():
        return pdg.findFundamentalMatrixBatch(d1, d2, 1.0, 0.999, 10000, seeds=seeds, offsets=doff, n_max=n_max)

    paths = {"ragged": ragged, "loop": loop, "ransac": ransac}
    for fn in paths.values():
        event_ms(fn)
    t = {k: [] for k in paths}
    outs = {}
    for _ in range(args.rounds):
        for k, fn in paths.items():
            ms, outs[k] = event_ms(fn)
            t[k].append(ms)
    g = outs["ragged"]
    same = all(torch.equal(g.R[p], R[0]) and torch.equal(g.t[p], tt[0]) and torch.equal(g.good[p], gd[0])
               for p, (R, tt, gd) in enumerate(outs["loop"]))
    for k in paths:
        res[k] = {"ms": med(t[k]), "pairs_per_s": 1e3 * P / med(t[k]), "all_ms": t[k]}
    res["ragged_equals_loop"] = bool(same)
    res["loop_over_ragged"] = med(t["loop"]) / med(t["ragged"])
    res["pose_share_of_ransac_plus_pose"] = med(t["ragged"]) / (med(t["ragged"]) + med(t["ransac"]))
    res["good_sum"] = int(g.good.sum().item())
    res["median_angle_deg_median"] = float(np.degrees(np.nanmedian(g.median_angle.cpu().numpy())))
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
