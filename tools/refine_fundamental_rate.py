#!/usr/bin/env python
"""Rate and effect of refine_fundamental_ragged on one GPU, against the ragged F RANSAC before it.

    python tools/refine_fundamental_rate.py [--pairs 512] [--rounds 5] [--max-iters 10] [--out FILE]

Workload: P = 512 synthetic two-view pairs of 500 to 3000 correspondences each (uniform, seeded) of general 3-D scenes,
camera 1 calibrated by K1 and camera 2 by a different K2 (so F is not an essential matrix in disguise); 70 % of the
rows are views of the scene with 0.3 px noise in both images, 30 % random pixels.  F and its mask come from the ragged
F RANSAC on the batch (findFundamentalMatrixBatch(..., offsets=, n_max=), px_th 1, conf 0.999, 10000 iterations), so the
refinement starts where a user's would.  Timed with CUDA events after one warm-up call of each path, alternating the
paths every round:
  refine   refine_fundamental_ragged(F, pts1, pts2, offsets, mask, max_iters, px_th=1) over the whole batch
  ransac   the ragged F RANSAC on the same batch, for the share the refinement takes
Also reported: the trial steps per pair (mean, largest), whether any cost rose, and the error of F to the planted
geometry before and after: the mean Sampson distance (px) of 300 noise-free held-out correspondences of each planted
scene under F.  The card's name, power limit and clocks are read before and after.  Prints one JSON line.
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
from pydegensac_b200.matching import refine_fundamental_ragged  # noqa: E402
from pydegensac_b200.scenes import _K, _rot  # noqa: E402
from match_batch_rate import card, emit, med  # noqa: E402
from pose_ragged_rate import event_ms  # noqa: E402

K2 = _K.copy(); K2[0, 0] *= 1.1; K2[1, 1] *= 1.07; K2[0, 2] += 7.0      # tests/test_pose_refine.K2


def synth(P, lo, hi, inlier_frac, n_hold=300, seed=0):
    """p1, p2 [rows, 2], offsets [P+1] and per pair the noise-free held-out views (q1, q2) of n_hold further points"""
    rng = np.random.default_rng(seed)
    ps1, ps2, hold, lengths = [], [], [], []
    for p in range(P):
        n = int(rng.integers(lo, hi + 1))
        R = _rot("y", rng.uniform(-0.3, 0.3)) @ _rot("x", rng.uniform(-0.1, 0.1))
        t = np.array([rng.uniform(0.5, 1.5), rng.uniform(-0.2, 0.2), rng.uniform(-0.3, 0.3)])
        X = np.c_[rng.uniform(-2, 2, n + n_hold), rng.uniform(-2, 2, n + n_hold), rng.uniform(4, 10, n + n_hold)]
        x1 = X @ _K.T
        x2 = (X @ R.T + t) @ K2.T
        h1, h2 = x1[:, :2] / x1[:, 2:3], x2[:, :2] / x2[:, 2:3]
        p1 = h1[:n] + 0.3 * rng.normal(size=(n, 2))
        p2 = h2[:n] + 0.3 * rng.normal(size=(n, 2))
        inl = rng.random(n) < inlier_frac
        p2[~inl] = rng.uniform(0, 640, (int((~inl).sum()), 2))
        ps1.append(p1); ps2.append(p2); hold.append((h1[n:], h2[n:])); lengths.append(n)
    off = np.r_[0, np.cumsum(lengths)].astype(np.int32)
    return np.concatenate(ps1), np.concatenate(ps2), off, hold


def geometry_error(F, q1, q2):
    """mean Sampson distance (px) of the correspondences (q1, q2) under F (x2^T F x1 = 0)"""
    h1, h2 = np.c_[q1, np.ones(len(q1))], np.c_[q2, np.ones(len(q2))]
    a, b = h1 @ F.T, h2 @ F
    r2 = (h2 * a).sum(1) ** 2 / (a[:, 0] ** 2 + a[:, 1] ** 2 + b[:, 0] ** 2 + b[:, 1] ** 2)
    return float(np.sqrt(r2).mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--min-rows", type=int, default=500)
    ap.add_argument("--max-rows", type=int, default=3000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--max-iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    P = args.pairs
    p1, p2, off, hold = synth(P, args.min_rows, args.max_rows, 0.7)
    d1, d2, doff = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (p1, p2, off))
    seeds = torch.arange(P, dtype=torch.int64, device=dev)
    n_max = int(np.diff(off).max())
    F, mask = pdg.findFundamentalMatrixBatch(d1, d2, 1.0, 0.999, 10000, seeds=seeds, offsets=doff, n_max=n_max)
    res = {"workload": "%d general pairs (K1 != K2), %d to %d rows each (%d in all), 70 %% true matches with 0.3 px "
                       "noise; F and mask from the ragged F RANSAC (px_th 1, conf 0.999, 10000 iterations); refine "
                       "max_iters %d, px_th 1" % (P, args.min_rows, args.max_rows, int(off[-1]), args.max_iters),
           "card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call"}

    def refine():
        return refine_fundamental_ragged(F, d1, d2, doff, mask, max_iters=args.max_iters, px_th=1.0)

    def ransac():
        return pdg.findFundamentalMatrixBatch(d1, d2, 1.0, 0.999, 10000, seeds=seeds, offsets=doff, n_max=n_max)

    paths = {"refine": refine, "ransac": ransac}
    for fn in paths.values():
        event_ms(fn)
    t = {k: [] for k in paths}
    outs = {}
    for _ in range(args.rounds):
        for k, fn in paths.items():
            ms, outs[k] = event_ms(fn)
            t[k].append(ms)
    for k in paths:
        res[k] = {"ms": med(t[k]), "pairs_per_s": 1e3 * P / med(t[k]), "all_ms": t[k]}
    res["refine_share_of_ransac_plus_refine"] = med(t["refine"]) / (med(t["refine"]) + med(t["ransac"]))
    f = outs["refine"]
    iters = f.iters.cpu().numpy()
    res["trial_steps_per_pair"] = {"mean": float(iters.mean()), "max": int(iters.max()),
                                   "at_max_iters": int((iters == args.max_iters).sum())}
    res["rows_used"] = int(f.n_used.sum().item())
    res["cost_rose_pairs"] = int((f.cost > f.cost0).sum().item())
    Fn, Ff = F.cpu().numpy().reshape(P, 3, 3), f.F.cpu().numpy()
    ok = [p for p in range(P) if Fn[p].any()]
    before = np.array([geometry_error(Fn[p], *hold[p]) for p in ok])
    after = np.array([geometry_error(Ff[p], *hold[p]) for p in ok])
    res["pairs_with_a_model"] = len(ok)
    res["heldout_sampson_distance_px"] = {"median_before": float(np.median(before)), "median_after": float(np.median(after)),
                                          "mean_before": float(before.mean()), "mean_after": float(after.mean()),
                                          "worst_before": float(before.max()), "worst_after": float(after.max()),
                                          "pairs_improved": int((after < before).sum())}
    res["inliers_px1"] = {"ransac_mask": int(mask.sum().item()), "refined_F": int(f.inliers.sum().item())}
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
