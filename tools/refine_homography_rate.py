#!/usr/bin/env python
"""Rate and effect of refine_homography_ragged on one GPU, against the ragged H RANSAC before it.

    python tools/refine_homography_rate.py [--pairs 512] [--rounds 5] [--max-iters 10] [--out FILE]

Workload: the planar batch of tools/pose_homography_rate.py (P = 512 two-view pairs of 500 to 3000 correspondences,
0.3 px noise on 70 % of the rows, random pixels for the rest).  H and its mask come from the ragged H RANSAC on the
batch (findHomographyBatch(..., offsets=, n_max=), px_th 2, conf 0.999, 10000 iterations), so the refinement starts
where a user's would.  Timed with CUDA events after one warm-up call of each path, alternating the paths every round:
  refine   refine_homography_ragged(H, pts1, pts2, offsets, mask, max_iters, px_th=2) over the whole batch
  ransac   the ragged H RANSAC on the same batch, for the share the refinement takes
Also reported: the trial steps per pair (mean, largest), and the error of H to the planted homography before and after
(mean transfer distance over a 9 x 7 grid of the 640 x 480 image).  The card's name, power limit and clocks are read
before and after.  Prints one JSON line.
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
from pydegensac_b200.matching import refine_homography_ragged  # noqa: E402
from match_batch_rate import card, emit, med  # noqa: E402
from pose_homography_rate import synth_planar  # noqa: E402
from pose_ragged_rate import event_ms  # noqa: E402

GRID = np.stack(np.meshgrid(np.linspace(0, 640, 9), np.linspace(0, 480, 7)), -1).reshape(-1, 2)


def transfer_error(H, Hp):
    h = np.c_[GRID, np.ones(len(GRID))]
    a, b = h @ H.T, h @ Hp.T
    return float(np.linalg.norm(a[:, :2] / a[:, 2:] - b[:, :2] / b[:, 2:], axis=1).mean())


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
    p1, p2, _, Hp, off = synth_planar(P, args.min_rows, args.max_rows, 0.7)
    d1, d2, doff = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (p1, p2, off))
    seeds = torch.arange(P, dtype=torch.int64, device=dev)
    n_max = int(np.diff(off).max())
    H, mask = pdg.findHomographyBatch(d1, d2, 2.0, 0.999, 10000, seeds=seeds, offsets=doff, n_max=n_max)
    res = {"workload": "%d planar pairs, %d to %d rows each (%d in all), 70 %% inliers at 0.3 px; H and mask from the "
                       "ragged H RANSAC (px_th 2, conf 0.999, 10000 iterations); refine max_iters %d, px_th 2"
                       % (P, args.min_rows, args.max_rows, int(off[-1]), args.max_iters),
           "card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call"}

    def refine():
        return refine_homography_ragged(H, d1, d2, doff, mask, max_iters=args.max_iters, px_th=2.0)

    def ransac():
        return pdg.findHomographyBatch(d1, d2, 2.0, 0.999, 10000, seeds=seeds, offsets=doff, n_max=n_max)

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
    res["trial_steps_mean"] = float(iters.mean())
    res["trial_steps_max"] = int(iters.max())
    res["cost_rose_pairs"] = int((f.cost > f.cost0).sum().item())
    Hn, Hf = H.cpu().numpy().reshape(P, 3, 3), f.H.cpu().numpy()
    ok = [p for p in range(P) if Hn[p].any()]
    before = np.array([transfer_error(Hn[p], Hp[p]) for p in ok])
    after = np.array([transfer_error(Hf[p], Hp[p]) for p in ok])
    res["pairs_with_a_model"] = len(ok)
    res["transfer_error_px"] = {"median_before": float(np.median(before)), "median_after": float(np.median(after)),
                                "mean_before": float(before.mean()), "mean_after": float(after.mean()),
                                "worst_before": float(before.max()), "worst_after": float(after.max()),
                                "pairs_improved": int((after < before).sum())}
    res["inliers_before"] = int(mask.sum().item())
    res["inliers_after"] = int(f.inliers.sum().item())
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
