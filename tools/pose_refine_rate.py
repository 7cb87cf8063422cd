#!/usr/bin/env python
"""Rate and effect of refine_pose_ragged on one GPU, against the ragged F RANSAC and pose steps before it.

    python tools/pose_refine_rate.py [--pairs 512] [--rounds 5] [--out FILE]

Workload: the batch of tools/pose_ragged_rate.py -- P = 512 synthetic two-view pairs of 500 to 3000 correspondences
each (uniform, seeded), 70 % of them views of random 3-D points with 0.3 px noise in both images and 30 % random
pixels -- but with nothing planted downstream: F and the inlier mask come from the ragged RANSAC
(findFundamentalMatrixBatch(..., offsets=), px_th 1, conf 0.999, 10000 iterations), the pose from
pose_from_fundamental_ragged on them, and the refinement runs on pose.in_front, as the pipeline does.
Timed with CUDA events after one warm-up call of each step, alternating the steps in every round:
  ransac   the ragged F RANSAC
  pose     pose_from_fundamental_ragged on its F and mask
  refine   refine_pose_ragged(pose.R, pose.t, ..., pose.in_front, max_iters=10, px_th=1)
Reported besides: trial steps per pair, the refinement's share of ransac + pose + refine, and the median rotation and
translation-direction errors against the planted poses before and after.  The card's name, power limit and clocks are
read before and after.  Needs a GPU.  Prints one JSON line.
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
from pydegensac_b200.matching import pose_from_fundamental_ragged, refine_pose_ragged  # noqa: E402
from pydegensac_b200.scenes import _K, _rot  # noqa: E402
from match_batch_rate import card, emit, med  # noqa: E402
from pose_ragged_rate import event_ms  # noqa: E402


def synth(P, lo, hi, inlier_frac, seed=0):
    """the scenes of pose_ragged_rate.synth (same seeded draws), returning the planted poses instead of F"""
    rng = np.random.default_rng(seed)
    ps1, ps2, Rs, ts, lengths = [], [], [], [], []
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
        ps1.append(p1); ps2.append(p2); Rs.append(R); ts.append(t / np.linalg.norm(t)); lengths.append(n)
    off = np.r_[0, np.cumsum(lengths)].astype(np.int32)
    return np.concatenate(ps1), np.concatenate(ps2), np.stack(Rs), np.stack(ts), off


def pose_errors(R, t, Rp, tp):
    """rotation angle of R Rp^T and angle between t and tp, radians, per pair"""
    tr = np.einsum("pij,pij->p", R, Rp)
    return np.arccos(np.clip((tr - 1) / 2, -1, 1)), np.arctan2(np.linalg.norm(np.cross(t, tp), axis=1), (t * tp).sum(1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--min-rows", type=int, default=500)
    ap.add_argument("--max-rows", type=int, default=3000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--max-iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")         # no GPU: torch raises here
    p1, p2, Rp, tp, off = synth(args.pairs, args.min_rows, args.max_rows, 0.7)
    P = args.pairs
    d1, d2, doff, dK = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (p1, p2, off, _K))
    seeds = torch.arange(P, dtype=torch.int64, device=dev)
    n_max = int(np.diff(off).max())
    res = {"workload": "%d pairs, %d to %d rows each (%d in all), 70 %% true matches with 0.3 px noise; F and mask from the "
                       "ragged RANSAC (px_th 1, conf 0.999, 10000 iterations), pose from them, refinement on pose.in_front, "
                       "max_iters %d, px_th 1" % (P, args.min_rows, args.max_rows, int(off[-1]), args.max_iters),
           "card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call"}
    state = {}

    def ransac():
        state["F"], state["mask"] = pdg.findFundamentalMatrixBatch(d1, d2, 1.0, 0.999, 10000, seeds=seeds, offsets=doff,
                                                                   n_max=n_max)

    def pose():
        state["pose"] = pose_from_fundamental_ragged(state["F"], dK, dK, d1, d2, doff, state["mask"])

    def refine():
        ps = state["pose"]
        state["fine"] = refine_pose_ragged(ps.R, ps.t, dK, dK, d1, d2, doff, ps.in_front, max_iters=args.max_iters,
                                           px_th=1.0)

    steps = {"ransac": ransac, "pose": pose, "refine": refine}
    for fn in steps.values():
        event_ms(fn)
    t = {k: [] for k in steps}
    for _ in range(args.rounds):
        for k, fn in steps.items():
            t[k].append(event_ms(fn)[0])
    for k in steps:
        res[k] = {"ms": med(t[k]), "pairs_per_s": 1e3 * P / med(t[k]), "all_ms": t[k]}
    total = sum(med(t[k]) for k in steps)
    res["refine_share_of_ransac_plus_pose_plus_refine"] = med(t["refine"]) / total
    ps, fine = state["pose"], state["fine"]
    iters = fine.iters.cpu().numpy()
    res["trial_steps_per_pair"] = {"mean": float(iters.mean()), "max": int(iters.max()),
                                   "at_max_iters": int((iters == args.max_iters).sum())}
    res["rows_used"] = int(fine.n_used.sum().item())
    res["row_passes_per_pair_mean"] = float(iters.mean()) + 2.0      # the start, one per trial step, the inlier rows
    c0, c1 = fine.cost0.cpu().numpy(), fine.cost.cpu().numpy()
    res["cost_px2_per_row_median"] = {"before": float(np.nanmedian(c0 / fine.n_used.cpu().numpy())),
                                      "after": float(np.nanmedian(c1 / fine.n_used.cpu().numpy()))}
    res["cost_never_rises"] = bool((c1 <= c0).all())
    eR0, et0 = pose_errors(ps.R.cpu().numpy(), ps.t.cpu().numpy(), Rp, tp)
    eR1, et1 = pose_errors(fine.R.cpu().numpy(), fine.t.cpu().numpy(), Rp, tp)
    res["rotation_error_deg"] = {"median_before": float(np.degrees(np.median(eR0))), "median_after": float(np.degrees(np.median(eR1))),
                                 "p90_before": float(np.degrees(np.quantile(eR0, 0.9))), "p90_after": float(np.degrees(np.quantile(eR1, 0.9)))}
    res["translation_direction_error_deg"] = {"median_before": float(np.degrees(np.median(et0))), "median_after": float(np.degrees(np.median(et1))),
                                              "p90_before": float(np.degrees(np.quantile(et0, 0.9))), "p90_after": float(np.degrees(np.quantile(et1, 0.9)))}
    res["pairs_improved"] = {"rotation": int((eR1 < eR0).sum()), "translation": int((et1 < et0).sum()), "of": P}
    res["inliers_px1"] = {"ransac_mask": int(state["mask"].sum().item()), "refined_F": int(fine.inliers.sum().item())}
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
