#!/usr/bin/env python
"""Calibrated two-view verification on one GPU: find_essential_ragged against the ragged F RANSAC followed by pose.

    python tools/essential_rate.py [--pairs 512] [--rounds 5] [--out FILE]

Workloads (seeded): P = 512 calibrated pairs of 500 to 3000 correspondences each, camera 1 at the origin and camera 2 at
a random rotation of up to ~30 degrees and a unit baseline, points 3-10 units in front of camera 1, 0.5 px Gaussian
noise; one batch with 30 % true rows, one with 70 %, and one planar batch (every point on one plane, 70 % true rows).
The rest are random pixels in image 2.  Per batch, the two paths alternate within the run:
  E path  find_essential_ragged(px_th 1, conf 0.999, max_iters 10000, refine_iters 10), then
          pose_from_fundamental_ragged(ess.F, K, K, ...) for the cheirality vote;
  F path  findFundamentalMatrixBatch(offsets=..., px_th 1, conf 0.999, max_iters 10000), then
          pose_from_fundamental_ragged(F, K, K, ...).
Each call pair is timed with CUDA events after one warm-up; the median over the rounds.  Reported per path: the time,
the RANSAC iterations per pair (mean, largest) and the median rotation and translation-direction errors of the pose
against the planted one.  The card's name, power limit and clocks are read before and after.  Prints one JSON line."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import pydegensac_b200 as pdg  # noqa: E402
from pydegensac_b200.matching import find_essential_ragged, pose_from_fundamental_ragged  # noqa: E402
from pydegensac_b200.scenes import _K  # noqa: E402
from match_batch_rate import card, emit, med  # noqa: E402
from pose_ragged_rate import event_ms  # noqa: E402

PX_TH, CONF, MAX_ITERS = 1.0, 0.999, 10000


def _rotation(rng, max_angle):
    w = rng.normal(size=3)
    w *= rng.uniform(0.0, max_angle) / np.linalg.norm(w)
    a = np.linalg.norm(w)
    W = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]]) / a
    return np.eye(3) + np.sin(a) * W + (1 - np.cos(a)) * W @ W


def synth(P, lo, hi, w, sigma, planar, seed):
    """pts1, pts2 [rows,2], offsets [P+1], planted R [P,3,3], t [P,3] (unit)"""
    rng = np.random.default_rng(seed)
    Ki = np.linalg.inv(_K)
    p1s, p2s, Rs, ts = [], [], [], []
    for _ in range(P):
        n = int(rng.integers(lo, hi + 1))
        R = _rotation(rng, np.radians(30.0))
        t = rng.normal(size=3)
        t /= np.linalg.norm(t)
        u = np.c_[rng.uniform(0, 640, n), rng.uniform(0, 480, n)]
        ray = np.c_[u, np.ones(n)] @ Ki.T
        if planar:
            nrm = np.array([0.2, -0.1, 1.0]) + 0.2 * rng.normal(size=3)
            z = 6.0 / (ray @ nrm)
        else:
            z = rng.uniform(3.0, 10.0, n)
        q = (ray * z[:, None] @ R.T + t) @ _K.T
        x2 = q[:, :2] / q[:, 2:] + sigma * rng.normal(size=(n, 2))
        x1 = u + sigma * rng.normal(size=(n, 2))
        out = rng.random(n) >= w
        x2[out] = np.c_[rng.uniform(0, 640, out.sum()), rng.uniform(0, 480, out.sum())]
        p1s.append(x1); p2s.append(x2); Rs.append(R); ts.append(t)
    off = np.r_[0, np.cumsum([len(x) for x in p1s])].astype(np.int32)
    return np.concatenate(p1s), np.concatenate(p2s), off, np.stack(Rs), np.stack(ts)


def pose_errors(R, t, Rt, tt):
    """rotation angle and translation-direction angle per pair (NaN for a pair without a pose)"""
    c = np.clip((np.einsum("pij,pij->p", R, Rt) - 1.0) / 2.0, -1.0, 1.0)
    er = np.arccos(c)
    nt = np.linalg.norm(t, axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        et = np.arccos(np.clip(np.einsum("pi,pi->p", t, tt) / nt, -1.0, 1.0))
    bad = nt == 0
    er[bad] = np.nan
    et[bad] = np.nan
    return er, et


def summary(e):
    return {"median": float(np.nanmedian(e)), "p90": float(np.nanpercentile(e, 90)), "no_pose": int(np.isnan(e).sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--min-rows", type=int, default=500)
    ap.add_argument("--max-rows", type=int, default=3000)
    ap.add_argument("--sigma", type=float, default=0.5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    P = args.pairs
    res = {"workload": "%d calibrated pairs of %d to %d rows per batch, %.1f px noise; px_th %g, conf %g, max_iters %d; "
                       "E path refine_iters 10" % (P, args.min_rows, args.max_rows, args.sigma, PX_TH, CONF, MAX_ITERS),
           "card": card(), "rounds": args.rounds,
           "timing": "CUDA events around each path (RANSAC + pose_from_fundamental_ragged), one warm-up each, the two "
                     "paths alternating within the run; median over the rounds"}
    dK = torch.from_numpy(_K).to(dev)
    seeds = torch.arange(P, dtype=torch.int64, device=dev)
    for name, w, planar, seed in (("w30", 0.3, False, 1), ("w70", 0.7, False, 2), ("planar_w70", 0.7, True, 3)):
        p1, p2, off, Rt, tt = synth(P, args.min_rows, args.max_rows, w, args.sigma, planar, seed)
        d1, d2, doff = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (p1, p2, off))
        n_max = int(np.diff(off).max())

        def e_path():
            ess = find_essential_ragged(d1, d2, dK, dK, doff, px_th=PX_TH, conf=CONF, max_iters=MAX_ITERS, seeds=seeds)
            return ess, pose_from_fundamental_ragged(ess.F, dK, dK, d1, d2, doff, ess.mask)

        def f_path():
            F, mask, stats = pdg.findFundamentalMatrixBatch(d1, d2, PX_TH, CONF, MAX_ITERS, seeds=seeds, offsets=doff,
                                                            n_max=n_max, return_stats=True)
            return stats, pose_from_fundamental_ragged(F, dK, dK, d1, d2, doff, mask)

        event_ms(e_path)
        event_ms(f_path)
        te, tf = [], []
        for _ in range(args.rounds):
            ms, eo = event_ms(e_path)
            te.append(ms)
            ms, fo = event_ms(f_path)
            tf.append(ms)
        ess, epose = eo
        stats, fpose = fo
        ie = ess.iters.cpu().numpy()
        i_f = stats[:, 0].cpu().numpy()
        er_e, et_e = pose_errors(epose.R.cpu().numpy(), epose.t.cpu().numpy(), Rt, tt)
        er_f, et_f = pose_errors(fpose.R.cpu().numpy(), fpose.t.cpu().numpy(), Rt, tt)
        res[name] = {
            "rows": int(off[-1]),
            "essential": {"call_ms": med(te), "all_ms": te, "iters_mean": float(ie.mean()), "iters_max": int(ie.max()),
                          "rotation_rad": summary(er_e), "translation_dir_rad": summary(et_e),
                          "inliers": int(ess.n_inliers.sum().item()),
                          "cost_rose_pairs": int((ess.cost > ess.cost0).sum().item())},
            "fundamental": {"call_ms": med(tf), "all_ms": tf, "iters_mean": float(i_f.mean()),
                            "iters_max": int(i_f.max()), "rotation_rad": summary(er_f),
                            "translation_dir_rad": summary(et_f)},
        }
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
