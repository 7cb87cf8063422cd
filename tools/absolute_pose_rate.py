#!/usr/bin/env python
"""Rate and accuracy of find_absolute_pose_ragged on one GPU, with cv2.solvePnPRansac on the host's CPU cores beside.

    python tools/absolute_pose_rate.py [--pairs 1024] [--rounds 5] [--out FILE]

Workload: P = 1024 views to register, each with 500 to 3000 2D-3D rows (uniform, seeded): points 2-10 units in front of
a camera with a random pose, observed through K with 0.5 px Gaussian noise; half the views have 30 % true rows, half
70 %, the rest are random pixels.  One call of find_absolute_pose_ragged(px_th 2, conf 0.999, max_iters 10000,
refine_iters 10) over the whole batch, timed with CUDA events after one warm-up call; the median of the rounds.
Also reported: the RANSAC iterations per view (mean, largest), the pose error to the planted pose (rotation angle, and
|t - t_true| over the 6-unit mean depth) before the local optimisation (refine_iters 0) and after it, and
cv2.solvePnPRansac (SOLVEPNP_P3P, the same threshold, confidence and iteration cap) over the same views in a process pool
of os.cpu_count() workers.  The card's name, power limit and clocks are read before and after.  Prints one JSON line.
"""
import argparse
import os
import sys
import time
from multiprocessing import Pool

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from pydegensac_b200.matching import find_absolute_pose_ragged  # noqa: E402
from pydegensac_b200.scenes import _K  # noqa: E402
from match_batch_rate import card, emit, med  # noqa: E402
from pose_ragged_rate import event_ms  # noqa: E402

PX_TH, CONF, MAX_ITERS = 2.0, 0.999, 10000


def _rotation(rng):
    q = rng.normal(size=4)
    a, b, c, d = q / np.linalg.norm(q)
    return np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])


def synth(P, lo, hi, sigma, seed=0):
    """x [rows,2], X [rows,3], offsets [P+1], planted (R [P,3,3], t [P,3]), inlier ratio per view"""
    rng = np.random.default_rng(seed)
    xs, Xs, Rs, ts, ws = [], [], [], [], []
    Ki = np.linalg.inv(_K)
    for p in range(P):
        n = int(rng.integers(lo, hi + 1))
        w = 0.3 if p % 2 == 0 else 0.7
        R, t = _rotation(rng), rng.uniform(-1, 1, 3)
        u = np.c_[rng.uniform(0, 640, n), rng.uniform(0, 480, n)]
        Pc = (np.c_[u, np.ones(n)] @ Ki.T) * rng.uniform(2, 10, n)[:, None]
        X = (Pc - t) @ R
        x = u + sigma * rng.normal(size=(n, 2))
        out = rng.random(n) >= w
        x[out] = np.c_[rng.uniform(0, 640, out.sum()), rng.uniform(0, 480, out.sum())]
        xs.append(x); Xs.append(X); Rs.append(R); ts.append(t); ws.append(w)
    off = np.r_[0, np.cumsum([len(x) for x in xs])].astype(np.int32)
    return np.concatenate(xs), np.concatenate(Xs), off, np.stack(Rs), np.stack(ts), np.array(ws)


def pose_errors(R, t, Rt, tt):
    c = np.clip((np.einsum("pij,pij->p", R, Rt) - 1.0) / 2.0, -1.0, 1.0)
    return np.arccos(c), np.linalg.norm(t - tt, axis=1) / 6.0


def _cv2_view(args):
    import cv2
    cv2.setNumThreads(1)
    x, X = args
    ok, rv, tv, inl = cv2.solvePnPRansac(X, x, _K, None, iterationsCount=MAX_ITERS, reprojectionError=PX_TH,
                                         confidence=CONF, flags=cv2.SOLVEPNP_P3P)
    if not ok:
        return np.zeros((3, 3)), np.zeros(3)
    return cv2.Rodrigues(rv)[0], tv.ravel()


def summary(e):
    return {"median": float(np.median(e)), "p90": float(np.percentile(e, 90)), "worst": float(e.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1024)
    ap.add_argument("--min-rows", type=int, default=500)
    ap.add_argument("--max-rows", type=int, default=3000)
    ap.add_argument("--sigma", type=float, default=0.5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true", help="skip cv2.solvePnPRansac")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    P = args.pairs
    x, X, off, Rt, tt, ws = synth(P, args.min_rows, args.max_rows, args.sigma)
    dx, dX, doff, dK = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (x, X, off, _K))
    seeds = torch.arange(P, dtype=torch.int64, device=dev)
    res = {"workload": "%d views, %d to %d 2D-3D rows each (%d in all), half at 30 %% and half at 70 %% true rows with "
                       "%.1f px noise; px_th %g, conf %g, max_iters %d, refine_iters 10"
                       % (P, args.min_rows, args.max_rows, int(off[-1]), args.sigma, PX_TH, CONF, MAX_ITERS),
           "card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call"}

    def call(refine_iters=10):
        return find_absolute_pose_ragged(dx, dX, dK, doff, px_th=PX_TH, conf=CONF, max_iters=MAX_ITERS, seeds=seeds,
                                         refine_iters=refine_iters)

    event_ms(call)
    t = []
    for _ in range(args.rounds):
        ms, out = event_ms(call)
        t.append(ms)
    res["call_ms"] = med(t)
    res["all_ms"] = t
    res["calls_per_s"] = 1e3 / med(t)
    res["views_per_s"] = 1e3 * P / med(t)
    iters = out.iters.cpu().numpy()
    res["iters"] = {"mean": float(iters.mean()), "max": int(iters.max()),
                    "mean_at_30pct": float(iters[ws == 0.3].mean()), "mean_at_70pct": float(iters[ws == 0.7].mean())}
    raw = call(refine_iters=0)
    R1, t1 = out.R.cpu().numpy(), out.t.cpu().numpy()
    R0, t0 = raw.R.cpu().numpy(), raw.t.cpu().numpy()
    er0, et0 = pose_errors(R0, t0, Rt, tt)
    er1, et1 = pose_errors(R1, t1, Rt, tt)
    res["pose_error_ransac"] = {"rotation_rad": summary(er0), "translation_over_depth": summary(et0)}
    res["pose_error_after_lo"] = {"rotation_rad": summary(er1), "translation_over_depth": summary(et1)}
    res["cost_rose_pairs"] = int((out.cost > out.cost0).sum().item())
    res["inliers"] = {"ransac": int(raw.n_inliers.sum().item()), "after_lo": int(out.n_inliers.sum().item())}
    if not args.no_cpu:
        jobs = [(x[off[p]:off[p + 1]], X[off[p]:off[p + 1]]) for p in range(P)]
        cores = os.cpu_count()
        with Pool(cores) as pool:
            pool.map(_cv2_view, jobs[:cores])            # warm-up: workers started, cv2 imported
            s = time.perf_counter()
            cv = pool.map(_cv2_view, jobs)
            wall = time.perf_counter() - s
        Rc, tc = np.stack([c[0] for c in cv]), np.stack([c[1] for c in cv])
        erc, etc = pose_errors(Rc, tc, Rt, tt)
        res["cv2_solvePnPRansac"] = {"cores": cores, "wall_s": wall, "views_per_s": P / wall,
                                     "pose_error": {"rotation_rad": summary(erc), "translation_over_depth": summary(etc)}}
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
