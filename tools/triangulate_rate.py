#!/usr/bin/env python
"""Rate and accuracy of triangulate_tracks_ragged on one GPU, with the numpy oracle on a subset of the tracks beside.

    python tools/triangulate_rate.py [--tracks 1000000] [--cameras 200] [--rounds 5] [--out FILE]

Workload (seeded): C = 200 cameras along a 20-unit line (centres 0.1 units apart with 0.1 units of jitter, rotations
below 0.1 rad, looking along +z, one K), T = 10^6 tracks.  A track's length is 2 + a geometric draw (p = 0.15) capped
at 20, and one track in a thousand has 200-400 observations; its cameras are consecutive from a random start (wrapping
around past the last camera), so its point, 4-12 units ahead and within 3 units sideways of their middle, is seen
from a spread of baselines.  Observations get 0.5 px Gaussian noise; 10 % of them are replaced by uniform random
pixels (outliers).  One call of triangulate_tracks_ragged(px_th 2, min_angle 1.5 deg, conf 0.999, max_iters 1000,
refine_iters 10) over the whole batch, timed with CUDA events after one warm-up call; the median of the rounds.
Also reported: the iterations per track (mean, largest), the share of tracks triangulated, the median 3D error to the
planted points with refine_iters 0 (the RANSAC point) and 10, and the numpy oracle (tests/triangulate_np.py, one CPU
core) on the first --cpu-tracks tracks, labelled as that.  The card's name, power limit and clocks are read before and
after.  Prints one JSON line.
"""
import argparse
import math
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from pydegensac_b200.matching import triangulate_tracks_ragged  # noqa: E402
from pydegensac_b200.scenes import _K, _rot  # noqa: E402
from match_batch_rate import card, emit, med  # noqa: E402
from pose_ragged_rate import event_ms  # noqa: E402

PX_TH, MIN_ANGLE, CONF, MAX_ITERS = 2.0, math.radians(1.5), 0.999, 1000


def synth(T, C, sigma, outliers, seed=0):
    """cams [obs] int32, pts [obs,2], R [C,3,3], t [C,3], offsets [T+1], planted points [T,3], is_outlier [obs]"""
    rng = np.random.default_rng(seed)
    R = np.stack([_rot("y", rng.uniform(-0.1, 0.1)) @ _rot("x", rng.uniform(-0.05, 0.05)) for _ in range(C)])
    centres = np.c_[0.1 * np.arange(C) - 0.05 * C, rng.uniform(-0.1, 0.1, C), rng.uniform(-0.1, 0.1, C)]
    t = -np.einsum("cij,cj->ci", R, centres)
    L = np.minimum(2 + rng.geometric(0.15, T) - 1, 20)
    tail = rng.random(T) < 1e-3
    L[tail] = rng.integers(200, 401, int(tail.sum()))
    off = np.r_[0, np.cumsum(L)].astype(np.int64)
    obs = int(off[-1])
    start = rng.integers(0, C, T)
    trk = np.repeat(np.arange(T), L)
    pos = np.arange(obs) - off[trk]
    cams = (start[trk] + pos) % C
    mid = centres[(start + (np.minimum(L, C) - 1) // 2) % C, 0]
    X = np.c_[mid + rng.uniform(-3, 3, T), rng.uniform(-2, 2, T), rng.uniform(4, 12, T)]
    p = np.einsum("oij,oj->oi", R[cams], X[trk]) + t[cams]
    q = p @ _K.T
    pts = q[:, :2] / q[:, 2:] + sigma * rng.normal(size=(obs, 2))
    out = rng.random(obs) < outliers
    pts[out] = np.c_[rng.uniform(0, 640, int(out.sum())), rng.uniform(0, 480, int(out.sum()))]
    return cams.astype(np.int32), pts, R, t, off.astype(np.int32), X, out


def summary(e):
    return {"median": float(np.median(e)), "p90": float(np.percentile(e, 90)), "worst": float(e.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tracks", type=int, default=1000000)
    ap.add_argument("--cameras", type=int, default=200)
    ap.add_argument("--sigma", type=float, default=0.5)
    ap.add_argument("--outliers", type=float, default=0.1)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cpu-tracks", type=int, default=2000, help="tracks run through the numpy oracle (0: none)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    T, C = args.tracks, args.cameras
    cams, pts, R, t, off, Xt, out = synth(T, C, args.sigma, args.outliers)
    L = np.diff(off)
    d = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (cams, pts, R, t, _K, off)]
    seeds = torch.arange(T, dtype=torch.int64, device=dev)
    res = {"workload": "%d tracks (%d observations; lengths 2-20, mean %.2f, and %d tracks of 200-400) over %d cameras "
                       "on a line, %.0f %% outlier observations, %.1f px noise; px_th %g, min_angle 1.5 deg, conf %g, "
                       "max_iters %d, refine_iters 10"
                       % (T, int(off[-1]), float(L[L <= 20].mean()), int((L > 20).sum()), C, 100 * args.outliers,
                          args.sigma, PX_TH, CONF, MAX_ITERS),
           "card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call"}

    def call(refine_iters=10):
        return triangulate_tracks_ragged(*d, px_th=PX_TH, min_angle=MIN_ANGLE, conf=CONF, max_iters=MAX_ITERS,
                                         seeds=seeds, refine_iters=refine_iters)

    event_ms(call)
    times = []
    for _ in range(args.rounds):
        ms, res_gpu = event_ms(call)
        times.append(ms)
    res["call_ms"] = med(times)
    res["all_ms"] = times
    res["tracks_per_s"] = 1e3 * T / med(times)
    iters = res_gpu.iters.cpu().numpy()
    n_in = res_gpu.n_inliers.cpu().numpy()
    res["iters"] = {"mean": float(iters.mean()), "max": int(iters.max()),
                    "mean_long_tracks": float(iters[L > 20].mean()) if (L > 20).any() else None}
    ok = n_in >= 2
    res["triangulated_share"] = float(ok.mean())
    raw = call(refine_iters=0)
    X1, X0 = res_gpu.X.cpu().numpy(), raw.X.cpu().numpy()
    both = ok & (raw.n_inliers.cpu().numpy() >= 2)
    res["error_3d_ransac"] = summary(np.linalg.norm(X0[both] - Xt[both], axis=1))
    res["error_3d_after_lo"] = summary(np.linalg.norm(X1[both] - Xt[both], axis=1))
    res["cost_rose_tracks"] = int((res_gpu.cost > res_gpu.cost0).sum().item())
    mask = res_gpu.mask.cpu().numpy()
    res["outlier_observations_kept"] = int((mask & out).sum())
    res["outlier_observations"] = int(out.sum())
    if args.cpu_tracks > 0:
        from tests import triangulate_np as o
        n = min(args.cpu_tracks, T)
        Kc = np.broadcast_to(_K, (C, 3, 3))
        s = time.perf_counter()
        ref = o.triangulate_tracks_ragged(cams[:off[n]], pts[:off[n]], R, t, Kc, off[:n + 1], px_th=PX_TH,
                                          min_angle=MIN_ANGLE, conf=CONF, max_iters=MAX_ITERS,
                                          seeds=np.arange(n, dtype=np.uint64))
        wall = time.perf_counter() - s
        same = sum(int(r["n_inliers"]) == int(n_in[j]) for j, r in enumerate(ref))
        res["numpy_oracle_subset"] = {"what": "tests/triangulate_np.py on one CPU core, first %d tracks" % n,
                                      "wall_s": wall, "tracks_per_s": n / wall, "same_n_inliers_as_gpu": same}
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
