#!/usr/bin/env python
"""Rate and accuracy of bundle_adjust_ragged on one GPU, with scipy.optimize.least_squares on a subset beside.

    python tools/bundle_adjust_rate.py [--tracks 100000] [--rounds 3] [--out FILE]

Workload (seeded): C = 80 cameras along an 8-unit line (centres 0.1 units apart with 0.1 units of jitter, rotations
below 0.1 rad, looking along +z, one K); cameras 0-15 held, 16-79 free (64).  T = 10^5 tracks; a track's length is
1 + a geometric draw (p = 0.2) capped at 20 (mean ~6), its cameras consecutive from a random start (wrapping around),
its point 4-12 units ahead and within 3 units sideways of their middle.  0.5 px Gaussian noise.  Start: the free
cameras rotated by ~2e-3 rad and moved by ~1e-2 units, every point moved by ~2e-2 units.  One call of
bundle_adjust_ragged(max_iters 50, squared error) timed with CUDA events after one warm-up call; the median of the
rounds, and the call time over the trial steps taken.  Errors against the planted scene before and after: the largest
and median rotation error of the free cameras and the median 3D point error.  CPU comparison: scipy's least_squares
(trf, jac_sparsity, 2-point differences) on the same cameras and the first --cpu-tracks tracks, labelled as that.
The card's name, power limit and clocks are read before and after.  Prints one JSON line.
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
from pydegensac_b200.matching import bundle_adjust_ragged  # noqa: E402
from pydegensac_b200.scenes import _K, _rot  # noqa: E402
from match_batch_rate import card, emit, med  # noqa: E402
from pose_ragged_rate import event_ms  # noqa: E402

N_HELD, MAX_ITERS = 16, 50


def expmap(w):
    a = np.linalg.norm(w)
    W = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    if a == 0.0:
        return np.eye(3)
    return np.eye(3) + np.sin(a) / a * W + 2.0 * (np.sin(0.5 * a) / a) ** 2 * W @ W


def synth(T, C, sigma, seed=0):
    """cams [obs] int32, pts [obs,2], planted (R, t, X), start (R, t, X), offsets [T+1]"""
    rng = np.random.default_rng(seed)
    R = np.stack([_rot("y", rng.uniform(-0.1, 0.1)) @ _rot("x", rng.uniform(-0.05, 0.05)) for _ in range(C)])
    centres = np.c_[0.1 * np.arange(C) - 0.05 * C, rng.uniform(-0.1, 0.1, C), rng.uniform(-0.1, 0.1, C)]
    t = -np.einsum("cij,cj->ci", R, centres)
    L = np.minimum(1 + rng.geometric(0.2, T), 20)
    off = np.r_[0, np.cumsum(L)].astype(np.int64)
    obs = int(off[-1])
    start = rng.integers(0, C, T)
    trk = np.repeat(np.arange(T), L)
    cams = (start[trk] + np.arange(obs) - off[trk]) % C
    mid = centres[(start + (L - 1) // 2) % C, 0]
    X = np.c_[mid + rng.uniform(-3, 3, T), rng.uniform(-2, 2, T), rng.uniform(4, 12, T)]
    q = (np.einsum("oij,oj->oi", R[cams], X[trk]) + t[cams]) @ _K.T
    pts = q[:, :2] / q[:, 2:] + sigma * rng.normal(size=(obs, 2))
    R0, t0 = R.copy(), t.copy()
    for c in range(N_HELD, C):
        R0[c] = expmap(2e-3 * rng.normal(size=3)) @ R[c]
        t0[c] = t[c] + 1e-2 * rng.normal(size=3)
    X0 = X + 2e-2 * rng.normal(size=X.shape)
    return cams.astype(np.int32), pts, (R, t, X), (R0, t0, X0), off.astype(np.int32)


def rot_err(Ra, Rb):
    c = (np.einsum("cij,cij->c", Ra, Rb) - 1) / 2
    return np.arccos(np.clip(c, -1, 1))


def errors(R, X, truth, free):
    e = rot_err(R[free], truth[0][free])
    return {"rotation_max_rad": float(e.max()), "rotation_median_rad": float(np.median(e)),
            "point_median": float(np.median(np.linalg.norm(X - truth[2], axis=1)))}


def scipy_subset(cams, pts, start, off, n, free, max_nfev):
    """least_squares(trf, jac_sparsity) on the free cameras and the first n tracks; returns wall time, cost0, cost"""
    from scipy.optimize import least_squares
    from scipy.sparse import lil_matrix
    R0, t0, X0 = start
    m = int(off[n])
    c, x = cams[:m], pts[:m]
    trk = np.repeat(np.arange(n), np.diff(off[:n + 1]))
    slot = np.full(len(R0), -1)
    slot[free] = np.arange(len(free))
    nc = 6 * len(free)

    def poses(v):
        R, t = R0.copy(), t0.copy()
        for q, k in enumerate(free):
            R[k] = expmap(v[6 * q:6 * q + 3]) @ R0[k]
            t[k] = t0[k] + v[6 * q + 3:6 * q + 6]
        return R, t

    def fun(v):
        R, t = poses(v)
        X = X0[:n] + v[nc:].reshape(n, 3)
        p = np.einsum("oij,oj->oi", R[c], X[trk]) + t[c]
        q = p @ _K.T
        return (q[:, :2] / q[:, 2:] - x).ravel()

    S = lil_matrix((2 * m, nc + 3 * n), dtype=int)
    for i in range(m):
        for r in (2 * i, 2 * i + 1):
            if slot[c[i]] >= 0:
                S[r, 6 * slot[c[i]]:6 * slot[c[i]] + 6] = 1
            S[r, nc + 3 * trk[i]:nc + 3 * trk[i] + 3] = 1
    v0 = np.zeros(nc + 3 * n)
    s = time.perf_counter()
    sol = least_squares(fun, v0, jac_sparsity=S, method="trf", x_scale="jac", max_nfev=max_nfev, xtol=1e-12,
                        ftol=1e-12)
    wall = time.perf_counter() - s
    return {"what": "scipy.optimize.least_squares(trf, jac_sparsity, 2-point) on one CPU process: the %d free cameras "
                    "and the first %d tracks (%d observations), max_nfev %d" % (len(free), n, m, max_nfev),
            "wall_s": wall, "nfev": int(sol.nfev), "cost0": float((fun(v0) ** 2).sum()),
            "cost": float(2 * sol.cost)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tracks", type=int, default=100000)
    ap.add_argument("--cameras", type=int, default=80)
    ap.add_argument("--sigma", type=float, default=0.5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--cpu-tracks", type=int, default=5000, help="tracks in the scipy comparison (0: none)")
    ap.add_argument("--cpu-nfev", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    T, C = args.tracks, args.cameras
    cams, pts, truth, start, off = synth(T, C, args.sigma)
    free = list(range(N_HELD, C))
    d = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (cams, pts, start[0], start[1], _K, off, start[2])]
    res = {"workload": "%d tracks (%d observations, mean length %.2f) over %d cameras on a line, %d held and %d free; "
                       "%.1f px noise; start: free cameras rotated ~2e-3 rad and moved ~1e-2, points moved ~2e-2; "
                       "squared error, max_iters %d"
                       % (T, int(off[-1]), float(np.diff(off).mean()), C, N_HELD, len(free), args.sigma, MAX_ITERS),
           "card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call"}

    def call():
        return bundle_adjust_ragged(*d, free=free, scale_gauge=None, max_iters=MAX_ITERS)

    event_ms(call)
    times = []
    for _ in range(args.rounds):
        ms, out = event_ms(call)
        times.append(ms)
    iters = int(out.iters[0])
    res["call_ms"] = med(times)
    res["all_ms"] = times
    res["trial_steps"] = iters
    res["ms_per_trial_step"] = med(times) / max(iters, 1)
    res["n_used"] = int(out.n_used[0])
    res["cost0"], res["cost"] = float(out.cost0[0]), float(out.cost[0])
    res["error_before"] = errors(start[0], start[2], truth, free)
    res["error_after"] = errors(out.R.cpu().numpy(), out.X.cpu().numpy(), truth, free)
    if args.cpu_tracks > 0:
        res["scipy_subset"] = scipy_subset(cams, pts, start, off, min(args.cpu_tracks, T), free, args.cpu_nfev)
        n = min(args.cpu_tracks, T)
        ds = [torch.from_numpy(np.ascontiguousarray(a)).to(dev)
              for a in (cams[:off[n]], pts[:off[n]], start[0], start[1], _K, off[:n + 1], start[2][:n])]
        ms, sub = event_ms(lambda: bundle_adjust_ragged(*ds, free=free, scale_gauge=None, max_iters=MAX_ITERS))
        res["gpu_subset"] = {"what": "bundle_adjust_ragged on the same subset", "call_ms": ms,
                             "trial_steps": int(sub.iters[0]), "cost0": float(sub.cost0[0]), "cost": float(sub.cost[0])}
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
