#!/usr/bin/env python
"""Rate and accuracy of bundle_adjust_pcg_ragged on one GPU, beside bundle_adjust_ragged and scipy.

    python tools/bundle_adjust_pcg_rate.py [--cameras 2000] [--tracks 400000] [--rounds 3] [--out FILE]

Workloads (seeded, tools/bundle_adjust_rate.synth: cameras on a line, tracks over consecutive cameras, 0.5 px noise,
cameras 16.. rotated by ~2e-3 rad and moved by ~1e-2, points moved by ~2e-2):
  large   --cameras cameras and --tracks tracks, cameras 16.. free, squared error, max_iters 50, at cg_tol 0.1 and
          0.01: call time (CUDA events, one warm-up call, median of --rounds), trial steps, CG iterations, the time
          of pcg_solve_kernel per CG iteration from torch.profiler in a run of its own, the bytes one CG iteration
          reads (from shapes: W twice and the gathers, below) over that time against 3.35 TB/s, and the errors
          against the planted scene before and after;
  dense   the 80-camera, 10^5-track workload of tools/bundle_adjust_rate.py through bundle_adjust_ragged and
          bundle_adjust_pcg_ragged, alternated in one process;
  scipy   least_squares (trf, jac_sparsity) of tools/bundle_adjust_rate.py on the first --cpu-tracks tracks of a
          100-camera scene with 84 free cameras, beside the new call on the same subset.
The card's name, power limit and clocks are read before and after.  Prints one JSON line.
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from pydegensac_b200.matching import bundle_adjust_pcg_ragged, bundle_adjust_ragged  # noqa: E402
from pydegensac_b200.scenes import _K  # noqa: E402
from bundle_adjust_rate import N_HELD, errors, scipy_subset, synth  # noqa: E402
from match_batch_rate import card, emit, med  # noqa: E402
from pose_ragged_rate import event_ms  # noqa: E402

MAX_ITERS = 50
HBM_BPS = 3.35e12


def cg_bytes(cams, T, free):
    """DRAM bytes of one CG iteration, from shapes: per used observation of a free camera W (144 B) and its slot
    (4 B) in the track pass, W (144 B), its track (4 B) and y of the track (24 B) in the camera pass; per track its
    offsets, V*^-1 and y (4 + 4 + 48 + 24 B).  The per-camera vectors stay in L2 and are not counted."""
    n = int(np.isin(cams, free).sum())
    return 320 * n + 80 * T


def solve_ms(call):
    """total time of pcg_solve_kernel in one call, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = call()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "pcg_solve_kernel" in e.key)
    return us / 1000.0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, default=2000)
    ap.add_argument("--tracks", type=int, default=400000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--cpu-tracks", type=int, default=3000)
    ap.add_argument("--cpu-nfev", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call"}
    # large
    C, T = args.cameras, args.tracks
    cams, pts, truth, start, off = synth(T, C, 0.5)
    free = list(range(N_HELD, C))
    # synth's tracks wrap around from the last camera to the first, which at this length joins cameras 200 units
    # apart: those tracks are masked out (not optimised)
    L = np.diff(off)
    keep = np.repeat(cams[off[:-1]] + L <= C, L)
    d = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (cams, pts, start[0], start[1], _K, off, start[2])]
    dm = torch.from_numpy(keep).to(dev)
    large = {"workload": "%d tracks (%d observations, %d in tracks that do not wrap around) over %d cameras on a line, "
                         "%d held and %d free; 0.5 px noise; squared error, max_iters %d"
                         % (T, int(off[-1]), int(keep.sum()), C, N_HELD, len(free), MAX_ITERS),
             "cg_bytes_per_iteration": cg_bytes(cams[keep], int((cams[off[:-1]] + L <= C).sum()), free),
             "error_before": errors(start[0], start[2], truth, free)}
    for tol in (0.1, 0.01):
        def call():
            return bundle_adjust_pcg_ragged(*d, mask=dm, free=free, scale_gauge=None, max_iters=MAX_ITERS, cg_tol=tol)
        event_ms(call)
        times = []
        for _ in range(args.rounds):
            ms, out = event_ms(call)
            times.append(ms)
        sms, _ = solve_ms(call)
        cg = int(out.cg_iters[0])
        r = {"call_ms": med(times), "all_ms": times, "trial_steps": int(out.iters[0]), "cg_iters": cg,
             "cost0": float(out.cost0[0]), "cost": float(out.cost[0]), "n_used": int(out.n_used[0]),
             "solve_kernel_ms": sms, "ms_per_cg_iteration": sms / max(cg, 1),
             "error_after": errors(out.R.cpu().numpy(), out.X.cpu().numpy(), truth, free)}
        r["cg_bytes_per_s"] = large["cg_bytes_per_iteration"] / (r["ms_per_cg_iteration"] * 1e-3)
        r["share_of_3_35_TBps"] = r["cg_bytes_per_s"] / HBM_BPS
        large["cg_tol_%g" % tol] = r
    res["large"] = large
    del d
    # the dense tool's workload through both entry points, alternated
    cams, pts, truth, start, off = synth(100000, 80, 0.5)
    free = list(range(N_HELD, 80))
    d = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (cams, pts, start[0], start[1], _K, off, start[2])]
    calls = {"bundle_adjust_ragged": lambda: bundle_adjust_ragged(*d, free=free, scale_gauge=None, max_iters=MAX_ITERS),
             "bundle_adjust_pcg_ragged": lambda: bundle_adjust_pcg_ragged(*d, free=free, scale_gauge=None,
                                                                          max_iters=MAX_ITERS)}
    times = {k: [] for k in calls}
    outs = {}
    for k in calls:
        event_ms(calls[k])
    for _ in range(args.rounds):
        for k in calls:
            ms, outs[k] = event_ms(calls[k])
            times[k].append(ms)
    res["dense_workload"] = {"workload": "tools/bundle_adjust_rate.py: 10^5 tracks (%d observations), 80 cameras, "
                                         "64 free" % int(off[-1])}
    for k in calls:
        o = outs[k]
        res["dense_workload"][k] = {"call_ms": med(times[k]), "all_ms": times[k], "trial_steps": int(o.iters[0]),
                                    "cost": float(o.cost[0]),
                                    "error_after": errors(o.R.cpu().numpy(), o.X.cpu().numpy(), truth, free)}
    res["dense_workload"]["bundle_adjust_pcg_ragged"]["cg_iters"] = int(outs["bundle_adjust_pcg_ragged"].cg_iters[0])
    del d
    # scipy on a subset with more than 64 free cameras
    if args.cpu_tracks > 0:
        cams, pts, truth, start, off = synth(args.cpu_tracks, 100, 0.5, seed=1)
        free = list(range(N_HELD, 100))
        res["scipy_subset"] = scipy_subset(cams, pts, start, off, args.cpu_tracks, free, args.cpu_nfev)
        ds = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (cams, pts, start[0], start[1], _K, off,
                                                                          start[2])]
        ms, sub = event_ms(lambda: bundle_adjust_pcg_ragged(*ds, free=free, scale_gauge=None, max_iters=MAX_ITERS))
        res["gpu_subset"] = {"what": "bundle_adjust_pcg_ragged on the same subset", "call_ms": ms,
                             "trial_steps": int(sub.iters[0]), "cg_iters": int(sub.cg_iters[0]),
                             "cost0": float(sub.cost0[0]), "cost": float(sub.cost[0])}
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
