#!/usr/bin/env python
"""Rate of bundle_adjust_intrinsics_ragged on one GPU, beside bundle_adjust_pcg_ragged on the same scene.

    python tools/bundle_adjust_intrinsics_rate.py [--cameras 2000] [--tracks 400000] [--rounds 2] [--out FILE]

The scene of tools/bundle_adjust_pcg_rate.py (tools/bundle_adjust_rate.synth: cameras on a line, tracks over
consecutive cameras, 0.5 px noise, cameras 16.. perturbed; tracks that wrap around masked out), cameras 16.. free,
squared error, max_iters 50, cg_tol 0.1, through three calls alternated in one process:
  pose_only      bundle_adjust_pcg_ragged with the scene's K;
  one_group      bundle_adjust_intrinsics_ragged, every camera in one group (f, cx, cy of K, k1 = k2 = 0), f and
                 (k1, k2) refined;
  group_per_cam  the same with one group per camera.
For each: the call time (CUDA events, one warm-up call, median of --rounds), the trial steps and CG iterations, the
time per trial step (call time over trial steps), and the time of the PCG kernel per CG iteration from torch.profiler
in a run of its own.  The card's name, power limit and clocks are read before and after.  Prints one JSON line.
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from pydegensac_b200.matching import bundle_adjust_intrinsics_ragged, bundle_adjust_pcg_ragged  # noqa: E402
from pydegensac_b200.scenes import _K  # noqa: E402
from bundle_adjust_rate import N_HELD, synth  # noqa: E402
from match_batch_rate import card, emit, med  # noqa: E402
from pose_ragged_rate import event_ms  # noqa: E402

MAX_ITERS = 50


def kernel_ms(call, name):
    """total device time of the kernels whose name contains `name` in one call, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = call()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if name in e.key)
    return us / 1000.0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, default=2000)
    ap.add_argument("--tracks", type=int, default=400000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call"}
    C, T = args.cameras, args.tracks
    cams, pts, truth, start, off = synth(T, C, 0.5)
    free = list(range(N_HELD, C))
    L = np.diff(off)
    keep = np.repeat(cams[off[:-1]] + L <= C, L)
    K = np.asarray(_K, np.float64)
    k1 = np.array([[K[0, 0], K[0, 2], K[1, 2], 0.0, 0.0]])
    d = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (cams, pts, start[0], start[1], K, off, start[2])]
    dm = torch.from_numpy(keep).to(dev)
    g1, k_1 = torch.zeros(C, dtype=torch.int32, device=dev), torch.from_numpy(k1).to(dev)
    gC, k_C = torch.arange(C, dtype=torch.int32, device=dev), torch.from_numpy(np.repeat(k1, C, 0)).to(dev)
    base = dict(mask=dm, free=free, scale_gauge=None, max_iters=MAX_ITERS)
    calls = {
        "pose_only": (lambda: bundle_adjust_pcg_ragged(*d, **base), "pcg_solve_kernel"),
        "one_group": (lambda: bundle_adjust_intrinsics_ragged(d[0], d[1], d[2], d[3], g1, k_1, d[5], d[6], **base),
                      "bai_solve_kernel"),
        "group_per_camera": (lambda: bundle_adjust_intrinsics_ragged(d[0], d[1], d[2], d[3], gC, k_C, d[5], d[6],
                                                                     **base), "bai_solve_kernel"),
    }
    res["workload"] = ("%d tracks (%d observations, %d in tracks that do not wrap around) over %d cameras on a line, "
                       "%d held and %d free; 0.5 px noise; squared error, max_iters %d, cg_tol 0.1; intrinsics: f and "
                       "(k1, k2) refined" % (T, int(off[-1]), int(keep.sum()), C, N_HELD, len(free), MAX_ITERS))
    times = {k: [] for k in calls}
    outs = {}
    for k, (call, _) in calls.items():
        event_ms(call)
    for _ in range(args.rounds):
        for k, (call, _) in calls.items():
            ms, outs[k] = event_ms(call)
            times[k].append(ms)
    for k, (call, kernel) in calls.items():
        sms, _ = kernel_ms(call, kernel)
        o = outs[k]
        steps, cg = int(o.iters[0]), int(o.cg_iters[0])
        r = {"call_ms": med(times[k]), "all_ms": times[k], "trial_steps": steps, "cg_iters": cg,
             "ms_per_trial_step": med(times[k]) / max(steps, 1), "solve_kernel_ms": sms,
             "ms_per_cg_iteration": sms / max(cg, 1), "cost0": float(o.cost0[0]), "cost": float(o.cost[0]),
             "n_used": int(o.n_used[0])}
        if hasattr(o, "intrinsics"):
            kk = o.intrinsics.cpu().numpy()
            r["f_range"] = [float(kk[:, 0].min()), float(kk[:, 0].max())]
        res[k] = r
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
