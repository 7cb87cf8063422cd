#!/usr/bin/env python
"""Rate and accuracy of average_rotations on one GPU, beside the numpy/scipy oracle on one CPU core.

    python tools/rotation_averaging_rate.py [--views 10000] [--edges 200000] [--rounds 5] [--out FILE]

Workload (seeded, synth below): --views views with random rotations, a path (v, v + 1) plus random long-range pairs up
to --edges edges, 1 deg of noise per axis on every relative rotation, 20 % of all edges (taken from the long-range
ones) replaced by random rotations; weights like a pose's support, 100-999 for an inlier edge and 10-99 for an outlier.
Default controls.  Reported: the call time (CUDA events around each call after one warm-up call, median of --rounds),
its split into the spanning-tree start and the IRLS by torch.profiler in a run of its own, the iterations and CG
iterations, the rotation errors of the start and of the result against the planted rotations (gauge aligned at view
0), and the oracle (tests/rotation_averaging_np.py) on the same graph pinned to one CPU core, with its largest
difference from the device.  The card's name, power limit and clocks are read before and after.  Prints one JSON line.
"""
import os

for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
    os.environ[_v] = "1"                          # the oracle on one core (set before numpy loads)
import argparse  # noqa: E402
import sys  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

TREE_KERNELS = ("ra_edges_kernel", "ra_views_kernel", "ra_count_kernel", "ra_scan_kernel", "ra_scatter_kernel",
                "ra_min_edge_kernel", "ra_hook_kernel", "ra_compress_kernel", "ra_tree_kernel")
IRLS_KERNELS = ("ra_residual_kernel", "ra_rhs_kernel", "ra_solve_kernel", "ra_decide_kernel")


def synth(n, P, seed, noise_deg=1.0, outlier_share=0.2):
    """(pairs int32 [P,2], R_rel [P,3,3], weights int32 [P], R_true [n,3,3]) of the workload above"""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    R = Rotation.random(n, random_state=rng).as_matrix()
    m = P - (n - 1)
    i = rng.integers(0, n, m)
    j = (i + rng.integers(1, n, m)) % n
    pairs = np.r_[np.c_[np.arange(n - 1), np.arange(1, n)], np.c_[i, j]].astype(np.int32)
    Re = np.einsum("pij,pkj->pik", R[pairs[:, 1]], R[pairs[:, 0]])
    Re = Rotation.from_rotvec(np.radians(noise_deg) * rng.normal(size=(P, 3))).as_matrix() @ Re
    bad = np.zeros(P, bool)
    bad[n - 1 + rng.choice(m, int(outlier_share * P), replace=False)] = True
    Re[bad] = Rotation.random(int(bad.sum()), random_state=rng).as_matrix()
    w = np.where(bad, rng.integers(10, 100, P), rng.integers(100, 1000, P)).astype(np.int32)
    return pairs, Re, w, R


def errors_deg(Rest, Rtrue):
    """median and largest angle in degrees between the estimated and planted rotations, gauge aligned at view 0"""
    from scipy.spatial.transform import Rotation
    G = Rest[0].T @ Rtrue[0]
    e = np.degrees(np.linalg.norm(Rotation.from_matrix((Rest @ G) @ np.swapaxes(Rtrue, 1, 2)).as_rotvec(), axis=1))
    return {"median_deg": float(np.median(e)), "max_deg": float(e.max())}


def split_ms(call):
    """device time of the start's kernels and of the IRLS kernels in one call, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    tree = irls = 0.0
    for e in prof.key_averages():
        if any(k in e.key for k in TREE_KERNELS):
            tree += e.device_time_total
        elif any(k in e.key for k in IRLS_KERNELS):
            irls += e.device_time_total
    return tree / 1000.0, irls / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=10000)
    ap.add_argument("--edges", type=int, default=200000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from match_batch_rate import card, emit, med
    from pose_ragged_rate import event_ms
    from pydegensac_b200.matching import average_rotations
    from tests import rotation_averaging_np as ra
    dev = torch.device("cuda:0")
    res = {"card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call"}
    n, P = args.views, args.edges
    pairs, Re, w, Rt = synth(n, P, 0)
    dR, dw = torch.from_numpy(Re).to(dev), torch.from_numpy(w).to(dev)
    res["workload"] = ("%d views, %d edges (a path and %d random pairs), 1 deg noise per axis, %d outlier edges (20 %%), "
                       "support weights; default controls" % (n, P, P - n + 1, int(0.2 * P)))

    def call(**kw):
        return average_rotations(pairs, dR, n, weights=dw, **kw)
    event_ms(call)
    times = []
    for _ in range(args.rounds):
        ms, out = event_ms(call)
        times.append(ms)
    _, start = event_ms(lambda: call(l1_iters=0, max_iters=0))
    tree_ms, irls_ms = split_ms(call)
    Rg = out.R.cpu().numpy()
    gpu = {"call_ms": med(times), "all_ms": times, "profiler_tree_ms": tree_ms, "profiler_irls_ms": irls_ms,
           "iters": out.iters.cpu().tolist(), "cg_iters": int(out.cg_iters[0]),
           "start_error": errors_deg(start.R.cpu().numpy(), Rt), "error": errors_deg(Rg, Rt),
           "outlier_edges_above_5deg": int((out.residual.cpu().numpy() > np.radians(5.0)).sum())}
    res["gpu"] = gpu
    if not args.no_oracle:
        try:
            os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})
        except (AttributeError, OSError):
            pass
        t0 = time.perf_counter()
        o = ra.average_rotations(pairs, Re, n, weights=w)
        res["oracle_one_cpu_core"] = {
            "what": "tests/rotation_averaging_np.py (numpy/scipy) on one CPU core of the GPU host, same graph and "
                    "controls", "seconds": time.perf_counter() - t0, "iters": o["iters"].tolist(),
            "cg_iters": int(o["cg_iters"]), "error": errors_deg(o["R"], Rt),
            "largest_abs_difference_from_gpu_R": float(np.abs(o["R"] - Rg).max())}
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
