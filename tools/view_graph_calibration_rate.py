#!/usr/bin/env python
"""Rate and accuracy of calibrate_view_graph on one GPU, beside the numpy/scipy oracle on one CPU core.

    python tools/view_graph_calibration_rate.py [--views 10000] [--edges 200000] [--rounds 5] [--out FILE]

Workloads (seeded, synth below), run twice: once with one camera group for every view (f = 800) and once with a group
per view (f uniform in [600, 1000]).  --views views on a sphere of radius 4 to 6 around the origin, each looking at a
point near the origin with a random roll; a path (v, v + 1) plus random pairs up to --edges edges; each F the planted
one with 1e-3 relative noise on the entries of its essential matrix, projected to rank 2; 5 % of the edges a
random rank-2 F.  The start is f0 = 0.96 f (768 for 800) with the planted principal point.  Default controls.  Reported: the call time (CUDA events
around each call after one warm-up call, median of --rounds), the trial steps and CG iterations, the relative focal
error at the start and at the result (median and largest over the groups), the inlier count and how many random
edges are among the inliers, and the oracle (tests/view_graph_calibration_np.py) on the same graph pinned to one CPU
core, with its largest theta difference from the device.  The card's name, power limit and clocks are read before and
after.  Prints one JSON line.
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


def synth(n, P, one_group, seed, noise=1e-3, outlier_share=0.05):
    """(pairs int32 [P,2], F [P,3,3], groups int32 [n], k_start [G,5], f_true [G]) of the workload above; the random
    edges are the last ones of the random pairs' draw, marked by F_bad below"""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1)[:, None]
    c = d * rng.uniform(4.0, 6.0, n)[:, None]
    z = rng.uniform(-0.5, 0.5, (n, 3)) - c
    z /= np.linalg.norm(z, axis=1)[:, None]
    up = rng.normal(size=(n, 3))
    x = np.cross(up, z)
    x /= np.linalg.norm(x, axis=1)[:, None]
    y = np.cross(z, x)
    R = np.stack([x, y, z], 1)
    t = -np.einsum("vij,vj->vi", R, c)
    G = 1 if one_group else n
    groups = (np.zeros(n) if one_group else np.arange(n)).astype(np.int32)
    f_true = np.full(G, 800.0) if one_group else rng.uniform(600.0, 1000.0, G)
    k_true = np.c_[f_true, np.full(G, 320.0), np.full(G, 240.0), np.zeros((G, 2))]
    m = P - (n - 1)
    i = rng.integers(0, n, m)
    j = (i + rng.integers(1, n, m)) % n
    pairs = np.r_[np.c_[np.arange(n - 1), np.arange(1, n)], np.c_[i, j]].astype(np.int32)
    pi, pj = pairs[:, 0], pairs[:, 1]
    Rr = np.einsum("pij,pkj->pik", R[pj], R[pi])
    tr = t[pj] - np.einsum("pij,pj->pi", Rr, t[pi])
    tx = np.zeros((P, 3, 3))
    tx[:, 0, 1], tx[:, 0, 2], tx[:, 1, 2] = -tr[:, 2], tr[:, 1], -tr[:, 0]
    tx[:, 1, 0], tx[:, 2, 0], tx[:, 2, 1] = tr[:, 2], -tr[:, 1], tr[:, 0]

    def kinv(k):
        Ki = np.zeros((len(k), 3, 3))
        Ki[:, 0, 0] = Ki[:, 1, 1] = 1.0 / k[:, 0]
        Ki[:, 0, 2], Ki[:, 1, 2], Ki[:, 2, 2] = -k[:, 1] / k[:, 0], -k[:, 2] / k[:, 0], 1.0
        return Ki
    E = np.einsum("pij,pjk->pik", tx, Rr)
    E /= np.linalg.norm(E, axis=(1, 2))[:, None, None]
    bad = np.zeros(P, bool)
    bad[n - 1 + rng.choice(m, int(outlier_share * P), replace=False)] = True
    E[bad] = rng.normal(size=(int(bad.sum()), 3, 3)) / 3.0
    E = E + noise * rng.normal(size=E.shape) / 3.0          # the noise is relative to the calibrated matrix
    U, s, Vt = np.linalg.svd(E)
    s[:, 2] = 0.0
    Ki, Kj = kinv(k_true[groups[pi]]), kinv(k_true[groups[pj]])
    F = np.einsum("pji,pjk,pkl->pil", Kj, np.einsum("pij,pj,pjk->pik", U, s, Vt), Ki)
    k_start = k_true.copy()
    k_start[:, 0] *= 0.96
    synth.F_bad = bad
    return pairs, F, groups, k_start, f_true


def focal_errors(f, f_true):
    e = np.abs(f / f_true - 1.0)
    return {"median": float(np.median(e)), "max": float(e.max())}


def run(dev, n, P, one_group, rounds, oracle):
    import torch
    from pose_ragged_rate import event_ms
    from match_batch_rate import med
    from pydegensac_b200.matching import calibrate_view_graph
    from tests import view_graph_calibration_np as vg
    pairs, F, groups, k0, f_true = synth(n, P, one_group, 0)
    bad = synth.F_bad
    dF, dg, dk = (torch.from_numpy(a).to(dev) for a in (F, groups, k0))

    def call():
        return calibrate_view_graph(pairs, dF, dg, dk)
    event_ms(call)
    times = []
    for _ in range(rounds):
        ms, out = event_ms(call)
        times.append(ms)
    f = out.intrinsics[:, 0].cpu().numpy()
    inl = out.inliers.cpu().numpy()
    res = {"workload": "%d views, %d edges (a path and %d random pairs), %s, 1e-3 relative noise on E, %d random F "
                       "(5 %%), start f0 = 0.96 f; default controls"
                       % (n, P, P - n + 1, "one group (f = 800)" if one_group else "a group per view (f in [600, 1000])",
                          int(bad.sum())),
           "call_ms": med(times), "all_ms": times, "iters": int(out.iters[0]), "cg_iters": int(out.cg_iters[0]),
           "n_used": int(out.n_used[0]), "inliers": int(inl.sum()), "random_edges_among_inliers": int(inl[bad].sum()),
           "refined_groups": int(out.refined.sum()), "start_focal_error": focal_errors(k0[:, 0], f_true),
           "focal_error": focal_errors(f, f_true)}
    if oracle:
        try:
            os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})
        except (AttributeError, OSError):
            pass
        t0 = time.perf_counter()
        o = vg.calibrate_view_graph(pairs, F, groups, k0)
        th = np.log(f / k0[:, 0])
        res["oracle_one_cpu_core"] = {
            "what": "tests/view_graph_calibration_np.py (numpy/scipy) on one CPU core of the GPU host, same graph and "
                    "controls", "seconds": time.perf_counter() - t0, "iters": int(o["iters"]),
            "cg_iters": int(o["cg_iters"]),
            "largest_abs_theta_difference_from_gpu": float(np.abs(np.where(o["refined"], o["theta"], 0.0) - th).max())}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=10000)
    ap.add_argument("--edges", type=int, default=200000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from match_batch_rate import card, emit
    dev = torch.device("cuda:0")
    res = {"card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call"}
    res["one_group"] = run(dev, args.views, args.edges, True, args.rounds, not args.no_oracle)
    res["group_per_view"] = run(dev, args.views, args.edges, False, args.rounds, not args.no_oracle)
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
