#!/usr/bin/env python
"""Rate and accuracy of global_positioning_ragged on one GPU, and its share of the global pipeline's device time.

    python tools/global_positioning_rate.py [--views 50,200,2000] [--tracks-per-view 500] [--rounds 3] [--out FILE]

Workload (seeded, synth below), for each size in --views: that many views along the x axis 0.3 apart with a few
degrees of rotation each, looking at --tracks-per-view points per view 4 to 6 ahead; each track is seen by 2 to 6
consecutive views, 0.5 px of pixel noise, and 2 % of the observations replaced by random pixels.  The planted rotations
go in, as rotation averaging would give them.  Default controls.  Reported per size: the call time (CUDA events around
each call after one warm-up call, median of --rounds), its device time by torch.profiler, the trial steps and CG
iterations, and the centre errors against the planted centres after a similarity alignment, after positioning and
after the next stages (triangulate_tracks_ragged on the positioning's inliers, then bundle_adjust_pcg_ragged for at
most 50 trial steps).  At the largest size, for positioning's share of the pipeline's device time: average_rotations
on the view graph of the same views (each view paired with its next 4, planted relative rotations with 1 deg of noise)
beside the positioning and the bundle adjustment.  The card's name, power limit and clocks are read before and after.
Prints one JSON line.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

K0 = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])


def synth(n, T, seed, noise_px=0.5, outliers=0.02):
    """(cams int32 [obs], pts [obs,2], R [n,3,3], offsets int32 [T+1], centres [n,3]) of the workload above"""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    R = Rotation.from_rotvec(np.radians(3.0) * rng.normal(size=(n, 3))).as_matrix()
    Cw = np.c_[0.3 * np.arange(n), 0.05 * rng.normal(size=(n, 2))]
    length = rng.integers(2, 7, T)
    first = rng.integers(0, n - 1, T)
    length = np.minimum(length, n - first)
    offsets = np.r_[0, np.cumsum(length)].astype(np.int32)
    X = np.c_[0.3 * (first + 0.5 * (length - 1)) + rng.uniform(-1.0, 1.0, T), rng.uniform(-1.0, 1.0, T),
              rng.uniform(4.0, 6.0, T)]
    trk = np.repeat(np.arange(T), length)
    cams = (first[trk] + np.arange(len(trk)) - offsets[trk]).astype(np.int32)
    p = np.einsum("ij,nj->ni", K0, np.einsum("nij,nj->ni", R[cams], X[trk] - Cw[cams]))
    pts = p[:, :2] / p[:, 2:] + noise_px * rng.normal(size=(len(trk), 2))
    bad = rng.random(len(trk)) < outliers
    pts[bad] = rng.uniform(0.0, 640.0, (int(bad.sum()), 2))
    return cams, pts, R, offsets, Cw


def align(est, ref):
    """The similarity s Q est + t closest to ref (Umeyama), applied to est"""
    me, mr = est.mean(0), ref.mean(0)
    A, B = est - me, ref - mr
    U, S, Vt = np.linalg.svd(B.T @ A)
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    Q = U @ D @ Vt
    s = np.trace(np.diag(S) @ D) / np.sum(A * A)
    return (s * (Q @ A.T)).T + mr


def centre_errors(R, t, Cw):
    """median and largest distance of the centres -R^T t from the planted ones after a similarity alignment"""
    Ce = -np.einsum("cji,cj->ci", R, t)
    ok = np.isfinite(Ce).all(1)
    e = np.linalg.norm(align(Ce[ok], Cw[ok]) - Cw[ok], axis=1)
    return {"median": float(np.median(e)), "max": float(e.max()), "baseline": 0.3}


def device_ms(call):
    """device time of one call's kernels and copies, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    return sum(e.self_device_time_total for e in prof.key_averages()) / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", default="50,200,2000")
    ap.add_argument("--tracks-per-view", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from scipy.spatial.transform import Rotation
    from match_batch_rate import card, emit, med
    from pose_ragged_rate import event_ms
    from pydegensac_b200.matching import (average_rotations, bundle_adjust_pcg_ragged, global_positioning_ragged,
                                          triangulate_tracks_ragged)
    dev = torch.device("cuda:0")
    res = {"card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call",
           "sizes": []}
    G = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    for n in (int(v) for v in args.views.split(",")):
        T = n * args.tracks_per_view
        cams, pts, R, offsets, Cw = synth(n, T, 0)
        dc, dp, dR, dK, do = G(cams), G(pts), G(R), G(K0), G(offsets)

        def call():
            return global_positioning_ragged(dc, dp, dR, dK, do)
        event_ms(call)
        times = []
        for _ in range(args.rounds):
            ms, out = event_ms(call)
            times.append(ms)
        gp_dev = device_ms(call)
        tr = triangulate_tracks_ragged(dc, dp, dR, out.t, dK, do, mask=out.inliers, px_th=3.0)

        def adjust():
            return bundle_adjust_pcg_ragged(dc, dp, dR, out.t, dK, do, tr.X, mask=tr.mask, loss_scale=1.0)
        ba = adjust()
        row = {"workload": "%d views on a line 0.3 apart, %d tracks over 2-6 consecutive views (%d observations), "
                           "0.5 px noise, 2 %% random pixels; planted rotations; default controls" % (n, T, len(cams)),
               "call_ms": med(times), "all_ms": times, "device_ms": gp_dev, "iters": int(out.iters[0]),
               "cg_iters": int(out.cg_iters[0]), "inlier_share": float(out.inliers.float().mean()),
               "cost0": float(out.cost0[0]), "cost": float(out.cost[0]),
               "centre_error_positioned": centre_errors(R, out.t.cpu().numpy(), Cw),
               "ba_iters": int(ba.iters[0]), "ba_cg_iters": int(ba.cg_iters[0]),
               "centre_error_after_triangulation_and_ba": centre_errors(ba.R.cpu().numpy(), ba.t.cpu().numpy(), Cw)}
        res["sizes"].append(row)
    # the stages either side at the largest size: rotation averaging on the view graph, bundle adjustment after
    pairs = np.array([(i, i + k) for i in range(n) for k in range(1, 5) if i + k < n], np.int32)
    rng = np.random.default_rng(1)
    Re = np.einsum("pij,pkj->pik", R[pairs[:, 1]], R[pairs[:, 0]])
    Re = Rotation.from_rotvec(np.radians(1.0) * rng.normal(size=(len(pairs), 3))).as_matrix() @ Re
    dRe = G(Re)
    ra_dev = device_ms(lambda: average_rotations(pairs, dRe, n))
    ba_dev = device_ms(adjust)
    total = ra_dev + gp_dev + ba_dev
    res["pipeline_device_ms"] = {"views": n, "average_rotations": ra_dev, "global_positioning": gp_dev,
                                 "bundle_adjust_pcg": ba_dev, "positioning_share": gp_dev / total,
                                 "what": "torch.profiler device time of one call each at the largest size; the BA "
                                         "(at most 50 trial steps) starts from the points triangulated on the "
                                         "positioning's inliers"}
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
