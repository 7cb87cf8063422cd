#!/usr/bin/env python
"""Rate of pose_from_homography_ragged on one GPU, against the ragged H RANSAC on the same batch, with
pose_from_fundamental_ragged re-timed in the same run.

    python tools/pose_homography_rate.py [--pairs 512] [--rounds 5] [--out FILE]

Workload: P = 512 synthetic planar two-view pairs of 500 to 3000 correspondences each (uniform, seeded): views of random
points on a random plane with 0.3 px noise for 70 % of the rows and random pixels for the rest; the mask given to the
pose steps is the planted inlier flag, H the planted homography and F the planted fundamental matrix (the F path's
workload of tools/pose_ragged_rate.py, same sizes).  Timed with CUDA events after one warm-up call of each path,
alternating the paths in every round:
  pose_h   one pose_from_homography_ragged call over the whole batch (candidates, vote, rows, median)
  pose_f   one pose_from_fundamental_ragged call over the F workload
  ransac   findHomographyBatch(..., offsets=, n_max=) on the planar batch (px_th 2, conf 0.999, 10000 iterations), the
           step before pose in the H branch, for the share pose takes
With --parent-lib, the pose_from_fundamental_ragged entry point of that build and of this one are also timed as two
raw C ABI calls on the same buffers, alternating with the rest, and their outputs compared byte for byte.
The card's name, power limit and clocks are read before and after.  Prints one JSON line.
"""
import argparse
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import pydegensac_b200 as pdg  # noqa: E402
from pydegensac_b200 import _cabi  # noqa: E402
from pydegensac_b200.matching import pose_from_fundamental_ragged, pose_from_homography_ragged  # noqa: E402
from pydegensac_b200.scenes import _K, _rot  # noqa: E402
from match_batch_rate import card, emit, med  # noqa: E402
from pose_ragged_rate import event_ms, synth  # noqa: E402


def synth_planar(P, lo, hi, inlier_frac, seed=0):
    rng = np.random.default_rng(seed)
    Ki = np.linalg.inv(_K)
    ps1, ps2, ms, Hs, lengths = [], [], [], [], []
    for p in range(P):
        n = int(rng.integers(lo, hi + 1))
        R = _rot("y", rng.uniform(-0.3, 0.3)) @ _rot("x", rng.uniform(-0.1, 0.1))
        t = np.array([rng.uniform(0.5, 1.5), rng.uniform(-0.2, 0.2), rng.uniform(-0.3, 0.3)])
        nrm = np.array([rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), 1.0])
        nrm /= np.linalg.norm(nrm)
        d = rng.uniform(4, 10)
        xy = np.c_[rng.uniform(-2, 2, n), rng.uniform(-2, 2, n)]
        X = np.c_[xy, (d - xy @ nrm[:2]) / nrm[2]]
        x1 = X @ _K.T
        x2 = (X @ R.T + t) @ _K.T
        p1 = x1[:, :2] / x1[:, 2:3] + 0.3 * rng.normal(size=(n, 2))
        p2 = x2[:, :2] / x2[:, 2:3] + 0.3 * rng.normal(size=(n, 2))
        inl = rng.random(n) < inlier_frac
        p2[~inl] = rng.uniform(0, 640, (int((~inl).sum()), 2))
        ps1.append(p1); ps2.append(p2); ms.append(inl); Hs.append(_K @ (R + np.outer(t, nrm) / d) @ Ki)
        lengths.append(n)
    off = np.r_[0, np.cumsum(lengths)].astype(np.int32)
    return np.concatenate(ps1), np.concatenate(ps2), np.concatenate(ms), np.stack(Hs), off


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--min-rows", type=int, default=500)
    ap.add_argument("--max-rows", type=int, default=3000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--parent-lib", default=None, help="another build of libdegensac_b200.so to time pose from F of")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    P = args.pairs
    p1, p2, mask, H, off = synth_planar(P, args.min_rows, args.max_rows, 0.7)
    f1, f2, fmask, F, foff = synth(P, args.min_rows, args.max_rows, 0.7)
    d1, d2, dm, dH, doff, dK = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (p1, p2, mask, H, off, _K))
    e1, e2, em, dF, eoff = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (f1, f2, fmask, F, foff))
    seeds = torch.arange(P, dtype=torch.int64, device=dev)
    n_max = int(np.diff(off).max())
    res = {"workload": "%d planar pairs, %d to %d rows each (%d in all), %.1f %% masked inliers; H planted; RANSAC "
                       "px_th 2, conf 0.999, 10000 iterations; pose_f on the F workload of pose_ragged_rate.py "
                       "(%d rows)" % (P, args.min_rows, args.max_rows, int(off[-1]), 100.0 * mask.mean(),
                                      int(foff[-1])),
           "card": card(), "rounds": args.rounds, "timing": "CUDA events around each call, after one warm-up call"}

    def pose_h():
        return pose_from_homography_ragged(dH, dK, dK, d1, d2, doff, dm)

    def pose_f():
        return pose_from_fundamental_ragged(dF, dK, dK, e1, e2, eoff, em)

    def ransac():
        return pdg.findHomographyBatch(d1, d2, 2.0, 0.999, 10000, seeds=seeds, offsets=doff, n_max=n_max)

    paths = {"pose_h": pose_h, "pose_f": pose_f, "ransac": ransac}
    if args.parent_lib:
        vp = ctypes.c_void_p
        rows = int(foff[-1])

        def abi(L):
            fn = L.dgb200_pose_from_fundamental_ragged_dev
            fn.argtypes = _cabi.lib().dgb200_pose_from_fundamental_ragged_dev.argtypes
            outs = [torch.empty(s, dtype=d, device=dev) for s, d in (((P, 9), torch.float64), ((P, 3), torch.float64),
                    ((P,), torch.int32), ((rows, 3), torch.float64), ((rows,), torch.uint8), ((rows,), torch.float64),
                    ((P,), torch.float64))]

            def call():
                rc = fn(vp(dF.data_ptr()), vp(dK.data_ptr()), vp(dK.data_ptr()), 0, vp(e1.data_ptr()), vp(e2.data_ptr()),
                        vp(eoff.data_ptr()), P, rows, 2, vp(em.data_ptr()), *[vp(o.data_ptr()) for o in outs],
                        vp(torch.cuda.current_stream(dev).cuda_stream))
                assert rc == 0
                return outs
            return call
        paths["pose_f_abi_this"] = abi(_cabi.lib())
        paths["pose_f_abi_parent"] = abi(ctypes.CDLL(os.path.abspath(args.parent_lib)))
    for fn in paths.values():
        event_ms(fn)
    t = {k: [] for k in paths}
    outs = {}
    for _ in range(args.rounds):
        for k, fn in paths.items():
            ms, outs[k] = event_ms(fn)
            t[k].append(ms)
    for k in paths:
        res[k] = {"ms": med(t[k]), "pairs_per_s": 1e3 * P / med(t[k]), "all_ms": t[k]}
    res["pose_h_share_of_ransac_plus_pose"] = med(t["pose_h"]) / (med(t["pose_h"]) + med(t["ransac"]))
    if args.parent_lib:
        res["parent_lib"] = args.parent_lib
        res["pose_f_abi_bytes_equal"] = all(torch.equal(a.view(torch.uint8), b.view(torch.uint8))
                                            for a, b in zip(outs["pose_f_abi_this"], outs["pose_f_abi_parent"]))
    g = outs["pose_h"]
    res["rotation_only_pairs"] = int(g.rotation_only.sum().item())
    res["good0_sum"] = int(g.good[:, 0].sum().item())
    res["good1_sum"] = int(g.good[:, 1].sum().item())
    res["median_angle_deg_median"] = float(np.degrees(np.nanmedian(g.median_angle.cpu().numpy())))
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
