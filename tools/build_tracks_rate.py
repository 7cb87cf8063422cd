#!/usr/bin/env python
"""Rate of build_tracks_ragged on one GPU, with scipy's connected components plus the numpy ordering on the CPU beside.

    python tools/build_tracks_rate.py [--images 1000] [--keypoints 8000] [--neighbours 20] [--rows 600] [--out FILE]

Workload (seeded): I images of n keypoints each.  Image i sees the scene points i * S .. i * S + n - 1 (S = n /
neighbours, so a point is seen by `neighbours` consecutive images), each at a keypoint of a per-image permutation.
Image i is paired with images i + 1 .. i + neighbours (when they exist); a pair's verified rows are up to --rows of the
points both images see, drawn at random, of which --wrong (0.5 %) join a random wrong keypoint instead: these merge
tracks into conflicting components.  Every row is in the mask.  Defaults: 1000 x 8000 = 8.0 M keypoints, 18 810 pairs,
11.1 M rows.  One build_tracks_ragged call over the whole batch (keypoint pixels copied), timed with CUDA events after
one warm-up call, median of --rounds (and the same without the keypoints, which leaves out the wrapper's gather of
1000 keypoint tensors into one bank); then a torch.profiler run of --rounds calls splits the device time between the
union phase (init, hook, compress kernels) and the ordering phase (the scans, scatter, rank, write and finish
kernels).  The output is compared byte for byte with the numpy oracle (tests/tracks_np.py), whose connected
components (scipy.sparse.csgraph) and ordering are timed on the CPU (one core), labelled as that.  The card's name,
power limit and clocks are read before and after.  Prints one JSON line.
"""
import argparse
import os
import re
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from pydegensac_b200.matching import build_tracks_ragged  # noqa: E402
from tests import tracks_np  # noqa: E402
from match_batch_rate import card, emit, med  # noqa: E402
from pose_ragged_rate import event_ms  # noqa: E402

UNION_KERNELS = ("tk_init_kernel", "tk_hook_kernel", "tk_compress_kernel")


def synth(I, n, nb, rows, wrong, seed=0):
    """pairs [P,2], idx1, idx2 [R] int32, offsets [P+1] int32, keypoint pixels [I*n, 2]"""
    rng = np.random.default_rng(seed)
    S = n // nb
    perm = np.stack([rng.permutation(n) for _ in range(I)]).astype(np.int32)   # perm[i][u - i S]: keypoint of point u
    pairs, i1, i2 = [], [], []
    for i in range(I):
        for d in range(1, nb + 1):
            j = i + d
            if j >= I:
                break
            common = n - d * S                        # points j S .. i S + n - 1
            if common <= 0:
                continue
            u = j * S + rng.choice(common, min(rows, common), replace=False)
            a, b = perm[i][u - i * S], perm[j][u - j * S]
            bad = rng.random(len(u)) < wrong
            b = np.where(bad, rng.integers(0, n, len(u)), b)
            pairs.append((i, j)); i1.append(a); i2.append(b.astype(np.int32))
    off = np.r_[0, np.cumsum([len(a) for a in i1])].astype(np.int32)
    kp = rng.uniform(0, 640, (I * n, 2))
    return np.array(pairs, np.int32), np.concatenate(i1), np.concatenate(i2), off, kp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=1000)
    ap.add_argument("--keypoints", type=int, default=8000)
    ap.add_argument("--neighbours", type=int, default=20)
    ap.add_argument("--rows", type=int, default=600)
    ap.add_argument("--wrong", type=float, default=0.005)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("build_tracks_rate: no CUDA device (this measurement runs on the GPU only)")
    dev = torch.device("cuda:0")
    I, n = args.images, args.keypoints
    pairs, i1, i2, off, kp = synth(I, n, args.neighbours, args.rows, args.wrong)
    counts = [n] * I
    d1, d2, doff = (torch.from_numpy(x).to(dev) for x in (i1, i2, off))
    kps = [k for k in torch.from_numpy(kp).to(dev).view(I, n, 2)]
    before = card()

    def call():
        return build_tracks_ragged(counts, pairs, d1, d2, doff, None, kps=kps)
    call()
    torch.cuda.synchronize()
    ms = [event_ms(call)[0] for _ in range(args.rounds)]
    ms_nokp = [event_ms(lambda: build_tracks_ragged(counts, pairs, d1, d2, doff, None))[0] for _ in range(args.rounds)]
    ts = call()
    got = {k: (None if v is None else v.cpu().numpy()) for k, v in ts._asdict().items()}
    # the kernels' device time by phase
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.rounds):
            call()
        torch.cuda.synchronize()
    union = order = 0.0
    per_kernel = {}
    for ev in prof.key_averages():
        if not re.search(r"tk_\w+?_kernel", ev.key):
            continue
        t = ev.device_time_total / 1000.0 / args.rounds if hasattr(ev, "device_time_total") else \
            ev.cuda_time_total / 1000.0 / args.rounds
        name = re.search(r"tk_\w+?_kernel", ev.key).group(0)
        per_kernel[name] = per_kernel.get(name, 0.0) + t
        if name in UNION_KERNELS:
            union += t
        else:
            order += t
    after = card()
    # the CPU oracle: the edges once, then components (scipy) and ordering (numpy) timed
    a, b = tracks_np.edges(counts, pairs, i1, i2, off)
    t0 = time.perf_counter()
    roots = tracks_np.component_roots(I * n, a, b)
    t1 = time.perf_counter()
    ref = tracks_np.tracks_from_roots(counts, roots, 2, kp)
    t2 = time.perf_counter()
    same = all(np.array_equal(got[k], ref[k]) for k in ("offsets", "cams", "kp", "track_of", "stats")) and \
        np.array_equal(got["pts"].view(np.uint64), ref["pts"].view(np.uint64))
    s = [int(v) for v in got["stats"]]
    res = {
        "tool": "build_tracks_rate", "card_before": before, "card_after": after,
        "images": I, "keypoints": I * n, "pairs": len(pairs), "rows": int(off[-1]), "edges": int(len(a)),
        "ms_per_call_median": med(ms), "ms_per_call": [round(x, 3) for x in ms],
        "ms_per_call_without_kps_median": med(ms_nokp),
        "device_ms_all_kernels": round(union + order, 3),
        "device_ms_union_phase": round(union, 3), "device_ms_ordering_phase": round(order, 3),
        "device_ms_per_kernel": {k: round(v, 3) for k, v in sorted(per_kernel.items())},
        "stats": {"tracks": s[0], "observations": s[1], "conflicting_components": s[2], "keypoints_in_them": s[3]},
        "equals_numpy_oracle_bytes": bool(same),
        "cpu_one_core_scipy_connected_components_ms": round(1000 * (t1 - t0), 1),
        "cpu_one_core_numpy_ordering_ms": round(1000 * (t2 - t1), 1),
    }
    emit(res, args.out)


if __name__ == "__main__":
    main()
