#!/usr/bin/env python
"""Rate of the batched descriptor matcher against a Python loop of single-pair calls, on one GPU.

    python tools/match_batch_rate.py [--parent-lib PATH] [--out FILE]

Workload: I = 64 synthetic images of n = 4000 descriptors (D = 128, float32), views of one set of 3-D points whose
descriptors agree up to noise (the planted true matches), plus clutter -- as in examples/gpu_pipeline.py.  P = 512 pairs:
image i against images i+1 .. i+8 (mod 64).  Timed, alternating, on the same inputs:
  loop   a Python loop of matching.match_descriptors over the P pairs (one call per pair, each reads its count back)
  batch  one matching.match_descriptors_batch over the P pairs
  batch+F  the batch followed by findFundamentalMatrixBatch(..., offsets=, n_max=) on its ragged output
and the single-pair call at n1 = n2 = 2000, D = 128 (device time per call from CUDA events over back-to-back calls),
through this build's library and, with --parent-lib, through another build of the same C entry point.
FLOP/s count 2 n1 n2 D per pair (the distance computations) against the H100 SXM data-sheet 67 TFLOP/s (FP32, dense).
The card's name, power limit and clocks are read in the same run.  Prints one JSON line.

    python tools/match_batch_rate.py --norm hamming --bytes 32 61 [--out FILE]

Binary descriptors (ORB: 32 bytes, AKAZE: 61) on the same scenes: the planted matches share a random code with each
bit flipped with probability 0.1 per view, the clutter is random bytes; match_descriptors(..., norm="hamming").  Per
byte count the same loop / batch / batch+F / single-call timings, and for 32 bytes the workaround without a Hamming
matcher: the bits unpacked to float32 (D = 256) through the L2 batch matcher on the same pairs.  Rates count
n1 n2 n_words 32-bit popcounts per pair (n_words = the row padded to 16 bytes, in words) against the POPC issue bound:
16 results per clock per SM (CUDA programming guide, arithmetic instruction throughput, compute capability 9.0) times
the SM count times the SM clock read right after the timed rounds.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pydegensac_b200 as pdg  # noqa: E402
from pydegensac_b200 import _cabi  # noqa: E402
from pydegensac_b200.matching import match_descriptors, match_descriptors_batch  # noqa: E402
from pydegensac_b200.scenes import _K, _rot  # noqa: E402

FP32_PEAK = 67e12   # NVIDIA H100 SXM data sheet, FP32 dense (a card allowed 700 W)


def flip_bits(codes, p, rng):
    bits = np.unpackbits(codes, axis=1)
    return np.packbits(bits ^ (rng.random(bits.shape) < p), axis=1)


def synth_images(n_img, n, D, seed=0, n_true_frac=0.6, binary=False):
    """binary: D-byte uint8 descriptors (shared codes with bits flipped, random clutter) in place of float32 ones"""
    rng = np.random.default_rng(seed)
    n_true = int(n * n_true_frac)
    X = np.c_[rng.uniform(-2, 2, n_true), rng.uniform(-2, 2, n_true), rng.uniform(5, 10, n_true)]
    code = rng.integers(0, 256, (n_true, D), dtype=np.uint8) if binary else rng.normal(size=(n_true, D)).astype(np.float32)
    kps, descs = [], []
    for i in range(n_img):
        R = _rot("y", 0.01 * i) @ _rot("x", 0.003 * i)
        t = np.array([0.05 * i, 0.01 * i, 0.0])
        x = (_K @ (R @ X.T + t[:, None])).T
        kp = np.r_[x[:, :2] / x[:, 2:3] + 0.1 * rng.normal(size=(n_true, 2)), rng.uniform(0, 640, (n - n_true, 2))]
        if binary:
            d = np.r_[flip_bits(code, 0.1, rng), rng.integers(0, 256, (n - n_true, D), dtype=np.uint8)]
        else:
            d = np.r_[code + 0.2 * rng.normal(size=code.shape).astype(np.float32),
                      rng.normal(size=(n - n_true, D)).astype(np.float32)]
        perm = rng.permutation(n)
        kps.append(kp[perm]); descs.append(d[perm])
    return kps, descs


def single_call_ms(L, d1, d2, reps, binary=False):
    """Device time per dgb200_match_descriptors_dev call of library L (CUDA events over `reps` back-to-back calls);
    binary: dgb200_match_binary_descriptors_dev on int32 rows of 32-bit words."""
    n1, D = d1.shape
    n2 = d2.shape[0]
    dev = d1.device
    mq = torch.empty(n1, dtype=torch.int32, device=dev)
    mt = torch.empty(n1, dtype=torch.int32, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    L.dgb200_match_workspace_bytes.restype = ctypes.c_size_t
    L.dgb200_match_workspace_bytes.argtypes = [ctypes.c_int, ctypes.c_int]
    ws = torch.empty(int(L.dgb200_match_workspace_bytes(n1, n2)), dtype=torch.uint8, device=dev)
    vp = ctypes.c_void_p
    ci = ctypes.c_int
    rt = ctypes.c_double if binary else ctypes.c_float
    fn = L.dgb200_match_binary_descriptors_dev if binary else L.dgb200_match_descriptors_dev
    fn.argtypes = [vp, ci, vp, ci, ci, rt, ci, vp, vp, ci, vp, vp, vp, vp, ci, ci, vp, vp, vp]
    st = torch.cuda.current_stream(dev)

    def call():
        rc = fn(vp(d1.data_ptr()), n1, vp(d2.data_ptr()), n2, D, rt(0.9), 1, None, None, 0, vp(mq.data_ptr()),
                vp(mt.data_ptr()), None, None, 0, n1, vp(cnt.data_ptr()), vp(ws.data_ptr()), vp(st.cuda_stream))
        assert rc == 0
    for _ in range(10):
        call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps, int(cnt.item()), mq[:int(cnt.item())].clone()


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the numbers still carry the torch device name
        out = "nvidia-smi unavailable: %s" % e
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": out.splitlines()[0] if out else ""}


def sm_clock_mhz():
    """current and maximum SM clock in MHz (nvidia-smi), or (None, None)"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        cur, mx = (float(x) for x in out.split(","))
        return cur, mx
    except Exception:
        return None, None


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def med(x):
    return float(np.median(x))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--n", type=int, default=4000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--neighbours", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--parent-lib", default=None, help="another build of libdegensac_b200.so to time the single call of")
    ap.add_argument("--norm", choices=("l2", "hamming"), default="l2")
    ap.add_argument("--bytes", type=int, nargs="+", default=[32, 61], help="binary descriptor lengths (--norm hamming)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.norm == "hamming":
        return main_hamming(args)
    dev = torch.device("cuda:0")
    kps, descs = synth_images(args.images, args.n, args.dim)
    dt = [torch.from_numpy(d).to(dev) for d in descs]
    kt = [torch.from_numpy(k).to(dev) for k in kps]
    pairs = np.array([(i, (i + k) % args.images) for i in range(args.images) for k in range(1, args.neighbours + 1)],
                     dtype=np.int32)
    P = len(pairs)
    flop = float(sum(2.0 * dt[q].shape[0] * dt[t].shape[0] * args.dim for q, t in pairs))
    seeds = torch.arange(P, dtype=torch.int64, device=dev)

    def loop():
        return [match_descriptors(dt[q], dt[t], kt[q], kt[t], 0.9, True) for q, t in pairs]

    def batch():
        return match_descriptors_batch(dt, pairs, kt, ratio=0.9, mutual=True)

    def batch_f():
        m = batch()
        return m, pdg.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                                 n_max=m.n_max)

    for fn in (loop, batch, batch_f):   # warm-up: module loads, allocator
        timed(fn)
    t_loop, t_batch, t_bf = [], [], []
    for _ in range(args.rounds):
        a, rl = timed(loop)
        b, rb = timed(batch)
        c, (mb, (F, mask)) = timed(batch_f)
        t_loop.append(a); t_batch.append(b); t_bf.append(c)
    # the two paths agree (bit for bit) on every pair
    off = rb.offsets.cpu().numpy()
    same = all(torch.equal(rb.idx1[off[p]:off[p + 1]], rl[p][0]) and torch.equal(rb.idx2[off[p]:off[p + 1]], rl[p][1])
               for p in range(P))
    matches = int(off[-1])
    inliers = int(mask[:matches].sum().item())
    res = {"workload": "match %d images x %d descriptors (D=%d), %d pairs (each image vs its %d successors), ratio 0.9, "
                       "mutual" % (args.images, args.n, args.dim, P, args.neighbours),
           "card": card(),
           "rounds": args.rounds,
           "loop": {"s": med(t_loop), "pairs_per_s": P / med(t_loop), "tflops": flop / med(t_loop) / 1e12,
                    "all_s": t_loop},
           "batch": {"s": med(t_batch), "pairs_per_s": P / med(t_batch), "tflops": flop / med(t_batch) / 1e12,
                     "frac_fp32_peak": flop / med(t_batch) / FP32_PEAK, "all_s": t_batch},
           "batch_plus_ragged_F": {"s": med(t_bf), "pairs_per_s": P / med(t_bf), "all_s": t_bf,
                                   "F": "px_th 0.5, conf 0.999, max_iters 10000, sampson", "inliers": inliers},
           "speedup_batch_vs_loop": med(t_loop) / med(t_batch),
           "matches": matches, "batch_equals_loop": bool(same),
           "flop_per_batch": flop, "fp32_peak_tflops_datasheet": FP32_PEAK / 1e12}
    # single-pair call, n1 = n2 = 2000
    d1, d2 = dt[0][:2000].contiguous(), dt[1][:2000].contiguous()
    single = {"n1": 2000, "n2": 2000, "D": args.dim, "mutual": True}
    libs = [("this_build", _cabi.lib())]
    if args.parent_lib:
        libs.append(("parent_build", ctypes.CDLL(os.path.abspath(args.parent_lib))))
    times = {k: [] for k, _ in libs}
    outs = {}
    for _ in range(args.rounds):
        for name, L in libs:
            ms, n, q = single_call_ms(L, d1, d2, 200)
            times[name].append(ms)
            outs[name] = (n, q)
    for name, _ in libs:
        single[name + "_ms"] = med(times[name])
        single[name + "_all_ms"] = times[name]
        single[name + "_tflops"] = 2.0 * 2000 * 2000 * args.dim / (med(times[name]) * 1e-3) / 1e12
    if args.parent_lib:
        single["same_matches"] = bool(outs["this_build"][0] == outs["parent_build"][0] and
                                      torch.equal(outs["this_build"][1], outs["parent_build"][1]))
    res["single_call"] = single
    res["card_after"] = card()
    emit(res, args.out)


def emit(res, out):
    line = json.dumps(res)
    print(line)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write(line + "\n")


def main_hamming(args):
    dev = torch.device("cuda:0")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pairs = np.array([(i, (i + k) % args.images) for i in range(args.images) for k in range(1, args.neighbours + 1)],
                     dtype=np.int32)
    P = len(pairs)
    seeds = torch.arange(P, dtype=torch.int64, device=dev)
    res = {"workload": "match %d images x %d binary descriptors, %d pairs (each image vs its %d successors), ratio 0.9, "
                       "mutual, norm hamming" % (args.images, args.n, P, args.neighbours),
           "card": card(), "rounds": args.rounds, "sm_count": sms,
           "popc_bound": "16 POPC results / clock / SM (CUDA programming guide, compute capability 9.0) x SMs x SM clock"}
    for B in args.bytes:
        kps, descs = synth_images(args.images, args.n, B, binary=True)
        dt = [torch.from_numpy(d).to(dev) for d in descs]
        kt = [torch.from_numpy(k).to(dev) for k in kps]
        W = (B + 15) // 16 * 4
        popc = float(sum(dt[q].shape[0] * dt[t].shape[0] * W for q, t in pairs))
        paths = {
            "loop": lambda: [match_descriptors(dt[q], dt[t], kt[q], kt[t], 0.9, True, norm="hamming") for q, t in pairs],
            "batch": lambda: match_descriptors_batch(dt, pairs, kt, ratio=0.9, mutual=True, norm="hamming"),
        }

        def batch_f():
            m = paths["batch"]()
            return m, pdg.findFundamentalMatrixBatch(m.pts1, m.pts2, 0.5, 0.999, 10000, seeds=seeds, offsets=m.offsets,
                                                     n_max=m.n_max)
        paths["batch_plus_ragged_F"] = batch_f
        if B == 32:
            # the workaround without a Hamming matcher: squared L2 on the unpacked bits is the Hamming distance
            bits = [torch.from_numpy(np.unpackbits(d, axis=1).astype(np.float32)).to(dev) for d in descs]
            paths["unpacked_f32_l2_batch"] = lambda: match_descriptors_batch(bits, pairs, kt, ratio=0.9, mutual=True)
        for fn in paths.values():   # warm-up: module loads, allocator
            timed(fn)
        t = {k: [] for k in paths}
        outs = {}
        for _ in range(args.rounds):
            for k, fn in paths.items():
                s, outs[k] = timed(fn)
                t[k].append(s)
        clk, clk_max = sm_clock_mhz()   # right after the timed rounds
        rb = outs["batch"]
        off = rb.offsets.cpu().numpy()
        same = all(torch.equal(rb.idx1[off[p]:off[p + 1]], outs["loop"][p][0]) and
                   torch.equal(rb.idx2[off[p]:off[p + 1]], outs["loop"][p][1]) for p in range(P))
        r = {"bytes": B, "n_words": W, "popc_per_batch": popc, "matches": int(off[-1]), "batch_equals_loop": bool(same),
             "sm_clock_mhz": clk, "sm_clock_max_mhz": clk_max}
        bound = 16.0 * sms * clk * 1e6 if clk else None
        for k in paths:
            r[k] = {"s": med(t[k]), "pairs_per_s": P / med(t[k]), "all_s": t[k]}
            if k != "unpacked_f32_l2_batch":
                r[k]["popc_per_s"] = popc / med(t[k])
                if bound:
                    r[k]["frac_popc_bound"] = popc / med(t[k]) / bound
        r["popc_bound_per_s"] = bound
        r["batch_plus_ragged_F"]["inliers"] = int(outs["batch_plus_ragged_F"][1][1][:int(off[-1])].sum().item())
        r["speedup_batch_vs_loop"] = med(t["loop"]) / med(t["batch"])
        if B == 32:
            r["speedup_batch_vs_unpacked_f32"] = med(t["unpacked_f32_l2_batch"]) / med(t["batch"])
        # single-pair call, n1 = n2 = 2000
        from pydegensac_b200.matching import _binary_words
        w1, w2 = _binary_words([dt[0][:2000]]), _binary_words([dt[1][:2000]])
        ms = med([single_call_ms(_cabi.lib(), w1, w2, 200, binary=True)[0] for _ in range(args.rounds)])
        r["single_call"] = {"n1": 2000, "n2": 2000, "n_words": W, "mutual": True, "ms": ms,
                            "popc_per_s": 2000.0 * 2000 * W / (ms * 1e-3)}
        res["B%d" % B] = r
    res["card_after"] = card()
    emit(res, args.out)


if __name__ == "__main__":
    main()
