#!/usr/bin/env python
"""Cost of one ATAN multicam call against one ATAN call per camera, on one GPU.

Workload: B = 1024 pairs of SVO's stock 752x480 FOV camera, 300 points + 80 segments per pair, levels 4 -> 2, bearings
given.  K in {1, 4, 64} cameras, each the stock camera with fx, fy, cx, cy perturbed by up to 2 % and d0 by up to 5 %;
the pairs are spread round-robin over the cameras.  For alignment and for tracking, one
plsvo_*_atan_multicam_batch_run over the batch is compared with K plsvo_*_atan_batch_run calls, one per camera's pairs.
It prints one JSON line with, per K and call:
  pairs_per_s : end-to-end pairs/s (median over --reps calls; the K-call form counts all K calls as one)
  kernel_ms   : device time of the alignment (and pose-optimiser) kernels over one call, from torch.profiler in a run of
                its own
The card's name and power limit are read in the same run.  Needs a GPU.

usage: python tools/bench_atan_multicam.py [--batch 1024] [--reps 10] [--warmup 2] [--ks 1,4,64]"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from bench_raw_track import card, kernel_ms, timed  # noqa: E402

STOCK = (752, 480, 0.511496, 0.802603, 0.530199, 0.496011, 0.934092)


def cameras(pkg, k, rng):
    w, h, fx, fy, cx, cy, d0 = STOCK
    if k == 1:
        return [pkg.ATANCamera(*STOCK)]
    p = lambda v, s: v * (1.0 + rng.uniform(-s, s))  # noqa: E731
    return [pkg.ATANCamera(w, h, p(fx, 0.02), p(fy, 0.02), p(cx, 0.02), p(cy, 0.02), p(d0, 0.05)) for _ in range(k)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ks", default="1,4,64")
    args = ap.parse_args()
    import plsvo_b200 as pkg
    from plsvo_b200 import synth

    rng = np.random.default_rng(9300)
    res = {"workload": f"B={args.batch} 752x480 FOV pairs, 300 points + 80 segments, levels 4->2", "card": card()}
    names = ["sparse_img_align", "pose_optimizer"]
    for k in (int(s) for s in args.ks.split(",")):
        cams = cameras(pkg, k, rng)
        cop = np.arange(args.batch) % k
        data, po, parts, po_parts, groups = synth.make_atan_multicam_batch(cams, cop, poseopt=True, n_pts=300, n_segs=80,
                                                                           seed=9400 + k, device="cuda")
        sia = pkg.SparseImgAlign(4, 2, 30)
        runs = {
            "align_one_call": lambda: sia.run(data, camera=cams, cam_of_pair=cop),
            "align_k_calls": lambda: [sia.run(p, camera=c) for p, c in zip(parts, cams)],
            "track_one_call": lambda: pkg.api.track(data, po, camera=cams, cam_of_pair=cop),
            "track_k_calls": lambda: [pkg.api.track(p, q, camera=c) for p, q, c in zip(parts, po_parts, cams)],
        }
        out = {}
        for name, fn in runs.items():
            med, best = timed(fn, args.reps, args.warmup)
            kms = kernel_ms(fn, names)
            out[name] = {"pairs_per_s": round(args.batch / med, 1), "best_pairs_per_s": round(args.batch / best, 1),
                         "kernel_ms": {n: round(v, 3) for n, v in kms.items() if v}}
        res[f"K={k}"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
