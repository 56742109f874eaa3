#!/usr/bin/env python
"""Cost of the ATAN (FOV) camera model in sparse image alignment on one GPU: plsvo_align_atan_batch_run against
plsvo_align_batch_run on the same workload.

Workload: B = 1024 VGA pairs (synth.make_align_batch, 300 points + 80 segments per pair, levels 4 -> 2), bearings given.
The ATAN call always runs upload -> launch -> download; the pinhole call is timed that way too (its three-leg form,
like for like) and through plsvo_align_batch_run, which streams a batch this size through the arrival gate.  It prints one JSON line with, per camera (pinhole; ATAN with
d0 = 0, 0.3, 0.93):
  pairs_per_s : end-to-end pairs/s of one call (median over --reps)
  kernel_ms   : device time of the alignment kernel over one call (torch.profiler)
  iters       : mean Gauss-Newton passes per pair (the distortion changes the optimisation, not only its cost per pass)
  patch_iters : mean patches evaluated per pair, and kernel ns per evaluated patch
The card's name and power limit are read in the same run.  Needs a GPU.

usage: python tools/bench_atan.py [--batch 1024] [--reps 10] [--warmup 2]"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from bench_raw_track import card, kernel_ms, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import plsvo_b200 as pkg
    from plsvo_b200 import synth

    data = synth.make_align_batch(batch=args.batch, n_pts=300, n_segs=80, seed=9100, device="cuda")
    sia = pkg.SparseImgAlign(4, 2, 30)

    def pinhole_plain():  # upload -> launch -> download, as the ATAN call runs
        sia.upload(data)
        sia.launch()
        return sia.download()

    w, h, cam = synth.VGA.width, synth.VGA.height, synth.VGA
    res = {"workload": f"B={args.batch} VGA pairs, 300 points + 80 segments, levels 4->2", "card": card()}
    runs = {"pinhole_plain": pinhole_plain, "pinhole_batch_run": lambda: sia.run(data)}
    for d0 in (0.0, 0.3, 0.93):
        at = pkg.ATANCamera(w, h, cam.fx / w, cam.fy / h, (cam.cx + 0.5) / w, (cam.cy + 0.5) / h, d0)
        d = data if d0 == 0.0 else _with_bearings(data, at)
        runs[f"atan_d0={d0}"] = (lambda d=d, at=at: sia.run(d, camera=at))
    for name, fn in runs.items():
        med, best = timed(fn, args.reps, args.warmup)
        out = fn()
        k = kernel_ms(fn, ["sparse_img_align"])["sparse_img_align"]
        pi = float(out.patch_iters.mean())
        res[name] = {"pairs_per_s": round(args.batch / med, 1), "best_pairs_per_s": round(args.batch / best, 1),
                     "kernel_ms": round(k, 3), "iters": round(float(out.iters.sum(1).mean()), 2), "patch_iters": round(pi, 1),
                     "kernel_ns_per_patch": round(k * 1e6 / (pi * args.batch), 3)}
    print(json.dumps(res))


def _with_bearings(data, at):
    import copy

    d = copy.copy(data)
    d.pt_f = np.ascontiguousarray(at.cam2world(data.pt_px))
    d.seg_sf = np.ascontiguousarray(at.cam2world(data.seg_spx))
    d.seg_ef = np.ascontiguousarray(at.cam2world(data.seg_epx))
    return d


if __name__ == "__main__":
    main()
