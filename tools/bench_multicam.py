#!/usr/bin/env python
"""Multicam batches on one GPU: one plsvo_align_multicam_batch_run over pairs from K differently calibrated cameras,
against what a caller does without it — K plsvo_align_batch_run calls of B/K pairs, one per camera.

Workload: B = 1024 VGA pairs (synth.make_multicam_batch, 300 points + 80 segments per pair, levels 4 -> 2), pairs of the
K cameras interleaved and randomly permuted, for K in {1, 4, 64}:
  K = 1  : synth.VGA
  K = 4  : synth.MULTICAM_K4, VGA and the TUM freiburg1/2/3 intrinsics
  K = 64 : one VGA sensor with individual calibrations, fx and fy within +-5 %, cx and cy within +-10 px
Arms, per K:
  multicam        : one plsvo_align_multicam_batch_run (upload -> launch -> download)
  per_camera      : K plsvo_align_batch_run calls of B/K pairs (a batch of 256 pairs or more streams through the arrival
                    gate)
  uniform_3leg    : K = 1 only, plsvo_align_upload / launch / download of the whole batch, like for like with multicam
  track_multicam  : one plsvo_track_multicam_batch_run;  track_per_camera: K plsvo_track_batch_run calls
It prints one JSON line with pairs_per_s (median over --reps), best_pairs_per_s and kernel_ms (device time of the
alignment kernels over one call, torch.profiler), and the card's name and power limit read in the same run.  Needs a GPU.

usage: python tools/bench_multicam.py [--batch 1024] [--reps 10] [--warmup 2]"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from bench_raw_track import card, kernel_ms, timed  # noqa: E402


def cameras_for(synth, K: int):
    if K == 1:
        return (synth.VGA,)
    if K == 4:
        return synth.MULTICAM_K4
    rng = np.random.default_rng(64)
    v = synth.VGA
    return tuple(synth.Camera(v.width, v.height, v.fx * s, v.fy * s, v.cx + dx, v.cy + dy)
                 for s, dx, dy in zip(rng.uniform(0.95, 1.05, K), rng.uniform(-10, 10, K), rng.uniform(-10, 10, K)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import plsvo_b200 as pkg
    from plsvo_b200 import synth

    B = args.batch
    res = {"workload": f"B={B} VGA pairs, 300 points + 80 segments, levels 4->2, K cameras interleaved", "card": card()}
    sia = pkg.SparseImgAlign(4, 2, 30)
    for K in (1, 4, 64):
        cams = cameras_for(synth, K)
        cam_of_pair = np.random.default_rng(K).permutation(np.arange(B) % K)
        al, po, cameras = synth.make_multicam_batch(cams, cam_of_pair, n_pts=300, n_segs=80, seed=9900, device="cuda",
                                                    poseopt=True)
        groups = []
        for k, cam in enumerate(cams):
            idx = np.flatnonzero(cam_of_pair == k)
            sa, sp = synth.take_pairs(al, idx), synth.take_pairs(po, idx)
            sa.cam, sp.fx = cam, cam.fx
            groups.append((sa, sp))

        def three_leg():
            sia.upload(al)
            sia.launch()
            return sia.download()

        runs = {"multicam": lambda: sia.run(al, cameras=cameras),
                "per_camera": lambda: [sia.run(sa) for sa, _ in groups]}
        if K == 1:
            runs["uniform_3leg"] = three_leg
        runs["track_multicam"] = lambda: pkg.api.track(al, po, cameras=cameras)
        runs["track_per_camera"] = lambda: [pkg.api.track(sa, sp) for sa, sp in groups]
        out = {}
        for name, fn in runs.items():
            med, best = timed(fn, args.reps, args.warmup)
            k = kernel_ms(fn, ["sparse_img_align"])["sparse_img_align"]
            out[name] = {"pairs_per_s": round(B / med, 1), "best_pairs_per_s": round(B / best, 1), "kernel_ms": round(k, 3)}
        res[f"K={K}"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
