#!/usr/bin/env python
"""Cost of findMatchDirect for frames from an ATAN (FOV) camera against the pinhole matcher, on one GPU.

Workload: --n candidates (default 200 000, about what a reprojector pass of a few hundred frames hands over) on 4 keyframes
and 4 current frames, 4 pyramid levels, a quarter of them edgelets, at VGA (640x480) and at SVO's stock ATAN size
(752x480).  Cameras: the undistorted pinhole (plsvo_match_direct_batch_run), ATAN with d0 = 0 and ATAN with d0 = 0.93
(plsvo_match_direct_atan_batch_run), all three with the same members fx_..cy_.
It prints one JSON line with, per size and camera:
  kernel_ms        : plsvo_last_kernel_ms (the kernel alone, CUDA events), median over --reps calls
  cands_per_s      : end-to-end candidates/s of Matcher.findMatchDirect (uploads, kernel, downloads), median over --reps
  cpu_cands_per_s  : the CPU oracle (ATAN oracle for the ATAN cameras, pinhole oracle otherwise) on every host thread
The card's name and power limit are read in the same run.  Needs a GPU.

usage: python tools/bench_atan_match.py [--n 200000] [--reps 20] [--warmup 3]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools")]

from bench_raw_track import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import plsvo_b200 as pkg
    from plsvo_b200 import synth

    import oracle_atan_match
    import oracle_lib

    abi = pkg.abi
    res = {"workload": f"{args.n} findMatchDirect candidates, 4 keyframes + 4 current frames, 4 levels, 25 % edgelets", "card": card(),
           "cpu_threads": os.cpu_count()}
    ctx = pkg.default_context()
    m = pkg.Matcher(10, ctx)
    for size in ("VGA", "EUROC"):
        base = getattr(synth, size)
        w, h = base.width, base.height
        cams = {d0: pkg.ATANCamera(w, h, base.fx / w, base.fy / h, (base.cx + 0.5) / w, (base.cy + 0.5) / h, d0) for d0 in (0.0, 0.93)}
        c0 = cams[0.0]
        pin = synth.Camera(w, h, c0.fx_, c0.fy_, c0.cx_, c0.cy_)
        out = {}
        for name, cam in (("pinhole", None), ("atan_d0=0", cams[0.0]), ("atan_d0=0.93", cams[0.93])):
            d = synth.make_match_batch(cam=pin, n=args.n, n_ref=4, n_cur=4, n_pyr_levels=4, seed=9900, device="cuda", atan=cam)
            fn = (lambda: m.findMatchDirect(d)) if cam is None else (lambda: m.findMatchDirect(d, camera=cam))
            kms = []

            def call():
                r = fn()
                kms.append(ctx.last_kernel_ms())
                return r

            med, best = timed(call, args.reps, args.warmup)
            got = fn()
            t0 = time.perf_counter()
            ref = oracle_lib.match_direct(abi, d, os.cpu_count()) if cam is None else oracle_atan_match.match_direct(abi, cam, d)
            cpu = time.perf_counter() - t0
            out[name] = {"kernel_ms": round(float(np.median(kms[args.warmup:])), 4), "cands_per_s": round(args.n / med, 1),
                         "best_cands_per_s": round(args.n / best, 1), "cpu_cands_per_s": round(args.n / cpu, 1),
                         "success_rate": round(float(got.success.mean()), 4),
                         "search_level_equal_to_oracle": round(float((got.search_level == ref.search_level).mean()), 6)}
        res[f"{w}x{h}"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
