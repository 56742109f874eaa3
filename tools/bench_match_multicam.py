#!/usr/bin/env python
"""Cost of one findMatchDirect call with a camera per image (plsvo_match_direct_multicam_batch_run) against one call per
camera (plsvo_match_direct_batch_run / plsvo_match_direct_atan_batch_run), on one GPU.

Workload: about --n candidates (default 200 000) from K in {1, 4, 64} cameras, each contributing 2 keyframes and 2 current
frames, 4 pyramid levels, a quarter of them edgelets.  Fleets: pinhole only and ATAN only at VGA (640x480), and pinhole
and ATAN cameras alternating over VGA and 752x480 (slot 752x480).  Every candidate pairs two images of one camera, so the
K one-camera calls can answer the same candidates; both arms run on identical images and candidates, the one-camera
calls on each camera's frames cut out of the slots.  The two arms alternate within each repetition.
It prints one JSON line with, per fleet and K, for each arm:
  kernel_ms    : plsvo_last_kernel_ms (the kernel alone, CUDA events), summed over the arm's calls, median over --reps
  cands_per_s  : end-to-end candidates/s of Matcher.findMatchDirect (uploads, kernel, downloads), median over --reps
  bytes_h2d / bytes_d2h : what the arm's calls copy, computed from the shapes (images, poses, candidates, camera table)
The card's name and power limit are read in the same run.  Needs a GPU.

usage: python tools/bench_match_multicam.py [--n 200000] [--reps 10] [--warmup 2] [--k 1,4,64]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from dataclasses import replace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

from bench_raw_track import card  # noqa: E402

CAND_H2D = 4 + 4 + 16 + 24 + 4 + 1 + 16 + 24 + 16 + 32  # indices, ref_px, ref_f, level, edgelet, grad, pos, px_cur, A_cur_ref
CAND_D2H = 16 + 1 + 4 + 32  # px_cur, success, search level, A_cur_ref


def shipped(d, n_cams=0):
    """(host->device, device->host) bytes of one call on d: every image level's rows (cut to its width), the poses, the
    per-candidate arrays, and with n_cams the camera table (80 bytes a camera) and the two image-index arrays."""
    img = sum(im.shape[0] * im.shape[1] * im.shape[2] for pyr in (d.ref_pyr, d.cur_pyr) for im in pyr.values())
    n_img = d.T_ref_w.shape[0] + d.T_cur_w.shape[0]
    table = 80 * n_cams + 4 * n_img if n_cams else 0
    return img + 56 * n_img + CAND_H2D * d.n + table, CAND_D2H * d.n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--k", default="1,4,64")
    args = ap.parse_args()
    import plsvo_b200 as pkg
    from plsvo_b200 import synth

    import match_multicam_cases as mc

    res = {"workload": f"~{args.n} findMatchDirect candidates, 2 keyframes + 2 current frames per camera, 4 levels, 25 % edgelets",
           "card": card()}
    ctx = pkg.default_context()
    m = pkg.Matcher(10, ctx)
    for fleet, sizes in (("pinhole", ((640, 480),)), ("atan", ((640, 480),)), ("mixed", mc.MIXED_SIZES)):
        for k in (int(x) for x in args.k.split(",")):
            cams = mc.fleet(pkg, synth, fleet, k, sizes)
            ref, cur = mc.images(k, 2)
            d, parts, groups = synth.make_match_multicam_batch(cams, ref, cur, n=args.n, n_pyr_levels=4, seed=9950 + k, device="cuda",
                                                               same_camera_frac=1.0)
            parts = [None if p is None else replace(p, ref_pyr={l: np.ascontiguousarray(v) for l, v in p.ref_pyr.items()},
                                                    cur_pyr={l: np.ascontiguousarray(v) for l, v in p.cur_pyr.items()}) for p in parts]
            used = [j for j, p in enumerate(parts) if p is not None]
            assert sum(len(groups[j]) for j in used) == d.n

            def per_image():
                return m.findMatchDirect(d, camera=cams, cam_of_ref=ref, cam_of_cur=cur), ctx.last_kernel_ms()

            def per_camera():
                outs, kms = [], 0.0
                for j in used:
                    outs.append(m.findMatchDirect(parts[j], camera=cams[j]) if mc.is_atan(cams[j]) else m.findMatchDirect(parts[j]))
                    kms += ctx.last_kernel_ms()
                return outs, kms

            arms = {"one_call": per_image, f"{len(used)}_calls": per_camera}
            t = {a: [] for a in arms}
            kms = {a: [] for a in arms}
            for rep in range(args.warmup + args.reps):
                for a, fn in arms.items():
                    t0 = time.perf_counter()
                    _, km = fn()
                    if rep >= args.warmup:
                        t[a].append(time.perf_counter() - t0)
                        kms[a].append(km)
            got, _ = per_image()
            outs, _ = per_camera()
            same = all(np.array_equal(got.px_cur[groups[j]].view(np.uint8), o.px_cur.view(np.uint8)) and
                       np.array_equal(got.success[groups[j]], o.success) for j, o in zip(used, outs))
            b_one = shipped(d, k)
            b_k = tuple(sum(x) for x in zip(*(shipped(parts[j]) for j in used)))
            row = {"n": d.n, "equal_outputs": bool(same), "success_rate": round(float(got.success.mean()), 4)}
            for a, b in (("one_call", b_one), (f"{len(used)}_calls", b_k)):
                row[a] = {"kernel_ms": round(float(np.median(kms[a])), 4), "cands_per_s": round(d.n / float(np.median(t[a])), 1),
                          "bytes_h2d": int(b[0]), "bytes_d2h": int(b[1])}
            res[f"{fleet}_K{k}"] = row
            print(json.dumps({f"{fleet}_K{k}": row}), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
