#!/usr/bin/env python
"""Raw frames from K differently calibrated lenses on one GPU: one plsvo_align_raw_multicam_batch_run against what a
caller does without it.

Workload: B = 1024 raw pairs (synth.make_raw_multicam_batch: each pair rendered through its own lens), 300 points + 80
segments per pair, levels 4 -> 2, pairs of the K cameras interleaved and randomly permuted, for:
  K = 1  : EuRoC cam0 (752x480, config/dataset_params.yaml)
  K = 4  : the four VGA lenses of tests/golden/undistort_cv2.json (strong barrel, pincushion, tangential only, d0 = 0)
  K = 64 : EuRoC sensors with individual calibrations: fx, fy +-5 %, cx, cy +-10 px, k1, k2 +-10 %
Arms, per K, raw frames in pageable and in pinned (plsvo_host_alloc) host memory:
  raw_multicam        : one plsvo_align_raw_multicam_batch_run
  per_camera_raw      : K plsvo_align_raw_batch_run calls of the camera's pairs
  host_rect_multicam  : cv2.remap of every frame with its camera's map (maps made beforehand, one thread), then one
                        plsvo_align_multicam_batch_run shipping level 0 (levels 1..4 derived on the device)
  track_raw_multicam / track_per_camera_raw : the track forms of the first two
Also: fused_kernel_us_per_frame, the device time of the rectify + pyramid kernel over one raw_multicam call divided by
its 2B frames (torch.profiler), for the pairs in their random order; and cold_map_build_ms, plsvo_last_map_build_ms of
the first call on a fresh context (K map builds).  It prints one JSON line with the card's name and power limit read in
the same run.  Needs a GPU.

usage: python tools/bench_raw_multicam.py [--batch 1024] [--reps 10] [--warmup 2]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from bench_raw_track import card, kernel_ms, timed  # noqa: E402

VGA4 = ("vga_strong_barrel_k3", "vga_pincushion", "vga_tangential_only", "vga_d0_zero_is_a_copy")


def lenses(K: int):
    """(width, height, fx, fy, cx, cy, d0..d4) of the K cameras."""
    with open(os.path.join(ROOT, "tests", "golden", "undistort_cv2.json")) as f:
        golden = json.load(f)["cameras"]
    if K == 4:
        return [golden[n]["params"] for n in VGA4]
    W, H, fx, fy, cx, cy, k1, k2, p1, p2, k3 = golden["euroc_dataset_params"]["params"]
    if K == 1:
        return [[W, H, fx, fy, cx, cy, k1, k2, p1, p2, k3]]
    rng = np.random.default_rng(64)
    s = rng.uniform(-1, 1, (K, 6))
    return [[W, H, fx * (1 + 0.05 * a), fy * (1 + 0.05 * b), cx + 10 * c, cy + 10 * d, k1 * (1 + 0.1 * e), k2 * (1 + 0.1 * g), p1, p2, k3]
            for a, b, c, d, e, g in s]


def pinned_copy(ctx, a):
    p = C.c_void_p()
    ctx.check(ctx.lib.plsvo_host_alloc(C.byref(p), a.nbytes), "plsvo_host_alloc")
    out = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(a.nbytes,)).reshape(a.shape)
    out[...] = a
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import cv2
    import plsvo_b200 as pkg
    from plsvo_b200 import synth

    B = args.batch
    res = {"workload": f"B={B} raw pairs, 300 points + 80 segments, levels 4->2, K lenses interleaved", "card": card()}
    for K in (1, 4, 64):
        ctx = pkg.api.Context(0)
        sia = pkg.SparseImgAlign(4, 2, 30, ctx=ctx)
        lens = lenses(K)
        cams = [synth.Camera(*p[:6]) for p in lens]
        dists = [tuple(p[6:]) for p in lens]
        pcs = [pkg.PinholeCamera(*p) for p in lens]
        cop = np.random.default_rng(K).permutation(np.arange(B) % K).astype(np.int32)
        al, po, (ref, cur), cameras = synth.make_raw_multicam_batch(cams, dists, cop, n_pts=300, n_segs=80, seed=9900,
                                                                    device="cuda", poseopt=True)
        al.ref_pyr = al.cur_pyr = {}
        raws = {"pageable": (ref, cur), "pinned": (pinned_copy(ctx, ref), pinned_copy(ctx, cur))}
        groups = []
        for k in range(K):
            idx = np.flatnonzero(cop == k)
            sa, sp = synth.take_pairs(al, idx), synth.take_pairs(po, idx)
            sa.cam, sp.fx = cams[k], abs(cams[k].fx)
            groups.append((k, idx, sa, sp))
        # a fresh context's first call builds every map
        cold = pkg.api.Context(0)
        pkg.SparseImgAlign(4, 2, 30, ctx=cold).run_raw(pcs, raws["pinned"], al, cam_of_pair=cop)
        out = {"cold_map_build_ms": cold.last_map_build_ms(), "n_maps_built": int(sum(abs(p[6]) > 1e-7 for p in lens))}
        cold.close()
        maps = [cv2.initUndistortRectifyMap(np.array([[p[2], 0, p[4]], [0, p[3], p[5]], [0, 0, 1]], np.float32),
                                            np.array(p[6:], np.float32), None,
                                            np.array([[p[2], 0, p[4]], [0, p[3], p[5]], [0, 0, 1]], np.float32), (p[0], p[1]),
                                            cv2.CV_16SC2) if abs(p[6]) > 1e-7 else None for p in lens]

        def host_rect(raw):
            r0, r1 = np.empty_like(raw[0]), np.empty_like(raw[1])
            for src, dst in ((raw[0], r0), (raw[1], r1)):
                for b in range(B):
                    m = maps[cop[b]]
                    dst[b] = cv2.remap(src[b], m[0], m[1], cv2.INTER_LINEAR) if m is not None else src[b]
            al.ref_pyr, al.cur_pyr = {0: r0}, {0: r1}
            try:
                return sia.run(al, cameras=cameras)
            finally:
                al.ref_pyr = al.cur_pyr = {}

        # each camera's frames as stacks of their own, in the same kind of host memory, made before the clock runs
        group_raws = {"pageable": [(ref[idx], cur[idx]) for _, idx, _, _ in groups]}
        group_raws["pinned"] = [(pinned_copy(ctx, a), pinned_copy(ctx, b)) for a, b in group_raws["pageable"]]
        for mem, raw in raws.items():
            graw = group_raws[mem]
            runs = {"raw_multicam": lambda: sia.run_raw(pcs, raw, al, cam_of_pair=cop),
                    "per_camera_raw": lambda: [sia.run_raw(pcs[k], graw[k], sa) for k, _, sa, _ in groups],
                    "host_rect_multicam": lambda: host_rect(raw),
                    "track_raw_multicam": lambda: pkg.api.track_raw(pcs, raw, al, po, ctx=ctx, cam_of_pair=cop),
                    "track_per_camera_raw": lambda: [pkg.api.track_raw(pcs[k], graw[k], sa, sp, ctx=ctx) for k, _, sa, sp in groups]}
            for name, fn in runs.items():
                med, best = timed(fn, args.reps, args.warmup)
                out.setdefault(name, {})[mem] = {"pairs_per_s": round(B / med, 1), "best_pairs_per_s": round(B / best, 1)}
        for name, fn in (("raw_multicam", lambda: sia.run_raw(pcs, raws["pinned"], al, cam_of_pair=cop)),
                         ("per_camera_raw", lambda: [sia.run_raw(pcs[k], group_raws["pinned"][k], sa) for k, _, sa, _ in groups])):
            k = kernel_ms(fn, ["undistort_pyramid", "sparse_img_align"])
            out[name]["kernel_ms"] = {n: round(v, 3) for n, v in k.items()}
        out["fused_kernel_us_per_frame"] = round(1e3 * out["raw_multicam"]["kernel_ms"]["undistort_pyramid"] / (2 * B), 3)
        res[f"K={K}"] = out
        ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
