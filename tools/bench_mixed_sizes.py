#!/usr/bin/env python
"""Pairs of several image sizes on one GPU: one multicam call over slot-sized batches (`sizes=`, every pair's frames in
the top-left corner of a slot of the largest width and height) against what a caller does without it — S multicam calls,
one per image size.

Workload: B = 1024 pairs, 300 points + 80 segments per pair, levels 4 -> 2, the sizes interleaved and randomly permuted:
  S = 2 : VGA 640x480 + EuRoC 752x480                 (slot 752x480)
  S = 3 : VGA + EuRoC + a KITTI-like 1241x376 camera  (slot 1241x480)
Arms, per S, from pageable and from pinned host buffers:
  mixed / per_size             : alignment, one call / S calls
  track_mixed / track_per_size : alignment + pose optimiser
  raw_mixed / raw_per_size     : raw frames of one distorted lens per size (plsvo_align_raw_multicam_batch_run)
It prints one JSON line with pairs_per_s (median over --reps), best_pairs_per_s, kernel_ms (device time of the
alignment kernels, and for raw of the fused rectify + pyramid kernel, over one call, torch.profiler, a run of its own),
the image bytes each arm ships (counted from shapes) and the card's name and power limit read in the same run.
Needs a GPU.

usage: python tools/bench_mixed_sizes.py [--batch 1024] [--reps 10] [--warmup 2]"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from bench_raw_track import card, kernel_ms, timed  # noqa: E402


def pinned(a):
    import torch

    t = torch.empty(a.shape, dtype=torch.uint8, pin_memory=True)
    out = t.numpy()
    out[...] = a
    return out


def pin_images(d):
    import copy

    d = copy.copy(d)
    d.ref_pyr = {l: pinned(v) for l, v in d.ref_pyr.items()}
    d.cur_pyr = {l: pinned(v) for l, v in d.cur_pyr.items()}
    return d


def image_bytes(d):
    return int(sum(v.nbytes for v in d.ref_pyr.values()) + sum(v.nbytes for v in d.cur_pyr.values()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import plsvo_b200 as pkg
    from plsvo_b200 import synth

    B = args.batch
    wide = synth.Camera(1241, 376, 718.856, 718.856, 607.1928, 185.2157)
    dists = {640: (-0.28, 0.07, 0.0, 0.0, 0.0), 752: synth.EUROC_DIST, 1241: (-0.1, 0.02, 0.0, 0.0, 0.0)}
    res = {"workload": f"B={B} pairs, 300 points + 80 segments, levels 4->2, S image sizes interleaved", "card": card()}
    sia = pkg.SparseImgAlign(4, 2, 30)
    for S, cams in ((2, (synth.VGA, synth.EUROC)), (3, (synth.VGA, synth.EUROC, wide))):
        g = np.random.default_rng(S).permutation(np.arange(B) % S)
        groups = [np.flatnonzero(g == k) for k in range(S)]
        al_parts, po_parts, raw_parts = [], [], []
        for k, (cam, idx) in enumerate(zip(cams, groups)):
            al, po, raw, _ = synth.make_raw_multicam_batch([cam], [dists[cam.width]], np.zeros(len(idx), int), n_pts=300, n_segs=80,
                                                           seed=9900 + k, device="cuda", poseopt=True)
            po.fx = cam.fx
            al_parts.append(al), po_parts.append(po), raw_parts.append(raw)
        al, sizes, raw = synth.merge_sizes(al_parts, groups, raws=raw_parts)
        po = synth.scatter_batches(po_parts, groups, B)
        k4 = np.zeros((B, 4))
        for cam, idx in zip(cams, groups):
            k4[idx] = (cam.fx, cam.fy, cam.cx, cam.cy)
        lenses = [pkg.PinholeCamera(c.width, c.height, c.fx, c.fy, c.cx, c.cy, *dists[c.width]) for c in cams]
        cop = g.astype(np.int32)
        raw_al = synth.take_pairs(al, np.arange(B))
        raw_al.ref_pyr = raw_al.cur_pyr = {}
        raw_sub = []
        for k, idx in enumerate(groups):
            sub = synth.take_pairs(al_parts[k], np.arange(len(idx)))
            sub.ref_pyr = sub.cur_pyr = {}
            raw_sub.append(sub)
        out = {"bytes": {"mixed": image_bytes(al), "per_size": sum(image_bytes(p) for p in al_parts),
                         "raw_mixed": int(raw[0].nbytes * 2), "raw_per_size": int(sum(r[0].nbytes * 2 for r in raw_parts))}}
        for mem in ("pageable", "pinned"):
            m_al = pin_images(al) if mem == "pinned" else al
            parts = [pin_images(p) for p in al_parts] if mem == "pinned" else al_parts
            m_raw = tuple(pinned(r) for r in raw) if mem == "pinned" else raw
            p_raw = [tuple(pinned(r) for r in rr) for rr in raw_parts] if mem == "pinned" else raw_parts
            runs = {
                "mixed": lambda: sia.run(m_al, cameras=k4, sizes=sizes),
                "per_size": lambda: [sia.run(p, cameras=k4[idx]) for p, idx in zip(parts, groups)],
                "track_mixed": lambda: pkg.api.track(m_al, po, cameras=k4, sizes=sizes),
                "track_per_size": lambda: [pkg.api.track(p, q, cameras=k4[idx]) for p, q, idx in zip(parts, po_parts, groups)],
                "raw_mixed": lambda: sia.run_raw(lenses, m_raw, raw_al, cam_of_pair=cop),
                "raw_per_size": lambda: [sia.run_raw([lenses[k]], p_raw[k], raw_sub[k], cam_of_pair=np.zeros(len(idx), np.int32))
                                         for k, idx in enumerate(groups)],
            }
            for name, fn in runs.items():
                med, best = timed(fn, args.reps, args.warmup)
                r = {"pairs_per_s": round(B / med, 1), "best_pairs_per_s": round(B / best, 1)}
                if mem == "pinned":
                    names = ["sparse_img_align"] + (["undistort_pyramid"] if name.startswith("raw") else [])
                    km = kernel_ms(fn, names)
                    r["kernel_ms"] = round(km["sparse_img_align"], 3)
                    if name.startswith("raw"):
                        r["fused_us_per_frame"] = round(1000.0 * km["undistort_pyramid"] / (2 * B), 4)
                out[f"{name}_{mem}"] = r
        res[f"S={S}"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
