#!/usr/bin/env python
"""Cost of one raw any-camera call (raw frames from distorted lenses and ATAN (FOV) cameras in one batch) against the
best a caller can do without it, on one GPU.

Workload: B = 1024 raw pairs in a 752x480 slot, 300 points + 80 segments per pair, levels 4 -> 2, bearings given.
Fleets of K in {2, 8, 64} cameras, all 752x480: the even ones EuRoC cam0 lenses (config/dataset_params.yaml) with fx, fy
perturbed by up to 5 %, cx, cy by up to 10 px and k1, k2 by up to 10 %; the odd ones SVO's stock FOV camera with fx, fy,
cx, cy perturbed by up to 2 % and d0 by up to 5 %.  The pairs are interleaved over the cameras
(synth.make_raw_any_camera_batch renders every pair through its own camera).  Arms, for alignment and for tracking, raw
frames in pageable and in pinned (plsvo_host_alloc) host memory:
  any_call   : one plsvo_*_raw_any_camera_batch_run over the batch
  two_calls  : one plsvo_*_raw_multicam_batch_run on the lens pairs and one plsvo_*_atan_multicam_batch_run on the ATAN
               pairs, shipping the ATAN frames' level 0 and deriving levels 1..4 on the device (so both arms ship the same
               image bytes); inputs split beforehand into the same kind of host memory, outputs scattered back
It prints one JSON line with, per fleet and arm:
  pairs_per_s  : end-to-end pairs/s, median of --reps calls, the four arms of a memory kind alternating call by call
  kernel_ms    : device time over one call (torch.profiler, in a run of its own) of the fused rectify / pyramid kernel,
                 the device pyramid kernel (levels derived from a shipped level 0), the map builds, the alignment and the
                 pose-optimiser kernels
  image_h2d_bytes : raw image bytes the call ships (both arms: 2B slot-sized frames)
  equal        : whether the arm's outputs are byte-identical to the any-camera call's
The card's name and power limit are read in the same run.  Needs a GPU.

usage: python tools/bench_raw_any_camera.py [--batch 1024] [--reps 10] [--warmup 2] [--ks 2,8,64]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from bench_any_camera import ALIGN_FIELDS, PO_FIELDS, STOCK, alternating, same, scatter  # noqa: E402
from bench_raw_track import card  # noqa: E402

KERNELS = (("fused_rectify_pyramid", "undistort_pyramid"), ("map_build", "undistort_map"), ("derive_pyramid", "pyramid_kernel"),
           ("align", "sparse_img_align"), ("pose_optimizer", "pose_optimizer"))


def fleet(pkg, k, rng):
    """k cameras of 752x480, the even ones perturbed EuRoC lenses and the odd ones perturbed stock ATAN cameras."""
    with open(os.path.join(ROOT, "tests", "golden", "undistort_cv2.json")) as f:
        W, H, fx, fy, cx, cy, k1, k2, p1, p2, k3 = json.load(f)["cameras"]["euroc_dataset_params"]["params"]
    w, h, afx, afy, acx, acy, d0 = STOCK
    p = lambda v, s: v * (1.0 + rng.uniform(-s, s))  # noqa: E731
    out = []
    for i in range(k):
        if i % 2 == 0:
            out.append(pkg.PinholeCamera(W, H, p(fx, 0.05), p(fy, 0.05), cx + rng.uniform(-10, 10), cy + rng.uniform(-10, 10),
                                         p(k1, 0.1), p(k2, 0.1), p1, p2, k3))
        else:
            out.append(pkg.ATANCamera(w, h, p(afx, 0.02), p(afy, 0.02), p(acx, 0.02), p(acy, 0.02), p(d0, 0.05)))
    return out


def pinned_copy(ctx, a, held):
    """a copy of `a` in pinned host memory (plsvo_host_alloc), its pointer appended to `held` for plsvo_host_free"""
    p = C.c_void_p()
    ctx.check(ctx.lib.plsvo_host_alloc(C.byref(p), a.nbytes), "plsvo_host_alloc")
    held.append(p)
    out = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(a.nbytes,)).reshape(a.shape)
    out[...] = a
    return out


def kernel_ms(fn):
    """Device time per kernel kind over one call of fn (torch.profiler); the fused kernel's name also holds
    "pyramid_kernel", so every event counts once, for the first kind it matches."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n, _ in KERNELS}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        for n, key in KERNELS:
            if key in ev.name:
                out[n] += ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
                break
    return {n: round(v, 3) for n, v in out.items() if v}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ks", default="2,8,64")
    args = ap.parse_args()
    import plsvo_b200 as pkg
    from plsvo_b200 import synth

    B = args.batch
    rng = np.random.default_rng(9800)
    res = {"workload": f"B={B} raw pairs in a 752x480 slot, 300 points + 80 segments, levels 4->2, half EuRoC lenses and half "
                       "ATAN cameras, interleaved", "card": card()}
    ctx = pkg.api.Context(0)
    sia = pkg.SparseImgAlign(4, 2, 30, ctx=ctx)
    for k in (int(s) for s in args.ks.split(",")):
        cams = fleet(pkg, k, rng)
        cop = (np.arange(B) % k).astype(np.int32)
        al, po, (ref, cur), _, _, _ = synth.make_raw_any_camera_batch(cams, cop, poseopt=True, n_pts=300, n_segs=80,
                                                                      seed=9900 + k, device="cuda")
        al.ref_pyr = al.cur_pyr = {}
        atan = np.array([isinstance(cams[c], pkg.ATANCamera) for c in cop])
        index = [np.flatnonzero(~atan), np.flatnonzero(atan)]
        tables = []
        for idx in index:
            used = sorted({int(c) for c in cop[idx]})
            tables.append(([cams[c] for c in used], np.array([used.index(c) for c in cop[idx]], np.int32)))
        subs = [synth.take_pairs(al, idx) for idx in index]
        po_subs = [synth.take_pairs(po, idx) for idx in index]
        held = []
        raws = {"pageable": (ref, cur), "pinned": (pinned_copy(ctx, ref, held), pinned_copy(ctx, cur, held))}
        out = {}
        results = {}
        for mem, raw in raws.items():
            lens_raw = tuple(pinned_copy(ctx, r[index[0]], held) if mem == "pinned" else r[index[0]] for r in raw)
            atan_l0 = tuple(pinned_copy(ctx, r[index[1]], held) if mem == "pinned" else r[index[1]] for r in raw)
            atan_sub = synth.take_pairs(subs[1], np.arange(len(index[1])))
            atan_sub.ref_pyr, atan_sub.cur_pyr = {0: atan_l0[0]}, {0: atan_l0[1]}

            def align_two_calls(lens_raw=lens_raw, atan_sub=atan_sub):
                outs = (sia.run_raw(tables[0][0], lens_raw, subs[0], cam_of_pair=tables[0][1]),
                        sia.run(atan_sub, camera=tables[1][0], cam_of_pair=tables[1][1]))
                return scatter(outs, index, B, ALIGN_FIELDS)

            def track_two_calls(lens_raw=lens_raw, atan_sub=atan_sub):
                outs = (pkg.api.track_raw(tables[0][0], lens_raw, subs[0], po_subs[0], ctx=ctx, cam_of_pair=tables[0][1]),
                        pkg.api.track(atan_sub, po_subs[1], ctx=ctx, camera=tables[1][0], cam_of_pair=tables[1][1]))
                return [scatter([o[j] for o in outs], index, B, f) for j, f in ((0, ALIGN_FIELDS), (1, PO_FIELDS))]

            runs = {"align_any_call": lambda raw=raw: sia.run_raw(cams, raw, al, cam_of_pair=cop),
                    "align_two_calls": align_two_calls,
                    "track_any_call": lambda raw=raw: pkg.api.track_raw(cams, raw, al, po, ctx=ctx, cam_of_pair=cop),
                    "track_two_calls": track_two_calls}
            med = alternating(runs, args.reps, args.warmup)
            for name in runs:
                out.setdefault(name, {})[mem] = {"pairs_per_s": round(B / med[name], 1)}
            results[mem] = runs
        runs = results["pinned"]
        ref_a, ref_t = runs["align_any_call"](), runs["track_any_call"]()
        tt = runs["track_two_calls"]()
        out["align_two_calls"]["equal"] = same(runs["align_two_calls"](), ref_a, ALIGN_FIELDS)
        out["track_two_calls"]["equal"] = same(tt[0], ref_t[0], ALIGN_FIELDS) and same(tt[1], ref_t[1], PO_FIELDS)
        for name, fn in runs.items():
            out[name]["kernel_ms"] = kernel_ms(fn)
            out[name]["image_h2d_bytes"] = int(ref.nbytes + cur.nbytes)
        res[f"K={k}"] = out
        del raws, results, runs, tt, ref_a, ref_t
        ctx.sync()
        for p in held:
            ctx.lib.plsvo_host_free(p)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
