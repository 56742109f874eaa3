#!/usr/bin/env python
"""Cost of one any-camera call (pinhole and ATAN pairs in one batch) against the best a caller can do without it, on one
GPU.

Workload: B = 1024 pairs, 300 points + 80 segments per pair, levels 4 -> 2, bearings given, in a 752x480 slot.  Fleets of
K in {2, 8, 64} cameras, half pinhole and half ATAN (SVO's stock FOV camera with fx, fy, cx, cy perturbed by up to 2 %
and d0 by up to 5 %; pinhole cameras with focal lengths 400..480), all 752x480, the pairs interleaved over the cameras.
Arms, for alignment and for tracking:
  any_call      : one plsvo_*_any_camera_batch_run over the batch
  two_calls     : one pinhole multicam call on the pinhole pairs and one ATAN multicam call on the ATAN pairs (inputs
                  split beforehand), the outputs scattered back into batch order
  K = 1 of each model: the any-camera call on a one-camera table against that model's per-pair multicam call, which
  measures what the tag and the second branch cost.
It prints one JSON line with, per fleet and arm:
  pairs_per_s  : end-to-end pairs/s, median of --reps calls, the arms alternating call by call
  kernel_ms    : device time of the alignment (and pose-optimiser) kernels over one call, from torch.profiler in a run of
                 its own
  camera_h2d_bytes : bytes of the per-pair camera arrays the call uploads (records, distortion terms, tags), from their
                 sizes; the batch's own arrays are the same for every arm
  equal        : whether the arm's outputs are byte-identical to the any-camera call's
The card's name and power limit are read in the same run.  Needs a GPU.

usage: python tools/bench_any_camera.py [--batch 1024] [--reps 10] [--warmup 2] [--ks 2,8,64]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from bench_raw_track import card, kernel_ms  # noqa: E402

STOCK = (752, 480, 0.511496, 0.802603, 0.530199, 0.496011, 0.934092)
ALIGN_FIELDS = ("T_cur_w", "n_tracked", "H", "seg_killed", "iters", "status", "patch_iters", "patch_levels")
PO_FIELDS = ("T_f_w", "cov", "estimated_scale", "error_init", "error_final", "num_obs_pt", "num_obs_ls", "pt_outlier",
             "seg_outlier", "iters", "status")
REC, TERMS, TAG = 40, 32, 4  # bytes per pair: plsvo_camera, four doubles, int32


def fleet(pkg, synth, k, rng):
    """k cameras of 752x480, the even ones pinhole and the odd ones ATAN."""
    w, h, fx, fy, cx, cy, d0 = STOCK
    p = lambda v, s: v * (1.0 + rng.uniform(-s, s))  # noqa: E731
    out = []
    for i in range(k):
        if i % 2 == 0:
            f = rng.uniform(400.0, 480.0)
            out.append(synth.Camera(w, h, f, f * rng.uniform(0.98, 1.02), p(375.5, 0.02), p(239.5, 0.02)))
        else:
            out.append(pkg.ATANCamera(w, h, p(fx, 0.02), p(fy, 0.02), p(cx, 0.02), p(cy, 0.02), p(d0, 0.05)))
    return out


def same(a, b, fields):
    return all(np.array_equal(np.asarray(getattr(a, f)).view(np.uint8), np.asarray(getattr(b, f)).view(np.uint8)) for f in fields)


def scatter(outs, index, B, fields):
    class R:
        pass

    r = R()
    for f in fields:
        v0 = getattr(outs[0], f)
        full = np.empty((B,) + v0.shape[1:], v0.dtype)
        for o, idx in zip(outs, index):
            full[idx] = getattr(o, f)
        setattr(r, f, full)
    return r


def alternating(fns, reps, warmup):
    """median seconds of every fn over `reps` rounds, the fns called in turn within each round"""
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    ts = {n: [] for n in fns}
    for _ in range(reps):
        for n, fn in fns.items():
            t0 = time.perf_counter()
            fn()
            ts[n].append(time.perf_counter() - t0)
    return {n: float(np.median(v)) for n, v in ts.items()}


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
    rng = np.random.default_rng(9500)
    res = {"workload": f"B={B} pairs in a 752x480 slot, 300 points + 80 segments, levels 4->2, half pinhole and half ATAN",
           "card": card()}
    names = ["sparse_img_align", "pose_optimizer"]
    sia = pkg.SparseImgAlign(4, 2, 30)

    def pin_kw(cams, cop):
        return dict(cameras=np.array([[cams[k].fx, cams[k].fy, cams[k].cx, cams[k].cy] for k in cop]),
                    sizes=np.array([[cams[k].width, cams[k].height] for k in cop], np.int32))

    for k in (int(s) for s in args.ks.split(",")):
        cams = fleet(pkg, synth, k, rng)
        cop = (np.arange(B) % k).astype(np.int32)
        data, po, _, _, _ = synth.make_any_camera_batch(cams, cop, poseopt=True, n_pts=300, n_segs=80, seed=9600 + k, device="cuda")
        pin = np.array([isinstance(cams[c], synth.Camera) for c in cop])
        index = [np.flatnonzero(pin), np.flatnonzero(~pin)]
        subs = [synth.take_pairs(data, idx) for idx in index]
        po_subs = [synth.take_pairs(po, idx) for idx in index]
        atan_ids = sorted({int(c) for c in cop[index[1]]})
        atan_kw = dict(camera=[cams[c] for c in atan_ids], cam_of_pair=np.array([atan_ids.index(c) for c in cop[index[1]]], np.int32))
        pkw = pin_kw(cams, cop[index[0]])

        def track_two_calls(subs, po_subs, pkw, atan_kw):
            outs = (pkg.api.track(subs[0], po_subs[0], **pkw), pkg.api.track(subs[1], po_subs[1], **atan_kw))
            return [scatter([o[j] for o in outs], index, B, f) for j, f in ((0, ALIGN_FIELDS), (1, PO_FIELDS))]

        runs = {
            "align_any_call": lambda: sia.run(data, camera=cams, cam_of_pair=cop),
            "align_two_calls": lambda: scatter([sia.run(subs[0], **pkw), sia.run(subs[1], **atan_kw)], index, B, ALIGN_FIELDS),
            "track_any_call": lambda: pkg.api.track(data, po, camera=cams, cam_of_pair=cop),
            "track_two_calls": lambda: track_two_calls(subs, po_subs, pkw, atan_kw),
        }
        med = alternating(runs, args.reps, args.warmup)
        n_pin, n_atan = len(index[0]), len(index[1])
        h2d = {"any_call": B * (REC + TERMS + TAG), "two_calls": n_pin * REC + n_atan * (REC + TERMS)}
        ref_a, ref_t = runs["align_any_call"](), runs["track_any_call"]()
        equal = {"align_two_calls": same(runs["align_two_calls"](), ref_a, ALIGN_FIELDS)}
        tt = runs["track_two_calls"]()
        equal["track_two_calls"] = same(tt[0], ref_t[0], ALIGN_FIELDS) and same(tt[1], ref_t[1], PO_FIELDS)
        out = {}
        for name, fn in runs.items():
            kms = kernel_ms(fn, names)
            out[name] = {"pairs_per_s": round(B / med[name], 1), "kernel_ms": {n: round(v, 3) for n, v in kms.items() if v},
                         "camera_h2d_bytes": h2d[name.split("_", 1)[1]]}
            if name in equal:
                out[name]["equal"] = equal[name]
        res[f"K={k}"] = out

    # K = 1 of each model: the any-camera kernel against its single-model twin on the same batch
    for model in ("pinhole", "atan"):
        cam = fleet(pkg, synth, 2, rng)[0 if model == "pinhole" else 1]
        cop = np.zeros(B, np.int32)
        data = synth.make_any_camera_batch([cam], cop, n_pts=300, n_segs=80, seed=9700, device="cuda")[0]
        twin = (lambda: sia.run(data, **pin_kw([cam], cop))) if model == "pinhole" else (lambda: sia.run(data, camera=[cam], cam_of_pair=cop))
        # a one-camera table of one model takes the single-model path in the API: call the any-camera entry point itself
        table = pkg.abi.make_match_cameras([cam])

        def any_call():
            batch, keep = pkg.abi.make_align_batch(data)
            out = pkg.abi.AlignOut(data.batch, data.n_segs)
            sia.ctx.check(sia.ctx.lib.plsvo_align_any_camera_batch_run(sia.ctx.handle, table, 1, cop.ctypes.data_as(
                pkg.abi.C.POINTER(pkg.abi.C.c_int32)), pkg.abi.C.byref(batch), pkg.abi.C.byref(sia.params),
                pkg.abi.C.byref(out.struct)), "plsvo_align_any_camera_batch_run")
            return out

        arms = {"any_call": any_call, "single_model_call": twin}
        med = alternating(arms, args.reps, args.warmup)
        out = {n: {"pairs_per_s": round(B / med[n], 1), "kernel_ms": {m: round(v, 3) for m, v in kernel_ms(fn, names).items() if v}}
               for n, fn in arms.items()}
        out["single_model_call"]["equal"] = same(twin(), any_call(), ALIGN_FIELDS)
        res[f"K=1 {model}"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
