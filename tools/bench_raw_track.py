#!/usr/bin/env python
"""Measurement of alignment and tracking from raw (distorted) frames on one GPU: plsvo_align_raw_batch_run and
plsvo_track_raw_batch_run against the two ways a caller with a real lens had before them.

Workload: B = 1024 pairs of the EuRoC camera (752x480, config/dataset_params.yaml) as one frame chain of 1025 raw frames
rendered through the lens (synth.make_raw_chain_batch), 300 points + 80 segments per pair, levels 4 -> 2.  It prints one
JSON line with:
  raw_align / raw_track   : end-to-end pairs/s of the one-call raw entry points, raw frames in pageable and in pinned
                            (plsvo_host_alloc) host memory; `copy_ms` is the host->device time of the raw stack alone at
                            the pinned rate measured in the same run, `copy_share` its share of the pinned call
  host_oracle_then_align  : (a) the C++ oracle's undistortion + pyramid on every host thread, then plsvo_align_batch_run
                            shipping level 2 only (levels 3, 4 derived on the device)
  device_roundtrip_align  : (b) plsvo_undistort_batch_run (levels 0..2 back to the host), then plsvo_align_batch_run
                            shipping level 2 only
  kernels                 : device time (torch.profiler) of undistort_pyramid_kernel for levels 2..4 against
                            undistort_remap_kernel + pyramid_kernel for levels 0..4, and the fused kernel's HBM bytes
                            (raw frames read, the map once, levels 2..4 written) per second against 3.35 TB/s
  h2d_peak                : tools/h2d_peak.py's pinned host->device rates of this box
The card's name and power limit are read in the same run.  Needs a GPU.

usage: python tools/bench_raw_track.py [--batch 1024] [--reps 10] [--warmup 2]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
HBM_BPS = 3.35e12


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True, timeout=30)
        name, power = (s.strip() for s in q.strip().splitlines()[0].split(","))
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"name": "unknown", "power_limit": f"not read ({type(e).__name__})"}


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), float(min(ts))


def kernel_ms(fn, names):
    """Device time of the kernels whose names contain one of `names`, summed over one call of fn (torch.profiler)."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        for n in names:
            if n in ev.name:
                out[n] += ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_raw_track: no CUDA device (this measurement has no CPU fallback)")
    import oracle_lib
    import plsvo_b200
    import undistort_oracle
    from plsvo_b200 import abi, synth

    B = args.batch
    data, raw = synth.make_raw_chain_batch(batch=B, n_pts=300, n_segs=80, seed=5150, device="cuda")
    po = synth.make_poseopt_batch(cam=data.cam, batch=B, n_pts=300, n_segs=80, seed=5151, T_gt=data.T_cur_w_gt)
    cam = plsvo_b200.PinholeCamera(data.cam.width, data.cam.height, data.cam.fx, data.cam.fy, data.cam.cx, data.cam.cy, *synth.EUROC_DIST)
    W, H = data.cam.width, data.cam.height
    ctx = plsvo_b200.api.Context(0)
    al = plsvo_b200.SparseImgAlign(4, 2, 30, ctx=ctx)
    rows = {"workload": {"batch": B, "frames": B + 1, "camera": f"{W}x{H} EuRoC", "n_pts": 300, "n_segs": 80, "levels": "4->2"}}

    # pinned copy of the raw stack
    p = C.c_void_p()
    ctx.check(ctx.lib.plsvo_host_alloc(C.byref(p), raw.nbytes), "plsvo_host_alloc")
    pinned = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(raw.nbytes,)).reshape(raw.shape)
    pinned[...] = raw
    first = al.run_raw(cam, raw, data)
    assert all(np.array_equal(getattr(first, f), getattr(al.run_raw(cam, pinned, data), f)) for f in ("T_cur_w", "n_tracked", "iters"))
    for what, fn in (("raw_align", lambda r: al.run_raw(cam, r, data)),
                     ("raw_track", lambda r: plsvo_b200.track_raw(cam, r, data, po, ctx=ctx))):
        med_pg, _ = timed(lambda: fn(raw), args.reps, args.warmup)
        med_pn, _ = timed(lambda: fn(pinned), args.reps, args.warmup)
        rows[what] = {"pageable_pairs_per_s": B / med_pg, "pinned_pairs_per_s": B / med_pn, "pageable_ms": 1e3 * med_pg,
                      "pinned_ms": 1e3 * med_pn, "kernel_ms": ctx.last_kernel_ms()}
    # pinned H2D rate of the raw stack alone
    d = torch.empty(raw.nbytes, dtype=torch.uint8, device="cuda")
    h = torch.from_numpy(pinned.reshape(-1))
    for _ in range(3):
        d.copy_(h, non_blocking=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(5):
        d.copy_(h, non_blocking=True)
    torch.cuda.synchronize()
    copy_ms = 1e3 * (time.perf_counter() - t0) / 5
    for what in ("raw_align", "raw_track"):
        rows[what]["copy_ms"] = copy_ms
        rows[what]["copy_share_of_pinned_call"] = copy_ms / rows[what]["pinned_ms"]

    # (a) C++ oracle undistortion + pyramid on every host thread, then alignment shipping level 2 only
    olib = oracle_lib.load(abi)
    olib.plsvo_oracle_pyramid_batch.restype = C.c_int
    olib.plsvo_oracle_pyramid_batch.argtypes = [C.POINTER(abi.PyramidBatch), C.POINTER(abi.PyramidResult), C.c_int]
    n_threads = max(1, olib.plsvo_oracle_hardware_threads())
    maps = undistort_oracle.undistort_map(abi, cam.struct)
    ulib = undistort_oracle.load(abi)
    n = B + 1
    levels, r = abi.pyramid_levels(n, H, W, 3)
    ub = abi.UndistortBatch(cam.struct, n, 1, raw.ctypes.data_as(C.POINTER(C.c_uint8)), raw.strides[1], raw.strides[0])
    pb = abi.PyramidBatch(n, W, H, 3, levels[0].ctypes.data_as(C.POINTER(C.c_uint8)), levels[0].strides[1], levels[0].strides[0])
    import dataclasses

    def host_oracle():
        ulib.plsvo_oracle_undistort_frames(C.byref(ub), maps[0].ctypes.data_as(C.POINTER(C.c_int16)),
                                           maps[1].ctypes.data_as(C.POINTER(C.c_uint16)), C.byref(r), n_threads)
        olib.plsvo_oracle_pyramid_batch(C.byref(pb), C.byref(r), n_threads)
        return al.run(dataclasses.replace(data, ref_pyr={}, cur_pyr={}, frame_pyr={2: levels[2]}))

    med, _ = timed(host_oracle, max(2, args.reps // 3), 1)
    rows["host_oracle_then_align"] = {"pairs_per_s": B / med, "ms": 1e3 * med, "cpu_threads": n_threads}

    # (b) device rectification round trip, then alignment shipping level 2 only
    def roundtrip():
        lv = cam.undistortImage(raw, 3, ctx)
        return al.run(dataclasses.replace(data, ref_pyr={}, cur_pyr={}, frame_pyr={2: lv[2]}))

    med, _ = timed(roundtrip, args.reps, args.warmup)
    rows["device_roundtrip_align"] = {"pairs_per_s": B / med, "ms": 1e3 * med}

    # kernels
    fused = kernel_ms(lambda: al.run_raw(cam, raw, data), ["undistort_pyramid_kernel"])["undistort_pyramid_kernel"]
    two = kernel_ms(lambda: cam.undistortImage(raw, 5, ctx), ["undistort_remap_kernel", "pyramid_kernel"])
    fused_bytes = raw.nbytes + W * H * 6 + n * sum(((W >> l) + 15) // 16 * 16 * (H >> l) for l in (2, 3, 4))
    rows["kernels"] = {"fused_levels_2_4_ms": fused, "remap_ms": two["undistort_remap_kernel"],
                       "pyramid_levels_0_4_ms": two["pyramid_kernel"],
                       "fused_hbm_bytes": fused_bytes, "fused_bytes_per_s": fused_bytes / (fused * 1e-3),
                       "fused_share_of_3_35_TBps": fused_bytes / (fused * 1e-3) / HBM_BPS}
    ctx.lib.plsvo_host_free(p)
    ctx.close()
    try:
        out = subprocess.check_output([sys.executable, os.path.join(ROOT, "tools", "h2d_peak.py")], text=True, timeout=300)
        rows["h2d_peak"] = json.loads(out.strip().splitlines()[-1])
    except Exception as e:  # noqa: BLE001
        rows["h2d_peak"] = f"not measured ({type(e).__name__})"
    print(json.dumps({"bench": "raw_track", "card": card(), **rows}))


if __name__ == "__main__":
    main()
