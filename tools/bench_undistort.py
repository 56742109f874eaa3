#!/usr/bin/env python
"""Measurement of PinholeCamera.undistortImage (plsvo_undistort_batch_run) on one GPU: B raw u8 frames -> rectified level 0
(cv::remap INTER_LINEAR with the camera's CV_16SC2 map) -> n_levels-deep pyramid, host in, host out.

Workloads: B = 256 frames of the EuRoC-style 752x480 camera of the reference's config/dataset_params.yaml and of a 720p
camera, each with n_levels = 1 (rectification alone) and 5 (the reference's pyramid depth).  Per workload it prints:
  e2e_frames_per_s : frames over the wall time of the synchronous call (uploads, kernels, downloads), map cached
  kernel_ms        : median device time of the remap + pyramid kernels (plsvo_last_kernel_ms), map cached
  map_build_ms     : device time of the one-off map build (first call on a fresh context)
  bytes            : bytes the kernels must move, from shapes: raw frames read + level 0 written by the remap, the
                     map's 6 B per pixel read once, level 0 read again + levels 1.. written by the pyramid kernel
  bytes_per_s, share_of_3_35_TBps : bytes over kernel_ms, against the H100 SXM data-sheet HBM3 bandwidth
  cpu_oracle_frames_per_s : the C++ oracle (oracle/undistort_oracle.cpp + plsvo_oracle.cpp's pyramid) on every host
                            thread, map prebuilt
  cpu_cv2_frames_per_s    : cv2.remap per frame + the oracle's pyramid on every host thread (only when cv2 imports)
The card's name and power limit are read in the same run.  Needs a GPU; prints one JSON line.

usage: python tools/bench_undistort.py [--batch 256] [--reps 20] [--warmup 3]"""
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

CAMERAS = {
    "752x480": (752, 480, 416.401549, 416.375319, 385.554786, 237.640332, -0.277970, 0.060647, -0.002097, 0.000373, 0.0),
    "1280x720": (1280, 720, 700.3, 699.8, 641.2, 362.9, -0.31, 0.11, 0.0006, -0.0004, -0.018),
}
HBM_BPS = 3.35e12


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True, timeout=30)
        name, power = (s.strip() for s in q.strip().splitlines()[0].split(","))
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"name": "unknown", "power_limit": f"not read ({type(e).__name__})"}


def level_bytes(W, H, n_levels):
    return sum((W >> l) * (H >> l) for l in range(n_levels))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-reps", type=int, default=3)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_undistort: no CUDA device (this measurement has no CPU fallback)")
    import plsvo_b200
    import oracle_lib
    import undistort_oracle
    from plsvo_b200 import abi

    olib = oracle_lib.load(abi)
    olib.plsvo_oracle_pyramid_batch.restype = C.c_int
    olib.plsvo_oracle_pyramid_batch.argtypes = [C.POINTER(abi.PyramidBatch), C.POINTER(abi.PyramidResult), C.c_int]
    n_threads = max(1, olib.plsvo_oracle_hardware_threads())
    try:
        import cv2
    except ImportError:
        cv2 = None
    B = args.batch
    rows = []
    for cam_name, p in CAMERAS.items():
        W, H = p[:2]
        raw = np.random.default_rng(7).integers(0, 256, (B, H, W), np.uint8)
        cam_s = abi.PinholeCamera(W, H, *p[2:6], (C.c_double * 5)(*p[6:]))
        maps = undistort_oracle.undistort_map(abi, cam_s)
        for n_levels in (1, 5):
            ctx = plsvo_b200.api.Context(0)
            cam = plsvo_b200.PinholeCamera(*p)
            first = cam.undistortImage(raw, n_levels, ctx)
            map_ms = ctx.last_map_build_ms()
            want = undistort_oracle.undistort(abi, cam_s, np.ascontiguousarray(raw[:4]), n_levels, n_threads=n_threads, maps=maps)
            exact = all(np.array_equal(first[l][:4], want[l]) for l in range(n_levels))
            for _ in range(args.warmup):
                cam.undistortImage(raw, n_levels, ctx)
            walls, kms = [], []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                cam.undistortImage(raw, n_levels, ctx)
                walls.append(time.perf_counter() - t0)
                kms.append(ctx.last_kernel_ms())
                assert ctx.last_map_build_ms() is None
            ctx.close()
            k_ms = float(np.median(kms))
            nbytes = B * W * H * 2 + W * H * 6 + (B * level_bytes(W, H, n_levels) if n_levels > 1 else 0)
            row = {"camera": cam_name, "batch": B, "n_levels": n_levels, "bit_exact_first_4_frames": exact,
                   "e2e_frames_per_s": B / float(np.median(walls)), "e2e_ms_median": 1e3 * float(np.median(walls)),
                   "kernel_ms": k_ms, "map_build_ms": map_ms, "bytes": nbytes, "bytes_per_s": nbytes / (k_ms * 1e-3),
                   "share_of_3_35_TBps": nbytes / (k_ms * 1e-3) / HBM_BPS}
            # CPU arms: the C++ oracle (map prebuilt, as vikit builds it once), and cv2.remap, each followed by the oracle's
            # pyramid on every host thread
            levels, r = abi.pyramid_levels(B, H, W, n_levels)
            pb = abi.PyramidBatch(B, W, H, n_levels, levels[0].ctypes.data_as(C.POINTER(C.c_uint8)), levels[0].strides[1],
                                  levels[0].strides[0])
            ub = abi.UndistortBatch(cam_s, B, 1, raw.ctypes.data_as(C.POINTER(C.c_uint8)), raw.strides[1], raw.strides[0])
            ulib = undistort_oracle.load(abi)
            ts = []
            for _ in range(args.cpu_reps):
                t0 = time.perf_counter()
                ulib.plsvo_oracle_undistort_frames(C.byref(ub), maps[0].ctypes.data_as(C.POINTER(C.c_int16)),
                                                   maps[1].ctypes.data_as(C.POINTER(C.c_uint16)), C.byref(r), n_threads)
                if n_levels > 1:
                    olib.plsvo_oracle_pyramid_batch(C.byref(pb), C.byref(r), n_threads)
                ts.append(time.perf_counter() - t0)
            row["cpu_oracle_frames_per_s"] = B / min(ts)
            row["cpu_threads"] = n_threads
            if cv2 is not None:
                m1, m2 = maps
                ts = []
                for _ in range(args.cpu_reps):
                    t0 = time.perf_counter()
                    for b in range(B):
                        cv2.remap(raw[b], m1, m2, cv2.INTER_LINEAR, dst=levels[0][b])
                    if n_levels > 1:
                        olib.plsvo_oracle_pyramid_batch(C.byref(pb), C.byref(r), n_threads)
                    ts.append(time.perf_counter() - t0)
                row["cpu_cv2_frames_per_s"] = B / min(ts)
                row["cv2_threads"] = cv2.getNumThreads()
            else:
                row["cpu_cv2_frames_per_s"] = "not measured (cv2 not importable)"
            rows.append(row)
    print(json.dumps({"bench": "undistort", "card": card(), "workloads": rows}))


if __name__ == "__main__":
    main()
