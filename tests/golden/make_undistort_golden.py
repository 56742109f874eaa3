"""Generates tests/golden/undistort_cv2.json: for each test camera of tests/test_undistort.py, the sha256 digests of what
OpenCV computes for vk::PinholeCamera::undistortImage — cv::initUndistortRectifyMap(K, D, I, K, size, CV_16SC2) with K
and D as float matrices, as rpg_vikit's constructor builds them, and cv::remap(raw, rect, map1, map2, INTER_LINEAR) of a
seeded random frame.  The cameras and the frame recipe are stored beside the digests, so the restatements can be
checked against OpenCV where cv2 is not installed.  Needs cv2; run from the repo root:
    python tests/golden/make_undistort_golden.py
"""
import hashlib
import json
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# name -> (width, height, fx, fy, cx, cy, d0, d1, d2, d3, d4)
CAMERAS = {
    "euroc_dataset_params": (752, 480, 416.401549, 416.375319, 385.554786, 237.640332, -0.277970, 0.060647, -0.002097, 0.000373, 0.0),
    "vga_strong_barrel_k3": (640, 480, 420.0, 421.5, 318.2, 241.7, -0.42, 0.21, 0.0, 0.0, -0.06),
    "vga_pincushion": (640, 480, 300.0, 300.0, 320.0, 240.0, 0.9, 0.6, 0.0, 0.0, 0.3),
    "vga_tangential_only": (640, 480, 500.0, 500.0, 319.5, 239.5, 1e-6, 0.0, 0.004, -0.003, 0.0),
    "vga_d0_zero_is_a_copy": (640, 480, 500.0, 500.0, 319.5, 239.5, 0.0, 0.2, 0.001, 0.001, 0.05),
    "hd720": (1280, 720, 700.3, 699.8, 641.2, 362.9, -0.31, 0.11, 0.0006, -0.0004, -0.018),
    "odd_641x479": (641, 479, 390.7, 388.1, 320.3, 238.9, -0.25, 0.07, 0.001, 0.0005, 0.0),
}
FRAME_SEED = 9100  # frame of camera k: np.random.default_rng(FRAME_SEED + k).integers(0, 256, (H, W), np.uint8)


def frame(k, width, height):
    return np.random.default_rng(FRAME_SEED + k).integers(0, 256, (height, width), np.uint8)


def digest(a) -> str:
    a = np.ascontiguousarray(a)
    return hashlib.sha256(f"{a.dtype.str}{a.shape}".encode() + a.tobytes()).hexdigest()


def main():
    out = {"opencv": cv2.__version__, "frame_seed": FRAME_SEED, "cameras": {}}
    for k, (name, cam) in enumerate(CAMERAS.items()):
        W, H, fx, fy, cx, cy, *d = cam
        img = frame(k, W, H)
        entry = {"params": list(cam), "index": k}
        if abs(d[0]) > 1e-7:
            K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
            map1, map2 = cv2.initUndistortRectifyMap(K, np.array(d, np.float32), np.eye(3), K, (W, H), cv2.CV_16SC2)
            entry.update(map1=digest(map1), map2=digest(map2), image=digest(cv2.remap(img, map1, map2, cv2.INTER_LINEAR)))
        else:  # vikit: undistortImage is raw.clone()
            entry.update(image=digest(img))
        out["cameras"][name] = entry
    with open(os.path.join(HERE, "undistort_cv2.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
