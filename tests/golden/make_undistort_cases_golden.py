"""Generates the OpenCV fixtures of tests/test_gpu_undistort_cases.py, for machines without cv2:
  * tests/golden/undistort_cases_cv2.json: sha256 digests of cv2's map1, map2 and remapped frame for every in-range and
    tie camera of tests/undistort_cases.py at the sizes listed in the file;
  * tests/golden/undistort_cases_cv2.npz: cv2's map1 and map2 themselves for the out-of-range cameras at the small sizes
    (SMALL_OOR_SIZES) and the camera with infinite coordinates, where cv2 4.x does not follow one rule the test could
    recompute (it saturates in its vectorised columns and wraps in its scalar tail).
cv::initUndistortRectifyMap(K, D, I, K, size, CV_16SC2) with K and D as float matrices, as rpg_vikit's PinholeCamera
builds them, and cv::remap(raw, rect, map1, map2, INTER_LINEAR).  Needs cv2; run from the repo root:
    python tests/golden/make_undistort_cases_golden.py
"""
import hashlib
import json
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import undistort_cases as uc  # noqa: E402

FRAME_SEED = 9300  # frame of a camera at W x H: undistort_cases.frames(1, H, W, FRAME_SEED)[0]


def digest(a) -> str:
    a = np.ascontiguousarray(a)
    return hashlib.sha256(f"{a.dtype.str}{a.shape}".encode() + a.tobytes()).hexdigest()


def cv_map(p):
    W, H, fx, fy, cx, cy, *d = p
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    return cv2.initUndistortRectifyMap(K, np.array(d, np.float32), np.eye(3), K, (W, H), cv2.CV_16SC2)


def digest_cases():
    """name@WxH -> camera: the in-range cameras at DIGEST_SIZES and the tie cameras."""
    out = {f"{n}@{W}x{H}": p for W, H in uc.DIGEST_SIZES for n, p in uc.in_range(W, H).items()}
    out.update({f"{n}@640x480": p for n, p in uc.TIES.items()})
    return out


def map_cases():
    """name@WxH -> camera: the out-of-range cameras at SMALL_OOR_SIZES and the infinite one."""
    out = {f"{n}@{W}x{H}": p for W, H in uc.SMALL_OOR_SIZES for n, p in uc.out_of_range(W, H).items()}
    out["inf@64x48"] = uc.INF
    return out


def main():
    digests = {}
    for key, p in digest_cases().items():
        W, H = p[:2]
        img = uc.frames(1, H, W, FRAME_SEED)[0]
        if abs(p[6]) > 1e-7:
            map1, map2 = cv_map(p)
            digests[key] = {"map1": digest(map1), "map2": digest(map2), "image": digest(cv2.remap(img, map1, map2, cv2.INTER_LINEAR))}
        else:  # vikit: undistortImage is raw.clone()
            digests[key] = {"image": digest(img)}
    with open(os.path.join(HERE, "undistort_cases_cv2.json"), "w") as f:
        json.dump({"opencv": cv2.__version__, "frame_seed": FRAME_SEED, "digests": digests}, f, indent=1)
        f.write("\n")
    maps = {}
    for key, p in map_cases().items():
        maps[key + ":map1"], maps[key + ":map2"] = cv_map(p)
    np.savez_compressed(os.path.join(HERE, "undistort_cases_cv2.npz"), opencv=np.array(cv2.__version__), **maps)


if __name__ == "__main__":
    main()
