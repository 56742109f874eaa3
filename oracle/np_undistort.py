"""np_undistort.py — an INDEPENDENT NumPy restatement of vk::PinholeCamera::undistortImage (rpg_vikit pinhole_camera.cpp) =
cv::initUndistortRectifyMap once (constructor) + cv::remap(raw, rect, map1, map2, INTER_LINEAR) per frame (OpenCV 3.4
imgproc undistort.cpp / imgwarp.cpp, scalar paths).  TEST INFRASTRUCTURE ONLY.

Written separately from oracle/undistort_oracle.cpp: the row recurrence as np.add.accumulate (sequential along a row),
the polynomial and the remap vectorised over the image.  NumPy's float64 operations are IEEE without FMA contraction."""
from __future__ import annotations

import numpy as np


def undistort_is_copy(d0) -> bool:
    """PinholeCamera's distortion_ flag is fabs(d0) > 1e-7; without it undistortImage is raw.clone()."""
    return not abs(float(d0)) > 1e-7


def cv_round(t):
    """cvRound: round half to even; out of int range (or NaN) gives INT_MIN like cvtsd2si.  int64 array."""
    r = np.rint(t)
    ok = (r >= -2147483648.0) & (r <= 2147483647.0)
    return np.where(ok, np.where(ok, r, 0).astype(np.int64), -2147483648).astype(np.int64)


def map_of_rounded(iu, iv):
    """The CV_16SC2 map from cvRound(u * 32), cvRound(v * 32) as OpenCV's scalar loop stores it: map1 = the (short) casts
    of iu >> 5, iv >> 5 (wrapping), map2 = (iv & 31) * 32 + (iu & 31)."""
    map1 = np.stack([(iu >> 5).astype(np.int16), (iv >> 5).astype(np.int16)], -1)  # (short) cast: wraps like C
    map2 = ((iv & 31) * 32 + (iu & 31)).astype(np.uint16)
    return map1, map2


def undistort_map(width, height, fx, fy, cx, cy, d0=0.0, d1=0.0, d2=0.0, d3=0.0, d4=0.0):
    """cv::initUndistortRectifyMap(cvK_, cvD_, I, cvK_, size, CV_16SC2) -> (map1 int16 [H,W,2], map2 uint16 [H,W]).
    cvK_ / cvD_ are Mat_<float>: every parameter is rounded to float first."""
    u32, v32 = undistort_coords(width, height, fx, fy, cx, cy, d0, d1, d2, d3, d4)
    return map_of_rounded(cv_round(u32), cv_round(v32))


def undistort_coords(width, height, fx, fy, cx, cy, d0=0.0, d1=0.0, d2=0.0, d3=0.0, d4=0.0):
    """u * 32 and v * 32 (float64 [H,W]) of every map entry, the values cvRound rounds."""
    fx, fy, cx, cy, k1, k2, p1, p2, k3 = (float(np.float32(v)) for v in (fx, fy, cx, cy, d0, d1, d2, d3, d4))
    # iR = (K R).inv(DECOMP_LU): OpenCV's closed-form 3x3 inverse (cofactors times 1/det3) of K with R = I
    m = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])
    det = m[0, 0] * (m[1, 1] * m[2, 2] - m[1, 2] * m[2, 1]) - m[0, 1] * (m[1, 0] * m[2, 2] - m[1, 2] * m[2, 0]) \
        + m[0, 2] * (m[1, 0] * m[2, 1] - m[1, 1] * m[2, 0])
    d = 1.0 / det
    ir = np.array([(m[1, 1] * m[2, 2] - m[1, 2] * m[2, 1]) * d, (m[0, 2] * m[2, 1] - m[0, 1] * m[2, 2]) * d,
                   (m[0, 1] * m[1, 2] - m[0, 2] * m[1, 1]) * d, (m[1, 2] * m[2, 0] - m[1, 0] * m[2, 2]) * d,
                   (m[0, 0] * m[2, 2] - m[0, 2] * m[2, 0]) * d, (m[0, 2] * m[1, 0] - m[0, 0] * m[1, 2]) * d,
                   (m[1, 0] * m[2, 1] - m[1, 1] * m[2, 0]) * d, (m[0, 1] * m[2, 0] - m[0, 0] * m[2, 1]) * d,
                   (m[0, 0] * m[1, 1] - m[0, 1] * m[1, 0]) * d])
    i = np.arange(height, dtype=np.float64)[:, None]

    def row_walk(step, a, b):  # _x = i*a + b, then _x += step pixel by pixel along the row
        seq = np.empty((height, width))
        seq[:, :1] = i * a + b
        seq[:, 1:] = step
        return np.add.accumulate(seq, axis=1)

    _x, _y, _w = row_walk(ir[0], ir[1], ir[2]), row_walk(ir[3], ir[4], ir[5]), row_walk(ir[6], ir[7], ir[8])
    w = 1.0 / _w
    x, y = _x * w, _y * w
    x2, y2 = x * x, y * y
    r2 = x2 + y2
    _2xy = 2 * x * y
    kr = 1 + ((k3 * r2 + k2) * r2 + k1) * r2
    u = fx * (x * kr + p1 * _2xy + p2 * (r2 + 2 * x2)) + cx
    v = fy * (y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy) + cy
    return u * 32, v * 32


def remap_linear(img, map1, map2):
    """cv::remap(img, out, map1, map2, INTER_LINEAR, BORDER_CONSTANT, 0) for u8 [..., H, W]: fixed-point bilinear,
    (sum p*w + 2^14) >> 15 with the 1/32-step weights of the interpolation table ((32-a)(32-b)*32, ...)."""
    img = np.asarray(img, np.uint8)
    H, W = img.shape[-2:]
    sx, sy = map1[..., 0].astype(np.int64), map1[..., 1].astype(np.int64)
    a, b = (map2 & 31).astype(np.int64), (map2 >> 5).astype(np.int64)
    acc = np.zeros(img.shape[:-2] + map2.shape, np.int64)
    for dy, dx, wt in ((0, 0, (32 - a) * (32 - b)), (0, 1, a * (32 - b)), (1, 0, (32 - a) * b), (1, 1, a * b)):
        xx, yy = sx + dx, sy + dy
        inside = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
        p = img[..., np.where(inside, yy, 0), np.where(inside, xx, 0)].astype(np.int64) * inside
        acc += p * (wt * 32)
    return ((acc + (1 << 14)) >> 15).astype(np.uint8)


def undistort_image(raw, width, height, fx, fy, cx, cy, d0=0.0, d1=0.0, d2=0.0, d3=0.0, d4=0.0):
    """PinholeCamera(width, height, fx, fy, cx, cy, d0..d4).undistortImage for u8 [..., H, W]."""
    raw = np.asarray(raw, np.uint8)
    if undistort_is_copy(d0):
        return raw.copy()
    return remap_linear(raw, *undistort_map(width, height, fx, fy, cx, cy, d0, d1, d2, d3, d4))
