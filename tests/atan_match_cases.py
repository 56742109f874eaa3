"""Cameras and candidate batches of the ATAN (FOV) findMatchDirect tests (tests/test_atan_match_cpu.py on the CPU,
tests/test_gpu_atan_match.py on the device).

A case is synth.make_match_batch(atan=camera) with rows overwritten by edge cases: the in-frame border (b = 6) at every
reference level on both sides, NaN warps, search levels clamped at n_pyr_levels - 1, edgelets with zero and
axis-aligned gradients, current frames rolled 45 and 135 degrees about the optical axis, and rows around the principal
point of an unmoved current frame, whose cam2world arguments fall inside r_d <= 0.01 and whose world2cam arguments fall
inside r < 0.001, so that both distortion cut-offs are reached from both sides."""
from __future__ import annotations

import math
from dataclasses import replace

import numpy as np
import torch


def camera(pkg, synth, size: str, d0: float):
    """The ATAN camera of synth's pinhole `size` (VGA, EUROC, ...) with distortion d0: fx_ = w fx, cx_ = w cx - 0.5."""
    c = getattr(synth, size)
    w, h = c.width, c.height
    return pkg.ATANCamera(w, h, c.fx / w, c.fy / h, (c.cx + 0.5) / w, (c.cy + 0.5) / h, d0)


def off_centre(pkg, d0: float = 0.93):
    """752x480 with fx_ != fy_ and the principal point away from the centre."""
    return pkg.ATANCamera(752, 480, 438.06 / 752, 384.0 / 480, 0.56, 0.43, d0)


def telephoto(pkg, d0: float = 0.93):
    """VGA with fx_ = fy_ = 6400: every ray lies within 0.07 of the axis, and the cut-off discs have radii of 64 px
    (cam2world) and 6.4 px (world2cam).  Only such a camera has candidates inside both: the du / dv samples of the warp
    lie 5 * 2^l px apart from the reference pixel, so with the pixel at -(2.5, 2.5) * 2^l from the principal point all three
    projections stay within 3.6 * 2^l px of it."""
    return pkg.ATANCamera(640, 480, 10.0, 6400.0 / 480, 0.5, 0.5, d0)


def pinhole_of(synth, cam):
    """The undistorted pinhole whose intrinsics are the ATAN camera's members."""
    return synth.Camera(cam.width, cam.height, cam.fx_, cam.fy_, cam.cx_, cam.cy_)


def with_camera(d, pin):
    return replace(d, cam=pin)


def _render_frames(synth, d, cam, which, T7):
    pose_attr, pyr_attr = ("T_ref_w", "ref_pyr") if which == "ref" else ("T_cur_w", "cur_pyr")
    T7 = np.ascontiguousarray(T7, np.float64)
    img = synth.Scene().render(d.cam, torch.tensor(T7), atan=cam)
    levels = synth.build_pyramid(img, max(getattr(d, pyr_attr)) + 1)
    pyr = getattr(d, pyr_attr)
    for l in pyr:
        pyr[l] = np.ascontiguousarray(np.concatenate([pyr[l], levels[l].numpy()]))
    first = getattr(d, pose_attr).shape[0]
    setattr(d, pose_attr, np.ascontiguousarray(np.concatenate([getattr(d, pose_attr), T7])))
    return first


def _Rt(synth, T7):
    R, t = synth.pose7_to_Rt(torch.tensor(np.asarray(T7, np.float64).reshape(-1, 7)))
    return R[0].numpy(), t[0].numpy()


def case(pkg, synth, cam, n: int = 1200, n_pyr_levels: int = 4, seed: int = 7600, rows: bool = True):
    """A candidate batch seen through `cam`, with the edge rows of the module docstring written over its first rows."""
    pin = pinhole_of(synth, cam)
    d = synth.make_match_batch(cam=pin, n=n, seed=seed, n_pyr_levels=n_pyr_levels, atan=cam)
    if rows:
        _edge_rows(synth, d, cam, np.random.default_rng(seed))
    return d


def _edge_rows(synth, d, cam, rng):
    W0, H0, L = d.cam.width, d.cam.height, d.n_pyr_levels
    r = 0

    def put(ref_px=None, level=None, **kw):
        nonlocal r
        assert r < d.n, "the batch is too small for its edge rows"
        if ref_px is not None:
            d.ref_px[r] = ref_px
            d.ref_f[r] = cam.cam2world(np.asarray(ref_px, np.float64))
        if level is not None:
            d.ref_level[r] = level
        for k, v in kw.items():
            getattr(d, k)[r] = v
        r += 1

    # the in-frame border (b = 6) at every reference level, both sides
    for l in range(L):
        s, W, H = 1 << l, W0 >> l, H0 >> l
        for o in (5, 6, W - 7, W - 6):
            put(((o + 0.5) * s, H0 / 2), l)
        for o in (5, 6, H - 7, H - 6):
            put((W0 / 2, (o + 0.5) * s), l)
    # NaN warps: a point at the centre of an identity reference frame (depth exactly 0) and a NaN point
    R0, t0 = _Rt(synth, d.T_ref_w[0])
    ident = _render_frames(synth, d, cam, "ref", [[0, 0, 0, 1, 0, 0, 0]])
    for k in range(2):
        put((W0 / 2 + 7 * k, H0 / 2), 0, ref_index=ident, pos=(0.0, 0.0, 0.0), is_edgelet=k)
        put(None, None, pos=(math.nan, 1.0, 2.0), is_edgelet=k)
    # a current frame 1 mm in front of a point 1 m ahead of the identity reference frame: the search level is clamped
    close = _render_frames(synth, d, cam, "cur", [[0, 0, 0, 1, 0, 0, -0.999]])
    for e in (0, 1):
        put((cam.cx_, cam.cy_), 0, ref_index=ident, cur_index=close, pos=(0.0, 0.0, 1.0), px_cur=(cam.cx_ + 0.3, cam.cy_ - 0.2), is_edgelet=e)
    # edgelets with zero and axis-aligned gradients
    for g in ((0.0, 0.0), (1.0, 0.0), (0.0, 1.0), (-0.0, -1.0)):
        for _ in range(2):
            put(None, None, is_edgelet=1, ref_grad=g)
    # current frames rolled 45 and 135 degrees about the optical axis of reference frame 0, candidates at the in-frame
    # border of every level (their warped 10x10 sample reaches outside the reference level)
    for ang in (math.pi / 4, 3 * math.pi / 4):
        c, s_ = math.cos(ang), math.sin(ang)
        Rz = np.array([[c, -s_, 0.0], [s_, c, 0.0], [0.0, 0.0, 1.0]])
        rolled = _render_frames(synth, d, cam, "cur", _pose7(synth, Rz @ R0, Rz @ t0))
        for l in range(L):
            sc, W, H = 1 << l, W0 >> l, H0 >> l
            if W - 7 < 6 or H - 7 < 6:
                continue
            for ox, oy in ((6, H // 2), (W - 7, H // 2), (W // 2, 6), (W // 2, H - 7)):
                p = np.array([(ox + 0.5) * sc, (oy + 0.5) * sc])
                q = p - (cam.cx_, cam.cy_)
                pc = np.array([c * q[0] - s_ * q[1], s_ * q[0] + c * q[1]]) + (cam.cx_, cam.cy_) + rng.uniform(-1, 1, 2)
                for e in (0, 1):
                    put(p, l, ref_index=0, cur_index=rolled, px_cur=pc, is_edgelet=e, pos=_on_ray(cam, R0, t0, p, 2.0))
    # both cut-offs from both sides: an unmoved current frame (reference frame 0's pose) and reference pixels around the
    # principal point and 5 * 2^l px left of / above it (where the du / dv samples of the warp fall on it)
    still = _render_frames(synth, d, cam, "cur", d.T_ref_w[:1])
    for l in range(min(L, 3)):
        st = 5.0 * (1 << l)
        for base in ((cam.cx_, cam.cy_), (cam.cx_ - st, cam.cy_), (cam.cx_, cam.cy_ - st), (cam.cx_ - st / 2, cam.cy_ - st / 2)):
            for off in ((0.0, 0.0), (0.2, -0.1), (1.5, 0.5), (-3.0, 2.0), (0.01 * cam.fx_ + 0.5, 0.0), (0.0, 0.01 * cam.fy_ - 0.5)):
                p = np.array(base) + off
                put(p, l, ref_index=0, cur_index=still, px_cur=p + rng.uniform(-0.5, 0.5, 2), is_edgelet=r % 2,
                    pos=_on_ray(cam, R0, t0, p, 1.5))
    return r


def _pose7(synth, R, t):
    return synth.pose7_from_Rt(torch.tensor(R[None]), torch.tensor(t[None])).numpy()


def _on_ray(cam, R, t, px, depth):
    """The world point at `depth` along the ATAN ray of pixel px of the frame T_f_w = (R, t)."""
    f = cam.cam2world(np.asarray(px, np.float64))
    return R.T @ (f * depth - t)


def cut_off_arguments(cam, d):
    """The arguments of the five camera calls of each row's warp matrix, in float64 NumPy (close to, not bit-equal with,
    the oracle's): r_d of the two cam2world calls [n, 2] and r of the three world2cam calls [n, 3]."""
    n = d.n
    lvl = (1 << d.ref_level.astype(np.int64)).astype(np.float64)
    du = d.ref_px + np.stack([5 * lvl, 0 * lvl], -1)
    dv = d.ref_px + np.stack([0 * lvl, 5 * lvl], -1)
    rd = np.stack([np.hypot((p[:, 0] - cam.cx_) / cam.fx_, (p[:, 1] - cam.cy_) / cam.fy_) for p in (du, dv)], -1)
    r = np.full((n, 3), np.nan)
    Rr, tr = _Rts(d.T_ref_w)
    Rc, tc = _Rts(d.T_cur_w)
    for i in range(n):
        R0, t0 = Rr[d.ref_index[i]], tr[d.ref_index[i]]
        R1, t1 = Rc[d.cur_index[i]], tc[d.cur_index[i]]
        depth = np.linalg.norm(-R0.T @ t0 - d.pos[i])
        xyz = d.ref_f[i] * depth
        pts = [xyz]
        for p in (du[i], dv[i]):
            f = cam.cam2world(p)
            pts.append(f * (xyz[2] / f[2]))
        R, t = R1 @ R0.T, t1 - R1 @ R0.T @ t0
        for k, p in enumerate(pts):
            q = R @ p + t
            r[i, k] = math.hypot(q[0] / q[2], q[1] / q[2])
    return rd, r


def _Rts(T7):
    R, t = [], []
    for T in T7:
        a, b = _Rt_np(T)
        R.append(a), t.append(b)
    return R, t


def _Rt_np(T):
    x, y, z, w = T[:4] / np.linalg.norm(T[:4])
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    return R, np.asarray(T[4:7], np.float64)


def transcendental_free(cam, d, margin: float = 0.98):
    """Rows whose five camera calls stay inside both cut-offs with a margin, so that neither tan nor atan is evaluated:
    every cam2world argument r_d <= 0.01 and every world2cam argument r < 0.001 (or d0 == 0: no row calls either)."""
    if cam.s_ == 0.0:
        return np.ones(d.n, bool)
    rd, r = cut_off_arguments(cam, d)
    return (rd <= 0.01 * margin).all(-1) & (r < 0.001 * margin).all(-1)
