"""The direct-matching kernels (csrc/align2d_kernel.cu) against the CPU oracle, on the exits, borders, levels and layouts
where they can go wrong.

align2d_kernel and align1d_kernel run feature_alignment::align2D / align1D, one thread per feature; match_direct_kernel
runs Matcher::findMatchDirect (in-frame test, affine warp, search level, warped patch, align2D / align1D at the search
level).  All three are bit-identical to the oracle, so every output array is compared whole and byte for byte; only NaN
payloads are made alike first (the x86 and the CUDA default NaN differ in their sign bit), so the sign of an infinity or of
a zero is compared too.  The cases:

  * features, for levels 0-4 of VGA, EuRoC (752x480), 641x479 and HD720:
    - a border sweep: floor(u) in {3, 4, 5, cols-6, cols-5, cols-4} with fractional parts {0, ulp, 0.5, 1 - ulp} (ulp: the
      spacing of float at the coordinate, at least 2^-20), and the same for v;
    - walkers, whose true position lies 1-3 px outside a bound: their template comes from a copy of the image shifted by
      4 px, so the loop leaves the frame at iteration 1 or later, at each of the four bounds;
    - random interior features, which reach every byte offset (floor(u) - 4) mod 4 of the unaligned 9-byte window;
    - degenerate templates: constant, stripes in x only or in y only, 0/255 noise, a checkerboard, a ramp (a singular H in
      align2D); align1D directions (1,0), (0,1), (0,0), (3,4), (4,-3) and (0.8,-0.6) across the ramp, and subnormal
      (h_inv infinite);
    - align1D back-off ties new_chi2 == chi2 (a template whose LK step on a flat image leaves every residual as it was);
    - starting points NaN, +-inf, +-1e10 and -0.0 (x86 turns an out-of-range conversion into INT_MIN, CUDA saturates);
    - n_iter in {0, 1, 2, 3, 10, 30, 100};
  * batch sizes 1, 127, 128, 129 and 2^17 + 1 drawn from those features: a feature's bytes do not depend on where it sits;
  * findMatchDirect: n_pyr_levels 1-8 on the four cameras; align_max_iter in {0, 1, 3, 10, 30}; reference points on
    both sides of the in-frame border (b = 6) at every reference level; NaN warps (the point at the reference camera
    centre gives A = 0, and a NaN point); warped patches partly outside the reference image (a current frame rolled 45
    degrees about the optical axis), with samples exactly on the last column and on the last row at every level; edgelets with zero and axis-aligned gradients; 40 reference and 40 current frames;
    NULL is_edgelet / search_level / A_cur_ref; A_cur_ref prefilled with a sentinel, which rejected rows must return;
    n_pyr_levels = 9, refused with PLSVO_ERR_INVALID;
  * host layouts: pyramids with padded rows and pitch, every other frame of a stack (both take the per-image copy), and
    pyramids that supply level 3 only.

test_direct_match_cases_cover_every_exit (no GPU) uses the oracle's decision statistics (oracle_lib.feature_align_stats,
oracle_lib.match_direct_stats) to check that the cases keep reaching what they are meant to reach."""
import ctypes as C
import functools
import math
import zlib

import numpy as np
import pytest
import torch

from _compare import assert_same_bytes

CAMS = ("VGA", "EUROC", "ODD", "HD720")
LEVELS = 5
N_ITERS = (0, 1, 2, 3, 10, 30, 100)
MATCH_ITERS = (0, 1, 3, 10, 30)
BATCH_SIZES = (1, 127, 128, 129, 2 ** 17 + 1)
SENTINEL = -7.25
# images of a feature case: 0 the frame, 1 a second view, 2-5 the frame shifted by 4 px right, left, down, up, 6 flat 128
SHIFT = 4
# a template row whose 8x8 patch has mean 128 and whose x-gradients sum to 0, but whose LK step on a flat 128 image is not 0:
# align1D along (1,0) from an integer row then moves u while every residual, and so chi2, stays the same bit for bit (the
# bilinear weights sum to 1 exactly there): new_chi2 == chi2 at every iteration after the first
TIE_ROW = (100, 156, 124, 124, 124, 124, 122, 122, 128, 128)


# ---- feature cases -----------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _frames(synth, cam_name):
    """The seven images of every level: {level: u8 [7, h, w]}."""
    cam = getattr(synth, cam_name)
    xi = torch.tensor([[0.01, -0.02, 0.01, 0.0, 0.0, 0.0], [0.03, 0.01, -0.02, 0.004, -0.006, 0.003]], dtype=torch.float64)
    img = synth.Scene().render(cam, synth.pose7_from_Rt(*synth.se3_exp_Rt(xi)))
    pyr = {}
    for l, p in enumerate(synth.build_pyramid(img, LEVELS)):
        a, b = p[0].numpy(), p[1].numpy()
        pyr[l] = np.ascontiguousarray(np.stack([a, b, np.roll(a, SHIFT, 1), np.roll(a, -SHIFT, 1), np.roll(a, SHIFT, 0),
                                                np.roll(a, -SHIFT, 0), np.full_like(a, 128)]))
    return pyr


def _ulp_fracs(c):
    e = max(2.0 ** -20, float(np.spacing(np.float32(c + 1))))
    return (0.0, e, 0.5, 1.0 - e)


def _degenerate_border(kind, rng):
    y, x = np.mgrid[0:10, 0:10]
    return {"constant": np.full((10, 10), 128), "xstripes": np.where(x % 2, 200, 50), "ystripes": np.where(y % 2, 200, 50),
            "saturated": rng.integers(0, 2, (10, 10)) * 255, "checker": np.where((x + y) % 2, 255, 0),
            "ramp": 40 + 3 * x + 4 * y}[kind].astype(np.uint8)


DEGENERATE = ("constant", "xstripes", "ystripes", "saturated", "checker", "ramp")
# align1D directions; (4,-3) and (0.8,-0.6) are across the ramp 3x + 4y (H00 exactly 0, and round-off), (0,1) across xstripes
DIRS = ((1.0, 0.0), (0.0, 1.0), (0.0, 0.0), (3.0, 4.0), (4.0, -3.0), (0.8, -0.6), (1e-40, 1e-40), (-1e-40, 2e-45))
SPECIAL = (math.nan, math.inf, -math.inf, 1e10, -1e10, -0.0)


@functools.lru_cache(maxsize=None)
def _features(synth, cam_name, seed=0):
    """All feature cases of one camera: (pyr, image_index, level, border, ref, px, dirs, group)."""
    cam = getattr(synth, cam_name)
    pyr = _frames(synth, cam_name)
    rng = np.random.default_rng(1000 + CAMS.index(cam_name) + 10 * seed)
    rows = []  # (image for the alignment, level, border, start u, start v, group)

    def add(img, l, border, u, v, group):
        rows.append((img, l, border, u, v, group))

    for l in range(LEVELS):
        A = pyr[l][0]
        h, w = A.shape

        def tmpl(src, x, y):
            x, y = int(min(max(x, 5), w - 5)), int(min(max(y, 5), h - 5))
            return pyr[l][src][y - 5:y + 5, x - 5:x + 5]

        # border sweep, on the other view (a real motion) and on the frame itself
        for c in (3, 4, 5, w - 6, w - 5, w - 4):
            for f in _ulp_fracs(c):
                y = rng.uniform(5, h - 5)
                add(int(rng.integers(0, 2)), l, tmpl(0, c, y), c + f, y, "border")
        for c in (3, 4, 5, h - 6, h - 5, h - 4):
            for f in _ulp_fracs(c):
                x = rng.uniform(5, w - 5)
                add(int(rng.integers(0, 2)), l, tmpl(0, x, c), x, c + f, "border")
        # walkers: true position 1-3 px outside a bound, start 2-4 px further in
        for k in (1, 2, 3):
            for step in (2, 3, 4):
                y, x = int(rng.integers(6, h - 6)), int(rng.integers(6, w - 6))
                add(0, l, tmpl(2, 4 - k + SHIFT, y), 4 - k + step + 0.25, y + 0.5, "walk-left")  # image 2: A moved right
                add(0, l, tmpl(3, w - 5 + k - SHIFT, y), w - 5 + k - step + 0.25, y + 0.5, "walk-right")
                add(0, l, tmpl(4, x, 4 - k + SHIFT), x + 0.5, 4 - k + step + 0.25, "walk-top")
                add(0, l, tmpl(5, x, h - 5 + k - SHIFT), x + 0.5, h - 5 + k - step + 0.25, "walk-bottom")
        # random interior features
        n_rand = 120
        for _ in range(n_rand):
            x, y = int(rng.integers(8, w - 8)) if w > 16 else w // 2, int(rng.integers(8, h - 8)) if h > 16 else h // 2
            add(int(rng.integers(0, 2)), l, tmpl(0, x, y), x + rng.uniform(-1.5, 1.5), y + rng.uniform(-1.5, 1.5), "random")
        for kind in DEGENERATE:
            for _ in range(len(DIRS)):
                add(0, l, _degenerate_border(kind, rng), rng.uniform(5, w - 5), rng.uniform(5, h - 5), kind)
        # back-off ties: on the flat image, walking right from the middle and from near the right bound
        for u0 in (w / 2 + 0.25, w - 9 + 0.5, w - 6 + 0.75):
            add(6, l, np.tile(np.array(TIE_ROW, np.uint8), (10, 1)), u0, float(h // 2), "tie")
        for s in SPECIAL:
            add(0, l, tmpl(0, w // 2, h // 2), s, h / 2, "special")
            add(0, l, tmpl(0, w // 2, h // 2), w / 2, s, "special")
        add(0, l, tmpl(0, w // 2, h // 2), -0.0, -0.0, "special")
        add(0, l, tmpl(0, w // 2, h // 2), math.nan, math.inf, "special")
    n = len(rows)
    image_index = np.array([r[0] for r in rows], np.int32)
    level = np.array([r[1] for r in rows], np.int32)
    border = np.ascontiguousarray(np.stack([r[2] for r in rows]).astype(np.uint8))
    ref = np.ascontiguousarray(border[:, 1:9, 1:9])
    px = np.array([[r[3], r[4]] for r in rows], np.float64)
    group = np.array([r[5] for r in rows])
    ang = rng.uniform(0, 2 * np.pi, n)
    dirs = np.stack([np.cos(ang), np.sin(ang)], -1).astype(np.float32)
    for kind in DEGENERATE:  # every special direction on every degenerate template, and on ordinary features
        idx = np.flatnonzero(group == kind)
        dirs[idx] = np.array(DIRS, np.float32)[np.arange(len(idx)) % len(DIRS)]
    idx = np.flatnonzero(group == "random")[: 4 * len(DIRS)]
    dirs[idx] = np.array(DIRS, np.float32)[np.arange(len(idx)) % len(DIRS)]
    dirs[group == "tie"] = (1, 0)
    for side, d in (("left", (1, 0)), ("right", (-1, 0)), ("top", (0, 1)), ("bottom", (0, -1))):  # align1D walks along the axis
        dirs[group == "walk-" + side] = d
    return pyr, image_index, level, border, ref, px, dirs, group


def _oracle_features(oracle, abi, synth, cam_name, kind, n_iter, stats=False):
    pyr, idx, lvl, border, ref, px, dirs, _ = _features(synth, cam_name)
    cam = getattr(synth, cam_name)
    return oracle.feature_align_stats(abi, kind, pyr, idx, lvl, border, ref, px, n_iter, cam.width, cam.height,
                                      dirs if kind == "1d" else None, stats=stats)


_ORACLE = {}


def _solved(key, fn):
    """Each case is solved once on the oracle per module."""
    if key not in _ORACLE:
        _ORACLE[key] = fn()
    return _ORACLE[key]


def _gpu_features(pkg, cam, kind, pyr, idx, lvl, border, ref, px, n_iter, dirs):
    if kind == "2d":
        return pkg.feature_alignment.align2D(pyr, idx, lvl, border, ref, n_iter, px, cam.width, cam.height)
    return pkg.feature_alignment.align1D(pyr, idx, lvl, dirs, border, ref, n_iter, px, cam.width, cam.height)


def _assert_features(got, want, what):
    for name, g, w in zip(("converged", "px", "h_inv"), got, want):
        assert_same_bytes(g, w, f"{what} {name}")


@pytest.mark.gpu
@pytest.mark.parametrize("n_iter", N_ITERS)
@pytest.mark.parametrize("kind", ("2d", "1d"))
@pytest.mark.parametrize("cam_name", CAMS)
def test_gpu_feature_alignment_cases(pkg, oracle, abi, synth, cam_name, kind, n_iter):
    pyr, idx, lvl, border, ref, px, dirs, _ = _features(synth, cam_name)
    want, _ = _solved(("f", cam_name, kind, n_iter), lambda: _oracle_features(oracle, abi, synth, cam_name, kind, n_iter))
    got = _gpu_features(pkg, getattr(synth, cam_name), kind, pyr, idx, lvl, border, ref, px, n_iter, dirs)
    _assert_features(got, want, f"{cam_name} align{kind} n_iter={n_iter}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ("2d", "1d"))
def test_gpu_feature_alignment_does_not_depend_on_the_batch(pkg, oracle, abi, synth, kind):
    """Batches of 1, 127, 128, 129 and 2^17 + 1 features drawn (with repeats, in a random order) from the VGA cases: every
    feature's bytes equal those it gets in the full batch, and the oracle's."""
    pyr, idx, lvl, border, ref, px, dirs, _ = _features(synth, "VGA")
    cam = synth.VGA
    full = _gpu_features(pkg, cam, kind, pyr, idx, lvl, border, ref, px, 10, dirs)
    want, _ = _solved(("f", "VGA", kind, 10), lambda: _oracle_features(oracle, abi, synth, "VGA", kind, 10))
    _assert_features(full, want, "full batch")
    rng = np.random.default_rng(5)
    for n in BATCH_SIZES:
        sel = rng.integers(0, len(idx), n)
        got = _gpu_features(pkg, cam, kind, pyr, idx[sel], lvl[sel], border[sel], ref[sel], px[sel], 10, dirs[sel])
        _assert_features(got, tuple(a[sel] for a in full), f"batch of {n}")


def _padded(pyr, rows=3, cols=21):
    """The same pyramid as views into arrays with `rows` spare rows and `cols` spare columns: pitch != width and
    stride != rows * pitch, so the host copies it image by image."""
    out = {}
    for l, a in pyr.items():
        big = np.full((a.shape[0], a.shape[1] + rows, a.shape[2] + cols), 77, np.uint8)
        big[:, :a.shape[1], :a.shape[2]] = a
        out[l] = big[:, :a.shape[1], :a.shape[2]]
    return out


def _every_other(pyr):
    """The same pyramid as every other frame of a stack whose other frames are garbage."""
    out = {}
    for l, a in pyr.items():
        big = np.empty((2 * a.shape[0],) + a.shape[1:], np.uint8)
        big[0::2] = a
        big[1::2] = 255 - a
        out[l] = big[0::2]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ("padded", "every-other", "level-3-only"))
@pytest.mark.parametrize("kind", ("2d", "1d"))
def test_gpu_feature_alignment_host_layouts(pkg, oracle, abi, synth, kind, layout):
    pyr, idx, lvl, border, ref, px, dirs, _ = _features(synth, "ODD")
    cam = synth.ODD
    want, _ = _solved(("f", "ODD", kind, 10), lambda: _oracle_features(oracle, abi, synth, "ODD", kind, 10))
    if layout == "level-3-only":
        sel = np.flatnonzero(lvl == 3)
        got = _gpu_features(pkg, cam, kind, {3: _padded({3: pyr[3]})[3]}, idx[sel], lvl[sel], border[sel], ref[sel], px[sel], 10,
                            dirs[sel])
        _assert_features(got, tuple(a[sel] for a in want), layout)
        return
    view = _padded(pyr) if layout == "padded" else _every_other(pyr)
    assert all(v.strides[0] != v.shape[1] * v.strides[1] for v in view.values())
    got = _gpu_features(pkg, cam, kind, view, idx, lvl, border, ref, px, 10, dirs)
    _assert_features(got, want, layout)


# ---- findMatchDirect cases ---------------------------------------------------------------------------------------------
def _append_frames(synth, d, which, T7):
    """Append frames with poses T7 [k,7] (rendered from the scene) to d's reference or current frames."""
    pose_attr, pyr_attr = ("T_ref_w", "ref_pyr") if which == "ref" else ("T_cur_w", "cur_pyr")
    T7 = np.ascontiguousarray(T7, np.float64)
    img = synth.Scene().render(d.cam, torch.tensor(T7))
    levels = synth.build_pyramid(img, max(getattr(d, pyr_attr)) + 1)
    pyr = getattr(d, pyr_attr)
    for l in pyr:
        pyr[l] = np.ascontiguousarray(np.concatenate([pyr[l], levels[l].numpy()]))
    first = getattr(d, pose_attr).shape[0]
    setattr(d, pose_attr, np.ascontiguousarray(np.concatenate([getattr(d, pose_attr), T7])))
    return first


def _edge_rows(synth, d, rng):
    """Overwrite the first rows of d with the edge cases; returns the number of rows used."""
    cam, L = d.cam, d.n_pyr_levels
    r, exact = 0, []

    def put(ref_px=None, level=None, **kw):
        nonlocal r
        if ref_px is not None:
            d.ref_px[r] = ref_px
        if level is not None:
            d.ref_level[r] = level
        for k, v in kw.items():
            getattr(d, k)[r] = v
        r += 1

    # the in-frame border (b = 6) at every reference level, both sides, first and last pixel of the level's cell
    for l in range(L):
        s, W, H = 1 << l, cam.width >> l, cam.height >> l
        for o in (5, 6, W - 7, W - 6):
            for f in (0.0, 1.0 - 2.0 ** -10):
                put(((o + f) * s, cam.height / 2), l)
        for o in (5, 6, H - 7, H - 6):
            for f in (0.0, 1.0 - 2.0 ** -10):
                put((cam.width / 2, (o + f) * s), l)
    # NaN warps: the point at the reference camera centre (an extra reference frame at the identity: A = 0), and NaN
    R0, t0 = torch.eye(3, dtype=torch.float64)[None], torch.zeros(1, 3, dtype=torch.float64)
    ident = _append_frames(synth, d, "ref", synth.pose7_from_Rt(R0, t0).numpy())
    for k in range(4):
        put((cam.width / 2 + 7 * k, cam.height / 2), 0, ref_index=ident, pos=(0.0, 0.0, 0.0), is_edgelet=k % 2)
        put(None, None, pos=(math.nan, 1.0, 2.0), is_edgelet=k % 2)
    # a current frame 1 mm in front of a point 1 m ahead of the identity frame: A ~ 1000, so the search level is clamped at
    # n_pyr_levels - 1 for every n_pyr_levels up to 8
    close = _append_frames(synth, d, "cur", synth.pose7_from_Rt(R0, torch.tensor([[0.0, 0.0, -0.999]], dtype=torch.float64)).numpy())
    for e in (0, 1):
        put((cam.cx, cam.cy), 0, ref_index=ident, cur_index=close, ref_f=(0.0, 0.0, 1.0), pos=(0.0, 0.0, 1.0),
            px_cur=(cam.cx + 0.3, cam.cy - 0.2), is_edgelet=e)
    # edgelets with zero and axis-aligned gradients
    for g in ((0.0, 0.0), (1.0, 0.0), (0.0, 1.0), (-0.0, -1.0)):
        for _ in range(2):
            put(None, None, is_edgelet=1, ref_grad=g)
    # warped patches partly outside the reference image: a current frame rolled 45 degrees about the optical axis of
    # reference frame 0, candidates at the in-frame border of every level (their 10x10 sample reaches 5 sqrt(2) px out)
    Rr, tr = synth.pose7_to_Rt(torch.tensor(d.T_ref_w[:1]))
    c, s_ = math.cos(math.pi / 4), math.sin(math.pi / 4)
    Rz = torch.tensor([[[c, -s_, 0.0], [s_, c, 0.0], [0.0, 0.0, 1.0]]], dtype=torch.float64)
    rolled = _append_frames(synth, d, "cur", synth.pose7_from_Rt(Rz @ Rr, (Rz @ tr[..., None])[..., 0]).numpy())
    for l in range(L):
        sc, W, H = 1 << l, cam.width >> l, cam.height >> l
        for ox, oy in ((6, H // 2), (W - 7, H // 2), (W // 2, 6), (W // 2, H - 7), (6, 6), (W - 7, H - 7)):
            p = np.array([(ox + 0.5) * sc, (oy + 0.5) * sc])
            q = p - (cam.cx, cam.cy)
            pc = np.array([c * q[0] - s_ * q[1], s_ * q[0] + c * q[1]]) + (cam.cx, cam.cy) + rng.uniform(-1, 1, 2)
            for e in (0, 1):
                put(p, l, ref_index=0, cur_index=rolled, px_cur=pc, is_edgelet=e)
    # rows that _on_bound moves so that a sample of the warped patch which a template gradient reads lands exactly on the
    # last column / row: a frame rolled 135 degrees reaches 6.4 px beyond the point with such a sample (45 degrees: 4.9)
    c3, s3 = math.cos(3 * math.pi / 4), math.sin(3 * math.pi / 4)
    Rz3 = torch.tensor([[[c3, -s3, 0.0], [s3, c3, 0.0], [0.0, 0.0, 1.0]]], dtype=torch.float64)
    rolled3 = _append_frames(synth, d, "cur", synth.pose7_from_Rt(Rz3 @ Rr, (Rz3 @ tr[..., None])[..., 0]).numpy())
    for l in range(L):
        sc, W, H = 1 << l, cam.width >> l, cam.height >> l
        if W - 7 >= 6 and H - 7 >= 6:
            for axis, (ox, oy) in enumerate(((W - 7, H // 2), (W // 2, H - 7))):
                p = np.array([(ox + 0.5) * sc, (oy + 0.5) * sc])
                q = p - (cam.cx, cam.cy)
                pc = np.array([c3 * q[0] - s3 * q[1], s3 * q[0] + c3 * q[1]]) + (cam.cx, cam.cy)
                f = np.array([(p[0] - cam.cx) / cam.fx, (p[1] - cam.cy) / cam.fy, 1.0])
                exact.append((r, axis))
                put(p, l, ref_index=0, cur_index=rolled3, px_cur=pc, is_edgelet=0, ref_f=f / np.linalg.norm(f))
    return r, exact


def _on_bound(d, exact):
    """Move the reference point of each (row, axis) of `exact` so that one sample of its warped 10x10 patch lands exactly on
    the last column (axis 0) or row (axis 1) of the reference level, where `q >= cols - 1` zeroes it.  The sample's float
    position is recomputed as warpAffine computes it (fp32, no contraction) from the warp the oracle returns; the warp moves
    a little with the point, so this repeats until the oracle counts such a sample in every row."""
    import oracle_lib
    import plsvo_b200

    abi = plsvo_b200.abi
    oracle_lib.load(abi)
    f32 = np.float32
    for _ in range(8):
        out, st = oracle_lib.match_direct_stats(abi, d)
        todo = [(i, a) for i, a in exact if st["on_bound"][i] == 0]
        if not todo:
            return
        for i, axis in todo:
            A00, A01, A10, A11 = out.A_cur_ref[i]
            l, sl = int(d.ref_level[i]), int(out.search_level[i])
            assert sl >= 0, (i, d.ref_px[i])
            invdet = 1.0 / (A00 * A11 - A10 * A01)
            R = (f32(A11 * invdet), f32(-A01 * invdet)) if axis == 0 else (f32(-A10 * invdet), f32(A00 * invdet))
            x, y = np.meshgrid(np.arange(10), np.arange(10))
            p0, p1 = f32(x - 5) * f32(1 << sl), f32(y - 5) * f32(1 << sl)
            t = (R[0] * p0 + R[1] * p1).astype(f32)  # fp32 products and sum, as in warpAffine
            t[[0, 0, 9, 9], [0, 9, 0, 9]] = -np.inf  # no template gradient reads the corners
            k = np.argmax(t)
            t_k = t.flat[k]
            bound = f32(((d.cam.width if axis == 0 else d.cam.height) >> l) - 1)
            pr = f32(bound - t_k)
            for cand in (pr, np.nextafter(pr, f32(np.inf)), np.nextafter(pr, f32(-np.inf))):
                if f32(t_k + cand) == bound:
                    pr = cand
                    break
            d.ref_px[i, axis] = float(pr) * (1 << l)
            f = np.array([(d.ref_px[i, 0] - d.cam.cx) / d.cam.fx, (d.ref_px[i, 1] - d.cam.cy) / d.cam.fy, 1.0])
            d.ref_f[i] = f / np.linalg.norm(f)  # the bearing of the moved point: the warp stays the roll
    raise AssertionError("no warped sample lands exactly on the last column / row")


@functools.lru_cache(maxsize=None)
def _match_case(synth, name):
    """findMatchDirect cases by name: ("levels", cam, L), ("iters",), ("many-frames",)."""
    if name[0] == "levels":
        _, cam_name, L = name
        seed = 7300 + 10 * CAMS.index(cam_name) + L
        d = synth.make_match_batch(cam=getattr(synth, cam_name), n=1200, seed=seed, n_pyr_levels=L)
    elif name[0] == "iters":
        d = synth.make_match_batch(cam=synth.VGA, n=3000, seed=7390, n_pyr_levels=5)
    else:
        # rendered on the CPU everywhere, so that the reference pin finds its recorded inputs on any machine
        d = synth.make_match_batch(cam=synth.VGA, n=4000, n_ref=40, n_cur=40, seed=7391, n_pyr_levels=4)
    _, exact = _edge_rows(synth, d, np.random.default_rng(zlib.crc32(repr(name).encode())))
    _on_bound(d, exact)
    return d


MATCH_CASES = [("levels", c, L) for c in CAMS for L in range(1, 9)] + [("iters",), ("many-frames",)]


def _oracle_match(oracle, abi, d, n_iter, out=None):
    d.n_iter = n_iter
    return oracle.match_direct(abi, d, oracle._n_threads(abi, 0), out=out)


def _assert_match(got, want, what):
    for f in ("px_cur", "success", "search_level", "A_cur_ref"):
        assert_same_bytes(getattr(got, f), getattr(want, f), f"{what} {f}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", MATCH_CASES, ids=lambda n: "-".join(map(str, n)))
def test_gpu_find_match_direct_cases(pkg, oracle, abi, synth, name):
    d = _match_case(synth, name)
    for n_iter in (MATCH_ITERS if name == ("iters",) else (10,)):
        want = _solved(("m", name, n_iter), lambda: _oracle_match(oracle, abi, d, n_iter))
        got = pkg.Matcher(n_iter).findMatchDirect(d)
        _assert_match(got, want, f"{name} align_max_iter={n_iter}")


@pytest.mark.gpu
def test_gpu_find_match_direct_null_pointers_and_sentinel(pkg, oracle, abi, synth):
    """A_cur_ref prefilled with a sentinel comes back with the sentinel in every rejected row; without is_edgelet every
    candidate runs align2D; NULL search_level and A_cur_ref leave px_cur and success as they are."""
    d = _match_case(synth, ("levels", "VGA", 5))
    ctx = pkg.default_context()

    def run_gpu(data, out):
        b, keep = abi.make_match_batch(data)
        assert ctx.lib.plsvo_match_direct_batch_run(ctx.handle, C.byref(b), C.byref(out.struct)) == abi.OK
        return out

    def sentinel_out():
        o = abi.MatchOut(d.n)
        o.A_cur_ref[:] = SENTINEL
        return o

    d.n_iter = 10
    got, want = run_gpu(d, sentinel_out()), _oracle_match(oracle, abi, d, 10, out=sentinel_out())
    _assert_match(got, want, "sentinel")
    rejected = want.search_level < 0
    assert rejected.any() and (got.A_cur_ref[rejected] == SENTINEL).all()
    # no is_edgelet (NULL pointers): every candidate is a point
    from dataclasses import replace

    dn = replace(d, is_edgelet=None, ref_grad=None)
    want_pts = _oracle_match(oracle, abi, dn, 10)
    _assert_match(run_gpu(dn, abi.MatchOut(d.n)), want_pts, "no is_edgelet")
    dz = replace(d, is_edgelet=np.zeros_like(d.is_edgelet))
    _assert_match(want_pts, _oracle_match(oracle, abi, dz, 10), "is_edgelet NULL vs all 0")
    # NULL search_level and A_cur_ref
    o = abi.MatchOut(d.n)
    o.struct.search_level = C.POINTER(C.c_int32)()
    o.struct.A_cur_ref = C.POINTER(C.c_double)()
    got = run_gpu(d, o)
    assert_same_bytes(got.px_cur, want.px_cur, "NULL outputs px_cur")
    assert_same_bytes(got.success, want.success, "NULL outputs success")


@pytest.mark.gpu
def test_gpu_find_match_direct_refuses_nine_levels(pkg, oracle, abi, synth):
    d = _match_case(synth, ("levels", "VGA", 8))
    ctx = pkg.default_context()
    d.n_iter = 10
    b, keep = abi.make_match_batch(d)
    b.n_pyr_levels = 9
    out = abi.MatchOut(d.n)
    assert ctx.lib.plsvo_match_direct_batch_run(ctx.handle, C.byref(b), C.byref(out.struct)) == abi.ERR_INVALID
    assert b"match batch description" in ctx.lib.plsvo_last_error(ctx.handle)
    # the context stays usable
    want = _solved(("m", ("levels", "VGA", 8), 10), lambda: _oracle_match(oracle, abi, d, 10))
    _assert_match(pkg.Matcher(10, ctx).findMatchDirect(d), want, "after the refusal")


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ("padded", "every-other", "ref-level-3-only"))
def test_gpu_find_match_direct_host_layouts(pkg, oracle, abi, synth, layout):
    from dataclasses import replace

    d = _match_case(synth, ("levels", "ODD", 5))
    want = _solved(("m", ("levels", "ODD", 5), 10), lambda: _oracle_match(oracle, abi, d, 10))
    if layout == "ref-level-3-only":
        sel = np.flatnonzero(d.ref_level == 3)
        sub = lambda a: None if a is None else np.ascontiguousarray(a[sel])  # noqa: E731
        ds = replace(d, ref_pyr={3: _padded({3: d.ref_pyr[3]})[3]}, ref_index=sub(d.ref_index), cur_index=sub(d.cur_index),
                     ref_px=sub(d.ref_px), ref_f=sub(d.ref_f), ref_level=sub(d.ref_level), is_edgelet=sub(d.is_edgelet),
                     ref_grad=sub(d.ref_grad), pos=sub(d.pos), px_cur=sub(d.px_cur), px_cur_gt=sub(d.px_cur_gt))
        got = pkg.Matcher(10).findMatchDirect(ds)
        for f in ("px_cur", "success", "search_level", "A_cur_ref"):
            assert_same_bytes(getattr(got, f), getattr(want, f)[sel], f"{layout} {f}")
        return
    view = _padded if layout == "padded" else _every_other
    dv = replace(d, ref_pyr=view(d.ref_pyr), cur_pyr=view(d.cur_pyr))
    _assert_match(_oracle_match(oracle, abi, dv, 10), want, f"{layout} (oracle)")
    _assert_match(pkg.Matcher(10).findMatchDirect(dv), want, layout)


# ---- coverage (no GPU) -------------------------------------------------------------------------------------------------
def test_direct_match_cases_cover_every_exit(oracle, abi, synth):
    """The cases above reach every exit of both aligners at iteration 0, 1 and n_iter - 1 and the iteration cap, singular
    systems in both, back-offs at iteration 1 and later, frame exits at each bound at every level, all four byte offsets
    at every level width, and, in findMatchDirect, every clamped n_pyr_levels, NaN warps, partial patches and NaN
    edgelet directions."""
    X = oracle
    for kind in ("2d", "1d"):
        exits = {X.DS_EXIT_FRAME, X.DS_EXIT_CONVERGED, X.DS_EXIT_CAP} | ({X.DS_EXIT_BACKOFF} if kind == "1d" else set())
        seen = set()
        for cam_name in CAMS:
            _, _, lvl, _, _, _, _, group = _features(synth, cam_name)
            for n_iter in N_ITERS:
                _, st = _oracle_features(oracle, abi, synth, cam_name, kind, n_iter, stats=True)
                if n_iter == 0:
                    assert (st["exit"] == X.DS_EXIT_NONE).all()
                    continue
                for e in exits:
                    for it in {0, 1, n_iter - 1}:
                        if (e == X.DS_EXIT_BACKOFF and it == 0) or (e == X.DS_EXIT_CAP and it != n_iter - 1):
                            continue
                        if ((st["exit"] == e) & (st["iter"] == it)).any():
                            seen.add((e, it == 0, it == 1, it == n_iter - 1))
                if n_iter != 10:
                    continue
                frame = st["exit"] == X.DS_EXIT_FRAME
                for l in range(LEVELS):
                    at = lvl == l
                    for k, b in enumerate(X.DS_BOUNDS):
                        assert (frame & at & (st["bound"] & (1 << k) != 0) & (st["iter"] >= 1)).any(), (cam_name, kind, l, b)
                    assert set(np.unique(st["offset"][at])) >= {0, 1, 2, 3}, (cam_name, kind, l)
                    # floor(u) and floor(v) on the first rejected pixel past each bound, and features that reach the last
                    # admissible one without leaving
                    for k in range(4):
                        assert (st["dist"][at & (group == "border"), k] == -1).any(), (cam_name, kind, l, k)
                        assert (st["dist"][at, k] == 0).any(), (cam_name, kind, l, k)
                assert (st["det_zero"] & st["hinv_nonfinite"]).any()
                if kind == "1d":
                    assert st["h_inv_nonfinite"].any()
                    back = st["exit"] == X.DS_EXIT_BACKOFF
                    assert (back & (st["iter"] == 1)).any() and (back & (st["iter"] >= 2)).any()
                    assert (st["tie"] & (group == "tie")).any() and not (st["tie"] & (group != "tie")).any()
        for e in exits:
            assert any(s[0] == e and s[1] for s in seen) or e in (X.DS_EXIT_BACKOFF, X.DS_EXIT_CAP), (kind, e, "iteration 0")
            assert any(s[0] == e and s[2] for s in seen), (kind, e, "iteration 1")
            assert any(s[0] == e and s[3] for s in seen), (kind, e, "iteration n_iter - 1")
    # findMatchDirect
    for cam_name in CAMS:
        for L in range(1, 9):
            d = _match_case(synth, ("levels", cam_name, L))
            d.n_iter = 10
            out, st = oracle.match_direct_stats(abi, d)
            ran = ~st["reject"]
            assert st["reject"].any() and ran.any()
            assert (st["clamped"] & (out.search_level == L - 1)).any(), (cam_name, L)
            assert st["nan_warp"].any() and (st["zeroed"] > 0).any() and st["nan_dir"].any(), (cam_name, L)
            assert (st["on_bound"] > 0).any(), (cam_name, L)
            assert (st["edgelet"] & ~st["nan_dir"] & ran).any()
    d = _match_case(synth, ("iters",))
    for n_iter in MATCH_ITERS:
        d.n_iter = n_iter
        out, st = oracle.match_direct_stats(abi, d)
        if n_iter:
            assert (st["exit"] == X.DS_EXIT_CAP).any() and (st["exit"] == X.DS_EXIT_CONVERGED).any()


def test_direct_stats_entry_points_compute_what_the_batch_ones_do(oracle, abi, synth):
    """plsvo_oracle_align{2,1}d_stats and plsvo_oracle_match_direct_stats run the same code as the batch entry points: their
    outputs are byte-identical."""
    pyr, idx, lvl, border, ref, px, dirs, _ = _features(synth, "ODD")
    for kind in ("2d", "1d"):
        for n_iter in (1, 10):
            plain, _ = _oracle_features(oracle, abi, synth, "ODD", kind, n_iter)
            with_stats, st = _oracle_features(oracle, abi, synth, "ODD", kind, n_iter, stats=True)
            _assert_features(with_stats, plain, f"align{kind} n_iter={n_iter}")
            assert len(st["exit"]) == len(idx)
    for name in (("levels", "ODD", 5), ("levels", "HD720", 8)):
        d = _match_case(synth, name)
        d.n_iter = 10
        out, st = oracle.match_direct_stats(abi, d)
        _assert_match(out, oracle.match_direct(abi, d, 4), str(name))
    # and the per-feature loop of oracle.align2d / align1d agrees with the batch entry point
    sel = np.arange(0, len(idx), 7)
    args = (pyr, idx[sel], lvl[sel])
    conv, p = oracle.align2d(abi, *args, border[sel], ref[sel], px[sel], 10)
    _assert_features((conv, p), oracle.align2d_batch(abi, *args, border[sel], ref[sel], px[sel], 10, synth.ODD.width, synth.ODD.height),
                     "align2d loop")
    conv, p, h = oracle.align1d(abi, *args, dirs[sel], border[sel], ref[sel], px[sel], 10)
    _assert_features((conv, p, h), oracle.align1d_batch(abi, *args, dirs[sel], border[sel], ref[sel], px[sel], 10, synth.ODD.width,
                                                        synth.ODD.height), "align1d loop")


PIN_FEATURES = [(c, k, n) for c in CAMS for k in ("2d", "1d") for n in N_ITERS]


@pytest.mark.parametrize("cam_name,kind,n_iter", PIN_FEATURES)
def test_direct_feature_cases_are_bit_identical_to_the_reference_tu(oracle, abi, synth, cam_name, kind, n_iter):
    """The feature cases (border sweep, walkers, degenerate templates and directions, NaN / inf / 1e10 / -0.0 starts) through
    the reference's own feature_alignment.cpp (oracle/_ref, or its recorded outputs)."""
    if not oracle.have_ref():
        pytest.skip("oracle/_ref is not built and no recorded outputs of it are present")
    pyr, idx, lvl, border, ref, px, dirs, _ = _features(synth, cam_name)
    got, _ = _oracle_features(oracle, abi, synth, cam_name, kind, n_iter)
    if kind == "2d":
        r = oracle.ref_align2d(abi, pyr, idx, lvl, border, ref, px, n_iter)
    else:
        r = oracle.ref_align1d(abi, pyr, idx, lvl, dirs, border, ref, px, n_iter)
    for k, g in enumerate(got):
        oracle.assert_ref_equal(g, r, str(k))


PIN_MATCH = MATCH_CASES


@pytest.mark.parametrize("name", PIN_MATCH, ids=lambda n: "-".join(map(str, n)))
def test_direct_match_cases_are_bit_identical_to_the_reference_tu(oracle, abi, synth, name):
    """The findMatchDirect cases (clamped search levels, the in-frame border at every level, NaN warps, partial patches,
    NaN edgelet directions) through the reference's own matcher.cpp, one fresh Matcher per candidate.  Points at the
    reference camera centre or NaN are left out: their viewing direction is NaN, so the reference's getCloseViewObs rejects
    them before findMatchDirect's own code runs (the kernel takes candidates after that choice)."""
    if not oracle.have_ref():
        pytest.skip("oracle/_ref is not built and no recorded outputs of it are present")
    d = _match_case(synth, name)
    rows = np.flatnonzero(~(np.isnan(d.pos).any(1) | (d.pos == 0).all(1)))
    for n_iter in (MATCH_ITERS if name == ("iters",) else (10,)):
        d.n_iter = n_iter
        o = oracle.match_direct(abi, d, 4)
        r = oracle.ref_match_direct(abi, d)
        for f in ("success", "search_level", "px_cur", "A_cur_ref"):
            oracle.assert_ref_equal(getattr(o, f), r, f, rows=rows, err_msg=f"{name} {n_iter}")
