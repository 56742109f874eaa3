"""The image-pyramid kernel (pyramid_kernel.cu, frame_utils::createImgPyramid = repeated vk::halfSample) through its three
callers: plsvo_pyramid_batch_run, plsvo_undistort_batch_run (the pyramid of the rectified frame) and the levels an
alignment or track call derives from the finest level it was given.

The reference is the integer definition, written here in NumPy: every level is (a + b + c + d) // 4 of the 2x2 blocks of
the level below, in uint16.  The cases:
  * sizes on both sides of the kernel's 16-byte row segments and 64-pixel tiles, with a top level of one row or one
    column, at 1, 2 and the deepest legal number of levels; one level more is refused;
  * byte patterns that check the packed 16-bit lanes and the truncation: all 0, all 255, a 0/255 checkerboard,
    one-pixel stripes, and blocks whose sum is 4k+3;
  * a level 0 inside wider rows and padded frames, outputs in padded arrays whose padding must stay untouched;
  * batches of up to 70 001 frames (more than gridDim.z holds), and one context reused across shapes;
  * the undistort entry point, with and without distortion;
  * level 7 derived from level 0 in the alignment, the ATAN alignment and the track call, which takes two launches of
    the kernel (its 64x64 tile holds levels 0..6), against the same calls with every level shipped and against the
    oracle."""
import copy
import ctypes as C
import os

import numpy as np
import pytest

from test_gpu_align import _check
from test_gpu_atan import atan_for, compare, oracle_atan, reference, through  # noqa: F401  (oracle_atan: fixture)
from test_undistort import ODD, PINCUSHION, cam_struct, remap_kernels, uo  # noqa: F401  (remap_kernels, uo: fixtures)
from test_zz_gpu_word_pitch import FIELDS

WIDTHS = (1, 2, 3, 15, 16, 17, 63, 64, 65, 127, 128, 129, 130, 192, 641, 1280)
HEIGHTS = (1, 2, 3, 63, 64, 65, 127, 128, 129, 479)
GUARD = 0xA5


def half(a):
    """vk::halfSample: the truncating mean of every 2x2 block, in uint16."""
    h, w = a.shape[1] // 2, a.shape[2] // 2
    x = a[:, : 2 * h, : 2 * w].astype(np.uint16)
    return ((x[:, 0::2, 0::2] + x[:, 0::2, 1::2] + x[:, 1::2, 0::2] + x[:, 1::2, 1::2]) // 4).astype(np.uint8)


def np_pyramid(img, n_levels):
    out = [np.asarray(img)]
    for _ in range(1, n_levels):
        out.append(half(out[-1]))
    return out


def deepest(w, h):
    """The deepest legal level count: every level at least one pixel, at most 7 levels."""
    return min(7, min(w, h).bit_length())


def pyramid_call(pkg, abi, img, n_levels, ctx=None, pad=(0, 0)):
    """plsvo_pyramid_batch_run on the u8 view img [B,H,W], passed with its own pitch and frame stride.  Levels 1.. go into
    arrays with pad = (rows, columns) of padding, filled with GUARD.  Returns (rc, message, levels, padded arrays)."""
    ctx = ctx or pkg.api.default_context()
    B, H, W = img.shape
    assert img.strides[2] == 1
    b = abi.PyramidBatch(B, W, H, n_levels, img.ctypes.data_as(C.POINTER(C.c_uint8)), img.strides[1], img.strides[0])
    r = abi.PyramidResult()
    bufs = [None]
    for l in range(1, min(n_levels, abi.MAX_LEVELS)):
        buf = np.full((B, (H >> l) + pad[0], (W >> l) + pad[1]), GUARD, np.uint8)
        bufs.append(buf)
        r.level[l] = buf.ctypes.data_as(C.POINTER(C.c_uint8))
        r.pitch[l], r.stride[l] = buf.strides[1], buf.strides[0]
    rc = ctx.lib.plsvo_pyramid_batch_run(ctx.handle, C.byref(b), C.byref(r))
    msg = (ctx.lib.plsvo_last_error(ctx.handle) or b"").decode() if rc != abi.OK else ""
    levels = [img] + [buf[:, : H >> l, : W >> l] for l, buf in enumerate(bufs) if l > 0]
    return rc, msg, levels, bufs


@pytest.fixture
def new_ctx(pkg):
    """Makes contexts for one test and closes them when it ends, whether it passed or not."""
    made = []

    def make():
        made.append(pkg.api.Context(0))
        return made[-1]

    yield make
    for ctx in made:
        ctx.close()


def counted(ctx, call):
    """(result of call(), kernels it launched on ctx)."""
    n = ctx.launch_count()
    out = call()
    return out, ctx.launch_count() - n


def check_pyramid(pkg, abi, img, n_levels, what, ctx=None, pad=(0, 0), want=None):
    rc, msg, got, bufs = pyramid_call(pkg, abi, img, n_levels, ctx, pad)
    assert rc == abi.OK, (what, rc, msg)
    want = want or np_pyramid(np.ascontiguousarray(img), n_levels)
    for l in range(1, n_levels):
        np.testing.assert_array_equal(got[l], want[l], err_msg=f"{what}: level {l}")
        h, w = want[l].shape[1:]
        assert (bufs[l][:, h:, :] == GUARD).all() and (bufs[l][:, :, w:] == GUARD).all(), f"{what}: level {l} wrote its padding"
    return got


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_numpy_reference_is_the_oracle_pyramid(oracle, abi):
    rng = np.random.default_rng(7000)
    for B, H, W in ((2, 1, 1), (1, 3, 17), (3, 65, 63), (2, 64, 130), (1, 129, 2)):
        img = rng.integers(0, 256, (B, H, W), dtype=np.uint8)
        n = deepest(W, H)
        for a, b in zip(np_pyramid(img, n), oracle.pyramid(abi, img, n)):
            np.testing.assert_array_equal(a, b)
    blocks = np.array([[[255, 255], [255, 254]]], np.uint8), np.array([[[0, 0], [1, 2]]], np.uint8)
    assert half(blocks[0])[0, 0, 0] == 254 and half(blocks[1])[0, 0, 0] == 0  # 4k+3 sums truncate


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("W", WIDTHS)
def test_every_size_and_level_count(pkg, abi, W):
    """Each width with every height, at 1, 2 and the deepest legal level count; one level more is refused."""
    rng = np.random.default_rng(7100 + W)
    for H in HEIGHTS:
        img = rng.integers(0, 256, (2, H, W), dtype=np.uint8)
        top = deepest(W, H)
        want = np_pyramid(img, top)
        for n in sorted({1, min(2, top), top}):
            check_pyramid(pkg, abi, img, n, f"{W}x{H}, {n} levels", want=want[:n])
        rc, msg, _, _ = pyramid_call(pkg, abi, img, top + 1)
        assert rc == abi.ERR_INVALID, (W, H, top + 1, rc)
        assert ("smaller than one pixel" if top < 7 else "pyramid batch description") in msg, (W, H, msg)


def patterns(rng, B, H, W):
    y, x = np.mgrid[:H, :W]
    out = {"zeros": np.zeros((B, H, W), np.uint8), "255": np.full((B, H, W), 255, np.uint8),
           "checkerboard": np.broadcast_to(((x + y) % 2 * 255).astype(np.uint8), (B, H, W)),
           "stripes_x": np.broadcast_to((x % 2 * 255).astype(np.uint8), (B, H, W)),
           "stripes_y": np.broadcast_to((y % 2 * 255).astype(np.uint8), (B, H, W))}
    # 2x2 blocks (k, k, k+1, k+2) in a random order: sum 4k+3, mean k, for k up to 253; and the two ends of the range
    k = rng.integers(0, 254, (B, (H + 1) // 2, (W + 1) // 2)).astype(np.int32)
    k[:, ::3, ::3] = 253
    k[:, 1::3, 1::3] = 0
    offs = np.array([0, 0, 1, 2], np.int32)[rng.permuted(np.tile(np.arange(4), (B, k.shape[1], k.shape[2], 1)), axis=-1)]
    blocks = (k[..., None] + offs).reshape(B, k.shape[1], k.shape[2], 2, 2).transpose(0, 1, 3, 2, 4)
    out["sum_4k_plus_3"] = blocks.reshape(B, 2 * k.shape[1], 2 * k.shape[2])[:, :H, :W].astype(np.uint8)
    out["random"] = rng.integers(0, 256, (B, H, W), dtype=np.uint8)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(8, 16), (65, 129), (64, 64), (127, 130), (479, 641), (720, 1280)])
def test_byte_patterns(pkg, abi, H, W):
    rng = np.random.default_rng(7200 + W)
    for name, img in patterns(rng, 3, H, W).items():
        img = np.ascontiguousarray(img)
        want = np_pyramid(img, deepest(W, H))
        if name == "sum_4k_plus_3":
            h, w = H // 2, W // 2  # every block's mean is its smallest pixel
            np.testing.assert_array_equal(want[1], img[:, : 2 * h, : 2 * w].reshape(3, h, 2, w, 2).min(axis=(2, 4)))
        check_pyramid(pkg, abi, img, deepest(W, H), f"{name} {W}x{H}", want=want)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(8, 16), (65, 129), (479, 641), (128, 1280)])
@pytest.mark.parametrize("layout", ["row_padded", "frame_padded", "both", "every_other_frame"])
def test_padded_input_and_output_layouts(pkg, abi, layout, H, W):
    """A level-0 view into wider rows (pitch0 > width), padded frames (stride0 != H * pitch0: copied frame by frame), and
    outputs written into padded arrays whose padding must stay as it was."""
    rng = np.random.default_rng(7300 + H)
    big = rng.integers(0, 256, (10, H + 3, W + 21), dtype=np.uint8)
    view = {"row_padded": lambda: np.ascontiguousarray(big[:, :H])[:, :, 5:W + 5],
            "frame_padded": lambda: np.ascontiguousarray(big[:, :, :W])[:, 1:H + 1],
            "both": lambda: big[:, 2:H + 2, 3:W + 3],
            "every_other_frame": lambda: big[::2, :H, :W]}[layout]()
    assert view.strides[1] != W or view.strides[0] != H * view.strides[1]
    for pad in ((0, 0), (2, 13), (1, 1)):
        check_pyramid(pkg, abi, view, deepest(W, H), f"{layout} {W}x{H} pad {pad}", pad=pad)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 37, 65535, 65536, 70001])
def test_batch_sizes(pkg, abi, B):
    """Frames sit on the kernel's gridDim.z (at most 65535): larger batches are launched in pieces."""
    img = np.random.default_rng(7400 + B).integers(0, 256, (B, 8, 16), dtype=np.uint8)
    check_pyramid(pkg, abi, img, 3, f"B={B}", pad=(1, 3))
    got = pkg.createImgPyramid(img, 3)
    for a, b in zip(got, np_pyramid(img, 3)):
        np.testing.assert_array_equal(a, b)


@pytest.mark.gpu
def test_one_context_large_small_large(pkg, abi, new_ctx):
    """Calls of different shapes on one context equal those of a fresh context: no byte of an earlier call shows through
    the device buffers' padding."""
    rng = np.random.default_rng(7500)
    ctx = new_ctx()
    for B, H, W, n in ((3, 720, 1280, 7), (5, 17, 33, 5), (2, 479, 641, 7), (9, 3, 129, 2), (4, 720, 1280, 7), (70001, 8, 16, 3)):
        img = rng.integers(0, 256, (B, H, W), dtype=np.uint8)
        got = check_pyramid(pkg, abi, img, n, f"reused context {B}x{W}x{H}", ctx=ctx, pad=(1, 7))
        fresh = check_pyramid(pkg, abi, img, n, f"fresh context {B}x{W}x{H}", ctx=new_ctx())
        for l in range(n):
            np.testing.assert_array_equal(got[l], fresh[l])


# ---- the undistort entry point: the pyramid of the rectified frame -------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("size", ["odd_641x479", "129x65"])
def test_undistort_copy_camera_every_level_count(pkg, new_ctx, size):
    """A camera without distortion: level 0 is the raw frame, levels 1.. its pyramid."""
    from test_undistort import params

    cam = pkg.PinholeCamera(*params(ODD)[:6]) if size.startswith("odd") else pkg.PinholeCamera(129, 65, 90.0, 90.0, 64.0, 32.0)
    assert (cam.width, cam.height) == ((641, 479) if size.startswith("odd") else (129, 65))
    raw = np.random.default_rng(7600).integers(0, 256, (3, cam.height, cam.width), dtype=np.uint8)
    want = np_pyramid(raw, 7)
    ctx = new_ctx()
    for n in range(1, 8):
        got = cam.undistortImage(raw, n, ctx)
        assert len(got) == n
        for l in range(n):
            np.testing.assert_array_equal(got[l], want[l], err_msg=f"{size}, {n} levels, level {l}")


@pytest.mark.gpu
def test_undistort_copy_camera_past_65535_frames(pkg):
    raw = np.random.default_rng(7700).integers(0, 256, (70001, 8, 16), dtype=np.uint8)
    got = pkg.PinholeCamera(16, 8, 12.0, 12.0, 7.5, 3.5).undistortImage(raw, 3)
    for l, want in enumerate(np_pyramid(raw, 3)):
        np.testing.assert_array_equal(got[l], want, err_msg=f"level {l}")


@pytest.mark.gpu
def test_undistort_distorted_camera_seven_levels(remap_kernels, uo, pkg, abi):
    from test_undistort import frames, params

    raw = frames(PINCUSHION, 3, seed=7800)
    got = pkg.PinholeCamera(*params(PINCUSHION)).undistortImage(raw, 7)
    rect = uo.undistort(abi, cam_struct(abi, PINCUSHION), raw, 1, n_threads=8)[0]
    want = np_pyramid(rect, 7)
    for l in range(7):
        np.testing.assert_array_equal(got[l], want[l], err_msg=f"level {l}")


# ---- levels the alignment derives -----------------------------------------------------------------------------------------
def big_cam(synth):
    """2048 x 1536: level 7 is 16 x 12 pixels.  make_align_batch's default margin (512 px at max_level 7) keeps the
    features inside level 7's in-frame box."""
    return synth.Camera(2048, 1536, 1400.0, 1400.0, 1023.5, 767.5)


def shipped(data, levels):
    o = copy.copy(data)
    o.ref_pyr = {l: data.ref_pyr[l] for l in levels}
    o.cur_pyr = {l: data.cur_pyr[l] for l in levels}
    return o


def in_range(data, max_level, min_level):
    return shipped(data, range(min_level, max_level + 1))


def same(got, want, what):
    for f in FIELDS:
        np.testing.assert_array_equal(getattr(got, f), getattr(want, f), err_msg=f"{what}: {f}")


@pytest.fixture(scope="module")
def level7(synth, abi, oracle, gen_device):
    """Eight pairs at 2048 x 1536, every level 0..7, and the oracle's alignment at levels 7 -> 5."""
    data = synth.make_align_batch(cam=big_cam(synth), batch=8, n_pts=300, n_segs=80, max_level=7, min_level=5, keep_levels_only=False,
                                  device=gen_device, seed=7900)
    ref = oracle.align(abi, data, abi.align_params(7, 5, 30), n_threads=8)
    return data, ref


def test_oracle_runs_level_7_on_every_pair(level7):
    data, ref = level7
    assert data.ref_pyr[7].shape[1:] == (12, 16)
    assert (ref.iters[:, 7] > 0).all(), ref.iters[:, 7]


def atan_kernels_or_skip(pkg, ex):
    if "without the ATAN alignment kernels" in str(ex) and os.environ.get("PLSVO_LIB"):
        pytest.skip(f"{os.environ['PLSVO_LIB']}: {ex}")
    raise ex


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["two_stacks", "chain", "three_leg", "atan", "track"])
def test_level_7_derived_from_level_0(pkg, abi, synth, oracle, gen_device, level7, monkeypatch, request, new_ctx, form):
    """Only level 0 shipped, max_level 7: levels 1..7 come from two launches of the pyramid kernel per frame stack.  Every
    output equals the same call with levels 5..7 shipped, byte for byte (one kernel variant pinned), and the oracle's
    alignment, which runs level-7 passes on every pair."""
    monkeypatch.setenv("PLSVO_VARIANT", "128,4")
    params = abi.align_params(7, 5, 30)
    ctx = new_ctx()
    stacks = 1 if form == "chain" else 2
    if form in ("two_stacks", "three_leg"):
        data, ref = level7

        def run(d):
            al = pkg.SparseImgAlign(7, 5, 30, ctx=ctx)
            if form == "two_stacks":
                return al.run(d)
            al.upload(d)
            al.launch()
            return al.download()
        (full, n_full), (lean, n_lean) = counted(ctx, lambda: run(in_range(data, 7, 5))), counted(ctx, lambda: run(shipped(data, [0])))
    elif form == "chain":
        data = synth.make_chain_batch(cam=big_cam(synth), batch=8, n_pts=300, n_segs=80, max_level=7, min_level=5, keep_levels_only=False,
                                      device=gen_device, seed=7910)
        ref = oracle.align(abi, data, params, n_threads=8)
        runs = []
        for levels in (range(5, 8), [0]):
            o = copy.copy(data)
            o.frame_pyr = synth.chain_frames(data, list(levels))
            runs.append(counted(ctx, lambda: pkg.SparseImgAlign(7, 5, 30, ctx=ctx).run(o)))
        (full, n_full), (lean, n_lean) = runs
    elif form == "atan":
        cam = atan_for(pkg, big_cam(synth), 0.3)
        data = synth.make_align_batch(cam=big_cam(synth), batch=8, n_pts=300, n_segs=80, max_level=7, min_level=5, keep_levels_only=False,
                                      device=gen_device, seed=7920, atan=cam)
        data = through(cam, data, lean=False)
        try:
            full, n_full = counted(ctx, lambda: pkg.SparseImgAlign(7, 5, 30, ctx=ctx).run(in_range(data, 7, 5), camera=cam))
        except pkg.api.PlsvoError as ex:
            atan_kernels_or_skip(pkg, ex)
        lean, n_lean = counted(ctx, lambda: pkg.SparseImgAlign(7, 5, 30, ctx=ctx).run(shipped(data, [0]), camera=cam))
        ref = reference(abi, request.getfixturevalue("oracle_atan"), cam, data)
    else:
        data, po = synth.make_track_batch(cam=big_cam(synth), batch=8, n_pts=300, n_segs=80, max_level=7, min_level=5,
                                          keep_levels_only=False, device=gen_device, seed=7930)
        ref = oracle.align(abi, data, params, n_threads=8)
        (fa, fp), n_full = counted(ctx, lambda: pkg.api.track(in_range(data, 7, 5), po, max_level=7, min_level=5, ctx=ctx))
        (la, lp), n_lean = counted(ctx, lambda: pkg.api.track(shipped(data, [0]), po, max_level=7, min_level=5, ctx=ctx))
        for f in ("T_f_w", "cov", "estimated_scale", "error_init", "error_final", "num_obs_pt", "num_obs_ls", "pt_outlier", "seg_outlier"):
            np.testing.assert_array_equal(getattr(lp, f), getattr(fp, f), err_msg=f)
        full, lean = fa, la
    assert (ref.iters[:, 7] > 0).all(), f"{form}: the oracle skips level 7 on some pair: {ref.iters[:, 7]}"
    assert n_lean - n_full == 2 * stacks, f"{form}: {n_lean} kernels with level 0 shipped, {n_full} with levels 5..7"
    same(lean, full, form)
    if form == "atan":
        compare(synth, lean, ref, "ATAN d0=0.3, level 0 -> 7")
    else:
        _check(synth, lean, ref)


@pytest.mark.gpu
def test_level_7_after_a_call_with_other_images(pkg, abi, synth, gen_device, level7, monkeypatch, new_ctx):
    """The derived-level buffers of a context hold the previous call's levels: a second call must overwrite all of them."""
    monkeypatch.setenv("PLSVO_VARIANT", "128,4")
    data, ref = level7
    other = synth.make_align_batch(cam=big_cam(synth), batch=8, n_pts=300, n_segs=80, max_level=7, min_level=5, keep_levels_only=False,
                                   device=gen_device, seed=7940)
    al = pkg.SparseImgAlign(7, 5, 30, ctx=new_ctx())
    al.run(shipped(other, [0]))
    lean = al.run(shipped(data, [0]))
    same(lean, pkg.SparseImgAlign(7, 5, 30, ctx=new_ctx()).run(in_range(data, 7, 5)), "second call on one context")
    _check(synth, lean, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["level_1_to_7", "level_0_to_6", "gated_level_0_to_6", "word_pitch_level_0_to_6"])
def test_derived_level_controls(pkg, abi, synth, oracle, gen_device, level7, monkeypatch, new_ctx, case):
    """One launch of the pyramid kernel per stack (level 1 -> 7, level 0 -> 6), and levels the alignment kernel derives
    itself, with no pyramid launch: the arrival-gated stream (256 pairs, level 0 shipped and aligned down to level 0), and
    a level 0 whose rows are word- but not 16-byte aligned.  The kernel counts pin each case to its path."""
    monkeypatch.setenv("PLSVO_VARIANT", "128,4")
    ctx = new_ctx()
    if case in ("level_1_to_7", "level_0_to_6"):
        data, ref = level7
        top, src = (7, 1) if case == "level_1_to_7" else (6, 0)
        full, n_full = counted(ctx, lambda: pkg.SparseImgAlign(top, 5, 30, ctx=ctx).run(in_range(data, top, 5)))
        lean, n_lean = counted(ctx, lambda: pkg.SparseImgAlign(top, 5, 30, ctx=ctx).run(shipped(data, [src])))
        assert (n_full, n_lean) == (1, 3), (case, n_full, n_lean)
        same(lean, full, case)
        _check(synth, lean, ref if top == 7 else oracle.align(abi, data, abi.align_params(6, 5, 30), n_threads=8))
        return
    if case == "gated_level_0_to_6":  # 256 pairs: the streamed call
        cam, B, n_pts, n_segs, lo = synth.Camera(1024, 768, 700.0, 700.0, 511.5, 383.5), 256, 60, 8, 0
    else:  # 756-byte rows
        cam, B, n_pts, n_segs, lo = synth.Camera(756, 768, 500.0, 500.0, 377.5, 383.5), 8, 300, 80, 4
    data = synth.make_align_batch(cam=cam, batch=B, n_pts=n_pts, n_segs=n_segs, max_level=6, min_level=lo, keep_levels_only=False,
                                  device=gen_device, seed=7950 + B)
    full, n_full = counted(ctx, lambda: pkg.SparseImgAlign(6, lo, 30, ctx=ctx).run(in_range(data, 6, lo)))
    lean, n_lean = counted(ctx, lambda: pkg.SparseImgAlign(6, lo, 30, ctx=ctx).run(shipped(data, [0])))
    assert (n_full, n_lean) == (1, 1), (case, n_full, n_lean)
    same(lean, full, case)
    if B <= 8:
        _check(synth, lean, oracle.align(abi, data, abi.align_params(6, lo, 30), n_threads=8))
