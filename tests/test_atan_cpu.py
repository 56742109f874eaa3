"""The ATAN (vk::ATANCamera) camera model without a GPU: the NumPy restatement (api.ATANCamera) against the C++ stand-in
(oracle/refdeps/vikit/atan_camera.h), its round trip, and the oracle's ATAN alignment path against its pinhole path when
the camera has no distortion (d0 = 0)."""
import copy

import numpy as np
import pytest


@pytest.fixture(scope="module")
def oracle_atan(abi):
    import oracle_atan

    oracle_atan.build()
    oracle_atan.load(abi)
    return oracle_atan


def vga_atan(pkg, synth, d0, cam=None):
    """The ATAN camera whose derived members equal the undistorted pinhole `cam`: fx_ = w fx, cx_ = w cx - 0.5."""
    cam = cam or synth.VGA
    w, h = cam.width, cam.height
    return pkg.ATANCamera(w, h, cam.fx / w, cam.fy / h, (cam.cx + 0.5) / w, (cam.cy + 0.5) / h, d0)


@pytest.mark.parametrize("d0", [0.0, 0.3, 0.93])
def test_numpy_camera_matches_the_cpp_stand_in(pkg, abi, synth, oracle_atan, d0):
    cam = vga_atan(pkg, synth, d0)
    rng = np.random.default_rng(11)
    px = np.stack([rng.uniform(0, 640, 4000), rng.uniform(0, 480, 4000)], -1)
    px[:4] = [[cam.cx_, cam.cy_], [cam.cx_ + 1e-3, cam.cy_], [0, 0], [639.5, 479.5]]  # centre, r < 0.01, corners
    f_np, f_cpp = cam.cam2world(px), oracle_atan.cam2world(abi, cam, px)
    np.testing.assert_allclose(f_np, f_cpp, rtol=0, atol=1e-15)
    xyz = np.concatenate([rng.uniform(-1, 1, (4000, 2)), rng.uniform(0.5, 3, (4000, 1))], -1)
    xyz[:2] = [[0, 0, 1], [1e-4, 0, 1]]  # r < 0.001: no distortion factor
    np.testing.assert_allclose(cam.world2cam(xyz), oracle_atan.world2cam(abi, cam, xyz), rtol=0, atol=1e-9)
    assert cam.errorMultiplier2() == oracle_atan.error_multiplier2(abi, cam) == 640 * cam.struct.fx
    # round trip world2cam(cam2world(px)) within 1e-9 px.  The model itself is not its own inverse near the principal
    # point: cam2world skips the distortion within r_d <= 0.01 of it, world2cam only within r < 0.001 — there (about 6 px
    # around the centre of a VGA image) the round trip misses by up to d0-dependent hundredths of a pixel, upstream too.
    rd = np.hypot((px[:, 0] - cam.cx_) / cam.fx_, (px[:, 1] - cam.cy_) / cam.fy_)
    ok = (rd > 0.01) | (d0 == 0.0)
    assert ok.sum() > 3900
    np.testing.assert_allclose(cam.world2cam(f_np)[ok], px[ok], rtol=0, atol=1e-9)
    np.testing.assert_allclose(oracle_atan.world2cam(abi, cam, f_cpp)[ok], px[ok], rtol=0, atol=1e-9)


def test_constructor_derives_the_members_as_documented(pkg):
    cam = pkg.ATANCamera(641, 479, 0.6, 0.8, 0.51, 0.49, 0.93)
    assert cam.fx_ == 641 * 0.6 and cam.fy_ == 479 * 0.8
    assert cam.cx_ == 0.51 * 641 - 0.5 and cam.cy_ == 0.49 * 479 - 0.5
    assert cam.tans_ == 2.0 * np.tan(0.93 / 2.0) and cam.s_inv_ == 1.0 / 0.93
    flat = pkg.ATANCamera(640, 480, 0.6, 0.8, 0.5, 0.5, 0.0)
    assert flat.tans_ == flat.s_inv_ == flat.tans_inv_ == 0.0


@pytest.mark.parametrize("levels", [(4, 2), (3, 0)])
def test_without_distortion_the_atan_path_is_the_pinhole_path(pkg, abi, synth, oracle, oracle_atan, levels):
    """d0 = 0: every output of the oracle's ATAN path equals its pinhole path's, bit for bit."""
    data = synth.make_align_batch(batch=6, n_pts=200, n_segs=40, max_level=levels[0], min_level=levels[1], seed=7100)
    cam = vga_atan(pkg, synth, 0.0)
    assert (cam.fx_, cam.fy_, cam.cx_, cam.cy_) == (synth.VGA.fx, synth.VGA.fy, synth.VGA.cx, synth.VGA.cy)
    pin = oracle.align(abi, data, n_threads=4)
    at = oracle_atan.align(abi, cam, data, n_threads=4)
    for f in ("T_cur_w", "n_tracked", "H", "seg_killed", "iters", "status", "patch_iters", "patch_levels"):
        np.testing.assert_array_equal(getattr(at, f), getattr(pin, f), err_msg=f)
    # and the bearings it forms itself (NULL pt_f / seg_sf / seg_ef) are the pinhole cam2world's
    lean = copy.copy(data)
    lean.pt_f = lean.seg_sf = lean.seg_ef = None
    np.testing.assert_array_equal(cam.cam2world(data.pt_px), oracle_atan.cam2world(abi, cam, data.pt_px.reshape(-1, 2)).reshape(data.pt_f.shape))
    at_lean = oracle_atan.align(abi, cam, lean, n_threads=4)
    full = copy.copy(data)
    full.pt_f = np.ascontiguousarray(cam.cam2world(data.pt_px))
    full.seg_sf, full.seg_ef = (np.ascontiguousarray(cam.cam2world(x)) for x in (data.seg_spx, data.seg_epx))
    ref = oracle.align(abi, full, n_threads=4)
    for f in ("T_cur_w", "n_tracked", "H", "seg_killed", "iters", "status"):
        np.testing.assert_array_equal(getattr(at_lean, f), getattr(ref, f), err_msg=f)


def test_distortion_changes_the_result(pkg, abi, synth, oracle_atan):
    """The distortion term is live: d0 = 0.3 and d0 = 0 align the same batch to different poses."""
    data = synth.make_align_batch(batch=4, n_pts=150, n_segs=30, seed=7200)
    a0 = oracle_atan.align(abi, vga_atan(pkg, synth, 0.0), data)
    a3 = oracle_atan.align(abi, vga_atan(pkg, synth, 0.3), data)
    assert not np.array_equal(a0.T_cur_w, a3.T_cur_w)


def test_abi_declares_the_atan_entry_points(abi):
    names = {n for n, _, _ in abi.ABI_SYMBOLS}
    assert {"plsvo_align_atan_batch_run", "plsvo_track_atan_batch_run"} <= names


@pytest.mark.parametrize("levels", [(4, 2), (3, 0)])
@pytest.mark.parametrize("d0", [0.0, 0.3, 0.93])
def test_oracle_atan_path_equals_the_reference_bit_for_bit(pkg, abi, synth, oracle_atan, d0, levels):
    """oracle/atan_oracle.cpp against the reference's own sparse_img_align.cpp driven with the stand-in vk::ATANCamera
    (oracle/_ref/libplsvo_atan_ref.so), on frames and features rendered through that camera; full and lean features."""
    if not oracle_atan.build_ref():
        pytest.skip("oracle/_ref/libplsvo_atan_ref.so is not built and the reference sources are absent")
    cam = vga_atan(pkg, synth, d0, synth.QVGA)
    data = synth.make_align_batch(cam=synth.QVGA, batch=4, n_pts=120, n_segs=24, max_level=levels[0], min_level=levels[1],
                                  seed=7300, atan=cam)
    data.pt_f = np.ascontiguousarray(cam.cam2world(data.pt_px))
    data.seg_sf, data.seg_ef = (np.ascontiguousarray(cam.cam2world(x)) for x in (data.seg_spx, data.seg_epx))
    lean = copy.copy(data)
    lean.pt_f = lean.seg_sf = lean.seg_ef = None
    for d in (data, lean):
        got, ref = oracle_atan.align(abi, cam, d, n_threads=4), oracle_atan.ref_align(abi, cam, d, n_threads=4)
        for f in ("T_cur_w", "n_tracked", "H", "seg_killed", "iters", "status"):
            np.testing.assert_array_equal(getattr(got, f), getattr(ref, f), err_msg=f)
        assert got.n_tracked.min() > 0
