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


# ------------------------------------------------------------------------------------------------
# the model in extended precision at the d0 values and cut-offs of tests/test_gpu_atan_cases.py
# ------------------------------------------------------------------------------------------------

EDGE_D0 = [-0.3, 1e-9, 0.93, 1.4, 2.4]
EPS = np.finfo(np.float64).eps


def _ld_cam2world(cam, px):
    """cam2world in np.longdouble from the camera's double members; also returns r_d and whether the factor applies."""
    L = np.longdouble
    px = np.asarray(px, L)
    x, y = (px[:, 0] - L(cam.cx_)) / L(cam.fx_), (px[:, 1] - L(cam.cy_)) / L(cam.fy_)
    rd = np.sqrt(x * x + y * y)
    r = np.tan(rd * L(cam.s_)) * L(cam.tans_inv_) if cam.s_ != 0.0 else rd
    applies = rd > L(0.01)
    factor = np.where(applies, r / np.where(applies, rd, 1), L(1))
    x, y = factor * x, factor * y
    n = np.sqrt(x * x + y * y + 1)
    return np.stack([x / n, y / n, 1 / n], -1), rd, applies


def _ld_world2cam(cam, xyz):
    L = np.longdouble
    xyz = np.asarray(xyz, L)
    u, v = xyz[:, 0] / xyz[:, 2], xyz[:, 1] / xyz[:, 2]
    r = np.sqrt(u * u + v * v)
    applies = ~((r < L(0.001)) | (cam.s_ == 0.0))
    f = L(cam.s_inv_) * np.arctan(r * L(cam.tans_)) / np.where(r > 0, r, 1)
    factor = np.where(applies, f, L(1))
    return np.stack([L(cam.cx_) + L(cam.fx_) * factor * u, L(cam.cy_) + L(cam.fy_) * factor * v], -1), applies


@pytest.mark.parametrize("d0", EDGE_D0)
def test_camera_model_against_extended_precision(pkg, abi, synth, oracle_atan, d0):
    """api.ATANCamera and the C++ stand-in against the model evaluated in long double: the same branch at both cut-offs
    (at r_d == 0.01 exactly and at r == 0 too) and within a few ulp, scaled by the conditioning of tan near pi/2."""
    import test_gpu_atan_cases as cases

    for cam in (vga_atan(pkg, synth, d0), cases._telephoto(pkg, synth, cases.C2W_FX, d0)[0]):
        _model_against_extended_precision(abi, oracle_atan, cases, cam, d0)


def _model_against_extended_precision(abi, oracle_atan, cases, cam, d0):
    rng = np.random.default_rng(12)
    c = np.array([cam.cx_, cam.cy_])
    px = np.concatenate([np.stack([rng.uniform(0, 640, 3000), rng.uniform(0, 480, 3000)], -1),
                         [c, cases.rd_exactly_001(cam) if cam.fx_ == cases.C2W_FX else c],  # the VGA camera has no such pixel
                         c + cases._in_annulus(rng, (200,), 0.0, 0.0099 * cam.fx_, (0, 0)),     # inside r_d <= 0.01
                         c + cases._in_annulus(rng, (200,), 0.0101 * cam.fx_, 0.011 * cam.fx_, (0, 0))])  # just outside
    ld, rd, applies = _ld_cam2world(cam, px)
    assert rd[3000] == 0 and cases.rd_of(cam, px[3001:3002])[0] == (0.01 if cam.fx_ == cases.C2W_FX else 0) and not applies[3000:3202].any() and applies[3202:].all()
    x = np.abs(rd * abs(d0)).astype(np.float64)
    kappa = np.where(x > 0, x * (1 + np.tan(x) ** 2) / np.maximum(np.abs(np.tan(x)), 1e-300), 1.0)  # relative condition of tan
    keep = np.abs(x - np.pi / 2) > 1e-3  # at the pole itself no precision is defined
    tol = 8 * EPS * (1 + kappa[keep, None])
    for got in (cam.cam2world(px), oracle_atan.cam2world(abi, cam, px)):
        assert (np.abs(got[keep] - ld[keep].astype(np.float64)) <= tol).all()
        # the branch: with the other one the bearing would be off by the factor's jump, far beyond the tolerance
        flat = px[~applies]
        xy = (flat - c) / [cam.fx_, cam.fy_]
        n = np.sqrt((xy ** 2).sum(1) + 1)
        np.testing.assert_array_equal(got[~applies], np.concatenate([xy / n[:, None], 1 / n[:, None]], 1))

    xyz = np.concatenate([rng.uniform(-1, 1, (3000, 2)), rng.uniform(0.5, 3, (3000, 1))], -1)
    ring = lambda r0, r1, n: np.concatenate([cases._in_annulus(rng, (n,), r0, r1, (0, 0)), np.ones((n, 1))], 1)
    xyz = np.concatenate([xyz, [[0, 0, 1], [0, 0, 2.5]], ring(0, 0.00099, 200), ring(0.00101, 0.0011, 200)])
    ld, applies = _ld_world2cam(cam, xyz)
    assert not applies[3000:3202].any() and applies[3202:].all() == (d0 != 0)
    for got in (cam.world2cam(xyz), oracle_atan.world2cam(abi, cam, xyz)):
        np.testing.assert_allclose(got, ld.astype(np.float64), rtol=8 * EPS, atol=8 * EPS * 640)
        np.testing.assert_array_equal(got[3000:3002], [c, c])  # r = 0: the guard, not 0/0


def test_atan_cases_fixtures_reach_their_branches(pkg, abi, synth, oracle_atan):
    """The fixtures of tests/test_gpu_atan_cases.py, built here as there: every cut-off fixture is inside (or just
    outside) its cut-off, r_d == 0.01 is hit exactly, d0 = 2.4 has feature pixels past pi/2, the non-square camera is told
    apart from its transpose by the oracle, and the world2cam pairs compared on the GPU stay inside r < 0.001."""
    import test_gpu_atan_cases as cases
    from test_gpu_align import ROT_TOL, TRANS_TOL

    cam, data = cases.cam2world_disc_batch(pkg, synth, "cpu")
    rd = cases.rd_of(cam, cases.feature_px(data))
    assert rd.max() == 0.01 and (rd == 0.01).sum() == data.batch and (rd == 0).sum() == data.batch
    cam, ring = cases.cam2world_disc_batch(pkg, synth, "cpu", ring=True)
    rd = cases.rd_of(cam, cases.feature_px(ring))
    assert rd.min() > 0.01 and rd.max() <= 0.011

    cam, data = cases.world2cam_disc_batch(pkg, synth, "cpu")
    flat = cases._telephoto(pkg, synth, cases.W2C_FX, 0.0)[0]
    r0 = cases.projected_r(data, data.T_cur_w)
    assert r0.max() < 0.0005 and r0[0, 0] == 0.0
    data = through(cam, data)
    inside, ref = cases.world2cam_inside_pairs(abi, oracle_atan, cam, flat, data)
    assert inside[0] and inside.sum() >= data.batch // 2, inside
    assert cases.projected_r(data, ref.T_cur_w)[inside].max() < 0.001

    cam, data = cases.d0_edge_batch(pkg, synth, "cpu", 2.4)
    assert (cases.rd_of(cam, cases.feature_px(data)) * 2.4 > np.pi / 2).sum() > 0

    cam, swapped = cases.nonsquare_cameras(pkg)
    assert (cam.fx_, cam.fy_) == (swapped.fy_, swapped.fx_) or abs(cam.fx_ - swapped.fy_) < 1e-12
    data = cases.nonsquare_batch(pkg, synth, "cpu")
    a, b = oracle_atan.align(abi, cam, data, n_threads=8), oracle_atan.align(abi, swapped, data, n_threads=8)
    ang, rel = synth.pose_error(a.T_cur_w, b.T_cur_w)
    assert ((ang > 100 * ROT_TOL) | (rel > 100 * TRANS_TOL)).all(), (ang.min(), rel.min())
    # the host model's entry takes the members the kernels receive: the same bytes as the normalised camera's
    m = oracle_atan.align_members(abi, cam, data, n_threads=8)
    for f in ("T_cur_w", "n_tracked", "H", "seg_killed", "iters", "status", "patch_iters", "patch_levels"):
        np.testing.assert_array_equal(getattr(m, f), getattr(a, f), err_msg=f)


def through(cam, data):
    """Full bearings of api.ATANCamera.cam2world, as test_gpu_atan.through(lean=False)."""
    d = copy.copy(data)
    d.pt_f = np.ascontiguousarray(cam.cam2world(data.pt_px))
    d.seg_sf, d.seg_ef = (np.ascontiguousarray(cam.cam2world(x)) for x in (data.seg_spx, data.seg_epx))
    return d
