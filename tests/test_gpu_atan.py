"""Alignment and tracking of frames from an ATAN (FOV) camera on the device (plsvo_align_atan_batch_run /
plsvo_track_atan_batch_run) against the CPU oracle's ATAN path (oracle/atan_oracle.cpp): cameras with no, mild and strong
distortion (frames and features rendered through that camera, synth.make_align_batch(atan=...)), batch sizes 1 / 37 /
1024, two level ranges, full and lean features, two stacks and frame chains, ragged counts and masks, levels derived on
the device, an odd-sized camera, the track call with the pose optimiser's outputs, and reference-typed frames through
the drop-in shim.  Where oracle/_ref is built, the comparison is with the reference's own SparseImgAlign through the
stand-in camera.  Counts, iterations, status
and flags must be equal and poses within the tolerance of tests/test_gpu_track.py; the number of pairs whose pose and H
are byte-identical is reported."""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oracle_atan(abi):
    import oracle_atan

    oracle_atan.build()
    oracle_atan.load(abi)
    return oracle_atan


def atan_for(pkg, cam, d0):
    w, h = cam.width, cam.height
    return pkg.ATANCamera(w, h, cam.fx / w, cam.fy / h, (cam.cx + 0.5) / w, (cam.cy + 0.5) / h, d0)


def through(camera, data, lean):
    """The batch's features as `camera` forms them: bearings are its cam2world of the pixels (NULL when lean: formed on
    the device and by the oracle).  The frames and 3-D points come from synth's ATAN rendering (make_*_batch(atan=...))."""
    d = copy.copy(data)
    if lean:
        d.pt_f = d.seg_sf = d.seg_ef = None
    else:
        d.pt_f = np.ascontiguousarray(camera.cam2world(data.pt_px))
        d.seg_sf = np.ascontiguousarray(camera.cam2world(data.seg_spx))
        d.seg_ef = np.ascontiguousarray(camera.cam2world(data.seg_epx))
    return d


def reference(abi, oracle_atan, cam, data):
    """The reference's own SparseImgAlign through the stand-in camera (oracle/_ref) where it is built, else the oracle."""
    if oracle_atan.ref_available():
        return oracle_atan.ref_align(abi, cam, data, n_threads=16)
    return oracle_atan.align(abi, cam, data, n_threads=16)


def ragged(data, seed):
    """Ragged counts and masks.  Every pair keeps at least a quarter of its points, except pair 0, which has no features
    at all (the early-out).  Pairs left with one to three points are not used: there a one-ulp difference in the
    projection flips an accept / reject decision of the almost unconstrained solve, on the pinhole path as on the ATAN
    one (measured on an H100: 7 of 1024 such pairs differ in iteration counts for the pinhole kernel, 9 for ATAN d0=0.93,
    all with pt_count <= 3), so they test the conditioning of the system, not the camera model."""
    rng = np.random.default_rng(seed)
    d = copy.copy(data)
    d.pt_count = rng.integers(d.n_pts // 4, d.n_pts + 1, d.batch).astype(np.int32)
    d.seg_count = rng.integers(0, d.n_segs + 1, d.batch).astype(np.int32)
    d.pt_count[0] = d.seg_count[0] = 0
    d.pt_valid = (rng.random((d.batch, d.n_pts)) > 0.1).astype(np.uint8)
    d.seg_valid = (rng.random((d.batch, d.n_segs)) > 0.1).astype(np.uint8)
    return d


def compare(synth, got, ref, what, data=None):
    np.testing.assert_array_equal(got.n_tracked, ref.n_tracked, err_msg=what)
    np.testing.assert_array_equal(got.iters, ref.iters, err_msg=what)
    np.testing.assert_array_equal(got.status, ref.status, err_msg=what)
    np.testing.assert_array_equal(got.seg_killed, ref.seg_killed, err_msg=what)
    ang, rel = synth.pose_error(got.T_cur_w, ref.T_cur_w)
    assert ang.max() <= 1e-5 and rel.max() <= 1e-4, (what, ang.max(), rel.max())
    same = int(np.sum(np.all(got.T_cur_w == ref.T_cur_w, 1) & np.all(got.H == ref.H, 1)))
    if data is not None:  # pairs without features return the input pose and H = 0 on both sides: always byte-identical
        empty = (data.pt_count == 0) & (data.seg_count == 0) if data.pt_count is not None else np.zeros(data.batch, bool)
        assert same >= int(empty.sum()), (what, same, int(empty.sum()))
    print(f"{what}: {same}/{got.T_cur_w.shape[0]} pairs byte-identical (pose and H); max rot err {ang.max():.2e}, rel-t {rel.max():.2e}")


CASES = [  # (d0, batch, levels, lean, chain, ragged); the frames are rendered through the ATAN camera of d0
    (0.0, 37, (4, 2), False, False, False),
    (0.3, 37, (4, 2), False, False, True),
    (0.93, 37, (4, 2), True, False, False),
    (0.3, 1, (3, 0), True, False, False),
    (0.93, 37, (3, 0), False, True, False),
    (0.3, 37, (4, 2), True, True, True),
    (0.93, 1024, (4, 2), False, False, True),
    (0.3, 1024, (4, 2), True, True, False),
]


@pytest.mark.parametrize("d0,batch,levels,lean,chain,rag", CASES)
def test_atan_alignment_matches_the_oracle(pkg, abi, synth, oracle_atan, gen_device, d0, batch, levels, lean, chain, rag):
    mk = synth.make_chain_batch if chain else synth.make_align_batch
    n_pts = 120 if batch == 1024 else 300
    cam = atan_for(pkg, synth.VGA, d0)
    data = mk(batch=batch, n_pts=n_pts, n_segs=40, max_level=levels[0], min_level=levels[1], seed=8100 + batch, device=gen_device,
              atan=cam)
    if chain:
        data.frame_pyr = synth.chain_frames(data)
    data = through(cam, data, lean)
    if rag:
        data = ragged(data, 8200 + batch)
    got = pkg.SparseImgAlign(levels[0], levels[1], 30).run(data, camera=cam)
    two_stacks = copy.copy(data)
    two_stacks.frame_pyr = None  # the oracle reads the same frames as two stacks
    ref = reference(abi, oracle_atan, cam, two_stacks)
    compare(synth, got, ref, f"d0={d0} B={batch} levels={levels} lean={lean} chain={chain} ragged={rag}", data)


def test_atan_alignment_levels_derived_on_the_device(pkg, abi, synth, oracle_atan, gen_device):
    """Lean features and only level min_level shipped: levels above it are half-sampled on the device."""
    cam = atan_for(pkg, synth.VGA, 0.93)
    data = through(cam, synth.make_align_batch(batch=37, n_pts=300, n_segs=40, seed=8150, device=gen_device, atan=cam), lean=True)
    ref = reference(abi, oracle_atan, cam, data)
    shipped = copy.copy(data)
    shipped.ref_pyr = {2: data.ref_pyr[2]}
    shipped.cur_pyr = {2: data.cur_pyr[2]}
    got = pkg.SparseImgAlign(4, 2, 30).run(shipped, camera=cam)
    compare(synth, got, ref, "d0=0.93 levels 3, 4 derived on the device")


@pytest.mark.parametrize("d0", [0.3, 0.93])
def test_atan_alignment_recovers_the_pose_of_an_atan_scene(pkg, synth, gen_device, d0):
    """Frames rendered through the ATAN camera: aligning them with that camera model converges to the true motion, and
    aligning them as if they were pinhole frames does markedly worse."""
    cam = atan_for(pkg, synth.VGA, d0)
    data = synth.make_align_batch(batch=16, n_pts=300, n_segs=80, seed=8600, device=gen_device, atan=cam)
    gpu = pkg.SparseImgAlign(4, 2, 30).run(data, camera=cam)
    ang0, rel0 = synth.pose_error(data.T_cur_w, data.T_cur_w_gt)
    ang, rel = synth.pose_error(gpu.T_cur_w, data.T_cur_w_gt)
    assert np.median(ang) < 0.2 * np.median(ang0) and np.median(rel) < 0.2 * np.median(rel0), (np.median(ang), np.median(ang0))
    pin = pkg.SparseImgAlign(4, 2, 30).run(data)  # the same frames and features, distortion ignored
    ang_p, rel_p = synth.pose_error(pin.T_cur_w, data.T_cur_w_gt)
    print(f"d0={d0}: median rot err {np.median(ang):.2e} (ATAN model) vs {np.median(ang_p):.2e} (pinhole model), initial {np.median(ang0):.2e}")
    assert np.median(rel) < np.median(rel_p)


def test_atan_alignment_odd_sized_camera(pkg, abi, synth, oracle_atan, gen_device):
    cam = atan_for(pkg, synth.ODD, 0.3)
    data = synth.make_align_batch(cam=synth.ODD, batch=37, n_pts=300, n_segs=40, seed=8300, device=gen_device, atan=cam)
    data = through(cam, data, lean=True)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, camera=cam)
    compare(synth, got, reference(abi, oracle_atan, cam, data), "641x479 d0=0.3")


def test_reference_typed_atan_frames_through_the_shim(pkg, abi, synth, oracle_atan, gen_device):
    """The reference's own Frame / Feature objects with a vk::ATANCamera through the drop-in SparseImgAlign::run: the shim
    finds the camera model through the frame and takes the ATAN path (same results as the direct ATAN call)."""
    if not oracle_atan.build_shimref():
        pytest.skip("oracle/_ref/libplsvo_atan_shimref.so is not built and the reference sources are absent")
    cam = atan_for(pkg, synth.VGA, 0.93)
    data = through(cam, synth.make_align_batch(batch=8, n_pts=300, n_segs=60, seed=8700, device=gen_device, atan=cam), lean=False)
    got = oracle_atan.shimref_align(abi, cam, data)
    direct = pkg.SparseImgAlign(4, 2, 30).run(data, camera=cam)
    # as tests/test_gpu_shim.py: the poses make a trip through the reference's SE3 (the quaternion is re-normalised), so
    # they agree to round-off; the decisions agree exactly
    np.testing.assert_array_equal(got.n_tracked, direct.n_tracked)
    np.testing.assert_array_equal(got.seg_killed, direct.seg_killed)
    ang, rel = synth.pose_error(got.T_cur_w, direct.T_cur_w)
    assert ang.max() <= 1e-9 and rel.max() <= 1e-8, (ang.max(), rel.max())
    pinhole = pkg.SparseImgAlign(4, 2, 30).run(data)
    assert not np.array_equal(got.T_cur_w, pinhole.T_cur_w)


@pytest.mark.parametrize("d0", [0.0, 0.93])
def test_atan_track_matches_the_oracle_chain(pkg, abi, synth, oracle, oracle_atan, gen_device, d0):
    cam = atan_for(pkg, synth.VGA, d0)
    al, po = synth.make_track_batch(batch=37, n_pts=300, n_segs=80, seed=8400, device=gen_device, atan=cam)
    al = through(cam, al, lean=False)
    po = copy.copy(po)
    po.fx = cam.errorMultiplier2()
    ao, pout = pkg.api.track(al, po, camera=cam)
    ra = reference(abi, oracle_atan, cam, al)
    compare(synth, ao, ra, f"track d0={d0}")
    po3 = copy.copy(po)
    po3.T_f_w = np.ascontiguousarray(ra.T_cur_w)
    rp = oracle.poseopt(abi, po3, abi.poseopt_params(2.0, 10, -1), n_threads=16)
    ang, rel = synth.pose_error(pout.T_f_w, rp.T_f_w)
    assert ang.max() <= 1e-5 and rel.max() <= 1e-4, (ang.max(), rel.max())
    for f in ("num_obs_pt", "num_obs_ls", "pt_outlier", "seg_outlier", "iters", "status"):
        np.testing.assert_array_equal(getattr(pout, f), getattr(rp, f), err_msg=f)


def test_malformed_atan_calls_are_rejected_before_anything_is_queued(pkg, abi, synth, gen_device):
    import ctypes as C

    data = synth.make_align_batch(batch=4, n_pts=32, n_segs=8, seed=8500, device=gen_device)
    ctx = pkg.default_context()
    batch, keep = abi.make_align_batch(data)
    params = abi.align_params()
    out = abi.AlignOut(data.batch, data.n_segs)
    good = atan_for(pkg, synth.VGA, 0.3)
    launches = ctx.launch_count()
    for bad in (abi.AtanCamera(641, 480, 0.65625, 0.875, 0.5, 0.5, 0.3),  # size differs from batch.cam
                abi.AtanCamera(640, 480, 0.0, 0.875, 0.5, 0.5, 0.3),      # fx <= 0
                abi.AtanCamera(640, 480, -0.6, 0.875, 0.5, 0.5, 0.3),
                abi.AtanCamera(640, 480, 0.65625, 0.875, 0.5, 0.5, float("nan"))):  # NaN d0
        rc = ctx.lib.plsvo_align_atan_batch_run(ctx.handle, C.byref(bad), C.byref(batch), C.byref(params), C.byref(out.struct))
        assert rc == abi.ERR_INVALID, rc
        assert b"plsvo_atan_camera" in ctx.lib.plsvo_last_error(ctx.handle)
    assert ctx.launch_count() == launches
    # the pinhole call on the same context is unaffected by the ATAN ones
    pin = pkg.SparseImgAlign(4, 2, 30).run(data)
    rc = ctx.lib.plsvo_align_atan_batch_run(ctx.handle, C.byref(good.struct), C.byref(batch), C.byref(params), C.byref(out.struct))
    assert rc == 0
    again = pkg.SparseImgAlign(4, 2, 30).run(data)
    np.testing.assert_array_equal(again.T_cur_w, pin.T_cur_w)
