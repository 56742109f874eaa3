"""Multicam batches on the device: frame pairs from differently calibrated pinhole cameras in one call
(plsvo_align_multicam_batch_run, plsvo_poseopt_multicam_batch_run, plsvo_track_multicam_batch_run).

The multicam kernels run the uniform kernels' expressions with the intrinsics read per pair, so every pair's outputs must
be byte-identical to the uniform three-leg call on that pair with batch->cam = its camera and the same kernel variant.
test_malformed_multicam_calls needs no kernel result: tests/test_multicam_cpu.py also runs it against the host model."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ALIGN_FIELDS = ("T_cur_w", "n_tracked", "H", "seg_killed", "iters", "status", "patch_iters", "patch_levels")
PO_FIELDS = ("T_f_w", "cov", "estimated_scale", "error_init", "error_final", "num_obs_pt", "num_obs_ls", "pt_outlier",
             "seg_outlier", "iters", "status")


def uniform_cameras(data):
    c = data.cam
    return np.tile([c.fx, c.fy, c.cx, c.cy], (data.batch, 1))


def three_leg(pkg, data, levels=(4, 2)):
    al = pkg.SparseImgAlign(levels[0], levels[1], 30)
    al.upload(data)
    al.launch()
    return al.download()


def assert_same(got, want, fields, rows=None, what="", want_rows=None):
    for f in fields:
        g, w = getattr(got, f), getattr(want, f)
        g = g if rows is None else g[rows]
        w = w if want_rows is None else w[want_rows]
        np.testing.assert_array_equal(g.view(np.uint8), w.view(np.uint8), err_msg=f"{what} {f}")


def ragged(data, seed, empty=(0,)):
    """Ragged point / segment counts, masked features, and the pairs `empty` without any feature."""
    rng = np.random.default_rng(seed)
    data.pt_count = rng.integers(0, data.n_pts + 1, data.batch).astype(np.int32)
    data.seg_count = rng.integers(0, data.n_segs + 1, data.batch).astype(np.int32)
    data.pt_valid = (rng.random((data.batch, data.n_pts)) > 0.1).astype(np.uint8)
    for b in empty:
        data.pt_count[b] = data.seg_count[b] = 0
    return data


def lean(data):
    """Bearings formed on the device from the pixels (cam2world through the pair's camera), depths instead of positions."""
    import plsvo_b200

    R, t = plsvo_b200.synth.pose7_to_Rt(torch.tensor(data.T_ref_w))
    ref_pos = -(R.transpose(-1, -2) @ t[..., None])[..., 0].numpy()
    data.pt_depth = np.ascontiguousarray(np.linalg.norm(data.pt_pos - ref_pos[:, None], axis=-1))
    data.pt_f = data.pt_pos = data.seg_sf = data.seg_ef = None
    return data


def derived_levels(data):
    """Only level 2 shipped: levels 3 and 4 are half-sampled on the device."""
    data.ref_pyr = {2: data.ref_pyr[2]}
    data.cur_pyr = {2: data.cur_pyr[2]}
    return data


# ---- uniform equivalence: cams[b] = batch->cam ----------------------------------------------------------------------


@pytest.mark.parametrize("batch", [37, 1024])
def test_uniform_cameras_equal_the_three_leg_call(pkg, synth, gen_device, batch):
    data = synth.make_align_batch(batch=batch, n_pts=300, n_segs=80, seed=9100 + batch, device=gen_device)
    want = three_leg(pkg, data)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, cameras=uniform_cameras(data))
    assert_same(got, want, ALIGN_FIELDS)


@pytest.mark.parametrize("variant", [f"{t},{b}" for t, b in
                                     ((64, 8), (96, 7), (96, 5), (128, 5), (128, 4), (160, 3), (192, 2), (256, 2))])
def test_uniform_cameras_every_variant(pkg, synth, gen_device, variant, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", variant)
    data = ragged(synth.make_align_batch(batch=37, n_pts=200, n_segs=60, seed=9200, device=gen_device), 9201)
    want = three_leg(pkg, data)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, cameras=uniform_cameras(data))
    assert_same(got, want, ALIGN_FIELDS, what=variant)


@pytest.mark.parametrize("case", ["chain", "lean", "derived_levels"])
def test_uniform_cameras_chain_lean_and_derived_levels(pkg, abi, synth, gen_device, case):
    if case == "chain":
        data = synth.make_chain_batch(batch=37, n_pts=300, n_segs=80, seed=9300, device=gen_device)
        data.frame_pyr = synth.chain_frames(data)
    else:
        data = synth.make_align_batch(batch=37, n_pts=300, n_segs=80, seed=9310, device=gen_device)
    if case == "lean":
        lean(data)
    if case == "derived_levels":
        derived_levels(data)
    want = three_leg(pkg, data)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, cameras=uniform_cameras(data))
    assert_same(got, want, ALIGN_FIELDS, what=case)
    assert (got.n_tracked > 0).any()


# ---- mixed batches: K = 4 cameras -----------------------------------------------------------------------------------


def mixed(synth, batch, seed, gen_device, poseopt=False):
    rng = np.random.default_rng(seed)
    cam_of_pair = rng.permutation(np.arange(batch) % 4)  # interleaved, then randomly permuted
    out = synth.make_multicam_batch(synth.MULTICAM_K4, cam_of_pair, n_pts=300, n_segs=80, seed=seed, device=gen_device,
                                    poseopt=poseopt)
    return cam_of_pair, out


@pytest.mark.parametrize("batch", [37, 1024])
def test_mixed_batch_equals_each_cameras_uniform_call(pkg, synth, gen_device, batch, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2" if batch <= 132 else "128,4")
    cam_of_pair, (data, cameras) = mixed(synth, batch, 9400 + batch, gen_device)
    ragged(data, 9401, empty=(0, batch // 2))
    got = pkg.SparseImgAlign(4, 2, 30).run(data, cameras=cameras)
    assert (got.status[[0, batch // 2]] == 1).all()
    for k, cam in enumerate(synth.MULTICAM_K4):
        idx = np.flatnonzero(cam_of_pair == k)
        sub = synth.take_pairs(data, idx)
        sub.cam = cam
        assert_same(got, three_leg(pkg, sub), ALIGN_FIELDS, rows=idx, what=f"camera {k}")
    # the intrinsics matter: the same pairs through one camera give other poses
    wrong = pkg.SparseImgAlign(4, 2, 30).run(data, cameras=uniform_cameras(data))
    assert not np.array_equal(wrong.T_cur_w, got.T_cur_w)


@pytest.mark.parametrize("case", ["lean", "derived_levels"])
def test_mixed_batch_lean_features_and_derived_levels(pkg, synth, gen_device, case, monkeypatch):
    """K = 4 cameras with fx != fy and distinct principal points: the bearings formed on the device (cam2world) and the
    levels derived on the device see each pair's own intrinsics."""
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    cam_of_pair, (data, cameras) = mixed(synth, 37, 9450, gen_device)
    ragged(data, 9451)
    (lean if case == "lean" else derived_levels)(data)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, cameras=cameras)
    assert (got.n_tracked > 0).sum() >= 25
    for k, cam in enumerate(synth.MULTICAM_K4):
        idx = np.flatnonzero(cam_of_pair == k)
        sub = synth.take_pairs(data, idx)
        sub.cam = cam
        assert_same(got, three_leg(pkg, sub), ALIGN_FIELDS, rows=idx, what=f"{case} camera {k}")
    # each camera's intrinsics reach every place they are read: transposed ones (fy, fx, cy, cx) give other results
    swapped = pkg.SparseImgAlign(4, 2, 30).run(data, cameras=np.ascontiguousarray(cameras[:, [1, 0, 3, 2]]))
    differs = ~np.all(swapped.T_cur_w == got.T_cur_w, axis=1)
    assert differs[got.n_tracked > 0].all()


def test_plans_at_the_shared_memory_limit(pkg, abi, synth, gen_device, monkeypatch):
    """Point counts up to the largest a <256,2> plan admits (no segments, so no image level is staged near the limit).
    The multicam kernels take static shared memory per CTA on top of the same dynamic plan: near the limit a pinned
    multicam call either runs, byte-identical to the uniform call, or is refused with PLSVO_ERR_INVALID by the planner —
    it never hands the runtime a plan that does not fit (PLSVO_ERR_CUDA).  Unpinned, it falls back to <128,4> as the
    uniform call does, and runs."""
    base = synth.make_align_batch(batch=2, n_pts=5800, n_segs=0, max_level=3, min_level=2, seed=9800, device=gen_device)

    def with_points(n):
        d = dataclasses.replace(base)
        d.pt_px, d.pt_f, d.pt_pos = (np.ascontiguousarray(a[:, :n]) for a in (base.pt_px, base.pt_f, base.pt_pos))
        return d

    ctx = pkg.Context(0)
    lib = ctx.lib
    ap = abi.align_params(3, 2, 30)
    runs = {}
    for n in range(5736, 5768):
        d = with_points(n)
        ab, keep = abi.make_align_batch(d)
        cams = abi.make_cameras(uniform_cameras(d), d.cam, d.batch)
        outs = {}
        for name, variant, multicam in (("uniform", "256,2", False), ("multicam", "256,2", True), ("fallback", "", True)):
            monkeypatch.setenv("PLSVO_VARIANT", variant)
            out = abi.AlignOut(d.batch, 0)
            if multicam:
                rc = lib.plsvo_align_multicam_batch_run(ctx.handle, cams, C.byref(ab), C.byref(ap), C.byref(out.struct))
            else:
                rc = lib.plsvo_align_upload(ctx.handle, C.byref(ab))
                rc = rc or lib.plsvo_align_launch(ctx.handle, C.byref(ap))
                rc = rc or lib.plsvo_align_download(ctx.handle, C.byref(out.struct))
            outs[name] = (rc, lib.plsvo_last_error(ctx.handle).decode(), out)
        runs[n] = outs
        (urc, _, uout), (mrc, mmsg, mout), (frc, fmsg, _) = outs["uniform"], outs["multicam"], outs["fallback"]
        assert mrc in (abi.OK, abi.ERR_INVALID), (n, mrc, mmsg)
        if mrc == abi.OK:
            assert urc == abi.OK, n
            assert_same(mout, uout, ("T_cur_w", "n_tracked", "H", "iters", "status"), what=f"n_pts={n}")
        else:
            assert "shared-memory plan" in mmsg, (n, mmsg)
        if urc == abi.OK:
            assert frc == abi.OK, (n, frc, fmsg)
    largest = max(n for n, o in runs.items() if o["uniform"][0] == abi.OK)
    assert largest < 5767, "the sweep does not reach the limit of the <256,2> plan"
    # 16 points below the limit there are far more than the static bytes left
    assert all(o["multicam"][0] == abi.OK for n, o in runs.items() if n <= largest - 16)
    ctx.close()


def test_mixed_batch_camera_groups_against_the_oracle(pkg, abi, synth, oracle, gen_device):
    cam_of_pair, (data, cameras) = mixed(synth, 48, 9500, gen_device)
    ragged(data, 9501)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, cameras=cameras)
    for k, cam in enumerate(synth.MULTICAM_K4):
        idx = np.flatnonzero(cam_of_pair == k)
        sub = synth.take_pairs(data, idx)
        sub.cam = cam
        ref = (oracle.ref_align if oracle.ref_available() else oracle.align)(abi, sub, n_threads=8)
        for f in ("n_tracked", "iters", "status", "seg_killed"):
            np.testing.assert_array_equal(getattr(got, f)[idx], getattr(ref, f), err_msg=f"camera {k} {f}")
        ang, rel = synth.pose_error(got.T_cur_w[idx], ref.T_cur_w)
        assert ang.max() <= 1e-5 and rel.max() <= 1e-4, (k, ang.max(), rel.max())


# ---- pose optimiser and track ---------------------------------------------------------------------------------------


@pytest.mark.parametrize("n_iter_ref", [None, 5])
def test_poseopt_per_frame_fx_equals_each_cameras_uniform_call(pkg, synth, n_iter_ref):
    cams = synth.MULTICAM_K4
    B = 4096
    cam_of_frame = np.random.default_rng(9600).permutation(np.arange(B) % 4)
    index = [np.flatnonzero(cam_of_frame == k) for k in range(4)]
    parts = [synth.make_poseopt_batch(cam=c, batch=len(i), n_pts=120, n_segs=30, seed=9600 + k)
             for k, (c, i) in enumerate(zip(cams, index))]
    po = synth.scatter_batches(parts, index, B)
    fx = synth.multicam_cameras(cams, cam_of_frame)[:, 0].copy()
    got = pkg.pose_optimizer.optimizeGaussNewton(2.0, 10, False, po, n_iter_ref=n_iter_ref, fx=fx)
    for k, idx in enumerate(index):
        sub = synth.take_pairs(po, idx)
        sub.fx = cams[k].fx
        want = pkg.pose_optimizer.optimizeGaussNewton(2.0, 10, False, sub, n_iter_ref=n_iter_ref)
        assert_same(got, want, PO_FIELDS, rows=idx, what=f"camera {k}")
    assert got.pt_outlier.any()


@pytest.mark.parametrize("chained", [True, False])
def test_track_equals_each_cameras_uniform_track(pkg, synth, gen_device, chained, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    cam_of_pair, (al, po, cameras) = mixed(synth, 37, 9700, gen_device, poseopt=True)
    ragged(al, 9701)
    ao, pout = pkg.api.track(al, po, chained=chained, po_n_iter_ref=3, cameras=cameras)
    for k, cam in enumerate(synth.MULTICAM_K4):
        idx = np.flatnonzero(cam_of_pair == k)
        sa, sp = synth.take_pairs(al, idx), synth.take_pairs(po, idx)
        sa.cam, sp.fx = cam, cam.fx
        wa, wp = pkg.api.track(sa, sp, chained=chained, po_n_iter_ref=3)
        assert_same(ao, wa, ALIGN_FIELDS, rows=idx, what=f"camera {k}")
        assert_same(pout, wp, PO_FIELDS, rows=idx, what=f"camera {k}")


# ---- argument handling ----------------------------------------------------------------------------------------------


def test_malformed_multicam_calls(pkg, abi, synth):
    """Each malformed call returns PLSVO_ERR_INVALID with its message before anything is queued; the context stays
    usable.  No kernel result is read, so the host model runs this too."""
    ctx = pkg.Context(0)
    lib = ctx.lib
    d = synth.make_align_batch(cam=synth.QVGA, batch=3, n_pts=16, n_segs=4, max_level=3, min_level=1, margin=32, seed=1)
    po = synth.make_poseopt_batch(cam=synth.QVGA, batch=3, n_pts=16, n_segs=4, seed=2)
    ab, keep_a = abi.make_align_batch(d)
    pb, keep_p = abi.make_poseopt_batch(po)
    ap, pp = abi.align_params(3, 1, 30), abi.poseopt_params()
    ao, pout = abi.AlignOut(3, 4), abi.PoseOptOut(3, 16, 4)

    def cams_with(**kw):
        k = uniform_cameras(d)
        cams = abi.make_cameras(k, d.cam, 3)
        for name, v in kw.items():
            setattr(cams[1], name, v)
        return cams

    def align(cams):
        return lib.plsvo_align_multicam_batch_run(ctx.handle, cams, C.byref(ab), C.byref(ap), C.byref(ao.struct))

    def track(cams, pbatch=pb):
        return lib.plsvo_track_multicam_batch_run(ctx.handle, cams, C.byref(ab), C.byref(ap), C.byref(pbatch), C.byref(pp),
                                                  C.byref(ao.struct), C.byref(pout.struct))

    def poseopt(fx):
        return lib.plsvo_poseopt_multicam_batch_run(ctx.handle, fx, C.byref(pb), C.byref(pp), C.byref(pout.struct))

    def err():
        return lib.plsvo_last_error(ctx.handle).decode()

    cases = [({}, None, "cams is NULL"), ({"width": 321}, 1, "cams[1] is 321x240"), ({"height": 0}, 1, "cams[1] is 320x0"),
             ({"fx": float("nan")}, 1, "non-finite"), ({"cy": float("inf")}, 1, "non-finite"), ({"fx": 0.0}, 1, "non-zero"),
             ({"fy": 0.0}, 1, "non-zero")]
    for kw, _, msg in cases:
        cams = None if not kw else cams_with(**kw)
        for call in (align, track):
            assert call(cams) == abi.ERR_INVALID, (kw, call.__name__)
            assert msg in err(), (kw, err())
    po_short = abi.make_poseopt_batch(synth.make_poseopt_batch(cam=synth.QVGA, batch=2, n_pts=16, n_segs=4, seed=3))[0]
    assert track(cams_with(), po_short) == abi.ERR_INVALID and "differ in size" in err()
    for fx, msg in ((None, "fx is NULL"), ([420.0, -1.0, 420.0], "fx[1]"), ([420.0, 420.0, 0.0], "fx[2]"),
                    ([np.nan, 420.0, 420.0], "fx[0]"), ([420.0, np.inf, 420.0], "fx[1]")):
        arr = None if fx is None else np.asarray(fx, np.float64).ctypes.data_as(C.POINTER(C.c_double))
        assert poseopt(arr) == abi.ERR_INVALID and msg in err(), (fx, err())
    # negative focal lengths are valid pinhole intrinsics (errorMultiplier2 is |fx|), and the Python mirror checks shapes
    with pytest.raises(pkg.api.PlsvoError, match="shape"):
        pkg.SparseImgAlign(3, 1, 30, ctx=ctx).run(d, cameras=np.zeros((2, 4)))
    with pytest.raises(pkg.api.PlsvoError, match="shape"):
        pkg.pose_optimizer.optimizeGaussNewton(2.0, 10, False, po, fx=np.ones(4), ctx=ctx)
    with pytest.raises(pkg.api.PlsvoError, match="not both"):
        pkg.SparseImgAlign(3, 1, 30, ctx=ctx).run(d, camera=object(), cameras=uniform_cameras(d))
    with pytest.raises(pkg.api.PlsvoError, match="not both"):
        pkg.api.track(d, po, camera=object(), cameras=uniform_cameras(d), ctx=ctx)
    ctx.close()


def test_valid_multicam_calls_after_rejections(pkg, synth):
    """A context that has rejected a multicam call runs the next one; a negative fx is accepted."""
    ctx = pkg.Context(0)
    d = synth.make_align_batch(cam=synth.QVGA, batch=3, n_pts=16, n_segs=4, max_level=3, min_level=1, margin=32, seed=1)
    with pytest.raises(pkg.api.PlsvoError):
        pkg.SparseImgAlign(3, 1, 30, ctx=ctx).run(d, cameras=np.full((3, 4), np.nan))
    cams = uniform_cameras(d)
    got = pkg.SparseImgAlign(3, 1, 30, ctx=ctx).run(d, cameras=cams)
    assert (got.n_tracked > 0).all()
    # a negative fx is valid: pair b equals the uniform call with batch->cam.fx negative (cJ takes |fx|)
    cams[1, 0] = -cams[1, 0]
    neg = pkg.SparseImgAlign(3, 1, 30, ctx=ctx).run(d, cameras=cams)
    flipped = dataclasses.replace(d)
    flipped.cam = dataclasses.replace(d.cam, fx=-d.cam.fx)
    al = pkg.SparseImgAlign(3, 1, 30, ctx=ctx)
    al.upload(flipped)
    al.launch()
    want = al.download()
    assert_same(neg, want, ALIGN_FIELDS, rows=[1], want_rows=[1], what="negative fx")
    assert_same(neg, got, ALIGN_FIELDS, rows=[0, 2], want_rows=[0, 2], what="the other pairs")
    assert not np.array_equal(neg.T_cur_w[1], got.T_cur_w[1])
    ctx.close()
