"""GPU tests of the round-2 boundary additions: the chained align -> pose-opt call (BASELINE config 4), pyramid levels
derived on the device, and feature depths passed instead of 3-D positions — all through the C ABI, all against the
oracle (or against the plain calls they must be equivalent to)."""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_chained_track_equals_two_separate_calls_and_the_reference_chain(pkg, abi, synth, oracle, gen_device):
    al, po = synth.make_track_batch(batch=24, n_pts=300, n_segs=80, seed=6100, device=gen_device)
    ao, pout = pkg.api.track(al, po)
    # (1) equivalent to the two public calls with the pose copied through the host
    a2 = pkg.SparseImgAlign(4, 2, 30).run(al)
    po2 = copy.copy(po)
    po2.T_f_w = np.ascontiguousarray(a2.T_cur_w)
    p2 = pkg.pose_optimizer.optimizeGaussNewton(2.0, 10, False, po2)
    np.testing.assert_array_equal(ao.T_cur_w, a2.T_cur_w)
    for f in ("T_f_w", "cov", "estimated_scale", "error_init", "error_final", "num_obs_pt", "num_obs_ls", "pt_outlier", "seg_outlier"):
        np.testing.assert_array_equal(getattr(pout, f), getattr(p2, f), err_msg=f)
    # (2) the same chain on the CPU checker: SparseImgAlign::run, then optimizeGaussNewton from its result
    ra = (oracle.ref_align if oracle.ref_available() else oracle.align)(abi, al, n_threads=8)
    po3 = copy.copy(po)
    po3.T_f_w = np.ascontiguousarray(ra.T_cur_w)
    rp = (oracle.ref_poseopt if oracle.ref_available() else oracle.poseopt)(abi, po3, abi.poseopt_params(2.0, 10, -1), n_threads=8)
    np.testing.assert_array_equal(ao.iters, ra.iters)
    ang, rel = synth.pose_error(pout.T_f_w, rp.T_f_w)
    assert ang.max() <= 1e-5 and rel.max() <= 1e-4, (ang.max(), rel.max())
    for f in ("num_obs_pt", "num_obs_ls", "pt_outlier", "seg_outlier"):
        np.testing.assert_array_equal(getattr(pout, f), getattr(rp, f), err_msg=f)


def test_chained_track_720p_combined_config(pkg, abi, synth, oracle, gen_device):
    """BASELINE config 4 shape: 720p, 500 points + 150 segments."""
    al, po = synth.make_track_batch(cam=synth.HD720, batch=6, n_pts=500, n_segs=150, seed=6200, device=gen_device)
    ao, pout = pkg.api.track(al, po)
    ra = oracle.align(abi, al, n_threads=8)
    po3 = copy.copy(po)
    po3.T_f_w = np.ascontiguousarray(ra.T_cur_w)
    rp = oracle.poseopt(abi, po3, abi.poseopt_params(2.0, 10, -1), n_threads=8)
    np.testing.assert_array_equal(ao.iters, ra.iters)
    ang, rel = synth.pose_error(pout.T_f_w, rp.T_f_w)
    assert ang.max() <= 1e-5 and rel.max() <= 1e-4
    np.testing.assert_array_equal(pout.pt_outlier, rp.pt_outlier)
    np.testing.assert_array_equal(pout.seg_outlier, rp.seg_outlier)


@pytest.mark.parametrize("batch", [12, 300])
def test_pyramid_levels_derived_on_the_device_are_bit_identical(pkg, synth, gen_device, batch, monkeypatch):
    """Only min_level is shipped; levels above it come from halfSample on the device (bit-exact with the host pyramid),
    so every output is identical — also through the arrival-gated host pipeline (batch >= 256)."""
    data = synth.make_align_batch(batch=batch, n_pts=100, n_segs=24, device=gen_device, seed=6300)
    if batch >= 256:  # the streamed host call and the three-leg API pick different CTA shapes by default; pin one, so that
        monkeypatch.setenv("PLSVO_VARIANT", "128,4")  # the comparison is about the derived levels alone
    full = pkg.SparseImgAlign(4, 2, 30).run(data)
    lean = copy.copy(data)
    lean.ref_pyr = {2: data.ref_pyr[2]}
    lean.cur_pyr = {2: data.cur_pyr[2]}
    got = pkg.SparseImgAlign(4, 2, 30).run(lean)
    for f in ("T_cur_w", "n_tracked", "H", "seg_killed", "iters", "status"):
        np.testing.assert_array_equal(getattr(got, f), getattr(full, f), err_msg=f)
    al = pkg.SparseImgAlign(4, 2, 30)  # three-leg API
    al.upload(lean)
    al.launch()
    np.testing.assert_array_equal(al.download().T_cur_w, full.T_cur_w)


def test_depths_instead_of_positions(pkg, abi, synth, oracle, gen_device):
    """pt_depth / seg_sdepth / seg_edepth = |pos - ref camera centre| replace the 3-D positions: same decisions, poses
    equal to round-off (the depth is formed on the host instead of on the device)."""
    import torch

    data = synth.make_align_batch(batch=16, n_pts=200, n_segs=48, device=gen_device, seed=6400)
    full = pkg.SparseImgAlign(4, 2, 30).run(data)
    R, t = synth.pose7_to_Rt(torch.tensor(data.T_ref_w))
    centre = -(R.transpose(1, 2) @ t[..., None])[..., 0].numpy()  # Frame::pos(), frame.h:131
    lean = copy.copy(data)
    lean.pt_depth = np.ascontiguousarray(np.linalg.norm(data.pt_pos - centre[:, None, :], axis=-1))
    lean.seg_sdepth = np.ascontiguousarray(np.linalg.norm(data.seg_spos - centre[:, None, :], axis=-1))
    lean.seg_edepth = np.ascontiguousarray(np.linalg.norm(data.seg_epos - centre[:, None, :], axis=-1))
    lean.pt_pos = lean.seg_spos = lean.seg_epos = None
    got = pkg.SparseImgAlign(4, 2, 30).run(lean)
    np.testing.assert_array_equal(got.iters, full.iters)
    np.testing.assert_array_equal(got.n_tracked, full.n_tracked)
    np.testing.assert_array_equal(got.seg_killed, full.seg_killed)
    ang, rel = synth.pose_error(got.T_cur_w, full.T_cur_w)
    assert ang.max() < 1e-10 and rel.max() < 1e-9


def test_bearings_derived_from_pixels_on_the_device(pkg, synth, gen_device):
    """pt_f / seg_sf / seg_ef = NULL: the device forms cam2world(px) as the reference's feature constructors do
    (feature.cpp:42,98-99).  Same decisions; poses equal to round-off (the generator normalises with torch)."""
    data = synth.make_align_batch(batch=16, n_pts=200, n_segs=48, device=gen_device, seed=6450)
    full = pkg.SparseImgAlign(4, 2, 30).run(data)
    lean = copy.copy(data)
    lean.pt_f = lean.seg_sf = lean.seg_ef = None
    got = pkg.SparseImgAlign(4, 2, 30).run(lean)
    np.testing.assert_array_equal(got.iters, full.iters)
    np.testing.assert_array_equal(got.n_tracked, full.n_tracked)
    np.testing.assert_array_equal(got.seg_killed, full.seg_killed)
    ang, rel = synth.pose_error(got.T_cur_w, full.T_cur_w)
    assert ang.max() < 1e-10 and rel.max() < 1e-9


def test_feature_counts_out_of_range_are_rejected(pkg, synth, gen_device):
    data = synth.make_align_batch(batch=4, n_pts=32, n_segs=8, device=gen_device, seed=6500)
    data.pt_count = np.array([32, 33, 1, 2], np.int32)
    with pytest.raises(pkg.api.PlsvoError):
        pkg.SparseImgAlign(4, 2, 30).run(data)
    data.pt_count = None
    data.seg_count = np.array([8, -1, 1, 2], np.int32)
    with pytest.raises(pkg.api.PlsvoError):
        pkg.SparseImgAlign(4, 2, 30).run(data)
    pd = synth.make_poseopt_batch(batch=4, n_pts=32, n_segs=8, seed=6501)
    pd.pt_count = np.array([32, 999, 1, 2], np.int32)
    with pytest.raises(pkg.api.PlsvoError):
        pkg.pose_optimizer.optimizeGaussNewton(2.0, 10, False, pd)


def test_gate_with_several_chunks_and_copy_streams(pkg, synth, gen_device, monkeypatch):
    """The arrival gate with more than one chunk on the copy stream (PLSVO_GATE_CHUNK=128, 3 chunks)."""
    data = synth.make_align_batch(batch=300, n_pts=64, n_segs=12, device=gen_device, seed=6600)
    al = pkg.SparseImgAlign(4, 2, 30)
    al.upload(data)  # the plain upload -> launch -> download sequence
    al.launch()
    plain = al.download()
    monkeypatch.setenv("PLSVO_GATE_CHUNK", "128")
    monkeypatch.setenv("PLSVO_VARIANT", "128,4")  # the CTA shape of the single-shot call: bitwise comparison of the gate alone
    for _ in range(2):
        gated = pkg.SparseImgAlign(4, 2, 30).run(data)
        for f in ("T_cur_w", "n_tracked", "iters", "H"):
            np.testing.assert_array_equal(getattr(plain, f), getattr(gated, f), err_msg=f)


def test_twenty_frame_sequence_chained_frame_to_frame(pkg, abi, synth, oracle, gen_device):
    """BASELINE config 1: 20-frame VGA sequences, each frame aligned against the previous one and refined by the pose
    optimiser, the estimate seeding the next frame (run_pipeline.cpp:312-451 / frame_handler_mono.cpp:263-340).
    The GPU chain (plsvo_track_batch_run per frame) against the same chain on the CPU checker: every frame inside the
    per-frame tolerance, identical alignment iteration counts and outlier flags, and the drift at frame 20 reported."""
    poses, steps = synth.make_sequence(n_seq=4, n_frames=20, n_pts=300, n_segs=80, seed=1000, device=gen_device)
    have_ref = oracle.ref_available()

    def cpu_step(al, po):
        ra = (oracle.ref_align if have_ref else oracle.align)(abi, al, n_threads=4)
        po.T_f_w = np.ascontiguousarray(ra.T_cur_w)
        return ra, (oracle.ref_poseopt if have_ref else oracle.poseopt)(abi, po, abi.poseopt_params(2.0, 10, -1), n_threads=4)

    est_gpu, it_gpu, out_gpu = synth.run_sequence(poses, steps, lambda al, po: pkg.api.track(al, po))
    est_cpu, it_cpu, out_cpu = synth.run_sequence(poses, steps, cpu_step)
    np.testing.assert_array_equal(it_gpu, it_cpu)
    np.testing.assert_array_equal(out_gpu, out_cpu)
    for k in range(1, 20):
        ang, rel = synth.pose_error(est_gpu[:, k], est_cpu[:, k])
        assert ang.max() <= 1e-5 and rel.max() <= 1e-4, (k, float(ang.max()), float(rel.max()))
    ang20, rel20 = synth.pose_error(est_gpu[:, 19], est_cpu[:, 19])
    ang_gt, rel_gt = synth.pose_error(est_gpu[:, 19], poses[:, 19])
    print(f"sequence drift at frame 20: GPU vs CPU chain {ang20.max():.2e} rad / {rel20.max():.2e}; GPU vs ground truth {ang_gt.max():.2e} rad / {rel_gt.max():.2e}")
    assert ang_gt.max() < 5e-3  # the chain tracks the trajectory
