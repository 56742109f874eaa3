"""GPU parity of the alignment kernel against the CPU oracle, through the C ABI.

Tolerance (BASELINE.json north_star): rotation <= 1e-5 rad, relative translation <= 1e-4 on
identical inputs.  Integer outputs (n_tracked, killed segments, per-level iteration counts, status)
must be equal on EVERY pair: the kernel reproduces the reference's sequential float chi2 bit for bit
and accumulates the normal equations per pixel in double, so the accept / rollback decision of the
Gauss-Newton loop never depends on summation order (DESIGN.md section 2).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROT_TOL = 1e-5
TRANS_TOL = 1e-4


def _run_both(pkg, abi, synth, oracle, data, max_level=4, min_level=2, n_iter=30):
    gpu = pkg.SparseImgAlign(max_level, min_level, n_iter, pkg.SparseImgAlign.GaussNewton, False, False).run(data)
    ref = oracle.align(abi, data, abi.align_params(max_level, min_level, n_iter), n_threads=8)
    return gpu, ref


def _check(synth, gpu, ref, exact_iters=True, mask=None):
    ang, rel = synth.pose_error(gpu.T_cur_w, ref.T_cur_w)
    if mask is not None:
        ang, rel = ang[mask], rel[mask]
    assert ang.max() <= ROT_TOL, f"rotation parity {ang.max():.3e}"
    assert rel.max() <= TRANS_TOL, f"translation parity {rel.max():.3e}"
    m = slice(None) if mask is None else mask
    np.testing.assert_array_equal(gpu.n_tracked[m], ref.n_tracked[m])
    np.testing.assert_array_equal(gpu.seg_killed[m], ref.seg_killed[m])
    np.testing.assert_array_equal(gpu.status[m], ref.status[m])
    if exact_iters:
        np.testing.assert_array_equal(gpu.iters[m], ref.iters[m])
    scale = np.abs(ref.H).max(axis=1, keepdims=True) + 1e-300
    same_it = (gpu.iters == ref.iters).all(axis=1)
    if mask is not None:
        same_it &= mask
    if same_it.any():
        assert (np.abs(gpu.H - ref.H)[same_it] / scale[same_it]).max() < 1e-9


def test_align_vga_points_and_segments(pkg, abi, synth, oracle, gen_device):
    data = synth.make_align_batch(batch=32, n_pts=300, n_segs=80, device=gen_device, seed=3000)
    gpu, ref = _run_both(pkg, abi, synth, oracle, data)
    _check(synth, gpu, ref)
    np.testing.assert_array_equal(gpu.patch_levels, ref.patch_levels)
    np.testing.assert_array_equal(gpu.patch_iters, ref.patch_iters)


@pytest.mark.parametrize("seed", [4100, 4101, 4102, 4103, 4104, 4105, 4106, 4107])
def test_align_parity_campaign_1024_pairs_per_seed(pkg, abi, synth, oracle, gen_device, seed):
    """8 seeds x 1024 C2-shaped pairs = 8192 pairs: every pair inside the tolerance, identical per-level iteration
    counts, n_tracked, killed segments and status; no chi2-order flag raised (status bits 2-4)."""
    data = synth.make_align_batch(batch=1024, n_pts=300, n_segs=80, device=gen_device, seed=seed)
    gpu = pkg.SparseImgAlign(4, 2, 30).run(data)
    ref = (oracle.ref_align if oracle.ref_available() else oracle.align)(abi, data, n_threads=64)
    ang, rel = synth.pose_error(gpu.T_cur_w, ref.T_cur_w)
    assert ang.max() <= ROT_TOL and rel.max() <= TRANS_TOL, (float(ang.max()), float(rel.max()))
    np.testing.assert_array_equal(gpu.iters, ref.iters)
    np.testing.assert_array_equal(gpu.n_tracked, ref.n_tracked)
    np.testing.assert_array_equal(gpu.seg_killed, ref.seg_killed)
    np.testing.assert_array_equal(gpu.status, ref.status)


def test_align_points_only(pkg, abi, synth, oracle, gen_device):
    data = synth.make_align_batch(batch=16, n_pts=300, n_segs=0, device=gen_device, seed=3100)
    gpu, ref = _run_both(pkg, abi, synth, oracle, data)
    _check(synth, gpu, ref)


def test_align_segments_only(pkg, abi, synth, oracle, gen_device):
    """Segments alone are an unstable problem in the reference: its segment weighting
    (H += H_*w/res_, Jres += Jres_*w, sparse_img_align.cpp:681-682) scales the GN step by the mean
    residual, so without points the iteration overshoots and often diverges chaotically (any
    rounding difference is amplified to radians).  Parity is therefore asserted on the pairs whose
    oracle result stays near the initial pose; the integer outputs must agree on all pairs."""
    data = synth.make_align_batch(batch=32, n_pts=0, n_segs=120, device=gen_device, seed=3200)
    gpu, ref = _run_both(pkg, abi, synth, oracle, data)
    moved, _ = synth.pose_error(ref.T_cur_w, data.T_cur_w)
    sane = moved < 0.02
    assert sane.sum() >= 4
    _check(synth, gpu, ref, exact_iters=True, mask=sane)
    np.testing.assert_array_equal(gpu.iters, ref.iters)  # same decisions on every pair, also the diverging ones


def test_align_converges_to_ground_truth(pkg, synth, gen_device):
    data = synth.make_align_batch(batch=16, n_pts=300, n_segs=80, device=gen_device, seed=3300)
    gpu = pkg.SparseImgAlign(4, 2, 30).run(data)
    ang0, rel0 = synth.pose_error(data.T_cur_w, data.T_cur_w_gt)
    ang, rel = synth.pose_error(gpu.T_cur_w, data.T_cur_w_gt)
    assert np.median(ang) < 0.2 * np.median(ang0)
    assert np.median(rel) < 0.2 * np.median(rel0)


def test_align_edge_cases(pkg, abi, synth, oracle, gen_device):
    """Invalid features (feat3D == NULL), ragged per-pair counts, empty pairs, features at the border."""
    data = synth.make_align_batch(batch=12, n_pts=96, n_segs=40, device=gen_device, seed=3400, margin=2)
    rng = np.random.default_rng(5)
    data.pt_valid = (rng.uniform(size=(12, 96)) > 0.2).astype(np.uint8)
    data.seg_valid = (rng.uniform(size=(12, 40)) > 0.2).astype(np.uint8)
    data.pt_count = rng.integers(1, 97, 12).astype(np.int32)
    data.seg_count = rng.integers(0, 41, 12).astype(np.int32)
    data.pt_count[3] = 0
    data.seg_count[3] = 0  # empty pair: run() returns 0 and leaves the pose untouched
    data.pt_count[5] = 0   # segments only
    data.seg_count[7] = 0  # points only
    gpu, ref = _run_both(pkg, abi, synth, oracle, data)
    _check(synth, gpu, ref)
    assert gpu.status[3] == 1 and gpu.n_tracked[3] == 0
    np.testing.assert_array_equal(gpu.T_cur_w[3], data.T_cur_w[3])


@pytest.mark.parametrize("levels", [(2, 0), (3, 1), (5, 3)])
def test_align_other_level_ranges(pkg, abi, synth, oracle, gen_device, levels):
    max_level, min_level = levels
    data = synth.make_align_batch(batch=6, n_pts=128, n_segs=32, max_level=max_level, min_level=min_level,
                                  device=gen_device, seed=3500 + max_level,
                                  motion_t=0.03 / (1 << (4 - min(4, max_level))), motion_r=0.01 / (1 << (4 - min(4, max_level))))
    gpu, ref = _run_both(pkg, abi, synth, oracle, data, max_level, min_level)
    _check(synth, gpu, ref)


def test_align_three_leg_api_matches_batch_run(pkg, synth, gen_device):
    data = synth.make_align_batch(batch=8, n_pts=200, n_segs=40, device=gen_device, seed=3600)
    al = pkg.SparseImgAlign(4, 2, 30)
    one = al.run(data)
    al.upload(data)
    al.launch()
    two = al.download()
    np.testing.assert_array_equal(one.T_cur_w, two.T_cur_w)  # deterministic reduction order
    np.testing.assert_array_equal(one.H, two.H)
    F = al.getFisherInformation()
    assert F.shape == (8, 6, 6)


def test_fp32_weight_matches_reference_expression(pkg):
    """w = 1/(1+|r|): the fp32 sequence must reproduce the reference's double-then-narrow value."""
    import ctypes as C

    ctx = pkg.api.default_context()
    bad = C.c_uint64(0)
    n = 1 << 26
    ctx.check(ctx.lib.plsvo_selftest_weight(ctx.handle, n, 12345, C.byref(bad)), "selftest")
    assert bad.value == 0, f"{bad.value} of {n} weights differ (scalar or packed form)"


def test_align_zero_residual_segment_raises_stop(pkg, abi, synth, oracle, gen_device):
    """Identical images: a segment with zero mean residual makes the reference divide by zero
    (sparse_img_align.cpp:681) -> NaN step -> stop_ (sticky) -> pose untouched.  Same on the GPU."""
    data = synth.make_align_batch(cam=synth.QVGA, batch=4, n_pts=40, n_segs=8, max_level=3, min_level=1, seed=21,
                                  margin=32, motion_t=0.0, motion_r=0.0, device=gen_device)
    gpu, ref = _run_both(pkg, abi, synth, oracle, data, 3, 1)
    np.testing.assert_array_equal(gpu.status, ref.status)
    assert (gpu.status == 2).all()
    np.testing.assert_array_equal(gpu.iters, ref.iters)
    ang, rel = synth.pose_error(gpu.T_cur_w, ref.T_cur_w)
    assert ang.max() < 1e-12


def test_align_720p_combined_config(pkg, abi, synth, oracle, gen_device):
    """BASELINE config 4 shape: 720p, 500 points + 150 segments (levels 4->2): larger per-pair state,
    the finest level is no longer staged in shared memory."""
    data = synth.make_align_batch(cam=synth.HD720, batch=6, n_pts=500, n_segs=150, device=gen_device, seed=3800)
    gpu, ref = _run_both(pkg, abi, synth, oracle, data)
    _check(synth, gpu, ref)


def test_align_segments_longer_than_a_warp(pkg, abi, synth, oracle, gen_device):
    """At level 0 a 700-px segment has more than 32 samples: the whole-warp loop (long-segment path)."""
    data = synth.make_align_batch(cam=synth.HD720, batch=4, n_pts=200, n_segs=12, max_level=2, min_level=0,
                                  device=gen_device, seed=3900, motion_t=0.004, motion_r=0.0012, margin=24)
    rng = np.random.default_rng(3)
    # stretch the segments: endpoints far apart inside the image
    import torch

    B, S = data.seg_spx.shape[:2]
    spx = np.stack([rng.uniform(40, 300, (B, S)), rng.uniform(40, 680, (B, S))], -1)
    epx = np.stack([rng.uniform(980, 1240, (B, S)), rng.uniform(40, 680, (B, S))], -1)
    scene = synth.Scene()
    R, t = synth.pose7_to_Rt(torch.tensor(data.T_ref_w))

    def lift(px):
        p = torch.tensor(px)
        d = torch.stack([(p[..., 0] - data.cam.cx) / data.cam.fx, (p[..., 1] - data.cam.cy) / data.cam.fy, torch.ones_like(p[..., 0])], -1)
        f = d / d.norm(dim=-1, keepdim=True)
        return f.numpy(), scene.intersect(R, t, d).numpy()

    data.seg_spx, data.seg_epx = np.ascontiguousarray(spx), np.ascontiguousarray(epx)
    data.seg_sf, data.seg_spos = (np.ascontiguousarray(x) for x in lift(spx))
    data.seg_ef, data.seg_epos = (np.ascontiguousarray(x) for x in lift(epx))
    data.seg_length = np.ascontiguousarray(np.linalg.norm(epx - spx, axis=-1))
    gpu, ref = _run_both(pkg, abi, synth, oracle, data, 2, 0)
    assert (data.seg_length / 16 > 32).any()
    _check(synth, gpu, ref)


def test_align_gated_host_pipeline_matches_single_shot(pkg, synth, gen_device, monkeypatch):
    """Default host-buffer path for >= 256 pairs: one persistent kernel gated on chunk arrivals while a copy
    stream streams the batch in.  Results must equal the plain upload -> launch -> download sequence."""
    data = synth.make_align_batch(batch=300, n_pts=64, n_segs=12, device=gen_device, seed=3750)
    al = pkg.SparseImgAlign(4, 2, 30)
    al.upload(data)  # the plain upload -> launch -> download sequence
    al.launch()
    plain = al.download()
    # the streamed call picks its own CTA shape (<192,2>): a different assignment of patches to threads, hence a different
    # order of the double-precision normal-equation sums — same decisions, poses equal to round-off
    for _ in range(2):
        gated = pkg.SparseImgAlign(4, 2, 30).run(data)
        np.testing.assert_array_equal(plain.n_tracked, gated.n_tracked)
        np.testing.assert_array_equal(plain.iters, gated.iters)
        ang, rel = synth.pose_error(gated.T_cur_w, plain.T_cur_w)
        assert ang.max() < 1e-11 and rel.max() < 1e-10
        np.testing.assert_allclose(gated.H, plain.H, rtol=1e-11, atol=1e-6)
    # with the same CTA shape on both paths the arrival gate must not change a single bit
    monkeypatch.setenv("PLSVO_VARIANT", "128,4")
    for _ in range(3):
        gated = pkg.SparseImgAlign(4, 2, 30).run(data)
        np.testing.assert_array_equal(plain.T_cur_w, gated.T_cur_w)
        np.testing.assert_array_equal(plain.n_tracked, gated.n_tracked)
        np.testing.assert_array_equal(plain.iters, gated.iters)
        np.testing.assert_array_equal(plain.H, gated.H)
