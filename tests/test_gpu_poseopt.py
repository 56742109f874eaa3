"""GPU parity of the pose-optimiser kernel against the CPU oracle, through the C ABI."""
from types import SimpleNamespace

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROT_TOL = 1e-5
TRANS_TOL = 1e-4
FIELDS = ("T_f_w", "status", "iters", "pt_outlier", "seg_outlier", "num_obs_pt", "num_obs_ls", "estimated_scale", "error_init",
          "error_final", "cov")


def _check(synth, gpu, ref, cov=True):
    """Pose to ROT_TOL / TRANS_TOL, bookkeeping exactly, scale and medians to round-off, and the covariance: its inf / NaN
    entries where the oracle has them (a singular A), the finite ones to 1e-6 of the frame's largest.  cov=False skips
    the covariance (n_iter = 0: the reference inverts an A it never set)."""
    ang, rel = synth.pose_error(gpu.T_f_w, ref.T_f_w)
    assert ang.max() <= ROT_TOL, f"rotation parity {ang.max():.3e}"
    assert rel.max() <= TRANS_TOL, f"translation parity {rel.max():.3e}"
    np.testing.assert_array_equal(gpu.status, ref.status)
    np.testing.assert_array_equal(gpu.iters, ref.iters)
    np.testing.assert_array_equal(gpu.pt_outlier, ref.pt_outlier)
    np.testing.assert_array_equal(gpu.seg_outlier, ref.seg_outlier)
    np.testing.assert_array_equal(gpu.num_obs_pt, ref.num_obs_pt)
    np.testing.assert_array_equal(gpu.num_obs_ls, ref.num_obs_ls)
    ok = ref.status == 0
    np.testing.assert_allclose(gpu.estimated_scale[ok], ref.estimated_scale[ok], rtol=1e-12)
    np.testing.assert_allclose(gpu.error_init[ok], ref.error_init[ok], rtol=1e-9)
    np.testing.assert_allclose(gpu.error_final[ok], ref.error_final[ok], rtol=1e-6)
    if not cov or not ok.any():
        return
    g, r = gpu.cov[ok], ref.cov[ok]
    for what, f in (("NaN", np.isnan), ("+inf", np.isposinf), ("-inf", np.isneginf)):
        np.testing.assert_array_equal(f(g), f(r), err_msg=f"covariance {what} entries")
    fin = np.isfinite(r)
    scale = np.abs(np.where(fin, r, 0.0)).max(axis=1, keepdims=True) + 1e-300
    with np.errstate(invalid="ignore"):
        err = np.where(fin, np.abs(g - r), 0.0)
    assert (err / scale).max() < 1e-6


def test_poseopt_9arg(pkg, abi, synth, oracle):
    data = synth.make_poseopt_batch(batch=64, n_pts=300, n_segs=80, seed=5000)
    gpu = pkg.pose_optimizer.optimizeGaussNewton(2.0, 10, False, data)
    ref = oracle.poseopt(abi, data, abi.poseopt_params(2.0, 10, -1), n_threads=8)
    _check(synth, gpu, ref)
    ang0, _ = synth.pose_error(data.T_f_w, data.T_f_w_gt)
    ang, _ = synth.pose_error(gpu.T_f_w, data.T_f_w_gt)
    assert np.median(ang) < 0.5 * np.median(ang0)


def test_poseopt_10arg_refinement(pkg, abi, synth, oracle):
    data = synth.make_poseopt_batch(batch=32, n_pts=300, n_segs=80, seed=5100)
    gpu = pkg.pose_optimizer.optimizeGaussNewton(2.0, 10, False, data, n_iter_ref=3)
    ref = oracle.poseopt(abi, data, abi.poseopt_params(2.0, 10, 3), n_threads=8)
    _check(synth, gpu, ref)


def test_poseopt_points_only_and_lines_dead(pkg, abi, synth, oracle):
    data = synth.make_poseopt_batch(batch=16, n_pts=200, n_segs=0, seed=5200)
    gpu = pkg.pose_optimizer.optimizeGaussNewton(2.0, 10, False, data)
    ref = oracle.poseopt(abi, data, abi.poseopt_params(2.0, 10, -1))
    _check(synth, gpu, ref)


def test_poseopt_edge_cases(pkg, abi, synth, oracle):
    data = synth.make_poseopt_batch(batch=10, n_pts=64, n_segs=24, seed=5300)
    rng = np.random.default_rng(9)
    data.pt_valid = (rng.uniform(size=(10, 64)) > 0.25).astype(np.uint8)
    data.seg_valid = (rng.uniform(size=(10, 24)) > 0.25).astype(np.uint8)
    data.pt_count = rng.integers(8, 65, 10).astype(np.int32)
    data.seg_count = rng.integers(0, 25, 10).astype(np.int32)
    data.pt_valid[2] = 0
    data.seg_valid[2] = 0  # no observations at all: early return, outputs untouched
    gpu = pkg.pose_optimizer.optimizeGaussNewton(2.0, 10, False, data)
    ref = oracle.poseopt(abi, data, abi.poseopt_params(2.0, 10, -1))
    _check(synth, gpu, ref)
    assert gpu.status[2] == 1
    np.testing.assert_array_equal(gpu.T_f_w[2], data.T_f_w[2])


def test_poseopt_many_ragged_frames_per_cta(pkg, abi, synth, oracle):
    """More frames than the grid has CTAs (16 per SM), so every CTA optimises a sequence of frames of different sizes:
    ragged point and segment counts, frames with no valid feature (status 1) and frames with a single point."""
    B = 2500
    data = synth.make_poseopt_batch(batch=B, n_pts=48, n_segs=12, seed=5400)
    rng = np.random.default_rng(11)
    data.pt_count = rng.integers(1, 49, B).astype(np.int32)
    data.seg_count = rng.integers(0, 13, B).astype(np.int32)
    data.pt_valid = (rng.uniform(size=(B, 48)) > 0.1).astype(np.uint8)
    data.seg_valid = (rng.uniform(size=(B, 12)) > 0.1).astype(np.uint8)
    data.pt_count[3::11] = 1
    data.seg_count[3::11] = 0
    data.pt_valid[3::11] = 1  # a single point
    data.pt_valid[::7] = 0
    data.seg_valid[::7] = 0  # nothing to optimise: early return
    gpu = pkg.pose_optimizer.optimizeGaussNewton(2.0, 10, False, data)
    ref = oracle.poseopt(abi, data, abi.poseopt_params(2.0, 10, -1), n_threads=8)
    # a handful of observations (two residual rows each) barely determines the 6-DoF pose, one point not at all: the steps
    # and the covariance of such a frame come from a singular or ill-conditioned system (one point: not even finite), so
    # they are round-off; those frames are held to the bookkeeping, which every frame must match
    vp = np.array([data.pt_valid[b, :data.pt_count[b]].sum() for b in range(B)])
    vs = np.array([data.seg_valid[b, :data.seg_count[b]].sum() for b in range(B)])
    few = (vp + vs > 0) & (vp + vs < 8)
    rows = lambda out, m: SimpleNamespace(**{f: getattr(out, f)[m] for f in FIELDS})
    _check(synth, rows(gpu, ~few), rows(ref, ~few))
    for f in ("status", "pt_outlier", "seg_outlier", "num_obs_pt", "num_obs_ls"):
        np.testing.assert_array_equal(getattr(gpu, f), getattr(ref, f), err_msg=f)
    assert (gpu.status[::7] == 1).all() and few.sum() > 100 and (~few).sum() > 1500
