"""Reference-typed bindings of the loops either side of the hot path (pl-svo_b200/host/plsvo_shim_next.{h,cpp}):

* plsvo::b200::DirectMatcher — every Matcher::findMatchDirect call of Reprojector::reprojectMap in one device call
  (src/reprojector.cpp:186-207, :236-387; src/matcher.cpp:159-275), with Point/LineSeg::getCloseViewObs on the host;
* plsvo::b200::DepthFilterB200 — DepthFilter::updateSeeds (src/depth_filter.cpp:262-471) with the per-seed work batched.

Both are checked on the reference's OWN objects (Point, LineSeg, PointFeat, LineFeat, Frame, PointSeed, LineSeed, Matcher,
DepthFilter) against the reference's own loops compiled from /root/reference (oracle/_ref): on the CPU with the C ABI
answered by the oracle (exact), on the GPU through the product library."""
import numpy as np
import pytest


def _need_ref(oracle, cpu):
    if not oracle.build_ref():
        pytest.skip("oracle/_ref needs the reference's sources (PLSVO_REFERENCE_ROOT)")
    if not (oracle.build_shimref_cpu() if cpu else oracle.build_shimref()):
        pytest.skip("the shim on reference types needs the reference's sources (PLSVO_REFERENCE_ROOT)")


def _check_match_scene(s, r, n_obs, n_ref):
    # the closest-view observation chosen by getCloseViewObs (host list logic) — and it is not always the batch's own one
    np.testing.assert_array_equal(s.pt_ref, r.pt_ref)
    np.testing.assert_array_equal(s.seg_ref, r.seg_ref)
    for f in ("pt_found", "pt_level", "seg_found", "seg_level"):
        np.testing.assert_array_equal(getattr(s, f), getattr(r, f), err_msg=f)
    for f in ("pt_px", "pt_A", "seg_spx", "seg_epx", "seg_A"):
        a, b = getattr(s, f), getattr(r, f)
        np.testing.assert_array_equal(np.isnan(a), np.isnan(b), err_msg=f)
        np.testing.assert_array_equal(a[~np.isnan(a)], b[~np.isnan(b)], err_msg=f)
    assert r.pt_found.mean() > 0.4 and r.seg_found.mean() > 0.15
    assert (~r.pt_found.astype(bool)).sum() > 10  # failures are exercised too


def _match_data(synth, seed, **kw):
    return synth.make_match_batch(n=1200, seed=seed, **kw)


@pytest.mark.parametrize("seed,n_obs,kw", [(7300, 3, {}), (7301, 1, dict(n_pyr_levels=5)), (7302, 2, dict(edgelet_frac=0.5))])
def test_direct_matcher_replays_the_reprojector_loop_cpu(oracle, abi, synth, seed, n_obs, kw):
    """Oracle-backed C ABI: what comes back in the reference's objects must equal the reference's own Matcher exactly."""
    _need_ref(oracle, cpu=True)
    d = _match_data(synth, seed, **kw)
    r = oracle.ref_match_scene(abi, d, n_obs)
    s = oracle.shimref_match_scene(abi, d, n_obs, cpu=True)
    _check_match_scene(s, r, n_obs, d.T_ref_w.shape[0])
    if n_obs > 1:  # some points are matched against a keyframe other than the one the flat batch names
        first = d.ref_index[: d.n]
        assert (r.pt_ref != first).mean() > 0.05


@pytest.mark.gpu
@pytest.mark.parametrize("seed,n_obs,kw", [(7310, 3, {}), (7311, 2, dict(n_pyr_levels=5, edgelet_frac=0.3))])
def test_direct_matcher_replays_the_reprojector_loop_gpu(pkg, oracle, abi, synth, seed, n_obs, kw):
    _need_ref(oracle, cpu=False)
    d = _match_data(synth, seed, **kw)
    r = oracle.ref_match_scene(abi, d, n_obs)
    s = oracle.shimref_match_scene(abi, d, n_obs)
    _check_match_scene(s, r, n_obs, d.T_ref_w.shape[0])


def _seed_data(synth, seed, n=900, **kw):
    pts = synth.make_seed_batch(n=n, seed=seed, **kw)
    lines = synth.make_line_seed_batch(n=n // 2, seed=seed, **{k: v for k, v in kw.items() if k != "edgelet_frac"})
    # the two batches share their random stream up to the poses: same keyframes, same current frames
    np.testing.assert_array_equal(pts.T_cur_w, lines.T_cur_w)
    np.testing.assert_array_equal(pts.T_ref_w, lines.T_ref_w)
    rng = np.random.default_rng(seed)
    pt_age = rng.integers(0, 5, pts.n).astype(np.int32)     # DepthFilter::Options::max_n_kfs = 3: ages 4 are erased
    seg_age = rng.integers(0, 5, lines.n).astype(np.int32)
    # push a share of the seeds to the edge of convergence so that this update converges them
    for d in (pts, lines):
        k = rng.uniform(size=d.n) < 0.35
        d.sigma2[k] = (d.z_range[k] / 200.0) ** 2 * rng.uniform(0.8, 1.6, k.sum()).astype(np.float32)
    k = rng.uniform(size=lines.n) < 0.5
    lines.sigma2_e[k] = (lines.z_range_e[k] / 200.0) ** 2 * rng.uniform(0.8, 1.6, k.sum()).astype(np.float32)
    return pts, lines, pt_age, seg_age


def _check_seed_scene(s, r, exact, pt_age, seg_age):
    assert set(np.unique(r.pt_fate)) == {0, 1, 2} and set(np.unique(r.seg_fate)) == {0, 1, 2}
    np.testing.assert_array_equal(r.pt_fate[pt_age > 3], 2)  # aged out
    np.testing.assert_array_equal(s.pt_fate[pt_age > 3], 2)
    if exact:
        for f in ("pt_fate", "seg_fate"):
            np.testing.assert_array_equal(getattr(s, f), getattr(r, f), err_msg=f)
        for f in ("pt_state", "pt_xyz", "pt_cb_sigma2", "pt_marks", "seg_state", "seg_xyz", "seg_cb_sigma2", "seg_marks"):
            a, b = getattr(s, f), getattr(r, f)
            assert a.shape == b.shape, f
            np.testing.assert_array_equal(np.isnan(a), np.isnan(b), err_msg=f)
            np.testing.assert_array_equal(a[~np.isnan(a)], b[~np.isnan(b)], err_msg=f)
        return
    # device: (a, b, mu, sigma2) agree to libm round-off (tests/test_depth_filter.py states the tolerances), so a seed sitting
    # on the convergence threshold may fall on the other side of it
    for kind, w in (("pt", 4), ("seg", 6)):
        fs, fr = getattr(s, kind + "_fate"), getattr(r, kind + "_fate")
        same = fs == fr
        assert same.mean() > 0.995, kind
        alive = same & (fr == 0)
        a, b = getattr(s, kind + "_state")[alive], getattr(r, kind + "_state")[alive]
        fin = np.isfinite(b).all(axis=1) & np.isfinite(a).all(axis=1)
        np.testing.assert_allclose(a[fin][:, 2::2], b[fin][:, 2::2], rtol=2e-6, atol=0, err_msg=kind + " mu")
        np.testing.assert_allclose(a[fin][:, 3::2], b[fin][:, 3::2], rtol=2e-4, atol=5e-7, err_msg=kind + " sigma2")
        np.testing.assert_allclose(a[fin][:, 0], b[fin][:, 0], rtol=5e-2, err_msg=kind + " a")
        np.testing.assert_allclose(a[fin][:, 1], b[fin][:, 1], rtol=5e-2, atol=1e-3, err_msg=kind + " b")
        conv = same & (fr == 1)
        assert conv.sum() > 10, kind
        xs, xr = getattr(s, kind + "_xyz")[conv], getattr(r, kind + "_xyz")[conv]
        np.testing.assert_allclose(xs, xr, rtol=1e-5, err_msg=kind + " xyz of the created 3-D feature")
    # detector marks on keyframes: positions are exact (integer search + bit-identical sub-pixel refinement); the count follows the fates
    if len(r.pt_marks):
        assert abs(len(s.pt_marks) - len(r.pt_marks)) <= 2
        if len(s.pt_marks) == len(r.pt_marks):
            np.testing.assert_array_equal(s.pt_marks, r.pt_marks)


@pytest.mark.parametrize("seed,keyframe,kw", [(9700, False, {}), (9701, True, dict(n_pyr_levels=5)), (9702, True, dict(baseline=0.25))])
def test_depth_filter_b200_replays_update_seeds_cpu(oracle, abi, synth, seed, keyframe, kw):
    _need_ref(oracle, cpu=True)
    pts, lines, pt_age, seg_age = _seed_data(synth, seed, **kw)
    r = oracle.ref_seed_scene(abi, pts, lines, pt_age, seg_age, keyframe)
    s = oracle.shimref_seed_scene(abi, pts, lines, pt_age, seg_age, keyframe, cpu=True)
    _check_seed_scene(s, r, True, pt_age, seg_age)
    assert (len(r.pt_marks) > 0) == keyframe and (len(r.seg_marks) > 0) == keyframe
    assert (r.pt_fate == 1).sum() > 20 and (r.seg_fate == 1).sum() > 5


@pytest.mark.gpu
@pytest.mark.parametrize("seed,keyframe,kw", [(9710, True, {}), (9711, False, dict(n_pyr_levels=5, baseline=0.25))])
def test_depth_filter_b200_replays_update_seeds_gpu(pkg, oracle, abi, synth, seed, keyframe, kw):
    _need_ref(oracle, cpu=False)
    pts, lines, pt_age, seg_age = _seed_data(synth, seed, n=1500, **kw)
    r = oracle.ref_seed_scene(abi, pts, lines, pt_age, seg_age, keyframe)
    s = oracle.shimref_seed_scene(abi, pts, lines, pt_age, seg_age, keyframe)
    _check_seed_scene(s, r, False, pt_age, seg_age)


def test_depth_filter_b200_with_every_seed_aged_out_makes_no_device_call(oracle, abi, synth):
    """Seeds older than max_n_kfs are erased before anything is packed: same fates as the reference, nothing updated."""
    _need_ref(oracle, cpu=True)
    pts, lines, _, _ = _seed_data(synth, 9720, n=120)
    old_p, old_s = np.full(pts.n, 9, np.int32), np.full(lines.n, 9, np.int32)
    r = oracle.ref_seed_scene(abi, pts, lines, old_p, old_s, True)
    s = oracle.shimref_seed_scene(abi, pts, lines, old_p, old_s, True, cpu=True)
    assert (r.pt_fate == 2).all() and (r.seg_fate == 2).all()
    np.testing.assert_array_equal(s.pt_fate, r.pt_fate)
    np.testing.assert_array_equal(s.seg_fate, r.seg_fate)
    assert len(s.pt_marks) == 0 and len(s.seg_marks) == 0


def test_direct_matcher_single_keyframe_single_observation(oracle, abi, synth):
    """One keyframe, one observation per map feature: getCloseViewObs has nothing to choose from."""
    _need_ref(oracle, cpu=True)
    d = synth.make_match_batch(n=200, n_ref=1, n_cur=2, seed=7330)
    r = oracle.ref_match_scene(abi, d, 1)
    s = oracle.shimref_match_scene(abi, d, 1, cpu=True)
    for f in ("pt_found", "pt_level", "pt_ref", "seg_found", "seg_level", "seg_ref"):
        np.testing.assert_array_equal(getattr(s, f), getattr(r, f), err_msg=f)
    for f in ("pt_px", "seg_spx", "seg_epx"):
        a, b = getattr(s, f), getattr(r, f)
        np.testing.assert_array_equal(a[~np.isnan(b)], b[~np.isnan(b)], err_msg=f)
    assert set(np.unique(r.pt_ref)) <= {-1, 0}


def _nan_warp_scene(synth):
    """A Reprojector pass where every eighth candidate, right after an ordinary one of the same current frame, is a point the
    warp of findMatchDirect cannot handle: at the camera centre of its keyframe (a keyframe at the identity: A would be 0)
    or NaN.  Returns (data, the special rows)."""
    import torch

    from test_gpu_direct_match_cases import _append_frames

    d = synth.make_match_batch(n=1200, seed=7320)
    R0, t0 = torch.eye(3, dtype=torch.float64)[None], torch.zeros(1, 3, dtype=torch.float64)
    ident = _append_frames(synth, d, "ref", synth.pose7_from_Rt(R0, t0).numpy())
    rows = np.arange(9, d.n, 8)
    d.cur_index[rows] = d.cur_index[rows - 1]
    d.ref_index[rows[::2]] = ident
    d.ref_px[rows] = (d.cam.cx + 3.25, d.cam.cy - 7.5)
    d.pos[rows[::2]] = 0.0
    d.pos[rows[1::2]] = (np.nan, 1.0, 2.0)
    return d, rows


@pytest.mark.parametrize("cpu", [True, pytest.param(False, marks=pytest.mark.gpu)], ids=["cpu", "gpu"])
def test_direct_matcher_never_warps_a_point_at_the_keyframe_centre_or_nan(pkg, oracle, abi, synth, cpu):
    """A point at its keyframe's camera centre, or a NaN point, would give findMatchDirect a NaN affine warp, where the
    reference's warpAffine keeps the previous candidate's patch and the kernel aligns a zero patch.  Neither reaches the warp:
    getCloseViewObs, which DirectMatcher runs on the host as Reprojector does, rejects it first (its viewing direction is
    zero or NaN, so the cosine is not above 0.5).  Both sides agree on every candidate; the special ones are not found and
    leave A_cur_ref_ as the candidate before them left it, i.e. no warp was computed for them."""
    _need_ref(oracle, cpu=cpu)
    d, rows = _nan_warp_scene(synth)
    r = oracle.ref_match_scene(abi, d, 1)
    s = oracle.shimref_match_scene(abi, d, 1, cpu=cpu)
    _check_match_scene(s, r, 1, d.T_ref_w.shape[0])
    for out in (r, s):
        assert not out.pt_found[rows].any()
        np.testing.assert_array_equal(out.pt_A[rows], out.pt_A[rows - 1])
        assert np.isfinite(out.pt_A[rows]).all()
