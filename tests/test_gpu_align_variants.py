"""Every compiled variant of the alignment kernel against the CPU oracle, at the shapes where the CTA size matters.

The variants (abi.ALIGN_VARIANTS: threads per CTA x resident CTAs per SM) share one source, but the CTA size changes the
chunk-to-warp mapping of the point rounds, which warps arrive early at the round barrier, the stride of the segment
rounds, the records of segments longer than a warp, the warps that chain the chi2 and sum the segment terms, and whether
the current image level is staged in shared memory.  The planner picks <256,2> for small batches and <128,4> for large
ones; PLSVO_VARIANT forces any of them (and fails rather than run another one).  Each case's oracle result is computed
once and compared with every variant, with the tolerances of test_gpu_align.py."""
import numpy as np
import pytest

from plsvo_b200 import abi as _abi
from test_gpu_align import _check

pytestmark = pytest.mark.gpu

VARIANTS = [f"{t},{b}" for t, b in _abi.ALIGN_VARIANTS]

# points per pair on both sides of the 32-patch chunks and of the rounds of 64 / 96 / 128 / 160 / 192 / 256 patches
BOUNDARY_COUNTS = [1, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 159, 160, 161, 191, 192, 193, 255, 256, 257, 300]


def _num_sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def _long_segments(synth, data, rng, n_long, atan=None):
    """Stretch the segments across a 720p image: about half of them nearly horizontal over more than 1024 px (more than
    64 samples at level 0: three trips of a warp), the rest anywhere (mostly two trips).  atan: the ATAN camera the
    frames were rendered through; the endpoints are then lifted through its rays."""
    import torch

    B, S = data.seg_spx.shape[:2]
    spx = np.stack([rng.uniform(40, 300, (B, S)), rng.uniform(40, 680, (B, S))], -1)
    epx = np.stack([rng.uniform(980, 1240, (B, S)), rng.uniform(40, 680, (B, S))], -1)
    spx[:, :n_long, 0] = rng.uniform(30, 110, (B, n_long))
    epx[:, :n_long, 0] = rng.uniform(1170, 1250, (B, n_long))
    epx[:, :n_long, 1] = np.clip(spx[:, :n_long, 1] + rng.uniform(-60, 60, (B, n_long)), 40, 680)
    scene = synth.Scene()
    R, t = synth.pose7_to_Rt(torch.tensor(data.T_ref_w))

    def lift(px):
        p = torch.tensor(px)
        if atan is not None:
            d = synth.atan_rays(atan, p[..., 0], p[..., 1])
        else:
            d = torch.stack([(p[..., 0] - data.cam.cx) / data.cam.fx, (p[..., 1] - data.cam.cy) / data.cam.fy, torch.ones_like(p[..., 0])], -1)
        return (d / d.norm(dim=-1, keepdim=True)).numpy(), scene.intersect(R, t, d).numpy()

    data.seg_spx, data.seg_epx = np.ascontiguousarray(spx), np.ascontiguousarray(epx)
    data.seg_sf, data.seg_spos = (np.ascontiguousarray(x) for x in lift(spx))
    data.seg_ef, data.seg_epos = (np.ascontiguousarray(x) for x in lift(epx))
    data.seg_length = np.ascontiguousarray(np.linalg.norm(epx - spx, axis=-1))
    return data


def _make(name, synth, dev, atan=None):
    """(data, max_level, min_level) of one case.  atan(cam): the ATAN camera of an image size, through which the frames
    are rendered and the features lifted (None: the pinhole camera)."""
    mk = synth.make_align_batch
    if atan is not None:
        def mk(cam=synth.VGA, **kw):
            return synth.make_align_batch(cam=cam, atan=atan(cam), **kw)

    if name == "vga":  # the bench shape
        return mk(batch=16, n_pts=300, n_segs=80, device=dev, seed=6000), 4, 2
    if name == "boundaries":
        n = len(BOUNDARY_COUNTS)
        d = mk(batch=n, n_pts=300, n_segs=80, device=dev, seed=6100)
        d.pt_count = np.array(BOUNDARY_COUNTS, np.int32)
        d.seg_count = np.array([[0, 1, 13, 31, 33, 80][i % 6] for i in range(n)], np.int32)
        return d, 4, 2
    if name == "edge":  # as test_align_edge_cases: masks, ragged counts, empty / points-only / segments-only pairs, border
        d = mk(batch=12, n_pts=96, n_segs=40, device=dev, seed=3400, margin=2)
        rng = np.random.default_rng(5)
        d.pt_valid = (rng.uniform(size=(12, 96)) > 0.2).astype(np.uint8)
        d.seg_valid = (rng.uniform(size=(12, 40)) > 0.2).astype(np.uint8)
        d.pt_count = rng.integers(1, 97, 12).astype(np.int32)
        d.seg_count = rng.integers(0, 41, 12).astype(np.int32)
        d.pt_count[3] = d.seg_count[3] = 0
        d.pt_count[5] = 0
        d.seg_count[7] = 0
        return d, 4, 2
    if name == "long_segments":
        d = mk(cam=synth.HD720, batch=4, n_pts=200, n_segs=12, max_level=2, min_level=0,
               device=dev, seed=6200, motion_t=0.004, motion_r=0.0012, margin=24)
        return _long_segments(synth, d, np.random.default_rng(6201), 6, atan and atan(synth.HD720)), 2, 0
    if name == "720p":  # the finest level is not staged in shared memory
        return mk(cam=synth.HD720, batch=6, n_pts=500, n_segs=150, device=dev, seed=6300), 4, 2
    if name in ("levels_5_3", "levels_2_0"):
        max_level, min_level = (5, 3) if name == "levels_5_3" else (2, 0)
        s = 1 << (4 - min(4, max_level))
        d = mk(batch=6, n_pts=128, n_segs=32, max_level=max_level, min_level=min_level, device=dev,
               seed=6400 + max_level, motion_t=0.03 / s, motion_r=0.01 / s)
        return d, max_level, min_level
    if name == "zero_motion":  # identical images: a segment's zero mean residual makes the step NaN, stop_ on every pair
        d = mk(cam=synth.QVGA, batch=4, n_pts=40, n_segs=8, max_level=3, min_level=1, seed=21, margin=32,
               motion_t=0.0, motion_r=0.0, device=dev)
        return d, 3, 1
    if name == "ragged_pairs_per_cta":  # about three pairs of different sizes per persistent CTA, one CTA per SM
        B = 3 * _num_sms()
        d = mk(batch=B, n_pts=72, n_segs=14, device=dev, seed=6500)
        rng = np.random.default_rng(6501)
        d.pt_count = rng.integers(0, 73, B).astype(np.int32)
        d.seg_count = rng.integers(0, 15, B).astype(np.int32)
        d.pt_count[::37] = 0
        d.seg_count[::37] = 0  # empty pairs in between
        d.pt_valid = (rng.uniform(size=(B, 72)) > 0.1).astype(np.uint8)
        return d, 4, 2
    if name.startswith("pts_"):  # thousands of points per pair
        n_pts = int(name[4:])
        return mk(batch=3, n_pts=n_pts, n_segs=80, device=dev, seed=6600 + n_pts), 4, 2
    raise KeyError(name)


CASES = ["vga", "boundaries", "edge", "long_segments", "720p", "levels_5_3", "levels_2_0", "zero_motion", "ragged_pairs_per_cta"]


@pytest.fixture(scope="module")
def case(abi, synth, oracle, gen_device):
    """name -> (data, max_level, min_level, oracle result), each built and solved once."""
    cache = {}
    solve = oracle.ref_align if oracle.ref_available() else oracle.align

    def get(name):
        if name not in cache:
            data, hi, lo = _make(name, synth, gen_device)
            cache[name] = (data, hi, lo, solve(abi, data, abi.align_params(hi, lo, 30), n_threads=16))
        return cache[name]

    return get


def _compared(synth, data, ref):
    """Pairs whose result is determined by the data, or None for all of them.  One or two valid points leave the 6-DoF
    problem underdetermined (a point patch's Jacobian has rank 2): its steps come from a singular system, i.e. from
    round-off, on the GPU as in the reference, so such pairs are not compared.  Segments alone are unstable in the
    reference (test_align_segments_only): those pairs are compared while the oracle stays near the initial pose."""
    B = data.batch
    n_pts = data.pt_count if data.pt_count is not None else np.full(B, data.n_pts)
    n_segs = data.seg_count if data.seg_count is not None else np.full(B, data.n_segs)
    valid = np.ones((B, data.n_pts), bool) if data.pt_valid is None else data.pt_valid.astype(bool)
    vp = (valid & (np.arange(data.n_pts) < n_pts[:, None])).sum(1)
    moved, _ = synth.pose_error(ref.T_cur_w, data.T_cur_w)
    out = ((vp > 0) & (vp < 3)) | ((vp == 0) & (n_segs > 0) & (moved >= 0.02))
    assert out.sum() <= max(1, B // 8), f"{out.sum()} of {B} pairs not compared"
    return ~out if out.any() else None


def _check_all(synth, data, gpu, ref):
    mask = _compared(synth, data, ref)
    _check(synth, gpu, ref, mask=mask)
    m = slice(None) if mask is None else mask
    if ref.patch_levels.any():  # the restated oracle counts patches; the reference's own code (oracle/_ref) does not
        np.testing.assert_array_equal(gpu.patch_levels[m], ref.patch_levels[m])
        np.testing.assert_array_equal(gpu.patch_iters[m], ref.patch_iters[m])
    assert not (gpu.status >> 2).any(), f"chi2-order flags raised: {np.unique(gpu.status)}"


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("variant", VARIANTS)
def test_variant_matches_the_oracle(pkg, synth, case, monkeypatch, variant, name):
    data, hi, lo, ref = case(name)
    monkeypatch.setenv("PLSVO_VARIANT", variant)
    al = pkg.SparseImgAlign(hi, lo, 30)
    if name == "ragged_pairs_per_cta":
        monkeypatch.setenv("PLSVO_CTAS_PER_SM", "1")
        al.upload(data)
        al.launch()
        gpu = al.download()
    else:
        gpu = al.run(data)
    if name == "zero_motion":  # NaN step, H is NaN, the pose stays where it was (test_align_zero_residual_segment_raises_stop)
        for f in ("status", "iters", "n_tracked", "seg_killed"):
            np.testing.assert_array_equal(getattr(gpu, f), getattr(ref, f), err_msg=f)
        assert (gpu.status == 2).all()
        ang, _ = synth.pose_error(gpu.T_cur_w, ref.T_cur_w)
        assert ang.max() < 1e-12
        return
    _check_all(synth, data, gpu, ref)
    if name == "edge":
        assert gpu.status[3] == 1 and gpu.n_tracked[3] == 0
        np.testing.assert_array_equal(gpu.T_cur_w[3], data.T_cur_w[3])


@pytest.mark.parametrize("variant", VARIANTS)
def test_image_staging_changes_no_bit(pkg, case, monkeypatch, variant):
    """The current level read from shared memory or through L2: the same bytes, so the same outputs bit for bit."""
    data = case("vga")[0]
    monkeypatch.setenv("PLSVO_VARIANT", variant)
    out = {}
    for staged in ("0", "1"):
        monkeypatch.setenv("PLSVO_IMG_SMEM", staged)
        out[staged] = pkg.SparseImgAlign(4, 2, 30).run(data)
    for f in ("T_cur_w", "n_tracked", "H", "seg_killed", "iters", "status", "patch_iters", "patch_levels"):
        np.testing.assert_array_equal(getattr(out["0"], f), getattr(out["1"], f), err_msg=f)


@pytest.mark.parametrize("variant", [None, "128,4"])
@pytest.mark.parametrize("n_pts", [2048, 4096])
def test_large_point_counts_keep_the_exact_chi2(pkg, synth, case, monkeypatch, n_pts, variant):
    """Thousands of points per pair: the opaque patches of the exact-order chi2 grow with the square of the point count
    (tests/test_chi2_order_cpu.py), and the kernel must still sum chi2 in the reference's order (status 0, no flag)."""
    data, _, _, ref = case(f"pts_{n_pts}")
    if variant:
        monkeypatch.setenv("PLSVO_VARIANT", variant)
    gpu = pkg.SparseImgAlign(4, 2, 30).run(data)
    np.testing.assert_array_equal(gpu.status, 0)
    _check(synth, gpu, ref)
