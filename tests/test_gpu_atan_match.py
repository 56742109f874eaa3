"""Matcher::findMatchDirect on the device for frames from an ATAN (FOV) camera (plsvo_match_direct_atan_batch_run,
Matcher.findMatchDirect(data, camera=ATANCamera)), held to its exactness contract (include/plsvo_b200.h):

1. A_cur_ref agrees with the oracle's within 1e-12 per entry (the device's tan / atan are not glibc's);
2. downstream of A_cur_ref everything is exact: success, search_level and px_cur equal byte for byte what the oracle's
   "given A" entry point computes from the device's own A_cur_ref;
3. rows whose A_cur_ref is bitwise equal to the oracle's match it byte for byte in every output;
4. rows that evaluate neither tan nor atan (d0 = 0, or inside both cut-offs) match the oracle byte for byte, A_cur_ref
   included; with d0 = 0 they also equal plsvo_match_direct_batch_run on the camera's members as pinhole intrinsics.

The cases (tests/atan_match_cases.py) are checked on the CPU to reach both cut-offs on both sides and every exit."""
import ctypes as C
from dataclasses import replace

import numpy as np
import pytest

import atan_match_cases as amc
from _compare import assert_same_bytes

A_TOL = 1e-12
SENTINEL = -12345.5


@pytest.fixture(scope="module")
def om(abi):
    import oracle_atan_match

    oracle_atan_match.build()
    oracle_atan_match.load(abi)
    return oracle_atan_match


def _assert_match(got, want, what, rows=slice(None), fields=("px_cur", "success", "search_level", "A_cur_ref")):
    if isinstance(rows, np.ndarray) and not rows.any():
        return
    for f in fields:
        assert_same_bytes(getattr(got, f)[rows], getattr(want, f)[rows], f"{what} {f}")


def check_contract(om, abi, cam, d, got, what):
    """The four clauses of the module docstring; returns (largest |A - A_oracle|, share of rows with bitwise-equal A)."""
    want = om.match_direct_members(abi, cam, d)
    live = want.search_level >= 0
    assert_same_bytes(got.search_level >= 0, live, f"{what} in-frame")
    # 1. A close to the oracle's (NaN where the oracle's is NaN)
    ga, wa = got.A_cur_ref[live], want.A_cur_ref[live]
    assert_same_bytes(np.isnan(ga), np.isnan(wa), f"{what} A NaN pattern")
    fin = np.isfinite(wa)
    diff = np.abs(ga[fin] - wa[fin])
    dmax = float(diff.max()) if diff.size else 0.0
    assert dmax <= A_TOL, f"{what}: |A - A_oracle| = {dmax:.3e}"
    # 2. downstream exact given the device's A
    given = om.match_direct_given_A(abi, d, np.where(live[:, None], got.A_cur_ref, 0.0))
    _assert_match(got, given, f"{what} given A", fields=("px_cur", "success", "search_level"))
    # 3. bitwise-equal A: every output equal
    same = live & (got.A_cur_ref.view(np.uint64) == want.A_cur_ref.view(np.uint64)).all(-1) | ~live
    _assert_match(got, want, f"{what} equal-A rows", rows=same)
    # 4. no transcendental call: every output equal
    free = amc.transcendental_free(cam, d)
    _assert_match(got, want, f"{what} transcendental-free rows", rows=free)
    return dmax, float(same[live].mean()) if live.any() else 1.0


CASES = ([("VGA", d0, L) for d0 in (0.3, 0.93) for L in range(1, 9)] + [("EUROC", d0, L) for d0 in (0.3, 0.93) for L in (1, 4, 5)] +
         [("off-centre", 0.93, 5), ("telephoto", 0.93, 4), ("telephoto", 0.3, 1)])


def _camera(pkg, synth, size, d0):
    if size == "off-centre":
        return amc.off_centre(pkg, d0)
    if size == "telephoto":
        return amc.telephoto(pkg, d0)
    return amc.camera(pkg, synth, size, d0)


@pytest.mark.gpu
@pytest.mark.parametrize("size,d0,L", CASES, ids=lambda v: str(v))
def test_gpu_atan_find_match_direct_meets_the_contract(pkg, abi, synth, om, size, d0, L):
    cam = _camera(pkg, synth, size, d0)
    d = amc.case(pkg, synth, cam, n=1500, n_pyr_levels=L, seed=8100 + 7 * L + int(10 * d0))
    got = pkg.Matcher(10).findMatchDirect(d, camera=cam)
    dmax, share = check_contract(om, abi, cam, d, got, f"{size} d0={d0} L={L}")
    print(f"{size} d0={d0} L={L}: max |dA| {dmax:.3e}, bitwise-equal A on {100 * share:.1f}% of in-frame rows")
    if size != "telephoto":  # at fx_ = 6400 a patch sees too little texture of the scene for most alignments to converge
        assert got.success.mean() > 0.3


@pytest.mark.gpu
@pytest.mark.parametrize("n_iter", (0, 1, 3, 10, 30))
def test_gpu_atan_find_match_direct_every_align_max_iter(pkg, abi, synth, om, n_iter):
    cam = amc.camera(pkg, synth, "EUROC", 0.93)
    d = amc.case(pkg, synth, cam, n=1500, n_pyr_levels=5, seed=8300)
    check_contract(om, abi, cam, d, pkg.Matcher(n_iter).findMatchDirect(d, camera=cam), f"align_max_iter={n_iter}")


@pytest.mark.gpu
@pytest.mark.parametrize("L", (1, 4, 8))
def test_gpu_atan_without_distortion_is_the_pinhole_matcher(pkg, abi, synth, om, L):
    """d0 = 0: no transcendental call anywhere, so every output equals the oracle's and the pinhole kernel's on the
    camera's members, byte for byte."""
    cam = amc.camera(pkg, synth, "VGA", 0.0)
    d = amc.case(pkg, synth, cam, n=1500, n_pyr_levels=L, seed=8400 + L)
    got = pkg.Matcher(10).findMatchDirect(d, camera=cam)
    _assert_match(got, om.match_direct_members(abi, cam, d), "oracle")
    _assert_match(got, pkg.Matcher(10).findMatchDirect(amc.with_camera(d, amc.pinhole_of(synth, cam))), "pinhole kernel")


@pytest.mark.gpu
def test_gpu_atan_batches_of_every_size_match_their_rows_in_the_full_batch(pkg, abi, synth, om):
    cam = amc.camera(pkg, synth, "VGA", 0.93)
    n = (1 << 17) + 1
    d = amc.case(pkg, synth, cam, n=n, n_pyr_levels=4, seed=8500)
    full = pkg.Matcher(10).findMatchDirect(d, camera=cam)
    sub_rows = np.arange(0, n, 64)
    sub = _take(d, sub_rows)
    check_contract(om, abi, cam, sub, _take_out(abi, full, sub_rows), "2^17+1 (every 64th row)")
    rng = np.random.default_rng(8501)
    for k in (1, 127, 128, 129):
        rows = np.sort(rng.choice(n, k, replace=False))
        got = pkg.Matcher(10).findMatchDirect(_take(d, rows), camera=cam)
        _assert_match(got, _take_out(abi, full, rows), f"batch of {k}")


def _take(d, rows):
    t = lambda a: None if a is None else np.ascontiguousarray(a[rows])  # noqa: E731
    return replace(d, ref_index=t(d.ref_index), cur_index=t(d.cur_index), ref_px=t(d.ref_px), ref_f=t(d.ref_f), ref_level=t(d.ref_level),
                   is_edgelet=t(d.is_edgelet), ref_grad=t(d.ref_grad), pos=t(d.pos), px_cur=t(d.px_cur), px_cur_gt=t(d.px_cur_gt))


def _take_out(abi, out, rows):
    o = abi.MatchOut(len(rows))
    for f in ("px_cur", "success", "search_level", "A_cur_ref"):
        getattr(o, f)[:] = getattr(out, f)[rows]
    return o


@pytest.mark.gpu
def test_gpu_atan_null_pointers_and_sentinel(pkg, abi, synth, om):
    cam = amc.camera(pkg, synth, "EUROC", 0.93)
    d = amc.case(pkg, synth, cam, n=1500, n_pyr_levels=5, seed=8600)
    d.n_iter = 10
    ctx = pkg.default_context()

    def run_gpu(data, out):
        b, keep = abi.make_match_batch(data)
        assert ctx.lib.plsvo_match_direct_atan_batch_run(ctx.handle, C.byref(cam.struct), C.byref(b), C.byref(out.struct)) == abi.OK
        return out

    o = abi.MatchOut(d.n)
    o.A_cur_ref[:] = SENTINEL
    got = run_gpu(d, o)
    rejected = got.search_level < 0
    assert rejected.any() and (got.A_cur_ref[rejected] == SENTINEL).all()
    ref = pkg.Matcher(10).findMatchDirect(d, camera=cam)
    _assert_match(got, ref, "sentinel", rows=~rejected)
    # NULL is_edgelet: every candidate runs align2D
    dn = replace(d, is_edgelet=None, ref_grad=None)
    got_n = run_gpu(dn, abi.MatchOut(d.n))
    check_contract(om, abi, cam, dn, got_n, "no is_edgelet")
    _assert_match(got_n, run_gpu(replace(d, is_edgelet=np.zeros_like(d.is_edgelet)), abi.MatchOut(d.n)), "NULL vs all-zero is_edgelet")
    # NULL search_level and A_cur_ref
    o = abi.MatchOut(d.n)
    o.struct.search_level = C.POINTER(C.c_int32)()
    o.struct.A_cur_ref = C.POINTER(C.c_double)()
    got = run_gpu(d, o)
    _assert_match(got, ref, "NULL outputs", fields=("px_cur", "success"))


@pytest.mark.gpu
def test_gpu_atan_rejects_bad_cameras_and_the_context_stays_usable(pkg, abi, synth, om):
    cam = amc.camera(pkg, synth, "VGA", 0.93)
    d = amc.case(pkg, synth, cam, n=400, n_pyr_levels=4, seed=8700)
    d.n_iter = 10
    ctx = pkg.default_context()
    b, keep = abi.make_match_batch(d)
    s = cam.struct
    bad = [abi.AtanCamera(s.width + 1, s.height, s.fx, s.fy, s.cx, s.cy, s.d0), abi.AtanCamera(s.width, s.height, float("nan"), s.fy, s.cx, s.cy, s.d0),
           abi.AtanCamera(s.width, s.height, s.fx, s.fy, s.cx, s.cy, float("inf")), abi.AtanCamera(s.width, s.height, 0.0, s.fy, s.cx, s.cy, s.d0),
           abi.AtanCamera(s.width, s.height, s.fx, -1.0, s.cx, s.cy, s.d0)]
    msgs = [b"size differs", b"non-finite", b"non-finite", b"positive", b"positive"]
    for c, m in zip(bad, msgs):
        out = abi.MatchOut(d.n)
        out.A_cur_ref[:] = SENTINEL
        assert ctx.lib.plsvo_match_direct_atan_batch_run(ctx.handle, C.byref(c), C.byref(b), C.byref(out.struct)) == abi.ERR_INVALID
        assert m in ctx.lib.plsvo_last_error(ctx.handle)
        assert (out.A_cur_ref == SENTINEL).all() and not out.success.any()  # nothing was queued
    got = pkg.Matcher(10, ctx).findMatchDirect(d, camera=cam)
    check_contract(om, abi, cam, d, got, "after the refusals")
    # the Python layer refuses a wrong size and a wrong camera type before the call
    with pytest.raises(pkg.api.PlsvoError):
        pkg.Matcher(10, ctx).findMatchDirect(d, camera=amc.camera(pkg, synth, "EUROC", 0.93))
    with pytest.raises(TypeError):
        pkg.Matcher(10, ctx).findMatchDirect(d, camera=amc.pinhole_of(synth, cam))


@pytest.mark.gpu
def test_gpu_atan_refines_towards_the_true_projection(pkg, abi, synth):
    cam = amc.camera(pkg, synth, "EUROC", 0.93)
    d = synth.make_match_batch(cam=amc.pinhole_of(synth, cam), n=3000, seed=8800, edgelet_frac=0.0, atan=cam)
    o = pkg.Matcher(10).findMatchDirect(d, camera=cam)
    ok = o.success.astype(bool)
    assert ok.mean() > 0.85
    before = np.abs(d.px_cur - d.px_cur_gt).max(axis=1)
    after = np.abs(o.px_cur - d.px_cur_gt).max(axis=1)
    assert np.median(after[ok]) < 0.35 * np.median(before[ok])


@pytest.mark.gpu
def test_gpu_direct_matcher_on_atan_frames_agrees_with_the_reference(pkg, abi, synth, om):
    """The reprojector pass over reference-typed frames holding a vk::ATANCamera, answered by the drop-in DirectMatcher on
    the device, against the reference's own Matcher on the same objects: chosen observations, found, search levels and
    refined positions identical, A_cur_ref_ within the contract's bound."""
    if not om.ref_available() or not om.build_shimref():
        pytest.skip("oracle/_ref's ATAN scene libraries are not built (the reference sources were not present)")
    cam = amc.camera(pkg, synth, "EUROC", 0.93)
    d = synth.make_match_batch(cam=amc.pinhole_of(synth, cam), n=1200, n_ref=4, n_cur=3, seed=8900, n_pyr_levels=4, atan=cam)
    ref = om.ref_match_scene(abi, cam, d, 3)
    shim = om.shimref_match_scene(abi, cam, d, 3)
    for k in ("pt_found", "pt_px", "pt_level", "pt_ref", "seg_found", "seg_spx", "seg_epx", "seg_level", "seg_ref"):
        assert_same_bytes(getattr(shim, k), getattr(ref, k), k)
    for k in ("pt_A", "seg_A"):
        a, b = getattr(shim, k), getattr(ref, k)
        assert_same_bytes(np.isnan(a), np.isnan(b), f"{k} NaN pattern")
        fin = np.isfinite(b)
        assert np.abs(a[fin] - b[fin]).max() <= A_TOL, k
    assert ref.pt_found.mean() > 0.5 and ref.seg_found.any()
