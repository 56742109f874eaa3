"""Matcher::findMatchDirect on the device with a camera per image, pinhole or ATAN (FOV), in padded slots
(plsvo_match_direct_multicam_batch_run, Matcher.findMatchDirect(data, camera=[...], cam_of_ref=, cam_of_cur=)), held to
its exactness contract (include/plsvo_b200.h):

1. a candidate whose two images share camera k equals, byte for byte, the one-camera call on k (plsvo_match_direct_batch_run
   for a pinhole, plsvo_match_direct_atan_batch_run for an ATAN camera) with the frames cut out of their slots;
2. a candidate whose two cameras are pinholes, cross-camera ones included, equals the two-camera oracle
   (oracle/multicam_match_oracle.cpp) byte for byte;
3. a candidate with an ATAN camera meets the ATAN matcher's contract against that oracle: A_cur_ref within 1e-12 per
   entry, everything downstream byte-exact against the oracle's "given A" entry point fed the device's A_cur_ref, rows
   with bitwise-equal A_cur_ref equal in every output, and rows that evaluate neither tan nor atan equal outright.

Batches come from synth.make_match_multicam_batch (tests/match_multicam_cases.py): pinhole, ATAN and mixed fleets of
K = 1, 4 and 64 cameras, of one size and of several."""
import ctypes as C
from dataclasses import replace

import numpy as np
import pytest

import match_multicam_cases as mc
from _compare import assert_same_bytes

A_TOL = 1e-12
SENTINEL = -12345.5
FIELDS = ("px_cur", "success", "search_level", "A_cur_ref")


@pytest.fixture(scope="module")
def om(abi):
    import oracle_multicam_match

    oracle_multicam_match.build()
    oracle_multicam_match.load(abi)
    return oracle_multicam_match


def _assert_match(got, want, what, rows, fields=FIELDS):
    rows = np.asarray(rows)
    if rows.size == 0:
        return
    for f in fields:
        assert_same_bytes(getattr(got, f)[rows], getattr(want, f)[rows], f"{what} {f}")


def _run(pkg, d, cams, ref, cur, n_iter=10):
    return pkg.Matcher(n_iter).findMatchDirect(d, camera=cams, cam_of_ref=ref, cam_of_cur=cur)


def _one_camera(pkg, part, cam, n_iter=10):
    m = pkg.Matcher(n_iter)
    return m.findMatchDirect(part, camera=cam) if mc.is_atan(cam) else m.findMatchDirect(part)


def _fleet_case(pkg, synth, gen_device, model, k, sizes, n, seed, per_cam=2, **kw):
    cams = mc.fleet(pkg, synth, model, k, sizes)
    ref, cur = mc.images(k, per_cam)
    d, parts, groups = synth.make_match_multicam_batch(cams, ref, cur, n=n, n_pyr_levels=4, seed=seed, device=gen_device, **kw)
    return cams, ref, cur, d, parts, groups


SMALL = ((200, 150), (160, 120), (240, 180))  # K = 64 fleets: many cameras, small frames


@pytest.mark.gpu
@pytest.mark.parametrize("model", ("pinhole", "atan", "mixed"))
@pytest.mark.parametrize("k,sizes", [(1, ((640, 480),)), (1, ((752, 480),)), (4, ((640, 480),)), (4, mc.MIXED_SIZES),
                                     (64, ((200, 150),)), (64, SMALL)], ids=["1-vga", "1-752", "4-one", "4-mixed", "64-one", "64-mixed"])
def test_same_camera_rows_equal_the_one_camera_calls(pkg, synth, gen_device, model, k, sizes):
    if k == 1 and model == "mixed":
        pytest.skip("one camera has one model")
    cams, ref, cur, d, parts, groups = _fleet_case(pkg, synth, gen_device, model, k, sizes, n=1500 if k < 64 else 4000,
                                                   seed=9100 + k + len(sizes), per_cam=2 if k < 64 else 1)
    got = _run(pkg, d, cams, ref, cur)
    checked = 0
    for j, (part, g) in enumerate(zip(parts, groups)):
        if part is None:
            continue
        want = _one_camera(pkg, part, cams[j])
        for f in FIELDS:
            assert_same_bytes(getattr(got, f)[g], getattr(want, f), f"camera {j} ({model}, {cams[j].width}x{cams[j].height}) {f}")
        checked += len(g)
    assert checked >= d.n // 3
    assert got.success.any()


def _cross_case(pkg, synth, gen_device, seed=9200, **kw):
    cams = mc.off_centre_mix(pkg, synth) + mc.fleet(pkg, synth, "mixed", 4, mc.MIXED_SIZES) + mc.atans(pkg, 3)[2:]  # the last: d0 = 0
    ref, cur = mc.images(len(cams), 2)
    d, parts, groups = synth.make_match_multicam_batch(cams, ref, cur, n=3000, n_pyr_levels=5, seed=seed, device=gen_device,
                                                       same_camera_frac=0.2, **kw)
    return cams, ref, cur, d


@pytest.mark.gpu
def test_pinhole_rows_equal_the_two_camera_oracle(pkg, abi, synth, gen_device, om):
    cams, ref, cur, d = _cross_case(pkg, synth, gen_device)
    got, want = _run(pkg, d, cams, ref, cur), om.match_direct(abi, cams, ref, cur, d)
    rows = mc.pinhole_rows(cams, ref, cur, d)
    cross = rows[ref[d.ref_index[rows]] != cur[d.cur_index[rows]]]
    assert len(cross) > 100
    _assert_match(got, want, "pinhole rows", rows)


@pytest.mark.gpu
def test_atan_rows_meet_the_atan_contract(pkg, abi, synth, gen_device, om):
    cams, ref, cur, d = _cross_case(pkg, synth, gen_device, seed=9210)
    got, want = _run(pkg, d, cams, ref, cur), om.match_direct(abi, cams, ref, cur, d)
    rows = np.setdiff1d(np.arange(d.n), mc.pinhole_rows(cams, ref, cur, d))
    assert len(rows) > 1000
    warped = rows[want.search_level[rows] >= 0]
    assert_same_bytes(got.search_level[rows] >= 0, want.search_level[rows] >= 0, "in-frame test")
    assert np.abs(got.A_cur_ref[warped] - want.A_cur_ref[warped]).max() <= A_TOL
    given = om.match_direct_given_A(abi, cams, ref, cur, d, np.where(np.isnan(got.A_cur_ref), 0.0, got.A_cur_ref))
    _assert_match(got, given, "downstream of the device's A_cur_ref", rows)
    same_A = warped[(got.A_cur_ref[warped].view(np.uint64) == want.A_cur_ref[warped].view(np.uint64)).all(1)]
    assert len(same_A) > len(warped) // 4
    _assert_match(got, want, "bitwise-equal A_cur_ref", same_A)
    plain = np.array([not mc.is_atan(c) or c.s_ == 0.0 for c in cams])  # d0 == 0: neither tan nor atan is evaluated
    free = rows[plain[ref[d.ref_index[rows]]] & plain[cur[d.cur_index[rows]]]]
    assert len(free) > 50
    _assert_match(got, want, "rows without tan / atan", free)


@pytest.mark.gpu
def test_random_padding_gives_the_bytes_of_zero_padding(pkg, synth, gen_device):
    cams = mc.off_centre_mix(pkg, synth)
    ref, cur = mc.images(3, 2)
    kw = dict(n=2000, n_pyr_levels=4, seed=9300, device=gen_device)
    d0 = synth.make_match_multicam_batch(cams, ref, cur, fill=0, **kw)[0]
    dr = synth.make_match_multicam_batch(cams, ref, cur, fill=np.random.Generator(np.random.PCG64(5)), **kw)[0]
    assert any((a != b).any() for a, b in zip(d0.ref_pyr.values(), dr.ref_pyr.values()))
    _assert_match(_run(pkg, dr, cams, ref, cur), _run(pkg, d0, cams, ref, cur), "random padding", np.arange(d0.n))


@pytest.mark.gpu
def test_edgelets_null_outputs_and_the_A_sentinel(pkg, abi, synth, gen_device, om):
    cams, ref, cur, d = _cross_case(pkg, synth, gen_device, seed=9400, edgelet_frac=0.6)
    d.n_iter = 10
    want = om.match_direct(abi, cams, ref, cur, d)
    rows = mc.pinhole_rows(cams, ref, cur, d)
    assert d.is_edgelet[rows].sum() > 300
    tab, r32, c32 = abi.make_match_cameras(cams), ref.astype(np.int32), cur.astype(np.int32)
    ctx = pkg.api.default_context()
    b, keep = abi.make_match_batch(d)
    out = abi.MatchOut(d.n)
    out.A_cur_ref[:] = SENTINEL
    nulls = abi.MatchResult(out.struct.px_cur, out.struct.success, None, None)
    i32 = C.POINTER(C.c_int32)
    for res in (out.struct, nulls):
        ctx.check(ctx.lib.plsvo_match_direct_multicam_batch_run(ctx.handle, tab, len(cams), r32.ctypes.data_as(i32), c32.ctypes.data_as(i32),
                                                                 C.byref(b), C.byref(res)), "plsvo_match_direct_multicam_batch_run")
        _assert_match(out, want, "edgelets", rows, ("px_cur", "success"))
    rejected = want.search_level == -1
    assert rejected.sum() > 5 and (out.A_cur_ref[rejected] == SENTINEL).all()
    _assert_match(out, want, "A_cur_ref", rows[~rejected[rows]], ("A_cur_ref",))
    no_edge = replace(d, is_edgelet=None, ref_grad=None)
    _assert_match(_run(pkg, no_edge, cams, ref, cur), om.match_direct(abi, cams, ref, cur, no_edge), "no edgelets", rows)


@pytest.mark.gpu
def test_in_frame_test_and_align_bounds_at_each_cameras_own_border(pkg, abi, synth, gen_device, om):
    """Reference pixels and projections placed across the right and bottom borders of cameras smaller than the slot: the
    in-frame test (b = 6 at the reference level) and align2D / align1D use the image's own camera, not the slot."""
    cams = [synth.Camera(640, 480, 420.0, 420.0, 319.5, 239.5), synth.Camera(400, 300, 262.0, 262.0, 199.5, 149.5),
            pkg.ATANCamera(320, 260, 0.66 * 1.5, 0.88 * 1.2, 0.5, 0.5, 0.0)]
    ref, cur = np.array([0, 1, 2, 1], np.int32), np.array([1, 2, 0, 2], np.int32)
    d = synth.make_match_multicam_batch(cams, ref, cur, n=2400, n_pyr_levels=4, seed=9500, device=gen_device, same_camera_frac=0.5)[0]
    rng = np.random.Generator(np.random.PCG64(9501))
    kr, kc = ref[d.ref_index], cur[d.cur_index]
    w = np.array([c.width for c in cams])[kr]
    h = np.array([c.height for c in cams])[kr]
    s = 1 << d.ref_level
    edge = rng.integers(0, 2, d.n).astype(bool)
    off = rng.integers(-8, 2, d.n) * s + rng.uniform(0, 1, d.n)
    d.ref_px[edge, 0] = (w[edge] // s[edge]) * s[edge] - 6 * s[edge] + off[edge]
    d.ref_px[~edge, 1] = (h[~edge] // s[~edge]) * s[~edge] - 6 * s[~edge] + off[~edge]
    wc = np.array([c.width for c in cams])[kc]
    d.px_cur[::3, 0] = wc[::3] - rng.uniform(0, 12, len(wc[::3]))
    got, want = _run(pkg, d, cams, ref, cur), om.match_direct(abi, cams, ref, cur, d)
    _assert_match(got, want, "borders", np.arange(d.n))
    small = kr != 0
    assert (got.search_level[small] == -1).sum() > 100 and (got.search_level[small] >= 0).sum() > 100


@pytest.mark.gpu
def test_every_batch_size_gives_the_rows_of_the_full_batch(pkg, synth, gen_device):
    cams = mc.fleet(pkg, synth, "mixed", 4, mc.MIXED_SIZES)
    ref, cur = mc.images(4, 2)
    d = synth.make_match_multicam_batch(cams, ref, cur, n=(1 << 17) + 1, n_pyr_levels=4, seed=9600, device=gen_device)[0]
    full = _run(pkg, d, cams, ref, cur)
    fields = ("ref_index", "cur_index", "ref_px", "ref_f", "ref_level", "is_edgelet", "ref_grad", "pos", "px_cur", "px_cur_gt")
    for n in (1, 129):
        for sel in (np.arange(n), np.arange(d.n - n, d.n)):
            part = replace(d, **{f: np.ascontiguousarray(getattr(d, f)[sel]) for f in fields})
            got = _run(pkg, part, cams, ref, cur)
            for f in FIELDS:
                assert_same_bytes(getattr(got, f), getattr(full, f)[sel], f"batch of {n} {f}")


@pytest.mark.gpu
def test_rejections_leave_the_context_usable(pkg, abi, synth, gen_device):
    cams = mc.off_centre_mix(pkg, synth)
    ref, cur = mc.images(3, 1)
    d = synth.make_match_multicam_batch(cams, ref, cur, n=300, n_pyr_levels=4, seed=9700, device=gen_device)[0]
    d.n_iter = 10
    ctx = pkg.api.default_context()
    b, keep = abi.make_match_batch(d)
    i32 = C.POINTER(C.c_int32)
    r32, c32 = ref.astype(np.int32), cur.astype(np.int32)

    def call(tab, n_cams, r, c):
        out = abi.MatchOut(d.n)
        out.A_cur_ref[:] = SENTINEL
        rc = ctx.lib.plsvo_match_direct_multicam_batch_run(ctx.handle, tab, n_cams, r, c, C.byref(b), C.byref(out.struct))
        return rc, out

    def tab_with(k, part, **kw):
        t = abi.make_match_cameras(cams)
        for f, v in kw.items():
            setattr(getattr(t[k], part) if part else t[k], f, v)
        return t

    good = abi.make_match_cameras(cams)
    pr, pc = r32.ctypes.data_as(i32), c32.ctypes.data_as(i32)
    big = np.array([0, 3, 1], np.int32)
    neg = np.array([0, -1, 1], np.int32)
    bad = [(None, 3, pr, pc), (good, 3, None, pc), (good, 3, pr, None), (good, 0, pr, pc), (good, 3, big.ctypes.data_as(i32), pc),
           (good, 3, pr, neg.ctypes.data_as(i32)), (tab_with(0, None, model=2), 3, pr, pc),
           (tab_with(0, "pinhole", cx=float("inf")), 3, pr, pc), (tab_with(0, "pinhole", fx=0.0), 3, pr, pc),
           (tab_with(1, "atan", fy=-0.5), 3, pr, pc), (tab_with(1, "atan", d0=float("nan")), 3, pr, pc),
           (tab_with(0, "pinhole", width=d.cam.width + 1), 3, pr, pc), (tab_with(1, "atan", height=d.cam.height + 1), 3, pr, pc),
           (tab_with(2, "atan", width=7), 3, pr, pc)]  # level n_pyr_levels - 1 = 3 of a 7-pixel-wide current camera
    for tab, n_cams, r, c in bad:
        rc, out = call(tab, n_cams, r, c)
        assert rc == abi.ERR_INVALID, ctx.lib.plsvo_last_error(ctx.handle)
        assert (out.A_cur_ref == SENTINEL).all() and not out.success.any()
    lvl = d.ref_level.copy()
    d.ref_level[:] = 3
    rc, _ = call(tab_with(2, "atan", width=7), 3, pr, (np.zeros(3, np.int32)).ctypes.data_as(i32))  # a keyframe camera at level 3
    assert rc == abi.ERR_INVALID and b"ref image" in ctx.lib.plsvo_last_error(ctx.handle)
    d.ref_level[:] = lvl
    b, keep = abi.make_match_batch(d)
    rc, out = call(good, 3, pr, pc)
    assert rc == abi.OK and out.success.any()
    with pytest.raises(pkg.api.PlsvoError):
        pkg.Matcher(10).findMatchDirect(d, camera=cams, cam_of_ref=ref)
