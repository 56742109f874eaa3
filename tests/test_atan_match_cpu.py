"""Matcher::findMatchDirect for ATAN (FOV) frames without a GPU: the oracle (oracle/atan_match_oracle.cpp) against the
reference's own matcher.cpp driven by the stand-in vk::ATANCamera, against the pinhole oracle when the camera has no
distortion, its "given A_cur_ref" entry point against itself, and the reach of the cases the GPU tests use
(tests/atan_match_cases.py): both distortion cut-offs on both sides, and every exit of the pinhole matcher."""
import hashlib

import numpy as np
import pytest

import atan_match_cases as amc
from _compare import assert_same_bytes

D0S = (0.0, 0.3, 0.93, -0.3, 2.4)


@pytest.fixture(scope="module")
def om(abi):
    import oracle_atan_match

    oracle_atan_match.build()
    oracle_atan_match.load(abi)
    return oracle_atan_match


def _assert_match(got, want, what, rows=slice(None)):
    for f in ("px_cur", "success", "search_level", "A_cur_ref"):
        assert_same_bytes(getattr(got, f)[rows], getattr(want, f)[rows], f"{what} {f}")


def _ref_rows(d):
    """Rows the reference's own matcher can be asked about: points at the reference camera centre or NaN have a NaN
    viewing direction, so its getCloseViewObs rejects them before findMatchDirect's own code runs (as in the pinhole pin,
    tests/test_gpu_direct_match_cases.py)."""
    return np.flatnonzero(~(np.isnan(d.pos).any(1) | (d.pos == 0).all(1)))


@pytest.mark.parametrize("d0", D0S)
@pytest.mark.parametrize("size", ("VGA", "EUROC"))
def test_atan_oracle_is_bit_identical_to_the_reference_matcher(pkg, abi, synth, om, size, d0):
    if not om.build_ref():
        pytest.skip("oracle/_ref/libplsvo_atan_match_ref.so is not built (the reference sources are not present)")
    cam = amc.camera(pkg, synth, size, d0)
    d = amc.case(pkg, synth, cam, n=900, n_pyr_levels=4, seed=7600 + int(100 * d0) % 97)
    _assert_match(om.match_direct(abi, cam, d), om.ref_match_direct(abi, cam, d), f"{size} d0={d0}", _ref_rows(d))


def test_atan_oracle_off_centre_and_telephoto_cameras_match_the_reference(pkg, abi, synth, om):
    if not om.build_ref():
        pytest.skip("oracle/_ref/libplsvo_atan_match_ref.so is not built (the reference sources are not present)")
    for cam in (amc.off_centre(pkg), amc.telephoto(pkg)):
        d = amc.case(pkg, synth, cam, n=600, n_pyr_levels=5, seed=7650)
        _assert_match(om.match_direct(abi, cam, d), om.ref_match_direct(abi, cam, d), f"fx_={cam.fx_}", _ref_rows(d))


@pytest.mark.parametrize("n_pyr_levels", (1, 3, 5, 8))
def test_without_distortion_the_atan_oracle_is_the_pinhole_oracle(pkg, abi, synth, oracle, om, n_pyr_levels):
    cam = amc.camera(pkg, synth, "VGA", 0.0)
    d = amc.case(pkg, synth, cam, n=800, n_pyr_levels=n_pyr_levels, seed=7700 + n_pyr_levels)
    pin = amc.pinhole_of(synth, cam)
    assert (pin.fx, pin.fy, pin.cx, pin.cy) == (cam.fx_, cam.fy_, cam.cx_, cam.cy_)
    _assert_match(om.match_direct(abi, cam, d), oracle.match_direct(abi, amc.with_camera(d, pin), 4), f"L={n_pyr_levels}")


@pytest.mark.parametrize("d0", (0.3, 0.93))
def test_given_A_entry_point_reproduces_the_oracle(pkg, abi, synth, om, d0):
    """Downstream of A_cur_ref the oracle reads no camera: fed its own warp matrices, the "given A" entry point returns every
    output byte for byte, including for rejected rows (whose A is not read)."""
    cam = amc.camera(pkg, synth, "EUROC", d0)
    d = amc.case(pkg, synth, cam, n=800, n_pyr_levels=5, seed=7800)
    want = om.match_direct(abi, cam, d)
    _assert_match(om.match_direct_given_A(abi, d, want.A_cur_ref), want, f"d0={d0}")
    # the members entry point (what the device kernel receives) computes the same bits as the constructor's
    _assert_match(om.match_direct_members(abi, cam, d), want, "members")


def test_atan_oracle_refines_towards_the_true_projection(pkg, abi, synth, om):
    cam = amc.camera(pkg, synth, "VGA", 0.93)
    d = synth.make_match_batch(cam=synth.VGA, n=1500, seed=7010, edgelet_frac=0.0, atan=cam)
    o = om.match_direct(abi, cam, d)
    ok = o.success.astype(bool)
    assert ok.mean() > 0.85
    before = np.abs(d.px_cur - d.px_cur_gt).max(axis=1)
    after = np.abs(o.px_cur - d.px_cur_gt).max(axis=1)
    assert np.median(after[ok]) < 0.35 * np.median(before[ok])


@pytest.mark.parametrize("size", ("VGA", "EUROC", "telephoto"))
def test_cases_reach_both_cut_offs_and_every_exit(pkg, abi, synth, om, size):
    cam = amc.telephoto(pkg) if size == "telephoto" else amc.camera(pkg, synth, size, 0.93)
    d = amc.case(pkg, synth, cam, n=900, n_pyr_levels=4, seed=7900)
    o = om.match_direct(abi, cam, d)
    rd, r = amc.cut_off_arguments(cam, d)
    live = o.search_level >= 0
    # cam2world: r_d <= 0.01 (no tan) and > 0.01; world2cam: r < 0.001 (no atan) and >= 0.001, on in-frame rows
    assert ((rd <= 0.01) & live[:, None]).any() and ((rd > 0.01) & live[:, None]).any()
    assert ((r < 0.001) & live[:, None]).any() and ((r >= 0.001) & live[:, None]).any()
    # rows that call neither tan nor atan (the GPU tests hold them to the oracle byte for byte): only a long focal length
    # fits the three projections of a warp into the 0.001 disc
    if size == "telephoto":
        assert amc.transcendental_free(cam, d)[live].sum() >= 4
    # the exits of findMatchDirect: in-frame rejection, NaN warp, clamped search level, align2D and align1D, each
    # converging and not
    assert (~live).any()
    assert np.isnan(o.A_cur_ref[live]).any()
    assert (o.search_level == d.n_pyr_levels - 1).any() and (o.search_level == 0).any()
    edge = d.is_edgelet.astype(bool)
    for sel in (edge & live, ~edge & live):
        assert o.success[sel].any() and not o.success[sel].all()


def test_synth_without_atan_is_unchanged(synth):
    """make_match_batch(atan=None) draws, renders and lifts exactly as before the atan argument existed: these digests were
    taken from the generator before it."""
    d = synth.make_match_batch(n=300, seed=7000)
    h = hashlib.sha256()
    for k in ("ref_pyr", "cur_pyr"):
        for l in sorted(getattr(d, k)):
            h.update(np.ascontiguousarray(getattr(d, k)[l]).tobytes())
    for k in ("T_ref_w", "T_cur_w", "ref_index", "cur_index", "ref_px", "ref_f", "ref_level", "is_edgelet", "ref_grad", "pos", "px_cur",
              "px_cur_gt"):
        h.update(np.ascontiguousarray(getattr(d, k)).tobytes())
    assert h.hexdigest() == SYNTH_DIGEST


SYNTH_DIGEST = "b3760a8a0f3300c69a40b9983d8c71683d83f4102fce909aa72462549bf5ff17"


def test_direct_matcher_replays_the_reprojector_loop_on_atan_frames_cpu(pkg, abi, synth, om):
    """The drop-in DirectMatcher on reference-typed frames holding a vk::ATANCamera, with the C ABI answered by the CPU
    oracle (oracle/atan_abi_on_oracle.cpp): it must find the camera through the frame, pack the candidates and replay the
    reprojector's per-candidate reads exactly as the reference's own Matcher leaves them, over map points and segments
    observed in up to three keyframes."""
    if not om.build_ref() or not om.build_shimref(cpu=True):
        pytest.skip("the reference sources are not present: oracle/_ref's ATAN scene libraries are not built")
    cam = amc.camera(pkg, synth, "EUROC", 0.93)
    d = synth.make_match_batch(cam=amc.pinhole_of(synth, cam), n=1200, n_ref=4, n_cur=3, seed=8900, n_pyr_levels=4, atan=cam)
    ref = om.ref_match_scene(abi, cam, d, 3)
    shim = om.shimref_match_scene(abi, cam, d, 3, cpu=True)
    for k in ("pt_found", "pt_px", "pt_level", "pt_A", "pt_ref", "seg_found", "seg_spx", "seg_epx", "seg_level", "seg_A", "seg_ref"):
        assert_same_bytes(getattr(shim, k), getattr(ref, k), k)
    assert ref.pt_found.mean() > 0.5 and ref.seg_found.any() and (ref.pt_ref >= 0).all()
