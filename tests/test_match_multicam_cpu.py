"""Matcher::findMatchDirect with a camera per image without a GPU: the two-camera oracle (oracle/multicam_match_oracle.cpp)
against the reference's own matcher.cpp driven by frames that hold distinct stand-in cameras, against the one-camera
pinhole and ATAN oracles when every image shares one camera, the layout of plsvo_match_camera, and the argument errors of
Matcher.findMatchDirect(data, camera=[...], cam_of_ref=, cam_of_cur=)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import match_multicam_cases as mc
from _compare import assert_same_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("px_cur", "success", "search_level", "A_cur_ref")


@pytest.fixture(scope="module")
def om(abi):
    import oracle_multicam_match

    oracle_multicam_match.build()
    oracle_multicam_match.load(abi)
    return oracle_multicam_match


def _assert_match(got, want, what, rows):
    for f in FIELDS:
        assert_same_bytes(getattr(got, f)[rows], getattr(want, f)[rows], f"{what} {f}")


def _ref_rows(d):
    """Rows the reference's own matcher can be asked about (see tests/test_atan_match_cpu.py: a point at the reference
    camera centre or NaN is rejected by getCloseViewObs before findMatchDirect's own code runs)."""
    return np.flatnonzero(~(np.isnan(d.pos).any(1) | (d.pos == 0).all(1)))


def _fleets(pkg, synth):
    return {
        "pinhole3": mc.pinholes(synth, 3),
        "atan3": mc.atans(pkg, 3, d0s=(0.0, 0.3, 0.93)),
        "mix": mc.fleet(pkg, synth, "mixed", 4),
        "sizes": mc.off_centre_mix(pkg, synth),
    }


@pytest.mark.parametrize("fleet", ("pinhole3", "atan3", "mix", "sizes"))
def test_two_camera_oracle_is_bit_identical_to_the_reference_matcher(pkg, abi, synth, om, fleet):
    if not om.build_ref():
        pytest.skip("oracle/_ref/libplsvo_multicam_match_ref.so is not built (the reference sources are not present)")
    cams = _fleets(pkg, synth)[fleet]
    ref, cur = mc.images(len(cams), 2)
    d, _, _ = synth.make_match_multicam_batch(cams, ref, cur, n=900, n_pyr_levels=4, seed=9800 + len(fleet), same_camera_frac=0.3)
    rows = _ref_rows(d)
    cross = rows[ref[d.ref_index[rows]] != cur[d.cur_index[rows]]]
    assert len(cross) > 300
    got, want = om.match_direct(abi, cams, ref, cur, d), om.ref_match_direct(abi, cams, ref, cur, d)
    _assert_match(got, want, fleet, rows)
    assert want.success[rows].mean() > 0.5 and (want.search_level[rows] == -1).any()


def test_with_one_camera_the_oracle_is_the_pinhole_and_the_atan_oracle(pkg, abi, synth, oracle, om):
    import oracle_atan_match

    oracle_atan_match.build()
    for cam in (synth.VGA, mc.atans(pkg, 1, sizes=((752, 480),))[0]):
        atan = mc.is_atan(cam)
        d = synth.make_match_batch(cam=synth.Camera(cam.width, cam.height, cam.fx_, cam.fy_, cam.cx_, cam.cy_) if atan else cam, n=900,
                                   n_pyr_levels=4, seed=9850, atan=cam if atan else None)
        ref, cur = np.zeros(d.T_ref_w.shape[0], np.int32), np.zeros(d.T_cur_w.shape[0], np.int32)
        got = om.match_direct(abi, [cam], ref, cur, d)
        want = oracle_atan_match.match_direct(abi, cam, d) if atan else oracle.match_direct(abi, d)
        _assert_match(got, want, "ATAN" if atan else "pinhole", np.arange(d.n))
        A = np.where(np.isnan(got.A_cur_ref), 0.0, got.A_cur_ref)
        _assert_match(om.match_direct_given_A(abi, [cam], ref, cur, d, A), oracle_atan_match.match_direct_given_A(abi, d, A), "given A",
                      np.arange(d.n))


def test_match_camera_layout_matches_the_header(abi, tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "plsvo_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %d %d\\n", sizeof(plsvo_match_camera), offsetof(plsvo_match_camera, reserved),'
                   ' offsetof(plsvo_match_camera, pinhole), offsetof(plsvo_match_camera, atan), PLSVO_CAMERA_PINHOLE, PLSVO_CAMERA_ATAN);\n'
                   "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    M = abi.MatchCamera
    assert got == [ctypes.sizeof(M), M.reserved.offset, M.pinhole.offset, M.atan.offset, abi.CAMERA_PINHOLE, abi.CAMERA_ATAN]



def test_findmatchdirect_argument_errors(pkg, synth):
    cams = mc.off_centre_mix(pkg, synth)
    ref, cur = mc.images(3, 1)
    d, _, _ = synth.make_match_multicam_batch(cams, ref, cur, n=20, n_pyr_levels=3, seed=9900)
    m = pkg.Matcher(10, ctx=object())  # every error below is raised before the library is reached
    err = pkg.api.PlsvoError
    for kw, msg in [(dict(camera=cams, cam_of_ref=ref), "cam_of_cur"), (dict(camera=cams, cam_of_cur=cur), "cam_of_ref"),
                    (dict(camera=cams[1], cam_of_ref=ref, cam_of_cur=cur), "sequence"), (dict(cam_of_ref=ref, cam_of_cur=cur), "sequence"),
                    (dict(camera=[], cam_of_ref=ref, cam_of_cur=cur), "empty"),
                    (dict(camera=cams[:2] + ["VGA"], cam_of_ref=ref, cam_of_cur=cur), "camera[2]"),
                    (dict(camera=cams, cam_of_ref=ref[:2], cam_of_cur=cur), "cam_of_ref must be integers of shape [3]"),
                    (dict(camera=cams, cam_of_ref=ref, cam_of_cur=cur.astype(np.float64)), "cam_of_cur must be integers"),
                    (dict(camera=tuple(cams), cam_of_ref=ref, cam_of_cur=np.stack([cur, cur])), "cam_of_cur must be integers")]:
        with pytest.raises(err, match=msg.replace("[", r"\[").replace("]", r"\]")):
            m.findMatchDirect(d, **kw)
    with pytest.raises(TypeError):  # the one-camera form is unchanged
        m.findMatchDirect(d, camera=synth.VGA)
