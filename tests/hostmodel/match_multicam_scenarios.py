"""Host-pipeline scenarios of the per-image-camera findMatchDirect entry point (plsvo_match_direct_multicam_batch_run),
run by tests/test_match_multicam_host_cpu.py in a subprocess with PLSVO_LIB pointing at the model library of
match_multicam_model.py, like scenarios.py, whose helpers they use.  TEST INFRASTRUCTURE ONLY — see fake_cuda.h.
`python match_multicam_scenarios.py` prints one JSON object {scenario: "ok" | error text}."""
from __future__ import annotations

import ctypes as C
import json
import os
import sys
import traceback

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from scenarios import abi, check, clean, lib, make_batch, pkg, run, synth  # noqa: E402

I32 = C.POINTER(C.c_int32)


def _fleet():
    """A QVGA pinhole, a 200x150 ATAN camera and a 280x240 pinhole in a 320x240 slot; two keyframes and three current
    frames, the last current frame seen through the smallest camera."""
    cams = [synth.Camera(320, 240, 210.0, 208.0, 159.5, 119.5), pkg.ATANCamera(200, 150, 0.9, 1.1, 0.5, 0.5, 0.93),
            synth.Camera(280, 240, 190.0, 190.0, 140.0, 118.0)]
    return cams, np.array([0, 2], np.int32), np.array([2, 0, 1], np.int32)


def _call(ctx, cams, n_cams, ref, cur, b, out):
    return ctx.lib.plsvo_match_direct_multicam_batch_run(ctx.handle, cams, n_cams, ref, cur, C.byref(b), C.byref(out.struct))


def s_match_multicam_rejections_leave_nothing_in_flight():
    """Every malformed camera table is refused before anything is queued (no copy of the caller's arrays, no kernel, the
    outputs untouched), with the index in the message, and the context works afterwards."""
    cams, ref, cur = _fleet()
    d, _, _ = synth.make_match_multicam_batch(cams, ref, cur, n=40, n_pyr_levels=3, seed=130)
    d.n_iter = 10
    ctx = pkg.api.Context(0)
    b, keep = abi.make_match_batch(d)
    good = abi.make_match_cameras(cams)
    p_ref, p_cur = ref.ctypes.data_as(I32), cur.ctypes.data_as(I32)

    def table(k, **kw):
        t = abi.make_match_cameras(cams)
        part = kw.pop("part")
        for f, v in kw.items():
            setattr(getattr(t[k], part) if part else t[k], f, v)
        return t

    bad_ref = np.array([0, 3], np.int32)
    bad_cur = np.array([2, -1, 1], np.int32)
    cases = [
        ((None, 3, p_ref, p_cur), b"NULL"), ((good, 3, None, p_cur), b"NULL"), ((good, 3, p_ref, None), b"NULL"),
        ((good, 0, p_ref, p_cur), b"n_cams"), ((good, 3, bad_ref.ctypes.data_as(I32), p_cur), b"cam_of_ref[1]"),
        ((good, 3, p_ref, bad_cur.ctypes.data_as(I32)), b"cam_of_cur[1]"),
        ((good, 2, p_ref, p_cur), b"cam_of_ref[1]"),
        ((table(1, part=None, model=7), 3, p_ref, p_cur), b"cams[1].model"),
        ((table(0, part="pinhole", fx=float("nan")), 3, p_ref, p_cur), b"cams[0] has a non-finite"),
        ((table(2, part="pinhole", fy=0.0), 3, p_ref, p_cur), b"cams[2].fx and fy"),
        ((table(1, part="atan", d0=float("inf")), 3, p_ref, p_cur), b"cams[1] (ATAN) has a non-finite"),
        ((table(1, part="atan", fx=-1.0), 3, p_ref, p_cur), b"cams[1] (ATAN) fx and fy"),
        ((table(2, part="pinhole", width=321), 3, p_ref, p_cur), b"cams[2] is 321x240"),
        ((table(1, part="atan", height=241), 3, p_ref, p_cur), b"cams[1] is 200x241"),
        ((table(1, part="atan", width=3), 3, p_ref, p_cur), b"cams[1] (current image 2)"),  # 3 >> 2 == 0 at the top level
    ]
    for (tab, n_cams, r, c), msg in cases:
        out = abi.MatchOut(d.n)
        out.A_cur_ref[:] = 7.0
        before = lib.fake_cuda_h2d_bytes()
        rc = _call(ctx, tab, n_cams, r, c, b, out)
        assert rc == abi.ERR_INVALID, (msg, rc)
        assert msg in ctx.lib.plsvo_last_error(ctx.handle), (msg, ctx.lib.plsvo_last_error(ctx.handle))
        assert lib.fake_cuda_h2d_bytes() == before, "a refused call queued copies"
        assert lib.fake_cuda_pending_ops() == 0 and lib.fake_cuda_pending_host_reads() == 0
        assert (out.A_cur_ref == 7.0).all() and not out.success.any()
    # a ref image's camera below one pixel at a candidate's level: a 6x6 keyframe camera asked at level 3
    tiny = cams[:2] + [synth.Camera(6, 6, 5.0, 5.0, 3.0, 3.0)]
    d4 = synth.make_match_multicam_batch(cams, ref, np.array([0, 0, 1], np.int32), n=40, n_pyr_levels=4, seed=132)[0]
    d4.n_iter = 10
    d4.ref_level[np.flatnonzero(ref[d4.ref_index] == 2)[0]] = 3
    b4, keep4 = abi.make_match_batch(d4)
    out = abi.MatchOut(d4.n)
    before = lib.fake_cuda_h2d_bytes()
    cur4 = np.array([0, 0, 1], np.int32)
    rc = _call(ctx, abi.make_match_cameras(tiny), 3, p_ref, cur4.ctypes.data_as(I32), b4, out)
    assert rc == abi.ERR_INVALID and b"cams[2] (ref image 1" in ctx.lib.plsvo_last_error(ctx.handle), ctx.lib.plsvo_last_error(ctx.handle)
    assert lib.fake_cuda_h2d_bytes() == before
    ok = make_batch(6, 10, 3, 133)  # the context is still usable
    check(run(ok, ctx=ctx), ok, "after the refused calls")


def s_match_multicam_accepted_call_reads_only_inside_each_camera():
    """An accepted call with pinhole and ATAN cameras of three sizes shows the model kernel (fake_match_multicam.cpp)
    in-bounds buffers for everything it reads — each image only inside its camera's region, the camera table and both
    index arrays — and records with the terms their models derive.  Then the context still works."""
    cams, ref, cur = _fleet()
    d, _, _ = synth.make_match_multicam_batch(cams, ref, cur, n=60, n_pyr_levels=3, seed=134)
    assert (d.cur_index == len(cur) - 1).any(), "a candidate must read the last current frame's camera index"
    d.n_iter = 10
    ctx = pkg.api.Context(0)
    out = pkg.Matcher(10, ctx=ctx).findMatchDirect(d, camera=cams, cam_of_ref=ref, cam_of_cur=cur)
    clean()
    assert (out.px_cur == d.px_cur).all() and not out.success.any() and (out.search_level == -1).all()
    ok = make_batch(6, 10, 3, 136)
    check(run(ok, ctx=ctx), ok, "after the per-image match call")


SCENARIOS = {k[2:]: v for k, v in list(globals().items()) if k.startswith("s_") and callable(v)}


def main(names):
    res = {}
    for name in names or SCENARIOS:
        try:
            lib.fake_cuda_clear_errors()
            SCENARIOS[name]()
            res[name] = "ok"
        except Exception:
            res[name] = traceback.format_exc(limit=6)
            lib.fake_cuda_drop_pending()
    print("RESULT " + json.dumps(res), flush=True)
    lib.fake_cuda_drop_pending()


if __name__ == "__main__":
    main(sys.argv[1:])
