"""Host-pipeline scenarios of the ATAN findMatchDirect entry point (plsvo_match_direct_atan_batch_run), run by
tests/test_atan_match_host_cpu.py in a subprocess with PLSVO_LIB pointing at libplsvo_hostmodel.so, like scenarios.py,
whose helpers they use.  TEST INFRASTRUCTURE ONLY — see fake_cuda.h.  `python atan_match_scenarios.py` prints one JSON
object {scenario: "ok" | error text}."""
from __future__ import annotations

import ctypes as C
import json
import os
import sys
import traceback

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from scenarios import abi, check, clean, lib, make_batch, pkg, run, synth  # noqa: E402


def s_atan_match_rejected_cameras_leave_nothing_in_flight():
    """plsvo_match_direct_atan_batch_run: a camera whose size differs from the batch's, a non-finite parameter, fx <= 0 or
    fy <= 0 is refused before anything is queued (no copy of the caller's arrays, no kernel, the outputs untouched), and
    the context works afterwards.  An accepted call then shows the model kernel (fake_atan_match.cpp) in-bounds buffers
    for everything it reads and the distortion terms vk::ATANCamera derives from d0."""
    d = synth.make_match_batch(cam=synth.QVGA, n=40, seed=120, n_pyr_levels=3)
    d.n_iter = 10
    ctx = pkg.api.Context(0)
    b, keep = abi.make_match_batch(d)
    w, h = synth.QVGA.width, synth.QVGA.height
    good = (w, h, 210.0 / w, 210.0 / h, 160.0 / w, 120.0 / h, 0.93)
    bads = [((w + 2,) + good[1:], b"size differs"), (good[:2] + (float("nan"),) + good[3:], b"non-finite"),
            (good[:6] + (float("-inf"),), b"non-finite"), (good[:2] + (0.0,) + good[3:], b"positive"), (good[:3] + (-2.0,) + good[4:], b"positive")]
    for args, msg in bads:
        out = abi.MatchOut(d.n)
        out.A_cur_ref[:] = 7.0
        before = lib.fake_cuda_h2d_bytes()
        rc = ctx.lib.plsvo_match_direct_atan_batch_run(ctx.handle, C.byref(abi.AtanCamera(*args)), C.byref(b), C.byref(out.struct))
        assert rc == abi.ERR_INVALID, (args, rc)
        assert msg in ctx.lib.plsvo_last_error(ctx.handle), ctx.lib.plsvo_last_error(ctx.handle)
        assert lib.fake_cuda_h2d_bytes() == before, "a refused camera queued copies"
        assert lib.fake_cuda_pending_ops() == 0 and lib.fake_cuda_pending_host_reads() == 0
        assert (out.A_cur_ref == 7.0).all() and not out.success.any()
    for cam in (good, good[:6] + (0.0,)):  # with and without distortion
        out = abi.MatchOut(d.n)
        out.A_cur_ref[:] = 7.0
        rc = ctx.lib.plsvo_match_direct_atan_batch_run(ctx.handle, C.byref(abi.AtanCamera(*cam)), C.byref(b), C.byref(out.struct))
        assert rc == abi.OK, (rc, ctx.lib.plsvo_last_error(ctx.handle))
        clean()
        assert (out.px_cur == d.px_cur).all() and not out.success.any() and (out.search_level == -1).all()
        assert (out.A_cur_ref == 7.0).all(), "A_cur_ref must come back as the caller passed it where the kernel leaves it"
    ok = make_batch(6, 10, 3, 121)  # the context is still usable
    check(run(ok, ctx=ctx), ok, "after the refused cameras")


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
