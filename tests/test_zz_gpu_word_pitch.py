"""Lean level shipping for image widths whose finest shipped level is word aligned but not 16-byte aligned (752-pixel-wide
cameras: level 2 has 188-byte rows).  The host layout of such a level is kept on the device, the pyramid kernel cannot read
it (16-byte row loads), so the coarser levels are halfSampled by the alignment kernel itself, pair by pair — the code the
arrival-gated stream uses, here on the small-batch staging block and the plain per-array copies
(tests/test_host_pipeline_cpu.py covers its host side without a GPU)."""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FIELDS = ("T_cur_w", "n_tracked", "H", "seg_killed", "iters", "status", "patch_iters", "patch_levels")


@pytest.mark.parametrize("no_small_upload", [None, "1"])
def test_levels_derived_from_a_word_aligned_level(pkg, abi, synth, oracle, gen_device, monkeypatch, no_small_upload):
    cam = synth.Camera(752, 480, 460.0, 460.0, 375.5, 239.5)
    data = synth.make_align_batch(cam=cam, batch=7, n_pts=120, n_segs=24, device=gen_device, seed=5300)
    assert data.ref_pyr[2].shape[2] == 188 and data.ref_pyr[4].shape[2] == 47
    if no_small_upload:  # None: the small-batch staging block
        monkeypatch.setenv("PLSVO_NO_SMALL_UPLOAD", no_small_upload)
    al = pkg.SparseImgAlign(4, 2, 30)
    full = al.run(data)
    lean = copy.copy(data)
    lean.ref_pyr, lean.cur_pyr = {2: data.ref_pyr[2]}, {2: data.cur_pyr[2]}
    out = al.run(lean)
    for f in FIELDS:
        np.testing.assert_array_equal(getattr(out, f), getattr(full, f), err_msg=f)
    ref = oracle.align(abi, data, abi.align_params(4, 2, 30), n_threads=8)
    ang, rel = synth.pose_error(out.T_cur_w, ref.T_cur_w)
    assert ang.max() <= 1e-5 and rel.max() <= 1e-4
    np.testing.assert_array_equal(out.iters, ref.iters)
    np.testing.assert_array_equal(out.n_tracked, ref.n_tracked)
