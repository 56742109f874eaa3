"""Frame chains (PLSVO_ALIGN_FRAME_CHAIN, include/plsvo_b200.h): a batch that replays one camera sequence — pair b =
(frame b, frame b+1), as FrameHandlerMono aligns them (src/frame_handler_mono.cpp:176,272) — ships ONE stack of B+1 frames
instead of a reference stack and a current stack.  The kernel is the same; only the upload differs, so every output must be
bit-identical to the two-stack form of the same batch on every host path (small-batch block, plain copies, repack of padded
layouts, arrival-gated stream, levels derived on the device), and parity with the oracle follows.
"""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FIELDS = ("T_cur_w", "n_tracked", "H", "seg_killed", "iters", "status", "patch_iters", "patch_levels")


def _chain(synth, data, levels=None):
    one = copy.copy(data)
    one.frame_pyr = synth.chain_frames(data, levels)
    return one


def _same(a, b):
    for f in FIELDS:
        np.testing.assert_array_equal(getattr(a, f), getattr(b, f), err_msg=f)


def test_frame_chain_small_batch_matches_two_stacks_and_the_oracle(pkg, abi, synth, oracle, gen_device):
    data = synth.make_chain_batch(batch=12, n_pts=300, n_segs=80, device=gen_device, seed=5200)
    al = pkg.SparseImgAlign(4, 2, 30)
    two = al.run(data)
    one = al.run(_chain(synth, data))
    _same(two, one)
    ref = oracle.align(abi, data, abi.align_params(4, 2, 30), n_threads=8)
    ang, rel = synth.pose_error(one.T_cur_w, ref.T_cur_w)
    assert ang.max() <= 1e-5 and rel.max() <= 1e-4
    np.testing.assert_array_equal(one.iters, ref.iters)
    np.testing.assert_array_equal(one.n_tracked, ref.n_tracked)
    # the alignment does its job on the chain: every pair ends close to the ground-truth motion
    ang, rel = synth.pose_error(one.T_cur_w, data.T_cur_w_gt)
    assert np.median(ang) < 2e-3


def test_frame_chain_three_leg_api(pkg, synth, gen_device):
    data = synth.make_chain_batch(batch=9, n_pts=150, n_segs=30, device=gen_device, seed=5210)
    al = pkg.SparseImgAlign(4, 2, 30)
    two = al.run(data)
    al.upload(_chain(synth, data))
    al.launch()
    one = al.download()
    _same(two, one)
    al.launch()  # device-resident relaunch reads the same stack again
    _same(two, al.download())


@pytest.mark.parametrize("no_small_upload", [None, "1"])
def test_frame_chain_small_block_and_plain_copies(pkg, synth, gen_device, monkeypatch, no_small_upload):
    """The small-batch staging block, and plain per-array copies with the block disabled."""
    data = synth.make_chain_batch(batch=26, n_pts=120, n_segs=24, device=gen_device, seed=5220)
    if no_small_upload:
        monkeypatch.setenv("PLSVO_NO_SMALL_UPLOAD", no_small_upload)
    al = pkg.SparseImgAlign(4, 2, 30)
    _same(al.run(data), al.run(_chain(synth, data)))


def test_frame_chain_levels_derived_on_the_device(pkg, synth, gen_device, monkeypatch):
    """Only the finest level is shipped; levels 3 and 4 of the B+1 frames come from the pyramid kernel."""
    data = synth.make_chain_batch(batch=20, n_pts=120, n_segs=24, device=gen_device, seed=5230)
    al = pkg.SparseImgAlign(4, 2, 30)
    full = al.run(data)
    _same(full, al.run(_chain(synth, data, levels=[2])))
    monkeypatch.setenv("PLSVO_NO_SMALL_UPLOAD", "1")
    _same(full, al.run(_chain(synth, data, levels=[2])))


@pytest.mark.parametrize("layout", ["row_padded", "frame_padded"])
def test_frame_chain_padded_host_layouts(pkg, synth, gen_device, monkeypatch, layout):
    """Host stacks whose rows / frames are padded take the repack path (one linear copy + device-side 2-D repack, or one
    2-D copy per frame)."""
    data = synth.make_chain_batch(batch=10, n_pts=100, n_segs=20, device=gen_device, seed=5240)
    two = pkg.SparseImgAlign(4, 2, 30).run(data)
    one = _chain(synth, data)
    for l, f in list(one.frame_pyr.items()):
        n, h, w = f.shape
        if layout == "row_padded":
            big = np.full((n, h, w + 3), 255, np.uint8)
            big[:, :, :w] = f
            one.frame_pyr[l] = big[:, :, :w]
        else:
            big = np.full((n, h + 1, w), 255, np.uint8)
            big[:, :h, :] = f
            one.frame_pyr[l] = big[:, :h, :]
        assert not one.frame_pyr[l].flags["C_CONTIGUOUS"]
    _same(two, pkg.SparseImgAlign(4, 2, 30).run(one))


@pytest.mark.parametrize("gate_chunk", [None, "128"])
def test_frame_chain_arrival_gated_stream(pkg, synth, gen_device, monkeypatch, gate_chunk):
    """Default host path for >= 256 pairs: the copy stream sends frames (b0, b1] of every chunk, the persistent kernel
    takes a pair once frame b+1 has landed and halfSamples both of its frames; the neighbour pair forms the same bytes."""
    data = synth.make_chain_batch(batch=300, n_pts=64, n_segs=12, device=gen_device, seed=5250)
    monkeypatch.setenv("PLSVO_VARIANT", "128,4")  # same CTA shape on every path: bitwise comparison
    al = pkg.SparseImgAlign(4, 2, 30)
    al.upload(data)  # the plain upload -> launch -> download sequence
    al.launch()
    plain = al.download()
    if gate_chunk:
        monkeypatch.setenv("PLSVO_GATE_CHUNK", gate_chunk)
    al = pkg.SparseImgAlign(4, 2, 30)
    for levels in (None, [2]):
        one = _chain(synth, data, levels)
        for _ in range(3):
            _same(plain, al.run(one))


def test_frame_chain_rejects_unknown_flags(pkg, abi, synth, gen_device):
    import ctypes as C

    data = synth.make_chain_batch(batch=2, n_pts=20, n_segs=4, device=gen_device, seed=5260)
    batch, keep = abi.make_align_batch(data)
    batch.flags = 6
    ctx = pkg.default_context()
    rc = ctx.lib.plsvo_align_upload(ctx.handle, C.byref(batch))
    assert rc == abi.ERR_INVALID
    assert b"flags" in ctx.lib.plsvo_last_error(ctx.handle)
