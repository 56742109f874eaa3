"""Scenarios of the host-pipeline model (run by tests/test_host_pipeline_cpu.py in a subprocess with PLSVO_LIB pointing at
libplsvo_hostmodel.so).  TEST INFRASTRUCTURE ONLY — see fake_cuda.h.

Every scenario drives the product's unchanged Python mirror (plsvo_b200.SparseImgAlign, api.track, ...) through the
product's unchanged host code; the model kernels return digests of the bytes they were given, which are compared with
the same digests computed here, in NumPy, from the caller's arrays.  `python scenarios.py` prints one JSON object
{scenario: "ok" | error text}."""
from __future__ import annotations

import contextlib
import copy
import ctypes as C
import json
import os
import sys
import traceback

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import plsvo_b200 as pkg  # noqa: E402
from plsvo_b200 import abi, synth  # noqa: E402

M64 = (1 << 64) - 1
K = 0x9E3779B97F4A7C15
LEVELS = (2, 3, 4)

lib = abi.load_library()
for _n, _r in (("fake_cuda_errors", C.c_char_p), ("fake_cuda_pending_host_reads", C.c_int), ("fake_cuda_pending_ops", C.c_int),
               ("fake_cuda_h2d_bytes", C.c_ulonglong), ("fake_cuda_live_blocks", C.c_int)):
    getattr(lib, _n).restype = _r


# ---- the digest of fake_kernels.cpp, restated ----
def dig_bytes(a) -> int:
    b = np.frombuffer(np.ascontiguousarray(a).tobytes(), np.uint8).astype(np.uint64)
    idx = (np.arange(b.size, dtype=np.uint64) + np.uint64(1)) * np.uint64(K)
    with np.errstate(over="ignore"):
        return int(((b + np.uint64(1)) * idx).sum(dtype=np.uint64))


def mix(h: int, v: int) -> int:
    return (h ^ ((v + K + ((h << 6) & M64) + (h >> 2)) & M64)) & M64


def dig_array(h: int, arr, b: int, count: int) -> int:
    if arr is None or arr.shape[1] == 0:  # not shipped (an empty array is not shipped either)
        return mix(h, 0x5151)
    return mix(h, dig_bytes(arr[b][:count]))


def expected(data):
    """(n_tracked digests [B] as int64, per-level digests [B, 2*levels]) for the batch as the kernel must see it."""
    B = data.batch
    out = np.zeros(B, np.uint64)
    levels = range(data.min_level, data.max_level + 1)
    lvl = np.zeros((B, 2 * len(levels)), np.float64)
    for b in range(B):
        h = 0
        for k, l in enumerate(levels):
            hr, hc = dig_bytes(data.ref_pyr[l][b]), dig_bytes(data.cur_pyr[l][b])
            h = mix(mix(h, hr), hc)
            lvl[b, 2 * k], lvl[b, 2 * k + 1] = float(hr >> 12), float(hc >> 12)
        npt = int(data.pt_count[b]) if data.pt_count is not None else data.n_pts
        nsg = int(data.seg_count[b]) if data.seg_count is not None else data.n_segs
        h = mix(h, dig_bytes(data.T_ref_w[b]))
        h = mix(h, dig_bytes(data.T_cur_w[b]))
        h = mix(h, npt * 65536 + nsg)
        for name in ("pt_px", "pt_f", "pt_pos", "pt_depth", "pt_valid"):
            h = dig_array(h, getattr(data, name, None), b, npt)
        if data.n_segs > 0:
            for name in ("seg_spx", "seg_epx", "seg_sf", "seg_ef", "seg_spos", "seg_epos", "seg_sdepth", "seg_edepth", "seg_length", "seg_valid"):
                h = dig_array(h, getattr(data, name, None), b, nsg)
        else:
            for _ in range(10):
                h = mix(h, 0x5151)
        out[b] = (h >> 1) | 1
    return out.view(np.int64), lvl


# ---- inputs: random bytes are as good as rendered scenes for a kernel that only digests them ----
def half(img):
    a = img.astype(np.int32)
    return ((a[:, 0::2, 0::2] + a[:, 0::2, 1::2] + a[:, 1::2, 0::2] + a[:, 1::2, 1::2]) >> 2).astype(np.uint8)


def pyramid(rng, n, cam, min_level=2, max_level=4):
    pyr = {min_level: rng.integers(0, 256, (n, cam.height >> min_level, cam.width >> min_level), dtype=np.uint8)}
    for l in range(min_level + 1, max_level + 1):
        pyr[l] = half(pyr[l - 1])
    return pyr


def make_batch(B, n_pts, n_segs, seed, cam=synth.VGA, chain=False, ragged=False, masks=False, min_level=2, max_level=4):
    rng = np.random.default_rng(seed)
    if chain:
        frames = pyramid(rng, B + 1, cam, min_level, max_level)
        ref = {l: np.ascontiguousarray(f[:-1]) for l, f in frames.items()}
        cur = {l: np.ascontiguousarray(f[1:]) for l, f in frames.items()}
    else:
        ref, cur = pyramid(rng, B, cam, min_level, max_level), pyramid(rng, B, cam, min_level, max_level)

    def r(*shape):
        return rng.standard_normal(shape)

    spx = rng.uniform(64, 400, (B, n_segs, 2))
    epx = spx + rng.uniform(-120, 120, (B, n_segs, 2))
    d = synth.AlignData(cam=cam, max_level=max_level, min_level=min_level, ref_pyr=ref, cur_pyr=cur, T_ref_w=r(B, 7), T_cur_w=r(B, 7), T_cur_w_gt=r(B, 7),
                        pt_px=rng.uniform(64, 400, (B, n_pts, 2)), pt_f=r(B, n_pts, 3), pt_pos=r(B, n_pts, 3), seg_spx=spx, seg_epx=epx,
                        seg_sf=r(B, n_segs, 3), seg_ef=r(B, n_segs, 3), seg_spos=r(B, n_segs, 3), seg_epos=r(B, n_segs, 3),
                        seg_length=np.linalg.norm(epx - spx, axis=-1))
    if ragged:
        d.pt_count = rng.integers(0, n_pts + 1, B).astype(np.int32)
        d.seg_count = rng.integers(0, n_segs + 1, B).astype(np.int32)
        d.pt_count[0], d.seg_count[0] = 0, 0  # the reference's early-out pair
    if masks:
        d.pt_valid = rng.integers(0, 2, (B, n_pts)).astype(np.uint8)
        d.seg_valid = rng.integers(0, 2, (B, n_segs)).astype(np.uint8)
    return d


def one_stack(data, levels=LEVELS):
    """The frame-chain form of a chain batch (PLSVO_ALIGN_FRAME_CHAIN): one stack of B+1 frames per shipped level."""
    o = copy.copy(data)
    o.frame_pyr = synth.chain_frames(data, list(levels))
    return o


def shipped(data, levels):
    """Same batch with only `levels` shipped (the rest is derived on the device)."""
    o = copy.copy(data)
    o.ref_pyr = {l: data.ref_pyr[l] for l in levels}
    o.cur_pyr = {l: data.cur_pyr[l] for l in levels}
    return o


def lean_features(data, rng):
    """Depth-only features without bearings (what bench.py's end-to-end leg ships)."""
    o = copy.copy(data)
    o.pt_depth = rng.uniform(1, 3, data.pt_px.shape[:2])
    o.seg_sdepth = rng.uniform(1, 3, data.seg_spx.shape[:2])
    o.seg_edepth = rng.uniform(1, 3, data.seg_spx.shape[:2])
    o.pt_pos = o.seg_spos = o.seg_epos = None
    o.pt_f = o.seg_sf = o.seg_ef = None
    return o


@contextlib.contextmanager
def env(**kw):
    old = {k: os.environ.get(k) for k in kw}
    for k, v in kw.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = str(v)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def clean():
    err = lib.fake_cuda_errors()
    assert not err, "model runtime recorded: " + err.decode()
    assert lib.fake_cuda_pending_host_reads() == 0, "host->device copies still queued after the call returned"


def check(out, data_as_kernel_sees_it, what=""):
    clean()
    want, lvl = expected(data_as_kernel_sees_it)
    got_lvl = out.H[:, : lvl.shape[1]]
    bad = np.nonzero(got_lvl != lvl)
    assert bad[0].size == 0, f"{what}: image level digests differ at (pair, 2*level_index+ref/cur) {list(zip(*bad))[:6]}"
    assert np.array_equal(out.n_tracked, want), f"{what}: pair digests differ at {np.nonzero(out.n_tracked != want)[0][:8]}"
    assert np.array_equal(out.T_cur_w, data_as_kernel_sees_it.T_cur_w), what
    npt = data_as_kernel_sees_it.pt_count if data_as_kernel_sees_it.pt_count is not None else data_as_kernel_sees_it.n_pts
    assert np.array_equal(out.patch_iters, np.broadcast_to(npt, out.patch_iters.shape)), what


def run(data, ctx=None, three_leg=False, **envs):
    """One plsvo_align_batch_run call, or (three_leg) the plsvo_align_upload / _launch / _download sequence."""
    with env(**envs):
        al = pkg.SparseImgAlign(data.max_level, data.min_level, 30, ctx=ctx or pkg.api.Context(0))
        if not three_leg:
            return al.run(data)
        al.upload(data)
        al.launch()
        return al.download()


# ---- scenarios ----
def s_plain_upload_launch_download():
    d = make_batch(5, 40, 9, 1)
    check(run(d, PLSVO_NO_SMALL_UPLOAD=1), d, "plain")
    d = make_batch(6, 33, 0, 2)  # no segments at all
    check(run(d, PLSVO_NO_SMALL_UPLOAD=1), d, "points only")


def s_small_batch_staging_block():
    for B in (1, 3, 12):
        d = make_batch(B, 40, 9, 10 + B, ragged=B > 1, masks=True)
        check(run(d), d, f"small B={B}")
    ctx = pkg.api.Context(0)  # staging block reused by consecutive calls of different sizes
    for B in (2, 9, 1, 9):
        d = make_batch(B, 25, 6, 20 + B)
        check(run(d, ctx=ctx), d, f"small, reused context B={B}")


def s_staging_block_grows_while_a_copy_is_queued():
    """upload() does not synchronise: a second, bigger upload must not free or refill the pinned staging block while the
    first upload's copy out of it is still queued (alignment and pose-optimiser uploads share the block)."""
    ctx = pkg.api.Context(0)
    al = pkg.SparseImgAlign(4, 2, 30, ctx=ctx)
    small, big = make_batch(1, 10, 2, 130), make_batch(14, 60, 12, 131)
    al.upload(small)
    al.upload(big)
    al.launch()
    check(al.download(), big, "second upload")
    al.upload(small)
    po = synth.make_poseopt_batch(batch=64, n_pts=60, n_segs=12, seed=132)
    out = pkg.pose_optimizer.optimizeGaussNewton(2.0, 10, False, po, ctx=ctx)  # refills (and grows) the shared block
    assert np.array_equal(out.T_f_w, po.T_f_w)
    al.launch()
    check(al.download(), small, "alignment upload before a pose-optimiser call")


def s_three_leg_api_and_relaunch():
    d = make_batch(7, 30, 8, 30)
    al = pkg.SparseImgAlign(4, 2, 30, ctx=pkg.api.Context(0))
    al.upload(d)
    al.launch()
    check(al.download(), d, "three-leg")
    al.launch()
    check(al.download(), d, "relaunch")
    d2 = shipped(d, [2])
    al.upload(d2)
    al.launch()
    check(al.download(), d, "three-leg, derived levels")
    al.launch()
    check(al.download(), d, "relaunch, derived levels")


def s_arrival_gated_stream():
    d = make_batch(300, 24, 6, 50, ragged=True)
    full_bytes = None
    for envs in ({}, {"PLSVO_GATE_CHUNK": 128}):
        h0 = lib.fake_cuda_h2d_bytes()
        check(run(d, **envs), d, f"gated {envs}")
        n_chunks = -(-d.batch // int(envs.get("PLSVO_GATE_CHUNK", 256)))
        moved = lib.fake_cuda_h2d_bytes() - h0 - 4 * n_chunks  # one 4-byte arrival flag per chunk
        full_bytes = full_bytes or moved
        assert moved == full_bytes, f"gated {envs}: {moved} bytes moved, {full_bytes} in the default configuration"
        check(run(shipped(d, [2]), **envs), d, f"gated, levels derived in the kernel {envs}")
    ctx = pkg.api.Context(0)  # consecutive calls on one context: buffers, flags and events are reused
    for seed in (51, 52):
        d = make_batch(257 + seed, 16, 4, seed)
        check(run(d, ctx=ctx, PLSVO_GATE_CHUNK=128), d, f"gated, reused context seed={seed}")
        check(run(make_batch(3, 16, 4, seed + 100), ctx=ctx), make_batch(3, 16, 4, seed + 100), "small call in between")


def s_padded_host_layouts():
    d = make_batch(10, 30, 8, 60)
    for layout in ("row_padded", "frame_padded", "both"):
        p = copy.copy(d)
        p.ref_pyr, p.cur_pyr = {}, {}
        for l in LEVELS:
            for src, dst in ((d.ref_pyr, p.ref_pyr), (d.cur_pyr, p.cur_pyr)):
                n, h, w = src[l].shape
                big = np.full((n, h + (layout != "row_padded"), w + 3 * (layout != "frame_padded")), 255, np.uint8)
                big[:, :h, :w] = src[l]
                dst[l] = big[:, :h, :w]
        check(run(p), d, layout)
        check(run(p, PLSVO_NO_SMALL_UPLOAD=1), d, f"{layout}, plain copies")


def s_lean_features():
    d = lean_features(make_batch(9, 30, 8, 70), np.random.default_rng(71))
    check(run(d), d, "lean small")
    check(run(shipped(d, [2]), PLSVO_NO_SMALL_UPLOAD=1), d, "lean, derived levels")
    d = lean_features(make_batch(260, 20, 5, 72), np.random.default_rng(73))
    check(run(shipped(d, [2])), d, "lean gated (the end-to-end leg of bench.py)")


def s_chain_every_host_path():
    # small block / plain copies, all levels shipped or derived (the arrival-gated stream: s_chain_arrival_gated_stream)
    d = make_batch(26, 30, 8, 80, chain=True, ragged=True)
    for envs in ({}, {"PLSVO_NO_SMALL_UPLOAD": 1}):
        check(run(one_stack(d), **envs), d, f"chain {envs}")
        check(run(one_stack(d, [2]), **envs), d, f"chain, derived levels {envs}")
    d = make_batch(3, 30, 8, 81, chain=True)
    check(run(one_stack(d)), d, "chain B=3 small block")
    d1 = make_batch(1, 30, 8, 82, chain=True)
    check(run(one_stack(d1)), d1, "chain of one pair")
    # three-leg form and relaunch
    al = pkg.SparseImgAlign(4, 2, 30, ctx=pkg.api.Context(0))
    al.upload(one_stack(d, [2]))
    al.launch()
    check(al.download(), d, "chain three-leg")
    al.launch()
    check(al.download(), d, "chain relaunch")


def s_chain_arrival_gated_stream():
    d = make_batch(300, 24, 6, 90, chain=True)
    two_stack_bytes = None
    for envs in ({}, {"PLSVO_GATE_CHUNK": 128}):
        for levels in (LEVELS, (2,)):
            h0 = lib.fake_cuda_h2d_bytes()
            check(run(shipped(d, levels), **envs), d, f"two stacks {envs} {levels}")
            h1 = lib.fake_cuda_h2d_bytes()
            check(run(one_stack(d, levels), **envs), d, f"chain gated {envs} {levels}")
            h2 = lib.fake_cuda_h2d_bytes()
            frame_bytes = sum(d.ref_pyr[l][0].nbytes for l in levels)
            # every frame crosses the link once: B+1 frames instead of 2B (the arrival flags, 4 bytes per chunk, are the slack:
            # VGA level 4 is not a multiple of 128 bytes, so a chain that ships it takes the ungated path)
            saved = (h1 - h0) - (h2 - h1) - (d.batch - 1) * frame_bytes
            assert 0 <= saved <= 16, f"chain {envs} {levels}: bytes moved {h1 - h0} vs {h2 - h1}"
    ctx = pkg.api.Context(0)  # chain and two-stack calls alternate on one context (the bench does exactly this)
    for seed in (91, 92):
        d = make_batch(256 + seed, 16, 4, seed, chain=True)
        check(run(shipped(d, [2]), ctx=ctx), d, "two stacks, reused context")
        check(run(one_stack(d, [2]), ctx=ctx), d, "chain, reused context")
        check(run(one_stack(d), ctx=ctx), d, "chain with all levels shipped, reused context")


def s_chain_padded_host_layouts():
    d = make_batch(10, 30, 8, 100, chain=True)
    for layout in ("row_padded", "frame_padded"):
        o = one_stack(d)
        for l, f in list(o.frame_pyr.items()):
            n, h, w = f.shape
            big = np.full((n, h + (layout == "frame_padded"), w + 3 * (layout == "row_padded")), 255, np.uint8)
            big[:, :h, :w] = f
            o.frame_pyr[l] = big[:, :h, :w]
        check(run(o), d, f"chain {layout}")
    # a chain whose frames are not 128-byte multiples must leave the gated path (QVGA level 4: 20 x 15 bytes)
    q = make_batch(260, 12, 3, 101, cam=synth.QVGA, chain=True)
    check(run(one_stack(q)), q, "chain with unaligned frames")


def s_rejected_inputs_leave_nothing_in_flight():
    d = make_batch(4, 10, 3, 110, chain=True)
    batch, keep = abi.make_align_batch(one_stack(d))
    ctx = pkg.api.Context(0)
    batch.flags = 6
    assert ctx.lib.plsvo_align_upload(ctx.handle, C.byref(batch)) == abi.ERR_INVALID
    assert b"flags" in ctx.lib.plsvo_last_error(ctx.handle)
    big = make_batch(300, 10, 3, 111, ragged=True)
    big.pt_count[299] = 11  # beyond n_pts: found by the sizing pass, after the gated copies have been queued
    b2, keep2 = abi.make_align_batch(big)
    out = abi.AlignOut(300, 3)
    rc = ctx.lib.plsvo_align_batch_run(ctx.handle, C.byref(b2), C.byref(abi.align_params(4, 2, 30)), C.byref(out.struct))
    assert rc == abi.ERR_INVALID, rc
    assert lib.fake_cuda_pending_host_reads() == 0, "the caller's arrays may still be read after an error return"
    missing = shipped(make_batch(300, 10, 3, 112), [3, 4])  # finest level neither shipped nor derivable
    b3, keep3 = abi.make_align_batch(missing)
    rc = ctx.lib.plsvo_align_batch_run(ctx.handle, C.byref(b3), C.byref(abi.align_params(4, 2, 30)), C.byref(out.struct))
    assert rc != abi.OK
    assert lib.fake_cuda_pending_host_reads() == 0
    ok = make_batch(300, 10, 3, 113)  # the context is still usable
    check(run(ok, ctx=ctx), ok, "after rejected calls")


def s_forced_variant_is_the_only_one_tried():
    """PLSVO_VARIANT selects the one kernel variant a call may run: a batch that variant cannot plan fails and names it,
    while the default plan of the same batch falls back to a variant that fits."""
    ctx = pkg.api.Context(0)

    def fits(n_pts, variant):
        d = make_batch(1, n_pts, 0, 160)
        try:
            out = run(d, ctx=ctx, PLSVO_VARIANT=variant)
        except pkg.api.PlsvoError as ex:
            assert f"PLSVO_VARIANT={variant} cannot run this batch" in str(ex) and "shared-memory plan" in str(ex), str(ex)
            clean()
            return False
        check(out, d, f"{variant}, {n_pts} points")
        return True

    # <256,2> needs more shared memory per point list than <128,4> (per-thread chi2 terms, cross-warp partials): find the
    # smallest point count it cannot plan
    lo, hi = 1000, 8000
    assert fits(lo, "256,2") and not fits(hi, "128,4")
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if fits(mid, "256,2") else (lo, mid)
    assert fits(hi, "128,4"), f"{hi} points: <128,4> should still fit where <256,2> stops"
    d = make_batch(1, hi, 0, 161)
    check(run(d, ctx=ctx), d, f"default plan of one pair (<256,2> first), {hi} points")
    for bad, why in (("128,3", "not compiled"), ("128x4", "threads,ctas")):
        try:
            run(make_batch(1, 10, 2, 162), ctx=ctx, PLSVO_VARIANT=bad)
        except pkg.api.PlsvoError as ex:
            assert why in str(ex), str(ex)
        else:
            raise AssertionError(f"PLSVO_VARIANT={bad} was accepted")
    clean()


def poseopt_expected(po, T=None):
    B = po.batch
    want = np.zeros(B, np.uint64)
    for b in range(B):
        npt = int(po.pt_count[b]) if getattr(po, "pt_count", None) is not None else po.n_pts
        nsg = int(po.seg_count[b]) if getattr(po, "seg_count", None) is not None else po.n_segs
        h = mix(0, dig_bytes((po.T_f_w if T is None else T)[b]))
        h = mix(h, npt * 65536 + nsg)
        for name, cnt in (("pt_f", npt), ("pt_pos", npt), ("pt_level", npt), ("pt_valid", npt), ("seg_line", nsg), ("seg_spos", nsg),
                          ("seg_epos", nsg), ("seg_level", nsg), ("seg_valid", nsg)):
            h = dig_array(h, getattr(po, name, None), b, cnt)
        want[b] = (h >> 1) | 1
    return want.view(np.int64)


def s_pose_optimiser_host_paths():
    """plsvo_poseopt_batch_run: one packed pinned block for small batches (the reference's own call is one frame), one copy
    per array for large ones; outputs come back in one block."""
    ctx = pkg.api.Context(0)
    for B, n_pts, n_segs, envs in ((1, 300, 80, {}), (7, 40, 9, {}), (7, 40, 0, {}), (64, 300, 80, {"PLSVO_NO_SMALL_UPLOAD": 1}),
                                   (2048, 300, 80, {}), (3, 20, 5, {})):
        po = synth.make_poseopt_batch(batch=B, n_pts=n_pts, n_segs=n_segs, seed=140 + B)
        with env(**envs):
            out = pkg.pose_optimizer.optimizeGaussNewton(2.0, 10, False, po, ctx=ctx)
        clean()
        assert np.array_equal(out.num_obs_pt, poseopt_expected(po)), f"pose-opt digests B={B}"
        assert np.array_equal(out.T_f_w, po.T_f_w)
        assert not out.status.any()


def s_pyramid_call():
    """plsvo_pyramid_batch_run with contiguous and padded level-0 stacks; the model kernel is the real truncating 2x2 mean."""
    rng = np.random.default_rng(150)
    for (B, h, w) in ((3, 480, 640), (2, 90, 161), (1, 64, 64)):
        img = rng.integers(0, 256, (B, h, w), dtype=np.uint8)
        want = [img]
        for _ in range(4):
            a = want[-1][:, : want[-1].shape[1] // 2 * 2, : want[-1].shape[2] // 2 * 2]
            want.append(half(a))
        got = pkg.api.createImgPyramid(img, 5, ctx=pkg.api.Context(0))
        clean()
        for l in range(5):
            assert np.array_equal(got[l], want[l]), f"pyramid level {l} of a {h}x{w} stack"


def s_track_chained_call():
    """plsvo_track_batch_run: the pose optimiser starts from the aligned poses on the device (here: T_cur_w passed through)."""
    d = make_batch(20, 30, 8, 120)
    B, n_pts, n_segs = 20, 30, 8
    po = synth.make_poseopt_batch(batch=B, n_pts=n_pts, n_segs=n_segs, seed=122)
    ao, pout = pkg.api.track(d, po, ctx=pkg.api.Context(0))
    check(ao, d, "track: alignment leg")
    assert np.array_equal(pout.num_obs_pt, poseopt_expected(po, T=d.T_cur_w)), "track: pose-opt digests"
    assert np.array_equal(pout.T_f_w, d.T_cur_w)
    clean()


def padded_view(stack, layout, rng):
    """The same images inside a bigger allocation: rows and / or frames padded with bytes the kernel must never see."""
    n, h, w = stack.shape
    pad_r = int(rng.integers(1, 5)) if layout in ("row", "both") else 0
    pad_f = int(rng.integers(1, 3)) if layout in ("frame", "both") else 0
    big = np.full((n, h + pad_f, w + pad_r), 255, np.uint8)
    big[:, :h, :w] = stack
    return big[:, :h, :w]


def s_randomised_configurations():
    """Differential test over random corners of the configuration space: camera size, level range, which levels are shipped,
    batch size on either side of the streaming threshold, feature counts down to none, ragged counts, masks, lean features,
    frame chains, padded host layouts, the one-call and three-leg forms, and the environment switches of the host path."""
    rng = np.random.default_rng(int(os.environ.get("PLSVO_FUZZ_SEED", 2024)))  # PLSVO_FUZZ_SEED / _ITERS: longer hunts by hand
    cams = [synth.Camera(w, h, 0.7 * w, 0.7 * w, w / 2 - 0.5, h / 2 - 0.5) for w, h in ((128, 96), (256, 192), (384, 128), (640, 480))]
    ctx = pkg.api.Context(0)  # one context for everything: every call inherits the buffers of a differently shaped one
    for it in range(int(os.environ.get("PLSVO_FUZZ_ITERS", 70))):
        cam = cams[int(rng.integers(0, 3 if it % 4 else 4))]
        min_level = int(rng.integers(0, 3))
        max_level = min(4, min_level + int(rng.integers(0, 3)))
        B = int(rng.integers(256, 400)) if it % 5 == 0 else int(rng.integers(1, 40))
        n_pts, n_segs = int(rng.integers(0, 50)), int(rng.integers(0, 12))
        if B >= 256:
            n_pts, n_segs = min(n_pts, 12), min(n_segs, 4)
            if cam.width == 640:
                cam = cams[1]
        chain = bool(rng.integers(0, 2))
        d = make_batch(B, n_pts, n_segs, 5000 + it, cam=cam, chain=chain, ragged=bool(rng.integers(0, 2)), masks=bool(rng.integers(0, 2)),
                       min_level=min_level, max_level=max_level)
        seen = d
        if rng.integers(0, 3) == 0 and n_pts + n_segs > 0:
            seen = d = lean_features(d, rng)
        top = int(rng.integers(min_level, max_level + 1))  # levels min..top are shipped, the rest derived on the device
        levels = list(range(min_level, top + 1))
        call = one_stack(d, levels) if chain else shipped(d, levels)
        layout = ["dense", "dense", "row", "frame", "both"][int(rng.integers(0, 5))]
        if layout != "dense":
            if chain:
                call.frame_pyr = {l: padded_view(f, layout, rng) for l, f in call.frame_pyr.items()}
            else:
                seed_pad = int(rng.integers(0, 1 << 30))
                call.ref_pyr = {l: padded_view(f, layout, np.random.default_rng(seed_pad + l)) for l, f in call.ref_pyr.items()}
                call.cur_pyr = {l: padded_view(f, layout, np.random.default_rng(seed_pad + l)) for l, f in call.cur_pyr.items()}
        pick = int(rng.integers(0, 8))  # one call or three legs, with and without the small block, gate chunk 256 or 128
        three_leg = bool(pick & 1)
        envs = {**({"PLSVO_NO_SMALL_UPLOAD": 1} if pick & 2 else {}), **({"PLSVO_GATE_CHUNK": 128} if pick & 4 else {})}
        what = (f"#{it}: {cam.width}x{cam.height} levels {min_level}..{max_level} shipped {levels} B={B} pts={n_pts} segs={n_segs} chain={chain} "
                f"layout={layout} lean={seen is not d or hasattr(d, 'pt_depth') and d.pt_depth is not None} three_leg={three_leg} env={envs}")
        try:
            out = run(call, ctx=ctx, three_leg=three_leg, **envs)
        except pkg.api.PlsvoError as ex:
            raise AssertionError(f"{what}: {ex}") from None
        check(out, seen, what)


def s_bench_chain_leg():
    """bench.py's `e2e_chain` leg (chain_leg, lean_copy, subset) against the host model: the leg's own bookkeeping — lean
    inputs, the one-stack view, bytes per call — on a cheap stand-in for the rendered trajectory."""
    import time as _time
    import types

    import torch

    sys.path.insert(0, ROOT)
    import bench

    class Event:
        def __init__(self, enable_timing=True):
            self.t = None

        def record(self, stream):
            self.t = _time.perf_counter()

        def elapsed_time(self, other):
            return 1e3 * (other.t - self.t)

    class Pinned:  # what torch.from_numpy(a).pin_memory() is used for: .numpy() and being kept alive
        def __init__(self, a):
            self.a = a

        def pin_memory(self):
            return self

        def numpy(self):
            return self.a

    fake_torch = types.SimpleNamespace(tensor=torch.tensor, from_numpy=Pinned,
                                       cuda=types.SimpleNamespace(synchronize=lambda dev: None, Event=Event))
    made = {}

    def cheap_chain(batch, n_pts, n_segs, device, seed):
        d = make_batch(batch, n_pts, n_segs, seed, chain=True)
        q = np.random.default_rng(seed).standard_normal((batch, 4))
        d.T_ref_w[:, :4] = q / np.linalg.norm(q, axis=1, keepdims=True)  # lean_copy turns the pose into a camera centre
        made["d"] = d
        return d

    fake_synth = types.SimpleNamespace(make_chain_batch=cheap_chain, chain_frames=synth.chain_frames, pose_error=synth.pose_error,
                                       pose7_to_Rt=synth.pose7_to_Rt)
    args = types.SimpleNamespace(n_pts=30, n_segs=8, steps=2)
    B = 260  # the streamed host path (>= 256 pairs), as in the bench
    al = pkg.SparseImgAlign(4, 2, 30, ctx=pkg.api.Context(0))
    h0 = lib.fake_cuda_h2d_bytes()
    ms, (cfull, out_c, h2d_chain, chk) = bench.chain_leg(args, al, fake_synth, fake_torch, "cpu", None, B, 0)
    clean()
    assert cfull is made["d"] and ms > 0
    assert chk["pairs"] == B and chk["iteration_counts_equal_to_two_stack_call"] == B
    assert chk["max_rot_rad_vs_two_stack_call"] == 0.0 and chk["max_rel_t_vs_two_stack_call"] == 0.0
    # what the kernel saw in the one-stack calls = the lean form of the batch (digest of the last call)
    lean, lean_bytes, _keep = bench.lean_copy(cfull, fake_torch)
    seen = copy.copy(lean)
    seen.ref_pyr, seen.cur_pyr = cfull.ref_pyr, cfull.cur_pyr  # levels 3 and 4 are derived on the device from the shipped one
    want, _lvl = expected(seen)
    assert np.array_equal(out_c.n_tracked, want), "chain leg: the kernel did not see the lean batch"
    # the leg's byte accounting equals what crossed the model link in one one-stack call (plus the arrival flags)
    moved = lib.fake_cuda_h2d_bytes() - h0
    two_stack, one_stack = lean_bytes, h2d_chain
    assert two_stack - one_stack == (B - 1) * cfull.ref_pyr[2][0].nbytes
    calls_one = 2 + args.steps
    assert 0 <= moved - (two_stack + calls_one * one_stack) <= 8 * (1 + calls_one), (moved, two_stack, one_stack)
    # the CPU-arm sample the bench takes afterwards
    sub = bench.subset(cfull, 16)
    assert sub.batch == 16 and np.array_equal(sub.ref_pyr[3], cfull.ref_pyr[3][:16])


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
            lib.fake_cuda_drop_pending()  # whatever is still queued may point at arrays of the failed scenario
    print("RESULT " + json.dumps(res), flush=True)
    lib.fake_cuda_drop_pending()


if __name__ == "__main__":
    main(sys.argv[1:])
