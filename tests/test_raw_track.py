"""Alignment and tracking of raw (distorted) frames: plsvo_align_raw_batch_run / plsvo_track_raw_batch_run rectify and
half-sample on the device (undistort_pyramid_kernel) and feed the pyramid straight to the alignment and pose-optimiser
kernels.  Every result must be byte-identical to plsvo_undistort_batch_run followed by the plain host-buffer
plsvo_align_batch_run / plsvo_track_batch_run on the rectified levels.

CPU: symbols, the ctypes layout, the kernel's spill report, the synthetic raw renderer, and this file's GPU tests against
the host model of the C ABI linked with the model kernels of tests/hostmodel/fake_undistort.cpp and fake_raw_pyramid.cpp."""
import ctypes as C
import importlib.util
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
with open(os.path.join(HERE, "golden", "undistort_cv2.json")) as _f:
    CAMS = json.load(_f)["cameras"]
EUROC, PINCUSHION, COPY, HD, ODD = "euroc_dataset_params", "vga_pincushion", "vga_d0_zero_is_a_copy", "hd720", "odd_641x479"
ALIGN_FIELDS = ("T_cur_w", "n_tracked", "H", "seg_killed", "iters", "status", "patch_iters", "patch_levels")
POSE_FIELDS = ("T_f_w", "cov", "estimated_scale", "error_init", "error_final", "num_obs_pt", "num_obs_ls", "pt_outlier",
               "seg_outlier", "iters", "status")


def params(name):
    return CAMS[name]["params"]


def nvcc():
    return shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)


def raw_frames(name, n, seed, pad=0):
    """n smooth textured u8 frames of the camera's size (cheap to make for thousands of frames), rows padded by `pad`."""
    W, H = params(name)[:2]
    rng = np.random.default_rng(seed)
    x, y = np.arange(W + pad, dtype=np.float32), np.arange(H, dtype=np.float32)
    out = np.empty((n, H, W + pad), np.uint8)
    noise = rng.integers(0, 24, (H, W + pad)).astype(np.float32)
    for f in range(n):
        a, b, c = rng.uniform(0.02, 0.2, 3)
        p = rng.uniform(0, 6.3, 3)
        img = 100 + 50 * np.sin(a * x + p[0])[None, :] + 50 * np.cos(b * y + p[1])[:, None] + 20 * np.sin(c * (x[None, :] + y[:, None]) + p[2])
        out[f] = np.clip(img + np.roll(noise, f, axis=1), 0, 255).astype(np.uint8)
    return out[:, :, :W] if pad else out


def features(synth, name, B, seed, max_level=4, min_level=2, n_pts=120, n_segs=24):
    """Features and poses for B pairs of the undistorted camera: a few generated pairs repeated (the raw frames, not the
    features, are what these tests vary), without image pyramids."""
    import dataclasses

    W, H, fx, fy, cx, cy = params(name)[:6]
    cam = synth.Camera(W, H, fx, fy, cx, cy)
    base = synth.make_align_batch(cam=synth.QVGA, batch=min(B, 4), n_pts=n_pts, n_segs=n_segs, seed=seed, max_level=max_level,
                                  min_level=min_level, margin=16)
    rep = lambda a: None if a is None else np.ascontiguousarray(np.resize(a, (B,) + a.shape[1:]))
    sx, sy = W / synth.QVGA.width, H / synth.QVGA.height
    scale = np.array([sx, sy])
    d = dataclasses.replace(base, cam=cam, ref_pyr={}, cur_pyr={}, frame_pyr=None)
    for f in ("T_ref_w", "T_cur_w", "T_cur_w_gt", "pt_f", "pt_pos", "seg_sf", "seg_ef", "seg_spos", "seg_epos", "pt_valid", "seg_valid"):
        setattr(d, f, rep(getattr(base, f)))
    d.pt_px, d.seg_spx, d.seg_epx = (rep(getattr(base, f) * scale) for f in ("pt_px", "seg_spx", "seg_epx"))
    d.seg_length = rep(np.linalg.norm(d.seg_epx - d.seg_spx, axis=-1)[: min(B, 4)])
    d.pt_f = d.seg_sf = d.seg_ef = None  # bearings formed on the device from the pixels (cam2world of the camera)
    return d


def camera(pkg, name):
    return pkg.PinholeCamera(*params(name))


def with_levels(data, rect, lo, hi, chain):
    """The AlignData of the host path: the rectified levels lo..hi as dense host stacks."""
    import dataclasses

    d = dataclasses.replace(data)
    if chain:
        d.frame_pyr = {l: np.ascontiguousarray(rect[l]) for l in range(lo, hi + 1)}
    else:
        B = data.batch
        d.ref_pyr = {l: np.ascontiguousarray(rect[l][:B]) for l in range(lo, hi + 1)}
        d.cur_pyr = {l: np.ascontiguousarray(rect[l][B:]) for l in range(lo, hi + 1)}
    return d


def host_path_align(pkg, cam, raw, data, hi, lo, ctx):
    """plsvo_undistort_batch_run, then the plain upload -> launch -> download sequence on the rectified levels."""
    frames = raw if not isinstance(raw, tuple) else np.concatenate(raw, 0)
    rect = cam.undistortImage(frames, hi + 1, ctx)
    al = pkg.SparseImgAlign(hi, lo, 30, ctx=ctx)
    al.upload(with_levels(data, rect, lo, hi, not isinstance(raw, tuple)))
    al.launch()
    return al.download(), rect


def assert_same(a, b, fields):
    for f in fields:
        np.testing.assert_array_equal(getattr(a, f), getattr(b, f), err_msg=f)


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_library_exports_the_raw_calls_and_the_fused_launcher(pkg):
    syms = subprocess.check_output(["nm", "-DC", "--defined-only", pkg.abi.LIB_PATH], text=True)
    assert "plsvo::undistort_pyramid_launch(" in syms
    assert re.search(r"\bplsvo_align_raw_batch_run\b", syms) and re.search(r"\bplsvo_track_raw_batch_run\b", syms)


def test_raw_frames_ctypes_layout_matches_the_header(pkg, tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "plsvo_b200.h"\nint main(void){printf("%zu %zu %zu %zu %zu %zu\\n",'
                   "sizeof(plsvo_raw_frames), offsetof(plsvo_raw_frames, cam), offsetof(plsvo_raw_frames, ref_raw),"
                   "offsetof(plsvo_raw_frames, cur_raw), offsetof(plsvo_raw_frames, pitch), offsetof(plsvo_raw_frames, stride));return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    R = pkg.abi.RawFrames
    assert got == [C.sizeof(R), R.cam.offset, R.ref_raw.offset, R.cur_raw.offset, R.pitch.offset, R.stride.offset]


@pytest.mark.skipif(nvcc() is None, reason="nvcc not found")
def test_fused_kernel_does_not_spill(tmp_path):
    spec = importlib.util.spec_from_file_location("plsvo_build_flags", os.path.join(ROOT, "pl-svo_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    flags = [f for f in mod.NVCC_FLAGS if f != "-shared"]
    res = subprocess.run([nvcc()] + flags + ["-Xptxas", "-v", "-c", "-o", str(tmp_path / "u.o"), "undistort_kernel.cu"],
                         cwd=os.path.join(ROOT, "pl-svo_b200", "csrc"), capture_output=True, text=True, check=True)
    log = res.stdout + res.stderr
    m = re.search(r"Compiling entry function '\S*undistort_pyramid_kernel\S*' for 'sm_90a'\s*\n"
                  r"(?:.*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\s*\n"
                  r"ptxas info\s*: Used (\d+) registers", log)
    assert m, "no ptxas report for undistort_pyramid_kernel:\n" + log[-3000:]
    stack, stores, loads, regs = map(int, m.groups())
    assert (stack, stores, loads) == (0, 0, 0) and regs <= 64, (stack, stores, loads, regs)


def test_synthetic_raw_render_rectifies_to_the_undistorted_render(synth, abi, oracle):
    """render_distorted, rectified by the C++ undistortion oracle, is Scene.render of the undistorted camera up to
    interpolation: a sanity check of the generator, with a loose bound, away from the border."""
    import torch
    import undistort_oracle

    undistort_oracle.build()
    cam, dist = synth.EUROC, synth.EUROC_DIST
    pose = torch.tensor([[1.0, 0.0, 0.0, 0.0, 0.02, -0.01, 0.0]], dtype=torch.float64)
    scene = synth.Scene()
    raw = synth.render_distorted(scene, cam, dist, pose).numpy()
    want = scene.render(cam, pose).numpy()[0].astype(np.int32)
    pc = abi.PinholeCamera(cam.width, cam.height, cam.fx, cam.fy, cam.cx, cam.cy, (C.c_double * 5)(*dist))
    got = undistort_oracle.undistort(abi, pc, raw, 1)[0][0].astype(np.int32)
    m = 40
    diff = np.abs(got - want)[m:-m, m:-m]
    assert np.median(diff) <= 3 and np.percentile(diff, 99) <= 25, (np.median(diff), np.percentile(diff, 99))
    assert np.abs(raw[0].astype(np.int32) - want).mean() > 2 * diff.mean()  # the lens does distort


@pytest.fixture(scope="module")
def raw_hostmodel(tmp_path_factory):
    spec = importlib.util.spec_from_file_location("plsvo_hostmodel_build", os.path.join(HERE, "hostmodel", "build.py"))
    hm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(hm)
    out = str(tmp_path_factory.mktemp("hostmodel") / "libplsvo_hostmodel_raw.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-Wno-unused-function", "-I" + hm.cuda_include(),
                    "-x", "c++", *hm.SOURCES, os.path.join(HERE, "hostmodel", "fake_undistort.cpp"),
                    os.path.join(HERE, "hostmodel", "fake_raw_pyramid.cpp"), "-o", out, "-lpthread", "-ldl", "-Wl,-Bsymbolic"], check=True)
    return out


@pytest.mark.parametrize("mode", ["lazy", "eager"])
def test_gpu_tests_of_this_file_against_the_host_model(oracle, raw_hostmodel, mode):
    """The GPU tests below on the unchanged host code of plsvo_abi.cu with the model CUDA runtime: the alignment and
    pose-optimiser "kernels" digest the bytes they are given, so byte-identical results mean the raw path hands them
    exactly the levels the host path ships; the model checks every access, the stream order and that no copy from the
    caller's arrays is pending when a call returns.  The oracle end-to-end test needs real kernels and is deselected."""
    env = dict(os.environ, PLSVO_LIB=raw_hostmodel, PLSVO_FAKE_CUDA=mode)
    p = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        "-k", "not oracle_end_to_end"], env=env, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0 and " skipped" not in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------------------- GPU
CASES = [  # camera, B, chain, (max_level, min_level)
    (EUROC, 1, True, (4, 2)), (EUROC, 3, False, (4, 2)), (EUROC, 3, True, (2, 0)), (PINCUSHION, 3, True, (4, 2)),
    (PINCUSHION, 1, False, (5, 3)), (COPY, 3, True, (4, 2)), (COPY, 3, False, (2, 0)), (HD, 3, True, (5, 3)), (HD, 1, False, (4, 2)),
    (ODD, 3, False, (4, 2)), (ODD, 3, True, (5, 3)), (ODD, 1, True, (2, 0)), (EUROC, 256, True, (4, 2)), (EUROC, 256, False, (2, 0)),
    (EUROC, 1024, True, (4, 2)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,chain,lv", CASES)
def test_gpu_align_raw_is_undistort_then_align(pkg, synth, name, B, chain, lv):
    hi, lo = lv
    ctx = pkg.api.Context(0)
    data = features(synth, name, B, seed=B + hi, max_level=hi, min_level=lo)
    raw = raw_frames(name, B + 1, seed=B) if chain else (raw_frames(name, B, seed=B), raw_frames(name, B, seed=B + 1))
    cam = camera(pkg, name)
    want, _ = host_path_align(pkg, cam, raw, data, hi, lo, ctx)
    got = pkg.SparseImgAlign(hi, lo, 30, ctx=ctx).run_raw(cam, raw, data)
    assert_same(got, want, ALIGN_FIELDS)
    assert ctx.last_kernel_ms() >= 0
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("chain", [True, False])
def test_gpu_padded_and_strided_raw_rows(pkg, synth, chain):
    B, W, H = 5, *params(EUROC)[:2]
    ctx = pkg.api.Context(0)
    data = features(synth, EUROC, B, seed=71)
    big = raw_frames(EUROC, 2 * (B + 1) + 2, seed=72, pad=41)
    cam = camera(pkg, EUROC)
    # padded rows; padded rows and every other frame
    for ref, cur in ((big[: B + 1], big[B + 1 : 2 * B + 1]), (big[::2][: B + 1], big[1::2][:B])):
        raw = ref if chain else (ref[:B], cur)
        assert ref.strides[1] != W
        want, _ = host_path_align(pkg, cam, raw, data, 4, 2, ctx)
        got = pkg.SparseImgAlign(4, 2, 30, ctx=ctx).run_raw(cam, raw, data)
        assert_same(got, want, ALIGN_FIELDS)
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_iter_ref", [None, 3])
@pytest.mark.parametrize("name,B,chain", [(EUROC, 3, True), (ODD, 3, False), (COPY, 2, True), (EUROC, 256, True)])
def test_gpu_track_raw_is_undistort_then_track(pkg, synth, name, B, chain, n_iter_ref):
    ctx = pkg.api.Context(0)
    data = features(synth, name, B, seed=90 + B)
    W, H, fx, fy, cx, cy = params(name)[:6]
    po = synth.make_poseopt_batch(cam=data.cam, batch=B, n_pts=data.n_pts, n_segs=data.n_segs, seed=91, T_gt=data.T_cur_w_gt)
    raw = raw_frames(name, B + 1, seed=B) if chain else (raw_frames(name, B, seed=B), raw_frames(name, B, seed=B + 1))
    cam = camera(pkg, name)
    frames = raw if chain else np.concatenate(raw, 0)
    rect = cam.undistortImage(frames, 5, ctx)
    want_a, want_p = pkg.api.track(with_levels(data, rect, 2, 4, chain), po, po_n_iter_ref=n_iter_ref, ctx=ctx)
    got_a, got_p = pkg.track_raw(cam, raw, data, po, po_n_iter_ref=n_iter_ref, ctx=ctx)
    assert_same(got_a, want_a, ALIGN_FIELDS)
    assert_same(got_p, want_p, POSE_FIELDS)
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,chain", [(EUROC, True), (ODD, False), (COPY, True)])
def test_gpu_rect_out_levels_are_undistort_image(pkg, synth, name, chain):
    B = 3
    ctx = pkg.api.Context(0)
    data = features(synth, name, B, seed=55)
    raw = raw_frames(name, B + 1, seed=56) if chain else (raw_frames(name, B, seed=56), raw_frames(name, B, seed=57))
    cam = camera(pkg, name)
    frames = raw if chain else np.concatenate(raw, 0)
    want = cam.undistortImage(frames, 7, ctx)
    al = pkg.SparseImgAlign(4, 2, 30, ctx=ctx)
    plain = al.run_raw(cam, raw, data)
    for levels in ([0], [1, 6], [0, 2, 3, 5], list(range(7))):
        out, rect = al.run_raw(cam, raw, data, rect_levels=levels)
        assert sorted(rect) == levels
        for l in levels:
            np.testing.assert_array_equal(rect[l], want[l], err_msg=f"level {l}")
        assert_same(out, plain, ALIGN_FIELDS)
    ctx.close()


@pytest.mark.gpu
def test_gpu_raw_path_against_the_oracle_end_to_end(pkg, abi, synth, oracle, gen_device):
    """Oracle undistortion -> oracle pyramid -> oracle alignment on seeded distorted frames of the analytic scene, against
    the raw path: the standard of tests/test_gpu_align.py.  On these noiseless frames the aligned poses must also be
    closer to ground truth than the initial guess by at least a factor of four in median rotation and translation
    (rectification's interpolation leaves an error of its own, so the raw path is held to ground truth that loosely)."""
    import undistort_oracle
    from test_gpu_align import _check

    undistort_oracle.build()
    data, raw = synth.make_raw_chain_batch(batch=4, n_pts=150, n_segs=30, seed=4242, device=gen_device)
    cam = pkg.PinholeCamera(*params(EUROC))
    gpu = pkg.SparseImgAlign(4, 2, 30).run_raw(cam, raw, data)
    rect = undistort_oracle.undistort(abi, cam.struct, raw, 5)
    data.ref_pyr = {l: np.ascontiguousarray(rect[l][:-1]) for l in range(2, 5)}
    data.cur_pyr = {l: np.ascontiguousarray(rect[l][1:]) for l in range(2, 5)}
    data.frame_pyr = None
    ref = oracle.align(abi, data, abi.align_params(4, 2, 30), n_threads=8)
    _check(synth, gpu, ref)
    a0, t0 = synth.pose_error(data.T_cur_w, data.T_cur_w_gt)
    a1, t1 = synth.pose_error(gpu.T_cur_w, data.T_cur_w_gt)
    assert np.median(a1) < 0.25 * np.median(a0) and np.median(t1) < 0.25 * np.median(t0), (a0, a1, t0, t1)


@pytest.mark.gpu
def test_gpu_context_reuse_cameras_and_sizes(pkg, synth):
    """raw -> plain -> raw on one context, two cameras alternating, an image-size change; the map-build time is reported
    exactly when a call built a map."""
    ctx = pkg.api.Context(0)
    B = 3
    built = []
    for k, name in enumerate([EUROC, EUROC, "vga_strong_barrel_k3", EUROC, ODD, COPY, EUROC]):
        data = features(synth, name, B, seed=300 + k)
        raw = raw_frames(name, B + 1, seed=310 + k)
        cam = camera(pkg, name)
        got = pkg.SparseImgAlign(4, 2, 30, ctx=ctx).run_raw(cam, raw, data)
        built.append(ctx.last_map_build_ms() is not None)
        want, _ = host_path_align(pkg, cam, raw, data, 4, 2, ctx)  # a plain call between raw calls
        assert_same(got, want, ALIGN_FIELDS)
    assert built == [True, False, True, True, True, False, True]
    ctx.close()


@pytest.mark.gpu
def test_gpu_validation_errors(pkg, abi, synth):
    ctx = pkg.api.Context(0)
    B, name = 2, ODD
    data = features(synth, name, B, seed=400)
    W, H = params(name)[:2]
    good_raw = raw_frames(name, B + 1, seed=401)
    cam = camera(pkg, name)

    def run(cam_params=None, raw=None, edit_batch=None, edit_raw=None, hi=4, lo=2, rect=None, track=False):
        c = pkg.PinholeCamera(*(cam_params or params(name)))
        rf, ab, keep = pkg.api._raw_call_args(c, good_raw if raw is None else raw, data)
        if edit_batch:
            edit_batch(ab)
        if edit_raw:
            edit_raw(rf)
        ap = abi.align_params(hi, lo, 30)
        out = abi.AlignOut(B, data.n_segs)
        r = rect(W, H) if rect else None
        rp = C.byref(r[1]) if r else None
        if track:
            po = synth.make_poseopt_batch(cam=data.cam, batch=B + 1, n_pts=4, n_segs=2, seed=3)
            pb, keep_p = abi.make_poseopt_batch(po)
            pp = abi.poseopt_params(2.0, 10, -1)
            po_out = abi.PoseOptOut(B + 1, 4, 2)
            rc = ctx.lib.plsvo_track_raw_batch_run(ctx.handle, C.byref(rf), C.byref(ab), C.byref(ap), C.byref(pb), C.byref(pp),
                                                   C.byref(out.struct), C.byref(po_out.struct), rp)
        else:
            rc = ctx.lib.plsvo_align_raw_batch_run(ctx.handle, C.byref(rf), C.byref(ab), C.byref(ap), C.byref(out.struct), rp)
        return rc, ctx.lib.plsvo_last_error(ctx.handle).decode()

    def with_param(i, v):
        p = list(params(name))
        p[i] = v
        return p

    def set_attr(**kw):
        def f(s):
            for k, v in kw.items():
                setattr(s, k, v)
        return f

    def image_in_batch(ab):
        ab.ref_img[3] = good_raw.ctypes.data_as(C.POINTER(C.c_uint8))

    def rect_narrow(W, H):
        levels, r = abi.pyramid_levels(B + 1, H, W, 3)
        r.pitch[2] = (W >> 2) - 1
        return levels, r

    def rect_level7(W, H):
        levels, r = abi.pyramid_levels(B + 1, H, W, 1)
        r.level[7] = r.level[0]
        r.pitch[7] = W
        return levels, r

    def rect_tiny(W, H):
        levels, r = abi.pyramid_levels(B + 1, H, W, 1)
        r.level[6] = r.level[0]
        r.pitch[6] = W
        return levels, r

    small = raw_frames(name, B + 1, seed=1)[:, :8, :8]  # an 8x8 camera with level 6 below one pixel

    def tiny_cam(ab):
        ab.cam.width, ab.cam.height = 8, 8

    cases = [
        (dict(cam_params=with_param(2, params(name)[2] + 1e-3)), "differ in width, height, fx, fy, cx or cy"),
        (dict(edit_batch=set_attr(flags=0)), "raw stack is NULL"),
        (dict(edit_batch=image_in_batch), "image pointers"),
        (dict(edit_raw=set_attr(ref_raw=None)), "raw stack is NULL"),
        (dict(edit_raw=lambda r: setattr(r, "cur_raw", r.ref_raw)), "cur_raw must be NULL"),
        (dict(edit_raw=set_attr(pitch=W - 1)), "pitch smaller"),
        (dict(cam_params=with_param(2, float("nan"))), "not finite"),
        (dict(cam_params=with_param(8, float("inf"))), "not finite"),
        (dict(cam_params=with_param(5, 1e300)), "not finite"),
        (dict(cam_params=with_param(3, 1e-60)), "non-zero"),
        (dict(hi=7, lo=2), "max_level > 6"),
        (dict(rect=rect_narrow), "rect_out: pitch"),
        (dict(rect=rect_level7), "level above 6"),
        (dict(raw=small, edit_batch=tiny_cam, cam_params=[8, 8] + params(name)[2:], rect=rect_tiny), "smaller than one pixel"),
        (dict(track=True), "batches differ in size"),
    ]
    for kw, msg in cases:
        rc, err = run(**kw)
        assert rc == abi.ERR_INVALID and msg in err, (kw, rc, err)
        rc, err = run()  # the context is still usable
        assert rc == abi.OK, err
    ctx.close()
