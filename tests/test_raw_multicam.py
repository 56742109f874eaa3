"""Raw frames from differently calibrated lenses in one batch: plsvo_align_raw_multicam_batch_run /
plsvo_track_raw_multicam_batch_run rectify every frame with its pair's camera (undistort_pyramid_multicam_kernel, one map
per camera from the context's multicam map cache) and align each pair with that camera's intrinsics (the multicam
kernels).  Pair b's results must be byte-identical to plsvo_align_raw_batch_run / plsvo_track_raw_batch_run on that pair
with its own camera and the same kernel variant.

CPU: symbols, the ctypes layout, the new kernel's ptxas report, the Python argument checks, this file's GPU tests against
the host model of the C ABI (tests/hostmodel/fake_raw_multicam.cpp with fake_undistort.cpp and fake_raw_pyramid.cpp: real
rectification arithmetic, digest alignment), and two faults seeded into plsvo_abi.cu that the model must notice."""
import ctypes as C
import importlib.util
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from test_raw_track import (ALIGN_FIELDS, CAMS, COPY, EUROC, ODD, POSE_FIELDS, assert_same, camera, features, params,
                            raw_frames)

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ABI_SOURCE = os.path.join(ROOT, "pl-svo_b200", "csrc", "plsvo_abi.cu")
VGA4 = ("vga_strong_barrel_k3", "vga_pincushion", "vga_tangential_only", "vga_d0_zero_is_a_copy")
# the host model rectifies and half-samples on the CPU: it runs the large batches at a size it can afford
MODEL = bool(os.environ.get("PLSVO_FAKE_CUDA"))
BIG = 64 if MODEL else 1024
# the host model's pose-optimiser digest writes only these outputs; the others hold whatever the buffer held
PO_FIELDS = ("T_f_w", "num_obs_pt", "status") if MODEL else POSE_FIELDS


@pytest.fixture(autouse=True)
def _host_model_is_clean(pkg):
    """Against the host model, every test must leave no model error (out-of-bounds access, unwritten map entries)."""
    yield
    if MODEL:
        lib = C.CDLL(os.environ["PLSVO_LIB"])
        lib.fake_cuda_errors.restype = C.c_char_p
        err = lib.fake_cuda_errors().decode()
        lib.fake_cuda_clear_errors()
        assert not err, err


def cams_of(pkg, names):
    return [camera(pkg, n) for n in names]


def sub_batch(synth, data, idx, name):
    """Pairs idx of a mixed batch as the one-camera batch of camera `name`."""
    sub = synth.take_pairs(data, idx)
    sub.cam = synth.Camera(*params(name)[:6])
    return sub


def with_bearings(data, names, cop):
    """Full bearings: pt_f, seg_sf, seg_ef lifted through every pair's own camera."""
    def lift(px, k):
        f = np.stack([(px[..., 0] - k[:, None, 2]) / k[:, None, 0], (px[..., 1] - k[:, None, 3]) / k[:, None, 1],
                      np.ones(px.shape[:2])], -1)
        return np.ascontiguousarray(f / np.linalg.norm(f, axis=-1, keepdims=True))

    k = np.array([params(names[c])[2:6] for c in cop], np.float64)
    data.pt_f, data.seg_sf, data.seg_ef = lift(data.pt_px, k), lift(data.seg_spx, k), lift(data.seg_epx, k)
    return data


def ragged(data, seed):
    rng = np.random.default_rng(seed)
    data.pt_count = rng.integers(0, data.n_pts + 1, data.batch).astype(np.int32)
    data.seg_count = rng.integers(0, data.n_segs + 1, data.batch).astype(np.int32)
    data.pt_count[0] = data.seg_count[0] = 0  # a pair without features
    return data


def per_camera_raw(pkg, synth, names, cop, raw, data, hi, lo, ctx):
    """Every camera's raw call on its own pairs, scattered back to batch order."""
    out = None
    for k in np.unique(cop):
        idx = np.flatnonzero(cop == k)
        got = pkg.SparseImgAlign(hi, lo, 30, ctx=ctx).run_raw(camera(pkg, names[k]), (raw[0][idx], raw[1][idx]),
                                                                sub_batch(synth, data, idx, names[k]))
        if out is None:
            out = {f: np.zeros((data.batch,) + getattr(got, f).shape[1:], getattr(got, f).dtype) for f in ALIGN_FIELDS}
        for f in ALIGN_FIELDS:
            out[f][idx] = getattr(got, f)
    return out


def assert_rows(got, want, what=""):
    for f in ALIGN_FIELDS:
        np.testing.assert_array_equal(getattr(got, f), want[f], err_msg=f"{what} {f}")


def mixed_raw(names, cop, seed):
    B = len(cop)
    return raw_frames(names[0], B, seed=seed), raw_frames(names[0], B, seed=seed + 1)


def nvcc():
    return shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_library_exports_the_raw_multicam_calls_and_launcher(pkg):
    syms = subprocess.check_output(["nm", "-DC", "--defined-only", pkg.abi.LIB_PATH], text=True)
    assert "plsvo::undistort_pyramid_multicam_launch(" in syms
    for n in ("plsvo_align_raw_multicam_batch_run", "plsvo_track_raw_multicam_batch_run"):
        assert re.search(rf"\b{n}\b", syms), n
    names = {n for n, _, _ in pkg.abi.ABI_SYMBOLS}
    assert {"plsvo_align_raw_multicam_batch_run", "plsvo_track_raw_multicam_batch_run"} <= names


def test_raw_multicam_frames_ctypes_layout_matches_the_header(pkg, tmp_path):
    fields = ("n_cams", "reserved", "cams", "cam_of_pair", "ref_raw", "cur_raw", "pitch", "stride")
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "plsvo_b200.h"\nint main(void){printf("%zu'
                   + " %zu" * len(fields) + '\\n", sizeof(plsvo_raw_multicam_frames)'
                   + "".join(f", offsetof(plsvo_raw_multicam_frames, {f})" for f in fields) + ");return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    R = pkg.abi.RawMulticamFrames
    assert got == [C.sizeof(R)] + [getattr(R, f).offset for f in fields]


@pytest.mark.skipif(nvcc() is None, reason="nvcc not found")
def test_multicam_fused_kernel_keeps_two_ctas_per_sm(tmp_path):
    spec = importlib.util.spec_from_file_location("plsvo_build_flags", os.path.join(ROOT, "pl-svo_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    flags = [f for f in mod.NVCC_FLAGS if f != "-shared"]
    res = subprocess.run([nvcc()] + flags + ["-Xptxas", "-v", "-c", "-o", str(tmp_path / "u.o"), "undistort_kernel.cu"],
                         cwd=os.path.join(ROOT, "pl-svo_b200", "csrc"), capture_output=True, text=True, check=True)
    log = res.stdout + res.stderr
    m = re.search(r"Compiling entry function '\S*undistort_pyramid_multicam_kernel\S*' for 'sm_90a'\s*\n"
                  r"(?:.*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\s*\n"
                  r"ptxas info\s*: Used (\d+) registers", log)
    assert m, "no ptxas report for undistort_pyramid_multicam_kernel:\n" + log[-3000:]
    stack, stores, loads, regs = map(int, m.groups())
    assert (stack, stores, loads) == (0, 0, 0) and regs <= 64, (stack, stores, loads, regs)


def test_python_argument_checks_need_no_library(pkg, synth):
    api = pkg.api
    data = features(synth, VGA4[0], 3, seed=1)
    cams = cams_of(pkg, VGA4[:2])
    raw = mixed_raw(VGA4, [0, 1, 0], 2)
    with pytest.raises(api.PlsvoError, match="sequence of PinholeCamera"):
        api._raw_call_args(cams[0], raw, data, [0, 1, 0])
    with pytest.raises(api.PlsvoError, match=r"shape \[3\]"):
        api._raw_call_args(cams, raw, data, [0, 1])
    with pytest.raises(api.PlsvoError, match="frame chains are not supported"):
        api._raw_call_args(cams, raw_frames(VGA4[0], 4, seed=3), data, [0, 1, 0])
    with pytest.raises(api.PlsvoError, match="at least one camera"):
        api._raw_call_args([], raw, data, [0, 1, 0])
    rf, ab, keep = api._raw_call_args(cams, raw, data, np.array([1, 0, 1]))
    assert rf.n_cams == 2 and [rf.cam_of_pair[b] for b in range(3)] == [1, 0, 1] and ab.flags == 0
    assert rf.cams[1].fx == params(VGA4[1])[2] and rf.pitch == 640 and rf.stride == 640 * 480


def test_raw_multicam_generator(synth):
    cams, dists = (synth.VGA, synth.TUM_FR1), ((-0.2, 0.05, 0.0, 0.0, 0.0), (0.1, 0.0, 0.001, 0.0, 0.0))
    al, (ref, cur), k = synth.make_raw_multicam_batch(cams, dists, [1, 0, 1], n_pts=8, n_segs=2, max_level=3, min_level=1)
    assert al.batch == 3 and ref.shape == cur.shape == (3, 480, 640) and ref.dtype == np.uint8
    np.testing.assert_array_equal(k[0], [cams[1].fx, cams[1].fy, cams[1].cx, cams[1].cy])
    import torch
    want = synth.render_distorted(synth.Scene(), cams[1], dists[1], torch.tensor(al.T_cur_w_gt[[2]])).numpy()
    np.testing.assert_array_equal(cur[2], want[0])


@pytest.fixture(scope="module")
def multicam_hostmodel(tmp_path_factory):
    return _build_model(str(tmp_path_factory.mktemp("hostmodel") / "libplsvo_hostmodel_raw_multicam.so"))


def _build_model(out, abi_source=ABI_SOURCE):
    spec = importlib.util.spec_from_file_location("plsvo_hostmodel_build", os.path.join(HERE, "hostmodel", "build.py"))
    hm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(hm)
    sources = [abi_source] + hm.SOURCES[1:]
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-Wno-unused-function", "-I" + hm.cuda_include(),
                    "-I" + os.path.join(ROOT, "pl-svo_b200", "csrc"), "-x", "c++", *sources,
                    *(os.path.join(HERE, "hostmodel", f) for f in ("fake_undistort.cpp", "fake_raw_pyramid.cpp", "fake_raw_multicam.cpp")),
                    "-o", out, "-lpthread", "-ldl", "-Wl,-Bsymbolic"], check=True)
    return out


def _run_model(lib, mode, k):
    env = dict(os.environ, PLSVO_LIB=lib, PLSVO_FAKE_CUDA=mode)
    for name in [n for n in env if n.startswith("PLSVO_") and n not in ("PLSVO_LIB", "PLSVO_FAKE_CUDA")]:
        del env[name]
    return subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-p", "no:cacheprovider",
                           "-k", k], env=env, capture_output=True, text=True, timeout=3000)


@pytest.mark.parametrize("mode", ["lazy", "eager"])
def test_gpu_tests_of_this_file_against_the_host_model(oracle, multicam_hostmodel, mode):
    """The GPU tests below on the unchanged host code of plsvo_abi.cu with the model CUDA runtime: rectification is
    computed for real, alignment and pose optimisation digest the bytes they are given; the model checks every access,
    the stream order, that no copy from the caller's arrays is pending when a call returns, and (the validation test) that
    a rejected call queued nothing.  The oracle end-to-end test needs real kernels and is deselected."""
    p = _run_model(multicam_hostmodel, mode, "not oracle_end_to_end")
    assert p.returncode == 0 and " skipped" not in p.stdout and " passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


FAULTS = {
    # the current frame of pair b is rectified with the camera of pair b + 1
    "current_frames_get_the_next_pairs_map": (
        [("    const int slot = slot_of_cam[in.cam_of_pair[f < B ? f : f - B]];\n",
          "    const int slot = slot_of_cam[in.cam_of_pair[f < B ? f : (f - B + 1) % B]];\n")],
        "mixed_k4"),
    # the missing maps are built after the fused kernel that reads them
    "map_build_queued_after_the_fused_launch": (
        [("      const int rc = map_launch(c, *slot_cam[m], c->mc_maps[m]->map1, c->mc_maps[m]->map2, s);\n"
          "      if (rc != PLSVO_OK) return rc;\n", ""),
         ("  CK(multicam ? undistort_pyramid_multicam_launch(r, d_visit, c->num_sms, s) : undistort_pyramid_launch(r, c->num_sms, s));\n",
          "  CK(multicam ? undistort_pyramid_multicam_launch(r, d_visit, c->num_sms, s) : undistort_pyramid_launch(r, c->num_sms, s));\n"
          "  if (multicam) for (auto& m : c->mc_maps) map_launch(c, m->cam, m->map1, m->map2, s);\n")],
        "mixed_k4 or cache"),
}


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_model_notices_seeded_fault(oracle, tmp_path, fault):
    edits, k = FAULTS[fault]
    src = open(ABI_SOURCE).read()
    for old, new in edits:
        assert src.count(old) == 1, f"the line this fault is seeded into has changed: {old!r}"
        src = src.replace(old, new)
    mutated = tmp_path / "plsvo_abi.cu"
    mutated.write_text(src)
    lib = _build_model(str(tmp_path / "libplsvo_hostmodel_fault.so"), str(mutated))
    p = _run_model(lib, "lazy", k)
    assert " passed" in p.stdout or " failed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]
    assert p.returncode != 0 and " failed" in p.stdout, f"{fault}: every test still passes — the model is blind to it"


# ---------------------------------------------------------------------------------------------------------------- GPU
K1_CASES = [(name, B, lv) for name in (EUROC, ODD, COPY) for B, lv in ((1, (4, 2)), (3, (2, 0)), (3, (6, 4)), (256, (5, 3)), (BIG, (6, 4)))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,lv", K1_CASES)
def test_gpu_k1_equals_the_raw_call(pkg, synth, name, B, lv, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2" if B <= 132 else "128,4")
    hi, lo = lv
    ctx = pkg.api.Context(0)
    data = features(synth, name, B, seed=B + hi, max_level=hi, min_level=lo)
    raw = (raw_frames(name, B, seed=B), raw_frames(name, B, seed=B + 1))
    cam = camera(pkg, name)
    want = pkg.SparseImgAlign(hi, lo, 30, ctx=ctx).run_raw(cam, raw, data)
    # one camera named by every pair, and the same camera listed twice (byte-equal cameras share one map)
    for cams, cop in (([cam], np.zeros(B, np.int32)), ([cam, cam], np.arange(B, dtype=np.int32) % 2)):
        got = pkg.SparseImgAlign(hi, lo, 30, ctx=ctx).run_raw(cams, raw, data, cam_of_pair=cop)
        assert_same(got, want, ALIGN_FIELDS)
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("B", [37, BIG])
@pytest.mark.parametrize("bearings", ["lean", "full"])
def test_gpu_mixed_k4_equals_each_cameras_raw_call(pkg, synth, B, bearings, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2" if B <= 132 else "128,4")
    ctx = pkg.api.Context(0)
    rng = np.random.default_rng(B)
    cop = rng.integers(0, 4, B).astype(np.int32)
    cop[:4] = (3, 0, 2, 1)  # every camera, in no particular order
    data = ragged(features(synth, VGA4[0], B, seed=7 + B), seed=B)
    if bearings == "full":
        data = with_bearings(data, VGA4, cop)
    raw = mixed_raw(VGA4, cop, seed=11 + B)
    got = pkg.SparseImgAlign(4, 2, 30, ctx=ctx).run_raw(cams_of(pkg, VGA4), raw, data, cam_of_pair=cop)
    assert_rows(got, per_camera_raw(pkg, synth, VGA4, cop, raw, data, 4, 2, ctx), "mixed K=4")
    # rect_out: every level of every frame is undistortImage of that frame with its own camera
    _, rect = pkg.SparseImgAlign(4, 2, 30, ctx=ctx).run_raw(cams_of(pkg, VGA4), raw, data, rect_levels=list(range(7)),
                                                            cam_of_pair=cop)
    frames, fcam = np.concatenate(raw, 0), np.concatenate([cop, cop])
    for k in range(4):
        idx = np.flatnonzero(fcam == k)
        want = camera(pkg, VGA4[k]).undistortImage(frames[idx], 7, ctx)
        for l in range(7):
            np.testing.assert_array_equal(rect[l][idx], want[l], err_msg=f"{VGA4[k]} level {l}")
    ctx.close()


def _variants():
    return ["64,8", "96,7", "96,5", "128,5", "128,4", "160,3", "192,2", "256,2"]


@pytest.mark.gpu
@pytest.mark.parametrize("variant", _variants())
def test_gpu_mixed_k4_every_variant(pkg, synth, variant, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", variant)
    ctx = pkg.api.Context(0)
    cop = np.array([2, 0, 3, 1, 0, 2], np.int32)
    data = features(synth, VGA4[0], len(cop), seed=21, n_pts=60, n_segs=12)
    raw = mixed_raw(VGA4, cop, seed=22)
    got = pkg.SparseImgAlign(4, 2, 30, ctx=ctx).run_raw(cams_of(pkg, VGA4), raw, data, cam_of_pair=cop)
    assert_rows(got, per_camera_raw(pkg, synth, VGA4, cop, raw, data, 4, 2, ctx), variant)
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_iter_ref", [None, 3])
@pytest.mark.parametrize("chained", [True, False])
def test_gpu_track_equals_each_cameras_track_raw(pkg, synth, chained, n_iter_ref, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    ctx = pkg.api.Context(0)
    cop = np.array([1, 3, 0, 2, 1, 0, 3], np.int32)
    B = len(cop)
    data = features(synth, VGA4[0], B, seed=31)
    po = synth.make_poseopt_batch(cam=data.cam, batch=B, n_pts=data.n_pts, n_segs=data.n_segs, seed=32, T_gt=data.T_cur_w_gt)
    raw = mixed_raw(VGA4, cop, seed=33)
    got_a, got_p = pkg.track_raw(cams_of(pkg, VGA4), raw, data, po, po_n_iter_ref=n_iter_ref, chained=chained, ctx=ctx,
                                 cam_of_pair=cop)
    for k in range(4):
        idx = np.flatnonzero(cop == k)
        sub = sub_batch(synth, data, idx, VGA4[k])
        sub_po = synth.take_pairs(po, idx)
        sub_po.fx = abs(params(VGA4[k])[2])  # errorMultiplier2 of the camera
        want_a, want_p = pkg.track_raw(camera(pkg, VGA4[k]), (raw[0][idx], raw[1][idx]), sub, sub_po, po_n_iter_ref=n_iter_ref,
                                       chained=chained, ctx=ctx)
        assert_same(_rows(got_a, idx, ALIGN_FIELDS), want_a, ALIGN_FIELDS)
        assert_same(_rows(got_p, idx, PO_FIELDS), want_p, PO_FIELDS)
    ctx.close()


def _rows(out, idx, fields):
    class R:
        pass

    r = R()
    for f in fields:
        setattr(r, f, getattr(out, f)[idx])
    return r


def euroc_fleet(n, seed):
    """n perturbed EuRoC calibrations: fx, fy +-5 %, cx, cy +-10 px, k1, k2 +-10 %."""
    rng = np.random.default_rng(seed)
    W, H, fx, fy, cx, cy, k1, k2, p1, p2, k3 = params(EUROC)
    out = []
    for _ in range(n):
        s = rng.uniform(-1, 1, 6)
        out.append([W, H, fx * (1 + 0.05 * s[0]), fy * (1 + 0.05 * s[1]), cx + 10 * s[2], cy + 10 * s[3], k1 * (1 + 0.1 * s[4]),
                    k2 * (1 + 0.1 * s[5]), p1, p2, k3])
    return out


@pytest.mark.gpu
def test_gpu_cache_k64(pkg, synth, monkeypatch):
    """64 perturbed EuRoC cameras: a repeat builds nothing, half new cameras build only those, results do not change
    across calls or with the pairs pre-grouped by camera, and the one-camera cache keeps its own behaviour in between."""
    monkeypatch.setenv("PLSVO_VARIANT", "128,4")
    ctx = pkg.api.Context(0)
    fleet = euroc_fleet(96, seed=5)
    K, B = 64, 128
    cop = np.random.default_rng(6).permutation(np.arange(B) % K).astype(np.int32)
    data = features(synth, EUROC, B, seed=41, n_pts=40, n_segs=8)
    raw = (raw_frames(EUROC, B, seed=42), raw_frames(EUROC, B, seed=43))
    al = pkg.SparseImgAlign(4, 2, 30, ctx=ctx)

    def run(cam_params, order=None):
        cams = [pkg.PinholeCamera(*p) for p in cam_params]
        n0 = ctx.launch_count()
        if order is None:
            out = al.run_raw(cams, raw, data, cam_of_pair=cop)
        else:
            out = al.run_raw(cams, (raw[0][order], raw[1][order]), synth.take_pairs(data, order), cam_of_pair=cop[order])
        return out, ctx.last_map_build_ms(), ctx.launch_count() - n0

    first, ms, n = run(fleet[:K])
    assert ms is not None and n == K + 2  # K map builds, the fused kernel, the alignment
    again, ms, n = run(fleet[:K])
    assert ms is None and n == 2
    assert_same(again, first, ALIGN_FIELDS)
    half = fleet[:K // 2] + fleet[K:K + K // 2]
    mixed, ms, n = run(half)
    assert ms is not None and n == K // 2 + 2
    assert_same(_rows(mixed, np.flatnonzero(cop < K // 2), ALIGN_FIELDS), _rows(first, np.flatnonzero(cop < K // 2), ALIGN_FIELDS),
                ALIGN_FIELDS)
    # one-camera raw calls and undistortImage between multicam calls: their own cache, built once
    one = pkg.PinholeCamera(*params(EUROC))
    sub = sub_batch(synth, data, [0, 1], EUROC)
    built = []
    for _ in range(2):
        al.run_raw(one, (raw[0][:2], raw[1][:2]), sub)
        built.append(ctx.last_map_build_ms() is not None)
        one.undistortImage(raw[0][:2], 1, ctx)
        built.append(ctx.last_map_build_ms() is not None)
        _, ms, n = run(half)
        assert ms is None and n == 2
    assert built == [True, False, False, False]
    # the same batch pre-grouped by camera gives the same pairs
    order = np.argsort(cop, kind="stable")
    grouped, ms, n = run(half, order)
    assert ms is None
    assert_same(grouped, _rows(mixed, order, ALIGN_FIELDS), ALIGN_FIELDS)
    ctx.close()


@pytest.mark.gpu
def test_gpu_raw_multicam_against_the_oracle_end_to_end(pkg, abi, synth, oracle, gen_device):
    """Three lenses of one image size: per camera, oracle undistortion -> oracle pyramid -> oracle alignment against the
    pairs of one multicam call, to the standard of tests/test_gpu_align.py; the aligned poses must also be closer to ground
    truth than the initial guess by a factor of four in median rotation and translation."""
    import undistort_oracle
    from test_gpu_align import _check

    undistort_oracle.build()
    cams = (synth.VGA, synth.TUM_FR1, synth.TUM_FR2)
    dists = ((-0.28, 0.07, 0.0, 0.0, 0.0), (0.15, -0.05, 0.001, -0.001, 0.0), (-0.1, 0.0, 0.0005, 0.0, 0.0))
    cop = np.array([0, 1, 2, 2, 0, 1], np.int32)
    data, (ref, cur), _ = synth.make_raw_multicam_batch(cams, dists, cop, n_pts=150, n_segs=30, seed=4343, device=gen_device)
    pcs = [pkg.PinholeCamera(c.width, c.height, c.fx, c.fy, c.cx, c.cy, *d) for c, d in zip(cams, dists)]
    data.ref_pyr = data.cur_pyr = {}
    gpu = pkg.SparseImgAlign(4, 2, 30).run_raw(pcs, (ref, cur), data, cam_of_pair=cop)
    for k in range(3):
        idx = np.flatnonzero(cop == k)
        sub = synth.take_pairs(data, idx)
        sub.cam = cams[k]
        r = undistort_oracle.undistort(abi, pcs[k].struct, np.concatenate([ref[idx], cur[idx]]), 5)
        n = len(idx)
        sub.ref_pyr = {l: np.ascontiguousarray(r[l][:n]) for l in range(2, 5)}
        sub.cur_pyr = {l: np.ascontiguousarray(r[l][n:]) for l in range(2, 5)}
        want = oracle.align(abi, sub, abi.align_params(4, 2, 30), n_threads=8)
        got = _rows(gpu, idx, ALIGN_FIELDS)
        _check(synth, got, want)
    a0, t0 = synth.pose_error(data.T_cur_w, data.T_cur_w_gt)
    a1, t1 = synth.pose_error(gpu.T_cur_w, data.T_cur_w_gt)
    assert np.median(a1) < 0.25 * np.median(a0) and np.median(t1) < 0.25 * np.median(t0), (a0, a1, t0, t1)


@pytest.mark.gpu
def test_gpu_validation_errors(pkg, abi, synth):
    """Every malformed call returns PLSVO_ERR_INVALID with its message before anything is queued (against the host
    model: no stream operation ran or is pending), and the context then runs a valid call."""
    ctx = pkg.api.Context(0)
    B, names = 3, VGA4[:2]
    W, H = params(names[0])[:2]
    data = features(synth, names[0], B, seed=400)
    good = mixed_raw(names, [0, 1, 0], 401)
    model = C.CDLL(os.environ["PLSVO_LIB"]) if MODEL else None

    def run(cam_params=None, cop=(0, 1, 0), edit_batch=None, edit_raw=None, hi=4, lo=2, rect=None, track=False, raw=None):
        cams = [pkg.PinholeCamera(*p) for p in (cam_params or [params(n) for n in names])]
        rf, ab, keep = pkg.api._raw_call_args(cams, good if raw is None else raw, data, np.array(cop))
        if edit_batch:
            edit_batch(ab)
        if edit_raw:
            edit_raw(rf)
        ap = abi.align_params(hi, lo, 30)
        out = abi.AlignOut(B, data.n_segs)
        r = rect() if rect else None
        rp = C.byref(r[1]) if r else None
        ops = model.fake_cuda_ops_run() if model else 0
        if track:
            po = synth.make_poseopt_batch(cam=data.cam, batch=B + 1, n_pts=4, n_segs=2, seed=3)
            pb, keep_p = abi.make_poseopt_batch(po)
            pp = abi.poseopt_params(2.0, 10, -1)
            po_out = abi.PoseOptOut(B + 1, 4, 2)
            rc = ctx.lib.plsvo_track_raw_multicam_batch_run(ctx.handle, C.byref(rf), C.byref(ab), C.byref(ap), C.byref(pb),
                                                            C.byref(pp), C.byref(out.struct), C.byref(po_out.struct), rp)
        else:
            rc = ctx.lib.plsvo_align_raw_multicam_batch_run(ctx.handle, C.byref(rf), C.byref(ab), C.byref(ap), C.byref(out.struct), rp)
        if model and rc != abi.OK:
            assert model.fake_cuda_pending_ops() == 0 and model.fake_cuda_ops_run() == ops, "a rejected call queued work"
        return rc, ctx.lib.plsvo_last_error(ctx.handle).decode()

    if model:
        model.fake_cuda_ops_run.restype = C.c_ulonglong

    def with_param(k, i, v):
        p = [list(params(n)) for n in names]
        p[k][i] = v
        return p

    def set_attr(**kw):
        def f(s):
            for k, v in kw.items():
                setattr(s, k, v)
        return f

    def image_in_batch(ab):
        ab.ref_img[3] = good[0].ctypes.data_as(C.POINTER(C.c_uint8))

    def rect_narrow():
        levels, r = abi.pyramid_levels(2 * B, H, W, 3)
        r.pitch[2] = (W >> 2) - 1
        return levels, r

    def rect_level7():
        levels, r = abi.pyramid_levels(2 * B, H, W, 1)
        r.level[7] = r.level[0]
        r.pitch[7] = W
        return levels, r

    cases = [
        (dict(edit_raw=set_attr(n_cams=0)), "n_cams must be at least 1"),
        (dict(edit_raw=set_attr(cams=None)), "n_cams must be at least 1"),
        (dict(edit_raw=set_attr(cam_of_pair=None)), "n_cams must be at least 1"),
        (dict(cop=(0, 2, 0)), "cam_of_pair[1] = 2 is outside [0, 2)"),
        (dict(cop=(0, 1, -1)), "cam_of_pair[2] = -1 is outside [0, 2)"),
        (dict(edit_raw=set_attr(n_cams=1)), "cam_of_pair[1] = 1 is outside [0, 1)"),
        (dict(cam_params=with_param(1, 0, W + 16)), "cams[1] is 656x480"),
        (dict(cam_params=with_param(1, 2, float("nan"))), "cams[1]: a parameter is not finite"),
        (dict(cam_params=with_param(0, 6, 1e300)), "cams[0]: a parameter is not finite"),
        (dict(cam_params=with_param(1, 3, 1e-60)), "cams[1]: fx and fy must be non-zero"),
        (dict(edit_batch=set_attr(flags=abi.ALIGN_FRAME_CHAIN)), "PLSVO_ALIGN_FRAME_CHAIN is not supported"),
        (dict(edit_batch=image_in_batch), "image pointers"),
        (dict(edit_raw=set_attr(cur_raw=None)), "raw stack is NULL"),
        (dict(edit_raw=set_attr(pitch=W - 1)), "pitch smaller"),
        (dict(hi=7, lo=2), "max_level > 6"),
        (dict(rect=rect_narrow), "rect_out: pitch"),
        (dict(rect=rect_level7), "level above 6"),
        (dict(track=True), "batches differ in size"),
    ]
    for kw, msg in cases:
        rc, err = run(**kw)
        assert rc == abi.ERR_INVALID and msg in err, (kw, rc, err)
        rc, err = run()  # the context is still usable
        assert rc == abi.OK, err
    ctx.close()
