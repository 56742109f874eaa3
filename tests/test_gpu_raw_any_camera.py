"""Raw frames from distorted lenses and ATAN (FOV) cameras in one batch (plsvo_align_raw_any_camera_batch_run,
plsvo_track_raw_any_camera_batch_run): pair b's camera is cams[cam_of_pair[b]], a plsvo_raw_camera whose tag picks the
model.  A lens pair's outputs must be byte-identical to plsvo_align_raw_multicam_batch_run on the lens pairs, an ATAN
pair's to plsvo_align_atan_multicam_batch_run on createImgPyramid of its raw frames, at the same kernel variant;
rect_out fed to plsvo_align_any_camera_batch_run must give the same bytes; the slot padding must not matter; only
distorted lenses build maps, in the cache the raw multicam calls keep; each model group agrees with its oracle.

CPU: the exports and ctypes layouts, the Python dispatch and synth.make_raw_any_camera_batch, this file's GPU tests
against the host model of the C ABI (real rectification and half-sampling by fake_mixed_sizes.cpp's fused kernel, each
pair aligned by its tag through fake_any_camera.cpp), and three faults seeded into plsvo_abi.cu that the model, with
every kernel answered by the CPU oracles, must notice."""
import ctypes as C
import functools
import importlib.util
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_atan_multicam import _oracle_lib, cop_of, slot_cam
from test_gpu_mixed_sizes import crop, interleave, rows
from test_gpu_multicam import ALIGN_FIELDS, PO_FIELDS, assert_same, lean, ragged
from test_raw_track import EUROC, ODD, features, params, raw_frames

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ABI_SOURCE = os.path.join(ROOT, "pl-svo_b200", "csrc", "plsvo_abi.cu")
MODEL = bool(os.environ.get("PLSVO_FAKE_CUDA"))
ORACLE_MODEL = bool(os.environ.get("PLSVO_FAKE_ORACLE"))
BIG = 16 if MODEL else 1024  # the host model renders and rectifies on the CPU
VARIANTS = ["64,8", "96,7", "96,5", "128,5", "128,4", "160,3", "192,2", "256,2"]
STOCK_ATAN = (752, 480, 0.511496, 0.802603, 0.530199, 0.496011, 0.934092)  # SVO's stock FOV camera


def stock(pkg):
    """EuRoC's cam0 lens and SVO's stock 752x480 ATAN camera."""
    return [pkg.PinholeCamera(*params(EUROC)), pkg.ATANCamera(*STOCK_ATAN)]


def fleet(pkg):
    """Eight cameras in one 752x480 slot: a lens and an ATAN camera at each of 752x480, 640x480, 641x479 and 320x240.
    The 320x240 lens has d0 = 0 (a copy whatever d1..d4); the ATAN cameras have d0 in {0.93, 0.3, 0, 0.93}."""
    return [pkg.PinholeCamera(*params(EUROC)), pkg.ATANCamera(752, 480, 0.5825, 0.8000, 0.5127, 0.4784, 0.93),
            pkg.PinholeCamera(*params("vga_strong_barrel_k3")), pkg.ATANCamera(640, 480, 0.6600, 0.9000, 0.4900, 0.5300, 0.3),
            pkg.PinholeCamera(*params(ODD)), pkg.ATANCamera(641, 479, 0.6500, 0.8700, 0.5000, 0.5000, 0.0),
            pkg.PinholeCamera(320, 240, 210.0, 205.0, 159.5, 119.5, 0.0, 0.2, 0.001, 0.0, 0.0),
            pkg.ATANCamera(320, 240, 0.6800, 0.8800, 0.5200, 0.4800, 0.93)]


def is_atan(pkg, cam):
    return isinstance(cam, pkg.ATANCamera)


def undistorted(synth, lens):
    s = lens.struct
    return synth.Camera(s.width, s.height, s.fx, s.fy, s.cx, s.cy)


def slot_of(synth, cams):
    return synth.Camera(max(c.width for c in cams), max(c.height for c in cams), 1.0, 1.0, 0.0, 0.0)


@functools.lru_cache(maxsize=4)
def _fleet_batch(K, B, seed, device, fill_key, n_pts, n_segs, poseopt):
    import plsvo_b200 as pkg

    synth = pkg.synth
    cams = stock(pkg) if K == 2 else fleet(pkg)
    cop = cop_of(interleave(len(cams), B, seed), B)
    fill = np.random.default_rng(fill_key[1]) if fill_key[0] == "rng" else fill_key[1]
    out = synth.make_raw_any_camera_batch(cams, cop, slot=slot_of(synth, cams), fill=fill, poseopt=poseopt, n_pts=n_pts,
                                          n_segs=n_segs, seed=seed, device=device)
    out[0].ref_pyr = out[0].cur_pyr = {}  # the raw calls read the raw frames only
    return cams, cop, out


def fleet_batch(K, B, seed, device, fill=0, n_pts=150, n_segs=40, poseopt=False):
    """(cams, cam_of_pair, data, (ref_raw, cur_raw)[, po]) of a fleet at B interleaved pairs; data is a fresh shallow copy
    (the tests replace its arrays, never write into them)."""
    import copy

    fill_key = ("rng", fill) if isinstance(fill, tuple) else ("byte", fill)
    cams, cop, out = _fleet_batch(K, B, seed, device, fill_key, n_pts, n_segs, poseopt)
    if poseopt:
        return cams, cop, copy.copy(out[0]), out[2], copy.copy(out[1])
    return cams, cop, copy.copy(out[0]), out[1]


def sub_table(cams, cop, idx):
    """The cameras pairs idx use, and their cam_of_pair into that list."""
    used = sorted(set(cop[idx].tolist()))
    return [cams[k] for k in used], np.array([used.index(k) for k in cop[idx]], np.int32)


def atan_levels(pkg, raw, idx, n_levels, ctx=None):
    """createImgPyramid of the raw frames of pairs idx (slot-sized: the truncating mean keeps every camera's region)."""
    ref = pkg.api.createImgPyramid(raw[0][idx], n_levels, ctx)
    cur = pkg.api.createImgPyramid(raw[1][idx], n_levels, ctx)
    return ref, cur


def per_model(pkg, synth, cams, cop, data, raw, hi, lo, ctx=None):
    """Pair b's outputs from its model's per-model call: the raw multicam call on the lens pairs, the ATAN multicam call
    on createImgPyramid of the ATAN pairs' raw frames."""
    want = {}
    atan = np.array([is_atan(pkg, cams[k]) for k in cop])
    for mask in (~atan, atan):
        idx = np.flatnonzero(mask)
        if not len(idx):
            continue
        table, k = sub_table(cams, cop, idx)
        sub = synth.take_pairs(data, idx)
        al = pkg.SparseImgAlign(hi, lo, 30, ctx=ctx)
        if mask is atan:
            ref, cur = atan_levels(pkg, raw, idx, hi + 1, ctx)
            sub.ref_pyr = {l: ref[l] for l in range(lo, hi + 1)}
            sub.cur_pyr = {l: cur[l] for l in range(lo, hi + 1)}
            got = al.run(sub, camera=table, cam_of_pair=k)
        else:
            got = al.run_raw(table, (raw[0][idx], raw[1][idx]), sub, cam_of_pair=k)
        for f in ALIGN_FIELDS:
            want.setdefault(f, np.zeros((data.batch,) + getattr(got, f).shape[1:], getattr(got, f).dtype))[idx] = getattr(got, f)
    return want


def assert_rows(got, want, what):
    for f in ALIGN_FIELDS:
        np.testing.assert_array_equal(getattr(got, f).view(np.uint8), want[f].view(np.uint8), err_msg=f"{what} {f}")


@pytest.fixture(autouse=True)
def _host_model_is_clean(pkg):
    yield
    if MODEL:
        lib = C.CDLL(os.environ["PLSVO_LIB"])
        lib.fake_cuda_errors.restype = C.c_char_p
        err = lib.fake_cuda_errors().decode()
        lib.fake_cuda_clear_errors()
        assert not err, err


@pytest.fixture(scope="module")
def oracle_atan(abi):
    import oracle_atan

    oracle_atan.build()
    oracle_atan.load(abi)
    return oracle_atan


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_library_exports_the_raw_any_camera_calls(pkg):
    syms = subprocess.check_output(["nm", "-D", "--defined-only", pkg.abi.LIB_PATH], text=True)
    names = {n for n, _, _ in pkg.abi.ABI_SYMBOLS}
    for n in ("plsvo_align_raw_any_camera_batch_run", "plsvo_track_raw_any_camera_batch_run"):
        assert re.search(rf"\b{n}\b", syms), n
        assert n in names, n


@pytest.mark.parametrize("struct,fields", [
    ("plsvo_raw_camera", ("model", "reserved", "pinhole", "atan")),
    ("plsvo_raw_any_camera_frames", ("n_cams", "reserved", "cams", "cam_of_pair", "ref_raw", "cur_raw", "pitch", "stride"))])
def test_ctypes_layout_matches_the_header(pkg, tmp_path, struct, fields):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "plsvo_b200.h"\nint main(void){printf("%zu'
                   + " %zu" * len(fields) + f'\\n", sizeof({struct})'
                   + "".join(f", offsetof({struct}, {f})" for f in fields) + ");return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    R = pkg.abi.RawCamera if struct == "plsvo_raw_camera" else pkg.abi.RawAnyCameraFrames
    assert got == [C.sizeof(R)] + [getattr(R, f).offset for f in fields]


def test_python_dispatch_and_tables(pkg, synth):
    api, abi = pkg.api, pkg.abi
    cams = stock(pkg)
    data = features(synth, EUROC, 3, seed=1)
    raw = (raw_frames(EUROC, 3, seed=2), raw_frames(EUROC, 3, seed=3))
    # an ATANCamera in the sequence takes the any-camera calls; PinholeCamera only keeps the raw multicam calls
    assert api._raw_any_camera(cams, [0, 1, 0]) and not api._raw_any_camera(cams[:1], [0, 0, 0])
    assert not api._raw_any_camera(cams, None) and not api._raw_any_camera(cams[1], [0, 0, 0])
    rf, ab, keep = api._raw_any_camera_args(cams, raw, data, np.array([1, 0, 1]))
    assert isinstance(rf, abi.RawAnyCameraFrames) and rf.n_cams == 2 and [rf.cam_of_pair[b] for b in range(3)] == [1, 0, 1]
    assert (rf.cams[0].model, rf.cams[1].model) == (abi.CAMERA_PINHOLE, abi.CAMERA_ATAN)
    assert rf.cams[0].pinhole.d[0] == params(EUROC)[6] and rf.cams[1].atan.d0 == STOCK_ATAN[6]
    assert rf.pitch == 752 and rf.stride == 752 * 480 and ab.flags == 0 and not any(ab.ref_img[l] for l in range(abi.MAX_LEVELS))
    rf, ab, keep = api._raw_call_args(cams[:1], raw, data, np.array([0, 0, 0]))
    assert isinstance(rf, abi.RawMulticamFrames)
    # anything else in the sequence is a PlsvoError, never a ctypes TypeError
    for bad in ([cams[0], cams[1], synth.VGA], [cams[1], 3]):
        assert api._raw_any_camera(bad, [0, 1, 0])
        with pytest.raises(api.PlsvoError, match="sequence of PinholeCamera and ATANCamera"):
            api._raw_any_camera_args(bad, raw, data, [0, 1, 0])
    with pytest.raises(api.PlsvoError, match="sequence of PinholeCamera"):
        api._raw_call_args([cams[0], synth.VGA], raw, data, [0, 1, 0])
    with pytest.raises(api.PlsvoError, match=r"shape \[3\]"):
        api._raw_any_camera_args(cams, raw, data, [0, 1])
    with pytest.raises(api.PlsvoError, match="frame chains are not supported"):
        api._raw_any_camera_args(cams, raw_frames(EUROC, 4, seed=3), data, [0, 1, 0])
    # the raw table as plsvo_match_camera records: a lens becomes the undistorted pinhole of its fx..cy
    m = abi.raw_to_match_cameras(abi.make_raw_cameras(cams))
    want = abi.make_match_cameras([undistorted(synth, cams[0]), cams[1]])
    assert bytes(m) == bytes(want)


def test_raw_any_camera_generator(pkg, synth):
    import torch

    cams = fleet(pkg)[4:]  # 641x479 lens, 641x479 ATAN d0 = 0, 320x240 copy lens, 320x240 ATAN
    cop = np.array([3, 0, 1, 3, 2])
    slot = synth.Camera(752, 480, 1.0, 1.0, 0.0, 0.0)
    data, (ref, cur), parts, groups = synth.make_raw_any_camera_batch(cams, cop, slot=slot, fill=255, n_pts=8, n_segs=2, seed=1)
    assert (data.cam.width, data.cam.height) == (752, 480) and ref.shape == cur.shape == (5, 480, 752)
    assert [g.tolist() for g in groups] == [[1], [2], [4], [0, 3]]
    assert parts[0].cam == undistorted(synth, cams[0]) and parts[3].cam.fx == cams[3].fx_
    # a lens pair's raw frame is the lens's render, an ATAN pair's the level 0 of its own pyramid
    s = cams[0].struct
    want = synth.render_distorted(synth.Scene(), parts[0].cam, tuple(s.d), torch.tensor(parts[0].T_cur_w_gt)).numpy()
    np.testing.assert_array_equal(cur[1, :479, :641], want[0])
    for l in parts[3].ref_pyr:
        np.testing.assert_array_equal(synth.build_pyramid(torch.tensor(ref[[0, 3], :240, :320]), l + 1)[l].numpy(), parts[3].ref_pyr[l])
    assert (ref[1, 479:] == 255).all() and (ref[0, :, 320:] == 255).all()
    np.testing.assert_allclose(parts[1].pt_f[0], cams[1].cam2world(parts[1].pt_px[0]), rtol=0, atol=1e-12)
    al, po, raw, parts, po_parts, groups = synth.make_raw_any_camera_batch(cams[:2], [1, 0, 1], poseopt=True, n_pts=8, n_segs=2,
                                                                            seed=2)
    assert po_parts[0].fx == abs(cams[0].struct.fx) and po_parts[1].fx == cams[1].fx_ and po.batch == 3
    assert raw[0].shape == (3, 479, 641)


@pytest.fixture(scope="module")
def raw_any_hostmodel(tmp_path_factory):
    return _build_model(str(tmp_path_factory.mktemp("hostmodel") / "libplsvo_hostmodel_raw_any_camera.so"))


# fake_mixed_sizes.cpp's multicam alignment and pose-optimiser launchers give way to those of fake_any_camera.cpp and
# fake_atan_multicam.cpp: only its fused rectify / pyramid kernel (frames of their own size in the slot) is linked in
MIXED_SIZES_RENAMES = ("align_multicam_kernel_static_smem", "align_multicam_kernel_prepare", "align_multicam_kernel_launch",
                       "poseopt_multicam_kernel_launch")


def _build_model(out, abi_source=ABI_SOURCE):
    """The stock model kernels, fake_undistort.cpp and fake_raw_pyramid.cpp (the map and one-camera fused kernels),
    fake_mixed_sizes.cpp's fused multicam kernel, fake_atan_multicam.cpp and fake_any_camera.cpp."""
    spec = importlib.util.spec_from_file_location("plsvo_hostmodel_build", os.path.join(HERE, "hostmodel", "build.py"))
    hm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(hm)
    cxx = ["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-Wall", "-Wno-unused-function", "-I" + hm.cuda_include(),
           "-I" + os.path.join(ROOT, "pl-svo_b200", "csrc")]
    mixed = out + ".mixed_sizes.o"
    subprocess.run(cxx + [f"-D{n}=mixed_sizes_unused_{n}" for n in MIXED_SIZES_RENAMES]
                   + ["-c", "-x", "c++", os.path.join(HERE, "hostmodel", "fake_mixed_sizes.cpp"), "-o", mixed], check=True)
    sources = [abi_source] + hm.SOURCES[1:] + [os.path.join(HERE, "hostmodel", f) for f in (
        "fake_undistort.cpp", "fake_raw_pyramid.cpp", "fake_atan_multicam.cpp", "fake_any_camera.cpp")]
    subprocess.run(cxx + ["-shared", "-x", "c++", *sources, "-x", "none", mixed, "-o", out, "-lpthread", "-ldl", "-Wl,-Bsymbolic"],
                   check=True)
    return out


def _run_here(lib, mode, k, oracle_lib=None):
    env = dict(os.environ, PLSVO_LIB=lib, PLSVO_FAKE_CUDA=mode)
    for name in [n for n in env if n.startswith("PLSVO_") and n not in ("PLSVO_LIB", "PLSVO_FAKE_CUDA")]:
        del env[name]
    if oracle_lib:
        env["PLSVO_FAKE_ORACLE"] = oracle_lib
    return subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-p", "no:cacheprovider",
                           "-k", k], env=env, capture_output=True, text=True, timeout=3000)


@pytest.mark.parametrize("mode", ["lazy", "eager"])
def test_gpu_tests_of_this_file_against_the_host_model(oracle, raw_any_hostmodel, mode):
    """The GPU tests below on the unchanged host code of plsvo_abi.cu with the model CUDA runtime: the model rectifies and
    half-samples for real, checks every access, the stream order and that a rejected call queued nothing, and digests
    each pair's own region at its own size through its model.  The oracle tests and the variant sweep need real kernels
    and are deselected."""
    p = _run_here(raw_any_hostmodel, mode, "not oracle and not every_variant")
    assert p.returncode == 0 and " skipped" not in p.stdout and " passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


FAULTS = {
    # an ATAN frame rectified with the map of the table's first distorted lens instead of copied
    "atan_frame_gets_a_lens_map": (
        "    return slot < 0 ? n_maps : slot;\n",
        "    return slot < 0 ? (n_maps && !is_lens(in, in.cam_of_pair[f < B ? f : f - B]) ? 0 : n_maps) : slot;\n",
        "fleet and full and 4_2"),
    # every pair given the model tag of cams[0] (a lens): the ATAN pairs run through the pinhole model
    "every_pair_gets_cams0_tag": (
        "    c->h_cam_models[i] = cams[k].model;\n",
        "    c->h_cam_models[i] = cams[0].model;\n",
        "fleet and full and 4_2"),
    # an ATAN frame's pose optimiser given the normalised fx instead of errorMultiplier2() = fx_
    "atan_track_gets_normalised_fx": (
        "      c->h_po_fx[b] = fabs(c->h_mc_cams[b].fx);\n",
        "      c->h_po_fx[b] = in.table && in.table[in.cam_of_pair[b]].model == PLSVO_CAMERA_ATAN ? in.table[in.cam_of_pair[b]].atan.fx\n"
        "                                                                                   : fabs(c->h_mc_cams[b].fx);\n",
        "track"),
}


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_model_notices_seeded_fault(oracle, oracle_atan, tmp_path, fault):
    old, new, k = FAULTS[fault]
    src = open(ABI_SOURCE).read()
    assert src.count(old) == 1, f"the line this fault is seeded into has changed: {old!r}"
    mutated = tmp_path / "plsvo_abi.cu"
    mutated.write_text(src.replace(old, new))
    lib = _build_model(str(tmp_path / "libplsvo_hostmodel_fault.so"), str(mutated))
    p = _run_here(lib, "lazy", k + " and not oracle", _oracle_lib(oracle, oracle_atan))
    assert " passed" in p.stdout or " failed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]
    assert p.returncode != 0 and " failed" in p.stdout, f"{fault}: every test still passes — the model is blind to it"


def test_unmutated_track_and_fleet_pass_on_the_oracle_model(oracle, oracle_atan, raw_any_hostmodel):
    """The control of the seeded faults: the same selections on the unmutated host code pass."""
    p = _run_here(raw_any_hostmodel, "lazy", "(track or (fleet and full and 4_2)) and not oracle", _oracle_lib(oracle, oracle_atan))
    assert p.returncode == 0 and " passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("lv", ["4_2", "6_4"])
@pytest.mark.parametrize("bearings", ["full", "lean"])
@pytest.mark.parametrize("B", [37, BIG])
@pytest.mark.parametrize("K", [2, 8])
def test_gpu_fleet_equals_per_model_calls(pkg, synth, gen_device, K, B, bearings, lv, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2" if B <= 132 else "128,4")
    hi, lo = map(int, lv.split("_"))
    cams, cop, data, raw = fleet_batch(K, B, seed=300 + K, device=gen_device)
    groups = [np.flatnonzero(cop == k) for k in range(len(cams))]
    ragged(data, seed=B + K, empty=(int(groups[-1][0]),))  # ragged counts, masks, and an empty pair
    if bearings == "lean":
        lean(data)
    got = pkg.SparseImgAlign(hi, lo, 30).run_raw(cams, raw, data, cam_of_pair=cop)
    assert_rows(got, per_model(pkg, synth, cams, cop, data, raw, hi, lo), f"K={K} B={B}")
    if not MODEL:
        assert all((got.n_tracked[idx] > 0).any() for idx in groups)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["lens", "atan"])
def test_gpu_one_model_table_equals_its_call(pkg, synth, gen_device, which, monkeypatch):
    """A table of one model (plus an unused camera of the other, which makes it an any-camera call) equals the raw
    multicam call, or the ATAN multicam call, on the whole batch."""
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    cams, cop, data, raw = fleet_batch(8, 37, seed=310, device=gen_device)
    keep = np.flatnonzero(np.array([is_atan(pkg, cams[k]) == (which == "atan") for k in cop]))
    table, k = sub_table(cams, cop, keep)
    data = synth.take_pairs(data, keep)
    raw = (raw[0][keep], raw[1][keep])
    other = pkg.ATANCamera(*STOCK_ATAN) if which == "lens" else pkg.PinholeCamera(*params(EUROC))
    got = pkg.SparseImgAlign(4, 2, 30).run_raw(table + [other], raw, data, cam_of_pair=k)
    if which == "lens":
        want = pkg.SparseImgAlign(4, 2, 30).run_raw(table, raw, data, cam_of_pair=k)
    else:
        ref, cur = atan_levels(pkg, raw, np.arange(len(keep)), 5)
        data.ref_pyr, data.cur_pyr = {l: ref[l] for l in (2, 3, 4)}, {l: cur[l] for l in (2, 3, 4)}
        want = pkg.SparseImgAlign(4, 2, 30).run(data, camera=table, cam_of_pair=k)
    assert_same(got, want, ALIGN_FIELDS)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 8])
def test_gpu_rect_out_and_the_any_camera_call(pkg, abi, synth, gen_device, K, monkeypatch):
    """rect_out holds undistortImage (lens) or createImgPyramid (ATAN) of every frame in its region and 0 outside; its
    levels 0..6, fed to plsvo_align_any_camera_batch_run with the table's plsvo_match_camera records, give the same
    bytes as the raw call."""
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    cams, cop, data, raw = fleet_batch(K, 37, seed=320 + K, device=gen_device)
    got, rect = pkg.SparseImgAlign(6, 4, 30).run_raw(cams, raw, data, cam_of_pair=cop, rect_levels=range(7))
    B = data.batch
    for k, cam in enumerate(cams):
        idx = np.flatnonzero(cop == k)
        frames = np.concatenate([raw[0][idx], raw[1][idx]])[:, : cam.height, : cam.width]
        want = (pkg.api.createImgPyramid(frames, 7) if is_atan(pkg, cam) else cam.undistortImage(frames, 7))
        at = np.concatenate([idx, B + idx])
        for l in range(7):
            h, w = cam.height >> l, cam.width >> l
            np.testing.assert_array_equal(rect[l][at, :h, :w], want[l], err_msg=f"camera {k} level {l}")
            assert not rect[l][at, h:].any() and not rect[l][at, :, w:].any(), f"camera {k} level {l} padding"
    d = synth.take_pairs(data, np.arange(B))
    d.ref_pyr = {l: np.ascontiguousarray(rect[l][:B]) for l in range(7)}
    d.cur_pyr = {l: np.ascontiguousarray(rect[l][B:]) for l in range(7)}
    ctx = pkg.Context(0)
    table = abi.raw_to_match_cameras(abi.make_raw_cameras(cams))
    ab, keep = abi.make_align_batch(d)
    out = abi.AlignOut(B, d.n_segs)
    rc = ctx.lib.plsvo_align_any_camera_batch_run(ctx.handle, table, len(cams), cop.ctypes.data_as(C.POINTER(C.c_int32)),
                                                   C.byref(ab), C.byref(abi.align_params(6, 4, 30)), C.byref(out.struct))
    assert rc == abi.OK, ctx.lib.plsvo_last_error(ctx.handle).decode()
    assert_same(out, got, ALIGN_FIELDS)
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_gpu_every_variant(pkg, synth, gen_device, variant, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", variant)
    cams, cop, data, raw = fleet_batch(2, 37, seed=330, device=gen_device, n_pts=100, n_segs=24)
    got = pkg.SparseImgAlign(4, 2, 30).run_raw(cams, raw, data, cam_of_pair=cop)
    assert_rows(got, per_model(pkg, synth, cams, cop, data, raw, 4, 2), variant)


@pytest.mark.gpu
@pytest.mark.parametrize("n_iter_ref", [None, 3])
@pytest.mark.parametrize("chained", [True, False])
def test_gpu_track_equals_per_model_track(pkg, synth, gen_device, chained, n_iter_ref, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    cams, cop, data, raw, po = fleet_batch(8, 16 if MODEL else 40, seed=340, device=gen_device, poseopt=True)
    fields = ("T_f_w", "num_obs_pt", "status") if MODEL and not ORACLE_MODEL else PO_FIELDS
    got_a, got_p = pkg.api.track_raw(cams, raw, data, po, po_n_iter_ref=n_iter_ref, chained=chained, cam_of_pair=cop)
    atan = np.array([is_atan(pkg, cams[k]) for k in cop])
    for mask in (~atan, atan):
        idx = np.flatnonzero(mask)
        table, k = sub_table(cams, cop, idx)
        sub, po_sub = synth.take_pairs(data, idx), synth.take_pairs(po, idx)
        if mask is atan:
            ref, cur = atan_levels(pkg, raw, idx, 5)
            sub.ref_pyr, sub.cur_pyr = {l: ref[l] for l in (2, 3, 4)}, {l: cur[l] for l in (2, 3, 4)}
            want_a, want_p = pkg.api.track(sub, po_sub, po_n_iter_ref=n_iter_ref, chained=chained, camera=table, cam_of_pair=k)
        else:
            want_a, want_p = pkg.api.track_raw(table, (raw[0][idx], raw[1][idx]), sub, po_sub, po_n_iter_ref=n_iter_ref,
                                               chained=chained, cam_of_pair=k)
        what = "atan" if mask is atan else "lens"
        assert_same(rows(got_a, idx), want_a, ALIGN_FIELDS, what=what)
        assert_same(rows(got_p, idx, fields), want_p, fields, what=what)


@pytest.mark.gpu
def test_gpu_padding_does_not_matter(pkg, synth, gen_device, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    outs, raws = [], []
    for fill in (0, 255, (7,)):  # (7,): random bytes
        cams, cop, data, raw = fleet_batch(8, 37, seed=350, device=gen_device, fill=fill)
        raws.append(raw[0])
        outs.append(pkg.SparseImgAlign(4, 2, 30).run_raw(cams, raw, data, cam_of_pair=cop, rect_levels=(0, 2, 4)))
    assert not np.array_equal(raws[0], raws[1]) and not np.array_equal(raws[0], raws[2])
    for o, levels in outs[1:]:
        assert_same(o, outs[0][0], ALIGN_FIELDS)
        for l in levels:
            np.testing.assert_array_equal(levels[l], outs[0][1][l])


@pytest.mark.gpu
def test_gpu_map_cache(pkg, synth, monkeypatch):
    """ATAN cameras build no map; a repeat builds nothing; the raw multicam calls share the cache and its rule (after a
    call it holds exactly the maps of the distorted lenses that call referenced)."""
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    ctx = pkg.api.Context(0)
    B = 6
    data = features(synth, EUROC, B, seed=51, n_pts=40, n_segs=8)
    raw = (raw_frames(EUROC, B, seed=52), raw_frames(EUROC, B, seed=53))
    lens_a, atan = stock(pkg)
    p = list(params(EUROC))
    p[6] *= 1.01
    lens_b = pkg.PinholeCamera(*p)
    copy_lens = pkg.PinholeCamera(*params(EUROC)[:6])
    al = pkg.SparseImgAlign(4, 2, 30, ctx=ctx)
    cop = np.array([0, 1, 1, 0, 1, 0], np.int32)

    def run(cams, any_camera=True):
        n0 = ctx.launch_count()
        out = al.run_raw(cams, raw, data, cam_of_pair=cop if any_camera or len(cams) > 1 else np.zeros(B, np.int32))
        return out, ctx.last_map_build_ms(), ctx.launch_count() - n0

    first, ms, n = run([lens_a, atan])
    assert ms is not None and n == 3  # one map, the fused kernel, the alignment
    again, ms, n = run([lens_a, atan])
    assert ms is None and n == 2
    assert_same(again, first, ALIGN_FIELDS)
    _, ms, n = run([atan, pkg.ATANCamera(752, 480, 0.6, 0.8, 0.5, 0.5, 0.0)])  # ATAN only: no map, and the cache empties
    assert ms is None and n == 2
    _, ms, n = run([copy_lens, atan])  # a d0 = 0 lens copies its frames: no map either
    assert ms is None and n == 2
    _, ms, n = run([lens_a, atan])
    assert ms is not None and n == 3
    # interleaved with raw multicam calls: one cache, one rule
    _, ms, n = run([lens_a], any_camera=False)
    assert ms is None and n == 2
    _, ms, n = run([lens_b, lens_a])
    assert ms is not None and n == 3
    _, ms, n = run([lens_b, atan])
    assert ms is None and n == 2
    _, ms, n = run([lens_a, lens_b])
    assert ms is not None and n == 3
    ctx.close()


@pytest.mark.gpu
def test_gpu_against_the_oracles(pkg, abi, synth, oracle, oracle_atan, gen_device):
    """Each lens group against oracle undistortion + the pinhole oracle, each ATAN group against the ATAN oracle, at
    tests/test_gpu_atan.py's tolerance; the aligned poses end closer to ground truth than the initial guess."""
    import undistort_oracle
    from test_gpu_atan import compare

    undistort_oracle.build()
    cams = fleet(pkg)
    cop = cop_of(interleave(len(cams), 32, 360), 32)
    data, raw, parts, groups = synth.make_raw_any_camera_batch(cams, cop, slot=slot_of(synth, cams), n_pts=200, n_segs=50,
                                                               seed=360, device=gen_device)
    got = pkg.SparseImgAlign(4, 2, 30).run_raw(cams, raw, data, cam_of_pair=cop)
    for k, cam in enumerate(cams):
        idx = np.flatnonzero(cop == k)
        if is_atan(pkg, cam):
            want = oracle_atan.align(abi, cam, crop(synth, data, idx, slot_cam(synth, cam)), n_threads=8)
        else:
            sub = synth.take_pairs(data, idx)
            sub.cam = undistorted(synth, cam)
            frames = np.ascontiguousarray(np.concatenate([raw[0][idx], raw[1][idx]])[:, : cam.height, : cam.width])
            r = undistort_oracle.undistort(abi, cam.struct, frames, 5)
            n = len(idx)
            sub.ref_pyr = {l: np.ascontiguousarray(r[l][:n]) for l in range(2, 5)}
            sub.cur_pyr = {l: np.ascontiguousarray(r[l][n:]) for l in range(2, 5)}
            want = oracle.align(abi, sub, abi.align_params(4, 2, 30), n_threads=8)
        compare(synth, rows(got, idx), want, f"camera {k} {cam.width}x{cam.height}")
    a0, t0 = synth.pose_error(data.T_cur_w, data.T_cur_w_gt)
    a1, t1 = synth.pose_error(got.T_cur_w, data.T_cur_w_gt)
    assert np.median(a1) < 0.25 * np.median(a0) and np.median(t1) < 0.25 * np.median(t0), (a0, a1, t0, t1)


@pytest.mark.gpu
def test_gpu_malformed_calls_queue_nothing(pkg, abi, synth):
    """Each malformed call returns PLSVO_ERR_INVALID with its message before anything is queued (against the host model:
    no stream operation ran or is pending); a valid call on the same context then succeeds."""
    ctx = pkg.Context(0)
    lib = ctx.lib
    model = C.CDLL(os.environ["PLSVO_LIB"]) if MODEL else None
    if model:
        model.fake_cuda_ops_run.restype = C.c_ulonglong
    B = 3
    data = features(synth, EUROC, B, seed=61, n_pts=16, n_segs=4)
    raw = (raw_frames(EUROC, B, seed=62), raw_frames(EUROC, B, seed=63))
    po = synth.make_poseopt_batch(cam=synth.EUROC, batch=B, n_pts=16, n_segs=4, seed=64)
    ab, keep_a = pkg.api._image_free_batch(data, False)
    pb, keep_p = abi.make_poseopt_batch(po)
    ao, pout = abi.AlignOut(B, 4), abi.PoseOptOut(B, 16, 4)
    cams = stock(pkg) + [pkg.ATANCamera(320, 240, 0.68, 0.88, 0.52, 0.48, 0.3)]
    img = np.zeros((B, 480, 752), np.uint8)

    def table(k=None, model=None, **kw):
        arr = abi.make_raw_cameras(cams)
        if k is not None:
            if model is not None:
                arr[k].model = model
            rec = arr[k].pinhole if arr[k].model == abi.CAMERA_PINHOLE else arr[k].atan
            for f, v in kw.items():
                if f.startswith("d") and f[1:].isdigit() and arr[k].model == abi.CAMERA_PINHOLE:
                    rec.d[int(f[1:])] = v
                else:
                    setattr(rec, f, v)
        return arr

    def run(arr=None, n_cams=3, cop=(0, 1, 0), hi=4, track=False, flags=0, po_batch=B, null_cams=False, image=False):
        arr = table() if arr is None else arr
        rf, keep_r = abi.make_raw_any_camera_frames(arr, np.zeros(B, np.int32), raw, B, slot=data.cam)
        rf.n_cams = n_cams
        cop_arr = None if cop is None else np.ascontiguousarray(cop, np.int32)
        rf.cam_of_pair = None if cop is None else cop_arr.ctypes.data_as(C.POINTER(C.c_int32))
        if null_cams:
            rf.cams = C.cast(None, C.POINTER(abi.RawCamera))
        ab.flags, pb.batch = flags, po_batch
        ab.ref_img[0] = img.ctypes.data_as(C.POINTER(C.c_uint8)) if image else None
        ops = model.fake_cuda_ops_run() if model else 0
        launches = ctx.launch_count()
        ap = abi.align_params(hi, 2, 30)
        if track:
            rc = lib.plsvo_track_raw_any_camera_batch_run(ctx.handle, C.byref(rf), C.byref(ab), C.byref(ap), C.byref(pb),
                                                          C.byref(abi.poseopt_params()), C.byref(ao.struct), C.byref(pout.struct),
                                                          None)
        else:
            rc = lib.plsvo_align_raw_any_camera_batch_run(ctx.handle, C.byref(rf), C.byref(ab), C.byref(ap), C.byref(ao.struct), None)
        if rc != abi.OK:
            assert ctx.launch_count() == launches, "a rejected call launched a kernel"
            if model:
                assert model.fake_cuda_pending_ops() == 0 and model.fake_cuda_ops_run() == ops, "a rejected call queued work"
        ab.flags, pb.batch, ab.ref_img[0] = 0, B, None
        return rc, lib.plsvo_last_error(ctx.handle).decode()

    nan = float("nan")
    NULLS = "n_cams must be at least 1, cams and cam_of_pair non-NULL"
    for kw, msg in (({"null_cams": True}, NULLS),
                    ({"cop": None}, NULLS),
                    ({"cop": None, "track": True}, NULLS),
                    ({"n_cams": 0}, NULLS),
                    ({"cop": (0, 3, 0)}, "cam_of_pair[1] = 3 is outside [0, 3)"),
                    ({"cop": (0, 1, -1), "track": True}, "cam_of_pair[2] = -1 is outside [0, 3)"),
                    ({"arr": table(1, model=7)}, "cams[1].model 7 is neither"),
                    ({"arr": table(0, fx=nan)}, "cams[0]: a parameter is not finite in float"),
                    ({"arr": table(0, d1=1e300)}, "cams[0]: a parameter is not finite in float"),
                    ({"arr": table(0, fy=0.0)}, "cams[0]: fx and fy must be non-zero"),
                    ({"arr": table(0, width=753)}, "cams[0] is 753x480"),
                    ({"arr": table(1, d0=nan)}, "cams[1] (ATAN) has a non-finite parameter"),
                    ({"arr": table(1, fx=-0.5)}, "cams[1] (ATAN) fx and fy must be positive"),
                    ({"arr": table(1, height=481)}, "cams[1] is 752x481"),
                    ({"arr": table(2, width=0), "track": True}, "cams[2] is 0x240"),  # unused: checked all the same
                    ({"arr": table(2, fy=nan)}, "cams[2] (ATAN) has a non-finite parameter"),
                    ({"arr": table(2, width=40, height=30), "hi": 6}, "cams[2] is 40x30: pyramid level 5 smaller than one pixel"),
                    ({"flags": abi.ALIGN_FRAME_CHAIN}, "PLSVO_ALIGN_FRAME_CHAIN is not supported"),
                    ({"image": True}, "image pointers in the alignment batch"),
                    ({"hi": 7}, "max_level > 6"),
                    ({"track": True, "po_batch": 2}, "batches differ in size")):
        rc, err = run(**kw)
        assert rc == abi.ERR_INVALID and msg in err, (kw, msg, err)
    for kw in ({}, {"track": True}):
        rc, err = run(**kw)
        assert rc == abi.OK, (kw, err)
    ctx.close()
