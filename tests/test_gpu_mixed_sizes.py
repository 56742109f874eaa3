"""Frame pairs of different image sizes in one multicam batch: batch->cam's size is the slot, and pair b's frames are
cams[b].width x cams[b].height in the top-left corner of their slots (plsvo_align_multicam_batch_run,
plsvo_track_multicam_batch_run, and the raw forms with cams[cam_of_pair[b]]).  Pair b's outputs must be byte-identical
to the multicam call on its size group at that size and to the one-camera call with its camera, at the same kernel
variant; the padding of the slots must not matter.

CPU: the Python argument handling and synth.merge_sizes, this file's GPU tests against the host model of the C ABI
(tests/hostmodel/fake_mixed_sizes.cpp: the model's multicam alignment digests each pair's own region, its rectification
works at each frame's camera size), and two faults seeded into plsvo_abi.cu that the model must notice."""
import ctypes as C
import dataclasses
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_multicam import ALIGN_FIELDS, PO_FIELDS, assert_same, lean, ragged
from test_raw_track import COPY, EUROC, ODD, camera, features, params, raw_frames

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ABI_SOURCE = os.path.join(ROOT, "pl-svo_b200", "csrc", "plsvo_abi.cu")
MODEL = bool(os.environ.get("PLSVO_FAKE_CUDA"))
BIG = 16 if MODEL else 1024  # the host model renders and rectifies on the CPU
VARIANTS = ["64,8", "96,7", "96,5", "128,5", "128,4", "160,3", "192,2", "256,2"]
RAW_LENSES = (EUROC, "vga_strong_barrel_k3", "vga_pincushion", COPY, ODD)


def cameras_of(synth):
    """VGA and TUM freiburg1 (one size, two calibrations), EuRoC, ODD, QVGA and a KITTI-like wide, short frame."""
    wide = synth.Camera(1241, 376, 718.856, 718.856, 607.1928, 185.2157)
    return (synth.VGA, synth.TUM_FR1, synth.EUROC, synth.ODD, synth.QVGA, wide)


@pytest.fixture(autouse=True)
def _host_model_is_clean(pkg):
    yield
    if MODEL:
        lib = C.CDLL(os.environ["PLSVO_LIB"])
        lib.fake_cuda_errors.restype = C.c_char_p
        err = lib.fake_cuda_errors().decode()
        lib.fake_cuda_clear_errors()
        assert not err, err


def interleave(n_groups, B, seed):
    """Group of every pair: every group present, in no particular order."""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, n_groups, B)
    g[:n_groups] = rng.permutation(n_groups)
    return [np.flatnonzero(g == k) for k in range(n_groups)]


def mixed(synth, cams, B, seed, device, fill=0, n_pts=150, n_segs=40):
    """One batch of B interleaved pairs of the cameras `cams` (slot: the largest width and height), with the per-pair
    intrinsics [B, 4] and sizes [B, 2]; and the groups (pair indices of every camera)."""
    groups = interleave(len(cams), B, seed)
    parts = [synth.make_align_batch(cam=c, batch=len(idx), n_pts=n_pts, n_segs=n_segs, seed=seed + 7 * k, device=device)
             for k, (c, idx) in enumerate(zip(cams, groups))]
    data, sizes = synth.merge_sizes(parts, groups, fill=fill)
    k = np.zeros((B, 4))
    for c, idx in zip(cams, groups):
        k[idx] = (c.fx, c.fy, c.cx, c.cy)
    return data, k, sizes, groups


def crop(synth, data, idx, cam):
    """Pairs idx of a slot batch as a batch of their own at `cam`'s size (its levels cut out of the slots)."""
    sub = synth.take_pairs(data, idx)
    sub.cam = cam
    for pyr in (sub.ref_pyr, sub.cur_pyr):
        for l in list(pyr):
            pyr[l] = np.ascontiguousarray(pyr[l][:, : cam.height >> l, : cam.width >> l])
    return sub


def rows(out, idx, fields=ALIGN_FIELDS):
    class R:
        pass

    r = R()
    for f in fields:
        setattr(r, f, getattr(out, f)[idx])
    return r


def per_size_and_per_camera(pkg, synth, data, k, sizes, cams, groups, hi=4, lo=2):
    """Pair b's outputs (a) from the multicam call on its size group at that size, (b) from the one-camera call with
    batch->cam = its camera, scattered to batch order."""
    by_size, by_cam = {}, {}
    for size in {(c.width, c.height) for c in cams}:
        idx = np.flatnonzero((sizes == size).all(1))
        cam = next(c for c in cams if (c.width, c.height) == size)
        got = pkg.SparseImgAlign(hi, lo, 30).run(crop(synth, data, idx, cam), cameras=k[idx])
        for f in ALIGN_FIELDS:
            by_size.setdefault(f, np.zeros((data.batch,) + getattr(got, f).shape[1:], getattr(got, f).dtype))[idx] = getattr(got, f)
    for cam, idx in zip(cams, groups):
        got = pkg.SparseImgAlign(hi, lo, 30).run(crop(synth, data, idx, cam))
        for f in ALIGN_FIELDS:
            by_cam.setdefault(f, np.zeros((data.batch,) + getattr(got, f).shape[1:], getattr(got, f).dtype))[idx] = getattr(got, f)
    return by_size, by_cam


def assert_rows(got, want, what):
    for f in ALIGN_FIELDS:
        np.testing.assert_array_equal(getattr(got, f).view(np.uint8), want[f].view(np.uint8), err_msg=f"{what} {f}")


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_merge_sizes_and_python_arguments(pkg, synth):
    a = synth.make_align_batch(cam=synth.QVGA, batch=2, n_pts=8, n_segs=2, seed=1)
    b = synth.make_align_batch(cam=synth.ODD, batch=1, n_pts=8, n_segs=2, seed=2)
    rng = np.random.default_rng(0)
    raws = [(np.full((2, 240, 320), 7, np.uint8),) * 2, (np.full((1, 479, 641), 9, np.uint8),) * 2]
    m, sizes, (ref, cur) = synth.merge_sizes([a, b], [[0, 2], [1]], fill=255, raws=raws)
    assert (m.cam.width, m.cam.height) == (641, 479) and sizes.tolist() == [[320, 240], [641, 479], [320, 240]]
    for l in m.ref_pyr:
        assert m.ref_pyr[l].shape == (3, 479 >> l, 641 >> l)
        np.testing.assert_array_equal(m.ref_pyr[l][2, : 240 >> l, : 320 >> l], a.ref_pyr[l][1])
        assert (m.ref_pyr[l][0, 240 >> l:] == 255).all() and (m.ref_pyr[l][0, :, 320 >> l:] == 255).all()
        np.testing.assert_array_equal(m.cur_pyr[l][1], b.cur_pyr[l][0])
    np.testing.assert_array_equal(m.pt_px[[0, 2]], a.pt_px)
    assert ref.shape == (3, 479, 641) and (ref[1] == 9).all() and (ref[0, :240, :320] == 7).all() and (ref[0, 240:] == 255).all()
    r = synth.merge_sizes([a, b], [[0, 2], [1]], fill=rng)[0]
    l = min(r.ref_pyr)
    assert not (r.ref_pyr[l][0, 240 >> l:] == r.ref_pyr[l][2, 240 >> l:]).all()
    with pytest.raises(ValueError, match="fit inside the slot"):
        synth.merge_sizes([a, b], [[0, 2], [1]], slot=synth.QVGA)
    cams = pkg.abi.make_cameras(np.ones((3, 4)), m.cam, 3, sizes)
    assert [(cams[i].width, cams[i].height) for i in range(3)] == [(320, 240), (641, 479), (320, 240)]
    assert (pkg.abi.make_cameras(np.ones((3, 4)), m.cam, 3)[1].width, pkg.abi.make_cameras(np.ones((3, 4)), m.cam, 3)[1].height) == (641, 479)
    with pytest.raises(pkg.api.PlsvoError, match="sizes must be"):
        pkg.api._cameras_arg(np.ones((3, 4)), m, np.ones((3, 3), np.int32))
    with pytest.raises(pkg.api.PlsvoError, match="sizes= needs cameras="):
        pkg.api._one_camera_model(None, None, sizes)
    # raw stacks of the slot's size with cameras of another size
    lenses = [camera(pkg, n) for n in ("vga_pincushion", ODD)]
    feats = synth.merge_sizes([features(synth, "vga_pincushion", 2, seed=3), features(synth, ODD, 1, seed=4)], [[0, 2], [1]])[0]
    assert (feats.cam.width, feats.cam.height) == (641, 480)
    stacks = (np.zeros((3, 480, 641), np.uint8), np.zeros((3, 480, 641), np.uint8))
    rf, ab, keep = pkg.api._raw_call_args(lenses, stacks, feats, np.array([0, 1, 0]))
    assert rf.pitch == 641 and rf.stride == 641 * 480 and rf.cams[0].width == 640 and rf.cams[1].height == 479


@pytest.fixture(scope="module")
def mixed_hostmodel(tmp_path_factory):
    return _build_model(str(tmp_path_factory.mktemp("hostmodel") / "libplsvo_hostmodel_mixed_sizes.so"))


def _build_model(out, abi_source=ABI_SOURCE):
    spec = importlib.util.spec_from_file_location("plsvo_hostmodel_build", os.path.join(HERE, "hostmodel", "build.py"))
    hm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(hm)
    sources = [abi_source] + hm.SOURCES[1:]
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-Wno-unused-function", "-I" + hm.cuda_include(),
                    "-I" + os.path.join(ROOT, "pl-svo_b200", "csrc"), "-x", "c++", *sources,
                    *(os.path.join(HERE, "hostmodel", f) for f in ("fake_undistort.cpp", "fake_raw_pyramid.cpp", "fake_mixed_sizes.cpp")),
                    "-o", out, "-lpthread", "-ldl", "-Wl,-Bsymbolic"], check=True)
    return out


def _run_model(lib, mode, k):
    env = dict(os.environ, PLSVO_LIB=lib, PLSVO_FAKE_CUDA=mode)
    for name in [n for n in env if n.startswith("PLSVO_") and n not in ("PLSVO_LIB", "PLSVO_FAKE_CUDA")]:
        del env[name]
    return subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-p", "no:cacheprovider",
                           "-k", k], env=env, capture_output=True, text=True, timeout=3000)


@pytest.mark.parametrize("mode", ["lazy", "eager"])
def test_gpu_tests_of_this_file_against_the_host_model(oracle, mixed_hostmodel, mode):
    """The GPU tests below on the unchanged host code of plsvo_abi.cu with the model CUDA runtime: the model checks every
    access and the stream order; its alignment digests each pair's own region at each level, so a pair handed the slot's
    size instead of its camera's differs from the per-size calls.  The oracle tests need real kernels and are deselected."""
    p = _run_model(mixed_hostmodel, mode, "not oracle and not every_variant")
    assert p.returncode == 0 and " skipped" not in p.stdout and " passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


FAULTS = {
    # every visit record of the fused kernel given the slot's map pitch instead of its camera's
    "visits_get_the_slot_map_pitch": (
        [("    rc = raw_multicam_maps(c, in, (int)B, s);\n    if (rc != PLSVO_OK) return rc;\n",
          "    rc = raw_multicam_maps(c, in, (int)B, s);\n    if (rc != PLSVO_OK) return rc;\n"
          "    for (RawVisit& v : c->h_visit) v.map_pitch = map_pitch_of(W);\n")],
        "raw"),
    # every pair of a raw multicam call aligned at the slot's size
    "raw_pairs_get_the_slot_size": (
        [("      c->h_mc_cams[b] = plsvo_camera{k.width, k.height, 0, 0, k.fx, k.fy, k.cx, k.cy};\n",
          "      c->h_mc_cams[b] = plsvo_camera{W, H, 0, 0, k.fx, k.fy, k.cx, k.cy};\n")],
        "raw"),
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
    p = _run_model(lib, "lazy", k + " and not oracle")
    assert " passed" in p.stdout or " failed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]
    assert p.returncode != 0 and " failed" in p.stdout, f"{fault}: every test still passes — the model is blind to it"


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("B", [37, BIG])
@pytest.mark.parametrize("bearings", ["full", "lean"])
@pytest.mark.parametrize("levels", ["shipped", "derived"])
def test_gpu_mixed_sizes_equal_per_size_and_per_camera_calls(pkg, synth, gen_device, B, bearings, levels, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2" if B <= 132 else "128,4")
    cams = cameras_of(synth)
    data, k, sizes, groups = mixed(synth, cams, B, seed=100 + B, device=gen_device)
    ragged(data, seed=B, empty=(int(groups[2][0]),))  # ragged counts, masks, and an empty EuRoC pair
    if bearings == "lean":
        lean(data)
    if levels == "derived":  # level 2 shipped, 3 and 4 half-sampled on the device
        data.ref_pyr, data.cur_pyr = {2: data.ref_pyr[2]}, {2: data.cur_pyr[2]}
    got = pkg.SparseImgAlign(4, 2, 30).run(data, cameras=k, sizes=sizes)
    by_size, by_cam = per_size_and_per_camera(pkg, synth, data, k, sizes, cams, groups)
    assert_rows(got, by_size, "per size group")
    assert_rows(got, by_cam, "per camera")
    if not MODEL:
        assert all((got.n_tracked[idx] > 0).any() for idx in groups)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_gpu_mixed_sizes_every_variant(pkg, synth, gen_device, variant, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", variant)
    cams = cameras_of(synth)
    data, k, sizes, groups = mixed(synth, cams, 37, seed=300, device=gen_device, n_pts=100, n_segs=24)
    ragged(data, seed=301)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, cameras=k, sizes=sizes)
    by_size, by_cam = per_size_and_per_camera(pkg, synth, data, k, sizes, cams, groups)
    assert_rows(got, by_size, variant)
    assert_rows(got, by_cam, variant)


@pytest.mark.gpu
def test_gpu_padding_does_not_matter(pkg, synth, gen_device, monkeypatch):
    """The same mixed batch with its padding filled with 0x00, 0xFF and random bytes: byte-identical results."""
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    cams = cameras_of(synth)
    outs = []
    for fill in (0, 255, np.random.default_rng(5)):
        data, k, sizes, _ = mixed(synth, cams, 37, seed=400, device=gen_device, fill=fill)
        outs.append(pkg.SparseImgAlign(4, 2, 30).run(data, cameras=k, sizes=sizes))
    for o in outs[1:]:
        assert_same(o, outs[0], ALIGN_FIELDS)


@pytest.mark.gpu
@pytest.mark.parametrize("n_iter_ref", [None, 3])
@pytest.mark.parametrize("chained", [True, False])
def test_gpu_track_equals_per_size_calls(pkg, synth, gen_device, chained, n_iter_ref, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    cams = cameras_of(synth)
    B = 40
    data, k, sizes, groups = mixed(synth, cams, B, seed=500, device=gen_device)
    po = synth.make_poseopt_batch(cam=synth.VGA, batch=B, n_pts=data.n_pts, n_segs=data.n_segs, seed=501, T_gt=data.T_cur_w_gt)
    fields = ("T_f_w", "num_obs_pt", "status") if MODEL else PO_FIELDS
    got_a, got_p = pkg.api.track(data, po, po_n_iter_ref=n_iter_ref, chained=chained, cameras=k, sizes=sizes)
    for size in {(c.width, c.height) for c in cams}:
        idx = np.flatnonzero((sizes == size).all(1))
        cam = next(c for c in cams if (c.width, c.height) == size)
        want_a, want_p = pkg.api.track(crop(synth, data, idx, cam), synth.take_pairs(po, idx), po_n_iter_ref=n_iter_ref,
                                   chained=chained, cameras=k[idx])
        assert_same(rows(got_a, idx), want_a, ALIGN_FIELDS, what=str(size))
        assert_same(rows(got_p, idx, fields), want_p, fields, what=str(size))


@pytest.mark.gpu
def test_gpu_frame_chain_of_one_size_in_a_larger_slot(pkg, abi, synth, gen_device, monkeypatch):
    """A chain of VGA frames in EuRoC-sized slots equals the plain VGA chain; a chain whose size changes is rejected."""
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    data = synth.make_chain_batch(cam=synth.VGA, batch=9, n_pts=150, n_segs=40, seed=600, device=gen_device)
    data.frame_pyr = synth.chain_frames(data)
    want = pkg.SparseImgAlign(4, 2, 30).run(data)
    slot = dataclasses.replace(synth.VGA, width=752)
    padded = dataclasses.replace(data, cam=slot, frame_pyr={})
    for l, f in data.frame_pyr.items():
        out = np.full((f.shape[0], 480 >> l, 752 >> l), 255, np.uint8)
        out[:, : f.shape[1], : f.shape[2]] = f
        padded.frame_pyr[l] = out
    k = np.tile([synth.VGA.fx, synth.VGA.fy, synth.VGA.cx, synth.VGA.cy], (9, 1))
    sizes = np.tile([640, 480], (9, 1)).astype(np.int32)
    got = pkg.SparseImgAlign(4, 2, 30).run(padded, cameras=k, sizes=sizes)
    assert_same(got, want, ALIGN_FIELDS)
    sizes[5] = (600, 480)
    with pytest.raises(pkg.api.PlsvoError, match=r"cams\[4\] is 640x480 and cams\[5\] is 600x480"):
        pkg.SparseImgAlign(4, 2, 30).run(padded, cameras=k, sizes=sizes)


@pytest.mark.gpu
def test_gpu_rejections_queue_nothing(pkg, abi, synth, gen_device):
    """Cameras larger than the slot, a level under one pixel for one pair's camera and a chain whose size changes are
    rejected before anything is queued (against the host model: no stream operation ran or is pending); then every
    existing malformed multicam case, and a valid call on the same context."""
    from test_gpu_multicam import test_malformed_multicam_calls

    ctx = pkg.Context(0)
    model = C.CDLL(os.environ["PLSVO_LIB"]) if MODEL else None
    if model:
        model.fake_cuda_ops_run.restype = C.c_ulonglong
    d = synth.make_align_batch(cam=synth.VGA, batch=3, n_pts=16, n_segs=4, seed=700, device=gen_device)
    ab, keep = abi.make_align_batch(d)
    k = np.tile([420.0, 420.0, 160.0, 120.0], (3, 1))
    ao = abi.AlignOut(3, 4)

    def run(sizes, hi=4, flags=0):
        ab.flags = flags
        ops = model.fake_cuda_ops_run() if model else 0
        cams = abi.make_cameras(k, d.cam, 3, np.array(sizes, np.int32))
        rc = ctx.lib.plsvo_align_multicam_batch_run(ctx.handle, cams, C.byref(ab), C.byref(abi.align_params(hi, 2, 30)), C.byref(ao.struct))
        if model and rc != abi.OK:
            assert model.fake_cuda_pending_ops() == 0 and model.fake_cuda_ops_run() == ops, "a rejected call queued work"
        return rc, ctx.lib.plsvo_last_error(ctx.handle).decode()

    ok = [(320, 240), (640, 480), (641 - 1, 479)]
    for sizes, hi, msg in (([(320, 240), (656, 480), (320, 240)], 4, "cams[1] is 656x480"),
                           ([(320, 240), (640, 481), (320, 240)], 4, "cams[1] is 640x481"),
                           ([(320, 240), (0, 480), (320, 240)], 4, "cams[1] is 0x480"),
                           ([(320, 240), (640, 480), (40, 30)], 6, "cams[2] is 40x30: pyramid level 5 smaller than one pixel")):
        rc, err = run(sizes, hi)
        assert rc == abi.ERR_INVALID and msg in err, (sizes, err)
        rc, err = run(ok)
        assert rc == abi.OK, err
    ctx.close()
    test_malformed_multicam_calls(pkg, abi, synth)


# ---- raw frames ------------------------------------------------------------------------------------------------------
def raw_mixed(pkg, synth, B, seed, fill=0):
    groups = interleave(len(RAW_LENSES), B, seed)
    parts = [features(synth, n, len(idx), seed=seed + k) for k, (n, idx) in enumerate(zip(RAW_LENSES, groups))]
    raws = [(raw_frames(n, len(idx), seed=seed + 11 * k), raw_frames(n, len(idx), seed=seed + 11 * k + 1))
            for k, (n, idx) in enumerate(zip(RAW_LENSES, groups))]
    data, sizes, raw = synth.merge_sizes(parts, groups, fill=fill, raws=raws)
    cop = np.zeros(B, np.int32)
    for kk, idx in enumerate(groups):
        cop[idx] = kk
    return data, raw, cop, groups, raws, parts


@pytest.mark.gpu
@pytest.mark.parametrize("B", [37, BIG])
def test_gpu_raw_mixed_sizes_equal_each_cameras_raw_call(pkg, synth, B, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2" if B <= 132 else "128,4")
    ctx = pkg.api.Context(0)
    data, raw, cop, groups, raws, parts = raw_mixed(pkg, synth, B, seed=800 + B)
    lenses = [camera(pkg, n) for n in RAW_LENSES]
    al = pkg.SparseImgAlign(4, 2, 30, ctx=ctx)
    got, rect = al.run_raw(lenses, raw, data, rect_levels=list(range(7)), cam_of_pair=cop)
    n0 = ctx.launch_count()
    again = al.run_raw(lenses, raw, data, cam_of_pair=cop)
    assert ctx.launch_count() - n0 == 2 and ctx.last_map_build_ms() is None  # the fused kernel and the alignment
    assert_same(again, got, ALIGN_FIELDS)
    frames_cam = np.concatenate([cop, cop])
    for kk, (name, idx) in enumerate(zip(RAW_LENSES, groups)):
        W, H = params(name)[:2]
        want = pkg.SparseImgAlign(4, 2, 30, ctx=ctx).run_raw(lenses[kk], raws[kk], parts[kk])
        assert_same(rows(got, idx), want, ALIGN_FIELDS, what=name)
        fidx = np.flatnonzero(frames_cam == kk)
        und = lenses[kk].undistortImage(np.concatenate(raws[kk]), 7, ctx)
        for l in range(7):
            np.testing.assert_array_equal(rect[l][fidx, : H >> l, : W >> l], und[l], err_msg=f"{name} level {l}")
            assert not rect[l][fidx, H >> l:].any() and not rect[l][fidx, :, W >> l:].any(), f"{name} level {l} padding"
    ctx.close()


@pytest.mark.gpu
def test_gpu_raw_padding_does_not_matter(pkg, synth, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    lenses = [camera(pkg, n) for n in RAW_LENSES]
    outs = []
    for fill in (0, 255, np.random.default_rng(9)):
        data, raw, cop, *_ = raw_mixed(pkg, synth, 23, seed=900, fill=fill)
        outs.append(pkg.SparseImgAlign(4, 2, 30).run_raw(lenses, raw, data, rect_levels=list(range(7)), cam_of_pair=cop))
    for o, rect in outs[1:]:
        assert_same(o, outs[0][0], ALIGN_FIELDS)
        for l in range(7):
            np.testing.assert_array_equal(rect[l], outs[0][1][l], err_msg=f"rect_out level {l}")


@pytest.mark.gpu
@pytest.mark.parametrize("chained", [True, False])
def test_gpu_raw_track_equals_each_cameras_track_raw(pkg, synth, chained, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    ctx = pkg.api.Context(0)
    B = 19
    data, raw, cop, groups, raws, parts = raw_mixed(pkg, synth, B, seed=1000)
    po = synth.make_poseopt_batch(cam=synth.VGA, batch=B, n_pts=data.n_pts, n_segs=data.n_segs, seed=1001, T_gt=data.T_cur_w_gt)
    fields = ("T_f_w", "num_obs_pt", "status") if MODEL else PO_FIELDS
    lenses = [camera(pkg, n) for n in RAW_LENSES]
    got_a, got_p = pkg.track_raw(lenses, raw, data, po, chained=chained, ctx=ctx, cam_of_pair=cop)
    for kk, (name, idx) in enumerate(zip(RAW_LENSES, groups)):
        sub_po = synth.take_pairs(po, idx)
        sub_po.fx = abs(params(name)[2])
        want_a, want_p = pkg.track_raw(lenses[kk], raws[kk], parts[kk], sub_po, chained=chained, ctx=ctx)
        assert_same(rows(got_a, idx), want_a, ALIGN_FIELDS, what=name)
        assert_same(rows(got_p, idx, fields), want_p, fields, what=name)
    ctx.close()


@pytest.mark.gpu
def test_gpu_raw_rejections(pkg, abi, synth):
    ctx = pkg.api.Context(0)
    data, raw, cop, *_ = raw_mixed(pkg, synth, 7, seed=1100)
    big = list(params(EUROC))
    big[0] = 768
    tiny = list(params(COPY))
    tiny[:2] = [40, 30]
    for lens, hi, msg in ((big, 4, "cams[0] is 768x480"), (tiny, 6, "pyramid level smaller than one pixel")):
        lenses = [pkg.PinholeCamera(*lens)] + [camera(pkg, n) for n in RAW_LENSES[1:]]
        with pytest.raises(pkg.api.PlsvoError, match=msg.replace("[", r"\[").replace("]", r"\]")):
            pkg.SparseImgAlign(hi, 2, 30, ctx=ctx).run_raw(lenses, raw, data, cam_of_pair=cop)
    pkg.SparseImgAlign(4, 2, 30, ctx=ctx).run_raw([camera(pkg, n) for n in RAW_LENSES], raw, data, cam_of_pair=cop)
    ctx.close()


# ---- oracle ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_mixed_sizes_against_the_oracle(pkg, abi, synth, oracle, gen_device):
    from test_gpu_align import _check

    cams = cameras_of(synth)
    data, k, sizes, groups = mixed(synth, cams, 24, seed=1200, device=gen_device, n_pts=200, n_segs=50)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, cameras=k, sizes=sizes)
    for cam, idx in zip(cams, groups):
        want = oracle.align(abi, crop(synth, data, idx, cam), abi.align_params(4, 2, 30), n_threads=8)
        _check(synth, rows(got, idx), want)


@pytest.mark.gpu
def test_gpu_raw_mixed_sizes_oracle_end_to_end(pkg, abi, synth, oracle, gen_device):
    """A VGA and a EuRoC lens in one batch: per camera, oracle undistortion -> oracle pyramid -> oracle alignment, and
    the poses closer to ground truth than the initial guess."""
    import undistort_oracle
    from test_gpu_align import _check

    undistort_oracle.build()
    cams, dists = (synth.VGA, synth.EUROC), ((-0.28, 0.07, 0.0, 0.0, 0.0), synth.EUROC_DIST)
    groups = interleave(2, 8, seed=1300)
    parts, raws = [], []
    for kk, (c, dd, idx) in enumerate(zip(cams, dists, groups)):
        d, r, _ = synth.make_raw_multicam_batch([c], [dd], np.zeros(len(idx), int), n_pts=150, n_segs=30, seed=1301 + kk,
                                                device=gen_device)
        parts.append(d)
        raws.append(r)
    data, sizes, raw = synth.merge_sizes(parts, groups, raws=raws)
    cop = np.zeros(8, np.int32)
    cop[groups[1]] = 1
    pcs = [pkg.PinholeCamera(c.width, c.height, c.fx, c.fy, c.cx, c.cy, *dd) for c, dd in zip(cams, dists)]
    data.ref_pyr = data.cur_pyr = {}
    gpu = pkg.SparseImgAlign(4, 2, 30).run_raw(pcs, raw, data, cam_of_pair=cop)
    for kk, idx in enumerate(groups):
        sub = synth.take_pairs(data, idx)
        sub.cam = cams[kk]
        r = undistort_oracle.undistort(abi, pcs[kk].struct, np.concatenate(raws[kk]), 5)
        n = len(idx)
        sub.ref_pyr = {l: np.ascontiguousarray(r[l][:n]) for l in range(2, 5)}
        sub.cur_pyr = {l: np.ascontiguousarray(r[l][n:]) for l in range(2, 5)}
        _check(synth, rows(gpu, idx), oracle.align(abi, sub, abi.align_params(4, 2, 30), n_threads=8))
    a0, t0 = synth.pose_error(data.T_cur_w, data.T_cur_w_gt)
    a1, t1 = synth.pose_error(gpu.T_cur_w, data.T_cur_w_gt)
    assert np.median(a1) < 0.25 * np.median(a0) and np.median(t1) < 0.25 * np.median(t0), (a0, a1, t0, t1)
