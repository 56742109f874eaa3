"""Frame pairs from pinhole and ATAN (FOV) cameras in one batch (plsvo_align_any_camera_batch_run,
plsvo_track_any_camera_batch_run): pair b's camera is cams[cam_of_pair[b]], a plsvo_match_camera whose tag picks the
model.  A pinhole pair's outputs must be byte-identical to plsvo_align_multicam_batch_run on that model's pairs with their
cameras, an ATAN pair's to plsvo_align_atan_multicam_batch_run, at the same kernel variant; the padding of the slots must
not matter; each model group agrees with its oracle.

CPU: the Python argument handling and synth.make_any_camera_batch, this file's GPU tests against the host model of the C
ABI (tests/hostmodel/fake_any_camera.cpp: every pair runs through the model's pinhole or ATAN kernel by its tag, at its
own size with its own camera), and three faults seeded into plsvo_abi.cu that the model, with every kernel answered by
the CPU oracles, must notice."""
import copy
import ctypes as C
import dataclasses
import os

import numpy as np
import pytest

from test_gpu_atan_multicam import _oracle_lib, cop_of, lean, slot_cam
from test_gpu_mixed_sizes import crop, interleave, rows
from test_gpu_multicam import ALIGN_FIELDS, PO_FIELDS, assert_same, ragged

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ABI_SOURCE = os.path.join(ROOT, "pl-svo_b200", "csrc", "plsvo_abi.cu")
MODEL = bool(os.environ.get("PLSVO_FAKE_CUDA"))
ORACLE_MODEL = bool(os.environ.get("PLSVO_FAKE_ORACLE"))
BIG = 16 if MODEL else 1024  # the host model renders on the CPU
VARIANTS = ["64,8", "96,7", "96,5", "128,5", "128,4", "160,3", "192,2", "256,2"]


def stock(pkg, synth):
    """A VGA pinhole camera and SVO's stock 752x480 ATAN camera."""
    return (synth.Camera(640, 480, 420.0, 420.0, 319.5, 239.5),
            pkg.ATANCamera(752, 480, 0.511496, 0.802603, 0.530199, 0.496011, 0.934092))


def fleet(pkg, synth):
    """Eight cameras in one 752x480 slot: a pinhole and an ATAN camera at each of 752x480, 640x480, 641x479 and 320x240,
    the ATAN ones with d0 in {0.93, 0.3, 0, -0.3}, non-square and off-centre."""
    return (synth.Camera(752, 480, 438.0, 385.0, 385.5, 229.5),
            pkg.ATANCamera(752, 480, 0.5825, 0.8000, 0.5127, 0.4784, 0.93),
            synth.Camera(640, 480, 517.3, 516.5, 318.6, 255.3),
            pkg.ATANCamera(640, 480, 0.6600, 0.9000, 0.4900, 0.5300, 0.3),
            synth.Camera(641, 479, 420.0, 425.0, 320.0, 239.0),
            pkg.ATANCamera(641, 479, 0.6500, 0.8700, 0.5000, 0.5000, 0.0),
            synth.Camera(320, 240, 210.0, 205.0, 159.5, 119.5),
            pkg.ATANCamera(320, 240, 0.6800, 0.8800, 0.5200, 0.4800, -0.3))


def is_pinhole(synth, cam):
    return isinstance(cam, synth.Camera)


def pinhole_args(cams, cop):
    """cameras= and sizes= of the pinhole multicam call for pairs of the pinhole cameras cams[cop[b]]"""
    return dict(cameras=np.array([[cams[k].fx, cams[k].fy, cams[k].cx, cams[k].cy] for k in cop]),
                sizes=np.array([[cams[k].width, cams[k].height] for k in cop], np.int32))


def per_model(pkg, synth, data, cams, cop, hi=4, lo=2):
    """Pair b's outputs from its own model's per-pair call on that model's pairs, in the same slots: the pinhole multicam
    call with the pinhole pairs' intrinsics and sizes, the ATAN multicam call with the ATAN pairs' cameras."""
    want = {}
    pin = np.array([is_pinhole(synth, cams[k]) for k in cop])
    for mask in (pin, ~pin):
        idx = np.flatnonzero(mask)
        if not len(idx):
            continue
        sub = synth.take_pairs(data, idx)
        if mask is pin:
            got = pkg.SparseImgAlign(hi, lo, 30).run(sub, **pinhole_args(cams, cop[idx]))
        else:
            atan = sorted(set(cop[idx].tolist()))
            remap = {k: i for i, k in enumerate(atan)}
            got = pkg.SparseImgAlign(hi, lo, 30).run(sub, camera=[cams[k] for k in atan],
                                                     cam_of_pair=np.array([remap[k] for k in cop[idx]], np.int32))
        for f in ALIGN_FIELDS:
            want.setdefault(f, np.zeros((data.batch,) + getattr(got, f).shape[1:], getattr(got, f).dtype))[idx] = getattr(got, f)
    return want


def assert_rows(got, want, what):
    for f in ALIGN_FIELDS:
        np.testing.assert_array_equal(getattr(got, f).view(np.uint8), want[f].view(np.uint8), err_msg=f"{what} {f}")


def fleet_batch(pkg, synth, cams, B, seed, device, fill=0, n_pts=150, n_segs=40):
    groups = interleave(len(cams), B, seed)
    cop = cop_of(groups, B)
    slot = synth.Camera(max(c.width for c in cams), max(c.height for c in cams), 1.0, 1.0, 0.0, 0.0)
    data, parts, groups = synth.make_any_camera_batch(cams, cop, slot=slot, fill=fill, n_pts=n_pts, n_segs=n_segs, seed=seed,
                                                      device=device)
    return cop, data, groups


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
def test_python_arguments_and_synth_helper(pkg, synth):
    cams = fleet(pkg, synth)
    cop = np.array([7, 6, 7, 6, 0])
    data, parts, groups = synth.make_any_camera_batch(cams, cop, fill=255, n_pts=8, n_segs=2, seed=1)
    assert (data.cam.width, data.cam.height) == (752, 480) and len(parts) == 3
    assert [g.tolist() for g in groups] == [[4], [1, 3], [0, 2]]
    assert (parts[1].cam.width, parts[1].cam.height) == (320, 240) and parts[1].cam == cams[6]
    assert parts[2].cam.fx == cams[7].fx_
    for l in data.ref_pyr:
        np.testing.assert_array_equal(data.ref_pyr[l][3, : 240 >> l, : 320 >> l], parts[1].ref_pyr[l][1])
        np.testing.assert_array_equal(data.ref_pyr[l][2, : 240 >> l, : 320 >> l], parts[2].ref_pyr[l][1])
        assert (data.ref_pyr[l][0, 240 >> l:] == 255).all()
    # an ATAN part's bearings go through the ATAN model, a pinhole part's through the pinhole one
    np.testing.assert_allclose(parts[2].pt_f[0], cams[7].cam2world(parts[2].pt_px[0]), rtol=0, atol=1e-12)
    al, po, parts, po_parts, groups = synth.make_any_camera_batch(cams[:2], [1, 0, 1], poseopt=True, n_pts=8, n_segs=2, seed=2)
    assert po_parts[0].fx == abs(cams[0].fx) and po_parts[1].fx == cams[1].fx_ and po.batch == 3
    np.testing.assert_array_equal(po.pt_f[[0, 2]], po_parts[1].pt_f)
    # dispatch: a sequence holding a synth.Camera takes the any-camera call; ATAN only keeps its path; anything else
    # (the distorted api.PinholeCamera) keeps the ATAN path's error
    E, arg = pkg.api.PlsvoError, pkg.api._any_cameras_arg
    arr, n, k = arg(list(cams), None, None, cop, data)
    assert n == 8 and k.dtype == np.int32 and k.tolist() == cop.tolist()
    assert [arr[i].model for i in range(8)] == [0, 1] * 4
    assert (arr[0].pinhole.width, arr[0].pinhole.fx) == (752, 438.0) and (arr[7].atan.width, arr[7].atan.d0) == (320, -0.3)
    assert arg([cams[1], cams[3]], None, None, cop % 2, data) is None
    raw = pkg.PinholeCamera(640, 480, 420, 420, 320, 240)
    assert arg([cams[0], raw], None, None, cop % 2, data) is None
    with pytest.raises(E, match="sequence of ATANCamera"):
        pkg.api._atan_cameras_arg([cams[0], raw], None, None, cop % 2, data)
    assert arg(list(cams), None, None, None, data) is None and arg(cams[0], None, None, cop, data) is None
    with pytest.raises(E, match="no cameras= or sizes="):
        arg(list(cams), np.ones((5, 4)), None, cop, data)
    with pytest.raises(E, match="no cameras= or sizes="):
        arg(list(cams), None, np.ones((5, 2), np.int32), cop, data)
    with pytest.raises(E, match="cam_of_pair must be"):
        arg(list(cams), None, None, cop[:4], data)
    with pytest.raises(E, match="cam_of_pair must be"):
        arg(list(cams), None, None, cop.astype(float), data)


@pytest.fixture(scope="module")
def any_hostmodel(tmp_path_factory):
    return _build_model(str(tmp_path_factory.mktemp("hostmodel") / "libplsvo_hostmodel_any_camera.so"))


def _build_model(out, abi_source=ABI_SOURCE):
    """The stock model kernels with fake_atan_multicam.cpp (the ATAN multicam launchers and the per-frame pose optimiser)
    and fake_any_camera.cpp (the any-camera and pinhole multicam launchers) linked next to them."""
    import importlib.util
    import subprocess

    spec = importlib.util.spec_from_file_location("plsvo_hostmodel_build", os.path.join(HERE, "hostmodel", "build.py"))
    hm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(hm)
    sources = [abi_source] + hm.SOURCES[1:] + [os.path.join(HERE, "hostmodel", f) for f in ("fake_atan_multicam.cpp", "fake_any_camera.cpp")]
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-Wno-unused-function", "-I" + hm.cuda_include(),
                    "-I" + os.path.join(ROOT, "pl-svo_b200", "csrc"), "-x", "c++", *sources, "-o", out, "-lpthread", "-ldl",
                    "-Wl,-Bsymbolic"], check=True)
    return out


@pytest.mark.parametrize("mode", ["lazy", "eager"])
def test_gpu_tests_of_this_file_against_the_host_model(oracle, any_hostmodel, mode):
    """The GPU tests below on the unchanged host code of plsvo_abi.cu with the model CUDA runtime: the model checks every
    access and the stream order, and digests each pair's own region at its own size.  The oracle tests and the
    shared-memory sweep need real kernels and are deselected."""
    p = _run_here(any_hostmodel, mode, "not oracle and not every_variant and not shared_memory")
    assert p.returncode == 0 and " skipped" not in p.stdout and " passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


def _run_here(lib, mode, k, oracle_lib=None):
    """_run_model of test_gpu_atan_multicam.py on this file."""
    import subprocess
    import sys

    env = dict(os.environ, PLSVO_LIB=lib, PLSVO_FAKE_CUDA=mode)
    for name in [n for n in env if n.startswith("PLSVO_") and n not in ("PLSVO_LIB", "PLSVO_FAKE_CUDA")]:
        del env[name]
    if oracle_lib:
        env["PLSVO_FAKE_ORACLE"] = oracle_lib
    return subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-p", "no:cacheprovider",
                           "-k", k], env=env, capture_output=True, text=True, timeout=3000)


FAULTS = {
    # every pair given the model tag of cams[0] (a pinhole): the ATAN pairs run through the pinhole model
    "every_pair_gets_cams0_tag": (
        "    c->h_cam_models[i] = cams[k].model;\n",
        "    c->h_cam_models[i] = cams[0].model;\n",
        "mixed and full and shipped"),
    # the ATAN pairs' distortion terms indexed by camera instead of by pair
    "terms_indexed_by_camera": (
        "    if (cams[k].model == PLSVO_CAMERA_ATAN) std::copy(&terms[4 * (size_t)k], &terms[4 * (size_t)k + 4], &c->h_atan_terms[4 * i]);\n",
        "    if (cams[k].model == PLSVO_CAMERA_ATAN) std::copy(&terms[4 * (size_t)(i % n_cams)], &terms[4 * (size_t)(i % n_cams) + 4], &c->h_atan_terms[4 * i]);\n",
        "mixed and full and shipped"),
    # the track call's pose optimiser given the normalised fx of an ATAN camera instead of errorMultiplier2() = fx_
    "track_gets_normalised_fx": (
        "  for (int i = 0; i < ab->batch; ++i) c->h_po_fx[i] = fabs(c->h_mc_cams[i].fx);\n",
        "  for (int i = 0; i < ab->batch; ++i)\n"
        "    c->h_po_fx[i] = cams[cam_of_pair[i]].model == PLSVO_CAMERA_ATAN ? cams[cam_of_pair[i]].atan.fx : fabs(c->h_mc_cams[i].fx);\n",
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


def test_unmutated_track_and_mixed_pass_on_the_oracle_model(oracle, oracle_atan, any_hostmodel):
    """The control of the seeded faults: the same selections on the unmutated host code pass."""
    p = _run_here(any_hostmodel, "lazy", "(track or (mixed and full and shipped)) and not oracle", _oracle_lib(oracle, oracle_atan))
    assert p.returncode == 0 and " passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("B", [37, BIG])
@pytest.mark.parametrize("which", ["pinhole", "atan"])
def test_gpu_one_model_table_equals_its_multicam_call(pkg, synth, gen_device, which, B, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2" if B <= 132 else "128,4")
    pin, atan = stock(pkg, synth)
    cams = [pin, synth.Camera(600, 450, 517.3, 516.5, 300.6, 225.3)] if which == "pinhole" else [atan, stock_vga_atan(pkg)]
    cop, data, groups = fleet_batch(pkg, synth, cams, B, seed=100 + B, device=gen_device)
    ragged(data, seed=B)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, camera=list(cams) + [synth.VGA], cam_of_pair=cop)
    if which == "pinhole":
        want = pkg.SparseImgAlign(4, 2, 30).run(data, **pinhole_args(cams, cop))
    else:
        want = pkg.SparseImgAlign(4, 2, 30).run(data, camera=list(cams), cam_of_pair=cop)
    assert_same(got, want, ALIGN_FIELDS)


def stock_vga_atan(pkg):
    return pkg.ATANCamera(640, 480, 0.65625, 0.875, 0.5, 0.5, 0.3)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_gpu_one_model_table_every_variant(pkg, synth, gen_device, variant, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", variant)
    for which, cam in enumerate(stock(pkg, synth)):
        cop, data, _ = fleet_batch(pkg, synth, [cam], 37, seed=200 + which, device=gen_device, n_pts=100, n_segs=24)
        got = pkg.SparseImgAlign(4, 2, 30).run(data, camera=[cam, synth.QVGA], cam_of_pair=cop)
        assert_rows(got, per_model(pkg, synth, data, [cam], cop), f"{variant} camera {which}")


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_gpu_mixed_every_variant(pkg, synth, gen_device, variant, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", variant)
    cams = stock(pkg, synth)
    cop, data, groups = fleet_batch(pkg, synth, cams, 37, seed=250, device=gen_device, n_pts=100, n_segs=24)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, camera=list(cams), cam_of_pair=cop)
    assert_rows(got, per_model(pkg, synth, data, cams, cop), variant)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [37, BIG])
@pytest.mark.parametrize("K", [2, 8])
@pytest.mark.parametrize("bearings", ["full", "lean"])
@pytest.mark.parametrize("levels", ["shipped", "derived"])
def test_gpu_mixed_fleet_equals_per_model_calls(pkg, synth, gen_device, B, K, bearings, levels, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2" if B <= 132 else "128,4")
    cams = stock(pkg, synth) if K == 2 else fleet(pkg, synth)
    cop, data, groups = fleet_batch(pkg, synth, cams, B, seed=300 + B + K, device=gen_device)
    ragged(data, seed=B, empty=(int(groups[-1][0]),))  # ragged counts, masks, and an empty pair
    if bearings == "lean":
        lean(data)
    if levels == "derived":  # level 2 shipped, 3 and 4 half-sampled on the device
        data.ref_pyr, data.cur_pyr = {2: data.ref_pyr[2]}, {2: data.cur_pyr[2]}
    got = pkg.SparseImgAlign(4, 2, 30).run(data, camera=list(cams), cam_of_pair=cop)
    assert_rows(got, per_model(pkg, synth, data, cams, cop), "per model")
    if not MODEL:
        assert all((got.n_tracked[idx] > 0).any() for idx in groups)


@pytest.mark.gpu
def test_gpu_d0_zero_atan_stays_atan(pkg, synth, gen_device, monkeypatch):
    """An ATAN camera with d0 = 0 next to a pinhole camera with its members: the tag, not the parameters, picks the model,
    so each pair equals its own model's call."""
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    atan = pkg.ATANCamera(640, 480, 0.65625, 0.875, 0.5, 0.5, 0.0)
    pin = synth.Camera(640, 480, atan.fx_, atan.fy_, atan.cx_, atan.cy_)
    cams = [pin, atan]
    cop, data, groups = fleet_batch(pkg, synth, cams, 37, seed=350, device=gen_device)
    lean(data)  # both models form the bearings: the ATAN one through its cam2world
    got = pkg.SparseImgAlign(4, 2, 30).run(data, camera=cams, cam_of_pair=cop)
    assert_rows(got, per_model(pkg, synth, data, cams, cop), "d0 = 0")


@pytest.mark.gpu
def test_gpu_padding_does_not_matter(pkg, synth, gen_device, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    cams = fleet(pkg, synth)
    outs = []
    for fill in (0, 255, np.random.default_rng(5)):
        cop, data, _ = fleet_batch(pkg, synth, cams, 37, seed=400, device=gen_device, fill=fill)
        outs.append(pkg.SparseImgAlign(4, 2, 30).run(data, camera=list(cams), cam_of_pair=cop))
    for o in outs[1:]:
        assert_same(o, outs[0], ALIGN_FIELDS)


@pytest.mark.gpu
def test_gpu_chains(pkg, synth, gen_device, monkeypatch):
    """A chain of one size whose cameras alternate models equals the same pairs as two stacks.  A size change inside a
    chain is rejected."""
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    vga = stock_vga_atan(pkg)
    data = synth.make_chain_batch(cam=slot_cam(synth, vga), batch=9, n_pts=150, n_segs=40, seed=600, device=gen_device, atan=vga)
    data.frame_pyr = synth.chain_frames(data)
    cams = [vga, synth.Camera(640, 480, 420.0, 420.0, 319.5, 239.5), pkg.ATANCamera(640, 480, 0.7, 0.9, 0.48, 0.52, 0.0),
            synth.Camera(640, 480, 517.3, 516.5, 318.6, 255.3)]
    cop = np.array([0, 1, 2, 3, 1, 0, 3, 2, 0], np.int32)
    chained = pkg.SparseImgAlign(4, 2, 30).run(data, camera=cams, cam_of_pair=cop)
    stacks = copy.copy(data)
    stacks.frame_pyr = None
    assert_same(chained, pkg.SparseImgAlign(4, 2, 30).run(stacks, camera=cams, cam_of_pair=cop), ALIGN_FIELDS, what="chained")
    assert_rows(chained, per_model(pkg, synth, stacks, cams, cop), "chain per model")
    qvga = synth.QVGA
    with pytest.raises(pkg.api.PlsvoError, match=r"cams\[4\] is 640x480 and cams\[5\] is 320x240"):
        pkg.SparseImgAlign(4, 2, 30).run(data, camera=cams + [qvga], cam_of_pair=np.array([0, 1, 2, 3, 1, 4, 4, 4, 4], np.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("n_iter_ref", [None, 3])
@pytest.mark.parametrize("chained", [True, False])
def test_gpu_track_equals_per_model_track(pkg, synth, gen_device, chained, n_iter_ref, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    cams = fleet(pkg, synth)
    B = 16 if MODEL else 40
    groups = interleave(len(cams), B, 500)
    cop = cop_of(groups, B)
    data, po, parts, po_parts, groups = synth.make_any_camera_batch(cams, cop, poseopt=True, n_pts=150, n_segs=40, seed=500,
                                                                    device=gen_device)
    fields = ("T_f_w", "num_obs_pt", "status") if MODEL and not ORACLE_MODEL else PO_FIELDS
    got_a, got_p = pkg.api.track(data, po, po_n_iter_ref=n_iter_ref, chained=chained, camera=list(cams), cam_of_pair=cop)
    pin = np.array([is_pinhole(synth, cams[k]) for k in cop])
    for mask in (pin, ~pin):
        idx = np.flatnonzero(mask)
        sub, po_sub = synth.take_pairs(data, idx), synth.take_pairs(po, idx)
        if mask is pin:
            kw = pinhole_args(cams, cop[idx])
        else:
            atan = sorted(set(cop[idx].tolist()))
            kw = dict(camera=[cams[k] for k in atan], cam_of_pair=np.array([atan.index(k) for k in cop[idx]], np.int32))
        want_a, want_p = pkg.api.track(sub, po_sub, po_n_iter_ref=n_iter_ref, chained=chained, **kw)
        what = "pinhole" if mask is pin else "atan"
        assert_same(rows(got_a, idx), want_a, ALIGN_FIELDS, what=what)
        assert_same(rows(got_p, idx, fields), want_p, fields, what=what)


@pytest.mark.gpu
def test_gpu_mixed_against_the_oracles(pkg, abi, synth, oracle, oracle_atan, gen_device):
    from test_gpu_atan import compare

    cams = fleet(pkg, synth)
    cop, data, groups = fleet_batch(pkg, synth, cams, 32, seed=700, device=gen_device, n_pts=200, n_segs=50)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, camera=list(cams), cam_of_pair=cop)
    for k, cam in enumerate(cams):
        idx = np.flatnonzero(cop == k)
        if is_pinhole(synth, cam):
            want = oracle.align(abi, crop(synth, data, idx, cam), abi.align_params(4, 2, 30), n_threads=8)
        else:
            want = oracle_atan.align(abi, cam, crop(synth, data, idx, slot_cam(synth, cam)), n_threads=8)
        compare(synth, rows(got, idx), want, f"camera {k} {cam.width}x{cam.height}")
    a0, t0 = synth.pose_error(data.T_cur_w, data.T_cur_w_gt)
    a1, t1 = synth.pose_error(got.T_cur_w, data.T_cur_w_gt)
    assert np.median(a1) < 0.25 * np.median(a0) and np.median(t1) < 0.25 * np.median(t0), (a0, a1, t0, t1)


@pytest.mark.gpu
def test_gpu_shared_memory_limit(pkg, abi, synth, gen_device, monkeypatch):
    """Point counts across the <256,2> limit: a pinned call runs, byte-identical to the pinned per-model calls, or is
    refused with the plan's message."""
    cams = stock(pkg, synth)[:1] + (stock_vga_atan(pkg),)
    base, _, _ = synth.make_any_camera_batch(cams, np.array([0, 1]), n_pts=5800, n_segs=0, max_level=3, min_level=2, seed=800,
                                             device=gen_device)
    ctx = pkg.Context(0)
    lib, ap = ctx.lib, abi.align_params(3, 2, 30)
    table, cop = abi.make_match_cameras(cams), np.array([0, 1], np.int32)
    pin = abi.make_cameras([[cams[0].fx, cams[0].fy, cams[0].cx, cams[0].cy]], base.cam, 1, sizes=[[640, 480]])
    atan = abi.make_atan_cameras([cams[1].struct], np.zeros(1, np.int32), 1)
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    ran = refused = 0
    for n in range(5736, 5768, 2):
        d = dataclasses.replace(base)
        d.pt_px, d.pt_f, d.pt_pos = (np.ascontiguousarray(a[:, :n]) for a in (base.pt_px, base.pt_f, base.pt_pos))
        ab, keep = abi.make_align_batch(d)
        out = abi.AlignOut(2, 0)
        rc = lib.plsvo_align_any_camera_batch_run(ctx.handle, table, 2, cop.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(ab),
                                                   C.byref(ap), C.byref(out.struct))
        msg = lib.plsvo_last_error(ctx.handle).decode()
        assert rc in (abi.OK, abi.ERR_INVALID), (n, rc, msg)
        if rc != abi.OK:
            assert "shared-memory plan" in msg, (n, msg)
            refused += 1
            continue
        ran += 1
        for b, (fn, cam) in enumerate(((lib.plsvo_align_multicam_batch_run, pin), (lib.plsvo_align_atan_multicam_batch_run, atan))):
            one, keep1 = abi.make_align_batch(synth.take_pairs(d, [b]))
            want = abi.AlignOut(1, 0)
            assert fn(ctx.handle, cam, C.byref(one), C.byref(ap), C.byref(want.struct)) == abi.OK, n
            assert_same(rows(out, [b], ("T_cur_w", "n_tracked", "H", "iters", "status")), want,
                        ("T_cur_w", "n_tracked", "H", "iters", "status"), what=f"n_pts={n} pair {b}")
    assert ran and refused, "the sweep does not cross the limit of the <256,2> plan"
    ctx.close()


@pytest.mark.gpu
def test_gpu_malformed_calls_queue_nothing(pkg, abi, synth, gen_device):
    """Each malformed call returns PLSVO_ERR_INVALID with its message before anything is queued (against the host model:
    no stream operation ran or is pending); a valid call on the same context then succeeds."""
    ctx = pkg.Context(0)
    lib = ctx.lib
    model = C.CDLL(os.environ["PLSVO_LIB"]) if MODEL else None
    if model:
        model.fake_cuda_ops_run.restype = C.c_ulonglong
    cams = [synth.VGA, stock_vga_atan(pkg)]
    d = synth.make_any_camera_batch(cams, np.array([0, 1, 0]), n_pts=16, n_segs=4, seed=900, device=gen_device)[0]
    po = synth.make_poseopt_batch(cam=synth.VGA, batch=3, n_pts=16, n_segs=4, seed=901)
    ab, keep_a = abi.make_align_batch(d)
    pb, keep_p = abi.make_poseopt_batch(po)
    ao, pout = abi.AlignOut(3, 4), abi.PoseOptOut(3, 16, 4)

    def table(k=None, model=None, **kw):
        arr = abi.make_match_cameras(cams)
        if k is not None:
            if model is not None:
                arr[k].model = model
            rec = arr[k].pinhole if arr[k].model == abi.CAMERA_PINHOLE and model is None else arr[k].atan
            for f, v in kw.items():
                setattr(rec, f, v)
        return arr

    def run(cams_arr=None, n_cams=2, cop=(0, 1, 0), hi=4, track=False, flags=0, po_batch=3, batch=3):
        cams_arr = table() if cams_arr is None else cams_arr
        cop_arr = None if cop is None else np.ascontiguousarray(cop, np.int32)
        cop_p = None if cop is None else cop_arr.ctypes.data_as(C.POINTER(C.c_int32))
        ab.flags, pb.batch, ab.batch = flags, po_batch, batch
        ops = model.fake_cuda_ops_run() if model else 0
        launches = ctx.launch_count()
        if track:
            rc = lib.plsvo_track_any_camera_batch_run(ctx.handle, cams_arr, n_cams, cop_p, C.byref(ab),
                                                      C.byref(abi.align_params(hi, 2, 30)), C.byref(pb),
                                                      C.byref(abi.poseopt_params()), C.byref(ao.struct), C.byref(pout.struct))
        else:
            rc = lib.plsvo_align_any_camera_batch_run(ctx.handle, cams_arr, n_cams, cop_p, C.byref(ab),
                                                      C.byref(abi.align_params(hi, 2, 30)), C.byref(ao.struct))
        if rc != abi.OK:
            assert ctx.launch_count() == launches, "a rejected call launched a kernel"
            if model:
                assert model.fake_cuda_pending_ops() == 0 and model.fake_cuda_ops_run() == ops, "a rejected call queued work"
        ab.flags, pb.batch, ab.batch = 0, 3, 3
        return rc, lib.plsvo_last_error(ctx.handle).decode()

    nan = float("nan")
    E = "cams or cam_of_pair is NULL"
    for kw, msg in (({"cams_arr": C.cast(None, C.POINTER(abi.MatchCamera))}, E),
                    ({"cop": None}, E),
                    ({"cop": None, "track": True}, E),
                    ({"n_cams": 0}, "n_cams must be at least 1"),
                    ({"n_cams": -3, "track": True}, "n_cams must be at least 1"),
                    ({"cop": (0, 2, 0)}, "cam_of_pair[1] = 2 is outside [0, 2)"),
                    ({"cop": (0, 1, -1), "track": True}, "cam_of_pair[2] = -1 is outside [0, 2)"),
                    ({"cams_arr": table(1, model=7)}, "cams[1].model 7 is neither"),
                    ({"cams_arr": table(0, fx=nan)}, "cams[0] has a non-finite fx, fy, cx or cy"),
                    ({"cams_arr": table(0, fy=0.0)}, "cams[0].fx and fy must be non-zero"),
                    ({"cams_arr": table(0, width=656)}, "cams[0] is 656x480"),
                    ({"cams_arr": table(1, d0=nan)}, "cams[1] (ATAN) has a non-finite parameter"),
                    ({"cams_arr": table(1, fx=-0.5)}, "cams[1] (ATAN) fx and fy must be positive"),
                    ({"cams_arr": table(1, height=481)}, "cams[1] is 640x481"),
                    ({"cams_arr": table(1, width=0), "track": True}, "cams[1] is 0x480"),
                    ({"cams_arr": table(0, width=40, height=30), "hi": 6}, "cams[0] is 40x30: pyramid level 5 smaller than one pixel"),
                    ({"cams_arr": table(1, width=320, height=240), "flags": abi.ALIGN_FRAME_CHAIN},
                     "cams[0] is 640x480 and cams[1] is 320x240"),
                    ({"batch": 0}, "batch/n_pts/n_segs out of range"),
                    ({"batch": -1, "po_batch": -1, "track": True}, "batch/n_pts/n_segs out of range"),
                    ({"track": True, "po_batch": 2}, "batches differ in size")):
        rc, err = run(**kw)
        assert rc == abi.ERR_INVALID and msg in err, (msg, err)
    for kw in ({}, {"track": True}):
        rc, err = run(**kw)
        assert rc == abi.OK, (kw, err)
    ctx.close()
