"""Frame pairs from differently calibrated ATAN (FOV) cameras in one batch (plsvo_align_atan_multicam_batch_run,
plsvo_track_atan_multicam_batch_run): batch->cam's size is the slot, and pair b's frames are cams[b].width x
cams[b].height in the top-left corner of their slots.  Pair b's outputs must be byte-identical to the one-camera ATAN
call (plsvo_align_atan_batch_run / plsvo_track_atan_batch_run) with cams[b] on its camera's pairs at their own size, at
the same kernel variant; the padding of the slots must not matter; each camera's pairs agree with the ATAN oracle.

CPU: the Python argument handling and synth.make_atan_multicam_batch, the oracle's sensitivity to the camera, this file's
GPU tests against the host model of the C ABI (tests/hostmodel/fake_atan_multicam.cpp: every pair runs through the
model's ATAN kernel at its own size with its own camera), and two faults seeded into plsvo_abi.cu that the model, with
every kernel answered by the CPU oracle, must notice."""
import copy
import ctypes as C
import dataclasses
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_mixed_sizes import crop, interleave, rows
from test_gpu_multicam import ALIGN_FIELDS, PO_FIELDS, assert_same, ragged

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ABI_SOURCE = os.path.join(ROOT, "pl-svo_b200", "csrc", "plsvo_abi.cu")
MODEL = bool(os.environ.get("PLSVO_FAKE_CUDA"))
ORACLE_MODEL = bool(os.environ.get("PLSVO_FAKE_ORACLE"))
BIG = 16 if MODEL else 1024  # the host model renders on the CPU
VARIANTS = ["64,8", "96,7", "96,5", "128,5", "128,4", "160,3", "192,2", "256,2"]
POSE_TOL = (1e-5, 1e-4)  # test_gpu_atan.compare: rotation (rad) and relative translation against the oracle


def fleet(pkg):
    """Four FOV cameras of four sizes: no, mild, strong and negative distortion, non-square and off-centre."""
    return (pkg.ATANCamera(752, 480, 0.5825, 0.8000, 0.5127, 0.4784, 0.93),
            pkg.ATANCamera(640, 480, 0.6600, 0.9000, 0.4900, 0.5300, 0.3),
            pkg.ATANCamera(641, 479, 0.6500, 0.8700, 0.5000, 0.5000, 0.0),
            pkg.ATANCamera(320, 240, 0.6800, 0.8800, 0.5200, 0.4800, -0.3))


def stock(pkg):
    """SVO's stock 752x480 camera (d0 = 0.93) and a VGA one with d0 = 0.3."""
    return (pkg.ATANCamera(752, 480, 0.511496, 0.802603, 0.530199, 0.496011, 0.934092),
            pkg.ATANCamera(640, 480, 0.65625, 0.875, 0.5, 0.5, 0.3))


def cop_of(groups, B):
    c = np.zeros(B, np.int32)
    for k, idx in enumerate(groups):
        c[idx] = k
    return c


def lean(data):
    """Bearings left to the camera's cam2world (on the device, and in the oracle)."""
    data.pt_f = data.seg_sf = data.seg_ef = None
    return data


def slot_cam(synth, cam):
    return synth.Camera(cam.width, cam.height, cam.fx_, cam.fy_, cam.cx_, cam.cy_)


def per_camera(pkg, synth, data, cams, groups, hi=4, lo=2):
    """Pair b's outputs from the one-camera ATAN call with its camera on its camera's pairs at their size."""
    want = {}
    for cam, idx in zip(cams, groups):
        got = pkg.SparseImgAlign(hi, lo, 30).run(crop(synth, data, idx, slot_cam(synth, cam)), camera=cam)
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
def test_python_arguments_and_synth_helper(pkg, synth):
    cams = fleet(pkg)
    cop = np.array([3, 1, 3, 1, 3])
    data, parts, groups = synth.make_atan_multicam_batch(cams, cop, fill=255, n_pts=8, n_segs=2, seed=1)
    assert (data.cam.width, data.cam.height) == (640, 480) and len(parts) == 2
    assert [g.tolist() for g in groups] == [[1, 3], [0, 2, 4]]
    assert (parts[1].cam.width, parts[1].cam.height) == (320, 240)
    for l in data.ref_pyr:
        np.testing.assert_array_equal(data.ref_pyr[l][2, : 240 >> l, : 320 >> l], parts[1].ref_pyr[l][1])
        assert (data.ref_pyr[l][0, 240 >> l:] == 255).all()
    al, po, parts, po_parts, groups = synth.make_atan_multicam_batch(cams[:2], [1, 0, 1], poseopt=True, n_pts=8, n_segs=2, seed=2)
    assert po_parts[0].fx == cams[0].fx_ and po_parts[1].fx == cams[1].fx_ and po.batch == 3
    np.testing.assert_array_equal(po.pt_f[[0, 2]], po_parts[1].pt_f)
    # argument handling: a sequence needs cam_of_pair, cam_of_pair needs a sequence of ATANCamera, no mixing
    E = pkg.api.PlsvoError
    with pytest.raises(E, match="needs cam_of_pair"):
        pkg.api._atan_cameras_arg(list(cams), None, None, None, data)
    with pytest.raises(E, match="sequence of ATANCamera"):
        pkg.api._atan_cameras_arg(cams[0], None, None, cop, data)
    with pytest.raises(E, match="sequence of ATANCamera"):
        pkg.api._atan_cameras_arg([cams[0], pkg.PinholeCamera(640, 480, 420, 420, 320, 240)], None, None, cop, data)
    with pytest.raises(E, match="no cameras= or sizes="):
        pkg.api._atan_cameras_arg(list(cams), np.ones((5, 4)), None, cop, data)
    with pytest.raises(E, match="no cameras= or sizes="):
        pkg.api._atan_cameras_arg(list(cams), None, np.ones((5, 2), np.int32), cop, data)
    with pytest.raises(E, match="cam_of_pair must be"):
        pkg.api._atan_cameras_arg(list(cams), None, None, cop[:4], data)
    with pytest.raises(E, match="indexes 4 cameras"):
        pkg.api._atan_cameras_arg(list(cams), None, None, np.array([0, 1, 2, 3, 4]), data)
    with pytest.raises(E, match="pass camera= .* or cameras="):
        pkg.api._atan_cameras_arg(cams[0], np.ones((5, 4)), None, None, data)
    assert pkg.api._atan_cameras_arg(cams[0], None, None, None, data) is None
    arr = pkg.api._atan_cameras_arg(list(cams), None, None, cop, data)
    assert [(arr[i].width, arr[i].d0) for i in (0, 1)] == [(320, -0.3), (640, 0.3)]


def test_oracle_is_sensitive_to_the_camera(pkg, abi, synth, oracle_atan):
    """Control for the per-camera comparisons: aligning one camera's pairs with another fleet camera's parameters (at
    this camera's size) moves their poses by far more than the tolerance of the oracle comparisons."""
    cams = fleet(pkg)
    own, other = cams[3], cams[1]
    swapped = pkg.ATANCamera(own.width, own.height, other.struct.fx, other.struct.fy, other.struct.cx, other.struct.cy,
                             other.struct.d0)
    data = synth.make_atan_multicam_batch([own], np.zeros(4, int), n_pts=150, n_segs=30, seed=50)[1][0]
    a = oracle_atan.align(abi, own, data, n_threads=8)
    b = oracle_atan.align(abi, swapped, data, n_threads=8)
    ang, rel = synth.pose_error(a.T_cur_w, b.T_cur_w)
    assert np.median(ang) > 100 * POSE_TOL[0] and np.median(rel) > 100 * POSE_TOL[1], (ang, rel)


@pytest.fixture(scope="module")
def atan_hostmodel(tmp_path_factory):
    return _build_model(str(tmp_path_factory.mktemp("hostmodel") / "libplsvo_hostmodel_atan_multicam.so"))


def _build_model(out, abi_source=ABI_SOURCE):
    spec = importlib.util.spec_from_file_location("plsvo_hostmodel_build", os.path.join(HERE, "hostmodel", "build.py"))
    hm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(hm)
    sources = [abi_source] + hm.SOURCES[1:] + [os.path.join(HERE, "hostmodel", "fake_atan_multicam.cpp")]
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-Wno-unused-function", "-I" + hm.cuda_include(),
                    "-I" + os.path.join(ROOT, "pl-svo_b200", "csrc"), "-x", "c++", *sources, "-o", out, "-lpthread", "-ldl",
                    "-Wl,-Bsymbolic"], check=True)
    return out


def _run_model(lib, mode, k, oracle_lib=None):
    env = dict(os.environ, PLSVO_LIB=lib, PLSVO_FAKE_CUDA=mode)
    for name in [n for n in env if n.startswith("PLSVO_") and n not in ("PLSVO_LIB", "PLSVO_FAKE_CUDA")]:
        del env[name]
    if oracle_lib:
        env["PLSVO_FAKE_ORACLE"] = oracle_lib
    return subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-p", "no:cacheprovider",
                           "-k", k], env=env, capture_output=True, text=True, timeout=3000)


@pytest.mark.parametrize("mode", ["lazy", "eager"])
def test_gpu_tests_of_this_file_against_the_host_model(oracle, atan_hostmodel, mode):
    """The GPU tests below on the unchanged host code of plsvo_abi.cu with the model CUDA runtime: the model checks every
    access and the stream order, and digests each pair's own region at its own size.  The oracle tests and the
    shared-memory sweep need real kernels and are deselected."""
    p = _run_model(atan_hostmodel, mode, "not oracle and not every_variant and not shared_memory")
    assert p.returncode == 0 and " skipped" not in p.stdout and " passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


def _oracle_lib(oracle, oracle_atan):
    return os.path.join(ROOT, "oracle", "libplsvo_oracle.so")


FAULTS = {
    # every pair aligned with the distortion terms of cams[0]
    "every_pair_gets_cams0_terms": (
        "  int rc = multicam_check(c, c->h_mc_cams.data(), b, p);\n",
        "  for (size_t i = 1; i < B; ++i) std::copy(&c->h_atan_terms[0], &c->h_atan_terms[4], &c->h_atan_terms[4 * i]);\n"
        "  int rc = multicam_check(c, c->h_mc_cams.data(), b, p);\n",
        "fleet and full and shipped"),
    # the track call's pose optimiser given the normalised fx instead of errorMultiplier2() = fx_
    "track_gets_normalised_fx": (
        "  for (int i = 0; i < ab->batch; ++i) c->h_po_fx[i] = c->h_mc_cams[i].fx;\n",
        "  for (int i = 0; i < ab->batch; ++i) c->h_po_fx[i] = cams[i].fx;\n",
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
    p = _run_model(lib, "lazy", k + " and not oracle", _oracle_lib(oracle, oracle_atan))
    assert " passed" in p.stdout or " failed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]
    assert p.returncode != 0 and " failed" in p.stdout, f"{fault}: every test still passes — the model is blind to it"


def test_unmutated_track_and_fleet_pass_on_the_oracle_model(oracle, oracle_atan, atan_hostmodel):
    """The control of the seeded faults: the same selection on the unmutated host code passes."""
    p = _run_model(atan_hostmodel, "lazy", "(track or (fleet and full and shipped)) and not oracle", _oracle_lib(oracle, oracle_atan))
    assert p.returncode == 0 and " passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("B", [37, BIG])
@pytest.mark.parametrize("which", [0, 1])
def test_gpu_one_camera_equals_the_atan_call(pkg, synth, gen_device, which, B, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2" if B <= 132 else "128,4")
    cam = stock(pkg)[which]
    data = synth.make_atan_multicam_batch([cam], np.zeros(B, int), n_pts=150, n_segs=40, seed=100 + B + which, device=gen_device)[0]
    ragged(data, seed=B)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, camera=[cam], cam_of_pair=np.zeros(B, np.int32))
    want = pkg.SparseImgAlign(4, 2, 30).run(data, camera=cam)
    assert_same(got, want, ALIGN_FIELDS)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
def test_gpu_one_camera_every_variant(pkg, synth, gen_device, variant, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", variant)
    for which, cam in enumerate(stock(pkg)):
        data = synth.make_atan_multicam_batch([cam], np.zeros(37, int), n_pts=100, n_segs=24, seed=200 + which, device=gen_device)[0]
        got = pkg.SparseImgAlign(4, 2, 30).run(data, camera=[cam], cam_of_pair=np.zeros(37, np.int32))
        assert_same(got, pkg.SparseImgAlign(4, 2, 30).run(data, camera=cam), ALIGN_FIELDS, what=f"{variant} camera {which}")


def fleet_batch(pkg, synth, B, seed, device, fill=0, n_pts=150, n_segs=40):
    cams = fleet(pkg)
    groups = interleave(len(cams), B, seed)
    cop = cop_of(groups, B)
    data, parts, groups = synth.make_atan_multicam_batch(cams, cop, slot=slot_cam(synth, cams[0]), fill=fill, n_pts=n_pts,
                                                         n_segs=n_segs, seed=seed, device=device)
    return cams, cop, data, groups


@pytest.mark.gpu
@pytest.mark.parametrize("B", [37, BIG])
@pytest.mark.parametrize("bearings", ["full", "lean"])
@pytest.mark.parametrize("levels", ["shipped", "derived"])
def test_gpu_fleet_equals_per_camera_atan_calls(pkg, synth, gen_device, B, bearings, levels, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2" if B <= 132 else "128,4")
    cams, cop, data, groups = fleet_batch(pkg, synth, B, seed=300 + B, device=gen_device)
    ragged(data, seed=B, empty=(int(groups[3][0]),))  # ragged counts, masks, and an empty 320x240 pair
    if bearings == "lean":
        lean(data)
    if levels == "derived":  # level 2 shipped, 3 and 4 half-sampled on the device
        data.ref_pyr, data.cur_pyr = {2: data.ref_pyr[2]}, {2: data.cur_pyr[2]}
    got = pkg.SparseImgAlign(4, 2, 30).run(data, camera=list(cams), cam_of_pair=cop)
    assert_rows(got, per_camera(pkg, synth, data, cams, groups), "per camera")
    if not MODEL:
        assert all((got.n_tracked[idx] > 0).any() for idx in groups)


@pytest.mark.gpu
def test_gpu_padding_does_not_matter(pkg, synth, gen_device, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    outs = []
    for fill in (0, 255, np.random.default_rng(5)):
        cams, cop, data, _ = fleet_batch(pkg, synth, 37, seed=400, device=gen_device, fill=fill)
        outs.append(pkg.SparseImgAlign(4, 2, 30).run(data, camera=list(cams), cam_of_pair=cop))
    for o in outs[1:]:
        assert_same(o, outs[0], ALIGN_FIELDS)


@pytest.mark.gpu
def test_gpu_chains(pkg, synth, gen_device, monkeypatch):
    """One camera: the chain equals the ATAN chain call.  Several cameras of one size: the chained batch equals the same
    pairs as two stacks.  A size change inside a chain is rejected."""
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    vga = stock(pkg)[1]
    data = synth.make_chain_batch(cam=slot_cam(synth, vga), batch=9, n_pts=150, n_segs=40, seed=600, device=gen_device, atan=vga)
    data.frame_pyr = synth.chain_frames(data)
    one = pkg.SparseImgAlign(4, 2, 30).run(data, camera=[vga], cam_of_pair=np.zeros(9, np.int32))
    assert_same(one, pkg.SparseImgAlign(4, 2, 30).run(data, camera=vga), ALIGN_FIELDS, what="one camera")
    cams = [vga, pkg.ATANCamera(640, 480, 0.62, 0.86, 0.51, 0.49, 0.5), pkg.ATANCamera(640, 480, 0.7, 0.9, 0.48, 0.52, 0.0)]
    cop = np.array([0, 1, 2, 2, 1, 0, 1, 2, 0], np.int32)
    chained = pkg.SparseImgAlign(4, 2, 30).run(data, camera=cams, cam_of_pair=cop)
    stacks = copy.copy(data)
    stacks.frame_pyr = None
    assert_same(chained, pkg.SparseImgAlign(4, 2, 30).run(stacks, camera=cams, cam_of_pair=cop), ALIGN_FIELDS, what="chained")
    qvga = pkg.ATANCamera(320, 240, 0.62, 0.86, 0.51, 0.49, 0.5)
    with pytest.raises(pkg.api.PlsvoError, match=r"cams\[4\] is 640x480 and cams\[5\] is 320x240"):
        pkg.SparseImgAlign(4, 2, 30).run(data, camera=cams + [qvga], cam_of_pair=np.array([0, 1, 2, 2, 1, 3, 3, 3, 3], np.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("n_iter_ref", [None, 3])
@pytest.mark.parametrize("chained", [True, False])
def test_gpu_track_equals_per_camera_atan_track(pkg, synth, gen_device, chained, n_iter_ref, monkeypatch):
    monkeypatch.setenv("PLSVO_VARIANT", "256,2")
    cams = fleet(pkg)
    B = 16 if MODEL else 40
    groups = interleave(len(cams), B, 500)
    cop = cop_of(groups, B)
    data, po, parts, po_parts, groups = synth.make_atan_multicam_batch(cams, cop, slot=slot_cam(synth, cams[0]), poseopt=True,
                                                                       n_pts=150, n_segs=40, seed=500, device=gen_device)
    fields = ("T_f_w", "num_obs_pt", "status") if MODEL and not ORACLE_MODEL else PO_FIELDS
    got_a, got_p = pkg.api.track(data, po, po_n_iter_ref=n_iter_ref, chained=chained, camera=list(cams), cam_of_pair=cop)
    for cam, idx, po_k in zip(cams, groups, po_parts):
        want_a, want_p = pkg.api.track(crop(synth, data, idx, slot_cam(synth, cam)), po_k, po_n_iter_ref=n_iter_ref,
                                       chained=chained, camera=cam)
        assert_same(rows(got_a, idx), want_a, ALIGN_FIELDS, what=f"{cam.width}x{cam.height}")
        assert_same(rows(got_p, idx, fields), want_p, fields, what=f"{cam.width}x{cam.height}")


@pytest.mark.gpu
def test_gpu_fleet_against_the_oracle(pkg, abi, synth, oracle_atan, gen_device):
    from test_gpu_atan import compare

    cams, cop, data, groups = fleet_batch(pkg, synth, 24, seed=700, device=gen_device, n_pts=200, n_segs=50)
    got = pkg.SparseImgAlign(4, 2, 30).run(data, camera=list(cams), cam_of_pair=cop)
    for cam, idx in zip(cams, groups):
        want = oracle_atan.align(abi, cam, crop(synth, data, idx, slot_cam(synth, cam)), n_threads=8)
        compare(synth, rows(got, idx), want, f"{cam.width}x{cam.height} d0={cam.s_}")
    a0, t0 = synth.pose_error(data.T_cur_w, data.T_cur_w_gt)
    a1, t1 = synth.pose_error(got.T_cur_w, data.T_cur_w_gt)
    assert np.median(a1) < 0.25 * np.median(a0) and np.median(t1) < 0.25 * np.median(t0), (a0, a1, t0, t1)


@pytest.mark.gpu
def test_gpu_shared_memory_limit(pkg, abi, synth, gen_device, monkeypatch):
    """Point counts across the <256,2> limit: a pinned call runs, byte-identical to the pinned uniform ATAN call, or is
    refused with the plan's message; an unpinned call runs wherever the pinned uniform ATAN call does."""
    cam = stock(pkg)[1]
    base = synth.make_atan_multicam_batch([cam], np.zeros(2, int), n_pts=5800, n_segs=0, max_level=3, min_level=2, seed=800,
                                          device=gen_device)[0]
    ctx = pkg.Context(0)
    lib, ap = ctx.lib, abi.align_params(3, 2, 30)
    arr = abi.make_atan_cameras([cam.struct], np.zeros(2, np.int32), 2)
    largest = 0
    for n in range(5736, 5768):
        d = dataclasses.replace(base)
        d.pt_px, d.pt_f, d.pt_pos = (np.ascontiguousarray(a[:, :n]) for a in (base.pt_px, base.pt_f, base.pt_pos))
        ab, keep = abi.make_align_batch(d)
        outs = {}
        for name, variant, multi in (("uniform", "256,2", False), ("pinned", "256,2", True), ("free", "", True)):
            monkeypatch.setenv("PLSVO_VARIANT", variant)
            out = abi.AlignOut(2, 0)
            fn = lib.plsvo_align_atan_multicam_batch_run if multi else lib.plsvo_align_atan_batch_run
            rc = fn(ctx.handle, arr if multi else C.byref(cam.struct), C.byref(ab), C.byref(ap), C.byref(out.struct))
            outs[name] = (rc, lib.plsvo_last_error(ctx.handle).decode(), out)
        (urc, _, uout), (prc, pmsg, pout), (frc, fmsg, _) = outs["uniform"], outs["pinned"], outs["free"]
        assert prc in (abi.OK, abi.ERR_INVALID), (n, prc, pmsg)
        if urc == abi.OK:
            largest = n
        if prc == abi.OK:
            assert urc == abi.OK, n
            assert_same(pout, uout, ("T_cur_w", "n_tracked", "H", "iters", "status"), what=f"n_pts={n}")
        else:
            assert "shared-memory plan" in pmsg, (n, pmsg)
        if urc == abi.OK:
            assert frc == abi.OK, (n, fmsg)
    assert 0 < largest < 5767, "the sweep does not reach the limit of the <256,2> plan"
    ctx.close()


@pytest.mark.gpu
def test_gpu_malformed_calls_queue_nothing(pkg, abi, synth, gen_device):
    """Each malformed call returns PLSVO_ERR_INVALID with its message before anything is queued (against the host model:
    no stream operation ran or is pending); a valid call on the same context then succeeds.  Batches of no pairs or a
    negative count are rejected before any per-pair host array is sized by them, by the pinhole multicam track call too."""
    ctx = pkg.Context(0)
    lib = ctx.lib
    model = C.CDLL(os.environ["PLSVO_LIB"]) if MODEL else None
    if model:
        model.fake_cuda_ops_run.restype = C.c_ulonglong
    vga = stock(pkg)[1]
    d = synth.make_atan_multicam_batch([vga], np.zeros(3, int), n_pts=16, n_segs=4, seed=900, device=gen_device)[0]
    po = synth.make_poseopt_batch(cam=slot_cam(synth, vga), batch=3, n_pts=16, n_segs=4, seed=901)
    ab, keep_a = abi.make_align_batch(d)
    pb, keep_p = abi.make_poseopt_batch(po)
    ao, pout = abi.AlignOut(3, 4), abi.PoseOptOut(3, 16, 4)
    good = vga.struct

    def cams_with(i, **kw):
        cs = [abi.AtanCamera(*(getattr(good, f) for f, _ in abi.AtanCamera._fields_)) for _ in range(3)]
        for f, v in kw.items():
            setattr(cs[i], f, v)
        return (abi.AtanCamera * 3)(*cs)

    pinhole = abi.make_cameras(np.tile([vga.fx_, vga.fy_, vga.cx_, vga.cy_], (3, 1)), d.cam, 3)

    def run(cams, hi=4, track=False, flags=0, po_batch=3, batch=3, pinhole_track=False):
        ab.flags, pb.batch, ab.batch = flags, po_batch, batch
        ops = model.fake_cuda_ops_run() if model else 0
        launches = ctx.launch_count()
        if pinhole_track:
            rc = lib.plsvo_track_multicam_batch_run(ctx.handle, pinhole, C.byref(ab), C.byref(abi.align_params(hi, 2, 30)), C.byref(pb),
                                                    C.byref(abi.poseopt_params()), C.byref(ao.struct), C.byref(pout.struct))
        elif track:
            rc = lib.plsvo_track_atan_multicam_batch_run(ctx.handle, cams, C.byref(ab), C.byref(abi.align_params(hi, 2, 30)), C.byref(pb),
                                                         C.byref(abi.poseopt_params()), C.byref(ao.struct), C.byref(pout.struct))
        else:
            rc = lib.plsvo_align_atan_multicam_batch_run(ctx.handle, cams, C.byref(ab), C.byref(abi.align_params(hi, 2, 30)),
                                                         C.byref(ao.struct))
        if rc != abi.OK:
            assert ctx.launch_count() == launches, "a rejected call launched a kernel"
            if model:
                assert model.fake_cuda_pending_ops() == 0 and model.fake_cuda_ops_run() == ops, "a rejected call queued work"
        ab.flags, pb.batch, ab.batch = 0, 3, 3
        return rc, lib.plsvo_last_error(ctx.handle).decode()

    nan = float("nan")
    for cams, kw, msg in ((None, {}, "cams is NULL"),
                          (cams_with(1, d0=nan), {}, "cams[1] has a non-finite parameter"),
                          (cams_with(2, cx=float("inf")), {}, "cams[2] has a non-finite parameter"),
                          (cams_with(0, fx=0.0), {}, "cams[0] fx and fy must be positive"),
                          (cams_with(1, fy=-0.5), {}, "cams[1] fx and fy must be positive"),
                          (cams_with(2, fx=1e308), {}, "cams[2] focal length out of range"),
                          (cams_with(1, width=656), {}, "cams[1] is 656x480"),
                          (cams_with(1, height=481), {}, "cams[1] is 640x481"),
                          (cams_with(1, width=0), {}, "cams[1] is 0x480"),
                          (cams_with(2, width=-4), {"track": True}, "cams[2] is -4x480"),
                          (cams_with(0), {"batch": -1}, "batch/n_pts/n_segs out of range"),
                          (cams_with(0), {"batch": 0}, "batch/n_pts/n_segs out of range"),
                          (cams_with(0), {"batch": -1, "po_batch": -1, "track": True}, "batch/n_pts/n_segs out of range"),
                          (cams_with(0), {"batch": 0, "po_batch": 0, "track": True}, "batch/n_pts/n_segs out of range"),
                          (cams_with(0), {"batch": -1, "po_batch": -1, "pinhole_track": True}, "batch/n_pts/n_segs out of range"),
                          (cams_with(2, width=40, height=30), {"hi": 6}, "cams[2] is 40x30: pyramid level 5 smaller than one pixel"),
                          (cams_with(2, width=320, height=240), {"flags": abi.ALIGN_FRAME_CHAIN}, "cams[1] is 640x480 and cams[2] is 320x240"),
                          (cams_with(0), {"track": True, "po_batch": 2}, "batches differ in size")):
        rc, err = run(cams, **kw)
        assert rc == abi.ERR_INVALID and msg in err, (msg, err)
    # the host model of this file has no pinhole multicam alignment kernels: there a valid pinhole call is refused
    for kw in ({}, {"track": True}) + (() if MODEL else ({"pinhole_track": True},)):
        rc, err = run(cams_with(0), **kw)
        assert rc == abi.OK, (kw, err)
    ctx.close()
