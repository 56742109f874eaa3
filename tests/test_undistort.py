"""Frame rectification: vk::PinholeCamera::undistortImage (cv::initUndistortRectifyMap CV_16SC2 + cv::remap INTER_LINEAR)
followed by createImgPyramid, bit-exact.

CPU: the C++ oracle (oracle/undistort_oracle.cpp) and the independent NumPy restatement (oracle/np_undistort.py) agree on
maps and images, and both equal OpenCV: live when cv2 is importable, and always through the digests of cv2's output
committed in tests/golden/undistort_cv2.json (tests/golden/make_undistort_golden.py).  GPU: the device output equals the
oracle on every level.  The GPU tests also run here against the host model of the C ABI, linked with the model kernels of
tests/hostmodel/fake_undistort.cpp (the oracle's map, the real remap)."""
import ctypes as C
import hashlib
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "undistort_cv2.json")) as _f:
    GOLD = json.load(_f)
CAMS = GOLD["cameras"]
NAMES = list(CAMS)
EUROC, PINCUSHION, COPY, HD, ODD = "euroc_dataset_params", "vga_pincushion", "vga_d0_zero_is_a_copy", "hd720", "odd_641x479"


def params(name):
    return CAMS[name]["params"]


def cam_struct(abi, name):
    W, H, fx, fy, cx, cy, *d = params(name)
    return abi.PinholeCamera(W, H, fx, fy, cx, cy, (C.c_double * 5)(*d))


def frame(name):
    """The seeded frame the committed digests were computed from."""
    W, H = params(name)[:2]
    return np.random.default_rng(GOLD["frame_seed"] + CAMS[name]["index"]).integers(0, 256, (H, W), np.uint8)


def frames(name, B, seed=0):
    W, H = params(name)[:2]
    return np.random.default_rng(seed).integers(0, 256, (B, H, W), np.uint8)


def digest(a) -> str:
    a = np.ascontiguousarray(a)
    return hashlib.sha256(f"{a.dtype.str}{a.shape}".encode() + a.tobytes()).hexdigest()


def np_oracle():
    import np_undistort as m

    return m


@pytest.fixture(scope="session")
def uo(oracle):
    import undistort_oracle

    undistort_oracle.build()
    return undistort_oracle


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", NAMES)
def test_cpp_and_numpy_restatements_agree(uo, abi, oracle, name):
    npo = np_oracle()
    raw = frames(name, 2, seed=5)
    lv = uo.undistort(abi, cam_struct(abi, name), raw, 3)
    for b in range(2):
        np.testing.assert_array_equal(lv[0][b], npo.undistort_image(raw[b], *params(name)))
    for l, want in enumerate(oracle.pyramid(abi, lv[0], 3)):
        np.testing.assert_array_equal(lv[l], want)
    if npo.undistort_is_copy(params(name)[6]):
        np.testing.assert_array_equal(lv[0], raw)
    else:
        m1, m2 = uo.undistort_map(abi, cam_struct(abi, name))
        n1, n2 = npo.undistort_map(*params(name))
        np.testing.assert_array_equal(m1, n1)
        np.testing.assert_array_equal(m2, n2)


@pytest.mark.parametrize("name", NAMES)
def test_restatements_match_committed_opencv_digests(uo, abi, oracle, name):
    """0 mismatches against OpenCV: maps and the remapped frame, from the digests of cv2's own output."""
    npo, e, img = np_oracle(), CAMS[name], frame(name)
    assert digest(uo.undistort(abi, cam_struct(abi, name), img[None], 1)[0][0]) == e["image"]
    assert digest(npo.undistort_image(img, *params(name))) == e["image"]
    assert ("map1" in e) == (not npo.undistort_is_copy(params(name)[6]))
    if "map1" in e:
        m1, m2 = uo.undistort_map(abi, cam_struct(abi, name))
        assert (digest(m1), digest(m2)) == (e["map1"], e["map2"])
        n1, n2 = npo.undistort_map(*params(name))
        assert (digest(n1), digest(n2)) == (e["map1"], e["map2"])


@pytest.mark.parametrize("name", NAMES)
def test_restatements_match_live_cv2(uo, abi, oracle, name):
    cv2 = pytest.importorskip("cv2")
    W, H, fx, fy, cx, cy, *d = params(name)
    raw = frames(name, 1, seed=11)[0]
    got = uo.undistort(abi, cam_struct(abi, name), raw[None], 1)[0][0]
    if np_oracle().undistort_is_copy(d[0]):
        np.testing.assert_array_equal(got, raw)
        return
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    map1, map2 = cv2.initUndistortRectifyMap(K, np.array(d, np.float32), np.eye(3), K, (W, H), cv2.CV_16SC2)
    m1, m2 = uo.undistort_map(abi, cam_struct(abi, name))
    np.testing.assert_array_equal(m1, map1)
    np.testing.assert_array_equal(m2, map2)
    np.testing.assert_array_equal(got, cv2.remap(raw, map1, map2, cv2.INTER_LINEAR))


def test_pincushion_camera_samples_far_outside_the_frame(uo, abi, oracle):
    """The border path is exercised: corners of the pincushion camera read pixels hundreds of pixels outside."""
    m1, _ = uo.undistort_map(abi, cam_struct(abi, PINCUSHION))
    W, H = params(PINCUSHION)[:2]
    assert m1[..., 0].min() < -500 and m1[..., 0].max() > W + 500 and m1[..., 1].min() < -300 and m1[..., 1].max() > H + 300


def test_library_defines_both_undistort_launchers(pkg):
    """plsvo_abi.cu reaches the two launchers through weak references (so that the host model links without them): the
    product library must define both, or plsvo_undistort_batch_run would only ever report them missing."""
    syms = subprocess.check_output(["nm", "-DC", "--defined-only", pkg.abi.LIB_PATH], text=True)
    assert "plsvo::undistort_map_launch(" in syms and "plsvo::undistort_remap_launch(" in syms


@pytest.fixture(scope="module")
def undistort_hostmodel(tmp_path_factory):
    """The host model of tests/hostmodel/build.py, linked with the model undistortion kernels of fake_undistort.cpp."""
    spec = importlib.util.spec_from_file_location("plsvo_hostmodel_build", os.path.join(HERE, "hostmodel", "build.py"))
    hm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(hm)
    out = str(tmp_path_factory.mktemp("hostmodel") / "libplsvo_hostmodel_undistort.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-Wno-unused-function", "-I" + hm.cuda_include(),
                    "-x", "c++", *hm.SOURCES, os.path.join(HERE, "hostmodel", "fake_undistort.cpp"), "-o", out, "-lpthread", "-ldl",
                    "-Wl,-Bsymbolic"], check=True)
    return out


@pytest.mark.parametrize("mode", ["lazy", "eager"])
def test_gpu_tests_of_this_file_against_the_host_model(uo, undistort_hostmodel, mode):
    """The GPU tests below, run against the unchanged host code of plsvo_abi.cu on the model CUDA runtime, with the map
    build answered by the oracle and the remap computed by the model kernel: uploads, layouts, the map cache, the
    validation exits and the downloads are checked without a GPU (the kernels are not).  No test may be skipped."""
    env = dict(os.environ, PLSVO_LIB=undistort_hostmodel, PLSVO_FAKE_CUDA=mode)
    p = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-p", "no:cacheprovider"],
                       env=env, capture_output=True, text=True, timeout=1200)
    assert p.returncode == 0 and " skipped" not in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def remap_kernels(pkg, abi):
    """Tests of a distorted camera need the map and remap kernels.  The library always has them (see
    test_library_defines_both_undistort_launchers); only the stock host model of the GPU pre-flight lacks them."""
    ctx = pkg.api.Context(0)
    cam = pkg.PinholeCamera(16, 16, 10.0, 10.0, 8.0, 8.0, -0.1)
    raw = np.zeros((1, 16, 16), np.uint8)
    levels, r = abi.pyramid_levels(1, 16, 16, 1)
    b = abi.UndistortBatch(cam.struct, 1, 1, raw.ctypes.data_as(C.POINTER(C.c_uint8)), 16, 256)
    rc = ctx.lib.plsvo_undistort_batch_run(ctx.handle, C.byref(b), C.byref(r))
    msg = ctx.lib.plsvo_last_error(ctx.handle).decode()
    ctx.close()
    if rc != abi.OK and "not linked" in msg and os.environ.get("PLSVO_LIB"):
        pytest.skip(f"{os.environ['PLSVO_LIB']}: {msg}")
    assert rc == abi.OK, msg


def need_kernels(request, name):
    if name != COPY:
        request.getfixturevalue("remap_kernels")


def _check_levels(got, want, n_levels):
    assert len(got) == n_levels
    for l in range(n_levels):
        assert got[l].shape == want[l].shape
        np.testing.assert_array_equal(got[l], want[l], err_msg=f"level {l}")


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("name", NAMES)
def test_gpu_undistort_is_bit_exact(request, uo, pkg, abi, oracle, name, B):
    need_kernels(request, name)
    raw = frames(name, B, seed=B)
    got = pkg.PinholeCamera(*params(name)).undistortImage(raw, 5)
    _check_levels(got, uo.undistort(abi, cam_struct(abi, name), raw, 5, n_threads=8), 5)


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,n_levels", [(EUROC, 256, 5), (EUROC, 3, 1), (HD, 3, 7), (ODD, 3, 7), (PINCUSHION, 3, 1), (COPY, 3, 7),
                                             (COPY, 2, 1)])
def test_gpu_undistort_batch_and_depth(request, uo, pkg, abi, oracle, name, B, n_levels):
    need_kernels(request, name)
    raw = frames(name, B, seed=100 + n_levels)
    got = pkg.PinholeCamera(*params(name)).undistortImage(raw, n_levels)
    _check_levels(got, uo.undistort(abi, cam_struct(abi, name), raw, n_levels, n_threads=8), n_levels)


@pytest.mark.gpu
def test_gpu_pyramid_levels_are_create_img_pyramid_of_the_rectified_frame(remap_kernels, uo, pkg, abi, oracle):
    raw = frames(ODD, 3, seed=21)
    got = pkg.PinholeCamera(*params(ODD)).undistortImage(raw, 6)
    rect = uo.undistort(abi, cam_struct(abi, ODD), raw, 1)[0]
    _check_levels(got, oracle.pyramid(abi, rect, 6), 6)
    _check_levels(got, pkg.createImgPyramid(rect, 6), 6)


@pytest.mark.gpu
def test_gpu_padded_pitch_and_strided_frames(remap_kernels, uo, pkg, abi, oracle):
    W, H = params(EUROC)[:2]
    base = np.random.default_rng(31).integers(0, 256, (6, H + 3, W + 37), np.uint8)
    cam = pkg.PinholeCamera(*params(EUROC))
    for raw in (base[:, :H, :W], base[::2, 1:H + 1, 5:W + 5]):  # padded rows; padded rows and every other frame
        assert raw.strides[1] != W
        _check_levels(cam.undistortImage(raw, 4), uo.undistort(abi, cam_struct(abi, EUROC), np.ascontiguousarray(raw), 4), 4)
    # padded, non-contiguous output levels through the C ABI
    raw = base[:, :H, :W]
    want = uo.undistort(abi, cam_struct(abi, EUROC), np.ascontiguousarray(raw), 3)
    outs, r = [], abi.PyramidResult()
    for l in range(3):
        h, w = H >> l, W >> l
        buf = np.full((6, h + 2, w + 19), 7, np.uint8)
        outs.append(buf)
        r.level[l] = buf.ctypes.data_as(C.POINTER(C.c_uint8))
        r.pitch[l], r.stride[l] = buf.strides[1], buf.strides[0]
    b = abi.UndistortBatch(cam.struct, 6, 3, raw.ctypes.data_as(C.POINTER(C.c_uint8)), raw.strides[1], raw.strides[0])
    ctx = pkg.api.default_context()
    ctx.check(ctx.lib.plsvo_undistort_batch_run(ctx.handle, C.byref(b), C.byref(r)), "plsvo_undistort_batch_run")
    for l in range(3):
        h, w = H >> l, W >> l
        np.testing.assert_array_equal(outs[l][:, :h, :w], want[l])
        assert (outs[l][:, h:, :] == 7).all() and (outs[l][:, :, w:] == 7).all(), "bytes outside the levels were written"


@pytest.mark.gpu
def test_gpu_two_cameras_alternating_in_one_context(remap_kernels, uo, pkg, abi, oracle):
    """The map is cached per context and keyed by the whole camera: a different camera rebuilds it, the same one does not."""
    ctx = pkg.api.Context(0)
    a, b = pkg.PinholeCamera(*params(EUROC)), pkg.PinholeCamera(*params("vga_strong_barrel_k3"))
    a2 = pkg.PinholeCamera(*params(EUROC)[:10], 0.001)  # same size, k3 differs
    built = []
    for k, (cam, name) in enumerate([(a, EUROC), (a, EUROC), (b, "vga_strong_barrel_k3"), (a, EUROC), (a2, None), (a, EUROC)]):
        raw = frames(EUROC if name is None else name, 2, seed=40 + k)
        got = cam.undistortImage(raw, 2, ctx)
        want = uo.undistort(abi, cam.struct, raw, 2)
        _check_levels(got, want, 2)
        built.append(ctx.last_map_build_ms() is not None)
        assert ctx.last_kernel_ms() >= 0
    assert built == [True, False, True, True, True, True]
    pkg.PinholeCamera(*params(COPY)).undistortImage(frames(COPY, 1), 1, ctx)
    assert ctx.last_map_build_ms() is None  # d0 = 0: no map
    ctx.close()


@pytest.mark.gpu
def test_gpu_validation_errors(uo, pkg, abi):
    ctx = pkg.api.Context(0)
    W, H = 64, 48
    good = [W, H, 50.0, 50.0, 32.0, 24.0, -0.2, 0.05, 0.0, 0.0, 0.0]
    raw = np.zeros((2, H, W), np.uint8)

    def run(cam_params=good, B=2, n_levels=2, img=raw, pitch0=None, out_edit=None):
        cam = pkg.PinholeCamera(*cam_params)
        b = abi.UndistortBatch(cam.struct, B, n_levels, img.ctypes.data_as(C.POINTER(C.c_uint8)) if img is not None else None,
                               raw.strides[1] if pitch0 is None else pitch0, raw.strides[0])
        levels, r = abi.pyramid_levels(2, H, W, max(1, min(n_levels, 7)))
        if out_edit:
            out_edit(r)
        rc = ctx.lib.plsvo_undistort_batch_run(ctx.handle, C.byref(b), C.byref(r))
        return rc, ctx.lib.plsvo_last_error(ctx.handle).decode()

    def with_param(i, v):
        p = list(good)
        p[i] = v
        return p

    def null_level(l):
        def f(r):
            r.level[l] = None
        return f

    def small_pitch(r):
        r.pitch[1] = (W >> 1) - 1

    cases = [
        (dict(B=0), "positive"), (dict(cam_params=with_param(0, 0)), "positive"), (dict(cam_params=with_param(1, -4)), "positive"),
        (dict(n_levels=0), "n_levels"), (dict(n_levels=8), "n_levels"), (dict(img=None), "img0"), (dict(pitch0=W - 1), "pitch0"),
        (dict(out_edit=null_level(0)), "output level missing"), (dict(out_edit=null_level(1)), "output level missing"),
        (dict(out_edit=small_pitch), "output pitch"), (dict(n_levels=7, cam_params=[8, 8] + good[2:]), "smaller than one pixel"),
        (dict(cam_params=with_param(2, float("nan"))), "not finite"), (dict(cam_params=with_param(8, float("inf"))), "not finite"),
        (dict(cam_params=with_param(5, 1e300)), "not finite"), (dict(cam_params=with_param(2, 0.0)), "non-zero"),
        (dict(cam_params=with_param(3, 0.0)), "non-zero"), (dict(cam_params=with_param(3, 1e-60)), "non-zero"),
    ]
    for kw, msg in cases:
        rc, err = run(**kw)
        assert rc == abi.ERR_INVALID and msg in err, (kw, rc, err)
    assert ctx.lib.plsvo_undistort_batch_run(ctx.handle, None, None) == abi.ERR_INVALID
    assert run(cam_params=with_param(6, 0.0))[0] == abi.OK  # the context is still usable
    with pytest.raises(pkg.api.PlsvoError):
        pkg.PinholeCamera(*good).undistortImage(np.zeros((1, H, W + 1), np.uint8), 1, ctx)
    ctx.close()
