"""The undistortion kernels (undistort_kernel.cu) against the CPU oracle, case by case: the map and remap kernels through
plsvo_undistort_batch_run, the fused rectify + pyramid kernel through plsvo_align_raw_batch_run /
plsvo_track_raw_batch_run with rect_out, and its multicam form through plsvo_align_raw_multicam_batch_run.

The reference of every GPU comparison is the CPU oracle: oracle/undistort_oracle.cpp for the rectified frame, then the
2x2 mean of tests/test_gpu_pyramid_cases.py level by level; every level is compared byte for byte.  The cases
(tests/undistort_cases.py):
  * cameras: barrel, pincushion, tangential-only, non-square, principal point off-centre and outside the frame, negative
    fx and/or fy, d0 = +-1e-7 (a copy) and +-1.0000001e-7 (a map), scaled to every frame size; three dyadic cameras whose
    map reaches exact cvRound ties; four cameras whose map leaves the int16 range (int16 wrap, int overflow to INT_MIN,
    infinite coordinates) and one whose u or v is infinite;
  * sizes on both sides of the remap tile (64 x 16) and the fused tile (64 x 64), every legal level count;
  * random frames, all 255 and a 0/255 checkerboard; padded and strided inputs, guarded padded outputs; batches on both
    sides of the remap's and the fused kernel's frame-run split; a multicam slot of mixed cameras and sizes.

Outside the int16 range the kernels keep OpenCV's scalar loop: (short)(cvRound(u * 32) >> 5) wraps, and a cvRound out
of int range (or of an infinite value) is INT_MIN, so map1 = (0, 0) there.  cv2 4.x agrees in its scalar tail columns
and saturates in its vectorised ones; the CPU section pins both, live when cv2 is importable and otherwise through
tests/golden/undistort_cases_cv2.{json,npz} (tests/golden/make_undistort_cases_golden.py).  Guard tests keep every
special camera special.  The GPU section also runs against the host model of the C ABI."""
import ctypes as C
import hashlib
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import np_undistort as npu
from test_gpu_pyramid_cases import deepest, new_ctx, np_pyramid  # noqa: F401  (new_ctx: fixture)
from test_raw_track import ALIGN_FIELDS, POSE_FIELDS
from test_undistort import remap_kernels, uo  # noqa: F401  (fixtures)
from undistort_cases import DIGEST_SIZES, HEIGHTS, INF, OOR_SIZES, SMALL_OOR_SIZES, TIES, WIDTHS, frames, in_range, out_of_range, special

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MODEL = bool(os.environ.get("PLSVO_FAKE_CUDA"))
# the host model's pose-optimiser digest writes only these outputs
PO_FIELDS = ("T_f_w", "num_obs_pt", "status") if MODEL else POSE_FIELDS
TINY = 2001 if MODEL else 70001  # the host model rectifies on the CPU
GUARD = 0xA5
INT_MIN = -2 ** 31
with open(os.path.join(HERE, "golden", "undistort_cases_cv2.json")) as _f:
    GOLD = json.load(_f)


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


def struct(abi, p):
    W, H, fx, fy, cx, cy, *d = p
    return abi.PinholeCamera(W, H, fx, fy, cx, cy, (C.c_double * 5)(*d))


def oracle_levels(uo, abi, p, raw, n_levels):
    """undistortImage by the C++ oracle, then the 2x2-mean pyramid: n_levels arrays [B, H>>l, W>>l]."""
    return np_pyramid(uo.undistort_level0(abi, struct(abi, p), raw, n_threads=8), n_levels)


def check_levels(got, want, what):
    assert len(got) >= len(want), what
    for l, w in enumerate(want):
        assert got[l].shape == w.shape, (what, l, got[l].shape, w.shape)
        np.testing.assert_array_equal(got[l], w, err_msg=f"{what}: level {l}")


def scalar(p):
    """u * 32, v * 32 and their cvRound of every entry of camera p's map (NumPy restatement)."""
    with np.errstate(all="ignore"):
        u, v = npu.undistort_coords(*p)
    return u, v, npu.cv_round(u), npu.cv_round(v)


def is_tie(t):
    with np.errstate(invalid="ignore"):
        return np.abs(t - np.floor(t)) == 0.5


def near_tie(t):
    with np.errstate(invalid="ignore"):
        return np.abs(np.abs(t - np.floor(t)) - 0.5) <= 1e-6


def wrapped(iu, iv):
    """Entries where (short)(i >> 5) is not i >> 5 in either coordinate."""
    s = np.stack([iu >> 5, iv >> 5], -1)
    return ((s < -32768) | (s > 32767)).any(-1)


def digest(a) -> str:
    a = np.ascontiguousarray(a)
    return hashlib.sha256(f"{a.dtype.str}{a.shape}".encode() + a.tobytes()).hexdigest()


def sm_count():
    """The device's SM count, as the launchers read it (the host model answers for its own device)."""
    if MODEL:
        v = C.c_int()
        assert C.CDLL(os.environ["PLSVO_LIB"]).cudaDeviceGetAttribute(C.byref(v), 16, 0) == 0  # cudaDevAttrMultiProcessorCount
        return v.value
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_in_range_cameras_stay_inside_int16_at_every_size():
    """Guard: the in-range cameras keep |u|, |v| < 32768 pixels at every size (finite, no wrap), the tie cameras too."""
    cams = [p for W in WIDTHS for H in HEIGHTS for p in in_range(W, H).values()] + list(TIES.values())
    for p in cams:
        u, v, _, _ = scalar(p)
        assert np.isfinite(u).all() and np.isfinite(v).all() and max(np.abs(u).max(), np.abs(v).max()) < 2 ** 20, p


@pytest.mark.parametrize("name", sorted(TIES))
def test_tie_cameras_reach_exact_ties_that_change_the_frame(name):
    """Guard: exact cvRound ties, and round half away from zero in their place changes a byte of a rectified test frame."""
    p = TIES[name]
    u, v, iu, iv = scalar(p)
    ties = is_tie(u) | is_tie(v)
    assert ties.sum() >= 1, name
    away = lambda t: (np.sign(t) * np.floor(np.abs(t) + 0.5)).astype(np.int64)  # noqa: E731
    raw = frames(2, p[1], p[0], seed=11)
    want = npu.remap_linear(raw, *npu.map_of_rounded(iu, iv))
    assert (npu.remap_linear(raw, *npu.map_of_rounded(away(u), away(v))) != want).any(), name


def test_out_of_range_cameras_reach_int_min_infinity_and_wrap():
    """Guard, at 640 x 480: every out-of-range camera wraps int16, the huge and the subnormal-fx ones reach INT_MIN, the
    subnormal-fx and the infinite camera reach infinite coordinates, the wrap camera puts wrapped entries inside the frame;
    and saturating in place of INT_MIN changes a byte of a rectified test frame."""
    cams = out_of_range(640, 480)
    st = {n: scalar(p) for n, p in cams.items()}
    st["inf"] = scalar(INF)
    for n, (u, v, iu, iv) in st.items():
        assert wrapped(iu, iv).any(), n
    for n in ("oor_huge", "oor_subnormal_fx", "inf"):
        assert ((st[n][2] == INT_MIN) | (st[n][3] == INT_MIN)).any(), n
    for n in ("oor_subnormal_fx", "inf"):
        assert (np.isinf(st[n][0]) | np.isinf(st[n][1])).any(), n
    u, v, iu, iv = st["oor_wrap"]
    m1, _ = npu.map_of_rounded(iu, iv)
    inside = wrapped(iu, iv) & (m1[..., 0] >= 0) & (m1[..., 0] < 640) & (m1[..., 1] >= 0) & (m1[..., 1] < 480)
    assert inside.sum() >= 1

    def saturating(t):
        with np.errstate(invalid="ignore"):
            r = np.rint(t)
            return np.where(np.isnan(r), INT_MIN, np.clip(np.nan_to_num(r, nan=0.0), INT_MIN, 2 ** 31 - 1)).astype(np.int64)

    changed = []
    for n, p in list(cams.items()) + [("inf", INF)]:
        u, v, iu, iv = st[n]
        raw = frames(2, p[1], p[0], seed=12)
        want = npu.remap_linear(raw, *npu.map_of_rounded(iu, iv))
        changed.append((npu.remap_linear(raw, *npu.map_of_rounded(saturating(u), saturating(v))) != want).any())
    assert any(changed), changed


CPU_CASES = {**{f"{n}@{W}x{H}": p for W, H in ((641, 479), (65, 17), (7, 3), (1, 1)) for n, p in in_range(W, H).items()}, **special()}


@pytest.mark.parametrize("key", list(CPU_CASES))
def test_cpp_and_numpy_restatements_agree(uo, abi, key):
    """Maps and rectified frames bit for bit, through infinite coordinates, int overflow and int16 wrap."""
    p = CPU_CASES[key]
    W, H = p[:2]
    raw = frames(2, H, W, seed=13)
    with np.errstate(all="ignore"):
        n1, n2 = npu.undistort_map(*p)
        img = npu.undistort_image(raw, *p)
    m1, m2 = uo.undistort_map(abi, struct(abi, p))
    np.testing.assert_array_equal(m1, n1)
    np.testing.assert_array_equal(m2, n2)
    np.testing.assert_array_equal(uo.undistort_level0(abi, struct(abi, p), raw), img)
    if npu.undistort_is_copy(p[6]):
        np.testing.assert_array_equal(img, raw)


def test_int_min_entries_are_map1_zero(uo, abi):
    """OpenCV's scalar loop: cvRound out of int range (or of an infinite value) is INT_MIN, and INT_MIN >> 5 casts to 0
    with low bits 0, so the coordinate samples column (or row) 0 at weight 32."""
    for p in (out_of_range(640, 480)["oor_huge"], INF):
        _, _, iu, iv = scalar(p)
        m1, m2 = uo.undistort_map(abi, struct(abi, p))
        assert (m1[..., 0][iu == INT_MIN] == 0).all() and ((m2 & 31)[iu == INT_MIN] == 0).all()
        assert (m1[..., 1][iv == INT_MIN] == 0).all() and ((m2 >> 5)[iv == INT_MIN] == 0).all()


def opencv_contract(p, c1, c2, what):
    """cv2's map (c1, c2) against the scalar-loop map of camera p, entry by entry, away from (1e-6 of) a rounding tie,
    where cv2's vectorised arithmetic may round the other way: where both scalar values fit int16, map1 and map2 are
    equal; elsewhere each map1 value is the scalar loop's (wrapped) value, its saturation, or -32768 when a coordinate
    left the int range.  Returns the counts of (wrapped, saturated) map1 values that differ from the other kind."""
    u, v, iu, iv = scalar(p)
    m1, m2 = npu.map_of_rounded(iu, iv)
    s = np.stack([iu >> 5, iv >> 5], -1)
    fit = ((s >= -32768) & (s <= 32767)).all(-1)
    far = ~(near_tie(u) | near_tie(v))
    a = fit & far
    np.testing.assert_array_equal(c1[a], m1[a], err_msg=f"{what}: map1 where the scalar value fits int16")
    np.testing.assert_array_equal(c2[a], m2[a], err_msg=f"{what}: map2 where the scalar value fits int16")
    sat = np.clip(s, -32768, 32767)
    overflow = ((iu == INT_MIN) | (iv == INT_MIN))[..., None]
    ok = (c1 == m1) | (c1 == sat) | ((c1 == -32768) & overflow)
    assert ok[~fit & far].all(), f"{what}: a map1 value outside the int16 range is neither wrapped nor saturated"
    kinds = ~fit[..., None] & far[..., None] & (m1 != sat)
    return int((kinds & (c1 == m1)).sum()), int((kinds & (c1 == sat)).sum())


def check_opencv_out_of_range(maps_of):
    """The out-of-range contract at the small sizes: the contract above; every entry equal where the frame is narrower
    than cv2's vector block (W < 8: the scalar loop only); both kinds where vectorised columns and a tail meet (61 x 45)."""
    kinds = {}
    for W, H in SMALL_OOR_SIZES:
        for n, p in out_of_range(W, H).items():
            c1, c2 = maps_of(f"{n}@{W}x{H}")
            kinds[(n, W)] = opencv_contract(p, c1, c2, f"{n}@{W}x{H}")
            if W < 8:
                m1, m2 = npu.map_of_rounded(*scalar(p)[2:])
                np.testing.assert_array_equal(c1, m1)
                np.testing.assert_array_equal(c2, m2)
    c1, c2 = maps_of("inf@64x48")
    opencv_contract(INF, c1, c2, "inf@64x48")
    wrap61 = sum(kinds[(n, 61)][0] for n in out_of_range(61, 45))
    sat61 = sum(kinds[(n, 61)][1] for n in out_of_range(61, 45))
    assert wrap61 > 0 and sat61 > 0, (wrap61, sat61)
    assert sum(kinds[(n, W)][0] for n in out_of_range(7, 5) for W in (7, 3)) > 0


def cv2_map(cv2, p):
    W, H, fx, fy, cx, cy, *d = p
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    return cv2.initUndistortRectifyMap(K, np.array(d, np.float32), np.eye(3), K, (W, H), cv2.CV_16SC2)


def golden_cases():
    """The cameras of the committed digests: the in-range cameras at DIGEST_SIZES and the tie cameras."""
    cases = {f"{n}@{W}x{H}": p for W, H in DIGEST_SIZES for n, p in in_range(W, H).items()}
    cases.update({f"{n}@640x480": p for n, p in TIES.items()})
    return cases


def test_committed_fixture_covers_the_cases():
    """The fixture was made from the cameras of undistort_cases as they stand: the same keys, by cv2 4.13."""
    assert set(GOLD["digests"]) == set(golden_cases())
    z = np.load(os.path.join(HERE, "golden", "undistort_cases_cv2.npz"))
    keys = {k.rsplit(":", 1)[0] for k in z.files if ":" in k}
    assert keys == {f"{n}@{W}x{H}" for W, H in SMALL_OOR_SIZES for n in out_of_range(W, H)} | {"inf@64x48"}
    assert GOLD["opencv"].startswith("4.13") and str(z["opencv"]).startswith("4.13")


@pytest.mark.parametrize("key", list(golden_cases()))
def test_in_range_maps_and_frames_match_committed_opencv_digests(uo, abi, key):
    p, e = golden_cases()[key], GOLD["digests"][key]
    W, H = p[:2]
    img = frames(1, H, W, GOLD["frame_seed"])[0]
    assert digest(uo.undistort_level0(abi, struct(abi, p), img[None])[0]) == e["image"]
    assert ("map1" in e) == (not npu.undistort_is_copy(p[6]))
    if "map1" in e:
        m1, m2 = uo.undistort_map(abi, struct(abi, p))
        assert (digest(m1), digest(m2)) == (e["map1"], e["map2"])


def test_out_of_range_maps_against_committed_opencv_maps():
    z = np.load(os.path.join(HERE, "golden", "undistort_cases_cv2.npz"))
    check_opencv_out_of_range(lambda key: (z[key + ":map1"], z[key + ":map2"]))


@pytest.mark.parametrize("key", list(golden_cases()))
def test_in_range_maps_and_frames_match_live_cv2(uo, abi, key):
    cv2 = pytest.importorskip("cv2")
    p = golden_cases()[key]
    W, H = p[:2]
    raw = frames(1, H, W, seed=14)[0]
    got = uo.undistort_level0(abi, struct(abi, p), raw[None])[0]
    if npu.undistort_is_copy(p[6]):
        np.testing.assert_array_equal(got, raw)
        return
    map1, map2 = cv2_map(cv2, p)
    m1, m2 = uo.undistort_map(abi, struct(abi, p))
    np.testing.assert_array_equal(m1, map1)
    np.testing.assert_array_equal(m2, map2)
    np.testing.assert_array_equal(got, cv2.remap(raw, map1, map2, cv2.INTER_LINEAR))


# at 640 x 480, of 307,200: map entries where cv2 4.13's map1 differs from the scalar loop's, and pixels of the frame
# frames(1, 480, 640, 9300)[0] rectified differently (DESIGN.md)
CV2_MAP_DIFFERENCES = {"oor_wrap": 91339, "oor_huge": 306501, "oor_f60": 224612, "oor_subnormal_fx": 306720}
CV2_FRAME_DIFFERENCES = {"oor_wrap": 6, "oor_huge": 237963, "oor_f60": 33, "oor_subnormal_fx": 306720}


def test_out_of_range_maps_against_live_cv2(uo, abi):
    cv2 = pytest.importorskip("cv2")
    check_opencv_out_of_range(lambda key: cv2_map(cv2, special()[key]))
    for W, H in OOR_SIZES[:2]:  # the VGA frames: saturation only at 640, a wrapping tail column at 641
        kinds = [opencv_contract(p, *cv2_map(cv2, p), f"{n}@{W}x{H}") for n, p in out_of_range(W, H).items()]
        assert sum(k[1] for k in kinds) > 0 and (sum(k[0] for k in kinds) > 0) == (W == 641), kinds
    img = frames(1, 480, 640, 9300)[0]
    for n, p in out_of_range(640, 480).items():
        c1, c2 = cv2_map(cv2, p)
        assert int((c1 != uo.undistort_map(abi, struct(abi, p))[0]).any(-1).sum()) == CV2_MAP_DIFFERENCES[n], n
        got = uo.undistort_level0(abi, struct(abi, p), img[None])[0]
        assert int((got != cv2.remap(img, c1, c2, cv2.INTER_LINEAR)).sum()) == CV2_FRAME_DIFFERENCES[n], n


# ---------------------------------------------------------------------------------------------------------------- host model
@pytest.fixture(scope="module")
def cases_hostmodel(tmp_path_factory):
    """The host model of tests/hostmodel/build.py with the undistortion, fused and mixed-size multicam model kernels."""
    spec = importlib.util.spec_from_file_location("plsvo_hostmodel_build", os.path.join(HERE, "hostmodel", "build.py"))
    hm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(hm)
    out = str(tmp_path_factory.mktemp("hostmodel") / "libplsvo_hostmodel_undistort_cases.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-Wno-unused-function", "-I" + hm.cuda_include(),
                    "-I" + os.path.join(ROOT, "pl-svo_b200", "csrc"), "-x", "c++", *hm.SOURCES,
                    *(os.path.join(HERE, "hostmodel", f) for f in ("fake_undistort.cpp", "fake_raw_pyramid.cpp", "fake_mixed_sizes.cpp")),
                    "-o", out, "-lpthread", "-ldl", "-Wl,-Bsymbolic"], check=True)
    return out


@pytest.mark.parametrize("mode", ["lazy", "eager"])
def test_gpu_tests_of_this_file_against_the_host_model(oracle, cases_hostmodel, mode):
    """The GPU tests below on the unchanged host code of plsvo_abi.cu with the model CUDA runtime: the map is the
    oracle's, remap and the fused kernels compute for real on the CPU, alignment and pose optimisation digest their
    inputs.  Layouts, uploads, the frame-run arithmetic's inputs, the slot padding and every access are checked; the
    device kernels are not.  No test may be skipped."""
    env = dict(os.environ, PLSVO_LIB=cases_hostmodel, PLSVO_FAKE_CUDA=mode)
    for name in [n for n in env if n.startswith("PLSVO_") and n not in ("PLSVO_LIB", "PLSVO_FAKE_CUDA")]:
        del env[name]
    p = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-p", "no:cacheprovider"],
                       env=env, capture_output=True, text=True, timeout=3000)
    assert p.returncode == 0 and " skipped" not in p.stdout and " passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------------------- GPU
# ---- plsvo_undistort_batch_run: map, remap, pyramid ------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("W", WIDTHS)
def test_undistort_every_camera_and_size(remap_kernels, uo, pkg, abi, new_ctx, W):
    """Every in-range camera at every height, at the deepest level count; the barrel camera at every smaller count, and
    one level more is refused."""
    ctx = new_ctx()
    for H in HEIGHTS:
        raw = frames(2, H, W, seed=W * 1000 + H)
        top = deepest(W, H)
        for name, p in in_range(W, H).items():
            want = oracle_levels(uo, abi, p, raw, top)
            check_levels(pkg.PinholeCamera(*p).undistortImage(raw, top, ctx), want, f"{name} {W}x{H}")
            if name == "barrel":
                for n in range(1, top):
                    check_levels(pkg.PinholeCamera(*p).undistortImage(raw, n, ctx), want[:n], f"{name} {W}x{H}, {n} levels")
                with pytest.raises(pkg.api.PlsvoError, match="smaller than one pixel" if top < 7 else "n_levels"):
                    pkg.PinholeCamera(*p).undistortImage(raw, top + 1, ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(special()))
def test_undistort_tie_and_out_of_range_cameras(remap_kernels, uo, pkg, abi, key):
    p = special()[key]
    W, H = p[:2]
    raw = frames(2, H, W, seed=21)
    top = deepest(W, H)
    check_levels(pkg.PinholeCamera(*p).undistortImage(raw, top), oracle_levels(uo, abi, p, raw, top), key)


def raw_views(W, H, n, seed):
    """Raw stacks of n frames in three layouts: rows padded to a pitch that is not a multiple of 4 with contiguous frames
    (one linear copy), padded rows in padded frames, and every other frame of such a stack."""
    rng = np.random.default_rng(seed)
    pad = 1 if (W + 1) % 4 else 2
    uniform = rng.integers(0, 256, (n, H, W + pad), dtype=np.uint8)[:, :, :W]
    big = rng.integers(0, 256, (2 * n, H + 3, W + 37), dtype=np.uint8)
    for a in (uniform, big):
        a[1] = 255
        y, x = np.mgrid[:H, :W]
        a[2, :H, :W] = (x + y) % 2 * 255
    return {"odd_pitch": uniform, "padded_frames": big[:n, 1:H + 1, 5:W + 5], "every_other_frame": big[::2, :H, :W]}


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", [(1, 3), (3, 17), (17, 15), (65, 63), (129, 65), (641, 479)])
def test_undistort_padded_input_and_guarded_outputs(remap_kernels, uo, pkg, abi, W, H):
    """Strided raw frames, and output levels in padded arrays: nothing outside a level's W x H changes."""
    ctx = pkg.api.default_context()
    n = deepest(W, H)
    cams = in_range(W, H)
    for layout, raw in raw_views(W, H, 4, seed=W + H).items():
        assert raw.strides[1] != W or raw.strides[0] != H * W
        for name in ("barrel", "neg_fx_fy", "d0_-1e-7_copy"):
            p = cams[name]
            want = oracle_levels(uo, abi, p, raw, n)
            outs, r = [], abi.PyramidResult()
            for l in range(n):
                buf = np.full((4, (H >> l) + 2, (W >> l) + 13), GUARD, np.uint8)
                outs.append(buf)
                r.level[l] = buf.ctypes.data_as(C.POINTER(C.c_uint8))
                r.pitch[l], r.stride[l] = buf.strides[1], buf.strides[0]
            b = abi.UndistortBatch(struct(abi, p), 4, n, raw.ctypes.data_as(C.POINTER(C.c_uint8)), raw.strides[1], raw.strides[0])
            ctx.check(ctx.lib.plsvo_undistort_batch_run(ctx.handle, C.byref(b), C.byref(r)), "plsvo_undistort_batch_run")
            for l in range(n):
                h, w = H >> l, W >> l
                np.testing.assert_array_equal(outs[l][:, :h, :w], want[l], err_msg=f"{layout} {name} level {l}")
                assert (outs[l][:, h:] == GUARD).all() and (outs[l][:, :, w:] == GUARD).all(), f"{layout} {name} level {l}: padding written"


@pytest.mark.gpu
def test_undistort_remap_frame_runs(remap_kernels, uo, pkg, abi, new_ctx):
    """A one-tile frame (at most 64 x 16): the remap kernel runs num_sms * 4 frame runs; batches on both sides of every
    split, and one batch of many tiny frames."""
    want = sm_count() * 4
    W, H = 61, 13
    p = in_range(W, H)["barrel"]
    ctx = new_ctx()
    rng = np.random.default_rng(31)
    for B in (1, want - 1, want, want + 1, 3 * want + 1):
        raw = rng.integers(0, 256, (B, H, W), dtype=np.uint8)
        raw[-1] = 255
        check_levels(pkg.PinholeCamera(*p).undistortImage(raw, 3, ctx), oracle_levels(uo, abi, p, raw, 3), f"B={B}")
    p = in_range(16, 8)["pincushion"]
    raw = rng.integers(0, 256, (TINY, 8, 16), dtype=np.uint8)
    check_levels(pkg.PinholeCamera(*p).undistortImage(raw, 3, ctx), oracle_levels(uo, abi, p, raw, 3), f"B={TINY}")


# ---- plsvo_align_raw_batch_run / plsvo_track_raw_batch_run with rect_out: the fused kernel ----------------------------------
def align_data(synth, p, B, seed, empty, hi=2, lo=1):
    """Features and poses for B pairs of camera p (a few generated pairs, scaled to its frame, repeated), without images;
    empty: no point and no segment in any pair (the cameras whose alignment would see non-finite bearings)."""
    import dataclasses

    W, H, fx, fy, cx, cy = p[:6]
    base = synth.make_align_batch(cam=synth.QVGA, batch=min(B, 4), n_pts=40, n_segs=8, seed=seed, max_level=hi, min_level=lo, margin=16)
    rep = lambda a: None if a is None else np.ascontiguousarray(np.resize(a, (B,) + a.shape[1:]))  # noqa: E731
    scale = np.array([W / synth.QVGA.width, H / synth.QVGA.height])
    d = dataclasses.replace(base, cam=synth.Camera(W, H, fx, fy, cx, cy), ref_pyr={}, cur_pyr={}, frame_pyr=None)
    for f in ("T_ref_w", "T_cur_w", "T_cur_w_gt", "pt_pos", "seg_spos", "seg_epos", "pt_valid", "seg_valid"):
        setattr(d, f, rep(getattr(base, f)))
    d.pt_px, d.seg_spx, d.seg_epx = (rep(getattr(base, f) * scale) for f in ("pt_px", "seg_spx", "seg_epx"))
    d.seg_length = rep(np.linalg.norm(d.seg_epx - d.seg_spx, axis=-1)[: min(B, 4)])
    d.pt_f = d.seg_sf = d.seg_ef = None  # bearings formed on the device from the pixels
    if empty:
        d.pt_count = np.zeros(B, np.int32)
        d.seg_count = np.zeros(B, np.int32)
    return d


def fused_case(pkg, synth, uo, abi, ctx, p, raw, chain, level_sets, empty, what, seed=0):
    """One raw alignment call per level set with rect_out, against the oracle's levels and the same call without it."""
    n = raw.shape[0]
    B = n - 1 if chain else n // 2
    data = align_data(synth, p, B, seed=seed, empty=empty)
    stacks = raw if chain else (raw[:B], raw[B:])
    cam = pkg.PinholeCamera(*p)
    plain = pkg.SparseImgAlign(2, 1, 30, ctx=ctx).run_raw(cam, stacks, data)
    want = oracle_levels(uo, abi, p, raw, max(max(s) for s in level_sets) + 1)
    for levels in level_sets:
        out, rect = pkg.SparseImgAlign(2, 1, 30, ctx=ctx).run_raw(cam, stacks, data, rect_levels=list(levels))
        assert sorted(rect) == sorted(levels)
        for l in levels:
            np.testing.assert_array_equal(rect[l], want[l], err_msg=f"{what}: rect_out {levels} level {l}")
        for f in ALIGN_FIELDS:
            np.testing.assert_array_equal(getattr(out, f), getattr(plain, f), err_msg=f"{what}: {f} with rect_out {levels}")


SUBSETS = [tuple(l for l in range(7) if m >> l & 1) for m in range(1, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("chain", [True, False], ids=["chain", "pair"])
@pytest.mark.parametrize("W,H", [(65, 127), (191, 64)])
def test_fused_every_level_subset(pkg, synth, uo, abi, new_ctx, W, H, chain):
    raw = frames(3, H, W, seed=41 + W)[:4 if not chain else 5]
    fused_case(pkg, synth, uo, abi, new_ctx(), in_range(W, H)["barrel"], raw, chain, SUBSETS, W < 127, f"{W}x{H}")


FUSED_SIZES = {64: 64, 65: 127, 127: 65, 129: 191, 191: 129, 641: 479, 752: 480, 1280: 720}


@pytest.mark.gpu
@pytest.mark.parametrize("W", list(FUSED_SIZES))
def test_fused_every_camera_layout_and_pitch(pkg, synth, uo, abi, new_ctx, W):
    """Every in-range camera, in turn as a chain or pairs and with raw rows at a pitch that is not a multiple of 4 (one
    linear copy), in padded frames, or every other frame of a stack."""
    H = FUSED_SIZES[W]
    ctx = new_ctx()
    for i, (name, p) in enumerate(in_range(W, H).items()):
        chain = i % 2 == 0
        layout, raw = list(raw_views(W, H, 5 if chain else 4, seed=W + i).items())[i % 3]
        fused_case(pkg, synth, uo, abi, ctx, p, raw, chain, [tuple(range(7)), (0, 3, 6)], W < 127, f"{name} {W}x{H} {layout}", seed=i)


@pytest.mark.gpu
@pytest.mark.parametrize("key", ["tie_k1@640x480", "tie_neg_fx_p1@640x480", "oor_wrap@641x479", "oor_huge@640x480",
                                 "oor_subnormal_fx@640x480", "inf@64x48"])
def test_fused_tie_and_out_of_range_cameras(pkg, synth, uo, abi, new_ctx, key):
    p = special()[key]
    W, H = p[:2]
    levels = tuple(range(deepest(W, H)))
    for chain in (True, False):
        raw = frames(3, H, W, seed=51)[:5 if chain else 4]
        fused_case(pkg, synth, uo, abi, new_ctx(), p, raw, chain, [levels], True, f"{key} chain={chain}")


@pytest.mark.gpu
@pytest.mark.parametrize("d0", [1e-7, -1e-7, 1.0000001e-7, -1.0000001e-7])
def test_fused_d0_threshold(pkg, synth, uo, abi, new_ctx, d0):
    """fabs(d0) > 1e-7 is a map: exactly 1e-7 copies the raw frame whatever d1..d4 are."""
    p = list(in_range(129, 65)["barrel"])
    p[6], p[7] = d0, 0.2
    raw = frames(3, 65, 129, seed=52)
    fused_case(pkg, synth, uo, abi, new_ctx(), tuple(p), raw, True, [tuple(range(7))], True, f"d0={d0}")
    if abs(d0) == 1e-7:
        np.testing.assert_array_equal(oracle_levels(uo, abi, tuple(p), raw, 1)[0], raw)


@pytest.mark.gpu
def test_fused_frame_runs(pkg, synth, uo, abi, new_ctx):
    """A one-tile frame (64 x 64): raw_pyramid_grid makes num_sms * 16 frame runs; frame counts on both sides of it."""
    want = sm_count() * 16
    p = in_range(64, 64)["pincushion"]
    ctx = new_ctx()
    rng = np.random.default_rng(61)
    for n, chain in ((2, True), (want - 1, True), (want, True), (want + 1, True), (3 * want + 1, True), (want, False), (want + 2, False)):
        raw = rng.integers(0, 256, (n, 64, 64), dtype=np.uint8)
        raw[-1] = 255
        fused_case(pkg, synth, uo, abi, ctx, p, raw, chain, [tuple(range(7))], True, f"{n} frames chain={chain}")


@pytest.mark.gpu
@pytest.mark.parametrize("chain", [True, False], ids=["chain", "pair"])
@pytest.mark.parametrize("name,W,H", [("barrel", 641, 479), ("non_square", 129, 191), ("d0_1.0000001e-7_map", 752, 480)])
def test_fused_track_raw_rect_out(pkg, synth, uo, abi, new_ctx, name, W, H, chain):
    """plsvo_track_raw_batch_run: rect_out equals the oracle; alignment and pose optimisation equal the call without it."""
    p = in_range(W, H)[name]
    B = 3
    raw = frames(4, H, W, seed=71)[:B + 1 if chain else 2 * B]
    stacks = raw if chain else (raw[:B], raw[B:])
    data = align_data(synth, p, B, seed=72, empty=False)
    po = synth.make_poseopt_batch(cam=data.cam, batch=B, n_pts=data.n_pts, n_segs=data.n_segs, seed=73, T_gt=data.T_cur_w_gt)
    ctx = new_ctx()
    cam = pkg.PinholeCamera(*p)
    levels = [0, 2, 5, 6]
    plain_a, plain_p = pkg.track_raw(cam, stacks, data, po, max_level=2, min_level=1, chained=chain, ctx=ctx)
    got_a, got_p, rect = pkg.track_raw(cam, stacks, data, po, max_level=2, min_level=1, chained=chain, ctx=ctx, rect_levels=levels)
    want = oracle_levels(uo, abi, p, raw, 7)
    for l in levels:
        np.testing.assert_array_equal(rect[l], want[l], err_msg=f"level {l}")
    for f in ALIGN_FIELDS:
        np.testing.assert_array_equal(getattr(got_a, f), getattr(plain_a, f), err_msg=f)
    for f in PO_FIELDS:
        np.testing.assert_array_equal(getattr(got_p, f), getattr(plain_p, f), err_msg=f)


# ---- the multicam raw call: undistort_pyramid_multicam_kernel ---------------------------------------------------------------
SLOT = (643, 482)
MULTICAM_DEEP = [  # name, camera: every one at least 64 x 64 (levels 0..6), widths 0..3 mod 4, smaller than the slot each way
    ("copy_129x65", in_range(129, 65)["d0_1e-7_copy"]), ("copy_65x482", in_range(65, 482)["d0_-1e-7_copy"]),
    ("barrel_130x66", in_range(130, 66)["barrel"]), ("neg_fx_fy_66x482", in_range(66, 482)["neg_fx_fy"]),
    ("pincushion_643x67", in_range(643, 67)["pincushion"]), ("map_643x482", in_range(*SLOT)["d0_1.0000001e-7_map"]),
    ("tie_k1", TIES["tie_k1"]), ("tie_neg_fx_p1", TIES["tie_neg_fx_p1"]), ("oor_wrap_641x479", out_of_range(641, 479)["oor_wrap"]),
    ("oor_subnormal_fx_640x480", out_of_range(640, 480)["oor_subnormal_fx"]),
]
MULTICAM_SHALLOW = MULTICAM_DEEP + [  # frames down to 3 x 2: levels 0..1
    ("oor_huge_61x45", out_of_range(61, 45)["oor_huge"]), ("oor_subnormal_fx_7x5", out_of_range(7, 5)["oor_subnormal_fx"]),
    ("oor_f60_3x2", out_of_range(3, 2)["oor_f60"]), ("inf_64x48", INF), ("tie_k1_k2", TIES["tie_k1_k2"]),
    ("barrel_3x482", in_range(3, 482)["barrel"]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("cams,levels", [(MULTICAM_DEEP, tuple(range(7))), (MULTICAM_SHALLOW, (0, 1))], ids=["levels_0_6", "levels_0_1"])
def test_multicam_slot_of_mixed_cameras_and_sizes(pkg, synth, uo, abi, new_ctx, cams, levels):
    """Every frame's levels equal the oracle at the frame's own size, with its own camera, and the slot's padding of every
    level is 0."""
    K = len(cams)
    B = 2 * K
    cop = np.random.default_rng(81).permutation(np.arange(B) % K).astype(np.int32)
    W, H = SLOT
    raw = np.random.default_rng(82).integers(0, 256, (2 * B, H, W), dtype=np.uint8)
    raw[1] = 255
    y, x = np.mgrid[:H, :W]
    raw[2] = (x + y) % 2 * 255
    slot_cam = (W, H, 500.0, 500.0, W / 2, H / 2, 0.0, 0.0, 0.0, 0.0, 0.0)
    data = align_data(synth, slot_cam, B, seed=83, empty=True)
    hi = max(levels)
    lenses = [pkg.PinholeCamera(*p) for _, p in cams]
    _, rect = pkg.SparseImgAlign(hi, 0, 30, ctx=new_ctx()).run_raw(lenses, (raw[:B], raw[B:]), data, rect_levels=list(levels), cam_of_pair=cop)
    frame_cam = np.concatenate([cop, cop])
    for k, (name, p) in enumerate(cams):
        Wk, Hk = p[:2]
        idx = np.flatnonzero(frame_cam == k)
        want = oracle_levels(uo, abi, p, raw[idx, :Hk, :Wk], hi + 1)
        for l in levels:
            got = rect[l][idx]
            np.testing.assert_array_equal(got[:, : Hk >> l, : Wk >> l], want[l], err_msg=f"{name} level {l}")
            assert not got[:, Hk >> l:].any() and not got[:, :, Wk >> l:].any(), f"{name} level {l}: slot padding is not 0"
