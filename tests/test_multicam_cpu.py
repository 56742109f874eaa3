"""Multicam batches without a GPU: the C ABI's argument checks of the three multicam entry points against the host model
(tests/hostmodel: plsvo_abi.cu compiled unchanged, without the multicam kernels), and the Python mirror's handling of
`cameras=` and `fx=`."""
import ctypes as C
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def hostmodel():
    spec = importlib.util.spec_from_file_location("plsvo_hostmodel_build", os.path.join(HERE, "hostmodel", "build.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.build()


def _host_model_env(lib):
    env = dict(os.environ, PLSVO_LIB=lib, PLSVO_FAKE_CUDA="lazy")
    for k in [k for k in env if k.startswith("PLSVO_") and k not in ("PLSVO_LIB", "PLSVO_FAKE_CUDA")]:
        del env[k]
    return env


def test_malformed_calls_are_rejected_before_the_kernel_check(hostmodel):
    """tests/test_gpu_multicam.py::test_malformed_multicam_calls against the host model: every malformed call returns
    PLSVO_ERR_INVALID with its message although the model has no multicam kernel, so validation comes first."""
    p = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_multicam.py"), "-q", "-m", "gpu",
                        "-p", "no:cacheprovider", "-k", "malformed"],
                       env=_host_model_env(hostmodel), capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "1 passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


_WELL_FORMED = r"""
import ctypes as C, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import plsvo_b200 as pkg
from plsvo_b200 import abi, synth
ctx = pkg.Context(0)
lib = ctx.lib
d = synth.make_align_batch(cam=synth.QVGA, batch=3, n_pts=16, n_segs=4, max_level=3, min_level=1, margin=32, seed=1)
po = synth.make_poseopt_batch(cam=synth.QVGA, batch=3, n_pts=16, n_segs=4, seed=2)
ab, ka = abi.make_align_batch(d)
pb, kp = abi.make_poseopt_batch(po)
ap, pp = abi.align_params(3, 1, 30), abi.poseopt_params()
ao, pout = abi.AlignOut(3, 4), abi.PoseOptOut(3, 16, 4)
k = np.tile([d.cam.fx, d.cam.fy, d.cam.cx, d.cam.cy], (3, 1))
k[1] = (-500.0, 480.0, 150.0, 130.0)  # any finite intrinsics with fx, fy != 0 are valid
cams = abi.make_cameras(k, d.cam, 3)
fx = np.array([210.0, 500.0, 1e-3])
rcs = [lib.plsvo_align_multicam_batch_run(ctx.handle, cams, C.byref(ab), C.byref(ap), C.byref(ao.struct)),
       lib.plsvo_track_multicam_batch_run(ctx.handle, cams, C.byref(ab), C.byref(ap), C.byref(pb), C.byref(pp),
                                          C.byref(ao.struct), C.byref(pout.struct)),
       lib.plsvo_poseopt_multicam_batch_run(ctx.handle, fx.ctypes.data_as(C.POINTER(C.c_double)), C.byref(pb), C.byref(pp),
                                            C.byref(pout.struct))]
msg = lib.plsvo_last_error(ctx.handle).decode()
# the context still runs a uniform call afterwards
rc_uniform = lib.plsvo_align_upload(ctx.handle, C.byref(ab))
print("RESULT", rcs, rc_uniform, msg)
"""


def test_well_formed_calls_reach_the_kernel_check(hostmodel, tmp_path):
    """Well-formed multicam calls pass validation and report the missing kernels (PLSVO_ERR_CUDA), as any call does in
    a library built without its kernels."""
    script = tmp_path / "well_formed.py"
    script.write_text(_WELL_FORMED)
    root = os.path.dirname(HERE)
    p = subprocess.run([sys.executable, str(script), root], env=_host_model_env(hostmodel), capture_output=True, text=True,
                       timeout=300)
    line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
    assert p.returncode == 0 and line, p.stdout[-2000:] + p.stderr[-2000:]
    assert line[0].startswith("RESULT [-2, -2, -2] 0 "), line[0]
    assert "without the multicam pose-optimiser kernel" in line[0]


# ---- the Python mirror ----------------------------------------------------------------------------------------------


def test_make_cameras_layout(abi, synth):
    k = np.arange(12, dtype=np.float64).reshape(3, 4) + 1.0
    cams = abi.make_cameras(k, synth.VGA, 3)
    assert C.sizeof(cams) == 3 * C.sizeof(abi.Camera) == 3 * 48
    for b in range(3):
        c = cams[b]
        assert (c.width, c.height, c.reserved0, c.reserved1) == (640, 480, 0, 0)
        assert (c.fx, c.fy, c.cx, c.cy) == tuple(k[b])
    with pytest.raises(ValueError):
        abi.make_cameras(k[:, :3], synth.VGA, 3)
    with pytest.raises(ValueError):
        abi.make_cameras(k, synth.VGA, 4)


def test_abi_declares_the_multicam_entry_points(abi):
    names = {n for n, _, _ in abi.ABI_SYMBOLS}
    assert {"plsvo_align_multicam_batch_run", "plsvo_poseopt_multicam_batch_run", "plsvo_track_multicam_batch_run"} <= names
    header = open(os.path.join(os.path.dirname(HERE), "include", "plsvo_b200.h")).read()
    for n in ("plsvo_align_multicam_batch_run", "plsvo_poseopt_multicam_batch_run", "plsvo_track_multicam_batch_run"):
        assert f"int {n}(" in header


def test_python_argument_checks_need_no_library(pkg, synth):
    """Shapes and the camera= / cameras= exclusion are checked before the library is called."""
    api = pkg.api
    d = synth.make_align_batch(cam=synth.QVGA, batch=3, n_pts=8, n_segs=2, max_level=3, min_level=1, margin=32, seed=1)
    with pytest.raises(api.PlsvoError, match="not both"):
        api._one_camera_model(object(), np.zeros((3, 4)))
    api._one_camera_model(None, np.zeros((3, 4)))
    api._one_camera_model(object(), None)
    with pytest.raises(api.PlsvoError, match=r"shape \[3, 4\]"):
        api._cameras_arg(np.zeros((3, 3)), d)
    with pytest.raises(api.PlsvoError, match=r"shape \[3, 4\]"):
        api._cameras_arg(np.zeros(12), d)
    cams = api._cameras_arg([[1, 2, 3, 4]] * 3, d)
    assert cams[2].fx == 1.0 and cams[2].cy == 4.0 and cams[0].width == 320
    with pytest.raises(api.PlsvoError, match=r"shape \[3\]"):
        api._frame_fx_arg(np.ones((3, 1)), 3)
    fx = api._frame_fx_arg([1, 2, 3], 3)
    assert fx.dtype == np.float64 and fx.flags.c_contiguous


def test_multicam_generator(synth):
    cams = synth.MULTICAM_K4
    cam_of_pair = np.array([2, 0, 3, 1, 0, 2, 3])
    al, cameras = synth.make_multicam_batch(cams, cam_of_pair, n_pts=8, n_segs=2, max_level=3, min_level=1, margin=32,
                                            seed=11)
    assert al.batch == 7 and cameras.shape == (7, 4)
    for b, k in enumerate(cam_of_pair):
        c = cams[k]
        assert tuple(cameras[b]) == (c.fx, c.fy, c.cx, c.cy)
        # the bearings are the pixels lifted through pair b's own camera
        px = al.pt_px[b]
        f = np.stack([(px[:, 0] - c.cx) / c.fx, (px[:, 1] - c.cy) / c.fy, np.ones(len(px))], -1)
        np.testing.assert_allclose(al.pt_f[b], f / np.linalg.norm(f, axis=-1, keepdims=True), rtol=0, atol=1e-12)
    # the pairs of one camera are that camera's own batch, in order
    one = synth.make_align_batch(cam=cams[0], batch=2, n_pts=8, n_segs=2, max_level=3, min_level=1, margin=32, seed=11)
    np.testing.assert_array_equal(al.ref_pyr[1][[1, 4]], one.ref_pyr[1])
    np.testing.assert_array_equal(al.T_ref_w[[1, 4]], one.T_ref_w)
    with pytest.raises(ValueError):
        synth.make_multicam_batch((synth.VGA, synth.QVGA), [0, 1])


def test_take_pairs(synth):
    d = synth.make_align_batch(cam=synth.QVGA, batch=5, n_pts=8, n_segs=2, max_level=3, min_level=1, margin=32, seed=1)
    d.pt_depth = np.arange(40.0).reshape(5, 8)  # an array set on the instance, as lean batches do
    sub = synth.take_pairs(d, [3, 1])
    assert sub.batch == 2 and sub.cam == d.cam
    for name in ("pt_depth", "pt_px", "pt_f", "T_ref_w", "seg_length"):
        np.testing.assert_array_equal(getattr(sub, name), getattr(d, name)[[3, 1]], err_msg=name)
    for l in d.ref_pyr:
        np.testing.assert_array_equal(sub.ref_pyr[l], d.ref_pyr[l][[3, 1]])
        np.testing.assert_array_equal(sub.cur_pyr[l], d.cur_pyr[l][[3, 1]])
    d.frame_pyr = synth.chain_frames(synth.make_chain_batch(cam=synth.QVGA, batch=5, n_pts=8, n_segs=2, max_level=3,
                                                            min_level=1, margin=32))
    with pytest.raises(ValueError, match="frame chains"):
        synth.take_pairs(d, [0])
