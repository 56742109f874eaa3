"""Loader of the CPU oracle's ATAN path (oracle/atan_oracle.cpp -> oracle/libplsvo_atan_oracle.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib: SparseImgAlign::run seen through vk::ATANCamera (the stand-in
oracle/refdeps/vikit/atan_camera.h), and that camera's cam2world / world2cam / errorMultiplier2.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libplsvo_atan_oracle.so")
# atan_camera.h and everything of refdeps/ it includes
SOURCES = [os.path.join(_HERE, f) for f in ("atan_oracle.cpp", "plsvo_oracle.cpp", os.path.join("refdeps", "vikit", "atan_camera.h"),
                                            os.path.join("refdeps", "vikit", "abstract_camera.h"), os.path.join("refdeps", "vikit", "math_utils.h"),
                                            os.path.join("refdeps", "Eigen", "Core"))]
# the flags of oracle/Makefile's libplsvo_oracle.so: strict IEEE without FMA contraction
CXXFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-math-errno", "-funroll-loops", "-std=c++17", "-fPIC", "-Wall",
            "-Wno-unused-variable", "-Wno-unused-function"]
_lib = None

# oracle/_ref/libplsvo_atan_ref.so: the reference's own translation units (oracle/Makefile's `ref` target: same sources,
# same flags) driven through the stand-in ATANCamera by atan_ref_harness.cpp.  Only where the reference sources exist.
REFERENCE_ROOT = os.environ.get("PLSVO_REFERENCE", "/root/reference")
REF_LIB_PATH = os.path.join(_HERE, "_ref", "libplsvo_atan_ref.so")
REF_SRCS = ("sparse_img_align.cpp", "pose_optimizer.cpp", "feature.cpp", "feature_alignment.cpp", "matcher.cpp", "config.cpp",
            "feature3D_impl.cpp", "depth_filter.cpp", "feature3D.cpp")
REF_CXXFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-math-errno", "-funroll-loops", "-std=c++17", "-fPIC", "-w", "-DNDEBUG"]
_ref_lib = None


def build(force: bool = False) -> str:
    deps = SOURCES + [os.path.join(_HERE, "..", "include", "plsvo_b200.h")]
    stale = not os.path.exists(LIB_PATH) or any(os.path.getmtime(f) > os.path.getmtime(LIB_PATH) for f in deps)
    if force or stale:
        subprocess.check_call([os.environ.get("CXX", "g++")] + CXXFLAGS + ["-I" + os.path.join(_HERE, "refdeps"), "-shared", "-o",
                                                                            LIB_PATH, os.path.join(_HERE, "atan_oracle.cpp"), "-lpthread"])
    return LIB_PATH


def load(abi):
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        build()
    lib = C.CDLL(LIB_PATH)
    P = C.POINTER
    lib.plsvo_oracle_atan_align_batch.restype = C.c_int
    lib.plsvo_oracle_atan_align_batch.argtypes = [P(abi.AtanCamera), P(abi.AlignBatch), P(abi.AlignParams), P(abi.AlignResult), C.c_int]
    lib.plsvo_oracle_atan_align_batch_members.restype = C.c_int
    lib.plsvo_oracle_atan_align_batch_members.argtypes = [C.c_double] * 5 + [P(abi.AlignBatch), P(abi.AlignParams), P(abi.AlignResult), C.c_int]
    for name in ("plsvo_oracle_atan_cam2world", "plsvo_oracle_atan_world2cam"):
        fn = getattr(lib, name)
        fn.restype = None
        fn.argtypes = [P(abi.AtanCamera), P(C.c_double), C.c_int, P(C.c_double)]
    lib.plsvo_oracle_atan_error_multiplier2.restype = C.c_double
    lib.plsvo_oracle_atan_error_multiplier2.argtypes = [P(abi.AtanCamera)]
    _lib = lib
    return lib


def align(abi, camera, data, params=None, n_threads: int = 1):
    """SparseImgAlign::run on an AlignData batch seen through `camera` (api.ATANCamera) -> abi.AlignOut."""
    lib = load(abi)
    params = params or abi.align_params(data.max_level, data.min_level)
    batch, keep = abi.make_align_batch(data)
    out = abi.AlignOut(data.batch, data.n_segs)
    rc = lib.plsvo_oracle_atan_align_batch(C.byref(camera.struct), C.byref(batch), C.byref(params), C.byref(out.struct), n_threads)
    if rc != 0:
        raise RuntimeError(f"ATAN oracle align failed rc={rc}")
    return out


def align_members(abi, camera, data, params=None, n_threads: int = 1):
    """align() with the camera given by its derived members fx_, fy_, cx_, cy_ and d0 (the device kernels' AlignArgs)."""
    lib = load(abi)
    params = params or abi.align_params(data.max_level, data.min_level)
    batch, keep = abi.make_align_batch(data)
    out = abi.AlignOut(data.batch, data.n_segs)
    rc = lib.plsvo_oracle_atan_align_batch_members(camera.fx_, camera.fy_, camera.cx_, camera.cy_, camera.s_, C.byref(batch), C.byref(params),
                                                   C.byref(out.struct), n_threads)
    if rc != 0:
        raise RuntimeError(f"ATAN oracle align failed rc={rc}")
    return out


def _call(abi, name, camera, x, n_out):
    lib = load(abi)
    x = np.ascontiguousarray(x, np.float64)
    n = x.shape[0]
    out = np.zeros((n, n_out))
    getattr(lib, name)(C.byref(camera.struct), x.ctypes.data_as(C.POINTER(C.c_double)), n, out.ctypes.data_as(C.POINTER(C.c_double)))
    return out


def cam2world(abi, camera, px):
    """[n, 2] pixels -> [n, 3] bearings of the stand-in vk::ATANCamera."""
    return _call(abi, "plsvo_oracle_atan_cam2world", camera, px, 3)


def world2cam(abi, camera, xyz):
    """[n, 3] camera-frame points -> [n, 2] pixels of the stand-in vk::ATANCamera."""
    return _call(abi, "plsvo_oracle_atan_world2cam", camera, xyz, 2)


def error_multiplier2(abi, camera) -> float:
    return load(abi).plsvo_oracle_atan_error_multiplier2(C.byref(camera.struct))


def build_ref(force: bool = False) -> str | None:
    """Build oracle/_ref/libplsvo_atan_ref.so where the reference sources are present.  Returns its path, or None when
    neither the sources nor a prebuilt library exist."""
    srcs = [os.path.join(REFERENCE_ROOT, "src", f) for f in REF_SRCS]
    harness = [os.path.join(_HERE, f) for f in ("atan_ref_harness.cpp", "ref_harness.cpp", "next_scenes.h")]
    if all(os.path.exists(s) for s in srcs):
        deps = srcs + harness + SOURCES[2:] + [os.path.join(_HERE, "..", "include", "plsvo_b200.h")]
        stale = not os.path.exists(REF_LIB_PATH) or any(os.path.getmtime(f) > os.path.getmtime(REF_LIB_PATH) for f in deps)
        if force or stale:
            os.makedirs(os.path.dirname(REF_LIB_PATH), exist_ok=True)
            subprocess.check_call([os.environ.get("CXX", "g++")] + REF_CXXFLAGS + ["-I" + os.path.join(_HERE, "refdeps"),
                                   "-I" + os.path.join(REFERENCE_ROOT, "include"), "-shared", "-o", REF_LIB_PATH] + srcs +
                                  [harness[0], "-lpthread"])
    return REF_LIB_PATH if os.path.exists(REF_LIB_PATH) else None


def ref_available() -> bool:
    return os.path.exists(REF_LIB_PATH)


def ref_align(abi, camera, data, params=None, n_threads: int = 1):
    """SparseImgAlign::run of the reference's own sparse_img_align.cpp, the frames seen through `camera` -> abi.AlignOut."""
    global _ref_lib
    if _ref_lib is None:
        lib = C.CDLL(REF_LIB_PATH)
        lib.plsvo_ref_atan_align_batch.restype = C.c_int
        lib.plsvo_ref_atan_align_batch.argtypes = [C.POINTER(abi.AtanCamera), C.POINTER(abi.AlignBatch), C.POINTER(abi.AlignParams),
                                                   C.POINTER(abi.AlignResult), C.c_int]
        _ref_lib = lib
    params = params or abi.align_params(data.max_level, data.min_level)
    batch, keep = abi.make_align_batch(data)
    out = abi.AlignOut(data.batch, data.n_segs)
    rc = _ref_lib.plsvo_ref_atan_align_batch(C.byref(camera.struct), C.byref(batch), C.byref(params), C.byref(out.struct), n_threads)
    if rc != 0:
        raise RuntimeError(f"reference ATAN align failed rc={rc}")
    return out


# oracle/_ref/libplsvo_atan_shimref.so: the reference's own objects with a vk::ATANCamera through the drop-in shim
# (atan_shimref_harness.cpp; sources and flags of oracle/Makefile's `shimref` target).  Needs the reference sources and
# the built CUDA library.
SHIMREF_LIB_PATH = os.path.join(_HERE, "_ref", "libplsvo_atan_shimref.so")
SHIMREF_REF_SRCS = ("feature.cpp", "feature3D.cpp", "feature3D_impl.cpp", "depth_filter.cpp", "matcher.cpp", "feature_alignment.cpp",
                    "config.cpp")
_shimref_lib = None


def build_shimref(force: bool = False) -> str | None:
    shim_dir = os.path.join(_HERE, "..", "pl-svo_b200", "host")
    csrc = os.path.join(_HERE, "..", "pl-svo_b200", "csrc")
    srcs = [os.path.join(REFERENCE_ROOT, "src", f) for f in SHIMREF_REF_SRCS]
    shim = [os.path.join(shim_dir, f) for f in ("plsvo_shim.cpp", "plsvo_shim_next.cpp")]
    if all(os.path.exists(s) for s in srcs) and os.path.exists(os.path.join(csrc, "libplsvo_b200.so")):
        deps = srcs + shim + [os.path.join(shim_dir, f) for f in ("plsvo_shim.h", "plsvo_shim_next.h")] + [
            os.path.join(_HERE, f) for f in ("atan_shimref_harness.cpp", "shimref_harness.cpp", "next_scenes.h")] + SOURCES[2:] + [
            os.path.join(_HERE, "..", "include", "plsvo_b200.h")]
        stale = not os.path.exists(SHIMREF_LIB_PATH) or any(os.path.getmtime(f) > os.path.getmtime(SHIMREF_LIB_PATH) for f in deps)
        if force or stale:
            os.makedirs(os.path.dirname(SHIMREF_LIB_PATH), exist_ok=True)
            subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-w", "-DNDEBUG", "-DPLSVO_SHIM_WITH_REFERENCE_HEADERS",
                                   "-I" + os.path.join(shim_dir, "overlay"), "-I" + os.path.join(_HERE, "refdeps"),
                                   "-I" + os.path.join(REFERENCE_ROOT, "include"), "-I" + os.path.join(_HERE, "..", "include"), "-I" + shim_dir,
                                   "-shared", "-o", SHIMREF_LIB_PATH] + srcs + shim + [os.path.join(_HERE, "atan_shimref_harness.cpp"),
                                   "-L" + csrc, "-lplsvo_b200", "-Wl,-rpath,$ORIGIN/../../pl-svo_b200/csrc", "-lpthread"])
    return SHIMREF_LIB_PATH if os.path.exists(SHIMREF_LIB_PATH) else None


def shimref_align(abi, camera, data, params=None):
    """plsvo::SparseImgAlign(...).run(ref, cur) of the shim on reference-typed frames with a vk::ATANCamera -> abi.AlignOut
    (T_cur_w, n_tracked, seg_killed)."""
    global _shimref_lib
    if _shimref_lib is None:
        lib = C.CDLL(SHIMREF_LIB_PATH)
        lib.plsvo_shimref_atan_align_batch.restype = C.c_int
        lib.plsvo_shimref_atan_align_batch.argtypes = [C.POINTER(abi.AtanCamera), C.POINTER(abi.AlignBatch), C.POINTER(abi.AlignParams),
                                                       C.POINTER(abi.AlignResult)]
        _shimref_lib = lib
    params = params or abi.align_params(data.max_level, data.min_level)
    batch, keep = abi.make_align_batch(data)
    out = abi.AlignOut(data.batch, data.n_segs)
    rc = _shimref_lib.plsvo_shimref_atan_align_batch(C.byref(camera.struct), C.byref(batch), C.byref(params), C.byref(out.struct))
    if rc != 0:
        raise RuntimeError(f"ATAN shimref align failed rc={rc}")
    return out
