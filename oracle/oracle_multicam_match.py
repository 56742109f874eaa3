"""Loader of the CPU oracle's per-image-camera matcher (oracle/multicam_match_oracle.cpp ->
oracle/libplsvo_multicam_match_oracle.so) and of its checker, the reference's own matcher.cpp with a stand-in camera per
frame (oracle/multicam_match_ref_harness.cpp -> oracle/_ref/libplsvo_multicam_match_ref.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib and oracle_atan_match: Matcher::findMatchDirect with ref image r seen through
cams[cam_of_ref[r]] and current image c through cams[cam_of_cur[c]], and the same matcher downstream of a given A_cur_ref.
`cams` is a sequence of api.ATANCamera / synth.Camera (undistorted pinhole), as Matcher.findMatchDirect takes it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle_atan

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libplsvo_multicam_match_oracle.so")
SOURCES = [os.path.join(_HERE, "multicam_match_oracle.cpp"), os.path.join(_HERE, "plsvo_oracle.cpp"),
           os.path.join(_HERE, "refdeps", "vikit", "atan_camera.h"), os.path.join(_HERE, "refdeps", "vikit", "pinhole_camera.h")]
_lib = None

REF_LIB_PATH = os.path.join(_HERE, "_ref", "libplsvo_multicam_match_ref.so")
_ref_lib = None


def build(force: bool = False) -> str:
    deps = SOURCES + [os.path.join(_HERE, "..", "include", "plsvo_b200.h")]
    stale = not os.path.exists(LIB_PATH) or any(os.path.getmtime(f) > os.path.getmtime(LIB_PATH) for f in deps)
    if force or stale:
        subprocess.check_call([os.environ.get("CXX", "g++")] + oracle_atan.CXXFLAGS + ["-I" + os.path.join(_HERE, "refdeps"), "-shared",
                                                                                      "-o", LIB_PATH, SOURCES[0], "-lpthread"])
    return LIB_PATH


def _cam_args(abi, P):
    return [P(abi.MatchCamera), C.c_int, P(C.c_int32), P(C.c_int32)]


def load(abi):
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        build()
    lib = C.CDLL(LIB_PATH)
    P = C.POINTER
    lib.plsvo_oracle_match_direct_multicam_batch.restype = C.c_int
    lib.plsvo_oracle_match_direct_multicam_batch.argtypes = _cam_args(abi, P) + [P(abi.MatchBatch), P(abi.MatchResult), C.c_int]
    lib.plsvo_oracle_match_direct_multicam_given_A.restype = C.c_int
    lib.plsvo_oracle_match_direct_multicam_given_A.argtypes = _cam_args(abi, P) + [P(C.c_double), P(abi.MatchBatch), P(abi.MatchResult),
                                                                                  C.c_int]
    _lib = lib
    return lib


def _threads(n_threads: int) -> int:
    return n_threads if n_threads > 0 else (os.cpu_count() or 1)


def _tables(abi, cams, cam_of_ref, cam_of_cur):
    ref = np.ascontiguousarray(cam_of_ref, np.int32)
    cur = np.ascontiguousarray(cam_of_cur, np.int32)
    i32 = C.POINTER(C.c_int32)
    arr = abi.make_match_cameras(cams)
    return [arr, len(cams), ref.ctypes.data_as(i32), cur.ctypes.data_as(i32)], (arr, ref, cur)


def match_direct(abi, cams, cam_of_ref, cam_of_cur, data, n_threads: int = 0):
    """Matcher::findMatchDirect on a synth.MatchData batch with a camera per image -> abi.MatchOut."""
    lib = load(abi)
    b, keep = abi.make_match_batch(data)
    args, keep2 = _tables(abi, cams, cam_of_ref, cam_of_cur)
    out = abi.MatchOut(data.n)
    rc = lib.plsvo_oracle_match_direct_multicam_batch(*args, C.byref(b), C.byref(out.struct), _threads(n_threads))
    if rc != 0:
        raise RuntimeError(f"multicam oracle match_direct failed rc={rc}")
    return out


def match_direct_given_A(abi, cams, cam_of_ref, cam_of_cur, data, A, n_threads: int = 0):
    """match_direct() downstream of the warp matrix, with A_cur_ref [n, 4] (row-major) given per candidate -> abi.MatchOut.
    Rows whose in-frame test fails are not read."""
    lib = load(abi)
    A = np.ascontiguousarray(A, np.float64).reshape(data.n, 4)
    b, keep = abi.make_match_batch(data)
    args, keep2 = _tables(abi, cams, cam_of_ref, cam_of_cur)
    out = abi.MatchOut(data.n)
    rc = lib.plsvo_oracle_match_direct_multicam_given_A(*args, A.ctypes.data_as(C.POINTER(C.c_double)), C.byref(b), C.byref(out.struct),
                                                        _threads(n_threads))
    if rc != 0:
        raise RuntimeError(f"multicam oracle match_direct_given_A failed rc={rc}")
    return out


def build_ref(force: bool = False) -> str | None:
    """Build oracle/_ref/libplsvo_multicam_match_ref.so where the reference sources are present.  Returns its path, or None
    when neither the sources nor a prebuilt library exist."""
    srcs = [os.path.join(oracle_atan.REFERENCE_ROOT, "src", f) for f in oracle_atan.REF_SRCS]
    harness = [os.path.join(_HERE, f) for f in ("multicam_match_ref_harness.cpp", "atan_ref_harness.cpp", "ref_harness.cpp", "next_scenes.h")]
    if all(os.path.exists(s) for s in srcs):
        deps = srcs + harness + SOURCES[2:] + [os.path.join(_HERE, "..", "include", "plsvo_b200.h")]
        stale = not os.path.exists(REF_LIB_PATH) or any(os.path.getmtime(f) > os.path.getmtime(REF_LIB_PATH) for f in deps)
        if force or stale:
            os.makedirs(os.path.dirname(REF_LIB_PATH), exist_ok=True)
            subprocess.check_call([os.environ.get("CXX", "g++")] + oracle_atan.REF_CXXFLAGS + [
                "-I" + os.path.join(_HERE, "refdeps"), "-I" + os.path.join(oracle_atan.REFERENCE_ROOT, "include"), "-shared", "-o",
                REF_LIB_PATH] + srcs + [harness[0], "-lpthread"])
    return REF_LIB_PATH if os.path.exists(REF_LIB_PATH) else None


def ref_available() -> bool:
    return os.path.exists(REF_LIB_PATH)


def ref_match_direct(abi, cams, cam_of_ref, cam_of_cur, data):
    """Matcher::findMatchDirect of the reference's own matcher.cpp, every frame holding its own camera -> abi.MatchOut."""
    global _ref_lib
    if _ref_lib is None:
        lib = C.CDLL(REF_LIB_PATH)
        lib.plsvo_ref_match_direct_multicam_batch.restype = C.c_int
        lib.plsvo_ref_match_direct_multicam_batch.argtypes = _cam_args(abi, C.POINTER) + [C.POINTER(abi.MatchBatch),
                                                                                         C.POINTER(abi.MatchResult)]
        _ref_lib = lib
    b, keep = abi.make_match_batch(data)
    args, keep2 = _tables(abi, cams, cam_of_ref, cam_of_cur)
    out = abi.MatchOut(data.n)
    rc = _ref_lib.plsvo_ref_match_direct_multicam_batch(*args, C.byref(b), C.byref(out.struct))
    if rc != 0:
        raise RuntimeError(f"reference multicam match_direct failed rc={rc}")
    return out
