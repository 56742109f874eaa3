"""Loader of the CPU oracle's ATAN matcher (oracle/atan_match_oracle.cpp -> oracle/libplsvo_atan_match_oracle.so), of
its checker, the reference's own matcher.cpp with the stand-in vk::ATANCamera (oracle/atan_match_ref_harness.cpp ->
oracle/_ref/libplsvo_atan_match_ref.so), and of the reprojector scene answered by the drop-in DirectMatcher on ATAN frames
(oracle/atan_match_shimref_harness.cpp -> oracle/_ref/libplsvo_atan_match_shimref{,_cpu}.so).

TEST INFRASTRUCTURE ONLY, like oracle_lib and oracle_atan: Matcher::findMatchDirect seen through vk::ATANCamera, and the
same matcher downstream of a given A_cur_ref.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle_atan

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libplsvo_atan_match_oracle.so")
SOURCES = [os.path.join(_HERE, "atan_match_oracle.cpp")] + oracle_atan.SOURCES[1:]
_lib = None

REF_LIB_PATH = os.path.join(_HERE, "_ref", "libplsvo_atan_match_ref.so")
_ref_lib = None


def build(force: bool = False) -> str:
    deps = SOURCES + [os.path.join(_HERE, "..", "include", "plsvo_b200.h")]
    stale = not os.path.exists(LIB_PATH) or any(os.path.getmtime(f) > os.path.getmtime(LIB_PATH) for f in deps)
    if force or stale:
        subprocess.check_call([os.environ.get("CXX", "g++")] + oracle_atan.CXXFLAGS + ["-I" + os.path.join(_HERE, "refdeps"), "-shared",
                                                                                      "-o", LIB_PATH, SOURCES[0], "-lpthread"])
    return LIB_PATH


def load(abi):
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        build()
    lib = C.CDLL(LIB_PATH)
    P = C.POINTER
    lib.plsvo_oracle_atan_match_direct_batch.restype = C.c_int
    lib.plsvo_oracle_atan_match_direct_batch.argtypes = [P(abi.AtanCamera), P(abi.MatchBatch), P(abi.MatchResult), C.c_int]
    lib.plsvo_oracle_atan_match_direct_members.restype = C.c_int
    lib.plsvo_oracle_atan_match_direct_members.argtypes = [C.c_double] * 5 + [P(abi.MatchBatch), P(abi.MatchResult), C.c_int]
    lib.plsvo_oracle_match_direct_given_A.restype = C.c_int
    lib.plsvo_oracle_match_direct_given_A.argtypes = [P(C.c_double), P(abi.MatchBatch), P(abi.MatchResult), C.c_int]
    _lib = lib
    return lib


def _threads(n_threads: int) -> int:
    return n_threads if n_threads > 0 else (os.cpu_count() or 1)


def match_direct(abi, camera, data, n_threads: int = 0, out=None):
    """Matcher::findMatchDirect on a synth.MatchData batch seen through `camera` (api.ATANCamera) -> abi.MatchOut."""
    lib = load(abi)
    b, keep = abi.make_match_batch(data)
    out = out or abi.MatchOut(data.n)
    rc = lib.plsvo_oracle_atan_match_direct_batch(C.byref(camera.struct), C.byref(b), C.byref(out.struct), _threads(n_threads))
    if rc != 0:
        raise RuntimeError(f"ATAN oracle match_direct failed rc={rc}")
    return out


def match_direct_members(abi, camera, data, n_threads: int = 0, out=None):
    """match_direct() with the camera given by its members fx_, fy_, cx_, cy_ and d0 (the device kernel's MatchArgs)."""
    lib = load(abi)
    b, keep = abi.make_match_batch(data)
    out = out or abi.MatchOut(data.n)
    rc = lib.plsvo_oracle_atan_match_direct_members(camera.fx_, camera.fy_, camera.cx_, camera.cy_, camera.s_, C.byref(b),
                                                    C.byref(out.struct), _threads(n_threads))
    if rc != 0:
        raise RuntimeError(f"ATAN oracle match_direct failed rc={rc}")
    return out


def match_direct_given_A(abi, data, A, n_threads: int = 0):
    """findMatchDirect downstream of the warp matrix, with A_cur_ref [n, 4] (row-major) given per candidate -> abi.MatchOut.
    Rows whose in-frame test fails are not read."""
    lib = load(abi)
    A = np.ascontiguousarray(A, np.float64).reshape(data.n, 4)
    b, keep = abi.make_match_batch(data)
    out = abi.MatchOut(data.n)
    rc = lib.plsvo_oracle_match_direct_given_A(A.ctypes.data_as(C.POINTER(C.c_double)), C.byref(b), C.byref(out.struct),
                                               _threads(n_threads))
    if rc != 0:
        raise RuntimeError(f"oracle match_direct_given_A failed rc={rc}")
    return out


def build_ref(force: bool = False) -> str | None:
    """Build oracle/_ref/libplsvo_atan_match_ref.so where the reference sources are present.  Returns its path, or None
    when neither the sources nor a prebuilt library exist."""
    srcs = [os.path.join(oracle_atan.REFERENCE_ROOT, "src", f) for f in oracle_atan.REF_SRCS]
    harness = [os.path.join(_HERE, f) for f in ("atan_match_ref_harness.cpp", "atan_ref_harness.cpp", "ref_harness.cpp", "next_scenes.h",
                                                "atan_next_scenes.h")]
    if all(os.path.exists(s) for s in srcs):
        deps = srcs + harness + oracle_atan.SOURCES[2:] + [os.path.join(_HERE, "..", "include", "plsvo_b200.h")]
        stale = not os.path.exists(REF_LIB_PATH) or any(os.path.getmtime(f) > os.path.getmtime(REF_LIB_PATH) for f in deps)
        if force or stale:
            os.makedirs(os.path.dirname(REF_LIB_PATH), exist_ok=True)
            subprocess.check_call([os.environ.get("CXX", "g++")] + oracle_atan.REF_CXXFLAGS + [
                "-I" + os.path.join(_HERE, "refdeps"), "-I" + os.path.join(oracle_atan.REFERENCE_ROOT, "include"), "-shared", "-o",
                REF_LIB_PATH] + srcs + [harness[0], "-lpthread"])
    return REF_LIB_PATH if os.path.exists(REF_LIB_PATH) else None


def ref_available() -> bool:
    return os.path.exists(REF_LIB_PATH)


def _load_ref(abi):
    global _ref_lib
    if _ref_lib is None:
        lib = C.CDLL(REF_LIB_PATH)
        lib.plsvo_ref_atan_match_direct_batch.restype = C.c_int
        lib.plsvo_ref_atan_match_direct_batch.argtypes = [C.POINTER(abi.AtanCamera), C.POINTER(abi.MatchBatch), C.POINTER(abi.MatchResult)]
        _ref_lib = lib
    return _ref_lib


def ref_match_direct(abi, camera, data):
    """Matcher::findMatchDirect of the reference's own matcher.cpp, the frames seen through `camera` -> abi.MatchOut."""
    lib = _load_ref(abi)
    b, keep = abi.make_match_batch(data)
    out = abi.MatchOut(data.n)
    rc = lib.plsvo_ref_atan_match_direct_batch(C.byref(camera.struct), C.byref(b), C.byref(out.struct))
    if rc != 0:
        raise RuntimeError(f"reference ATAN match_direct failed rc={rc}")
    return out


class _WithCamera:
    """fn(camera, batch, n_obs, out) presented as fn(batch, n_obs, out), the shape oracle_lib._match_scene calls (it sets
    restype / argtypes on what it is given, which this ignores)."""

    def __init__(self, fn, abi, camera):
        import oracle_lib

        fn.restype = C.c_int
        fn.argtypes = [C.POINTER(abi.AtanCamera), C.POINTER(abi.MatchBatch), C.c_int, C.POINTER(oracle_lib.SceneMatchOut)]
        self.fn, self.camera = fn, camera

    def __call__(self, b, n_obs, out):
        return self.fn(C.byref(self.camera.struct), b, n_obs, out)


def ref_match_scene(abi, camera, data, n_obs=3):
    """Reprojector-style pass of the reference's own Matcher over map points / segments observed in n_obs keyframes, every
    frame seen through `camera` (oracle_lib.ref_match_scene with an ATAN camera)."""
    import oracle_lib

    return oracle_lib._match_scene(_WithCamera(_load_ref(abi).plsvo_ref_atan_match_scene, abi, camera), abi, data, n_obs)


SHIMREF_LIB_PATH = os.path.join(_HERE, "_ref", "libplsvo_atan_match_shimref.so")
SHIMREF_CPU_LIB_PATH = os.path.join(_HERE, "_ref", "libplsvo_atan_match_shimref_cpu.so")
_shimref_libs = {}


def build_shimref(force: bool = False, cpu: bool = False) -> str | None:
    """oracle/_ref/libplsvo_atan_match_shimref.so (the shim on the product library) or, with cpu, ..._cpu.so (the shim on
    the C ABI answered by the CPU oracle).  Needs the reference sources (and, without cpu, the built CUDA library)."""
    shim_dir = os.path.join(_HERE, "..", "pl-svo_b200", "host")
    csrc = os.path.join(_HERE, "..", "pl-svo_b200", "csrc")
    out = SHIMREF_CPU_LIB_PATH if cpu else SHIMREF_LIB_PATH
    srcs = [os.path.join(oracle_atan.REFERENCE_ROOT, "src", f) for f in oracle_atan.SHIMREF_REF_SRCS]
    shim = [os.path.join(shim_dir, f) for f in ("plsvo_shim.cpp", "plsvo_shim_next.cpp")]
    harness = [os.path.join(_HERE, f) for f in ("atan_match_shimref_harness.cpp", "atan_shimref_harness.cpp", "shimref_harness.cpp",
                                                "next_scenes.h", "atan_next_scenes.h")]
    backend = ([os.path.join(_HERE, f) for f in ("abi_on_oracle.cpp", "atan_abi_on_oracle.cpp", "atan_match_oracle.cpp")] if cpu else [])
    if all(os.path.exists(s) for s in srcs) and (cpu or os.path.exists(os.path.join(csrc, "libplsvo_b200.so"))):
        deps = srcs + shim + harness + backend + [os.path.join(shim_dir, f) for f in ("plsvo_shim.h", "plsvo_shim_next.h")] + \
            oracle_atan.SOURCES[1:] + [os.path.join(_HERE, "..", "include", "plsvo_b200.h")]
        stale = not os.path.exists(out) or any(os.path.getmtime(f) > os.path.getmtime(out) for f in deps)
        if force or stale:
            os.makedirs(os.path.dirname(out), exist_ok=True)
            flags = ["-O2", "-std=c++17", "-fPIC", "-w", "-DNDEBUG", "-DPLSVO_SHIM_WITH_REFERENCE_HEADERS"]
            if cpu:
                flags[1:1] = ["-march=x86-64-v3", "-ffp-contract=off"]  # the oracle's flags (oracle/Makefile's shimref-cpu)
            link = ["-Wl,-Bsymbolic", "-lpthread"] if cpu else ["-L" + csrc, "-lplsvo_b200", "-Wl,-rpath,$ORIGIN/../../pl-svo_b200/csrc",
                                                               "-lpthread"]
            subprocess.check_call([os.environ.get("CXX", "g++")] + flags + [
                "-I" + os.path.join(shim_dir, "overlay"), "-I" + os.path.join(_HERE, "refdeps"),
                "-I" + os.path.join(oracle_atan.REFERENCE_ROOT, "include"), "-I" + os.path.join(_HERE, "..", "include"), "-I" + shim_dir,
                "-shared", "-o", out] + srcs + shim + [harness[0]] + backend + link)
    return out if os.path.exists(out) else None


def shimref_match_scene(abi, camera, data, n_obs=3, cpu: bool = False):
    """The same pass as ref_match_scene answered by plsvo::b200::DirectMatcher (one C-ABI call per frame: on the GPU, or
    with cpu on the oracle-backed adapter)."""
    path = SHIMREF_CPU_LIB_PATH if cpu else SHIMREF_LIB_PATH
    if path not in _shimref_libs:
        _shimref_libs[path] = C.CDLL(path)
    import oracle_lib

    return oracle_lib._match_scene(_WithCamera(_shimref_libs[path].plsvo_shimref_atan_match_scene, abi, camera), abi, data, n_obs)
