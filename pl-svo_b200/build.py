"""In-tree build of libplsvo_b200.so with nvcc for sm_90a (no JIT cache, the .so travels with the repo)."""
from __future__ import annotations

import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
SOURCES = ["align_kernel.cu", "poseopt_kernel.cu", "pyramid_kernel.cu", "align2d_kernel.cu", "structopt_kernel.cu", "undistort_kernel.cu",
           "plsvo_abi.cu"]
HEADERS = ["device_math.cuh", "exact_math.cuh", "halfsample.cuh", "internal.h", os.path.join("..", "..", "include", "plsvo_b200.h")]
OUT = os.path.join(CSRC, "libplsvo_b200.so")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
    "-diag-suppress", "177",
]


def is_stale() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    # this file holds NVCC_FLAGS (the target architecture): a library built with other flags is stale too
    return os.path.getmtime(__file__) > t or any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return OUT
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libplsvo_b200.so")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT] + SOURCES
    subprocess.check_call(cmd, cwd=CSRC)
    return OUT


def build_variant(tag: str, defines: list[str], verbose: bool = False) -> str:
    """A/B builds of the library with preprocessor switches (e.g. PLSVO_FP32_SUMS, PLSVO_TREE_CHI2), loaded through
    PLSVO_LIB; used by A/B measurements, never by the product path."""
    out = os.path.join(CSRC, f"libplsvo_b200_{tag}.so")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cmd = [nvcc] + NVCC_FLAGS + [f"-D{d}" for d in defines] + (["-Xptxas", "-v"] if verbose else []) + ["-o", out] + SOURCES
    subprocess.check_call(cmd, cwd=CSRC)
    return out


HOST = os.path.join(_HERE, "host")
SHIM_OUT = os.path.join(HOST, "libplsvo_shim.so")
SHIM_SOURCES = ["plsvo_shim.cpp", "shim_harness.cpp"]


def build_shim(force: bool = False) -> str:
    """The signature-preserving C++ shim (host side above the C ABI) + its test harness, built against the
    compat stand-in types (the reference's own headers are not available in this image)."""
    deps = [os.path.join(HOST, f) for f in SHIM_SOURCES + ["plsvo_shim.h", "plsvo_compat.h"]] + [OUT]
    if not force and os.path.exists(SHIM_OUT) and all(os.path.getmtime(d) <= os.path.getmtime(SHIM_OUT) for d in deps):
        return SHIM_OUT
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", SHIM_OUT] + SHIM_SOURCES + [
        "-L" + CSRC, "-lplsvo_b200", "-Wl,-rpath,$ORIGIN/../csrc"]
    subprocess.check_call(cmd, cwd=HOST)
    return SHIM_OUT
