"""Loader of the CPU restatement of vk::PinholeCamera::undistortImage (oracle/undistort_oracle.cpp ->
oracle/libplsvo_undistort_oracle.so).  TEST INFRASTRUCTURE ONLY, like oracle_lib: the product package never imports it.
Levels below the rectified frame come from oracle_lib's createImgPyramid restatement."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, "undistort_oracle.cpp")
LIB_PATH = os.path.join(_HERE, "libplsvo_undistort_oracle.so")
# the flags of oracle/Makefile: strict IEEE (no FMA contraction), portable to the GPU box's host
CXXFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-math-errno", "-std=c++17", "-fPIC", "-Wall"]
_lib = None


def build(force: bool = False) -> str:
    hdr = os.path.join(_HERE, "..", "include", "plsvo_b200.h")
    if force or not os.path.exists(LIB_PATH) or any(os.path.getmtime(f) > os.path.getmtime(LIB_PATH) for f in (SRC, hdr)):
        subprocess.check_call([os.environ.get("CXX", "g++"), *CXXFLAGS, "-shared", "-o", LIB_PATH + ".tmp", SRC, "-lpthread"])
        os.replace(LIB_PATH + ".tmp", LIB_PATH)
    return LIB_PATH


def load(abi):
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        lib = C.CDLL(LIB_PATH)
        P = C.POINTER
        lib.plsvo_oracle_undistort_map.restype = C.c_int
        lib.plsvo_oracle_undistort_map.argtypes = [P(abi.PinholeCamera), P(C.c_int16), P(C.c_uint16), C.c_size_t]
        lib.plsvo_oracle_undistort_frames.restype = C.c_int
        lib.plsvo_oracle_undistort_frames.argtypes = [P(abi.UndistortBatch), P(C.c_int16), P(C.c_uint16), P(abi.PyramidResult), C.c_int]
        _lib = lib
    return _lib


def undistort_map(abi, cam):
    """cv::initUndistortRectifyMap as vk::PinholeCamera builds it: abi.PinholeCamera -> (map1 int16 [H,W,2], map2 uint16 [H,W])."""
    map1 = np.zeros((cam.height, cam.width, 2), np.int16)
    map2 = np.zeros((cam.height, cam.width), np.uint16)
    if load(abi).plsvo_oracle_undistort_map(C.byref(cam), map1.ctypes.data_as(C.POINTER(C.c_int16)),
                                            map2.ctypes.data_as(C.POINTER(C.c_uint16)), cam.width) != 0:
        raise RuntimeError("oracle undistort_map failed")
    return map1, map2


def undistort_level0(abi, cam, raw, n_threads: int = 1, maps=None):
    """undistortImage of u8 [B,H,W] raw frames (any row pitch / frame stride) -> rectified frames [B,H,W].
    maps = undistort_map(...) reuses a map, as the camera's constructor builds it once."""
    B, H, W = raw.shape
    assert raw.dtype == np.uint8 and raw.strides[2] == 1 and (W, H) == (cam.width, cam.height)
    b = abi.UndistortBatch(cam, B, 1, raw.ctypes.data_as(C.POINTER(C.c_uint8)), raw.strides[1], raw.strides[0])
    levels, r = abi.pyramid_levels(B, H, W, 1)
    if maps is None and abs(cam.d[0]) > 1e-7:
        maps = undistort_map(abi, cam)
    m1 = maps[0].ctypes.data_as(C.POINTER(C.c_int16)) if maps is not None else None
    m2 = maps[1].ctypes.data_as(C.POINTER(C.c_uint16)) if maps is not None else None
    if load(abi).plsvo_oracle_undistort_frames(C.byref(b), m1, m2, C.byref(r), n_threads) != 0:
        raise RuntimeError("oracle undistort failed")
    return levels[0]


def undistort(abi, cam, raw, n_levels: int = 1, n_threads: int = 1, maps=None):
    """vk::PinholeCamera::undistortImage + createImgPyramid restated -> list of levels, level 0 rectified."""
    return oracle_lib.pyramid(abi, undistort_level0(abi, cam, raw, n_threads, maps), n_levels)
