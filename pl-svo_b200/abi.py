"""ctypes mirror of include/plsvo_b200.h and the loader of the CUDA library.

There is no CPU fallback: `load_library()` raises if libplsvo_b200.so has not been built, and
every entry point of the library itself returns PLSVO_ERR_NO_DEVICE without a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

MAX_LEVELS = 8
PATCH_AREA = 16

OK = 0
ERR_INVALID = -1
ERR_CUDA = -2
ERR_NO_DEVICE = -3
ERR_STATE = -4

_u8p = C.POINTER(C.c_uint8)
_f64p = C.POINTER(C.c_double)
_i32p = C.POINTER(C.c_int32)
_i64p = C.POINTER(C.c_int64)
_u32p = C.POINTER(C.c_uint32)


class Camera(C.Structure):
    _fields_ = [
        ("width", C.c_int32),
        ("height", C.c_int32),
        ("reserved0", C.c_int32),
        ("reserved1", C.c_int32),
        ("fx", C.c_double),
        ("fy", C.c_double),
        ("cx", C.c_double),
        ("cy", C.c_double),
    ]


class AlignParams(C.Structure):
    _fields_ = [
        ("max_level", C.c_int32),
        ("min_level", C.c_int32),
        ("n_iter", C.c_int32),
        ("reserved", C.c_int32),
        ("eps", C.c_double),
    ]


ALIGN_FRAME_CHAIN = 1  # PLSVO_ALIGN_FRAME_CHAIN (include/plsvo_b200.h)


class AlignBatch(C.Structure):
    _fields_ = [
        ("batch", C.c_int32),
        ("n_pts", C.c_int32),
        ("n_segs", C.c_int32),
        ("flags", C.c_int32),  # 0 or ALIGN_FRAME_CHAIN
        ("cam", Camera),
        ("ref_img", _u8p * MAX_LEVELS),
        ("cur_img", _u8p * MAX_LEVELS),
        ("img_pitch", C.c_size_t * MAX_LEVELS),
        ("img_stride", C.c_size_t * MAX_LEVELS),
        ("T_ref_w", _f64p),
        ("T_cur_w", _f64p),
        ("pt_count", _i32p),
        ("pt_px", _f64p),
        ("pt_f", _f64p),
        ("pt_pos", _f64p),
        ("pt_valid", _u8p),
        ("seg_count", _i32p),
        ("seg_spx", _f64p),
        ("seg_epx", _f64p),
        ("seg_sf", _f64p),
        ("seg_ef", _f64p),
        ("seg_spos", _f64p),
        ("seg_epos", _f64p),
        ("seg_length", _f64p),
        ("seg_valid", _u8p),
        ("pt_depth", _f64p),
        ("seg_sdepth", _f64p),
        ("seg_edepth", _f64p),
    ]


class AlignResult(C.Structure):
    _fields_ = [
        ("T_cur_w", _f64p),
        ("n_tracked", _i64p),
        ("H", _f64p),
        ("seg_killed", _u8p),
        ("iters", _i32p),
        ("status", _i32p),
        ("patch_iters", _u32p),
        ("patch_levels", _u32p),
    ]


class PoseOptParams(C.Structure):
    _fields_ = [("reproj_thresh", C.c_double), ("n_iter", C.c_int32), ("n_iter_ref", C.c_int32)]


class PoseOptBatch(C.Structure):
    _fields_ = [
        ("batch", C.c_int32),
        ("n_pts", C.c_int32),
        ("n_segs", C.c_int32),
        ("reserved", C.c_int32),
        ("fx", C.c_double),
        ("T_f_w", _f64p),
        ("pt_count", _i32p),
        ("pt_f", _f64p),
        ("pt_pos", _f64p),
        ("pt_level", _i32p),
        ("pt_valid", _u8p),
        ("seg_count", _i32p),
        ("seg_line", _f64p),
        ("seg_spos", _f64p),
        ("seg_epos", _f64p),
        ("seg_level", _i32p),
        ("seg_valid", _u8p),
    ]


class PoseOptResult(C.Structure):
    _fields_ = [
        ("T_f_w", _f64p),
        ("cov", _f64p),
        ("estimated_scale", _f64p),
        ("error_init", _f64p),
        ("error_final", _f64p),
        ("num_obs_pt", _i64p),
        ("num_obs_ls", _i64p),
        ("pt_outlier", _u8p),
        ("seg_outlier", _u8p),
        ("iters", _i32p),
        ("status", _i32p),
    ]


class PyramidBatch(C.Structure):
    _fields_ = [("batch", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("n_levels", C.c_int32),
                ("img0", _u8p), ("pitch0", C.c_size_t), ("stride0", C.c_size_t)]


class PyramidResult(C.Structure):
    _fields_ = [("level", _u8p * MAX_LEVELS), ("pitch", C.c_size_t * MAX_LEVELS), ("stride", C.c_size_t * MAX_LEVELS)]


class PinholeCamera(C.Structure):
    """plsvo_pinhole_camera: the distorted vk::PinholeCamera constructor arguments."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double),
                ("cy", C.c_double), ("d", C.c_double * 5)]


class UndistortBatch(C.Structure):
    _fields_ = [("cam", PinholeCamera), ("batch", C.c_int32), ("n_levels", C.c_int32), ("img0", _u8p), ("pitch0", C.c_size_t),
                ("stride0", C.c_size_t)]


class RawFrames(C.Structure):
    """plsvo_raw_frames: the distorted camera and the raw frame stacks of plsvo_align_raw_batch_run /
    plsvo_track_raw_batch_run."""
    _fields_ = [("cam", PinholeCamera), ("ref_raw", _u8p), ("cur_raw", _u8p), ("pitch", C.c_size_t), ("stride", C.c_size_t)]


def make_raw_frames(cam: PinholeCamera, raw, batch: int):
    """plsvo_raw_frames for `batch` pairs from raw u8 frames: one array [B+1,H,W] (a frame chain) or a pair (ref, cur) of
    [B,H,W] arrays with the same strides.  Rows may be padded.  Returns (struct, chain, keepalive)."""
    chain = not isinstance(raw, (tuple, list))
    stacks = [np.asarray(raw)] if chain else [np.asarray(x) for x in raw]
    if not chain and len(stacks) != 2:
        raise ValueError("raw frames: one [B+1,H,W] chain or a (ref, cur) pair of [B,H,W] stacks")
    for s in stacks:
        if s.dtype != np.uint8 or s.ndim != 3 or s.strides[2] != 1 or s.shape[1:] != (cam.height, cam.width):
            raise ValueError(f"raw frames must be u8 [n,{cam.height},{cam.width}] with unit column stride")
        if s.shape[0] != batch + (1 if chain else 0):
            raise ValueError(f"raw frames: {s.shape[0]} frames for {batch} pairs" + (" (a chain has B+1)" if chain else ""))
        if s.strides != stacks[0].strides:
            raise ValueError("raw frames: both stacks must have the same layout")
    r = RawFrames(cam, stacks[0].ctypes.data_as(_u8p), None if chain else stacks[1].ctypes.data_as(_u8p),
                  stacks[0].strides[1], stacks[0].strides[0])
    return r, chain, stacks


def pyramid_levels(B: int, H: int, W: int, n_levels: int):
    """Contiguous u8 output levels [B, H>>l, W>>l] for l < n_levels and the plsvo_pyramid_result pointing at all of them."""
    r = PyramidResult()
    levels = []
    for l in range(n_levels):
        out = np.empty((B, H >> l, W >> l), np.uint8)
        levels.append(out)
        r.level[l] = out.ctypes.data_as(_u8p)
        r.pitch[l] = out.strides[1]
        r.stride[l] = out.strides[0]
    return levels, r


class Align2DBatch(C.Structure):
    _fields_ = [("n_features", C.c_int32), ("n_images", C.c_int32), ("width", C.c_int32), ("height", C.c_int32),
                ("n_iter", C.c_int32), ("reserved", C.c_int32),
                ("img", _u8p * MAX_LEVELS), ("img_pitch", C.c_size_t * MAX_LEVELS), ("img_stride", C.c_size_t * MAX_LEVELS),
                ("image_index", _i32p), ("level", _i32p), ("ref_patch_with_border", _u8p), ("ref_patch", _u8p), ("px", _f64p)]


class Align2DResult(C.Structure):
    _fields_ = [("px", _f64p), ("converged", _u8p)]


class Align1DBatch(C.Structure):
    _fields_ = [("features", Align2DBatch), ("dir", C.POINTER(C.c_float))]


class Align1DResult(C.Structure):
    _fields_ = [("px", _f64p), ("converged", _u8p), ("h_inv", _f64p)]


class MatchBatch(C.Structure):
    _fields_ = [("n_features", C.c_int32), ("n_ref_images", C.c_int32), ("n_cur_images", C.c_int32), ("n_pyr_levels", C.c_int32),
                ("n_iter", C.c_int32), ("reserved", C.c_int32), ("cam", Camera),
                ("ref_img", _u8p * MAX_LEVELS), ("ref_pitch", C.c_size_t * MAX_LEVELS), ("ref_stride", C.c_size_t * MAX_LEVELS),
                ("cur_img", _u8p * MAX_LEVELS), ("cur_pitch", C.c_size_t * MAX_LEVELS), ("cur_stride", C.c_size_t * MAX_LEVELS),
                ("T_ref_w", _f64p), ("T_cur_w", _f64p), ("ref_index", _i32p), ("cur_index", _i32p), ("ref_px", _f64p),
                ("ref_f", _f64p), ("ref_level", _i32p), ("is_edgelet", _u8p), ("ref_grad", _f64p), ("pos", _f64p),
                ("px_cur", _f64p)]


class StructOptBatch(C.Structure):
    _fields_ = [("n_points", C.c_int32), ("n_segs", C.c_int32), ("n_frames", C.c_int32), ("n_iter_pts", C.c_int32),
                ("n_iter_segs", C.c_int32), ("reserved", C.c_int32), ("T_f_w", _f64p),
                ("pt_obs_begin", _i32p), ("pt_obs_frame", _i32p), ("pt_obs_f", _f64p), ("pt_pos", _f64p),
                ("seg_obs_begin", _i32p), ("seg_obs_frame", _i32p), ("seg_obs_sf", _f64p), ("seg_obs_ef", _f64p),
                ("seg_spos", _f64p), ("seg_epos", _f64p)]


class StructOptResult(C.Structure):
    _fields_ = [("pt_pos", _f64p), ("seg_spos", _f64p), ("seg_epos", _f64p), ("pt_iters", _i32p), ("seg_iters", _i32p)]


_f32p = C.POINTER(C.c_float)


class SeedBatch(C.Structure):
    _fields_ = [("n_seeds", C.c_int32), ("n_ref_images", C.c_int32), ("n_cur_images", C.c_int32), ("n_pyr_levels", C.c_int32),
                ("n_iter", C.c_int32), ("max_epi_search_steps", C.c_int32), ("align_1d", C.c_uint8), ("subpix_refinement", C.c_uint8),
                ("epi_search_edgelet_filtering", C.c_uint8), ("reserved0", C.c_uint8 * 5),
                ("epi_search_edgelet_max_angle", C.c_double), ("seed_convergence_sigma2_thresh", C.c_double), ("cam", Camera),
                ("ref_img", _u8p * MAX_LEVELS), ("ref_pitch", C.c_size_t * MAX_LEVELS), ("ref_stride", C.c_size_t * MAX_LEVELS),
                ("cur_img", _u8p * MAX_LEVELS), ("cur_pitch", C.c_size_t * MAX_LEVELS), ("cur_stride", C.c_size_t * MAX_LEVELS),
                ("T_ref_w", _f64p), ("T_cur_w", _f64p), ("ref_index", _i32p), ("cur_index", _i32p), ("ref_px", _f64p),
                ("ref_f", _f64p), ("ref_level", _i32p), ("is_edgelet", _u8p), ("ref_grad", _f64p),
                ("a", _f32p), ("b", _f32p), ("mu", _f32p), ("z_range", _f32p), ("sigma2", _f32p)]


class SeedResult(C.Structure):
    _fields_ = [("a", _f32p), ("b", _f32p), ("mu", _f32p), ("sigma2", _f32p), ("status", _i32p), ("converged", _u8p),
                ("depth", _f64p), ("px_cur", _f64p)]


class LineSeedBatch(C.Structure):
    _fields_ = [("seeds", SeedBatch), ("ref_sf", _f64p), ("ref_ef", _f64p), ("mu_e", _f32p), ("z_range_e", _f32p), ("sigma2_e", _f32p)]


class LineSeedResult(C.Structure):
    _fields_ = [("seeds", SeedResult), ("mu_e", _f32p), ("sigma2_e", _f32p), ("depth_e", _f64p), ("px_cur_e", _f64p)]


SEED_NOT_VISIBLE, SEED_NO_MATCH, SEED_UPDATED = 0, 1, 2


class MatchResult(C.Structure):
    _fields_ = [("px_cur", _f64p), ("success", _u8p), ("search_level", _i32p), ("A_cur_ref", _f64p)]


# ------------------------------------------------------------------------------------------------
# numpy <-> struct helpers
# ------------------------------------------------------------------------------------------------

_CT = {np.dtype(np.float32): C.POINTER(C.c_float), np.dtype(np.uint8): _u8p, np.dtype(np.float64): _f64p, np.dtype(np.int32): _i32p,
       np.dtype(np.int64): _i64p, np.dtype(np.uint32): _u32p}


def _ptr(a, dtype):
    """Pointer to a C-contiguous numpy array of `dtype`, or NULL for None."""
    if a is None:
        return _CT[np.dtype(dtype)]()
    if not isinstance(a, np.ndarray) or a.dtype != np.dtype(dtype) or not a.flags.c_contiguous:
        raise TypeError(f"expected C-contiguous {np.dtype(dtype)} array, got {type(a)} {getattr(a, 'dtype', None)}")
    return a.ctypes.data_as(_CT[np.dtype(dtype)])


# Compiled variants of the alignment kernel as (threads per CTA, resident CTAs per SM), the values PLSVO_VARIANT accepts
# ("threads,ctas"): kAlignVariants in csrc/plsvo_abi.cu.  A variant missing here is missing from the parity tests.
ALIGN_VARIANTS = ((64, 8), (96, 7), (96, 5), (128, 5), (128, 4), (160, 3), (192, 2), (256, 2))


def align_params(max_level=4, min_level=2, n_iter=30, eps=1e-6) -> AlignParams:
    return AlignParams(max_level, min_level, n_iter, 0, eps)


def poseopt_params(reproj_thresh=2.0, n_iter=10, n_iter_ref=-1) -> PoseOptParams:
    return PoseOptParams(reproj_thresh, n_iter, n_iter_ref)


def make_align_batch(d):
    """Build a plsvo_align_batch from an AlignData-like object.  Returns (struct, keepalive)."""
    b = AlignBatch()
    keep = [d]
    b.batch, b.n_pts, b.n_segs = d.batch, d.n_pts, d.n_segs
    cam = d.cam
    b.cam = Camera(cam.width, cam.height, 0, 0, cam.fx, cam.fy, cam.cx, cam.cy)
    frame_pyr = getattr(d, "frame_pyr", None)
    if frame_pyr is not None:
        # frame chain (PLSVO_ALIGN_FRAME_CHAIN): one stack of B+1 frames per level, pair b = (frame b, frame b+1)
        b.flags = ALIGN_FRAME_CHAIN
        for l, f in frame_pyr.items():
            assert f.dtype == np.uint8 and f.ndim == 3 and f.shape[0] == d.batch + 1 and f.strides[2] == 1
            b.ref_img[l] = f.ctypes.data_as(_u8p)
            b.img_pitch[l] = f.strides[1]
            b.img_stride[l] = f.strides[0]
    for l in range(MAX_LEVELS):
        if frame_pyr is None and l in d.ref_pyr:
            r, c = d.ref_pyr[l], d.cur_pyr[l]
            assert r.dtype == np.uint8 and r.ndim == 3 and r.shape == c.shape
            assert r.strides[2] == 1 and c.strides == r.strides
            b.ref_img[l] = r.ctypes.data_as(_u8p)
            b.cur_img[l] = c.ctypes.data_as(_u8p)
            b.img_pitch[l] = r.strides[1]
            b.img_stride[l] = r.strides[0]
    b.T_ref_w = _ptr(d.T_ref_w, np.float64)
    b.T_cur_w = _ptr(d.T_cur_w, np.float64)
    b.pt_count = _ptr(d.pt_count, np.int32)
    b.pt_px = _ptr(d.pt_px, np.float64)
    b.pt_f = _ptr(getattr(d, "pt_f", None), np.float64)
    b.pt_pos = _ptr(getattr(d, "pt_pos", None), np.float64)
    b.pt_depth = _ptr(getattr(d, "pt_depth", None), np.float64)
    b.pt_valid = _ptr(d.pt_valid, np.uint8)
    b.seg_count = _ptr(d.seg_count, np.int32)
    if d.n_segs > 0:
        b.seg_spx = _ptr(d.seg_spx, np.float64)
        b.seg_epx = _ptr(d.seg_epx, np.float64)
        b.seg_sf = _ptr(getattr(d, "seg_sf", None), np.float64)
        b.seg_ef = _ptr(getattr(d, "seg_ef", None), np.float64)
        b.seg_spos = _ptr(getattr(d, "seg_spos", None), np.float64)
        b.seg_epos = _ptr(getattr(d, "seg_epos", None), np.float64)
        b.seg_sdepth = _ptr(getattr(d, "seg_sdepth", None), np.float64)
        b.seg_edepth = _ptr(getattr(d, "seg_edepth", None), np.float64)
        b.seg_length = _ptr(d.seg_length, np.float64)
        b.seg_valid = _ptr(d.seg_valid, np.uint8)
    return b, keep


class AlignOut:
    """Owns the output arrays of one alignment batch and the plsvo_align_result pointing at them."""

    def __init__(self, batch: int, n_segs: int):
        self.T_cur_w = np.zeros((batch, 7))
        self.n_tracked = np.zeros(batch, np.int64)
        self.H = np.zeros((batch, 36))
        self.seg_killed = np.zeros((batch, max(n_segs, 1)), np.uint8)
        self.iters = np.zeros((batch, MAX_LEVELS), np.int32)
        self.status = np.zeros(batch, np.int32)
        self.patch_iters = np.zeros(batch, np.uint32)
        self.patch_levels = np.zeros(batch, np.uint32)
        r = AlignResult()
        r.T_cur_w = _ptr(self.T_cur_w, np.float64)
        r.n_tracked = _ptr(self.n_tracked, np.int64)
        r.H = _ptr(self.H, np.float64)
        r.seg_killed = _ptr(self.seg_killed, np.uint8) if n_segs > 0 else _u8p()
        r.iters = _ptr(self.iters, np.int32)
        r.status = _ptr(self.status, np.int32)
        r.patch_iters = _ptr(self.patch_iters, np.uint32)
        r.patch_levels = _ptr(self.patch_levels, np.uint32)
        self.struct = r
        if n_segs == 0:
            self.seg_killed = self.seg_killed[:, :0]


def make_poseopt_batch(d):
    b = PoseOptBatch()
    b.batch, b.n_pts, b.n_segs = d.batch, d.n_pts, d.n_segs
    b.fx = d.fx
    b.T_f_w = _ptr(d.T_f_w, np.float64)
    b.pt_count = _ptr(d.pt_count, np.int32)
    b.pt_f = _ptr(getattr(d, "pt_f", None), np.float64)
    b.pt_pos = _ptr(d.pt_pos, np.float64)
    b.pt_level = _ptr(d.pt_level, np.int32)
    b.pt_valid = _ptr(d.pt_valid, np.uint8)
    b.seg_count = _ptr(d.seg_count, np.int32)
    if d.n_segs > 0:
        b.seg_line = _ptr(d.seg_line, np.float64)
        b.seg_spos = _ptr(getattr(d, "seg_spos", None), np.float64)
        b.seg_epos = _ptr(getattr(d, "seg_epos", None), np.float64)
        b.seg_sdepth = _ptr(getattr(d, "seg_sdepth", None), np.float64)
        b.seg_edepth = _ptr(getattr(d, "seg_edepth", None), np.float64)
        b.seg_level = _ptr(d.seg_level, np.int32)
        b.seg_valid = _ptr(d.seg_valid, np.uint8)
    return b, [d]


class PoseOptOut:
    def __init__(self, batch: int, n_pts: int, n_segs: int):
        self.T_f_w = np.zeros((batch, 7))
        self.cov = np.zeros((batch, 36))
        self.estimated_scale = np.zeros(batch)
        self.error_init = np.zeros(batch)
        self.error_final = np.zeros(batch)
        self.num_obs_pt = np.zeros(batch, np.int64)
        self.num_obs_ls = np.zeros(batch, np.int64)
        self.pt_outlier = np.zeros((batch, max(n_pts, 1)), np.uint8)
        self.seg_outlier = np.zeros((batch, max(n_segs, 1)), np.uint8)
        self.iters = np.zeros((batch, 2), np.int32)
        self.status = np.zeros(batch, np.int32)
        r = PoseOptResult()
        r.T_f_w = _ptr(self.T_f_w, np.float64)
        r.cov = _ptr(self.cov, np.float64)
        r.estimated_scale = _ptr(self.estimated_scale, np.float64)
        r.error_init = _ptr(self.error_init, np.float64)
        r.error_final = _ptr(self.error_final, np.float64)
        r.num_obs_pt = _ptr(self.num_obs_pt, np.int64)
        r.num_obs_ls = _ptr(self.num_obs_ls, np.int64)
        r.pt_outlier = _ptr(self.pt_outlier, np.uint8)
        r.seg_outlier = _ptr(self.seg_outlier, np.uint8) if n_segs > 0 else _u8p()
        r.iters = _ptr(self.iters, np.int32)
        r.status = _ptr(self.status, np.int32)
        self.struct = r
        if n_segs == 0:
            self.seg_outlier = self.seg_outlier[:, :0]


# ------------------------------------------------------------------------------------------------
# library loading
# ------------------------------------------------------------------------------------------------

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libplsvo_b200.so")

# every symbol include/plsvo_b200.h declares: (name, restype, argtypes)
_P = C.POINTER
ABI_SYMBOLS = [
    ("plsvo_ctx_create", C.c_int, [C.c_int, C.c_void_p, _P(C.c_void_p)]),
    ("plsvo_ctx_destroy", None, [C.c_void_p]),
    ("plsvo_last_error", C.c_char_p, [C.c_void_p]),
    ("plsvo_ctx_stream", C.c_void_p, [C.c_void_p]),
    ("plsvo_sync", C.c_int, [C.c_void_p]),
    ("plsvo_host_alloc", C.c_int, [_P(C.c_void_p), C.c_size_t]),
    ("plsvo_host_free", C.c_int, [C.c_void_p]),
    ("plsvo_align_upload", C.c_int, [C.c_void_p, _P(AlignBatch)]),
    ("plsvo_align_launch", C.c_int, [C.c_void_p, _P(AlignParams)]),
    ("plsvo_align_download", C.c_int, [C.c_void_p, _P(AlignResult)]),
    ("plsvo_align_batch_run", C.c_int, [C.c_void_p, _P(AlignBatch), _P(AlignParams), _P(AlignResult)]),
    ("plsvo_poseopt_upload", C.c_int, [C.c_void_p, _P(PoseOptBatch)]),
    ("plsvo_poseopt_launch", C.c_int, [C.c_void_p, _P(PoseOptParams)]),
    ("plsvo_poseopt_download", C.c_int, [C.c_void_p, _P(PoseOptResult)]),
    ("plsvo_poseopt_batch_run", C.c_int, [C.c_void_p, _P(PoseOptBatch), _P(PoseOptParams), _P(PoseOptResult)]),
    ("plsvo_track_upload", C.c_int, [C.c_void_p, _P(AlignBatch), _P(PoseOptBatch)]),
    ("plsvo_track_launch", C.c_int, [C.c_void_p, _P(AlignParams), _P(PoseOptParams)]),
    ("plsvo_track_batch_run", C.c_int, [C.c_void_p, _P(AlignBatch), _P(AlignParams), _P(PoseOptBatch), _P(PoseOptParams),
                                        _P(AlignResult), _P(PoseOptResult)]),
    ("plsvo_pyramid_batch_run", C.c_int, [C.c_void_p, _P(PyramidBatch), _P(PyramidResult)]),
    ("plsvo_undistort_batch_run", C.c_int, [C.c_void_p, _P(UndistortBatch), _P(PyramidResult)]),
    ("plsvo_last_map_build_ms", C.c_int, [C.c_void_p, _P(C.c_float)]),
    ("plsvo_align_raw_batch_run", C.c_int, [C.c_void_p, _P(RawFrames), _P(AlignBatch), _P(AlignParams), _P(AlignResult),
                                            _P(PyramidResult)]),
    ("plsvo_track_raw_batch_run", C.c_int, [C.c_void_p, _P(RawFrames), _P(AlignBatch), _P(AlignParams), _P(PoseOptBatch),
                                            _P(PoseOptParams), _P(AlignResult), _P(PoseOptResult), _P(PyramidResult)]),
    ("plsvo_align2d_batch_run", C.c_int, [C.c_void_p, _P(Align2DBatch), _P(Align2DResult)]),
    ("plsvo_align1d_batch_run", C.c_int, [C.c_void_p, _P(Align1DBatch), _P(Align1DResult)]),
    ("plsvo_match_direct_batch_run", C.c_int, [C.c_void_p, _P(MatchBatch), _P(MatchResult)]),
    ("plsvo_seed_update_batch_run", C.c_int, [C.c_void_p, _P(SeedBatch), _P(SeedResult)]),
    ("plsvo_line_seed_update_batch_run", C.c_int, [C.c_void_p, _P(LineSeedBatch), _P(LineSeedResult)]),
    ("plsvo_structopt_batch_run", C.c_int, [C.c_void_p, _P(StructOptBatch), _P(StructOptResult)]),
    ("plsvo_last_kernel_ms", C.c_int, [C.c_void_p, _P(C.c_float)]),
    ("plsvo_launch_count", C.c_int64, [C.c_void_p]),
    ("plsvo_selftest_weight", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, _P(C.c_uint64)]),
    ("plsvo_version", C.c_char_p, []),
]

_lib = None


def load_library(path: str | None = None):
    """dlopen libplsvo_b200.so and type every ABI symbol.  Raises if the library is missing."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or os.environ.get("PLSVO_LIB") or LIB_PATH
    if not os.path.exists(p):
        raise RuntimeError(
            f"{p} not found: the CUDA extension has not been built (run `python __graft_entry__.py build`). "
            "There is no CPU fallback for the PL-SVO hot path."
        )
    lib = C.CDLL(p)
    for name, res, args in ABI_SYMBOLS:
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if path is None:
        _lib = lib
    return lib


def make_align2d_batch(pyr, image_index, level, border, ref, px, n_iter, width, height):
    """pyr: {level: u8 [n_images,h,w]}; border u8 [n,10,10]; ref u8 [n,8,8]; px f64 [n,2]."""
    b = Align2DBatch()
    keep = [pyr, image_index, level, border, ref, px]
    b.n_features, b.n_iter = len(image_index), n_iter
    b.width, b.height = width, height
    for l, im in pyr.items():
        assert im.dtype == np.uint8 and im.ndim == 3 and im.strides[2] == 1
        b.n_images = im.shape[0]
        b.img[l] = im.ctypes.data_as(_u8p)
        b.img_pitch[l] = im.strides[1]
        b.img_stride[l] = im.strides[0]
    b.image_index = _ptr(image_index, np.int32)
    b.level = _ptr(level, np.int32)
    b.ref_patch_with_border = _ptr(border.reshape(len(image_index), -1), np.uint8)
    b.ref_patch = _ptr(ref.reshape(len(image_index), -1), np.uint8)
    b.px = _ptr(px, np.float64)
    return b, keep


def make_match_batch(d):
    """Build a plsvo_match_batch from a synth.MatchData-like object.  Returns (struct, keepalive)."""
    b = MatchBatch()
    b.n_features, b.n_ref_images, b.n_cur_images = d.n, d.T_ref_w.shape[0], d.T_cur_w.shape[0]
    b.n_pyr_levels, b.n_iter = d.n_pyr_levels, d.n_iter
    b.cam = Camera(d.cam.width, d.cam.height, 0, 0, d.cam.fx, d.cam.fy, d.cam.cx, d.cam.cy)
    for pyr, img, pitch, stride in ((d.ref_pyr, b.ref_img, b.ref_pitch, b.ref_stride), (d.cur_pyr, b.cur_img, b.cur_pitch, b.cur_stride)):
        for l, im in pyr.items():  # any u8 [n,h,w] view with unit column stride (padded rows, every other frame, ...)
            if not isinstance(im, np.ndarray) or im.dtype != np.uint8 or im.ndim != 3 or im.strides[2] != 1 or min(im.strides) < 0:
                raise TypeError(f"pyramid level {l}: expected a u8 [n,h,w] array with unit column stride")
            img[l] = im.ctypes.data_as(_u8p)
            pitch[l], stride[l] = im.strides[1], im.strides[0]
    b.T_ref_w, b.T_cur_w = _ptr(d.T_ref_w, np.float64), _ptr(d.T_cur_w, np.float64)
    b.ref_index, b.cur_index = _ptr(d.ref_index, np.int32), _ptr(d.cur_index, np.int32)
    b.ref_px, b.ref_f, b.ref_level = _ptr(d.ref_px, np.float64), _ptr(d.ref_f, np.float64), _ptr(d.ref_level, np.int32)
    b.is_edgelet, b.ref_grad = _ptr(d.is_edgelet, np.uint8), _ptr(d.ref_grad, np.float64)
    b.pos, b.px_cur = _ptr(d.pos, np.float64), _ptr(d.px_cur, np.float64)
    return b, [d]


class MatchOut:
    """Owns the output arrays of one findMatchDirect batch and the plsvo_match_result pointing at them."""

    def __init__(self, n: int):
        self.px_cur = np.zeros((n, 2))
        self.success = np.zeros(n, np.uint8)
        self.search_level = np.zeros(n, np.int32)
        self.A_cur_ref = np.full((n, 4), np.nan)  # Matcher::A_cur_ref_ row-major; NaN where the in-frame test fails
        self.struct = MatchResult(_ptr(self.px_cur, np.float64), _ptr(self.success, np.uint8), _ptr(self.search_level, np.int32),
                                  _ptr(self.A_cur_ref, np.float64))


def make_structopt_batch(d):
    """Build a plsvo_structopt_batch from a synth.StructOptData-like object.  Returns (struct, keepalive)."""
    b = StructOptBatch()
    b.n_points, b.n_segs, b.n_frames = d.pt_pos.shape[0], d.seg_spos.shape[0], d.T_f_w.shape[0]
    b.n_iter_pts, b.n_iter_segs = d.n_iter_pts, d.n_iter_segs
    b.T_f_w = _ptr(d.T_f_w, np.float64)
    b.pt_obs_begin, b.pt_obs_frame = _ptr(d.pt_obs_begin, np.int32), _ptr(d.pt_obs_frame, np.int32)
    b.pt_obs_f, b.pt_pos = _ptr(d.pt_obs_f, np.float64), _ptr(d.pt_pos, np.float64)
    b.seg_obs_begin, b.seg_obs_frame = _ptr(d.seg_obs_begin, np.int32), _ptr(d.seg_obs_frame, np.int32)
    b.seg_obs_sf, b.seg_obs_ef = _ptr(d.seg_obs_sf, np.float64), _ptr(d.seg_obs_ef, np.float64)
    b.seg_spos, b.seg_epos = _ptr(d.seg_spos, np.float64), _ptr(d.seg_epos, np.float64)
    return b, [d]


class StructOptOut:
    def __init__(self, n_points: int, n_segs: int):
        self.pt_pos = np.zeros((n_points, 3))
        self.seg_spos = np.zeros((n_segs, 3))
        self.seg_epos = np.zeros((n_segs, 3))
        self.pt_iters = np.zeros(n_points, np.int32)
        self.seg_iters = np.zeros(n_segs, np.int32)
        self.struct = StructOptResult(_ptr(self.pt_pos, np.float64), _ptr(self.seg_spos, np.float64), _ptr(self.seg_epos, np.float64),
                                      _ptr(self.pt_iters, np.int32), _ptr(self.seg_iters, np.int32))


def make_seed_batch(d):
    """Build a plsvo_seed_batch from a synth.SeedData-like object.  Returns (struct, keepalive)."""
    b = SeedBatch()
    b.n_seeds, b.n_ref_images, b.n_cur_images = d.n, d.T_ref_w.shape[0], d.T_cur_w.shape[0]
    b.n_pyr_levels, b.n_iter, b.max_epi_search_steps = d.n_pyr_levels, d.n_iter, d.max_epi_search_steps
    b.align_1d, b.subpix_refinement, b.epi_search_edgelet_filtering = int(d.align_1d), int(d.subpix_refinement), int(d.edgelet_filtering)
    b.epi_search_edgelet_max_angle, b.seed_convergence_sigma2_thresh = d.edgelet_max_angle, d.convergence_thresh
    b.cam = Camera(d.cam.width, d.cam.height, 0, 0, d.cam.fx, d.cam.fy, d.cam.cx, d.cam.cy)
    for l, im in d.ref_pyr.items():
        b.ref_img[l] = _ptr(im, np.uint8)
        b.ref_pitch[l], b.ref_stride[l] = im.strides[1], im.strides[0]
    for l, im in d.cur_pyr.items():
        b.cur_img[l] = _ptr(im, np.uint8)
        b.cur_pitch[l], b.cur_stride[l] = im.strides[1], im.strides[0]
    b.T_ref_w, b.T_cur_w = _ptr(d.T_ref_w, np.float64), _ptr(d.T_cur_w, np.float64)
    b.ref_index, b.cur_index = _ptr(d.ref_index, np.int32), _ptr(d.cur_index, np.int32)
    b.ref_px, b.ref_f, b.ref_level = _ptr(d.ref_px, np.float64), _ptr(d.ref_f, np.float64), _ptr(d.ref_level, np.int32)
    b.is_edgelet, b.ref_grad = _ptr(d.is_edgelet, np.uint8), _ptr(d.ref_grad, np.float64)
    b.a, b.b, b.mu = _ptr(d.a, np.float32), _ptr(d.b, np.float32), _ptr(d.mu, np.float32)
    b.z_range, b.sigma2 = _ptr(d.z_range, np.float32), _ptr(d.sigma2, np.float32)
    return b, [d]


class SeedOut:
    """Owns the output arrays of one seed-update batch and the plsvo_seed_result pointing at them."""

    def __init__(self, n: int):
        self.a, self.b = np.zeros(n, np.float32), np.zeros(n, np.float32)
        self.mu, self.sigma2 = np.zeros(n, np.float32), np.zeros(n, np.float32)
        self.status = np.zeros(n, np.int32)
        self.converged = np.zeros(n, np.uint8)
        self.depth = np.zeros(n)
        self.px_cur = np.zeros((n, 2))
        self.struct = SeedResult(_ptr(self.a, np.float32), _ptr(self.b, np.float32), _ptr(self.mu, np.float32), _ptr(self.sigma2, np.float32),
                                 _ptr(self.status, np.int32), _ptr(self.converged, np.uint8), _ptr(self.depth, np.float64),
                                 _ptr(self.px_cur, np.float64))


def make_line_seed_batch(d):
    """Build a plsvo_line_seed_batch from a synth.LineSeedData-like object (a SeedData for the start point plus the
    end-point fields).  Returns (struct, keepalive)."""
    base, keep = make_seed_batch(d)
    b = LineSeedBatch()
    b.seeds = base
    b.ref_sf, b.ref_ef = _ptr(d.ref_sf, np.float64), _ptr(d.ref_ef, np.float64)
    b.mu_e, b.z_range_e, b.sigma2_e = _ptr(d.mu_e, np.float32), _ptr(d.z_range_e, np.float32), _ptr(d.sigma2_e, np.float32)
    return b, keep


class LineSeedOut(SeedOut):
    def __init__(self, n: int):
        super().__init__(n)
        self.mu_e, self.sigma2_e = np.zeros(n, np.float32), np.zeros(n, np.float32)
        self.depth_e = np.zeros(n)
        self.px_cur_e = np.zeros((n, 2))  # Matcher::px_cur_ of the end-point search
        self.line_struct = LineSeedResult(self.struct, _ptr(self.mu_e, np.float32), _ptr(self.sigma2_e, np.float32),
                                          _ptr(self.depth_e, np.float64), _ptr(self.px_cur_e, np.float64))
