"""Host-side mirror of the reference's interface for the hot path, over the C ABI.

The reference's boundary is two C++ symbols (SURVEY.md §8b):

    plsvo::SparseImgAlign(max_level, min_level, n_iter, method, display, verbose).run(ref, cur)
        include/plsvo/sparse_img_align.h:56-70, src/sparse_img_align.cpp:40-95
    plsvo::pose_optimizer::optimizeGaussNewton(reproj_thresh, n_iter[, n_iter_ref], verbose, frame, ...)
        include/plsvo/pose_optimizer.h:47-64

This module keeps the same names and argument meaning for *batches* of frame pairs / frames held
in flat arrays (synth.AlignData / synth.PoseOptData).  The C++ shim that keeps the exact
FramePtr signatures lives in pl-svo_b200/host/.  All compute happens in libplsvo_b200.so on
the GPU; nothing here falls back to the CPU.
"""
from __future__ import annotations

import ctypes as C

from . import abi


class PlsvoError(RuntimeError):
    pass


class Context:
    """A device context (plsvo_ctx): one CUDA device + stream + reusable device buffers."""

    def __init__(self, device: int = 0, stream: int | None = None):
        self.lib = abi.load_library()
        h = C.c_void_p()
        rc = self.lib.plsvo_ctx_create(device, C.c_void_p(stream or 0), C.byref(h))
        if rc != abi.OK:
            msg = self.lib.plsvo_last_error(None)
            raise PlsvoError(f"plsvo_ctx_create failed rc={rc}: {msg.decode() if msg else ''}")
        self.handle = h

    def check(self, rc: int, what: str):
        if rc != abi.OK:
            msg = self.lib.plsvo_last_error(self.handle)
            raise PlsvoError(f"{what} failed rc={rc}: {msg.decode() if msg else ''}")

    @property
    def stream(self) -> int:
        return int(self.lib.plsvo_ctx_stream(self.handle) or 0)

    def sync(self):
        self.check(self.lib.plsvo_sync(self.handle), "plsvo_sync")

    def last_kernel_ms(self) -> float:
        """Device time of the kernel of the last pyramid / align2D / align1D call (plsvo_last_kernel_ms)."""
        ms = C.c_float(0)
        self.check(self.lib.plsvo_last_kernel_ms(self.handle, C.byref(ms)), "plsvo_last_kernel_ms")
        return float(ms.value)

    def last_map_build_ms(self) -> float | None:
        """Device time of the map build made by the last PinholeCamera.undistortImage call on this context, or None when
        that call reused the cached map or needed none (plsvo_last_map_build_ms)."""
        ms = C.c_float(0)
        self.check(self.lib.plsvo_last_map_build_ms(self.handle, C.byref(ms)), "plsvo_last_map_build_ms")
        return None if ms.value < 0 else float(ms.value)

    def launch_count(self) -> int:
        return int(self.lib.plsvo_launch_count(self.handle))

    def close(self):
        if getattr(self, "handle", None):
            self.lib.plsvo_ctx_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_ctx: Context | None = None


def default_context() -> Context:
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(0)
    return _default_ctx


class SparseImgAlign:
    """Batched counterpart of plsvo::SparseImgAlign (src/sparse_img_align.cpp:40-52)."""

    GaussNewton = 0
    LevenbergMarquardt = 1  # accepted for signature parity; the reference only ever passes GaussNewton

    def __init__(self, max_level: int, min_level: int, n_iter: int, method: int = 0,
                 display: bool = False, verbose: bool = False, ctx: Context | None = None, eps: float = 1e-6):
        if method != self.GaussNewton:
            raise PlsvoError("only Method::GaussNewton is on the hot path (frame_handler_mono.cpp:272-273)")
        self.params = abi.align_params(max_level, min_level, n_iter, eps)
        self.ctx = ctx or default_context()
        self.last = None

    # three-leg form (device-resident between legs)
    def upload(self, data):
        batch, self._keep = abi.make_align_batch(data)
        self._shape = (data.batch, data.n_segs)
        self.ctx.check(self.ctx.lib.plsvo_align_upload(self.ctx.handle, C.byref(batch)), "plsvo_align_upload")

    def launch(self):
        self.ctx.check(self.ctx.lib.plsvo_align_launch(self.ctx.handle, C.byref(self.params)), "plsvo_align_launch")

    def download(self) -> abi.AlignOut:
        out = abi.AlignOut(*self._shape)
        self.ctx.check(self.ctx.lib.plsvo_align_download(self.ctx.handle, C.byref(out.struct)), "plsvo_align_download")
        self.last = out
        return out

    def run(self, data, camera: "ATANCamera | None" = None, cameras=None, sizes=None, cam_of_pair=None) -> abi.AlignOut:
        """run(ref_frames, cur_frames) for a whole batch: returns poses, n_tracked (the reference's
        return value, sparse_img_align.cpp:94), H, killed-segment flags.  camera: an ATANCamera when the frames come from
        one (plsvo_align_atan_batch_run; data.cam then only gives the image size); None for the undistorted pinhole
        data.cam.  cameras: array-like [B, 4] of undistorted pinhole (fx, fy, cx, cy), one row per pair, when the pairs
        come from differently calibrated cameras (plsvo_align_multicam_batch_run).  sizes: with cameras, array-like
        [B, 2] of every pair's (width, height) when the pairs' frames differ in size: data.cam's size is then the slot
        each pair's frames sit in, top-left (synth.merge_sizes builds such a batch); data.cam's size for every pair
        when None.  cam_of_pair: [B] indices into `camera`, then a sequence of ATANCamera, when the pairs come from
        differently calibrated ATAN cameras (plsvo_align_atan_multicam_batch_run): pair b is aligned with
        camera[cam_of_pair[b]], its frames that camera's size in the top-left corner of data.cam's slot.  A sequence
        that also holds undistorted pinhole cameras (synth.Camera) aligns pinhole and ATAN pairs in one call
        (plsvo_align_any_camera_batch_run), each pair with its own camera's model."""
        any_cams = _any_cameras_arg(camera, cameras, sizes, cam_of_pair, data)
        atan_cams = None if any_cams else _atan_cameras_arg(camera, cameras, sizes, cam_of_pair, data)
        batch, keep = abi.make_align_batch(data)
        out = abi.AlignOut(data.batch, data.n_segs)
        if any_cams:
            cams, n_cams, cop = any_cams
            self.ctx.check(self.ctx.lib.plsvo_align_any_camera_batch_run(self.ctx.handle, cams, n_cams,
                                                                         cop.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(batch),
                                                                         C.byref(self.params), C.byref(out.struct)),
                           "plsvo_align_any_camera_batch_run")
            self.last = out
            return out
        if atan_cams is not None:
            self.ctx.check(self.ctx.lib.plsvo_align_atan_multicam_batch_run(self.ctx.handle, atan_cams, C.byref(batch),
                                                                            C.byref(self.params), C.byref(out.struct)),
                           "plsvo_align_atan_multicam_batch_run")
            self.last = out
            return out
        if cameras is not None:
            cams = _cameras_arg(cameras, data, sizes)
            self.ctx.check(self.ctx.lib.plsvo_align_multicam_batch_run(self.ctx.handle, cams, C.byref(batch),
                                                                       C.byref(self.params), C.byref(out.struct)),
                           "plsvo_align_multicam_batch_run")
            self.last = out
            return out
        if camera is not None:
            camera._check(data)
            self.ctx.check(self.ctx.lib.plsvo_align_atan_batch_run(self.ctx.handle, C.byref(camera.struct), C.byref(batch),
                                                                   C.byref(self.params), C.byref(out.struct)),
                           "plsvo_align_atan_batch_run")
            self.last = out
            return out
        self.ctx.check(
            self.ctx.lib.plsvo_align_batch_run(self.ctx.handle, C.byref(batch), C.byref(self.params), C.byref(out.struct)),
            "plsvo_align_batch_run",
        )
        self.last = out
        return out

    def run_raw(self, camera: "PinholeCamera", raw, data, rect_levels=None, cam_of_pair=None):
        """run() on raw (distorted) frames: each frame is rectified with `camera` (PinholeCamera.undistortImage) and
        half-sampled on the device, and the pyramid never leaves it.  raw: a [B+1,H,W] frame chain, or a (ref, cur) pair
        of [B,H,W] stacks; rows may be padded.  data describes features, poses and the undistorted camera as for run()
        (its images are ignored).  Results are byte-identical to undistortImage followed by the plain host-buffer run().
        rect_levels: levels to bring back as well; returns (AlignOut, {level: [n_frames, H>>l, W>>l]}) then, the frames
        in stack order (the chain, or the reference frames followed by the current ones).
        cam_of_pair: [B] indices into `camera`, then a sequence of PinholeCamera, when the pairs come from differently
        calibrated lenses (plsvo_align_raw_multicam_batch_run): pair b is rectified with camera[cam_of_pair[b]] and
        aligned with its fx, fy, cx, cy.  data.cam gives only the image size of the slot every frame sits in; a camera
        may be smaller, and its frames then occupy its own size in the top-left corner of their slots (of the raw
        stacks and of the rect_levels arrays, whose rest is 0).  raw must then be a (ref, cur) pair of stacks.  A
        sequence that also holds ATANCamera entries aligns lens and ATAN pairs in one call
        (plsvo_align_raw_any_camera_batch_run): an ATAN pair's frames are not rectified but half-sampled as they are
        and aligned through the ATAN model; its rect_levels entries are that pyramid."""
        any_camera = _raw_any_camera(camera, cam_of_pair)
        rf, batch, keep = (_raw_any_camera_args if any_camera else _raw_call_args)(camera, raw, data, cam_of_pair)
        levels, r = _rect_outputs(camera if cam_of_pair is None else data.cam, rf, data.batch, rect_levels)
        out = abi.AlignOut(data.batch, data.n_segs)
        fn, name = ((self.ctx.lib.plsvo_align_raw_batch_run, "plsvo_align_raw_batch_run") if cam_of_pair is None else
                    (self.ctx.lib.plsvo_align_raw_any_camera_batch_run, "plsvo_align_raw_any_camera_batch_run") if any_camera else
                    (self.ctx.lib.plsvo_align_raw_multicam_batch_run, "plsvo_align_raw_multicam_batch_run"))
        self.ctx.check(fn(self.ctx.handle, C.byref(rf), C.byref(batch), C.byref(self.params), C.byref(out.struct),
                          C.byref(r) if r is not None else None), name)
        self.last = out
        return out if rect_levels is None else (out, levels)

    def getFisherInformation(self):
        """H_ / (5e-4 * 255^2), sparse_img_align.cpp:97-102 (per pair)."""
        if self.last is None:
            raise PlsvoError("run() has not been called")
        return self.last.H.reshape(-1, 6, 6) / (5e-4 * 255 * 255)


class pose_optimizer:
    """Namespace mirror of plsvo::pose_optimizer (include/plsvo/pose_optimizer.h:47-64)."""

    @staticmethod
    def optimizeGaussNewton(reproj_thresh: float, n_iter: int, verbose: bool, data, n_iter_ref: int | None = None,
                            ctx: Context | None = None, fx=None) -> abi.PoseOptOut:
        """9-argument overload when n_iter_ref is None, 10-argument overload otherwise.  fx: array-like [B] of the
        frames' errorMultiplier2 when they differ (plsvo_poseopt_multicam_batch_run); data.fx is then not used."""
        ctx = ctx or default_context()
        params = abi.poseopt_params(reproj_thresh, n_iter, -1 if n_iter_ref is None else n_iter_ref)
        batch, keep = abi.make_poseopt_batch(data)
        out = abi.PoseOptOut(data.batch, data.n_pts, data.n_segs)
        if fx is not None:
            fxa = _frame_fx_arg(fx, data.batch)
            ctx.check(ctx.lib.plsvo_poseopt_multicam_batch_run(ctx.handle, abi._ptr(fxa, fxa.dtype), C.byref(batch),
                                                               C.byref(params), C.byref(out.struct)),
                      "plsvo_poseopt_multicam_batch_run")
            return out
        ctx.check(
            ctx.lib.plsvo_poseopt_batch_run(ctx.handle, C.byref(batch), C.byref(params), C.byref(out.struct)),
            "plsvo_poseopt_batch_run",
        )
        return out


def track(align_data, poseopt_data, max_level: int = 4, min_level: int = 2, n_iter: int = 30, reproj_thresh: float = 2.0,
          po_n_iter: int = 10, po_n_iter_ref: int | None = None, chained: bool = True, ctx: Context | None = None,
          camera: "ATANCamera | None" = None, cameras=None, sizes=None, cam_of_pair=None):
    """FrameHandlerMono::processFrame's two hot-path calls back to back (src/frame_handler_mono.cpp:272-274, :327-329):
    SparseImgAlign::run on every pair, then pose_optimizer::optimizeGaussNewton on every frame, the pose staying on the
    device in between (chained=True: the pose optimiser starts from the aligned pose of the same batch index).
    camera: an ATANCamera when the frames come from one (plsvo_track_atan_batch_run); poseopt_data.fx is then its
    errorMultiplier2().  cameras: array-like [B, 4] of per-pair undistorted pinhole (fx, fy, cx, cy)
    (plsvo_track_multicam_batch_run); frame b's errorMultiplier2 is then |cameras[b, 0]| and poseopt_data.fx is not used.
    sizes: with cameras, [B, 2] of every pair's (width, height), as for SparseImgAlign.run.
    cam_of_pair: with a sequence of ATANCamera as `camera`, as for SparseImgAlign.run
    (plsvo_track_atan_multicam_batch_run); frame b's errorMultiplier2 is then its camera's fx_ and poseopt_data.fx is
    not used.  With pinhole cameras (synth.Camera) in the sequence too (plsvo_track_any_camera_batch_run), frame b's
    errorMultiplier2 is |fx| of a pinhole camera and fx_ of an ATAN camera.
    Returns (AlignOut, PoseOptOut)."""
    any_cams = _any_cameras_arg(camera, cameras, sizes, cam_of_pair, align_data)
    atan_cams = None if any_cams else _atan_cameras_arg(camera, cameras, sizes, cam_of_pair, align_data)
    ctx = ctx or default_context()
    ap = abi.align_params(max_level, min_level, n_iter)
    pp = abi.poseopt_params(reproj_thresh, po_n_iter, -1 if po_n_iter_ref is None else po_n_iter_ref)
    ab, keep_a = abi.make_align_batch(align_data)
    pb, keep_p = abi.make_poseopt_batch(poseopt_data)
    if chained:
        pb.T_f_w = abi._f64p()
    ao = abi.AlignOut(align_data.batch, align_data.n_segs)
    po = abi.PoseOptOut(poseopt_data.batch, poseopt_data.n_pts, poseopt_data.n_segs)
    if any_cams:
        cams, n_cams, cop = any_cams
        ctx.check(ctx.lib.plsvo_track_any_camera_batch_run(ctx.handle, cams, n_cams, cop.ctypes.data_as(C.POINTER(C.c_int32)),
                                                           C.byref(ab), C.byref(ap), C.byref(pb), C.byref(pp),
                                                           C.byref(ao.struct), C.byref(po.struct)),
                  "plsvo_track_any_camera_batch_run")
        return ao, po
    if atan_cams is not None:
        ctx.check(ctx.lib.plsvo_track_atan_multicam_batch_run(ctx.handle, atan_cams, C.byref(ab), C.byref(ap), C.byref(pb),
                                                              C.byref(pp), C.byref(ao.struct), C.byref(po.struct)),
                  "plsvo_track_atan_multicam_batch_run")
        return ao, po
    if cameras is not None:
        cams = _cameras_arg(cameras, align_data, sizes)
        ctx.check(ctx.lib.plsvo_track_multicam_batch_run(ctx.handle, cams, C.byref(ab), C.byref(ap), C.byref(pb), C.byref(pp),
                                                         C.byref(ao.struct), C.byref(po.struct)),
                  "plsvo_track_multicam_batch_run")
        return ao, po
    if camera is not None:
        camera._check(align_data)
        ctx.check(ctx.lib.plsvo_track_atan_batch_run(ctx.handle, C.byref(camera.struct), C.byref(ab), C.byref(ap), C.byref(pb),
                                                     C.byref(pp), C.byref(ao.struct), C.byref(po.struct)),
                  "plsvo_track_atan_batch_run")
        return ao, po
    ctx.check(ctx.lib.plsvo_track_batch_run(ctx.handle, C.byref(ab), C.byref(ap), C.byref(pb), C.byref(pp), C.byref(ao.struct),
                                            C.byref(po.struct)), "plsvo_track_batch_run")
    return ao, po


def _one_camera_model(camera, cameras, sizes=None):
    if camera is not None and cameras is not None:
        raise PlsvoError("pass camera= (one ATAN camera) or cameras= (pinhole intrinsics per pair), not both")
    if sizes is not None and cameras is None:
        raise PlsvoError("sizes= needs cameras= (the pinhole intrinsics of every pair)")


def _atan_cameras_arg(camera, cameras, sizes, cam_of_pair, data):
    """plsvo_atan_camera[B] of the ATAN multicam calls when `camera` is a sequence of ATANCamera indexed by cam_of_pair;
    None for the other camera arguments, which _one_camera_model checks."""
    if cam_of_pair is None:
        _one_camera_model(camera, cameras, sizes)
        if isinstance(camera, (list, tuple)):
            raise PlsvoError("camera= is one ATANCamera; a sequence of them needs cam_of_pair=")
        return None
    if cameras is not None or sizes is not None:
        raise PlsvoError("cam_of_pair= selects ATAN cameras per pair: pass no cameras= or sizes= with it")
    if isinstance(camera, ATANCamera) or not isinstance(camera, (list, tuple)) or not all(isinstance(c, ATANCamera) for c in camera):
        raise PlsvoError("with cam_of_pair, camera must be a sequence of ATANCamera")
    try:
        return abi.make_atan_cameras([c.struct for c in camera], cam_of_pair, data.batch)
    except ValueError as e:
        raise PlsvoError(str(e)) from None


def _any_cameras_arg(camera, cameras, sizes, cam_of_pair, data):
    """(plsvo_match_camera[K], K, cam_of_pair as int32 [B]) of the any-camera calls when `camera` is a sequence of
    ATANCamera and undistorted pinhole cameras (synth.Camera) with at least one of the latter, indexed by cam_of_pair;
    None otherwise, for _atan_cameras_arg to handle (a sequence of ATANCamera only, or one holding anything else).  The
    values (index ranges, camera sizes and parameters) are the C ABI's to check."""
    import numpy as np

    from .synth import Camera as UndistortedPinhole

    if cam_of_pair is None or not isinstance(camera, (list, tuple)):
        return None
    if not any(isinstance(c, UndistortedPinhole) for c in camera):
        return None
    if not all(isinstance(c, (UndistortedPinhole, ATANCamera)) for c in camera):
        return None
    if cameras is not None or sizes is not None:
        raise PlsvoError("cam_of_pair= selects a camera per pair: pass no cameras= or sizes= with it")
    k = np.ascontiguousarray(cam_of_pair)
    if k.shape != (data.batch,) or not np.issubdtype(k.dtype, np.integer):
        raise PlsvoError(f"cam_of_pair must be integers of shape [{data.batch}], got {k.dtype} {list(k.shape)}")
    k = k.astype(np.int32)
    return abi.make_match_cameras(camera), len(camera), k


def _cameras_arg(cameras, data, sizes=None):
    """plsvo_camera[B] for the multicam calls: `cameras` [B, 4] rows (fx, fy, cx, cy), and `sizes` [B, 2] rows
    (width, height) or data.cam's image size."""
    import numpy as np

    k = np.asarray(cameras, dtype=np.float64)
    if k.shape != (data.batch, 4):
        raise PlsvoError(f"cameras must have shape [{data.batch}, 4] (fx, fy, cx, cy per pair), got {list(k.shape)}")
    try:
        return abi.make_cameras(k, data.cam, data.batch, sizes)
    except ValueError as e:
        raise PlsvoError(str(e)) from None


def _frame_fx_arg(fx, batch: int):
    import numpy as np

    fxa = np.ascontiguousarray(fx, dtype=np.float64)
    if fxa.shape != (batch,):
        raise PlsvoError(f"fx must have shape [{batch}] (errorMultiplier2 per frame), got {list(fxa.shape)}")
    return fxa


def _raw_call_args(camera, raw, align_data, cam_of_pair=None):
    """plsvo_raw_frames (plsvo_raw_multicam_frames when cam_of_pair is given, `camera` then a sequence of PinholeCamera)
    and an image-free plsvo_align_batch (flags from the layout of `raw`) for the raw-frame calls."""
    if cam_of_pair is None:
        rf, chain, keep_r = abi.make_raw_frames(camera.struct, raw, align_data.batch)
    else:
        try:
            structs = [c.struct for c in camera]
        except (TypeError, AttributeError):
            raise PlsvoError("with cam_of_pair, camera must be a sequence of PinholeCamera") from None
        try:
            rf, keep_r = abi.make_raw_multicam_frames(structs, cam_of_pair, raw, align_data.batch, slot=align_data.cam)
        except ValueError as e:
            raise PlsvoError(str(e)) from None
        chain = False
    batch, keep_a = _image_free_batch(align_data, chain)
    return rf, batch, (keep_r, keep_a)


def _image_free_batch(align_data, chain: bool):
    """plsvo_align_batch of the raw-frame calls: no image pointers (the images come from the raw frames)."""
    batch, keep_a = abi.make_align_batch(align_data)
    for l in range(abi.MAX_LEVELS):
        batch.ref_img[l] = batch.cur_img[l] = None
        batch.img_pitch[l] = batch.img_stride[l] = 0
    batch.flags = abi.ALIGN_FRAME_CHAIN if chain else 0
    return batch, keep_a


def _raw_any_camera(camera, cam_of_pair) -> bool:
    """A raw call with cam_of_pair whose camera sequence holds an ATANCamera: the raw any-camera calls.  A sequence of
    PinholeCamera only keeps the raw multicam calls."""
    return cam_of_pair is not None and isinstance(camera, (list, tuple)) and any(isinstance(c, ATANCamera) for c in camera)


def _raw_any_camera_args(camera, raw, align_data, cam_of_pair):
    """plsvo_raw_any_camera_frames and an image-free plsvo_align_batch for the raw any-camera calls: `camera` a sequence
    of PinholeCamera (distorted lenses) and ATANCamera, indexed by cam_of_pair."""
    if not all(isinstance(c, (PinholeCamera, ATANCamera)) for c in camera):
        raise PlsvoError("with cam_of_pair, camera must be a sequence of PinholeCamera and ATANCamera")
    try:
        rf, keep_r = abi.make_raw_any_camera_frames(abi.make_raw_cameras(camera), cam_of_pair, raw, align_data.batch,
                                                    slot=align_data.cam)
    except ValueError as e:
        raise PlsvoError(str(e)) from None
    batch, keep_a = _image_free_batch(align_data, False)
    return rf, batch, (keep_r, keep_a)


def _rect_outputs(camera, rf, B: int, rect_levels):
    """Host arrays for the rectified levels a raw-frame call brings back, and the plsvo_pyramid_result (or None)."""
    import numpy as np

    if rect_levels is None:
        return None, None
    n = B + 1 if not rf.cur_raw else 2 * B
    r = abi.PyramidResult()
    levels = {}
    for l in rect_levels:
        out = np.empty((n, camera.height >> l, camera.width >> l), np.uint8)
        levels[l] = out
        r.level[l] = out.ctypes.data_as(C.POINTER(C.c_uint8))
        r.pitch[l], r.stride[l] = out.strides[1], out.strides[0]
    return levels, r


def track_raw(camera, raw, align_data, poseopt_data, max_level: int = 4, min_level: int = 2, n_iter: int = 30,
              reproj_thresh: float = 2.0, po_n_iter: int = 10, po_n_iter_ref: int | None = None, chained: bool = True,
              ctx: Context | None = None, rect_levels=None, cam_of_pair=None):
    """track() on raw (distorted) frames, rectified with `camera` on the device (see SparseImgAlign.run_raw for `raw`,
    `rect_levels` and `cam_of_pair`; with cam_of_pair, frame b's errorMultiplier2 is |fx| of its camera and
    poseopt_data.fx is not used; fx_ for an ATANCamera in the sequence, plsvo_track_raw_any_camera_batch_run).
    Returns (AlignOut, PoseOptOut), plus the dict of rectified levels when rect_levels is given."""
    ctx = ctx or default_context()
    ap = abi.align_params(max_level, min_level, n_iter)
    pp = abi.poseopt_params(reproj_thresh, po_n_iter, -1 if po_n_iter_ref is None else po_n_iter_ref)
    any_camera = _raw_any_camera(camera, cam_of_pair)
    rf, ab, keep_a = (_raw_any_camera_args if any_camera else _raw_call_args)(camera, raw, align_data, cam_of_pair)
    pb, keep_p = abi.make_poseopt_batch(poseopt_data)
    if chained:
        pb.T_f_w = abi._f64p()
    levels, r = _rect_outputs(camera if cam_of_pair is None else align_data.cam, rf, align_data.batch, rect_levels)
    ao = abi.AlignOut(align_data.batch, align_data.n_segs)
    po = abi.PoseOptOut(poseopt_data.batch, poseopt_data.n_pts, poseopt_data.n_segs)
    fn, name = ((ctx.lib.plsvo_track_raw_batch_run, "plsvo_track_raw_batch_run") if cam_of_pair is None else
                (ctx.lib.plsvo_track_raw_any_camera_batch_run, "plsvo_track_raw_any_camera_batch_run") if any_camera else
                (ctx.lib.plsvo_track_raw_multicam_batch_run, "plsvo_track_raw_multicam_batch_run"))
    ctx.check(fn(ctx.handle, C.byref(rf), C.byref(ab), C.byref(ap), C.byref(pb), C.byref(pp), C.byref(ao.struct), C.byref(po.struct),
                 C.byref(r) if r is not None else None), name)
    return (ao, po) if rect_levels is None else (ao, po, levels)


def createImgPyramid(img_level_0, n_levels: int, ctx: Context | None = None):
    """Batched frame_utils::createImgPyramid (src/frame.cpp:171-180): u8 images [B,H,W] -> list of levels
    (level 0 is the input array itself), each the truncating 2x2 half-sample of the previous one."""
    import numpy as np

    ctx = ctx or default_context()
    img = np.ascontiguousarray(img_level_0, dtype=np.uint8)
    B, H, W = img.shape
    b = abi.PyramidBatch(B, W, H, n_levels, img.ctypes.data_as(C.POINTER(C.c_uint8)), img.strides[1], img.strides[0])
    r = abi.PyramidResult()
    levels = [img]
    for l in range(1, n_levels):
        out = np.empty((B, H >> l, W >> l), np.uint8)
        levels.append(out)
        r.level[l] = out.ctypes.data_as(C.POINTER(C.c_uint8))
        r.pitch[l] = out.strides[1]
        r.stride[l] = out.strides[0]
    ctx.check(ctx.lib.plsvo_pyramid_batch_run(ctx.handle, C.byref(b), C.byref(r)), "plsvo_pyramid_batch_run")
    return levels


class PinholeCamera:
    """vk::PinholeCamera(width, height, fx, fy, cx, cy, d0, d1, d2, d3, d4) (rpg_vikit pinhole_camera.cpp), for the one
    call the pipeline makes on every raw frame, undistortImage (app/run_pipeline.cpp:409-414)."""

    def __init__(self, width: int, height: int, fx: float, fy: float, cx: float, cy: float,
                 d0: float = 0.0, d1: float = 0.0, d2: float = 0.0, d3: float = 0.0, d4: float = 0.0):
        self.struct = abi.PinholeCamera(int(width), int(height), fx, fy, cx, cy, (C.c_double * 5)(d0, d1, d2, d3, d4))

    @property
    def width(self) -> int:
        return self.struct.width

    @property
    def height(self) -> int:
        return self.struct.height

    def undistortImage(self, raw, n_levels: int = 1, ctx: Context | None = None):
        """Batched undistortImage followed by frame_utils::createImgPyramid: u8 raw frames [B,H,W] (rows may be padded)
        -> list of n_levels arrays [B, H>>l, W>>l], level 0 the rectified frames, bit-identical to cv::remap with the
        camera's CV_16SC2 map.  The map is built on the device once per camera and context."""
        import numpy as np

        ctx = ctx or default_context()
        raw = np.asarray(raw)
        if raw.dtype != np.uint8 or raw.ndim != 3 or raw.strides[2] != 1:
            raise PlsvoError("undistortImage: raw frames must be u8 [B,H,W] with unit column stride")
        B, H, W = raw.shape
        if (W, H) != (self.width, self.height):
            raise PlsvoError(f"undistortImage: frames are {W}x{H}, the camera is {self.width}x{self.height}")
        b = abi.UndistortBatch(self.struct, B, n_levels, raw.ctypes.data_as(C.POINTER(C.c_uint8)), raw.strides[1], raw.strides[0])
        levels, r = abi.pyramid_levels(B, H, W, max(0, min(n_levels, abi.MAX_LEVELS)))
        ctx.check(ctx.lib.plsvo_undistort_batch_run(ctx.handle, C.byref(b), C.byref(r)), "plsvo_undistort_batch_run")
        return levels


class ATANCamera:
    """vk::ATANCamera(width, height, fx, fy, cx, cy, d0), the FOV model (fx..cy normalised by the image size), as
    app/run_pipeline.cpp builds it for cam_model ATAN.  Frames from it are aligned and tracked without rectification:
    pass it as `camera=` to SparseImgAlign.run and track (a sequence of them with cam_of_pair= for one camera per pair), and
    to Matcher.findMatchDirect.  world2cam / cam2world / errorMultiplier2 restate the model in
    NumPy (float64, the constructor's derived members and operation order; include/plsvo_b200.h states the formulas)."""

    def __init__(self, width: int, height: int, fx: float, fy: float, cx: float, cy: float, d0: float):
        import math

        self.struct = abi.AtanCamera(int(width), int(height), fx, fy, cx, cy, d0)
        self.fx_, self.fy_ = float(width) * fx, float(height) * fy
        self.cx_, self.cy_ = cx * float(width) - 0.5, cy * float(height) - 0.5
        self.s_ = float(d0)
        self.s_inv_ = self.tans_ = self.tans_inv_ = 0.0
        if self.s_ != 0.0:
            self.tans_ = 2.0 * math.tan(self.s_ / 2.0)
            self.tans_inv_ = 1.0 / self.tans_
            self.s_inv_ = 1.0 / self.s_

    @property
    def width(self) -> int:
        return self.struct.width

    @property
    def height(self) -> int:
        return self.struct.height

    def errorMultiplier2(self) -> float:
        return self.fx_

    def world2cam(self, xyz):
        """[..., 3] points in the camera frame -> [..., 2] pixels (world2cam(project2d(xyz)))."""
        import numpy as np

        xyz = np.asarray(xyz, np.float64)
        u, v = xyz[..., 0] / xyz[..., 2], xyz[..., 1] / xyz[..., 2]
        r = np.sqrt(u * u + v * v)
        with np.errstate(divide="ignore", invalid="ignore"):
            f = self.s_inv_ * np.arctan(r * self.tans_) / r
        factor = np.where((r < 0.001) | (self.s_ == 0.0), 1.0, f)
        return np.stack([self.cx_ + self.fx_ * (factor * u), self.cy_ + self.fy_ * (factor * v)], axis=-1)

    def cam2world(self, px):
        """[..., 2] pixels -> [..., 3] unit bearing vectors."""
        import numpy as np

        px = np.asarray(px, np.float64)
        x, y = (px[..., 0] - self.cx_) / self.fx_, (px[..., 1] - self.cy_) / self.fy_
        rd = np.sqrt(x * x + y * y)
        r = np.tan(rd * self.s_) * self.tans_inv_ if self.s_ != 0.0 else rd
        with np.errstate(divide="ignore", invalid="ignore"):
            factor = np.where(rd > 0.01, r / rd, 1.0)
        x, y = factor * x, factor * y
        n = np.sqrt((x * x + y * y) + 1.0)
        return np.stack([x / n, y / n, 1.0 / n], axis=-1)

    def _check(self, data):
        if (data.cam.width, data.cam.height) != (self.width, self.height):
            raise PlsvoError(f"ATANCamera is {self.width}x{self.height}, the batch's frames are {data.cam.width}x{data.cam.height}")


class feature_alignment:
    """Namespace mirror of plsvo::feature_alignment (include/plsvo/feature_alignment.h:49-55)."""

    @staticmethod
    def align2D(cur_pyr, image_index, level, ref_patch_with_border, ref_patch, n_iter, cur_px_estimate,
                width: int, height: int, ctx: Context | None = None):
        """Batched align2D (src/feature_alignment.cpp:160-290): returns (converged [n] bool, px [n,2])."""
        import numpy as np

        ctx = ctx or default_context()
        image_index = np.ascontiguousarray(image_index, np.int32)
        level = np.ascontiguousarray(level, np.int32)
        border = np.ascontiguousarray(ref_patch_with_border, np.uint8)
        ref = np.ascontiguousarray(ref_patch, np.uint8)
        px = np.ascontiguousarray(cur_px_estimate, np.float64)
        b, keep = abi.make_align2d_batch(cur_pyr, image_index, level, border, ref, px, n_iter, width, height)
        out_px = np.zeros_like(px)
        conv = np.zeros(len(image_index), np.uint8)
        r = abi.Align2DResult(out_px.ctypes.data_as(C.POINTER(C.c_double)), conv.ctypes.data_as(C.POINTER(C.c_uint8)))
        ctx.check(ctx.lib.plsvo_align2d_batch_run(ctx.handle, C.byref(b), C.byref(r)), "plsvo_align2d_batch_run")
        return conv.astype(bool), out_px

    @staticmethod
    def align1D(cur_pyr, image_index, level, dir, ref_patch_with_border, ref_patch, n_iter, cur_px_estimate,
                width: int, height: int, ctx: Context | None = None):
        """Batched align1D (src/feature_alignment.cpp:40-157): returns (converged [n] bool, px [n,2], h_inv [n])."""
        import numpy as np

        ctx = ctx or default_context()
        image_index = np.ascontiguousarray(image_index, np.int32)
        level = np.ascontiguousarray(level, np.int32)
        border = np.ascontiguousarray(ref_patch_with_border, np.uint8)
        ref = np.ascontiguousarray(ref_patch, np.uint8)
        px = np.ascontiguousarray(cur_px_estimate, np.float64)
        d = np.ascontiguousarray(dir, np.float32)
        feats, keep = abi.make_align2d_batch(cur_pyr, image_index, level, border, ref, px, n_iter, width, height)
        b = abi.Align1DBatch(feats, d.ctypes.data_as(C.POINTER(C.c_float)))
        out_px = np.zeros_like(px)
        conv = np.zeros(len(image_index), np.uint8)
        h_inv = np.zeros(len(image_index), np.float64)
        r = abi.Align1DResult(out_px.ctypes.data_as(C.POINTER(C.c_double)), conv.ctypes.data_as(C.POINTER(C.c_uint8)),
                              h_inv.ctypes.data_as(C.POINTER(C.c_double)))
        ctx.check(ctx.lib.plsvo_align1d_batch_run(ctx.handle, C.byref(b), C.byref(r)), "plsvo_align1d_batch_run")
        return conv.astype(bool), out_px, h_inv


class Matcher:
    """Batched counterpart of plsvo::Matcher::findMatchDirect (include/plsvo/matcher.h:104-107, src/matcher.cpp:159-211)
    for candidates whose reference observation has already been chosen (getCloseViewObs stays host-side list logic)."""

    def __init__(self, align_max_iter: int = 10, ctx: Context | None = None):
        self.align_max_iter = align_max_iter  # Matcher::Options::align_max_iter
        self.ctx = ctx or default_context()

    def findMatchDirect(self, data, camera: "ATANCamera | list | None" = None, cam_of_ref=None, cam_of_cur=None) -> abi.MatchOut:
        """data: synth.MatchData-like batch -> px_cur (refined, level-0 pixels), success flags, search levels.
        camera: an ATANCamera when the keyframes and current frames come from one (plsvo_match_direct_atan_batch_run;
        data.cam then only gives the image size); None for the undistorted pinhole of data.cam.  Or a sequence of cameras,
        each an ATANCamera or an undistorted pinhole given as a synth.Camera, with cam_of_ref [n_ref_images] and
        cam_of_cur [n_cur_images] indexing it: every image is seen through its own camera
        (plsvo_match_direct_multicam_batch_run; data.cam then only gives the slot size, synth.make_match_multicam_batch)."""
        data.n_iter = self.align_max_iter
        multi = _match_cameras_arg(camera, cam_of_ref, cam_of_cur, data)
        if camera is not None and multi is None:
            if not isinstance(camera, ATANCamera):
                raise TypeError(f"findMatchDirect: camera must be an ATANCamera or None, not {type(camera).__name__}")
            camera._check(data)
        b, keep = abi.make_match_batch(data)
        out = abi.MatchOut(data.n)
        if multi is not None:
            cams, ref, cur = multi
            self.ctx.check(self.ctx.lib.plsvo_match_direct_multicam_batch_run(
                self.ctx.handle, cams, len(cams), ref.ctypes.data_as(C.POINTER(C.c_int32)), cur.ctypes.data_as(C.POINTER(C.c_int32)),
                C.byref(b), C.byref(out.struct)), "plsvo_match_direct_multicam_batch_run")
        elif camera is not None:
            self.ctx.check(self.ctx.lib.plsvo_match_direct_atan_batch_run(self.ctx.handle, C.byref(camera.struct), C.byref(b),
                                                                          C.byref(out.struct)), "plsvo_match_direct_atan_batch_run")
        else:
            self.ctx.check(self.ctx.lib.plsvo_match_direct_batch_run(self.ctx.handle, C.byref(b), C.byref(out.struct)),
                           "plsvo_match_direct_batch_run")
        return out


def _match_cameras_arg(camera, cam_of_ref, cam_of_cur, data):
    """(plsvo_match_camera[K], cam_of_ref, cam_of_cur as int32 arrays) of the per-image match call when `camera` is a
    sequence; None for one camera or none.  Mismatched arguments raise PlsvoError; the values (index ranges, camera sizes
    and parameters) are the C ABI's to check."""
    import numpy as np

    seq = isinstance(camera, (list, tuple))
    if not seq:
        if cam_of_ref is not None or cam_of_cur is not None:
            raise PlsvoError("cam_of_ref= and cam_of_cur= select cameras per image: camera must then be a sequence of cameras")
        return None
    if cam_of_ref is None or cam_of_cur is None:
        raise PlsvoError("camera= as a sequence needs cam_of_ref= and cam_of_cur=")
    if len(camera) == 0:
        raise PlsvoError("camera= is an empty sequence")
    for k, c in enumerate(camera):
        if not isinstance(c, ATANCamera) and not all(hasattr(c, f) for f in ("width", "height", "fx", "fy", "cx", "cy")):
            raise PlsvoError(f"camera[{k}] must be an ATANCamera or a synth.Camera, not {type(c).__name__}")
    ref, cur = (np.ascontiguousarray(x) for x in (cam_of_ref, cam_of_cur))
    for name, x, n in (("cam_of_ref", ref, data.T_ref_w.shape[0]), ("cam_of_cur", cur, data.T_cur_w.shape[0])):
        if x.shape != (n,) or not np.issubdtype(x.dtype, np.integer):
            raise PlsvoError(f"{name} must be integers of shape [{n}] (a camera per image), got {x.dtype} {list(x.shape)}")
    return abi.make_match_cameras(camera), ref.astype(np.int32), cur.astype(np.int32)


def optimizeStructure(data, ctx: Context | None = None) -> abi.StructOptOut:
    """Batched Point::optimize / LineSeg::optimize (src/feature3D_impl.cpp:36-174) as FrameHandlerBase::optimizeStructure
    (src/frame_handler_base.cpp:202-237) applies them: data = synth.StructOptData-like CSR observation lists."""
    ctx = ctx or default_context()
    b, keep = abi.make_structopt_batch(data)
    out = abi.StructOptOut(b.n_points, b.n_segs)
    ctx.check(ctx.lib.plsvo_structopt_batch_run(ctx.handle, C.byref(b), C.byref(out.struct)), "plsvo_structopt_batch_run")
    return out


class DepthFilter:
    """Batched counterpart of plsvo::DepthFilter::updatePointSeeds (src/depth_filter.cpp:270-365): visibility test,
    Matcher::findEpipolarMatchDirect, computeTau and the Gaussian x Beta update of every seed; seed ageing, point creation
    and the detector's occupancy grid stay on the host."""

    def __init__(self, ctx: Context | None = None):
        self.ctx = ctx or default_context()

    def updateLineSeeds(self, data) -> abi.LineSeedOut:
        """Batched body of DepthFilter::updateLineSeeds (src/depth_filter.cpp:367-471): data = synth.LineSeedData-like."""
        b, keep = abi.make_line_seed_batch(data)
        out = abi.LineSeedOut(data.n)
        self.ctx.check(self.ctx.lib.plsvo_line_seed_update_batch_run(self.ctx.handle, C.byref(b), C.byref(out.line_struct)),
                       "plsvo_line_seed_update_batch_run")
        return out

    def updatePointSeeds(self, data) -> abi.SeedOut:
        b, keep = abi.make_seed_batch(data)
        out = abi.SeedOut(data.n)
        self.ctx.check(self.ctx.lib.plsvo_seed_update_batch_run(self.ctx.handle, C.byref(b), C.byref(out.struct)),
                       "plsvo_seed_update_batch_run")
        return out
