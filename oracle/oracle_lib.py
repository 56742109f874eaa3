"""Loader of the CPU oracle (oracle/libplsvo_oracle.so).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package (pl-svo_b200/) never imports this.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libplsvo_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "plsvo_oracle.cpp")
    hdr = os.path.join(_HERE, "..", "include", "plsvo_b200.h")
    stale = (not os.path.exists(LIB_PATH)) or any(
        os.path.exists(f) and os.path.getmtime(f) > os.path.getmtime(LIB_PATH) for f in (src, hdr)
    )
    if force or stale:
        subprocess.check_call(["make", "-C", _HERE, "-B" if force else "-s"] + ([] if force else []))
    return LIB_PATH


def load(abi):
    """abi = the pl-svo_b200.abi module (struct definitions are shared with the product header)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        build()
    lib = C.CDLL(LIB_PATH)
    P = C.POINTER
    lib.plsvo_oracle_align_batch.restype = C.c_int
    lib.plsvo_oracle_align_batch.argtypes = [P(abi.AlignBatch), P(abi.AlignParams), P(abi.AlignResult), C.c_int, C.c_int]
    lib.plsvo_oracle_align_trace.restype = C.c_int
    lib.plsvo_oracle_align_trace.argtypes = [P(abi.AlignBatch), P(abi.AlignParams), C.c_int, P(C.c_double), C.c_int, P(C.c_int)]
    lib.plsvo_oracle_trace_stride.restype = C.c_int
    lib.plsvo_oracle_poseopt_batch.restype = C.c_int
    lib.plsvo_oracle_poseopt_batch.argtypes = [P(abi.PoseOptBatch), P(abi.PoseOptParams), P(abi.PoseOptResult), C.c_int]
    for name, n_in in (("plsvo_oracle_se3_exp", 1), ("plsvo_oracle_se3_inverse", 1), ("plsvo_oracle_se3_mul", 2),
                       ("plsvo_oracle_solve6", 2), ("plsvo_oracle_inverse6", 1)):
        fn = getattr(lib, name)
        fn.restype = None
        fn.argtypes = [P(C.c_double)] * (n_in + 1)
    lib.plsvo_oracle_half_sample.restype = None
    lib.plsvo_oracle_half_sample.argtypes = [C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_size_t, C.POINTER(C.c_uint8), C.c_size_t]
    lib.plsvo_oracle_align2d.restype = C.c_int
    lib.plsvo_oracle_align2d.argtypes = [C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_size_t, C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), C.c_int, C.POINTER(C.c_double)]
    lib.plsvo_oracle_align1d.restype = C.c_int
    lib.plsvo_oracle_align1d.argtypes = [C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_size_t, C.POINTER(C.c_float), C.POINTER(C.c_uint8),
                                         C.POINTER(C.c_uint8), C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    lib.plsvo_oracle_hardware_threads.restype = C.c_int
    _lib = lib
    return lib


def align(abi, data, params=None, n_threads: int = 1, flags: int = 0):
    """Run the oracle's SparseImgAlign restatement on an AlignData batch -> abi.AlignOut."""
    lib = load(abi)
    params = params or abi.align_params(data.max_level, data.min_level)
    batch, keep = abi.make_align_batch(data)
    out = abi.AlignOut(data.batch, data.n_segs)
    rc = lib.plsvo_oracle_align_batch(C.byref(batch), C.byref(params), C.byref(out.struct), n_threads, flags)
    if rc != 0:
        raise RuntimeError(f"oracle align failed rc={rc}")
    return out


def align_trace(abi, data, pair: int, params=None, max_records: int = 512):
    lib = load(abi)
    params = params or abi.align_params(data.max_level, data.min_level)
    batch, keep = abi.make_align_batch(data)
    stride = lib.plsvo_oracle_trace_stride()
    rec = np.zeros((max_records, stride))
    n = C.c_int(0)
    rc = lib.plsvo_oracle_align_trace(C.byref(batch), C.byref(params), pair,
                                      rec.ctypes.data_as(C.POINTER(C.c_double)), max_records, C.byref(n))
    if rc != 0:
        raise RuntimeError(f"oracle trace failed rc={rc}")
    return rec[: n.value]


def poseopt(abi, data, params=None, n_threads: int = 1):
    lib = load(abi)
    params = params or abi.poseopt_params()
    batch, keep = abi.make_poseopt_batch(data)
    out = abi.PoseOptOut(data.batch, data.n_pts, data.n_segs)
    rc = lib.plsvo_oracle_poseopt_batch(C.byref(batch), C.byref(params), C.byref(out.struct), n_threads)
    if rc != 0:
        raise RuntimeError(f"oracle poseopt failed rc={rc}")
    return out


# exit reasons of a Gauss-Newton loop in poseopt_stats
PO_EXIT_NONE, PO_EXIT_CHI2, PO_EXIT_NAN, PO_EXIT_EPS, PO_EXIT_CAP = range(5)
PO_MEDIANS = ("mad_pt", "mad_ls", "init", "final")
PO_STAT_ITERS = 32


def poseopt_stats(abi, data, params=None, n_threads: int = 1):
    """The restated pose optimiser with a record of every frame's decisions -> (abi.PoseOptOut, stats).  The outputs are
    those of poseopt.  stats is a dict of arrays over the batch; [.., 2] is (main loop, refinement loop):
      exit [B,2]            PO_EXIT_*: chi2 rise, NaN step, EPS, iteration cap, or no iteration (also: no observation)
      fallback [B,2]        some solve's A has an unpivoted LDL^T pivot not above 1e-13 * max|diag A| (the GPU's register
                            solve then hands the system to the pivoted one)
      scale_pt, scale_ls [B]  the two MAD scales, before the fx factor
      med_count, med_tie [B,4]  per PO_MEDIANS: the live count, and whether the key of rank n // 2 is tied with a neighbour
      out_margin_pt, out_margin_ls [B]  smallest |e - thr| / thr of the outlier decisions (inf: none, or thr infinite)
      chi2_margin, eps_margin [B,2]  smallest relative margin of the new_chi2 > chi2 and norm_max(dT) <= EPS decisions
      iter_margin [B,2,PO_STAT_ITERS]  the smaller of the two at each iteration (inf: no such decision)"""
    lib = load(abi)
    params = params or abi.poseopt_params()
    batch, keep = abi.make_poseopt_batch(data)
    out = abi.PoseOptOut(data.batch, data.n_pts, data.n_segs)
    lib.plsvo_oracle_poseopt_stats_stride.restype = C.c_int
    stride = lib.plsvo_oracle_poseopt_stats_stride()
    assert stride == 20 + 2 * PO_STAT_ITERS
    st = np.zeros((data.batch, stride))
    fn = lib.plsvo_oracle_poseopt_stats
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(abi.PoseOptBatch), C.POINTER(abi.PoseOptParams), C.POINTER(abi.PoseOptResult), C.POINTER(C.c_double), C.c_int]
    rc = fn(C.byref(batch), C.byref(params), C.byref(out.struct), st.ctypes.data_as(C.POINTER(C.c_double)), n_threads)
    if rc != 0:
        raise RuntimeError(f"oracle poseopt_stats failed rc={rc}")
    return out, {
        "exit": st[:, 0:2].astype(np.int32), "fallback": st[:, 2:4] != 0, "scale_pt": st[:, 4].copy(), "scale_ls": st[:, 5].copy(),
        "med_count": st[:, 6:10].astype(np.int64), "med_tie": st[:, 10:14] != 0, "out_margin_pt": st[:, 14].copy(),
        "out_margin_ls": st[:, 15].copy(), "chi2_margin": st[:, 16:18].copy(), "eps_margin": st[:, 18:20].copy(),
        "iter_margin": st[:, 20:].reshape(-1, 2, PO_STAT_ITERS).copy()}


def pyramid(abi, img0, n_levels: int):
    """frame_utils::createImgPyramid restated: u8 [B,H,W] -> list of levels."""
    lib = load(abi)
    img0 = np.ascontiguousarray(img0, np.uint8)
    levels = [img0]
    u8p = C.POINTER(C.c_uint8)
    for _ in range(1, n_levels):
        prev = levels[-1]
        B, H, W = prev.shape
        out = np.empty((B, H // 2, W // 2), np.uint8)
        for b in range(B):
            lib.plsvo_oracle_half_sample(prev[b].ctypes.data_as(u8p), W, H, prev.strides[1], out[b].ctypes.data_as(u8p), out.strides[1])
        levels.append(out)
    return levels


def align2d(abi, cur_pyr, image_index, level, border, ref, px, n_iter):
    """feature_alignment::align2D restated, looped over features -> (converged [n] bool, px [n,2])."""
    lib = load(abi)
    u8p, dp = C.POINTER(C.c_uint8), C.POINTER(C.c_double)
    out = np.array(px, np.float64, copy=True)
    conv = np.zeros(len(image_index), bool)
    border = np.ascontiguousarray(border, np.uint8)
    ref = np.ascontiguousarray(ref, np.uint8)
    for i in range(len(image_index)):
        im = np.ascontiguousarray(cur_pyr[int(level[i])][int(image_index[i])])
        p = out[i].copy()
        conv[i] = bool(lib.plsvo_oracle_align2d(im.ctypes.data_as(u8p), im.shape[1], im.shape[0], im.strides[0],
                                                border[i].ctypes.data_as(u8p), ref[i].ctypes.data_as(u8p), n_iter,
                                                p.ctypes.data_as(dp)))
        out[i] = p
    return conv, out


# ---- align2D / align1D / findMatchDirect over whole batches, on all cores, optionally with each feature's decisions --------
# The record of one feature (plsvo_oracle_direct_stats_stride() doubles, laid out at DirectStats in plsvo_oracle.cpp)
DS_EXIT_NONE, DS_EXIT_FRAME, DS_EXIT_CONVERGED, DS_EXIT_CAP, DS_EXIT_BACKOFF = range(5)
DS_BOUNDS = ("left", "top", "right", "bottom")  # the order of stats["dist"] columns and of the stats["bound"] bits


def _n_threads(abi, n_threads):
    return n_threads or max(1, load(abi).plsvo_oracle_hardware_threads())


def _direct_stats(st):
    singular = st[:, 2].astype(np.int64)
    return {"exit": st[:, 0].astype(np.int32), "iter": st[:, 1].astype(np.int32), "det_zero": (singular & 1) != 0,
            "hinv_nonfinite": (singular & 2) != 0, "h_inv_nonfinite": (singular & 4) != 0, "conv_margin": st[:, 3].copy(),
            "backoff_margin": st[:, 4].copy(), "tie": st[:, 5] != 0, "dist": st[:, 6:10].copy(), "bound": st[:, 10].astype(np.int32),
            "offset": st[:, 11].astype(np.int32), "reject": st[:, 12] != 0, "nan_warp": st[:, 13] != 0, "clamped": st[:, 14] != 0,
            "zeroed": st[:, 15].astype(np.int32), "nan_dir": st[:, 16] != 0, "edgelet": st[:, 17] != 0,
            "on_bound": st[:, 18].astype(np.int32)}


def _stats_fn(lib, name, batch_t, result_t):
    fn = getattr(lib, name)
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(batch_t), C.POINTER(result_t), C.POINTER(C.c_double), C.c_int]
    return fn


def feature_align_stats(abi, kind, cur_pyr, image_index, level, border, ref, px, n_iter, width, height, dirs=None, n_threads=0,
                        stats=True):
    """align2D (kind "2d") or align1D (kind "1d", along dirs) over a batch, through plsvo_oracle_align{2,1}d_batch or, with
    stats, through plsvo_oracle_align{2,1}d_stats, which run the same code and also record each feature's decisions.
    cur_pyr: {level: u8 [n_images,h,w]} (views with unit column stride are fine).  Returns ((converged, px) for "2d" or
    (converged, px, h_inv) for "1d", stats); stats is None without stats, else a dict of arrays over the features:
      exit, iter            DS_EXIT_* and the iteration the loop ended at (n_iter - 1 at the cap, -1 without an iteration)
      det_zero, hinv_nonfinite, h_inv_nonfinite   a singular H: det == 0, a non-finite Hinv entry, a non-finite h_inv
      conv_margin, backoff_margin   smallest relative margin of the convergence and of the back-off test (inf: none)
      tie                   a back-off test compared equal chi2 values
      dist [n,4]            smallest distance of floor(u), floor(v) to each in-frame bound (DS_BOUNDS; negative = outside)
      bound                 the bounds a frame exit failed, bit k = DS_BOUNDS[k]
      offset                (floor(u) - 4) & 3 at the first iteration inside the frame, else -1"""
    assert kind in ("2d", "1d")
    lib = load(abi)
    pyr = cur_pyr if isinstance(cur_pyr, dict) else dict(enumerate(cur_pyr))
    image_index = np.ascontiguousarray(image_index, np.int32)
    level = np.ascontiguousarray(level, np.int32)
    border = np.ascontiguousarray(border, np.uint8)
    ref = np.ascontiguousarray(ref, np.uint8)
    px = np.ascontiguousarray(px, np.float64)
    n = len(image_index)
    b, keep = abi.make_align2d_batch(pyr, image_index, level, border, ref, px, n_iter, width, height)
    out_px, conv = np.zeros((n, 2)), np.zeros(n, np.uint8)
    dp, u8p = C.POINTER(C.c_double), C.POINTER(C.c_uint8)
    st = np.zeros((n, lib.plsvo_oracle_direct_stats_stride())) if stats else None
    if kind == "2d":
        r = abi.Align2DResult(out_px.ctypes.data_as(dp), conv.ctypes.data_as(u8p))
        name, bt, rt, arg = "plsvo_oracle_align2d", abi.Align2DBatch, abi.Align2DResult, b
    else:
        d = np.ascontiguousarray(dirs, np.float32)
        h_inv = np.zeros(n)
        arg = abi.Align1DBatch(b, d.ctypes.data_as(C.POINTER(C.c_float)))
        r = abi.Align1DResult(out_px.ctypes.data_as(dp), conv.ctypes.data_as(u8p), h_inv.ctypes.data_as(dp))
        name, bt, rt = "plsvo_oracle_align1d", abi.Align1DBatch, abi.Align1DResult
    nt = _n_threads(abi, n_threads)
    if stats:
        rc = _stats_fn(lib, name + "_stats", bt, rt)(C.byref(arg), C.byref(r), st.ctypes.data_as(dp), nt)
    else:
        fn = getattr(lib, name + "_batch")
        fn.restype, fn.argtypes = C.c_int, [C.POINTER(bt), C.POINTER(rt), C.c_int]
        rc = fn(C.byref(arg), C.byref(r), nt)
    if rc != 0:
        raise RuntimeError(f"oracle {name} failed rc={rc}")
    outs = (conv.astype(bool), out_px) if kind == "2d" else (conv.astype(bool), out_px, h_inv)
    return outs, (_direct_stats(st) if stats else None)


def align2d_batch(abi, cur_pyr, image_index, level, border, ref, px, n_iter, width, height, n_threads=0):
    """align2d on all cores (plsvo_oracle_align2d_batch) -> (converged [n] bool, px [n,2])."""
    return feature_align_stats(abi, "2d", cur_pyr, image_index, level, border, ref, px, n_iter, width, height, None, n_threads, False)[0]


def align1d_batch(abi, cur_pyr, image_index, level, dirs, border, ref, px, n_iter, width, height, n_threads=0):
    """align1d on all cores (plsvo_oracle_align1d_batch) -> (converged [n] bool, px [n,2], h_inv [n])."""
    return feature_align_stats(abi, "1d", cur_pyr, image_index, level, border, ref, px, n_iter, width, height, dirs, n_threads, False)[0]


def match_direct_stats(abi, data, n_threads=0, out=None):
    """match_direct through plsvo_oracle_match_direct_stats -> (abi.MatchOut, stats): the stats of feature_align_stats
    (exit kind "none" where the candidate never reaches alignment) and, per candidate:
      reject     failed the reference in-frame test       nan_warp   the affine warp is NaN (the patch stays zero)
      clamped    the search level stopped at n_pyr_levels - 1 with D > 3
      zeroed     border-patch pixels set to 0 because they lie outside the reference image
      nan_dir    an edgelet whose warped gradient direction is NaN;   edgelet   aligned with align1D
      on_bound   border-patch samples exactly on the last column or row of the reference image (zeroed, as outside)
    out: an abi.MatchOut to write into (e.g. with A_cur_ref prefilled), else a fresh one."""
    lib = load(abi)
    b, keep = abi.make_match_batch(data)
    out = out or abi.MatchOut(data.n)
    st = np.zeros((data.n, lib.plsvo_oracle_direct_stats_stride()))
    fn = _stats_fn(lib, "plsvo_oracle_match_direct_stats", abi.MatchBatch, abi.MatchResult)
    rc = fn(C.byref(b), C.byref(out.struct), st.ctypes.data_as(C.POINTER(C.c_double)), _n_threads(abi, n_threads))
    if rc != 0:
        raise RuntimeError(f"oracle match_direct_stats failed rc={rc}")
    return out, _direct_stats(st)


# ---- oracle/_ref: the reference's own translation units (oracle/ref_harness.cpp, Makefile target `ref`) ----
REF_LIB_PATH = os.path.join(_HERE, "_ref", "libplsvo_ref.so")
REFERENCE_ROOT = os.environ.get("PLSVO_REFERENCE_ROOT", "/root/reference")
_ref_lib = None


def build_ref(force: bool = False) -> str | None:
    """Build oracle/_ref/libplsvo_ref.so when the reference sources are present (authoring container only).
    Returns the path, or None when neither the sources nor a prebuilt library exist."""
    srcs = [os.path.join(REFERENCE_ROOT, "src", f) for f in ("sparse_img_align.cpp", "pose_optimizer.cpp", "feature.cpp", "feature_alignment.cpp", "matcher.cpp", "config.cpp", "feature3D_impl.cpp", "depth_filter.cpp")]
    if all(os.path.exists(s) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "ref", f"REFERENCE={REFERENCE_ROOT}"] + (["-B"] if force else ["-s"]))
    return REF_LIB_PATH if os.path.exists(REF_LIB_PATH) else None


SHIMREF_LIB_PATH = os.path.join(_HERE, "_ref", "libplsvo_shimref.so")
_shimref_lib = None


def build_shimref(force: bool = False) -> str | None:
    """oracle/_ref/libplsvo_shimref.so: reference-typed Frame / Feature objects driven through the shim compiled in
    reference-headers mode (oracle/shimref_harness.cpp).  Needs /root/reference and the built CUDA library to build."""
    if os.path.exists(os.path.join(REFERENCE_ROOT, "src", "feature.cpp")) and os.path.exists(
            os.path.join(_HERE, "..", "pl-svo_b200", "csrc", "libplsvo_b200.so")):
        subprocess.check_call(["make", "-C", _HERE, "shimref", f"REFERENCE={REFERENCE_ROOT}"] + (["-B"] if force else ["-s"]))
    return SHIMREF_LIB_PATH if os.path.exists(SHIMREF_LIB_PATH) else None


SHIMREF_CPU_LIB_PATH = os.path.join(_HERE, "_ref", "libplsvo_shimref_cpu.so")
_shimref_cpu_lib = None


def build_shimref_cpu(force: bool = False) -> str | None:
    """oracle/_ref/libplsvo_shimref_cpu.so: the same harness + shim with the C ABI answered by the CPU oracle
    (oracle/abi_on_oracle.cpp) — checks the shim's packing of reference objects without a GPU."""
    if os.path.exists(os.path.join(REFERENCE_ROOT, "src", "feature.cpp")):
        subprocess.check_call(["make", "-C", _HERE, "shimref-cpu", f"REFERENCE={REFERENCE_ROOT}"] + (["-B"] if force else ["-s"]))
    return SHIMREF_CPU_LIB_PATH if os.path.exists(SHIMREF_CPU_LIB_PATH) else None


def load_shimref(abi, cpu: bool = False):
    global _shimref_lib, _shimref_cpu_lib
    if cpu:
        if _shimref_cpu_lib is None:
            lib = C.CDLL(SHIMREF_CPU_LIB_PATH)
            P = C.POINTER
            lib.plsvo_shimref_align_batch.restype = C.c_int
            lib.plsvo_shimref_align_batch.argtypes = [P(abi.AlignBatch), P(abi.AlignParams), P(abi.AlignResult)]
            lib.plsvo_shimref_poseopt_batch.restype = C.c_int
            lib.plsvo_shimref_poseopt_batch.argtypes = [P(abi.PoseOptBatch), P(abi.PoseOptParams), P(abi.PoseOptResult)]
            _shimref_cpu_lib = lib
        return _shimref_cpu_lib
    if _shimref_lib is None:
        lib = C.CDLL(SHIMREF_LIB_PATH)
        P = C.POINTER
        lib.plsvo_shimref_align_batch.restype = C.c_int
        lib.plsvo_shimref_align_batch.argtypes = [P(abi.AlignBatch), P(abi.AlignParams), P(abi.AlignResult)]
        lib.plsvo_shimref_poseopt_batch.restype = C.c_int
        lib.plsvo_shimref_poseopt_batch.argtypes = [P(abi.PoseOptBatch), P(abi.PoseOptParams), P(abi.PoseOptResult)]
        _shimref_lib = lib
    return _shimref_lib


def shimref_align(abi, data, params=None, cpu: bool = False):
    """plsvo::SparseImgAlign(...).run(ref, cur) of the shim on reference-typed frames -> abi.AlignOut
    (T_cur_w, n_tracked, seg_killed; H holds getFisherInformation() = H / (5e-4 * 255^2))."""
    lib = load_shimref(abi, cpu)
    params = params or abi.align_params(data.max_level, data.min_level)
    batch, keep = abi.make_align_batch(data)
    out = abi.AlignOut(data.batch, data.n_segs)
    rc = lib.plsvo_shimref_align_batch(C.byref(batch), C.byref(params), C.byref(out.struct))
    if rc != 0:
        raise RuntimeError(f"shimref align failed rc={rc}")
    return out


def shimref_poseopt(abi, data, params=None, cpu: bool = False):
    lib = load_shimref(abi, cpu)
    params = params or abi.poseopt_params()
    batch, keep = abi.make_poseopt_batch(data)
    out = abi.PoseOptOut(data.batch, data.n_pts, data.n_segs)
    rc = lib.plsvo_shimref_poseopt_batch(C.byref(batch), C.byref(params), C.byref(out.struct))
    if rc != 0:
        raise RuntimeError(f"shimref poseopt failed rc={rc}")
    return out


def ref_available() -> bool:
    return os.path.exists(REF_LIB_PATH)


# ---- recorded reference outputs (tests/golden/reference.npz.xz) --------------------------------------------------------
# The reference's sources are not part of this repository, so oracle/_ref can only be built where they are present.
# Everywhere else the @_recorded ref_* calls answer from outputs recorded from oracle/_ref for the exact inputs the tests
# give them (keyed by a hash of the inputs), so that those tests keep comparing against the reference itself.  A call
# with inputs that were never recorded raises.  PLSVO_RECORD_REF=1 adds the outputs of every live @_recorded call (and
# the digests of every assert_ref_equal comparison) when the process exits.
GOLDEN_REF_PATH = os.path.join(_HERE, "..", "tests", "golden", "reference.npz.xz")
_golden_ref = None


def have_ref() -> bool:
    """oracle/_ref is built here (or can be), or recorded outputs of it are present."""
    return bool(build_ref()) or os.path.exists(GOLDEN_REF_PATH)


def _golden_archive() -> dict:
    global _golden_ref
    if _golden_ref is None:
        import io
        import lzma

        _golden_ref = {}
        if os.path.exists(GOLDEN_REF_PATH):
            with open(GOLDEN_REF_PATH, "rb") as f, np.load(io.BytesIO(lzma.decompress(f.read()))) as z:
                _golden_ref = {k: z[k] for k in z.files}
    return _golden_ref


def _save_golden_archive():
    import io
    import lzma

    buf = io.BytesIO()
    np.savez(buf, **_golden_archive())
    with open(GOLDEN_REF_PATH, "wb") as f:
        f.write(lzma.compress(buf.getvalue(), preset=9 | lzma.PRESET_EXTREME))


def _digest(h, x):
    if isinstance(x, np.ndarray):
        x = np.ascontiguousarray(x)
        h.update(f"a{x.dtype.str}{x.shape}".encode())
        h.update(x.tobytes())
    elif isinstance(x, C.Structure):
        h.update(b"s" + type(x).__name__.encode() + bytes(x))
    elif isinstance(x, dict):
        for k in sorted(x):
            h.update(f"k{k!r}".encode())
            _digest(h, x[k])
    elif isinstance(x, (list, tuple)):
        h.update(b"l%d" % len(x))
        for v in x:
            _digest(h, v)
    elif hasattr(x, "__dict__") and not isinstance(x, type):
        _digest(h, {k: v for k, v in vars(x).items() if not k.startswith("_")})
    elif x is None or isinstance(x, (bool, int, float, str, np.generic)):
        h.update(repr(x).encode())
    else:
        _digest(h, np.asarray(x))


def _pack(x, name, d, ints_only=False):
    if isinstance(x, tuple):
        d[name + "~tuple"] = np.array(len(x))
        for i, v in enumerate(x):
            _pack(v, f"{name}~{i}", d, ints_only)
    elif isinstance(x, np.ndarray):
        if not ints_only or x.dtype.kind in "biu":
            d[name] = x
    else:
        for k, v in vars(x).items():
            if isinstance(v, np.ndarray) and (not ints_only or v.dtype.kind in "biu"):
                d[f"{name}.{k}"] = v


class _Tuple(tuple):
    """A ref_* call's tuple of outputs, with the key of the call (assert_ref_equal)."""


def _unpack(z, name):
    if name + "~tuple" in z:
        return _Tuple(_unpack(z, f"{name}~{i}") for i in range(int(z[name + "~tuple"])))
    if name in z:
        return z[name].copy()
    if not any(k.startswith(name + ".") for k in z):
        return None  # a floating-point element of the tuple: only digests of it are recorded
    r = _Rec()
    for k in z:
        if k.startswith(name + "."):
            setattr(r, k[len(name) + 1:], z[k].copy())
    return r


_record_pending = False


def _record(key, value):
    """Add one entry to the archive; the archive is written once, when the process exits."""
    global _record_pending
    _golden_archive()[key] = value
    if not _record_pending:
        import atexit

        atexit.register(_save_golden_archive)
        _record_pending = True


def _recorded(fn):
    """Answer fn(abi, *args) from oracle/_ref when it is built, else from the recording of the same call.

    Only the integer outputs are recorded whole; the floating-point outputs are compared through assert_ref_equal, which
    records a digest of exactly what it compared (storing them whole would not keep the repository small)."""
    import functools
    import hashlib

    @functools.wraps(fn)
    def call(abi, *args, n_threads=None, **kw):
        h = hashlib.sha256(fn.__name__.encode())
        _digest(h, (list(args), kw))
        key = f"{fn.__name__}-{h.hexdigest()[:16]}"
        if not ref_available():
            z = _golden_archive()
            if key + "~tuple" not in z and key + "~call" not in z and not any(k.startswith(key + ".") for k in z):
                raise KeyError(f"{fn.__name__}: oracle/_ref is not built and these inputs were not recorded ({key})")
            out = _unpack(z, key)
        else:
            out = fn(abi, *args, **kw) if n_threads is None else fn(abi, *args, n_threads=n_threads, **kw)
            if os.environ.get("PLSVO_RECORD_REF"):
                d = {key + "~call": np.array(0)}
                _pack(out, key, d, ints_only=True)
                for k, v in d.items():
                    _record(k, v)
        out = _Tuple(out) if isinstance(out, tuple) else out
        out._ref_key = key
        return out

    return call


def _canonical_digest(x) -> np.ndarray:
    """sha256 of an array under np.testing.assert_array_equal's equality: every NaN alike, -0.0 == 0.0."""
    import hashlib

    x = np.ascontiguousarray(x)
    if x.dtype.kind == "f":
        x = np.where(np.isnan(x), np.array(np.nan, x.dtype), x + x.dtype.type(0))
    h = hashlib.sha256(f"{x.dtype.str}{x.shape}".encode())
    h.update(x.tobytes())
    return np.frombuffer(h.digest(), np.uint8)


def assert_ref_equal(actual, ref_out, field: str, rows=None, err_msg: str = ""):
    """np.testing.assert_array_equal(actual[rows], ref_out.<field>[rows]) for the output of a @_recorded ref_* call.  Without
    oracle/_ref the reference side is the digest recorded for this call, field and row selection."""
    sel = slice(None) if rows is None else rows
    got = np.asarray(actual)[sel]
    key = f"{ref_out._ref_key}:{field}:{_canonical_digest(np.asarray(rows if rows is not None else [])).tobytes().hex()[:16]}"
    want = ref_out[int(field)] if isinstance(ref_out, tuple) else getattr(ref_out, field, None)
    if want is not None:
        np.testing.assert_array_equal(got, want[sel], err_msg=err_msg)
        if ref_available() and os.environ.get("PLSVO_RECORD_REF"):
            _record(key, _canonical_digest(want[sel]))
        return
    if key not in _golden_archive():
        raise KeyError(f"{field}: oracle/_ref is not built and this comparison was not recorded ({key})")
    assert np.array_equal(_canonical_digest(got), _golden_archive()[key]), \
        f"{field} differs from the reference's recorded output {err_msg}"


def load_ref(abi):
    global _ref_lib
    if _ref_lib is not None:
        return _ref_lib
    if not os.path.exists(REF_LIB_PATH):
        raise FileNotFoundError(f"{REF_LIB_PATH} is not built (needs {REFERENCE_ROOT}; run `make -C oracle ref`)")
    lib = C.CDLL(REF_LIB_PATH)
    P = C.POINTER
    lib.plsvo_ref_align_batch.restype = C.c_int
    lib.plsvo_ref_align_batch.argtypes = [P(abi.AlignBatch), P(abi.AlignParams), P(abi.AlignResult), C.c_int]
    lib.plsvo_ref_poseopt_batch.restype = C.c_int
    lib.plsvo_ref_poseopt_batch.argtypes = [P(abi.PoseOptBatch), P(abi.PoseOptParams), P(abi.PoseOptResult), C.c_int]
    lib.plsvo_ref_describe.restype = C.c_char_p
    u8p, dp = P(C.c_uint8), P(C.c_double)
    lib.plsvo_ref_align2d.restype = C.c_int
    lib.plsvo_ref_align2d.argtypes = [u8p, C.c_int, C.c_int, C.c_size_t, u8p, u8p, C.c_int, dp]
    lib.plsvo_ref_align1d.restype = C.c_int
    lib.plsvo_ref_align1d.argtypes = [u8p, C.c_int, C.c_int, C.c_size_t, P(C.c_float), u8p, u8p, C.c_int, dp, dp]
    _ref_lib = lib
    return lib


@_recorded
def ref_align(abi, data, params=None, n_threads: int = 1):
    """SparseImgAlign::run of the reference's own sparse_img_align.cpp on an AlignData batch -> abi.AlignOut."""
    lib = load_ref(abi)
    params = params or abi.align_params(data.max_level, data.min_level)
    batch, keep = abi.make_align_batch(data)
    out = abi.AlignOut(data.batch, data.n_segs)
    rc = lib.plsvo_ref_align_batch(C.byref(batch), C.byref(params), C.byref(out.struct), n_threads)
    if rc != 0:
        raise RuntimeError(f"reference align failed rc={rc}")
    return out


@_recorded
def ref_poseopt(abi, data, params=None, n_threads: int = 1):
    """pose_optimizer::optimizeGaussNewton of the reference's own pose_optimizer.cpp -> abi.PoseOptOut."""
    lib = load_ref(abi)
    params = params or abi.poseopt_params()
    batch, keep = abi.make_poseopt_batch(data)
    out = abi.PoseOptOut(data.batch, data.n_pts, data.n_segs)
    rc = lib.plsvo_ref_poseopt_batch(C.byref(batch), C.byref(params), C.byref(out.struct), n_threads)
    if rc != 0:
        raise RuntimeError(f"reference poseopt failed rc={rc}")
    return out


@_recorded
def ref_align2d(abi, cur_pyr, image_index, level, border, ref, px, n_iter):
    """feature_alignment::align2D of the reference's own feature_alignment.cpp, looped over features."""
    lib = load_ref(abi)
    u8p, dp = C.POINTER(C.c_uint8), C.POINTER(C.c_double)
    out = np.array(px, np.float64, copy=True)
    conv = np.zeros(len(image_index), bool)
    border = np.ascontiguousarray(border, np.uint8)
    ref = np.ascontiguousarray(ref, np.uint8)
    for i in range(len(image_index)):
        im = np.ascontiguousarray(cur_pyr[int(level[i])][int(image_index[i])])
        p = out[i].copy()
        conv[i] = bool(lib.plsvo_ref_align2d(im.ctypes.data_as(u8p), im.shape[1], im.shape[0], im.strides[0],
                                             border[i].ctypes.data_as(u8p), ref[i].ctypes.data_as(u8p), n_iter,
                                             p.ctypes.data_as(dp)))
        out[i] = p
    return conv, out


def _align1d_loop(fn, cur_pyr, image_index, level, dirs, border, ref, px, n_iter):
    u8p, dp, fp = C.POINTER(C.c_uint8), C.POINTER(C.c_double), C.POINTER(C.c_float)
    out = np.array(px, np.float64, copy=True)
    conv = np.zeros(len(image_index), bool)
    h_inv = np.zeros(len(image_index))
    border = np.ascontiguousarray(border, np.uint8)
    ref = np.ascontiguousarray(ref, np.uint8)
    dirs = np.ascontiguousarray(dirs, np.float32)
    for i in range(len(image_index)):
        im = np.ascontiguousarray(cur_pyr[int(level[i])][int(image_index[i])])
        p = out[i].copy()
        h = C.c_double(0)
        conv[i] = bool(fn(im.ctypes.data_as(u8p), im.shape[1], im.shape[0], im.strides[0], dirs[i].ctypes.data_as(fp),
                          border[i].ctypes.data_as(u8p), ref[i].ctypes.data_as(u8p), n_iter, p.ctypes.data_as(dp), C.byref(h)))
        out[i] = p
        h_inv[i] = h.value
    return conv, out, h_inv


def align1d(abi, cur_pyr, image_index, level, dirs, border, ref, px, n_iter):
    """feature_alignment::align1D restated -> (converged [n], px [n,2], h_inv [n])."""
    return _align1d_loop(load(abi).plsvo_oracle_align1d, cur_pyr, image_index, level, dirs, border, ref, px, n_iter)


@_recorded
def ref_align1d(abi, cur_pyr, image_index, level, dirs, border, ref, px, n_iter):
    """feature_alignment::align1D of the reference's own feature_alignment.cpp."""
    return _align1d_loop(load_ref(abi).plsvo_ref_align1d, cur_pyr, image_index, level, dirs, border, ref, px, n_iter)


def match_direct(abi, data, n_threads: int = 1, out=None):
    """Matcher::findMatchDirect restated, over a synth.MatchData batch -> abi.MatchOut (out, if given, is written into)."""
    lib = load(abi)
    lib.plsvo_oracle_match_direct_batch.restype = C.c_int
    lib.plsvo_oracle_match_direct_batch.argtypes = [C.POINTER(abi.MatchBatch), C.POINTER(abi.MatchResult), C.c_int]
    b, keep = abi.make_match_batch(data)
    out = out or abi.MatchOut(data.n)
    rc = lib.plsvo_oracle_match_direct_batch(C.byref(b), C.byref(out.struct), n_threads)
    if rc != 0:
        raise RuntimeError(f"oracle match_direct failed rc={rc}")
    return out


@_recorded
def ref_match_direct(abi, data):
    """Matcher::findMatchDirect of the reference's own matcher.cpp -> abi.MatchOut."""
    lib = load_ref(abi)
    lib.plsvo_ref_match_direct_batch.restype = C.c_int
    lib.plsvo_ref_match_direct_batch.argtypes = [C.POINTER(abi.MatchBatch), C.POINTER(abi.MatchResult)]
    b, keep = abi.make_match_batch(data)
    out = abi.MatchOut(data.n)
    rc = lib.plsvo_ref_match_direct_batch(C.byref(b), C.byref(out.struct))
    if rc != 0:
        raise RuntimeError(f"reference match_direct failed rc={rc}")
    return out


def structopt(abi, data, n_threads: int = 1):
    """Point::optimize / LineSeg::optimize restated -> abi.StructOptOut."""
    lib = load(abi)
    lib.plsvo_oracle_structopt_batch.restype = C.c_int
    lib.plsvo_oracle_structopt_batch.argtypes = [C.POINTER(abi.StructOptBatch), C.POINTER(abi.StructOptResult), C.c_int]
    b, keep = abi.make_structopt_batch(data)
    out = abi.StructOptOut(b.n_points, b.n_segs)
    rc = lib.plsvo_oracle_structopt_batch(C.byref(b), C.byref(out.struct), n_threads)
    if rc != 0:
        raise RuntimeError(f"oracle structopt failed rc={rc}")
    return out


# exit reasons of Point::optimize / LineSeg::optimize in structopt_stats (the same numbers as PO_EXIT_*)
SO_EXIT_NONE, SO_EXIT_CHI2, SO_EXIT_NAN, SO_EXIT_EPS, SO_EXIT_CAP = range(5)
SO_CAUSE_CHI2, SO_CAUSE_NAN, SO_CAUSE_EPS = 1, 2, 4
# the six transposition pairs (tr[0], tr[1]) of a pivoted 3x3 LDLT; bit 2 * tr[0] + tr[1] - 1 of "pivots"
SO_PIVOTS = ((0, 1), (0, 2), (1, 1), (1, 2), (2, 1), (2, 2))


def structopt_stats(abi, data, n_threads: int = 1):
    """The restated structure optimisation with a record of every point's and every segment end's decisions ->
    (abi.StructOptOut, pt_stats, seg_stats).  The outputs are those of structopt.  pt_stats is a dict of arrays over the
    points, seg_stats the same over [n_segs, 2] (the s and e ends):
      exit, exit_it       SO_EXIT_* and the iteration it was taken at (-1: n_iter = 0); a segment's ends share them
      cause               bits SO_CAUSE_*: what this end did at the exit (for a segment: which end caused it)
      pivots              bitmask over the LDLTs factored, bit k for the transposition pair SO_PIVOTS[k]
      zero                some LDLT took the k == 0 early return (the whole diagonal of A is 0 or NaN)
      d_zeroed            in an LDLT without the early return, the pseudo-inverse tolerance zeroed a finite D entry
      d_ratio             smallest min|D| / max|D| over the LDLTs factored
      A [.., 3, 3], b [.., 3]  the first iteration's normal equations; cond: the 2-norm condition number of that A (inf
                          when singular, NaN when not finite)"""
    lib = load(abi)
    lib.plsvo_oracle_structopt_stats_stride.restype = C.c_int
    stride = lib.plsvo_oracle_structopt_stats_stride()
    assert stride == 19
    fn = lib.plsvo_oracle_structopt_stats
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(abi.StructOptBatch), C.POINTER(abi.StructOptResult), C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int]
    b, keep = abi.make_structopt_batch(data)
    out = abi.StructOptOut(b.n_points, b.n_segs)
    pst = np.zeros((max(b.n_points, 1), stride))
    sst = np.zeros((max(b.n_segs, 1), 2, stride))
    dp = C.POINTER(C.c_double)
    rc = fn(C.byref(b), C.byref(out.struct), pst.ctypes.data_as(dp), sst.ctypes.data_as(dp), _n_threads(abi, n_threads))
    if rc != 0:
        raise RuntimeError(f"oracle structopt_stats failed rc={rc}")

    def unpack(st):
        A = st[..., 7:16].reshape(st.shape[:-1] + (3, 3)).copy()
        cond = np.full(st.shape[:-1], np.nan)
        fin = np.isfinite(A).all((-2, -1))
        if fin.any():
            with np.errstate(divide="ignore", invalid="ignore"):
                s = np.linalg.svd(A[fin], compute_uv=False)
                cond[fin] = np.where(s[..., -1] > 0, s[..., 0] / s[..., -1], np.inf)
        return {"exit": st[..., 0].astype(np.int32), "exit_it": st[..., 1].astype(np.int32), "cause": st[..., 2].astype(np.int32),
                "pivots": st[..., 3].astype(np.int32), "zero": st[..., 4] != 0, "d_zeroed": st[..., 5] != 0,
                "d_ratio": st[..., 6].copy(), "A": A, "b": st[..., 16:19].copy(), "cond": cond}

    return out, unpack(pst[: b.n_points]), unpack(sst[: b.n_segs])


@_recorded
def ref_structopt(abi, data):
    """Point::optimize / LineSeg::optimize of the reference's own feature3D_impl.cpp -> abi.StructOptOut (iters not observable)."""
    lib = load_ref(abi)
    lib.plsvo_ref_structopt_batch.restype = C.c_int
    lib.plsvo_ref_structopt_batch.argtypes = [C.POINTER(abi.StructOptBatch), C.POINTER(abi.StructOptResult)]
    b, keep = abi.make_structopt_batch(data)
    out = abi.StructOptOut(b.n_points, b.n_segs)
    rc = lib.plsvo_ref_structopt_batch(C.byref(b), C.byref(out.struct))
    if rc != 0:
        raise RuntimeError(f"reference structopt failed rc={rc}")
    return out


def seed_update(abi, data, n_threads: int = 1):
    """DepthFilter::updatePointSeeds body restated, over a synth.SeedData batch -> abi.SeedOut."""
    lib = load(abi)
    lib.plsvo_oracle_seed_update_batch.restype = C.c_int
    lib.plsvo_oracle_seed_update_batch.argtypes = [C.POINTER(abi.SeedBatch), C.POINTER(abi.SeedResult), C.c_int]
    b, keep = abi.make_seed_batch(data)
    out = abi.SeedOut(data.n)
    rc = lib.plsvo_oracle_seed_update_batch(C.byref(b), C.byref(out.struct), n_threads)
    if rc != 0:
        raise RuntimeError(f"oracle seed_update failed rc={rc}")
    return out


@_recorded
def ref_seed_update(abi, data):
    """DepthFilter::updatePointSeeds of the reference's own depth_filter.cpp + matcher.cpp -> abi.SeedOut
    (a, b, mu, sigma2 only; status is -1 where the reference erased the seed, 0 otherwise)."""
    lib = load_ref(abi)
    lib.plsvo_ref_seed_update_batch.restype = C.c_int
    lib.plsvo_ref_seed_update_batch.argtypes = [C.POINTER(abi.SeedBatch), C.POINTER(abi.SeedResult)]
    b, keep = abi.make_seed_batch(data)
    out = abi.SeedOut(data.n)
    rc = lib.plsvo_ref_seed_update_batch(C.byref(b), C.byref(out.struct))
    if rc != 0:
        raise RuntimeError(f"reference seed_update failed rc={rc}")
    return out


def line_seed_update(abi, data, n_threads: int = 1):
    """DepthFilter::updateLineSeeds body restated -> abi.LineSeedOut."""
    lib = load(abi)
    lib.plsvo_oracle_line_seed_update_batch.restype = C.c_int
    lib.plsvo_oracle_line_seed_update_batch.argtypes = [C.POINTER(abi.LineSeedBatch), C.POINTER(abi.LineSeedResult), C.c_int]
    b, keep = abi.make_line_seed_batch(data)
    out = abi.LineSeedOut(data.n)
    rc = lib.plsvo_oracle_line_seed_update_batch(C.byref(b), C.byref(out.line_struct), n_threads)
    if rc != 0:
        raise RuntimeError(f"oracle line_seed_update failed rc={rc}")
    return out


SEARCH_STATS_FIELDS = ("steps", "rejected", "level", "first_best", "last_best", "no_win")


def seed_search_stats(abi, data, n_threads: int = 1):
    """The restated point- or line-seed update (by the type of `data`) with a record of every epipolar ZMSSD search ->
    (abi.SeedOut or abi.LineSeedOut, stats).  stats is a dict of int32 arrays [n] (point seeds) or [n, 2] (line seeds: start
    point, end point), one per SEARCH_STATS_FIELDS: the step count n_steps + 1 (-1 where no search was reached), whether
    max_epi_search_steps rejected it, the search level, the first and the last step whose score equals the final best (-1:
    none), and whether no score beat PatchScore::threshold().  The outputs are those of seed_update / line_seed_update."""
    lib = load(abi)
    line = getattr(data, "ref_sf", None) is not None
    st = np.zeros((data.n, 2 if line else 1, len(SEARCH_STATS_FIELDS)), np.int32)
    ip = C.POINTER(C.c_int32)
    if line:
        fn = lib.plsvo_oracle_line_seed_search_stats
        fn.argtypes = [C.POINTER(abi.LineSeedBatch), C.POINTER(abi.LineSeedResult), ip, C.c_int]
        b, keep = abi.make_line_seed_batch(data)
        out = abi.LineSeedOut(data.n)
        res = out.line_struct
    else:
        fn = lib.plsvo_oracle_seed_search_stats
        fn.argtypes = [C.POINTER(abi.SeedBatch), C.POINTER(abi.SeedResult), ip, C.c_int]
        b, keep = abi.make_seed_batch(data)
        out = abi.SeedOut(data.n)
        res = out.struct
    fn.restype = C.c_int
    rc = fn(C.byref(b), C.byref(res), st.ctypes.data_as(ip), n_threads)
    if rc != 0:
        raise RuntimeError(f"oracle seed_search_stats failed rc={rc}")
    if not line:
        st = st[:, 0]
    return out, {k: np.ascontiguousarray(st[..., j]) for j, k in enumerate(SEARCH_STATS_FIELDS)}


@_recorded
def ref_line_seed_update(abi, data):
    """DepthFilter::updateLineSeeds of the reference's own depth_filter.cpp + matcher.cpp -> abi.LineSeedOut (state only)."""
    lib = load_ref(abi)
    lib.plsvo_ref_line_seed_update_batch.restype = C.c_int
    lib.plsvo_ref_line_seed_update_batch.argtypes = [C.POINTER(abi.LineSeedBatch), C.POINTER(abi.LineSeedResult)]
    b, keep = abi.make_line_seed_batch(data)
    out = abi.LineSeedOut(data.n)
    rc = lib.plsvo_ref_line_seed_update_batch(C.byref(b), C.byref(out.line_struct))
    if rc != 0:
        raise RuntimeError(f"reference line_seed_update failed rc={rc}")
    return out


def _optimize_structure(fn, abi, data, pt_last, seg_last, max_n_pts, max_n_segs, frame_id):
    from plsvo_b200 import abi as _abi  # noqa: F401

    batch, keep = abi.make_structopt_batch(data)
    out = abi.StructOptOut(data.pt_pos.shape[0], data.seg_spos.shape[0])
    pl = np.ascontiguousarray(pt_last, dtype=np.int32).copy()
    sl = np.ascontiguousarray(seg_last, dtype=np.int32).copy()
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(abi.StructOptBatch), C.POINTER(abi.StructOptResult), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                   C.c_int, C.c_int, C.c_int]
    rc = fn(C.byref(batch), C.byref(out.struct), pl.ctypes.data_as(C.POINTER(C.c_int32)), sl.ctypes.data_as(C.POINTER(C.c_int32)),
            max_n_pts, max_n_segs, frame_id)
    if rc != 0:
        raise RuntimeError(f"optimize_structure failed rc={rc}")
    return out, pl, sl


def ref_optimize_structure(abi, data, pt_last, seg_last, max_n_pts, max_n_segs, frame_id=77):
    """FrameHandlerBase::optimizeStructure with the reference's own Point::optimize / LineSeg::optimize (oracle/_ref)."""
    return _optimize_structure(load_ref(abi).plsvo_ref_optimize_structure, abi, data, pt_last, seg_last, max_n_pts, max_n_segs, frame_id)


def shimref_optimize_structure(abi, data, pt_last, seg_last, max_n_pts, max_n_segs, frame_id=77, cpu: bool = False):
    """The same call on reference-typed objects through the shim's plsvo::b200::optimizeStructure (C ABI: GPU, or the
    oracle-backed adapter with cpu=True)."""
    return _optimize_structure(load_shimref(abi, cpu).plsvo_shimref_optimize_structure, abi, data, pt_last, seg_last, max_n_pts,
                               max_n_segs, frame_id)


# ---- reference-typed scenes for the loops either side of the hot path (oracle/next_scenes.h) ---------------------------
class SceneMatchOut(C.Structure):
    _fields_ = [("pt_found", C.POINTER(C.c_uint8)), ("pt_px", C.POINTER(C.c_double)), ("pt_level", C.POINTER(C.c_int32)),
                ("pt_A", C.POINTER(C.c_double)), ("pt_ref", C.POINTER(C.c_int32)), ("seg_found", C.POINTER(C.c_uint8)),
                ("seg_spx", C.POINTER(C.c_double)), ("seg_epx", C.POINTER(C.c_double)), ("seg_level", C.POINTER(C.c_int32)),
                ("seg_A", C.POINTER(C.c_double)), ("seg_ref", C.POINTER(C.c_int32))]


class SceneSeedOut(C.Structure):
    _fields_ = [("pt_fate", C.POINTER(C.c_int32)), ("pt_state", C.POINTER(C.c_float)), ("pt_xyz", C.POINTER(C.c_double)),
                ("pt_cb_sigma2", C.POINTER(C.c_double)), ("n_pt_marks", C.POINTER(C.c_int32)), ("pt_marks", C.POINTER(C.c_double)),
                ("seg_fate", C.POINTER(C.c_int32)), ("seg_state", C.POINTER(C.c_float)), ("seg_xyz", C.POINTER(C.c_double)),
                ("seg_cb_sigma2", C.POINTER(C.c_double)), ("n_seg_marks", C.POINTER(C.c_int32)), ("seg_marks", C.POINTER(C.c_double))]


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class _Rec:
    pass


def _match_scene(fn, abi, data, n_obs):
    n, m = data.n, data.n // 2
    r = _Rec()
    r.pt_found, r.pt_px, r.pt_level = np.zeros(n, np.uint8), np.full((n, 2), np.nan), np.full(n, -99, np.int32)
    r.pt_A, r.pt_ref = np.full((n, 4), np.nan), np.full(n, -99, np.int32)
    r.seg_found, r.seg_spx, r.seg_epx = np.zeros(m, np.uint8), np.full((m, 2), np.nan), np.full((m, 2), np.nan)
    r.seg_level, r.seg_A, r.seg_ref = np.full(m, -99, np.int32), np.full((m, 4), np.nan), np.full(m, -99, np.int32)
    out = SceneMatchOut(_p(r.pt_found, C.c_uint8), _p(r.pt_px, C.c_double), _p(r.pt_level, C.c_int32), _p(r.pt_A, C.c_double),
                        _p(r.pt_ref, C.c_int32), _p(r.seg_found, C.c_uint8), _p(r.seg_spx, C.c_double), _p(r.seg_epx, C.c_double),
                        _p(r.seg_level, C.c_int32), _p(r.seg_A, C.c_double), _p(r.seg_ref, C.c_int32))
    b, keep = abi.make_match_batch(data)
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(abi.MatchBatch), C.c_int, C.POINTER(SceneMatchOut)]
    rc = fn(C.byref(b), n_obs, C.byref(out))
    if rc != 0:
        raise RuntimeError(f"match scene failed rc={rc}")
    return r


def ref_match_scene(abi, data, n_obs=3):
    """Reprojector-style pass with the reference's own Matcher::findMatchDirect + Point/LineSeg::getCloseViewObs (oracle/_ref)
    over map points / segments observed in n_obs keyframes."""
    return _match_scene(load_ref(abi).plsvo_ref_match_scene, abi, data, n_obs)


def shimref_match_scene(abi, data, n_obs=3, cpu: bool = False):
    """The same pass answered by plsvo::b200::DirectMatcher (one C-ABI call per frame: GPU, or the oracle-backed adapter)."""
    return _match_scene(load_shimref(abi, cpu).plsvo_shimref_match_scene, abi, data, n_obs)


def _seed_scene(fn, abi, pts, lines, pt_age, seg_age, is_keyframe):
    n, m = pts.n, (lines.n if lines is not None else 0)
    r = _Rec()
    r.pt_fate, r.pt_state, r.pt_xyz = np.full(n, -1, np.int32), np.full((n, 4), np.nan, np.float32), np.full((n, 3), np.nan)
    r.pt_cb_sigma2, r.n_pt_marks, r.pt_marks = np.full(n, np.nan), np.zeros(1, np.int32), np.full((n + 1, 2), np.nan)
    r.seg_fate, r.seg_state, r.seg_xyz = np.full(m + 1, -1, np.int32), np.full((m + 1, 6), np.nan, np.float32), np.full((m + 1, 6), np.nan)
    r.seg_cb_sigma2, r.n_seg_marks, r.seg_marks = np.full((m + 1, 2), np.nan), np.zeros(1, np.int32), np.full((m + 1, 4), np.nan)
    out = SceneSeedOut(_p(r.pt_fate, C.c_int32), _p(r.pt_state, C.c_float), _p(r.pt_xyz, C.c_double), _p(r.pt_cb_sigma2, C.c_double),
                       _p(r.n_pt_marks, C.c_int32), _p(r.pt_marks, C.c_double), _p(r.seg_fate, C.c_int32), _p(r.seg_state, C.c_float),
                       _p(r.seg_xyz, C.c_double), _p(r.seg_cb_sigma2, C.c_double), _p(r.n_seg_marks, C.c_int32), _p(r.seg_marks, C.c_double))
    pb, keep = abi.make_seed_batch(pts)
    lb, lkeep = abi.make_line_seed_batch(lines) if lines is not None else (None, None)
    pa = np.ascontiguousarray(pt_age, np.int32) if pt_age is not None else None
    sa = np.ascontiguousarray(seg_age, np.int32) if seg_age is not None else None
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(abi.SeedBatch), C.POINTER(abi.LineSeedBatch), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int,
                   C.POINTER(SceneSeedOut)]
    rc = fn(C.byref(pb), C.byref(lb) if lb is not None else None, _p(pa, C.c_int32) if pa is not None else None,
            _p(sa, C.c_int32) if sa is not None else None, int(is_keyframe), C.byref(out))
    if rc != 0:
        raise RuntimeError(f"seed scene failed rc={rc}")
    r.seg_fate, r.seg_state, r.seg_xyz, r.seg_cb_sigma2 = r.seg_fate[:m], r.seg_state[:m], r.seg_xyz[:m], r.seg_cb_sigma2[:m]
    r.pt_marks, r.seg_marks = r.pt_marks[: r.n_pt_marks[0]], r.seg_marks[: r.n_seg_marks[0]]
    return r


def ref_seed_scene(abi, pts, lines=None, pt_age=None, seg_age=None, is_keyframe=False):
    """DepthFilter::updateSeeds of the reference's own depth_filter.cpp (real ageing, convergence, callbacks, detector marks)."""
    return _seed_scene(load_ref(abi).plsvo_ref_seed_scene, abi, pts, lines, pt_age, seg_age, is_keyframe)


def shimref_seed_scene(abi, pts, lines=None, pt_age=None, seg_age=None, is_keyframe=False, cpu: bool = False):
    """The same update through plsvo::b200::DepthFilterB200 (two C-ABI calls per frame: GPU, or the oracle-backed adapter)."""
    return _seed_scene(load_shimref(abi, cpu).plsvo_shimref_seed_scene, abi, pts, lines, pt_age, seg_age, is_keyframe)


def last_loop_seconds(abi, shim: bool, cpu: bool = False) -> float:
    """Wall-clock seconds of the loop under test in the last *_match_scene / *_seed_scene call (scene construction excluded)."""
    if shim:
        fn = load_shimref(abi, cpu).plsvo_shimref_last_loop_seconds
    else:
        fn = load_ref(abi).plsvo_ref_last_loop_seconds
    fn.restype = C.c_double
    fn.argtypes = []
    return float(fn())
