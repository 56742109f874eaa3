/*
 * plsvo_b200.h — C ABI of the H100-native (sm_90a) PL-SVO per-frame optimisation path.
 *
 * Two entry-point families, one per reference symbol they replace:
 *
 *   plsvo_align_*    replaces  plsvo::SparseImgAlign::run()
 *                    (reference: include/plsvo/sparse_img_align.h:56-70,
 *                     src/sparse_img_align.cpp:54-95; call sites
 *                     src/frame_handler_mono.cpp:272-274 and :418-420)
 *   plsvo_poseopt_*  replaces  plsvo::pose_optimizer::optimizeGaussNewton()
 *                    (reference: include/plsvo/pose_optimizer.h:47-64,
 *                     src/pose_optimizer.cpp:38-260 (9-arg) and :262-582 (10-arg);
 *                     call site src/frame_handler_mono.cpp:327-329)
 *
 * The reference has no FFI layer: its boundary is two C++ link-time symbols that take
 * boost::shared_ptr<Frame>.  The C++ shim in pl-svo_b200/host/ keeps those two signatures
 * and packs Frame / Feature lists into the flat arrays declared here (INTEGRATION.md).
 *
 * Conventions
 *   - plain C types only, caller-allocated outputs, int return codes, no exceptions.
 *   - a batch is B independent frame pairs (align) or B independent frames (pose-opt).
 *   - SE3 poses are 7 doubles {qx,qy,qz,qw,tx,ty,tz}: the unit quaternion (Eigen coeffs()
 *     order) and translation that the reference's Sophus::SE3 stores (include/plsvo/frame.h:62).
 *   - 6x6 matrices are 36 doubles (symmetric, so row/column order is immaterial).
 *   - every call is stream-ordered on the context's stream; *_download and *_batch
 *     synchronise before returning.
 *   - there is NO CPU fallback: without a CUDA device every call returns PLSVO_ERR_NO_DEVICE.
 */
#ifndef PLSVO_B200_H_
#define PLSVO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PLSVO_MAX_LEVELS 8   /* pyramid levels addressable through the ABI (reference uses 5) */
#define PLSVO_PATCH_AREA 16  /* 4x4 patch, include/plsvo/sparse_img_align.h:48-50 */

/* return codes */
#define PLSVO_OK 0
#define PLSVO_ERR_INVALID (-1)    /* bad argument / inconsistent batch description */
#define PLSVO_ERR_CUDA (-2)       /* CUDA runtime error, see plsvo_last_error() */
#define PLSVO_ERR_NO_DEVICE (-3)  /* no usable CUDA device: there is no CPU path */
#define PLSVO_ERR_STATE (-4)      /* launch/download without a prior upload */

typedef struct plsvo_ctx plsvo_ctx;

/* Undistorted pinhole camera: what vk::PinholeCamera::world2cam / errorMultiplier2 /
 * isInFrame use when the handler is given the undistorted model (app/run_pipeline.cpp:786-795). */
typedef struct plsvo_camera {
  int32_t width, height; /* level-0 image size */
  int32_t reserved0, reserved1;
  double fx, fy, cx, cy;
} plsvo_camera;

/* ------------------------------------------------------------------------------------------
 * Sparse image alignment
 * ---------------------------------------------------------------------------------------- */

/* SparseImgAlign constructor arguments (src/sparse_img_align.cpp:40-52); defaults at the call
 * site are max_level=4, min_level=2, n_iter=30 (src/frame_handler_mono.cpp:272-273,
 * src/config.cpp:98-99); eps is hard-coded 1e-6 in the reference (:51). */
typedef struct plsvo_align_params {
  int32_t max_level;
  int32_t min_level;
  int32_t n_iter;
  int32_t reserved;
  double eps;
} plsvo_align_params;

/* One batch of B frame pairs.  All pairs share the camera (plsvo_align_multicam_batch_run below takes pinhole intrinsics
 * per pair) and the array strides n_pts/n_segs;
 * per-pair feature counts may be smaller (pt_count/seg_count) and individual features may be
 * flagged invalid (feat3D == NULL in the reference).
 *
 * Images: for pyramid level l in [min_level,max_level], image of pair b starts at
 * ref_img[l] + b*img_stride[l] with row pitch img_pitch[l] bytes and (width>>l) x (height>>l)
 * u8 pixels (Frame::img_pyr_, include/plsvo/frame.h:64).  Levels outside the range may be NULL.
 * Levels ABOVE the lowest provided one may also be NULL inside the range: they are then derived on the device by
 * repeated vk::halfSample (the truncating 2x2 mean of frame_utils::createImgPyramid, src/frame.cpp:171-180 —
 * bit-identical to the host pyramid), which saves their host->device copy; this needs 16-byte aligned, 16-byte
 * pitched rows of the source level.
 *
 * The reference only ever uses the distance of a 3-D feature from the reference camera centre
 * (`(pos_ - ref_pos).norm()`, sparse_img_align.cpp:229,337-340).  A caller that already holds these distances may pass
 * them in pt_depth / seg_sdepth / seg_edepth and leave pt_pos / seg_spos / seg_epos NULL (16 bytes less per point,
 * 32 per segment over PCIe).
 *
 * pt_f / seg_sf / seg_ef may be NULL when the camera is the undistorted pinhole `cam`: the bearing vectors are then
 * formed on the device exactly as the reference's feature constructors form them, `cam_->cam2world(px)`
 * (src/feature.cpp:42,98-99; vk::PinholeCamera::cam2world = ((u-cx)/fx, (v-cy)/fy, 1).normalized()).  24 bytes less
 * per point, 48 per segment.
 *
 * Frame chains (flags & PLSVO_ALIGN_FRAME_CHAIN).  FrameHandlerMono aligns consecutive frames: the current frame of
 * one call is the reference frame of the next (src/frame_handler_mono.cpp:272 `run(last_frame_, new_frame_)`, :176
 * `last_frame_ = new_frame_`).  A batch that replays such a sequence — pair b = (frame b, frame b+1) — gives
 * ref_img[l] as a stack of B+1 frames (frame k at ref_img[l] + k*img_stride[l]) and leaves cur_img[l] NULL: every
 * frame crosses the host link and sits in device memory once instead of twice (B+1 frames instead of 2B).  Everything
 * else (poses, the features of each pair's reference frame, outputs) is per pair as before; results are bit-identical
 * to the same batch given as two stacks.
 */
#define PLSVO_ALIGN_FRAME_CHAIN 1 /* plsvo_align_batch.flags: ref_img holds B+1 chained frames, cur_img is ignored */

typedef struct plsvo_align_batch {
  int32_t batch;   /* B */
  int32_t n_pts;   /* array stride: points per pair   (Frame::pt_fts_,  frame.h:65) */
  int32_t n_segs;  /* array stride: segments per pair (Frame::seg_fts_, frame.h:66) */
  int32_t flags;   /* 0 or PLSVO_ALIGN_FRAME_CHAIN (was `reserved`: zero keeps the two-stack layout) */
  plsvo_camera cam;

  const uint8_t* ref_img[PLSVO_MAX_LEVELS];
  const uint8_t* cur_img[PLSVO_MAX_LEVELS];
  size_t img_pitch[PLSVO_MAX_LEVELS];
  size_t img_stride[PLSVO_MAX_LEVELS];

  const double* T_ref_w; /* [B][7]  ref_frame->T_f_w_ */
  const double* T_cur_w; /* [B][7]  cur_frame->T_f_w_ on entry (initial guess) */

  const int32_t* pt_count;  /* [B] or NULL (= n_pts)  : pt_fts_.size() */
  const double* pt_px;      /* [B][n_pts][2]  PointFeat::px  (level-0 pixels) */
  const double* pt_f;       /* [B][n_pts][3]  PointFeat::f   (unit bearing), or NULL = cam2world(px) */
  const double* pt_pos;     /* [B][n_pts][3]  PointFeat::feat3D->pos_ (world) */
  const uint8_t* pt_valid;  /* [B][n_pts] or NULL (= all valid): feat3D != NULL */

  const int32_t* seg_count; /* [B] or NULL (= n_segs) : seg_fts_.size() */
  const double* seg_spx;    /* [B][n_segs][2] LineFeat::spx */
  const double* seg_epx;    /* [B][n_segs][2] LineFeat::epx */
  const double* seg_sf;     /* [B][n_segs][3] LineFeat::sf, or NULL = cam2world(spx) */
  const double* seg_ef;     /* [B][n_segs][3] LineFeat::ef, or NULL = cam2world(epx) */
  const double* seg_spos;   /* [B][n_segs][3] LineFeat::feat3D->spos_ */
  const double* seg_epos;   /* [B][n_segs][3] LineFeat::feat3D->epos_ */
  const double* seg_length; /* [B][n_segs]    LineFeat::length */
  const uint8_t* seg_valid; /* [B][n_segs] or NULL: feat3D != NULL */

  const double* pt_depth;   /* [B][n_pts]  or NULL: |pos_ - ref_frame->pos()| (then pt_pos may be NULL) */
  const double* seg_sdepth; /* [B][n_segs] or NULL: |spos_ - ref_frame->pos()| (then seg_spos may be NULL) */
  const double* seg_edepth; /* [B][n_segs] or NULL: |epos_ - ref_frame->pos()| (then seg_epos may be NULL) */
} plsvo_align_batch;

/* Caller-allocated outputs; any pointer may be NULL to skip that output. */
typedef struct plsvo_align_result {
  double* T_cur_w;        /* [B][7]  cur_frame->T_f_w_ on return (sparse_img_align.cpp:92) */
  int64_t* n_tracked;     /* [B]     return value of run(): n_meas_/16 (:94) */
  double* H;              /* [B][36] H_ of the last evaluated iteration (getFisherInformation, :97-102) */
  uint8_t* seg_killed;    /* [B][n_segs] 1 where the reference sets ref seg feat3D = NULL (:687-688) */
  int32_t* iters;         /* [B][PLSVO_MAX_LEVELS] residual passes executed at each level (index = level) */
  int32_t* status;        /* [B] bit0: early-out "no features" (:58-62); bit1: solver stop_ was raised */
  uint32_t* patch_iters;  /* [B] sum over executed passes of patches evaluated (roofline accounting) */
  uint32_t* patch_levels; /* [B] sum over levels of patches precomputed (roofline accounting) */
} plsvo_align_result;

/* ------------------------------------------------------------------------------------------
 * Pose optimiser
 * ---------------------------------------------------------------------------------------- */

/* Arguments of pose_optimizer::optimizeGaussNewton (pose_optimizer.h:47-64); defaults
 * reproj_thresh=2.0, n_iter=10, n_iter_ref=3 (src/config.cpp:102-104).  n_iter_ref < 0
 * selects the 9-argument overload (no refinement loop). */
typedef struct plsvo_poseopt_params {
  double reproj_thresh;
  int32_t n_iter;
  int32_t n_iter_ref;
} plsvo_poseopt_params;

typedef struct plsvo_poseopt_batch {
  int32_t batch;   /* B frames */
  int32_t n_pts;   /* array stride */
  int32_t n_segs;  /* array stride */
  int32_t reserved;
  double fx;       /* frame->cam_->errorMultiplier2() */

  const double* T_f_w;      /* [B][7] frame->T_f_w_ on entry */

  const int32_t* pt_count;  /* [B] or NULL */
  const double* pt_f;       /* [B][n_pts][3]  PointFeat::f */
  const double* pt_pos;     /* [B][n_pts][3]  feat3D->pos_ */
  const int32_t* pt_level;  /* [B][n_pts]     Feature::level */
  const uint8_t* pt_valid;  /* [B][n_pts] or NULL */

  const int32_t* seg_count; /* [B] or NULL */
  const double* seg_line;   /* [B][n_segs][3] LineFeat::line */
  const double* seg_spos;   /* [B][n_segs][3] feat3D->spos_ */
  const double* seg_epos;   /* [B][n_segs][3] feat3D->epos_ */
  const int32_t* seg_level; /* [B][n_segs] */
  const uint8_t* seg_valid; /* [B][n_segs] or NULL */
} plsvo_poseopt_batch;

typedef struct plsvo_poseopt_result {
  double* T_f_w;            /* [B][7]  frame->T_f_w_ on return */
  double* cov;              /* [B][36] frame->Cov_ (pose_optimizer.cpp:199) */
  double* estimated_scale;  /* [B] */
  double* error_init;       /* [B] */
  double* error_final;      /* [B] */
  int64_t* num_obs_pt;      /* [B] */
  int64_t* num_obs_ls;      /* [B] */
  uint8_t* pt_outlier;      /* [B][n_pts]  1 where the reference sets feat3D = NULL (:218) */
  uint8_t* seg_outlier;     /* [B][n_segs] (:239) */
  int32_t* iters;           /* [B][2] GN passes executed in the main / refinement loop */
  int32_t* status;          /* [B] bit0: early return "no observations" (:88-89), outputs untouched */
} plsvo_poseopt_result;

/* ------------------------------------------------------------------------------------------
 * Context, memory, execution
 * ---------------------------------------------------------------------------------------- */

/* device: CUDA ordinal.  stream: a cudaStream_t to run on, or NULL to create a private one. */
int plsvo_ctx_create(int device, void* stream, plsvo_ctx** out);
void plsvo_ctx_destroy(plsvo_ctx* ctx);
/* last error text of this context (or of ctx creation when ctx == NULL) */
const char* plsvo_last_error(const plsvo_ctx* ctx);
/* the cudaStream_t all work of this context is ordered on */
void* plsvo_ctx_stream(plsvo_ctx* ctx);
int plsvo_sync(plsvo_ctx* ctx);

/* page-locked host memory for batch arrays (keeps the H2D/D2H legs at PCIe speed) */
int plsvo_host_alloc(void** ptr, size_t bytes);
int plsvo_host_free(void* ptr);

/* Alignment.  upload: host arrays -> device layout (async).  launch: the whole coarse-to-fine
 * optimisation of every pair, device-resident in and out (async).  download: device -> host
 * outputs, then synchronise.  plsvo_align_batch_run = upload + launch + download.
 * Every one-call form (plsvo_*_batch_run) has finished with the caller's arrays when it returns, whatever it returns:
 * an error found after copies had been queued first drains every stream of the context. */
int plsvo_align_upload(plsvo_ctx* ctx, const plsvo_align_batch* batch);
int plsvo_align_launch(plsvo_ctx* ctx, const plsvo_align_params* params);
int plsvo_align_download(plsvo_ctx* ctx, const plsvo_align_result* out);
int plsvo_align_batch_run(plsvo_ctx* ctx, const plsvo_align_batch* batch,
                          const plsvo_align_params* params, const plsvo_align_result* out);

/* Pose optimiser, same three legs. */
int plsvo_poseopt_upload(plsvo_ctx* ctx, const plsvo_poseopt_batch* batch);
int plsvo_poseopt_launch(plsvo_ctx* ctx, const plsvo_poseopt_params* params);
int plsvo_poseopt_download(plsvo_ctx* ctx, const plsvo_poseopt_result* out);
int plsvo_poseopt_batch_run(plsvo_ctx* ctx, const plsvo_poseopt_batch* batch,
                            const plsvo_poseopt_params* params, const plsvo_poseopt_result* out);

/* The two hot-path calls of FrameHandlerMono::processFrame back to back (src/frame_handler_mono.cpp:272-274 sparse
 * image alignment, :327-329 pose optimisation) for a batch of frames, with the pose staying on the device in between:
 * frame b of `po_batch` starts from the alignment result of pair b of `al_batch` when po_batch->T_f_w is NULL
 * (otherwise from the poses given).  `al_out` may be NULL.  Equivalent to plsvo_align_batch_run followed by
 * plsvo_poseopt_batch_run with T_f_w = the aligned poses, minus one device->host->device trip and one sync.
 * plsvo_track_upload / plsvo_track_launch are its two device-side legs (results: plsvo_align_download and
 * plsvo_poseopt_download). */
int plsvo_track_upload(plsvo_ctx* ctx, const plsvo_align_batch* al_batch, const plsvo_poseopt_batch* po_batch);
int plsvo_track_launch(plsvo_ctx* ctx, const plsvo_align_params* al_params, const plsvo_poseopt_params* po_params);
int plsvo_track_batch_run(plsvo_ctx* ctx, const plsvo_align_batch* al_batch, const plsvo_align_params* al_params,
                          const plsvo_poseopt_batch* po_batch, const plsvo_poseopt_params* po_params,
                          const plsvo_align_result* al_out, const plsvo_poseopt_result* po_out);

/* ------------------------------------------------------------------------------------------
 * Image pyramid (SURVEY.md §8f "next", rank 2): frame_utils::createImgPyramid, src/frame.cpp:171-180,
 * i.e. repeated vk::halfSample (truncating 2x2 mean), for B frames.  Host in, host out.
 * level[0] of the result may be NULL (level 0 is the input); n_levels <= 7.
 * ---------------------------------------------------------------------------------------- */
typedef struct plsvo_pyramid_batch {
  int32_t batch, width, height, n_levels;
  const uint8_t* img0; /* [B] level-0 images: image b at img0 + b*stride0, rows pitch0 bytes */
  size_t pitch0, stride0;
} plsvo_pyramid_batch;

typedef struct plsvo_pyramid_result {
  uint8_t* level[PLSVO_MAX_LEVELS]; /* caller-allocated; level l holds (width>>l) x (height>>l) pixels */
  size_t pitch[PLSVO_MAX_LEVELS];
  size_t stride[PLSVO_MAX_LEVELS];
} plsvo_pyramid_result;

int plsvo_pyramid_batch_run(plsvo_ctx* ctx, const plsvo_pyramid_batch* in, const plsvo_pyramid_result* out);

/* ------------------------------------------------------------------------------------------
 * Frame rectification: vk::PinholeCamera::undistortImage (rpg_vikit pinhole_camera.cpp), as app/run_pipeline.cpp
 * calls it on every raw frame before FrameHandlerMono::addImage, for B frames, followed by createImgPyramid.
 * The camera carries the distorted vk::PinholeCamera constructor arguments.  As there, fabs(d0) <= 1e-7 means no
 * distortion (the frame is copied, whatever d1..d4 are); otherwise the map is cv::initUndistortRectifyMap of the
 * float-rounded K and (k1,k2,p1,p2,k3) = (d0..d4), CV_16SC2, and each frame is cv::remap(raw, rect, map1, map2,
 * INTER_LINEAR) with a constant border of 0 — bit-identical to OpenCV's fixed-point path.
 * The map is built on the device once per camera and cached in the context; a call with another camera (or image
 * size) rebuilds it.  Host in, host out, synchronous.  level[0] of the result is required and receives the
 * rectified frame; levels 1..n_levels-1 are its half-sampled pyramid (as plsvo_pyramid_batch_run); n_levels <= 7.
 * ---------------------------------------------------------------------------------------- */
typedef struct plsvo_pinhole_camera {
  int32_t width, height;
  double fx, fy, cx, cy;
  double d[5]; /* d0..d4 = k1, k2, p1, p2, k3 */
} plsvo_pinhole_camera;

typedef struct plsvo_undistort_batch {
  plsvo_pinhole_camera cam;
  int32_t batch, n_levels;
  const uint8_t* img0; /* [B] raw frames of cam.width x cam.height: frame b at img0 + b*stride0, rows pitch0 bytes */
  size_t pitch0, stride0;
} plsvo_undistort_batch;

int plsvo_undistort_batch_run(plsvo_ctx* ctx, const plsvo_undistort_batch* in, const plsvo_pyramid_result* out);

/* device time (CUDA events) of the map build the last plsvo_undistort_batch_run call made, or -1 in *ms when that
 * call reused the context's cached map or needed none (d0 = 0).  After a raw multicam call: the time of all the map
 * builds it made.  plsvo_last_kernel_ms never includes it. */
int plsvo_last_map_build_ms(plsvo_ctx* ctx, float* ms);

/* ------------------------------------------------------------------------------------------
 * Alignment and tracking of raw frames: plsvo_undistort_batch_run followed by plsvo_align_batch_run /
 * plsvo_track_batch_run in one call, without the rectified pyramid leaving the device.  One kernel rectifies each frame
 * (the context's cached map, as plsvo_undistort_batch_run) and half-samples it, and stores only the levels alignment
 * reads plus those asked for in rect_out.  Results are byte-identical to the two calls chained through the host, with
 * plsvo_align_batch_run / plsvo_track_batch_run on their plain upload -> launch -> download sequence (the one they take
 * below 256 pairs; the arrival-gated path they take for larger batches uses another CTA shape and agrees to round-off).
 * The raw calls always take the plain sequence.
 *
 * - `batch` describes features, poses and the UNDISTORTED camera exactly as for plsvo_align_batch_run; every
 *   ref_img[l] / cur_img[l] must be NULL (the images come from `raw`).  batch->cam must equal raw->cam in width, height,
 *   fx, fy, cx and cy (run_pipeline builds both cameras from the same values).  flags = PLSVO_ALIGN_FRAME_CHAIN takes
 *   B+1 raw frames in ref_raw, pair b = (frame b, frame b+1), and cur_raw must be NULL.
 * - fabs(raw->cam.d[0]) <= 1e-7 means no distortion: the raw frame is level 0 as it is.
 * - max_level <= 6 (one 64x64 level-0 tile per CTA holds levels 0..6).
 * - rect_out may be NULL.  Each non-NULL rect_out->level[l] (l <= 6) receives rectified level l of every frame in stack
 *   order: the B+1 frames of a chain, or the B reference frames followed by the B current frames.  Levels left NULL are
 *   not copied back, and not written at all unless alignment reads them.
 * - Malformed input (K mismatch, image pointers in `batch`, a NULL raw stack, cur_raw with a chain, pitch < width,
 *   non-finite parameters or zero fx / fy after rounding to float, max_level > 6, a rect_out level too narrow or smaller
 *   than one pixel) returns PLSVO_ERR_INVALID with a message.  As every one-call form, these have finished with the
 *   caller's arrays when they return, whatever they return.
 * - plsvo_last_kernel_ms covers the rectify + pyramid kernel and the alignment (and pose-optimiser) kernels;
 *   plsvo_last_map_build_ms reports a map build this call made.
 * ---------------------------------------------------------------------------------------- */
typedef struct plsvo_raw_frames {
  plsvo_pinhole_camera cam; /* the distorted camera; d0..d4 as for plsvo_undistort_batch */
  const uint8_t* ref_raw;   /* [B] raw frames of cam.width x cam.height, or [B+1] with PLSVO_ALIGN_FRAME_CHAIN */
  const uint8_t* cur_raw;   /* [B] raw frames; must be NULL with PLSVO_ALIGN_FRAME_CHAIN */
  size_t pitch, stride;     /* host layout of both stacks: frame k at ref_raw + k*stride, rows pitch bytes */
} plsvo_raw_frames;

int plsvo_align_raw_batch_run(plsvo_ctx* ctx, const plsvo_raw_frames* raw, const plsvo_align_batch* batch,
                              const plsvo_align_params* params, const plsvo_align_result* out,
                              const plsvo_pyramid_result* rect_out);
int plsvo_track_raw_batch_run(plsvo_ctx* ctx, const plsvo_raw_frames* raw, const plsvo_align_batch* al_batch,
                              const plsvo_align_params* al_params, const plsvo_poseopt_batch* po_batch,
                              const plsvo_poseopt_params* po_params, const plsvo_align_result* al_out,
                              const plsvo_poseopt_result* po_out, const plsvo_pyramid_result* rect_out);

/* ------------------------------------------------------------------------------------------
 * Raw frames from differently calibrated distorted cameras in one batch: the raw-frame calls above with the multicam
 * calls' per-pair intrinsics below.  cams[k] are distorted vk::PinholeCamera arguments (d0..d4 as for
 * plsvo_undistort_batch); both frames of pair b are rectified with cams[cam_of_pair[b]], and the pair is then aligned
 * with that camera's fx, fy, cx, cy as its undistorted intrinsics (run_pipeline builds both cameras from the same
 * values).  In the track call frame b's errorMultiplier2 is |fx| of that camera.  Of batch->cam only width and height
 * are used: they are the slot.
 * - Slot: every frame of both raw stacks, and of every rect_out level, occupies a slot of batch->cam's size (the raw
 *   stacks at `pitch` and `stride`).  A camera may be smaller than the slot in either dimension: its frames are its
 *   width x height in the top-left corner of their slots, at level l (width >> l) x (height >> l).  Raw bytes outside
 *   that region are never read; cv::remap's constant border applies at the camera's own size.
 * - Pair b's outputs are byte for byte those of plsvo_align_raw_batch_run / plsvo_track_raw_batch_run on that pair with
 *   raw->cam = cams[cam_of_pair[b]], batch->cam carrying its intrinsics, and the same kernel variant.
 * - rect_out as for the raw calls: every non-NULL level, the B reference frames followed by the B current frames, each
 *   rectified with its own camera (plsvo_undistort_batch_run of that frame at the camera's size) in its slot's region,
 *   the rest of the slot 0.  Cameras with fabs(d0) <= 1e-7 copy the frame and may be mixed with distorted ones.
 * - The maps are built on the device once per camera and kept in a cache of the context separate from the one-camera
 *   cache of plsvo_undistort_batch_run and the raw calls: after a call it holds the maps of exactly the distorted cameras
 *   that call referenced (equal cameras, byte for byte, share one map).  plsvo_last_map_build_ms reports the device time
 *   of the builds the call made, or -1 when it made none.
 * - n_cams < 1, NULL cams or cam_of_pair, an index outside [0, n_cams), a camera wider or taller than batch->cam, or
 *   below 1 pixel in either dimension, or whose parameters plsvo_undistort_batch_run rejects, a level (aligned or asked
 *   of rect_out) smaller than one pixel for a camera some pair references, PLSVO_ALIGN_FRAME_CHAIN (a chained frame
 *   belongs to two pairs), and everything the raw calls reject return PLSVO_ERR_INVALID before anything is queued.  A library built without the
 *   multicam kernels returns PLSVO_ERR_CUDA.  The calls always run upload -> launch -> download and have finished with
 *   the caller's arrays when they return, whatever they return.
 * - Lenses and ATAN (FOV) cameras in one batch: plsvo_*_raw_any_camera_batch_run below.
 * - Out of scope: a ragged (unpadded) frame layout, frame chains, the arrival-gated path.
 * ---------------------------------------------------------------------------------------- */
typedef struct plsvo_raw_multicam_frames {
  int32_t n_cams, reserved;
  const plsvo_pinhole_camera* cams; /* [n_cams] distorted cameras (d0..d4 as plsvo_undistort_batch), each fits the slot */
  const int32_t* cam_of_pair;       /* [B] index into cams: the camera of both frames of pair b */
  const uint8_t* ref_raw;           /* [B] raw frames, one slot (batch->cam's size) each */
  const uint8_t* cur_raw;           /* [B] raw frames, one slot (batch->cam's size) each */
  size_t pitch, stride;             /* host layout of both stacks, as plsvo_raw_frames */
} plsvo_raw_multicam_frames;

int plsvo_align_raw_multicam_batch_run(plsvo_ctx* ctx, const plsvo_raw_multicam_frames* raw, const plsvo_align_batch* batch,
                                       const plsvo_align_params* params, const plsvo_align_result* out,
                                       const plsvo_pyramid_result* rect_out);
int plsvo_track_raw_multicam_batch_run(plsvo_ctx* ctx, const plsvo_raw_multicam_frames* raw,
                                       const plsvo_align_batch* al_batch, const plsvo_align_params* al_params,
                                       const plsvo_poseopt_batch* po_batch, const plsvo_poseopt_params* po_params,
                                       const plsvo_align_result* al_out, const plsvo_poseopt_result* po_out,
                                       const plsvo_pyramid_result* rect_out);

/* ------------------------------------------------------------------------------------------
 * Alignment and tracking of frames from an ATAN (FOV) camera: vk::ATANCamera, the model app/run_pipeline.cpp builds when
 * cam_model selects it.  On that path the frames are not rectified: SparseImgAlign projects every patch through the
 * distorted model (cam_->world2cam, src/sparse_img_align.cpp:425,584) and the feature constructors form bearings with
 * its cam2world.  These calls are plsvo_align_batch_run / plsvo_track_batch_run with that camera model.
 *
 * plsvo_atan_camera holds the constructor's arguments ATANCamera(width, height, fx, fy, cx, cy, d0), fx..cy normalised
 * by the image size.  The library derives the rest as the constructor does: fx_ = width fx, fy_ = height fy,
 * cx_ = cx width - 0.5, cy_ = cy height - 0.5, s_ = d0, tans_ = 2 tan(s_/2) (no distortion when s_ == 0), and
 *   world2cam(uv): r = |uv|, factor = (r < 0.001 || s_ == 0) ? 1 : atan(r tans_) / (s_ r), px = (cx_ + fx_ factor u, ...)
 *   cam2world(px): d = ((x - cx_)/fx_, (y - cy_)/fy_), r = s_ ? tan(|d| s_) / tans_ : |d|,
 *                  (factor d, 1).normalized() with factor = |d| > 0.01 ? r / |d| : 1
 *   errorMultiplier2() = fx_.
 * - `batch` (al_batch) is as for plsvo_align_batch_run, including frame chains, NULL bearings (formed on the device with
 *   the ATAN cam2world) and NULL levels derived on the device.  batch->cam.width / height must equal the camera's; its
 *   other fields are ignored.
 * - The pose optimiser is camera-free: po_batch->fx is errorMultiplier2() = fx_ = width fx.
 * - These calls always run upload -> launch -> download on the context's stream, as the raw-frame calls do: the
 *   arrival-gated path plsvo_align_batch_run takes for 256 pairs and more is not used.
 * - A size mismatch, a non-finite parameter, fx <= 0 or fy <= 0 returns PLSVO_ERR_INVALID before anything is queued.
 *   A library built without the ATAN kernels returns PLSVO_ERR_CUDA.
 * ---------------------------------------------------------------------------------------- */
typedef struct plsvo_atan_camera {
  int32_t width, height;
  double fx, fy, cx, cy, d0;
} plsvo_atan_camera;

int plsvo_align_atan_batch_run(plsvo_ctx* ctx, const plsvo_atan_camera* cam, const plsvo_align_batch* batch,
                               const plsvo_align_params* params, const plsvo_align_result* out);
int plsvo_track_atan_batch_run(plsvo_ctx* ctx, const plsvo_atan_camera* cam, const plsvo_align_batch* al_batch,
                               const plsvo_align_params* al_params, const plsvo_poseopt_batch* po_batch,
                               const plsvo_poseopt_params* po_params, const plsvo_align_result* al_out,
                               const plsvo_poseopt_result* po_out);

/* ------------------------------------------------------------------------------------------
 * Multicam batches: frame pairs from differently calibrated undistorted pinhole cameras in one call, e.g. a fleet of
 * identical sensors with individual calibrations, or a mix of datasets and image sizes.  These are
 * plsvo_align_batch_run / plsvo_poseopt_batch_run / plsvo_track_batch_run with the intrinsics and image size taken per
 * pair.
 * - Slot: of batch->cam only width and height are used; they are the slot.  Every pair's frames occupy slots of that
 *   size in the image stacks, at the batch's pitches and strides.  Pair b's frames are cams[b].width x cams[b].height
 *   in the top-left corner of their slots, at level l (width >> l) x (height >> l).  cams[b] may be smaller than the
 *   slot in either dimension; the bytes outside its region (the padding) are never read in a way that reaches a
 *   result.  Levels derived on the device need no care: the truncating 2x2 mean keeps the region.  In a frame chain
 *   pairs b and b+1 share a frame, so cams[b] and cams[b+1] must have one size.
 * - Alignment: pair b uses cams[b].fx, fy, cx, cy wherever plsvo_align_batch_run uses batch->cam's: world2cam, cam2world
 *   of bearings not shipped, and the Jacobian factor |fx| / 2^level; and cams[b]'s size wherever it uses the image
 *   size.  Everything else of `batch` is as for plsvo_align_batch_run: full or
 *   lean bearings, depths, ragged counts and masks, PLSVO_ALIGN_FRAME_CHAIN, NULL levels derived on the device, every
 *   kernel variant (PLSVO_VARIANT).  Pair b's outputs are byte for byte those of plsvo_align_batch_run on the same pair
 *   with batch->cam = cams[b] (its frames cut out of the slots) and the same kernel variant.  The slot size enters the
 *   shared-memory plan, so the variant a call picks may differ from that of the one-camera call: pin it to compare.
 * - Pose optimiser: frame b uses fx[b] (its errorMultiplier2) wherever plsvo_poseopt_batch_run uses batch->fx; the
 *   track call uses |cams[b].fx|, vk::PinholeCamera::errorMultiplier2().  po_batch->fx is ignored by both.
 * - These calls always run upload -> launch -> download on the context's stream, as the ATAN and raw-frame calls do
 *   (not the arrival-gated path), and have finished with the caller's arrays when they return, whatever they return.
 * - NULL cams or fx, a cams[b] wider or taller than batch->cam or below 1 pixel in either dimension, a level (shipped, or
 *   up to max_level) smaller than one pixel for a cams[b], a frame chain whose size changes between consecutive pairs,
 *   a non-finite fx, fy, cx or cy, fx or fy equal to 0,
 *   a non-finite or non-positive fx[b], or (track) batch sizes that differ return PLSVO_ERR_INVALID before anything is
 *   queued.  A library built without the multicam kernels returns PLSVO_ERR_CUDA.
 * - The multicam kernels keep the pair's intrinsics in 128 bytes of shared memory per CTA.  A batch whose shared-memory
 *   plan lies within that of the limit is planned for the next kernel variant, as any batch that does not fit; with no
 *   variant left, or PLSVO_VARIANT pinned, it returns PLSVO_ERR_INVALID (DESIGN.md §4.11).
 * - Raw frames: plsvo_*_raw_multicam_batch_run above.
 * - ATAN (FOV) cameras per pair: plsvo_*_atan_multicam_batch_run below.  Pinhole and ATAN pairs in one batch:
 *   plsvo_*_any_camera_batch_run below.
 * - Out of scope: a ragged (unpadded) frame layout, the arrival-gated streamed path, separate upload / launch / download legs, dist.align_sharded, the seed updates
 *   and the drop-in shim (one frame per call, nothing to batch).  Direct matching with a camera per image:
 *   plsvo_match_direct_multicam_batch_run.
 * ---------------------------------------------------------------------------------------- */
int plsvo_align_multicam_batch_run(plsvo_ctx* ctx, const plsvo_camera* cams /* [B] */, const plsvo_align_batch* batch,
                                   const plsvo_align_params* params, const plsvo_align_result* out);
int plsvo_poseopt_multicam_batch_run(plsvo_ctx* ctx, const double* fx /* [B] errorMultiplier2 */,
                                     const plsvo_poseopt_batch* batch, const plsvo_poseopt_params* params,
                                     const plsvo_poseopt_result* out);
int plsvo_track_multicam_batch_run(plsvo_ctx* ctx, const plsvo_camera* cams /* [B] */, const plsvo_align_batch* al_batch,
                                   const plsvo_align_params* al_params, const plsvo_poseopt_batch* po_batch,
                                   const plsvo_poseopt_params* po_params, const plsvo_align_result* al_out,
                                   const plsvo_poseopt_result* po_out);

/* ------------------------------------------------------------------------------------------
 * Multicam ATAN batches: frame pairs from differently calibrated ATAN (FOV) cameras in one call, e.g. a fleet of FOV-lens
 * sensors with individual fx, fy, cx, cy and d0, of one size or several.  These are plsvo_align_atan_batch_run /
 * plsvo_track_atan_batch_run with the camera taken per pair, in the slot layout of the multicam calls above.
 * - Slot: of batch->cam only width and height are used; they are the slot.  Pair b's frames are
 *   cams[b].width x cams[b].height in the top-left corner of their slots, as for plsvo_align_multicam_batch_run.
 * - Alignment: pair b uses cams[b]'s members fx_, fy_, cx_, cy_, s_, s_inv_, tans_, tans_inv_ (derived from its constructor
 *   arguments exactly as plsvo_align_atan_batch_run derives them) wherever that call uses the batch's camera.  Everything
 *   else of `batch` is as for plsvo_align_atan_batch_run: full or lean bearings, depths, ragged counts and masks,
 *   PLSVO_ALIGN_FRAME_CHAIN (frames of one size), NULL levels derived on the device, every kernel variant.  Pair b's
 *   outputs are byte for byte those of plsvo_align_atan_batch_run on the same pair with cams[b] at its own size (its
 *   frames cut out of the slots) and the same kernel variant.
 * - Track: frame b's errorMultiplier2 is fx_ = cams[b].width * cams[b].fx; po_batch->fx is ignored.
 * - These calls always run upload -> launch -> download on the context's stream (not the arrival-gated path) and have
 *   finished with the caller's arrays when they return, whatever they return.
 * - NULL cams; a cams[b] wider or taller than the slot, below one pixel, or with a level (shipped, or up to max_level)
 *   smaller than one pixel; a frame chain whose size changes between consecutive pairs; a non-finite parameter, fx <= 0
 *   or fy <= 0, or a derived focal length out of range for any cams[b] (the index is in the message); or (track) batch
 *   sizes that differ return PLSVO_ERR_INVALID before anything is queued.  A library built without the ATAN multicam
 *   kernels returns PLSVO_ERR_CUDA.
 * - The kernels keep the pair's members, size and distortion terms in 128 bytes of shared memory per CTA, planned for as
 *   for the multicam kernels (DESIGN.md §4.14).
 * - Pinhole and ATAN pairs in one batch: plsvo_*_any_camera_batch_run below.
 * - Out of scope: raw frames, the arrival-gated path, a ragged layout, the seed updates and the drop-in shim.  Direct
 *   matching with a camera per image: plsvo_match_direct_multicam_batch_run.
 * ---------------------------------------------------------------------------------------- */
int plsvo_align_atan_multicam_batch_run(plsvo_ctx* ctx, const plsvo_atan_camera* cams /* [B] */, const plsvo_align_batch* batch,
                                        const plsvo_align_params* params, const plsvo_align_result* out);
int plsvo_track_atan_multicam_batch_run(plsvo_ctx* ctx, const plsvo_atan_camera* cams /* [B] */, const plsvo_align_batch* al_batch,
                                        const plsvo_align_params* al_params, const plsvo_poseopt_batch* po_batch,
                                        const plsvo_poseopt_params* po_params, const plsvo_align_result* al_out,
                                        const plsvo_poseopt_result* po_out);

/* ------------------------------------------------------------------------------------------
 * Feature alignment (SURVEY.md §8f "next", rank 1): feature_alignment::align2D,
 * include/plsvo/feature_alignment.h:49-55, src/feature_alignment.cpp:160-290 (scalar path) — the 8x8
 * inverse-compositional refinement Matcher::findMatchDirect runs per feature (src/matcher.cpp:201).
 * n features; feature i searches pyramid level level[i] of frame image_index[i].
 * ---------------------------------------------------------------------------------------- */
typedef struct plsvo_align2d_batch {
  int32_t n_features, n_images, width, height; /* width/height = level-0 size of the frames */
  int32_t n_iter, reserved;
  const uint8_t* img[PLSVO_MAX_LEVELS]; /* cur_img per level: frame b at img[l] + b*img_stride[l] */
  size_t img_pitch[PLSVO_MAX_LEVELS];
  size_t img_stride[PLSVO_MAX_LEVELS];
  const int32_t* image_index;           /* [n] */
  const int32_t* level;                 /* [n] */
  const uint8_t* ref_patch_with_border; /* [n][10*10] */
  const uint8_t* ref_patch;             /* [n][8*8]   */
  const double* px;                     /* [n][2] cur_px_estimate on entry (pixels of the search level) */
} plsvo_align2d_batch;

typedef struct plsvo_align2d_result {
  double* px;         /* [n][2] cur_px_estimate on return */
  uint8_t* converged; /* [n]    return value of align2D */
} plsvo_align2d_result;

int plsvo_align2d_batch_run(plsvo_ctx* ctx, const plsvo_align2d_batch* in, const plsvo_align2d_result* out);

/* ---- feature_alignment::align1D (SURVEY.md §8f rank 1, "next") --------------------------------
 * Replaces, for n features at once, include/plsvo/feature_alignment.h:39-46 /
 * src/feature_alignment.cpp:40-157:
 *     bool align1D(const cv::Mat& cur_img, const Vector2f& dir, uint8_t* ref_patch_with_border,
 *                  uint8_t* ref_patch, const int n_iter, Vector2d& cur_px_estimate, double& h_inv);
 * the 1-DoF variant Matcher::findMatchDirect / findEpipolarMatchDirect use for edgelets
 * (src/matcher.cpp:195,331,400,497): the patch may only move along `dir`.  Same feature arrays as
 * plsvo_align2d_batch plus one direction per feature. */
typedef struct plsvo_align1d_batch {
  plsvo_align2d_batch features; /* images, image_index, level, patches, px — as for align2D */
  const float* dir;             /* [n][2] direction in which the patch is allowed to move */
} plsvo_align1d_batch;

typedef struct plsvo_align1d_result {
  double* px;         /* [n][2] cur_px_estimate on return */
  uint8_t* converged; /* [n]    return value of align1D */
  double* h_inv;      /* [n]    h_inv on return (:75) */
} plsvo_align1d_result;

int plsvo_align1d_batch_run(plsvo_ctx* ctx, const plsvo_align1d_batch* in, const plsvo_align1d_result* out);

/* ---- Matcher::findMatchDirect (SURVEY.md §8f rank 1, "next") ----------------------------------
 * Replaces, for n (3D feature, current frame) candidates at once, include/plsvo/matcher.h:104-107 /
 * src/matcher.cpp:159-211:
 *     bool Matcher::findMatchDirect(const Point& pt, const Frame& cur_frame, Vector2d& px_cur);
 * i.e. everything after pt.getCloseViewObs() has picked the reference observation ref_ftr_ (list
 * logic, stays on the host): the in-frame test of the reference patch (:169-171), the affine warp
 * matrix (warp::getWarpMatrixAffine, :42-71), the search level (warp::getBestSearchLevel, :73-87), the
 * warped 10x10 reference patch (warp::warpAffine, :89-133, bilinear vk::interpolateMat_8u), the 8x8
 * patch cut out of it (:148-157) and the align2D / align1D refinement at the search level (:189-208).
 * The line-segment overload (:241-275) is the same computation on the two end points
 * (precomputeRefPatch, :213-232, + align2D): pass each end point as one feature and AND the flags.
 * Both frames use the same undistorted pinhole camera (app/run_pipeline.cpp:786-795). */
typedef struct plsvo_match_batch {
  int32_t n_features;
  int32_t n_ref_images;   /* keyframes holding the reference observations */
  int32_t n_cur_images;   /* current frames */
  int32_t n_pyr_levels;   /* Config::nPyrLevels(): the search level is < n_pyr_levels (:180) */
  int32_t n_iter;         /* Matcher::Options::align_max_iter (10, matcher.h:85) */
  int32_t reserved;
  plsvo_camera cam;
  const uint8_t* ref_img[PLSVO_MAX_LEVELS]; /* ref_ftr_->frame->img_pyr_[l]: frame r at ref_img[l] + r*ref_stride[l] */
  size_t ref_pitch[PLSVO_MAX_LEVELS];
  size_t ref_stride[PLSVO_MAX_LEVELS];
  const uint8_t* cur_img[PLSVO_MAX_LEVELS]; /* cur_frame.img_pyr_[l] */
  size_t cur_pitch[PLSVO_MAX_LEVELS];
  size_t cur_stride[PLSVO_MAX_LEVELS];
  const double* T_ref_w;      /* [n_ref_images][7] ref_ftr_->frame->T_f_w_ */
  const double* T_cur_w;      /* [n_cur_images][7] cur_frame.T_f_w_ */
  const int32_t* ref_index;   /* [n] keyframe of the reference observation */
  const int32_t* cur_index;   /* [n] current frame */
  const double* ref_px;       /* [n][2] ref_ftr_->px (level-0 pixels) */
  const double* ref_f;        /* [n][3] ref_ftr_->f */
  const int32_t* ref_level;   /* [n]    ref_ftr_->level */
  const uint8_t* is_edgelet;  /* [n] or NULL: PointFeat::type == EDGELET -> align1D along A_cur_ref*grad */
  const double* ref_grad;     /* [n][2] or NULL: PointFeat::grad */
  const double* pos;          /* [n][3] pt.pos_ (world) */
  const double* px_cur;       /* [n][2] px_cur on entry: the projection estimate (level-0 pixels) */
} plsvo_match_batch;

typedef struct plsvo_match_result {
  double* px_cur;        /* [n][2] px_cur on return (untouched where the in-frame test fails) */
  uint8_t* success;      /* [n]    return value of findMatchDirect */
  int32_t* search_level; /* [n]    Matcher::search_level_ (-1 where the in-frame test fails) */
  double* A_cur_ref;     /* [n][4] or NULL: Matcher::A_cur_ref_ row-major (A00 A01 A10 A11), which Reprojector::refine reads for
                          *        edgelets (src/reprojector.cpp:318-320); untouched where the in-frame test fails */
} plsvo_match_result;

int plsvo_match_direct_batch_run(plsvo_ctx* ctx, const plsvo_match_batch* in, const plsvo_match_result* out);

/* ---- Matcher::findMatchDirect for frames from an ATAN (FOV) camera -------------------------------
 * plsvo_match_direct_batch_run with the keyframes and the current frames seen through vk::ATANCamera(*cam), the model of
 * plsvo_atan_camera above (in a reference pipeline with cam_model ATAN both are the same camera object).  Of
 * findMatchDirect only warp::getWarpMatrixAffine reads the camera model: its two cam_ref.cam2world and three
 * cam_cur.world2cam calls use the ATAN formulas.  The in-frame test reads the image size only, and everything downstream
 * of A_cur_ref (search level, warped patch, edgelet direction, align2D / align1D) is unchanged.
 * - `in` is as for plsvo_match_direct_batch_run.  in->cam.width / height must equal the camera's; the other fields of
 *   in->cam are ignored.
 * - A size mismatch, a non-finite parameter, fx <= 0 or fy <= 0 returns PLSVO_ERR_INVALID before anything is queued, and
 *   the context stays usable.  A library built without the ATAN matching kernel returns PLSVO_ERR_CUDA.
 * - Exactness: the device's atan and tan may differ from glibc's by an ulp or two, so A_cur_ref agrees with the reference
 *   to round-off (each entry within 1e-12; the entries are O(1)).  Everything downstream of A_cur_ref is exact: search
 *   level, success and px_cur are byte for byte what the reference computes from the returned A_cur_ref.  A candidate
 *   whose five projections call neither tan nor atan (d0 == 0, or every argument inside both cut-offs) matches the
 *   reference byte for byte, A_cur_ref included.
 * - Out of scope: the depth-filter seed updates (findEpipolarMatchDirect) for ATAN frames, raw frames.  A camera per
 *   image, pinhole and ATAN candidates in one call: plsvo_match_direct_multicam_batch_run below. */
int plsvo_match_direct_atan_batch_run(plsvo_ctx* ctx, const plsvo_atan_camera* cam, const plsvo_match_batch* in,
                                      const plsvo_match_result* out);

/* ---- Matcher::findMatchDirect for images from differently calibrated cameras --------------------
 * plsvo_match_direct_batch_run with a camera per image, pinhole or ATAN, in the padded slots of the multicam calls: one
 * call serves the keyframes and current frames of many visual-odometry streams.  In the reference the cameras belong to
 * the frames (ref_ftr_->frame->cam_ and cur_frame.cam_, src/matcher.cpp:168-176), and a candidate may pair a keyframe
 * and a current frame from different cameras.
 * - Slot: of in->cam only width and height are used; they are the slot.  Every image sits in a slot-sized frame at the
 *   batch's pitches and strides.  Ref image r's camera is cams[cam_of_ref[r]], current image c's cams[cam_of_cur[c]];
 *   the image's pixels are that camera's width x height in the top-left corner, at level l (width >> l) x (height >> l).
 *   The bytes outside that region (the padding) never reach a result.
 * - Candidate i reads its ref image's camera for the in-frame test, the warpAffine bounds and cam2world in
 *   getWarpMatrixAffine; its current image's camera for world2cam in getWarpMatrixAffine and the align2D / align1D bounds
 *   at the search level.
 * - A pinhole camera (model PLSVO_CAMERA_PINHOLE) is plsvo_match_batch::cam of plsvo_match_direct_batch_run: size and
 *   fx..cy in pixels.  An ATAN camera (PLSVO_CAMERA_ATAN) is the constructor's arguments, as for
 *   plsvo_match_direct_atan_batch_run, and its members are derived exactly as that call derives them.  The other member
 *   of the record is ignored.
 * - Exactness: a candidate whose two images share camera k gives byte for byte the outputs of the one-camera call
 *   (plsvo_match_direct_batch_run or plsvo_match_direct_atan_batch_run with k, the frames cut out of their slots).  A
 *   candidate with two pinhole cameras matches the reference byte for byte; one with an ATAN camera meets the contract of
 *   plsvo_match_direct_atan_batch_run.
 * - NULL cams, cam_of_ref or cam_of_cur; n_cams < 1; an index outside [0, n_cams); an unknown model; a pinhole camera
 *   with a non-finite fx, fy, cx or cy or with fx or fy equal to 0; an ATAN camera plsvo_match_direct_atan_batch_run
 *   rejects; a camera wider or taller than the slot; or a camera used at a level below one pixel (a ref image's at its
 *   candidates' ref_level, a current image's at n_pyr_levels - 1) returns PLSVO_ERR_INVALID, with the index in the
 *   message, before anything is queued; the context stays usable.  A library built without the kernel returns
 *   PLSVO_ERR_CUDA.
 * - Out of scope: the depth-filter seed updates per camera, raw frames, a ragged frame layout, a camera per candidate. */
#define PLSVO_CAMERA_PINHOLE 0
#define PLSVO_CAMERA_ATAN 1
typedef struct plsvo_match_camera {
  int32_t model, reserved;
  plsvo_camera pinhole;   /* model PINHOLE: size and fx..cy in pixels, as plsvo_match_batch::cam */
  plsvo_atan_camera atan; /* model ATAN: the constructor's arguments, as for plsvo_match_direct_atan_batch_run */
} plsvo_match_camera;

int plsvo_match_direct_multicam_batch_run(plsvo_ctx* ctx, const plsvo_match_camera* cams, int32_t n_cams,
                                          const int32_t* cam_of_ref /* [n_ref_images] */,
                                          const int32_t* cam_of_cur /* [n_cur_images] */, const plsvo_match_batch* in,
                                          const plsvo_match_result* out);

/* ------------------------------------------------------------------------------------------
 * Any-camera batches: frame pairs from pinhole and ATAN (FOV) cameras in one call, e.g. rectified EuRoC / TUM streams next
 * to SVO's 752x480 FOV camera.  These are plsvo_align_multicam_batch_run / plsvo_align_atan_multicam_batch_run (and the
 * track calls) with pair b's camera, and its model, taken from a table: cams[cam_of_pair[b]], the records of
 * plsvo_match_direct_multicam_batch_run, so that one camera table serves matching and alignment.
 * - Slot: of batch->cam only width and height are used; they are the slot.  Pair b's frames are its camera's width x
 *   height in the top-left corner of their slots, as for plsvo_align_multicam_batch_run.
 * - The model tag decides the model, never the parameters: an ATAN camera with d0 = 0 stays ATAN (the two models do not
 *   compute the same bits, DESIGN.md §4.10).  A pinhole camera is plsvo_camera in pixels; an ATAN camera is the
 *   constructor's arguments, its members derived exactly as plsvo_align_atan_batch_run derives them.
 * - Exactness: a pinhole pair's outputs are byte for byte those of plsvo_align_multicam_batch_run on that pair with that
 *   camera's plsvo_camera; an ATAN pair's those of plsvo_align_atan_multicam_batch_run on that pair with that
 *   plsvo_atan_camera; both at the same kernel variant.
 * - Everything else of `batch` is as for those calls: full or lean bearings (lean ones formed with the pair's own model's
 *   cam2world), depths, ragged counts and masks, NULL levels derived on the device, every kernel variant (PLSVO_VARIANT)
 *   and PLSVO_ALIGN_FRAME_CHAIN, in which consecutive pairs need cameras of one size.
 * - Track: frame b's errorMultiplier2 is |fx| of a pinhole camera and fx_ = width * fx of an ATAN camera; po_batch->fx is
 *   ignored.
 * - These calls always run upload -> launch -> download on the context's stream (not the arrival-gated path) and have
 *   finished with the caller's arrays when they return, whatever they return.
 * - NULL cams or cam_of_pair; n_cams < 1; a cam_of_pair[b] outside [0, n_cams); an unknown model; a camera of the table
 *   that plsvo_align_multicam_batch_run (pinhole) or plsvo_align_atan_multicam_batch_run (ATAN) would reject — wider or
 *   taller than the slot, below one pixel at a shipped or aligned level, non-finite or zero intrinsics; every camera of
 *   the table is checked, and the camera index is in the message; a size change between consecutive pairs of a frame
 *   chain (the pair indices are in the message); a batch <= 0; or (track) batch sizes that differ return
 *   PLSVO_ERR_INVALID before anything is queued, and the context stays usable.  A library built without the any-camera
 *   kernels returns PLSVO_ERR_CUDA.
 * - The kernels keep the pair's camera, size, distortion terms and model tag in 128 bytes of shared memory per CTA,
 *   planned for as for the multicam kernels (DESIGN.md §4.17).
 * - Raw (distorted pinhole) frames next to ATAN frames: plsvo_*_raw_any_camera_batch_run below.
 * - Out of scope: the arrival-gated path, separate upload / launch / download legs, dist.align_sharded, a ragged layout,
 *   the seed updates and the drop-in shim.
 * ---------------------------------------------------------------------------------------- */
int plsvo_align_any_camera_batch_run(plsvo_ctx* ctx, const plsvo_match_camera* cams, int32_t n_cams,
                                     const int32_t* cam_of_pair /* [B] */, const plsvo_align_batch* batch,
                                     const plsvo_align_params* params, const plsvo_align_result* out);
int plsvo_track_any_camera_batch_run(plsvo_ctx* ctx, const plsvo_match_camera* cams, int32_t n_cams,
                                     const int32_t* cam_of_pair /* [B] */, const plsvo_align_batch* al_batch,
                                     const plsvo_align_params* al_params, const plsvo_poseopt_batch* po_batch,
                                     const plsvo_poseopt_params* po_params, const plsvo_align_result* al_out,
                                     const plsvo_poseopt_result* po_out);

/* ------------------------------------------------------------------------------------------
 * Raw any-camera batches: raw frames from distorted pinhole lenses and from ATAN (FOV) cameras in one call, e.g. raw
 * EuRoC / TUM streams next to SVO's 752x480 FOV camera.  Pair b's camera is cams[cam_of_pair[b]], and its tag picks
 * what happens to both of the pair's frames:
 *   PLSVO_CAMERA_PINHOLE: `pinhole` is the distorted lens, as for plsvo_undistort_batch; fabs(d0) <= 1e-7 means no
 *     distortion.
 *     The frames are rectified on the device with that lens's map and aligned as an undistorted pinhole with its fx, fy,
 *     cx, cy: what plsvo_align_raw_multicam_batch_run does for that pair.
 *   PLSVO_CAMERA_ATAN: `atan` is the constructor's arguments, as plsvo_align_atan_batch_run.  The frames are used as they
 *     are (the pipeline never rectifies FOV frames), half-sampled into their pyramid and aligned through the ATAN model:
 *     what plsvo_align_atan_multicam_batch_run does with that pair's pyramid.
 * One fused rectify / pyramid kernel runs over every frame, then one alignment kernel (and, track, the pose optimiser).
 * - Slot: as for plsvo_align_raw_multicam_batch_run, of batch->cam only width and height are used.  Every camera fits in
 *   the slot, and a pair's frames sit in the top-left corner of their slots (raw stacks at `pitch` and `stride`).
 * - The tag decides the model, never the parameters: a lens with d0 = 0 is a pinhole that copies its frame; an ATAN
 *   camera with d0 = 0 stays ATAN.
 * - Exactness, at the same kernel variant: a lens pair's outputs are byte for byte those of
 *   plsvo_align_raw_multicam_batch_run on that pair with that lens; an ATAN pair's those of
 *   plsvo_align_atan_multicam_batch_run on that pair with that camera, its levels createImgPyramid of its raw frames.
 *   Equivalently, feeding rect_out to plsvo_align_any_camera_batch_run, with the table mapped to plsvo_match_camera
 *   records (a lens becomes the undistorted pinhole of its fx..cy), gives the same bytes for every pair.
 * - Track: frame b's errorMultiplier2 is |fx| of a lens and fx_ = width * fx of an ATAN camera; po_batch->fx is ignored.
 * - rect_out as for the raw calls: every non-NULL level, the B reference frames followed by the B current frames, each
 *   holding the pyramid the pipeline builds (rectified for a lens, the frame itself for an ATAN camera) in its slot's
 *   region, the rest of the slot 0.
 * - Maps: only distorted lenses build maps.  These calls share the cache of the raw multicam calls and its rule: after a
 *   call it holds exactly the maps of the distorted lenses that call referenced.  plsvo_last_map_build_ms works as there.
 * - NULL cams or cam_of_pair; n_cams < 1; a cam_of_pair[b] outside [0, n_cams); an unknown model; a table camera that
 *   plsvo_align_raw_multicam_batch_run (lens) or plsvo_align_any_camera_batch_run (ATAN) would reject, every camera of the
 *   table checked, used or not; a level (aligned or asked of rect_out) below one pixel for a camera some pair
 *   references; PLSVO_ALIGN_FRAME_CHAIN; image pointers in `batch`; max_level > 6; or (track) batch sizes that differ
 *   return PLSVO_ERR_INVALID, with the camera or pair index in the message, before anything is queued, and the context
 *   stays usable.  A library built without the fused multicam launcher or the any-camera kernels returns PLSVO_ERR_CUDA.
 * - These calls always run upload -> launch -> download on the context's stream (not the arrival-gated path) and have
 *   finished with the caller's arrays when they return, whatever they return.
 * - Out of scope: frame chains (a chained frame belongs to two pairs), the arrival-gated path, separate upload / launch /
 *   download legs, a ragged layout, the seed updates and the drop-in shim, rectifying ATAN frames.
 * ---------------------------------------------------------------------------------------- */
typedef struct plsvo_raw_camera {
  int32_t model, reserved;        /* PLSVO_CAMERA_PINHOLE or PLSVO_CAMERA_ATAN */
  plsvo_pinhole_camera pinhole;   /* PINHOLE: the distorted lens, as for plsvo_undistort_batch; fabs(d0) <= 1e-7: no distortion */
  plsvo_atan_camera atan;         /* ATAN: the constructor's arguments, as plsvo_align_atan_batch_run */
} plsvo_raw_camera;

typedef struct plsvo_raw_any_camera_frames {
  int32_t n_cams, reserved;
  const plsvo_raw_camera* cams;   /* [n_cams] */
  const int32_t* cam_of_pair;     /* [B] index into cams: the camera of both frames of pair b */
  const uint8_t* ref_raw;         /* [B] raw frames, one slot (batch->cam's size) each */
  const uint8_t* cur_raw;         /* [B] raw frames, one slot (batch->cam's size) each */
  size_t pitch, stride;           /* host layout of both stacks, as plsvo_raw_multicam_frames */
} plsvo_raw_any_camera_frames;

int plsvo_align_raw_any_camera_batch_run(plsvo_ctx* ctx, const plsvo_raw_any_camera_frames* raw, const plsvo_align_batch* batch,
                                         const plsvo_align_params* params, const plsvo_align_result* out,
                                         const plsvo_pyramid_result* rect_out);
int plsvo_track_raw_any_camera_batch_run(plsvo_ctx* ctx, const plsvo_raw_any_camera_frames* raw,
                                         const plsvo_align_batch* al_batch, const plsvo_align_params* al_params,
                                         const plsvo_poseopt_batch* po_batch, const plsvo_poseopt_params* po_params,
                                         const plsvo_align_result* al_out, const plsvo_poseopt_result* po_out,
                                         const plsvo_pyramid_result* rect_out);

/* ---- Structure optimisation: Point::optimize / LineSeg::optimize (SURVEY.md §8f rank 3, "next") ---
 * Replaces, for a batch of 3D features, include/plsvo/feature3D.h:120,157 / src/feature3D_impl.cpp:36-95,
 * 97-174 as driven by FrameHandlerBase::optimizeStructure (src/frame_handler_base.cpp:202-237):
 *     void Point::optimize(const size_t n_iter);     void LineSeg::optimize(const size_t n_iter);
 * 3x3 Gauss-Newton on the reprojection error (unit plane) of a 3D point over its observations obs_
 * (a LineSeg optimises its two end points with a coupled accept/roll-back/convergence test).
 * Observations are given in CSR form, in obs_ list order (the summation order of the reference). */
typedef struct plsvo_structopt_batch {
  int32_t n_points, n_segs, n_frames;
  int32_t n_iter_pts;  /* Config::structureOptimNumIter() */
  int32_t n_iter_segs; /* Config::structureOptimNumIterSegs() */
  int32_t reserved;
  const double* T_f_w;           /* [n_frames][7] (*it)->frame->T_f_w_ of the observing keyframes */
  const int32_t* pt_obs_begin;   /* [n_points+1] offsets into pt_obs_* */
  const int32_t* pt_obs_frame;   /* [n_pt_obs]   index into T_f_w */
  const double* pt_obs_f;        /* [n_pt_obs][3] PointFeat::f */
  const double* pt_pos;          /* [n_points][3] Point::pos_ on entry */
  const int32_t* seg_obs_begin;  /* [n_segs+1] */
  const int32_t* seg_obs_frame;  /* [n_seg_obs] */
  const double* seg_obs_sf;      /* [n_seg_obs][3] LineFeat::sf */
  const double* seg_obs_ef;      /* [n_seg_obs][3] LineFeat::ef */
  const double* seg_spos;        /* [n_segs][3] LineSeg::spos_ on entry */
  const double* seg_epos;        /* [n_segs][3] LineSeg::epos_ on entry */
} plsvo_structopt_batch;

typedef struct plsvo_structopt_result {
  double* pt_pos;   /* [n_points][3] Point::pos_ on return */
  double* seg_spos; /* [n_segs][3] */
  double* seg_epos; /* [n_segs][3] */
  int32_t* pt_iters;  /* [n_points] or NULL: GN iterations executed (diagnostic) */
  int32_t* seg_iters; /* [n_segs] or NULL */
} plsvo_structopt_result;

int plsvo_structopt_batch_run(plsvo_ctx* ctx, const plsvo_structopt_batch* in, const plsvo_structopt_result* out);

/* ---- Depth-filter point-seed update (SURVEY.md §8f rank 4, "next") ------------------------------
 * Replaces, for n point seeds at once, the body of DepthFilter::updatePointSeeds (src/depth_filter.cpp:270-365):
 * visibility test of the seed in the current frame (:291-304), inverse-depth search range (:307-308),
 *     bool Matcher::findEpipolarMatchDirect(ref_frame, cur_frame, ref_ftr, d_estimate, d_min, d_max, depth)
 * (include/plsvo/matcher.h, src/matcher.cpp:277-420: epipolar segment, affine warp, edgelet pre-selection, ZMSSD
 * search along the epipolar line or direct alignment when it is shorter than 2 px, sub-pixel align2D/align1D,
 * depthFromTriangulation :135-146), DepthFilter::computeTau (:568-584) and the Gaussian x Beta update
 * DepthFilter::updatePointSeed (:489-512, Vogiatzis & Hernandez 2011).  The list logic around it (seed ageing,
 * creating a Point from a converged seed, the detector's occupancy grid) stays on the host; `converged` reports
 * the reference's test sqrt(sigma2) < z_range / seed_convergence_sigma2_thresh (:334).
 * Images must be dense (pitch == width of the level): the reference indexes the ZMSSD patch with Mat::cols (:380-382). */
typedef struct plsvo_seed_batch {
  int32_t n_seeds;
  int32_t n_ref_images;
  int32_t n_cur_images;
  int32_t n_pyr_levels;          /* Config::nPyrLevels() */
  int32_t n_iter;                /* Matcher::Options::align_max_iter (10) */
  int32_t max_epi_search_steps;  /* Matcher::Options::max_epi_search_steps (1000) */
  uint8_t align_1d;              /* Matcher::Options::align_1d (false) */
  uint8_t subpix_refinement;     /* Matcher::Options::subpix_refinement (true) */
  uint8_t epi_search_edgelet_filtering; /* (true) */
  uint8_t reserved0[5];
  double epi_search_edgelet_max_angle;   /* (0.7) */
  double seed_convergence_sigma2_thresh; /* DepthFilter::Options (200.0) */
  plsvo_camera cam;
  const uint8_t* ref_img[PLSVO_MAX_LEVELS];
  size_t ref_pitch[PLSVO_MAX_LEVELS];
  size_t ref_stride[PLSVO_MAX_LEVELS];
  const uint8_t* cur_img[PLSVO_MAX_LEVELS];
  size_t cur_pitch[PLSVO_MAX_LEVELS];
  size_t cur_stride[PLSVO_MAX_LEVELS];
  const double* T_ref_w;     /* [n_ref_images][7] it->ftr->frame->T_f_w_ */
  const double* T_cur_w;     /* [n_cur_images][7] frame->T_f_w_ */
  const int32_t* ref_index;  /* [n] */
  const int32_t* cur_index;  /* [n] */
  const double* ref_px;      /* [n][2] it->ftr->px */
  const double* ref_f;       /* [n][3] it->ftr->f */
  const int32_t* ref_level;  /* [n]    it->ftr->level */
  const uint8_t* is_edgelet; /* [n] or NULL */
  const double* ref_grad;    /* [n][2] or NULL */
  const float* a;            /* [n] PointSeed::a on entry */
  const float* b;            /* [n] */
  const float* mu;           /* [n] inverse depth mean */
  const float* z_range;      /* [n] */
  const float* sigma2;       /* [n] */
} plsvo_seed_batch;

#define PLSVO_SEED_NOT_VISIBLE 0 /* behind the camera / outside the image: seed untouched (:296-304) */
#define PLSVO_SEED_NO_MATCH 1    /* findEpipolarMatchDirect failed: b += 1 (:312-317) */
#define PLSVO_SEED_UPDATED 2     /* Bayesian update applied (:320-325) */

typedef struct plsvo_seed_result {
  float* a;           /* [n] PointSeed state on return */
  float* b;
  float* mu;
  float* sigma2;
  int32_t* status;    /* [n] PLSVO_SEED_* */
  uint8_t* converged; /* [n] */
  double* depth;      /* [n] z of findEpipolarMatchDirect (NaN unless status == UPDATED) */
  double* px_cur;     /* [n][2] Matcher::px_cur_ (diagnostic; NaN where no position was computed) */
} plsvo_seed_result;

int plsvo_seed_update_batch_run(plsvo_ctx* ctx, const plsvo_seed_batch* in, const plsvo_seed_result* out);

/* Line-seed variant: the body of DepthFilter::updateLineSeeds (src/depth_filter.cpp:367-471).  A LineSeed carries one
 * inverse-depth Gaussian per end point and a shared Beta (a, b).  Both end points are searched with
 * Matcher::findEpipolarMatchDirectSegmentEndpoint (src/matcher.cpp:420-588) — which, as in the reference, warps and
 * searches around the segment feature's own px / f (its mid point, base Feature fields) for BOTH depth hypotheses and
 * has no edgelet pre-selection — then computeTau uses the end-point bearings sf / ef (:415-418) and
 * DepthFilter::updateLineSeed (:514-565) updates both Gaussians and takes a = max(a_s, a_e), b = min(b_s, b_e).
 * `seeds` describes the start point: ref_px / ref_f = LineFeat::px / f, mu / z_range / sigma2 = mu_s / z_range_s / sigma2_s;
 * is_edgelet / ref_grad are ignored. */
typedef struct plsvo_line_seed_batch {
  plsvo_seed_batch seeds;
  const double* ref_sf;    /* [n][3] LineFeat::sf */
  const double* ref_ef;    /* [n][3] LineFeat::ef */
  const float* mu_e;       /* [n] */
  const float* z_range_e;  /* [n] */
  const float* sigma2_e;   /* [n] */
} plsvo_line_seed_batch;

typedef struct plsvo_line_seed_result {
  plsvo_seed_result seeds; /* a, b, mu_s, sigma2_s, status, converged (both end points), depth = z_s, px_cur of the start search */
  float* mu_e;             /* [n] */
  float* sigma2_e;         /* [n] */
  double* depth_e;         /* [n] z_e (NaN unless status == UPDATED) */
  double* px_cur_e;        /* [n][2] or NULL: Matcher::px_cur_ of the end-point search — what matcherls_.px_cur_ holds when
                            *        DepthFilter::updateLineSeeds marks the detector grid on keyframes (:426-430); NaN where the
                            *        end-point search did not run or computed no position */
} plsvo_line_seed_result;

int plsvo_line_seed_update_batch_run(plsvo_ctx* ctx, const plsvo_line_seed_batch* in, const plsvo_line_seed_result* out);

/* device time (CUDA events on the context's stream) of the kernel launched by the last
 * plsvo_pyramid / align2d / align1d / match_direct / seed_update / structopt _batch_run call: the kernel alone,
 * without the host<->device copies those calls also make.  For plsvo_undistort_batch_run it covers the remap and
 * pyramid kernels; a map build that call made is not included (plsvo_last_map_build_ms reports it).  For the raw-frame
 * calls it covers the rectify + pyramid kernel and the alignment (and pose-optimiser) kernels.  Measurement aid,
 * no reference counterpart. */
int plsvo_last_kernel_ms(plsvo_ctx* ctx, float* ms);

/* number of kernels this context has launched since creation (bench "gpu_launches") */
int64_t plsvo_launch_count(const plsvo_ctx* ctx);

/* Device self-test of the fp32 weight kernel: evaluates w = 1/(1+a) with the product's fp32
 * sequence and with the reference's double-then-narrow expression (sparse_img_align.cpp:479) for
 * n pseudo-random a in [0,256) plus all n_exhaustive first float bit patterns of [0,256), and
 * returns the number of bitwise mismatches. */
int plsvo_selftest_weight(plsvo_ctx* ctx, uint32_t n, uint32_t seed, uint64_t* mismatches);

/* library build info: "plsvo_b200 <version> sm_90a" */
const char* plsvo_version(void);

#ifdef __cplusplus
}
#endif
#endif /* PLSVO_B200_H_ */
