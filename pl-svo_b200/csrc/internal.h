// internal.h — kernel argument blocks and launch entry points shared by the .cu files.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/plsvo_b200.h"

namespace plsvo {

constexpr int kCacheRows = 12;  // float4 rows per patch: 4 ref + 4 dx + 4 dy

// Device-layout description of one alignment batch (all pointers are device pointers).
struct AlignArgs {
  int B, n_pts, n_segs;
  int max_level, min_level, n_iter;
  double eps;
  int width, height;
  double fx, fy, cx, cy;
  // pyramid level l of pair b: img[l] + b*stride[l], rows pitch[l] bytes (pitch multiple of 16)
  const uint8_t* ref_img[PLSVO_MAX_LEVELS];
  const uint8_t* cur_img[PLSVO_MAX_LEVELS];
  uint32_t pitch[PLSVO_MAX_LEVELS];
  size_t stride[PLSVO_MAX_LEVELS];
  uint8_t img_in_smem[PLSVO_MAX_LEVELS];  // stage the cur level in shared memory with a bulk copy
  const double* T_ref_w;
  const double* T_cur_w;
  const int32_t* pt_count;
  const double* pt_px;
  const double* pt_f;
  const double* pt_pos;
  const uint8_t* pt_valid;
  const int32_t* seg_count;
  const double* seg_spx;
  const double* seg_epx;
  const double* seg_sf;
  const double* seg_ef;
  const double* seg_spos;
  const double* seg_epos;
  const double* seg_length;
  const uint8_t* seg_valid;
  const double* pt_depth;    // optional: |pos - ref_pos| per point (then pt_pos may be null)
  const double* seg_sdepth;  // optional: per segment start / end point
  const double* seg_edepth;
  // outputs
  double* out_T;
  long long* out_n_tracked;
  double* out_H;
  uint8_t* out_seg_killed;
  int32_t* out_iters;
  int32_t* out_status;
  uint32_t* out_patch_iters;
  uint32_t* out_patch_levels;
  // work distribution + per-CTA workspace
  unsigned int* work_counter;
  // arrival gate of the host-buffer pipeline: pair b may be touched once *arrived > b / gate_chunk
  // (a copy stream bumps it after each chunk of the batch has landed); gate_chunk == 0: no gate.
  const unsigned int* arrived;
  int gate_chunk;
  int max_patches;      // patch slots per pair: n_pts + max segment samples
  int max_seg_patches;  // segment sample slots per pair
  int max_seg_slots;    // lane slots of the segment groups per pair (multiple of 32)
  int smem_img_bytes;   // bytes of the image staging buffer
  float4* ws_cache;     // [grid][kCacheRows][max_patches] reference-patch cache (ref, dx, dy rows)
  double* ws_segpx;     // [grid][2][max_seg_patches] 2-D centre of every segment sample (precompute only)
  double* ws_rec;       // [grid][2][rec_cap*threads] parked Sxr, Syr of the samples of segments longer than a warp
  int rec_cap;          // 32-sample trips of the longest segment, <= 32
  double* ws_gram;      // [grid][max_seg_patches][3] Sxx, Sxy, Syy of every segment sample, unless gram_in_smem
  int gram_in_smem;     // 1: they sit in shared memory, 3 * 8 * max_seg_patches bytes behind align_smem_bytes()
  int derive_from;      // >= 0: the CTA forms levels (derive_from, max_level] of its pair by halfSample (gated pipeline)
  // vk::ATANCamera distortion (read by the ATAN kernels only; fx, fy, cx, cy above then hold fx_, fy_, cx_, cy_):
  // s_ = d0, s_inv_ = 1/s_, tans_ = 2 tan(s_/2), tans_inv_ = 1/tans_, all zero when s_ == 0
  double atan_s, atan_s_inv, atan_tans, atan_tans_inv;
  // [B] camera of every pair (the multicam kernels read its fx, fy, cx, cy instead of fx, fy, cx, cy above)
  const plsvo_camera* cams;
  // [B][4] s_, s_inv_, tans_, tans_inv_ of every pair's vk::ATANCamera (read by the ATAN multicam kernels only, instead
  // of atan_s..atan_tans_inv above; a.cams[b] then holds the pair's members fx_, fy_, cx_, cy_ and its size)
  const double* atan_terms;
  // [B] model tag of every pair, PLSVO_CAMERA_PINHOLE or PLSVO_CAMERA_ATAN (read by the any-camera kernels only: a.cams[b]
  // then holds a pinhole pair's fx..cy or an ATAN pair's members, and a.atan_terms[b] an ATAN pair's distortion terms)
  const int32_t* cam_models;
};

// Opaque chi2 patches (16 float terms each) the alignment kernel can hold per Gauss-Newton pass: the patches whose 16
// additions may carry the float accumulator across a power of two, chained term by term.  The classification margin
// grows with the patch index, so their number grows with the square of the point count; this leaves at least a factor
// of two over the count the exact-order model of tests/test_chi2_order_cpu.py gives, at every point count shared memory
// admits.  A pass that still overflows it flags status bit 2 and approximates the chi2.
__host__ __device__ inline int align_opq_cap(int n_pts) { return 48 + (int)((long long)n_pts * n_pts / 131072); }

// shared memory the kernel needs for a configuration (host + device agree through this)
size_t align_smem_bytes(int n_pts, int n_segs, int max_patches, int max_seg_slots, int img_bytes, int threads);
// kernel variants are compiled per (threads per CTA, resident CTAs per SM the register budget allows):
// (64,8) (96,7) (96,5) (128,5) (128,4) (160,3) (192,2) (256,2)
cudaError_t align_kernel_prepare(int threads, int min_blocks, size_t smem_bytes, int* ctas_per_sm);
cudaError_t weight_selftest_launch(uint32_t n, uint32_t seed, unsigned long long* d_mismatch, cudaStream_t s);
cudaError_t align_kernel_launch(const AlignArgs& a, int grid, int threads, int min_blocks, size_t smem_bytes,
                                cudaStream_t s);
// The same kernel variants with the vk::ATANCamera projection (plsvo_align_atan_batch_run).  Weak references for the
// reason given at undistort_map_launch below: the host-pipeline model of the tests need not provide them, and the ATAN
// entry points then report them missing.  The library always links align_kernel.cu.
__attribute__((weak)) cudaError_t align_atan_kernel_prepare(int threads, int min_blocks, size_t smem_bytes, int* ctas_per_sm);
__attribute__((weak)) cudaError_t align_atan_kernel_launch(const AlignArgs& a, int grid, int threads, int min_blocks,
                                                           size_t smem_bytes, cudaStream_t s);
// The same kernel variants with per-pair pinhole intrinsics, AlignArgs::cams (plsvo_align_multicam_batch_run).  Weak for
// the same reason.  They hold the current pair's intrinsics in static shared memory, which the runtime reserves per CTA
// next to the dynamic region (128 bytes on sm_90a: the 32 of the intrinsics, padded to the dynamic region's alignment);
// align_multicam_kernel_static_smem reports the compiled size (cudaFuncAttributes::sharedSizeBytes), and the plan of
// these kernels (and of no other) takes it into account.
__attribute__((weak)) cudaError_t align_multicam_kernel_static_smem(int threads, int min_blocks, size_t* bytes);
__attribute__((weak)) cudaError_t align_multicam_kernel_prepare(int threads, int min_blocks, size_t smem_bytes,
                                                                int* ctas_per_sm);
__attribute__((weak)) cudaError_t align_multicam_kernel_launch(const AlignArgs& a, int grid, int threads, int min_blocks,
                                                               size_t smem_bytes, cudaStream_t s);
// The same kernel variants with a vk::ATANCamera per pair, AlignArgs::cams and AlignArgs::atan_terms
// (plsvo_align_atan_multicam_batch_run).  Weak for the same reason; their static shared memory (the pair's members, size
// and distortion terms, 72 bytes padded to 128 on sm_90a) is reported and planned for as for the multicam kernels.
__attribute__((weak)) cudaError_t align_atan_multicam_kernel_static_smem(int threads, int min_blocks, size_t* bytes);
__attribute__((weak)) cudaError_t align_atan_multicam_kernel_prepare(int threads, int min_blocks, size_t smem_bytes,
                                                                     int* ctas_per_sm);
__attribute__((weak)) cudaError_t align_atan_multicam_kernel_launch(const AlignArgs& a, int grid, int threads, int min_blocks,
                                                                    size_t smem_bytes, cudaStream_t s);
// The same kernel variants with a pinhole or ATAN camera per pair, AlignArgs::cams, atan_terms and cam_models
// (plsvo_align_any_camera_batch_run).  Weak for the same reason; their static shared memory (the pair's camera, size,
// distortion terms and model tag, 80 bytes padded to 128 on sm_90a) is planned for as for the multicam kernels.
__attribute__((weak)) cudaError_t align_any_camera_kernel_static_smem(int threads, int min_blocks, size_t* bytes);
__attribute__((weak)) cudaError_t align_any_camera_kernel_prepare(int threads, int min_blocks, size_t smem_bytes,
                                                                  int* ctas_per_sm);
__attribute__((weak)) cudaError_t align_any_camera_kernel_launch(const AlignArgs& a, int grid, int threads, int min_blocks,
                                                                 size_t smem_bytes, cudaStream_t s);

// ---------------------------------------------------------------------------------------------
struct PoseOptArgs {
  int B, n_pts, n_segs;
  double fx, reproj_thresh;
  int n_iter, n_iter_ref;
  const double* T_f_w;
  const int32_t* pt_count;
  const double* pt_f;
  const double* pt_pos;
  const int32_t* pt_level;
  const uint8_t* pt_valid;
  const int32_t* seg_count;
  const double* seg_line;
  const double* seg_spos;
  const double* seg_epos;
  const int32_t* seg_level;
  const uint8_t* seg_valid;
  double* out_T;
  double* out_cov;
  double* out_scale;
  double* out_err_init;
  double* out_err_final;
  long long* out_num_pt;
  long long* out_num_ls;
  uint8_t* out_pt_outlier;
  uint8_t* out_seg_outlier;
  int32_t* out_iters;
  int32_t* out_status;
  const double* fx_frame;  // [B] errorMultiplier2 of every frame (read by the multicam kernel only, instead of fx)
};
size_t poseopt_smem_bytes(int n_pts, int n_segs);
cudaError_t poseopt_kernel_launch(const PoseOptArgs& a, size_t smem_bytes, cudaStream_t s);
// The same kernel with a.fx_frame (plsvo_poseopt_multicam_batch_run, plsvo_track_multicam_batch_run).  Weak, as the
// alignment launchers above.
__attribute__((weak)) cudaError_t poseopt_multicam_kernel_launch(const PoseOptArgs& a, size_t smem_bytes, cudaStream_t s);


// ---------------------------------------------------------------------------------------------
struct PyramidArgs {
  int B, width, height, n_levels;  // n_levels <= 7 (64x64 level-0 tiles)
  uint8_t* level[PLSVO_MAX_LEVELS];  // device, [B][rows_l][pitch_l]; level[0] is the input
  uint32_t pitch[PLSVO_MAX_LEVELS];
  size_t stride[PLSVO_MAX_LEVELS];
};
cudaError_t pyramid_kernel_launch(const PyramidArgs& a, cudaStream_t s);

// ---------------------------------------------------------------------------------------------
// vk::PinholeCamera::undistortImage: the CV_16SC2 map of cv::initUndistortRectifyMap, then cv::remap INTER_LINEAR.
// The two launchers are weak references: plsvo_abi.cu is also compiled, unchanged, into the host-pipeline model of the
// tests, whose model kernels need not provide them; plsvo_undistort_batch_run then reports them missing.  The library
// always links undistort_kernel.cu.
constexpr int kRemapTileW = 64;  // map rows are padded to a multiple of this (whole tiles load without bounds checks)
struct UndistortMapArgs {
  int width, height, map_pitch;                 // map_pitch: entries per map row
  double fx, fy, cx, cy, k1, k2, p1, p2, k3;    // already rounded to float (vikit's Mat_<float> cvK_ / cvD_)
  short2* map1;                                 // [height][map_pitch] (x, y) source pixel
  uint16_t* map2;                               // [height][map_pitch] (iv & 31) * 32 + (iu & 31)
};
__attribute__((weak)) cudaError_t undistort_map_launch(const UndistortMapArgs& a, cudaStream_t s);

struct RemapArgs {
  int B, width, height, map_pitch;
  const short2* map1;
  const uint16_t* map2;
  const uint8_t* src;  // [B][height][src_pitch] raw frames (src_pitch multiple of 16)
  uint32_t src_pitch;
  size_t src_stride;
  uint8_t* dst;        // [B][height][dst_pitch] rectified frames: pyramid level 0 (dst_pitch multiple of 16)
  uint32_t dst_pitch;
  size_t dst_stride;
};
__attribute__((weak)) cudaError_t undistort_remap_launch(const RemapArgs& a, int num_sms, cudaStream_t s);

// Rectification and half-sampling in one kernel (the raw-frame alignment calls): each CTA forms a 64x64 tile of
// rectified level 0 from the raw frame with the remap arithmetic above (or copies it when map1 is NULL: no distortion),
// half-samples it down to n_levels - 1, and stores only the levels whose level[l] is non-NULL.  Weak for the same reason
// as the two launchers above.
struct RawPyramidArgs {
  int B, width, height, n_levels, map_pitch;       // n_levels <= 7
  const short2* map1;                              // NULL: copy the raw frame (fabs(d0) <= 1e-7)
  const uint16_t* map2;
  const uint8_t* src;                              // [B][height][src_pitch] raw frames
  size_t src_pitch, src_stride;
  uint8_t* level[PLSVO_MAX_LEVELS];                // [B][rows_l][pitch_l], or NULL: level not stored
  uint32_t pitch[PLSVO_MAX_LEVELS];                // multiples of 16
  size_t stride[PLSVO_MAX_LEVELS];
};
__attribute__((weak)) cudaError_t undistort_pyramid_launch(const RawPyramidArgs& a, int num_sms, cudaStream_t s);
struct RawVisit {           // one frame of a multicam raw batch and the map it is rectified with
  const short2* map1;       // its camera's map ([height][map_pitch], as RawPyramidArgs::map1), or NULL: copy the frame
  const uint16_t* map2;
  int32_t frame;            // index into src and every level
  int32_t width, height;    // its camera's image size: the frame's region in the top-left corner of the slot
  int32_t map_pitch;        // entries per row of its camera's map
};
// The same kernel for frames of several cameras (plsvo_*_raw_multicam_batch_run): visit[0..a.B) lists every frame once,
// in the order the CTAs' frame runs take them, each with its camera's map and size (a.map1 / a.map2 / a.map_pitch are
// not read).  a.width x a.height is the slot: every frame's camera fits in it, and a frame's raw image and levels occupy
// their camera's size in the slot's top-left corner.  The kernel writes nothing of a level outside that region.
__attribute__((weak)) cudaError_t undistort_pyramid_multicam_launch(const RawPyramidArgs& a, const RawVisit* visit, int num_sms,
                                                                    cudaStream_t s);


// ---------------------------------------------------------------------------------------------
struct Align2DArgs {
  int n, n_iter, width, height;
  const uint8_t* img[PLSVO_MAX_LEVELS];  // device, [n_images][rows_l][pitch_l]
  uint32_t pitch[PLSVO_MAX_LEVELS];
  size_t stride[PLSVO_MAX_LEVELS];
  const int32_t* image_index;
  const int32_t* level;
  const uint8_t* ref_patch_with_border;  // [n][100]
  const uint8_t* ref_patch;              // [n][64]
  const double* px;                      // [n][2]
  double* out_px;
  uint8_t* out_converged;
  const float* dir;   // align1D only: [n][2]
  double* out_h_inv;  // align1D only: [n]
};
cudaError_t align2d_kernel_launch(const Align2DArgs& a, cudaStream_t s);
cudaError_t align1d_kernel_launch(const Align2DArgs& a, cudaStream_t s);

// ---------------------------------------------------------------------------------------------
// One camera of the per-image kernel, as the host derives it from a plsvo_match_camera: the pinhole's fx..cy, or the
// vk::ATANCamera members fx_..cy_ and distortion terms s_, s_inv_, tans_, tans_inv_ (zero for a pinhole).
struct MatchCamRecord {
  double fx, fy, cx, cy;
  int32_t width, height;
  int32_t model, reserved;  // PLSVO_CAMERA_PINHOLE or PLSVO_CAMERA_ATAN
  double s, s_inv, tans, tans_inv;
};
struct MatchArgs {
  int n, n_iter, n_pyr_levels, width, height;
  double fx, fy, cx, cy;
  const uint8_t* ref_img[PLSVO_MAX_LEVELS];  // device, [n_ref][rows_l][pitch_l]
  uint32_t ref_pitch[PLSVO_MAX_LEVELS];
  size_t ref_stride[PLSVO_MAX_LEVELS];
  const uint8_t* cur_img[PLSVO_MAX_LEVELS];
  uint32_t cur_pitch[PLSVO_MAX_LEVELS];
  size_t cur_stride[PLSVO_MAX_LEVELS];
  const double* T_ref_w;  // [n_ref][7]
  const double* T_cur_w;  // [n_cur][7]
  const int32_t* ref_index;
  const int32_t* cur_index;
  const double* ref_px;
  const double* ref_f;
  const int32_t* ref_level;
  const uint8_t* is_edgelet;  // may be null
  const double* ref_grad;     // may be null
  const double* pos;
  const double* px_cur;
  double* out_px;
  uint8_t* out_success;
  int32_t* out_level;
  double* out_A;  // [n][4] or null
  // vk::ATANCamera distortion (read by the ATAN kernel only; fx, fy, cx, cy above then hold fx_, fy_, cx_, cy_):
  // s_ = d0, s_inv_ = 1/s_, tans_ = 2 tan(s_/2), tans_inv_ = 1/tans_, all zero when s_ == 0
  double atan_s, atan_s_inv, atan_tans, atan_tans_inv;
  // A camera per image (the per-image kernel only; width / height above are then the slot): image r of the keyframes
  // is seen through cams[cam_of_ref[r]], image c of the current frames through cams[cam_of_cur[c]]
  const MatchCamRecord* cams;  // device, [n_cams]
  const int32_t* cam_of_ref;          // device, [n_ref_images]
  const int32_t* cam_of_cur;          // device, [n_cur_images]
};
cudaError_t match_direct_kernel_launch(const MatchArgs& a, cudaStream_t s);
// The same kernel with the vk::ATANCamera warp matrix (plsvo_match_direct_atan_batch_run).  Weak, as the ATAN alignment
// launchers: the host-pipeline model of the tests need not provide it, and the ATAN entry point then reports it missing.
__attribute__((weak)) cudaError_t match_direct_atan_kernel_launch(const MatchArgs& a, cudaStream_t s);
// The same kernel with a camera per image (plsvo_match_direct_multicam_batch_run).  Weak, for the same reason.
__attribute__((weak)) cudaError_t match_direct_multicam_kernel_launch(const MatchArgs& a, cudaStream_t s);

// ---------------------------------------------------------------------------------------------
struct SeedArgs {
  int n, n_iter, n_pyr_levels, width, height, max_epi_search_steps;
  int spw;           // seeds per warp; -1: chosen by the launch functions from the batch size
  int serial_steps;  // steps of an epipolar search walked by the seed's own thread before the warp takes over; -1: automatic
  int align_1d, subpix_refinement, edgelet_filtering;
  double edgelet_max_angle, convergence_thresh;
  double fx, fy, cx, cy;
  const uint8_t* ref_img[PLSVO_MAX_LEVELS];
  uint32_t ref_pitch[PLSVO_MAX_LEVELS];
  size_t ref_stride[PLSVO_MAX_LEVELS];
  const uint8_t* cur_img[PLSVO_MAX_LEVELS];
  uint32_t cur_pitch[PLSVO_MAX_LEVELS];
  size_t cur_stride[PLSVO_MAX_LEVELS];
  const double* T_ref_w;
  const double* T_cur_w;
  const int32_t* ref_index;
  const int32_t* cur_index;
  const double* ref_px;
  const double* ref_f;
  const int32_t* ref_level;
  const uint8_t* is_edgelet;  // may be null
  const double* ref_grad;     // may be null
  const float* a;
  const float* b;
  const float* mu;
  const float* z_range;
  const float* sigma2;
  // line seeds only
  const double* ref_sf;
  const double* ref_ef;
  const float* mu_e;
  const float* z_range_e;
  const float* sigma2_e;
  float* out_mu_e;
  float* out_sigma2_e;
  double* out_depth_e;
  double* out_px_cur_e;  // [n][2]
  float* out_a;
  float* out_b;
  float* out_mu;
  float* out_sigma2;
  int32_t* out_status;
  uint8_t* out_converged;
  double* out_depth;
  double* out_px_cur;
};
cudaError_t seed_update_kernel_launch(const SeedArgs& a, cudaStream_t s);
cudaError_t line_seed_update_kernel_launch(const SeedArgs& a, cudaStream_t s);

// ---------------------------------------------------------------------------------------------
struct StructOptArgs {
  int n_points, n_segs, n_iter_pts, n_iter_segs;
  const double* T_f_w;
  const int32_t* pt_obs_begin;
  const int32_t* pt_obs_frame;
  const double* pt_obs_f;
  const double* pt_pos;
  const int32_t* seg_obs_begin;
  const int32_t* seg_obs_frame;
  const double* seg_obs_sf;
  const double* seg_obs_ef;
  const double* seg_spos;
  const double* seg_epos;
  double* out_pt_pos;
  double* out_seg_spos;
  double* out_seg_epos;
  int32_t* out_pt_iters;
  int32_t* out_seg_iters;
};
cudaError_t structopt_kernel_launch(const StructOptArgs& a, cudaStream_t s);

}  // namespace plsvo
