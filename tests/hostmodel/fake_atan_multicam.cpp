// fake_atan_multicam.cpp — model kernels of the ATAN multicam calls (a vk::ATANCamera per pair, frames of the pair's own
// size in slots of the batch's size) for the host-pipeline model.  TEST INFRASTRUCTURE ONLY (see fake_cuda.h).
// tests/test_gpu_atan_multicam.py links it into a model library of its own, next to the stock model kernels; the stock
// model lacks these launchers, and plsvo_abi.cu reaches them through weak references.
//
//   alignment      : every pair as a batch of one through the stock model's ATAN launcher, at its camera's size
//                    (a.cams[b].width x height, which must fit the slot) with its own members fx_..cy_ (a.cams[b]) and
//                    distortion terms (a.atan_terms[b]), which must be those vk::ATANCamera derives from s_.  In digest
//                    mode the digest covers the pair's own region of every level; with PLSVO_FAKE_ORACLE the pair is
//                    answered by plsvo_oracle_atan_align_batch_members with its own camera, so a pair handed another
//                    pair's camera differs from the one-camera call on its group.
//   pose optimiser : digest mode: the stock digest, after the per-frame fx have been bounds-checked.  The digest does not
//                    cover fx, so in the lazy and eager digest runs a wrong errorMultiplier2 goes unnoticed.  With
//                    PLSVO_FAKE_ORACLE every frame is a batch of one through the stock launcher with fx = fx_frame[b], so a
//                    frame handed the wrong errorMultiplier2 differs from the one-camera track call: only that mode
//                    catches such a fault.
#include <math.h>
#include <string.h>
#include <stdlib.h>

#include "../../pl-svo_b200/csrc/internal.h"
#include "fake_cuda.h"

namespace plsvo {

cudaError_t align_atan_multicam_kernel_static_smem(int, int, size_t* bytes) {
  *bytes = 128;
  return cudaSuccess;
}

cudaError_t align_atan_multicam_kernel_prepare(int threads, int min_blocks, size_t smem_bytes, int* ctas_per_sm) {
  return align_kernel_prepare(threads, min_blocks, smem_bytes, ctas_per_sm);
}

namespace {
template <class T>
void move(T*& ptr, size_t n) {
  if (ptr) ptr += n;
}

// pair b of an ATAN multicam batch as a uniform ATAN batch of one at its camera's size, with its camera's members
AlignArgs one_pair(const AlignArgs& a, int b) {
  AlignArgs p = a;
  const size_t np = (size_t)a.n_pts, ns = (size_t)a.n_segs, pb = (size_t)b;
  p.B = 1;
  const plsvo_camera& k = a.cams[b];
  p.width = k.width, p.height = k.height, p.fx = k.fx, p.fy = k.fy, p.cx = k.cx, p.cy = k.cy;
  const double* t = a.atan_terms + 4 * pb;
  p.atan_s = t[0], p.atan_s_inv = t[1], p.atan_tans = t[2], p.atan_tans_inv = t[3];
  p.cams = nullptr, p.atan_terms = nullptr;
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) move(p.ref_img[l], pb * a.stride[l]), move(p.cur_img[l], pb * a.stride[l]);
  move(p.T_ref_w, 7 * pb), move(p.T_cur_w, 7 * pb), move(p.pt_count, pb), move(p.seg_count, pb);
  move(p.pt_px, 2 * np * pb), move(p.pt_f, 3 * np * pb), move(p.pt_pos, 3 * np * pb), move(p.pt_valid, np * pb), move(p.pt_depth, np * pb);
  move(p.seg_spx, 2 * ns * pb), move(p.seg_epx, 2 * ns * pb), move(p.seg_sf, 3 * ns * pb), move(p.seg_ef, 3 * ns * pb);
  move(p.seg_spos, 3 * ns * pb), move(p.seg_epos, 3 * ns * pb), move(p.seg_length, ns * pb), move(p.seg_valid, ns * pb);
  move(p.seg_sdepth, ns * pb), move(p.seg_edepth, ns * pb);
  move(p.out_T, 7 * pb), move(p.out_n_tracked, pb), move(p.out_H, 36 * pb), move(p.out_seg_killed, ns * pb);
  move(p.out_iters, (size_t)PLSVO_MAX_LEVELS * pb), move(p.out_status, pb), move(p.out_patch_iters, pb), move(p.out_patch_levels, pb);
  return p;
}

bool same_bits(double x, double y) { return memcmp(&x, &y, sizeof x) == 0; }
}  // namespace

// The pairs' cameras are device data the host uploaded on `s` before this launch: the stream catches up first so that
// they can be read here, then every pair is one launch of the stock ATAN model kernel, the work counter cleared in between
// as the host clears it before a launch.
cudaError_t align_atan_multicam_kernel_launch(const AlignArgs& a, int grid, int threads, int min_blocks, size_t smem_bytes,
                                              cudaStream_t s) {
  cudaError_t e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return e;
  if (!fakecuda::check(a.cams, (size_t)a.B * sizeof(plsvo_camera), "ATAN multicam align kernel: cams") ||
      !fakecuda::check(a.atan_terms, (size_t)a.B * 4 * sizeof(double), "ATAN multicam align kernel: atan_terms"))
    return cudaErrorIllegalAddress;
  for (int b = 0; b < a.B; ++b) {
    const plsvo_camera& k = a.cams[b];
    if (k.width < 1 || k.height < 1 || k.width > a.width || k.height > a.height) {
      fakecuda::error("ATAN multicam align kernel: a pair's camera does not fit the slot");
      return cudaErrorInvalidValue;
    }
    const double* t = a.atan_terms + 4 * (size_t)b;
    const double tans = t[0] != 0.0 ? 2.0 * tan(t[0] / 2.0) : 0.0;
    if (!same_bits(t[1], t[0] != 0.0 ? 1.0 / t[0] : 0.0) || !same_bits(t[2], tans) || !same_bits(t[3], t[0] != 0.0 ? 1.0 / tans : 0.0)) {
      fakecuda::error("ATAN multicam align kernel: a pair's distortion terms are not those vk::ATANCamera derives from its s_");
      return cudaErrorInvalidValue;
    }
    if (b > 0) {
      unsigned int* wc = a.work_counter;
      e = fakecuda::enqueue(s, [wc]() {
        if (fakecuda::check(wc, 4, "work counter")) *wc = 0;
        return true;
      });
      if (e != cudaSuccess) return e;
    }
    e = align_atan_kernel_launch(one_pair(a, b), grid, threads, min_blocks, smem_bytes, s);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t poseopt_multicam_kernel_launch(const PoseOptArgs& a, size_t smem_bytes, cudaStream_t s) {
  cudaError_t e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return e;
  if (!fakecuda::check(a.fx_frame, (size_t)a.B * sizeof(double), "multicam pose-optimiser kernel: fx_frame"))
    return cudaErrorIllegalAddress;
  const char* orc = getenv("PLSVO_FAKE_ORACLE");
  if (!orc || !*orc) return poseopt_kernel_launch(a, smem_bytes, s);
  const size_t np = (size_t)a.n_pts, ns = (size_t)a.n_segs, npo = np ? np : 1, nso = ns ? ns : 1;
  for (int b = 0; b < a.B; ++b) {
    PoseOptArgs p = a;
    const size_t pb = (size_t)b;
    p.B = 1, p.fx = a.fx_frame[b], p.fx_frame = nullptr;
    move(p.T_f_w, 7 * pb), move(p.pt_count, pb), move(p.seg_count, pb);
    move(p.pt_f, 3 * np * pb), move(p.pt_pos, 3 * np * pb), move(p.pt_level, np * pb), move(p.pt_valid, np * pb);
    move(p.seg_line, 3 * ns * pb), move(p.seg_spos, 3 * ns * pb), move(p.seg_epos, 3 * ns * pb), move(p.seg_level, ns * pb);
    move(p.seg_valid, ns * pb);
    move(p.out_T, 7 * pb), move(p.out_cov, 36 * pb), move(p.out_scale, pb), move(p.out_err_init, pb), move(p.out_err_final, pb);
    move(p.out_num_pt, pb), move(p.out_num_ls, pb), move(p.out_pt_outlier, npo * pb), move(p.out_seg_outlier, nso * pb);
    move(p.out_iters, 2 * pb), move(p.out_status, pb);
    e = poseopt_kernel_launch(p, smem_bytes, s);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace plsvo
