// fake_any_camera.cpp — model kernels of the any-camera calls (a pinhole or ATAN camera per pair, chosen by a model tag,
// frames of the pair's own size in slots of the batch's size) and of the pinhole multicam calls they are compared with,
// for the host-pipeline model.  TEST INFRASTRUCTURE ONLY (see fake_cuda.h).  tests/test_gpu_any_camera.py links it into a
// model library of its own, next to the stock model kernels and fake_atan_multicam.cpp (the ATAN multicam launchers and
// the per-frame pose optimiser); plsvo_abi.cu reaches all of them through weak references.
//
//   alignment : every pair as a batch of one through the stock model's pinhole or ATAN launcher, by its tag
//               (a.cam_models[b]), at its camera's size (a.cams[b].width x height, which must fit the slot) with its own
//               fx..cy (a.cams[b]) and, for an ATAN pair, its distortion terms (a.atan_terms[b]), which must be those
//               vk::ATANCamera derives from s_.  The pinhole multicam launcher is the same with every tag pinhole.  In
//               digest mode the digest covers the pair's own region of every level; with PLSVO_FAKE_ORACLE the pair is
//               answered by its model's oracle with its own camera, so a pair handed another pair's camera, terms or
//               model differs from its model's per-pair call.
#include <math.h>
#include <string.h>

#include "../../pl-svo_b200/csrc/internal.h"
#include "fake_cuda.h"

namespace plsvo {

namespace {
template <class T>
void move(T*& ptr, size_t n) {
  if (ptr) ptr += n;
}

// pair b of a per-pair batch as a uniform batch of one at its camera's size, with its camera (and, ATAN, its terms)
AlignArgs one_pair(const AlignArgs& a, int b, bool atan) {
  AlignArgs p = a;
  const size_t np = (size_t)a.n_pts, ns = (size_t)a.n_segs, pb = (size_t)b;
  p.B = 1;
  const plsvo_camera& k = a.cams[b];
  p.width = k.width, p.height = k.height, p.fx = k.fx, p.fy = k.fy, p.cx = k.cx, p.cy = k.cy;
  p.atan_s = p.atan_s_inv = p.atan_tans = p.atan_tans_inv = 0.0;
  if (atan) {
    const double* t = a.atan_terms + 4 * pb;
    p.atan_s = t[0], p.atan_s_inv = t[1], p.atan_tans = t[2], p.atan_tans_inv = t[3];
  }
  p.cams = nullptr, p.atan_terms = nullptr, p.cam_models = nullptr;
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

// The pairs' cameras are device data the host uploaded on `s` before this launch: the stream catches up first so that
// they can be read here, then every pair is one launch of the stock model kernel of its model, the work counter cleared
// in between as the host clears it before a launch.  any: the tags and terms are read (the any-camera kernels); else
// every pair is pinhole (the pinhole multicam kernels).
cudaError_t launch_per_pair(const AlignArgs& a, int grid, int threads, int min_blocks, size_t smem_bytes, cudaStream_t s, bool any) {
  cudaError_t e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return e;
  const char* what = any ? "any-camera align kernel" : "multicam align kernel";
  if (!fakecuda::check(a.cams, (size_t)a.B * sizeof(plsvo_camera), what)) return cudaErrorIllegalAddress;
  if (any && (!fakecuda::check(a.cam_models, (size_t)a.B * sizeof(int32_t), "any-camera align kernel: cam_models") ||
              !fakecuda::check(a.atan_terms, (size_t)a.B * 4 * sizeof(double), "any-camera align kernel: atan_terms")))
    return cudaErrorIllegalAddress;
  for (int b = 0; b < a.B; ++b) {
    const plsvo_camera& k = a.cams[b];
    if (k.width < 1 || k.height < 1 || k.width > a.width || k.height > a.height) {
      fakecuda::error("per-pair align kernel: a pair's camera does not fit the slot");
      return cudaErrorInvalidValue;
    }
    const int model = any ? a.cam_models[b] : PLSVO_CAMERA_PINHOLE;
    if (model != PLSVO_CAMERA_PINHOLE && model != PLSVO_CAMERA_ATAN) {
      fakecuda::error("any-camera align kernel: a pair's model tag is neither pinhole nor ATAN");
      return cudaErrorInvalidValue;
    }
    if (model == PLSVO_CAMERA_ATAN) {
      const double* t = a.atan_terms + 4 * (size_t)b;
      const double tans = t[0] != 0.0 ? 2.0 * tan(t[0] / 2.0) : 0.0;
      if (!same_bits(t[1], t[0] != 0.0 ? 1.0 / t[0] : 0.0) || !same_bits(t[2], tans) || !same_bits(t[3], t[0] != 0.0 ? 1.0 / tans : 0.0)) {
        fakecuda::error("any-camera align kernel: an ATAN pair's distortion terms are not those vk::ATANCamera derives from its s_");
        return cudaErrorInvalidValue;
      }
    }
    if (b > 0) {
      unsigned int* wc = a.work_counter;
      e = fakecuda::enqueue(s, [wc]() {
        if (fakecuda::check(wc, 4, "work counter")) *wc = 0;
        return true;
      });
      if (e != cudaSuccess) return e;
    }
    const bool atan = model == PLSVO_CAMERA_ATAN;
    e = atan ? align_atan_kernel_launch(one_pair(a, b, true), grid, threads, min_blocks, smem_bytes, s)
             : align_kernel_launch(one_pair(a, b, false), grid, threads, min_blocks, smem_bytes, s);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}
}  // namespace

cudaError_t align_multicam_kernel_static_smem(int, int, size_t* bytes) {
  *bytes = 128;
  return cudaSuccess;
}

cudaError_t align_multicam_kernel_prepare(int threads, int min_blocks, size_t smem_bytes, int* ctas_per_sm) {
  return align_kernel_prepare(threads, min_blocks, smem_bytes, ctas_per_sm);
}

cudaError_t align_multicam_kernel_launch(const AlignArgs& a, int grid, int threads, int min_blocks, size_t smem_bytes, cudaStream_t s) {
  return launch_per_pair(a, grid, threads, min_blocks, smem_bytes, s, false);
}

cudaError_t align_any_camera_kernel_static_smem(int, int, size_t* bytes) {
  *bytes = 128;
  return cudaSuccess;
}

cudaError_t align_any_camera_kernel_prepare(int threads, int min_blocks, size_t smem_bytes, int* ctas_per_sm) {
  return align_kernel_prepare(threads, min_blocks, smem_bytes, ctas_per_sm);
}

cudaError_t align_any_camera_kernel_launch(const AlignArgs& a, int grid, int threads, int min_blocks, size_t smem_bytes,
                                           cudaStream_t s) {
  return launch_per_pair(a, grid, threads, min_blocks, smem_bytes, s, true);
}

}  // namespace plsvo
