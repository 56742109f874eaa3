// fake_mixed_sizes.cpp — model kernels of the multicam calls with per-pair image sizes (frames smaller than the batch's
// slot) for the host-pipeline model.  TEST INFRASTRUCTURE ONLY (see fake_cuda.h).  tests/test_gpu_mixed_sizes.py links it,
// with fake_undistort.cpp and fake_raw_pyramid.cpp, into a model library of its own, in place of fake_raw_multicam.cpp
// (whose kernels work at the slot's size, which is every frame's size in the batches of tests/test_raw_multicam.py); the
// stock model lacks these launchers, and plsvo_abi.cu reaches them through weak references.
//
//   undistort_pyramid_multicam : the real computation of undistort_pyramid_kernel, frame by frame in the visit order, each
//                                frame at its visit record's camera size (which must fit the slot, a.width x a.height)
//                                with the map the record names (or a copy).  Every frame must be visited exactly once;
//                                every map is bounds-checked, at the record's map pitch, against its own device block,
//                                and a map entry no map kernel has written (the model's 0xCD poison) is an error.  Only
//                                the frame's own region of every level is written, as the real kernel does.
//   alignment                  : the digest kernel of fake_kernels.cpp run pair by pair, each pair as a batch of one at
//                                its camera's size (a.cams[b].width x height, which must fit the slot): the digest
//                                covers the pair's own region of every level and nothing of the slot's padding.  The
//                                digest does not cover the intrinsics; the -m gpu tests compare the real kernels' results.
//   pose optimiser             : the digest kernel of fake_kernels.cpp, after the per-frame fx have been bounds-checked.
#include <vector>

#include "../../pl-svo_b200/csrc/internal.h"
#include "fake_cuda.h"

namespace plsvo {

cudaError_t undistort_pyramid_multicam_launch(const RawPyramidArgs& a0, const RawVisit* visit, int, cudaStream_t s) {
  const RawPyramidArgs a = a0;
  return fakecuda::enqueue(s, [a, visit]() {
    if (!fakecuda::check(visit, (size_t)a.B * sizeof(RawVisit), "raw multicam pyramid kernel: visit list")) return true;
    std::vector<int> seen((size_t)a.B, 0);
    std::vector<uint8_t> cur, next;
    for (int i = 0; i < a.B; ++i) {
      const RawVisit v = visit[i];
      if (v.frame < 0 || v.frame >= a.B || seen[v.frame]++) {
        fakecuda::error("raw multicam pyramid kernel: the visit list does not name every frame exactly once");
        return true;
      }
      const int b = v.frame, W = v.width, H = v.height;
      if (W < 1 || H < 1 || W > a.width || H > a.height || v.map_pitch < W || v.map_pitch % 64 != 0) {
        fakecuda::error("raw multicam pyramid kernel: a frame's size does not fit the slot, or its map pitch is not whole tiles");
        return true;
      }
      cur.assign((size_t)W * H, 0);
      // the real kernel reads whole 64-entry tiles of every map row the frame covers
      const size_t mspan = (size_t)(H - 1) * v.map_pitch + (size_t)(W + 63) / 64 * 64;
      if (v.map1) {
        if (!fakecuda::check(v.map1, mspan * sizeof(short2), "raw multicam pyramid kernel: map1") ||
            !fakecuda::check(v.map2, mspan * 2, "raw multicam pyramid kernel: map2"))
          return true;
      }
      const uint8_t* src = a.src + (size_t)b * a.src_stride;
      if (!fakecuda::check(src, (size_t)(H - 1) * a.src_pitch + W, "raw multicam pyramid kernel: raw frame")) return true;
      auto px = [&](int x, int y) -> uint32_t {
        return ((unsigned)x < (unsigned)W && (unsigned)y < (unsigned)H) ? src[(size_t)y * a.src_pitch + x] : 0u;
      };
      for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
          if (!v.map1) {
            cur[(size_t)y * W + x] = (uint8_t)px(x, y);
            continue;
          }
          const size_t e = (size_t)y * v.map_pitch + x;
          if (v.map2[e] >= 1024) {  // m2 = (iv & 31) * 32 + (iu & 31)
            fakecuda::error("raw multicam pyramid kernel: reads a map entry no map kernel has written");
            return true;
          }
          const int sx = v.map1[e].x, sy = v.map1[e].y, fa = v.map2[e] & 31, fb = v.map2[e] >> 5;
          const uint32_t w = px(sx, sy) * (32 - fa) * (32 - fb) + px(sx + 1, sy) * fa * (32 - fb) + px(sx, sy + 1) * (32 - fa) * fb +
                             px(sx + 1, sy + 1) * fa * fb;
          cur[(size_t)y * W + x] = (uint8_t)((w * 32 + (1u << 14)) >> 15);
        }
      int cols = W, rows = H;
      for (int l = 0; l < a.n_levels; ++l) {
        if (l > 0) {  // vk::halfSample of the previous level
          const int c2 = cols >> 1, r2 = rows >> 1;
          next.assign((size_t)c2 * r2, 0);
          for (int y = 0; y < r2; ++y)
            for (int x = 0; x < c2; ++x) {
              const uint8_t* p = cur.data() + (size_t)(2 * y) * cols + 2 * x;
              next[(size_t)y * c2 + x] = (uint8_t)(((int)p[0] + (int)p[1] + (int)p[cols] + (int)p[cols + 1]) / 4);
            }
          cur.swap(next);
          cols = c2, rows = r2;
        }
        if (!a.level[l]) continue;
        uint8_t* dst = a.level[l] + (size_t)b * a.stride[l];
        if (a.pitch[l] % 16 != 0) fakecuda::error("raw multicam pyramid kernel: level pitch not a multiple of 16");
        if (!fakecuda::check(dst, a.stride[l], "raw multicam pyramid kernel: output level")) return true;
        for (int y = 0; y < rows; ++y)
          for (int x = 0; x < cols; ++x) dst[(size_t)y * a.pitch[l] + x] = cur[(size_t)y * cols + x];
      }
    }
    return true;
  });
}

cudaError_t align_multicam_kernel_static_smem(int, int, size_t* bytes) {
  *bytes = 128;
  return cudaSuccess;
}

cudaError_t align_multicam_kernel_prepare(int threads, int min_blocks, size_t smem_bytes, int* ctas_per_sm) {
  return align_kernel_prepare(threads, min_blocks, smem_bytes, ctas_per_sm);
}

namespace {
// pair b of a multicam batch as a batch of one at its camera's size: every per-pair pointer moved to the pair's entry
AlignArgs one_pair(const AlignArgs& a, int b) {
  AlignArgs p = a;
  const size_t np = (size_t)a.n_pts, ns = (size_t)a.n_segs, pb = (size_t)b;
  auto move = [](auto*& ptr, size_t n) {
    if (ptr) ptr += n;
  };
  p.B = 1;
  p.width = a.cams[b].width, p.height = a.cams[b].height;
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) move(p.ref_img[l], pb * a.stride[l]), move(p.cur_img[l], pb * a.stride[l]);
  move(p.T_ref_w, 7 * pb), move(p.T_cur_w, 7 * pb), move(p.pt_count, pb), move(p.seg_count, pb);
  move(p.pt_px, 2 * np * pb), move(p.pt_f, 3 * np * pb), move(p.pt_pos, 3 * np * pb), move(p.pt_valid, np * pb), move(p.pt_depth, np * pb);
  move(p.seg_spx, 2 * ns * pb), move(p.seg_epx, 2 * ns * pb), move(p.seg_sf, 3 * ns * pb), move(p.seg_ef, 3 * ns * pb);
  move(p.seg_spos, 3 * ns * pb), move(p.seg_epos, 3 * ns * pb), move(p.seg_length, ns * pb), move(p.seg_valid, ns * pb);
  move(p.seg_sdepth, ns * pb), move(p.seg_edepth, ns * pb);
  move(p.out_T, 7 * pb), move(p.out_n_tracked, pb), move(p.out_H, 36 * pb), move(p.out_seg_killed, ns * pb);
  move(p.out_iters, (size_t)PLSVO_MAX_LEVELS * pb), move(p.out_status, pb), move(p.out_patch_iters, pb), move(p.out_patch_levels, pb);
  move(p.cams, pb);
  return p;
}
}  // namespace

// The pairs' sizes are device data the host uploaded on `s` before this launch: the stream catches up first so that they
// can be read here, then every pair is one launch of the digest kernel, the work counter cleared in between as the host
// clears it before a launch.
cudaError_t align_multicam_kernel_launch(const AlignArgs& a, int grid, int threads, int min_blocks, size_t smem_bytes, cudaStream_t s) {
  cudaError_t e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return e;
  if (!fakecuda::check(a.cams, (size_t)a.B * sizeof(plsvo_camera), "multicam align kernel: cams")) return cudaErrorIllegalAddress;
  for (int b = 0; b < a.B; ++b) {
    const plsvo_camera& k = a.cams[b];
    if (k.width < 1 || k.height < 1 || k.width > a.width || k.height > a.height) {
      fakecuda::error("multicam align kernel: a pair's camera does not fit the slot");
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
    e = align_kernel_launch(one_pair(a, b), grid, threads, min_blocks, smem_bytes, s);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t poseopt_multicam_kernel_launch(const PoseOptArgs& a, size_t smem_bytes, cudaStream_t s) {
  const PoseOptArgs args = a;
  cudaError_t e = fakecuda::enqueue(s, [args]() {
    fakecuda::check(args.fx_frame, (size_t)args.B * sizeof(double), "multicam pose-optimiser kernel: fx_frame");
    return true;
  });
  return e != cudaSuccess ? e : poseopt_kernel_launch(a, smem_bytes, s);
}

}  // namespace plsvo
