// fake_raw_multicam.cpp — model kernels of the raw multicam calls for the host-pipeline model.  TEST INFRASTRUCTURE ONLY
// (see fake_cuda.h).  tests/test_raw_multicam.py links it, with fake_undistort.cpp and fake_raw_pyramid.cpp, into a
// model library of its own; the stock model lacks these launchers, and plsvo_abi.cu reaches them through weak references.
//
//   undistort_pyramid_multicam : the real computation of undistort_pyramid_kernel, frame by frame in the visit order, each
//                                frame with the map its visit record names (or a copy).  Every frame must be visited
//                                exactly once; every map is bounds-checked against its own device block, and a map
//                                entry no map kernel has written (the model's 0xCD poison) is an error.
//   alignment / pose optimiser : the digest kernels of fake_kernels.cpp, after the per-pair intrinsics / per-frame fx
//                                have been bounds-checked.  The digest does not cover the intrinsics; the -m gpu tests
//                                compare the real kernels' results.
#include <vector>

#include "../../pl-svo_b200/csrc/internal.h"
#include "fake_cuda.h"

namespace plsvo {

cudaError_t undistort_pyramid_multicam_launch(const RawPyramidArgs& a0, const RawVisit* visit, int, cudaStream_t s) {
  const RawPyramidArgs a = a0;
  return fakecuda::enqueue(s, [a, visit]() {
    const int W = a.width, H = a.height;
    if (!fakecuda::check(visit, (size_t)a.B * sizeof(RawVisit), "raw multicam pyramid kernel: visit list")) return true;
    std::vector<int> seen((size_t)a.B, 0);
    std::vector<uint8_t> cur((size_t)W * H), next;
    for (int i = 0; i < a.B; ++i) {
      const RawVisit v = visit[i];
      if (v.frame < 0 || v.frame >= a.B || seen[v.frame]++) {
        fakecuda::error("raw multicam pyramid kernel: the visit list does not name every frame exactly once");
        return true;
      }
      const int b = v.frame;
      const size_t mspan = (size_t)(H - 1) * a.map_pitch + W;
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
          const size_t e = (size_t)y * a.map_pitch + x;
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
      cur.assign((size_t)W * H, 0);
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

cudaError_t align_multicam_kernel_launch(const AlignArgs& a, int grid, int threads, int min_blocks, size_t smem_bytes, cudaStream_t s) {
  const AlignArgs args = a;
  cudaError_t e = fakecuda::enqueue(s, [args]() {
    fakecuda::check(args.cams, (size_t)args.B * sizeof(plsvo_camera), "multicam align kernel: cams");
    return true;
  });
  return e != cudaSuccess ? e : align_kernel_launch(a, grid, threads, min_blocks, smem_bytes, s);
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
