// fake_raw_pyramid.cpp — model kernel of the fused rectify + pyramid launcher for the host-pipeline model.  TEST
// INFRASTRUCTURE ONLY (see fake_cuda.h).  tests/test_raw_track.py links it, with fake_undistort.cpp, into a model library
// of its own; the stock model lacks the launcher, and plsvo_abi.cu reaches it through a weak reference.
//
//   undistort_pyramid : the real computation: fixed-point bilinear on the map it is given (or a copy of the raw frame
//                       when there is no map), then the truncating 2x2 mean level by level; only the levels it is given
//                       are stored.
// Every byte the real kernel would read or write is bounds-checked against the model's device blocks.
#include <vector>

#include "../../pl-svo_b200/csrc/internal.h"
#include "fake_cuda.h"

namespace plsvo {

cudaError_t undistort_pyramid_launch(const RawPyramidArgs& a0, int, cudaStream_t s) {
  const RawPyramidArgs a = a0;
  return fakecuda::enqueue(s, [a]() {
    const int W = a.width, H = a.height;
    if (a.map1) {
      const size_t mspan = (size_t)(H - 1) * a.map_pitch + W;
      if (!fakecuda::check(a.map1, mspan * sizeof(short2), "raw pyramid kernel: map1") ||
          !fakecuda::check(a.map2, mspan * 2, "raw pyramid kernel: map2"))
        return true;
    }
    std::vector<uint8_t> cur((size_t)W * H), next;
    for (int b = 0; b < a.B; ++b) {
      const uint8_t* src = a.src + (size_t)b * a.src_stride;
      if (!fakecuda::check(src, (size_t)(H - 1) * a.src_pitch + W, "raw pyramid kernel: raw frame")) return true;
      auto px = [&](int x, int y) -> uint32_t {
        return ((unsigned)x < (unsigned)W && (unsigned)y < (unsigned)H) ? src[(size_t)y * a.src_pitch + x] : 0u;
      };
      for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
          if (!a.map1) {
            cur[(size_t)y * W + x] = (uint8_t)px(x, y);
            continue;
          }
          const size_t e = (size_t)y * a.map_pitch + x;
          const int sx = a.map1[e].x, sy = a.map1[e].y, fa = a.map2[e] & 31, fb = a.map2[e] >> 5;
          const uint32_t v = px(sx, sy) * (32 - fa) * (32 - fb) + px(sx + 1, sy) * fa * (32 - fb) + px(sx, sy + 1) * (32 - fa) * fb +
                             px(sx + 1, sy + 1) * fa * fb;
          cur[(size_t)y * W + x] = (uint8_t)((v * 32 + (1u << 14)) >> 15);
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
        if (a.pitch[l] % 16 != 0) fakecuda::error("raw pyramid kernel: level pitch not a multiple of 16");
        if (!fakecuda::check(dst, a.stride[l], "raw pyramid kernel: output level")) return true;
        for (int y = 0; y < rows; ++y)
          for (int x = 0; x < cols; ++x) dst[(size_t)y * a.pitch[l] + x] = cur[(size_t)y * cols + x];
      }
      cur.assign((size_t)W * H, 0);
    }
    return true;
  });
}

}  // namespace plsvo
