// fake_undistort.cpp — model kernels of the undistortion launchers for the host-pipeline model.  TEST INFRASTRUCTURE
// ONLY (see fake_cuda.h).  tests/test_undistort.py links it with the sources of tests/hostmodel/build.py into a model
// library of its own; the stock model lacks these launchers, and plsvo_abi.cu reaches them through weak references.
//
//   map   : the CPU oracle's map (oracle/undistort_oracle.cpp, included here), written with the device map's row pitch.
//   remap : the real computation: fixed-point bilinear on the map it is given, border 0.
// Every byte the real kernels would read or write is bounds-checked against the model's device blocks.
#include <vector>

#include "../../oracle/undistort_oracle.cpp"
#include "../../pl-svo_b200/csrc/internal.h"
#include "fake_cuda.h"

namespace plsvo {

cudaError_t undistort_map_launch(const UndistortMapArgs& a0, cudaStream_t s) {
  const UndistortMapArgs a = a0;
  return fakecuda::enqueue(s, [a]() {
    const size_t span = (size_t)(a.height - 1) * a.map_pitch + a.width;
    if (!fakecuda::check(a.map1, span * sizeof(short2), "undistort map kernel: map1") ||
        !fakecuda::check(a.map2, span * sizeof(uint16_t), "undistort map kernel: map2"))
      return true;
    const plsvo_pinhole_camera cam{a.width, a.height, a.fx, a.fy, a.cx, a.cy, {a.k1, a.k2, a.p1, a.p2, a.k3}};
    if (plsvo_oracle_undistort_map(&cam, reinterpret_cast<int16_t*>(a.map1), a.map2, (size_t)a.map_pitch) != PLSVO_OK)
      fakecuda::error("undistort map kernel: camera refused");
    return true;
  });
}

cudaError_t undistort_remap_launch(const RemapArgs& a0, int, cudaStream_t s) {
  const RemapArgs a = a0;
  return fakecuda::enqueue(s, [a]() {
    const size_t mspan = (size_t)(a.height - 1) * a.map_pitch + a.width;
    const size_t sspan = (size_t)(a.height - 1) * a.src_pitch + a.width, dspan = (size_t)(a.height - 1) * a.dst_pitch + a.width;
    if (!fakecuda::check(a.map1, mspan * sizeof(short2), "remap kernel: map1") || !fakecuda::check(a.map2, mspan * 2, "remap kernel: map2"))
      return true;
    for (int b = 0; b < a.B; ++b) {
      const uint8_t* src = a.src + (size_t)b * a.src_stride;
      uint8_t* dst = a.dst + (size_t)b * a.dst_stride;
      if (!fakecuda::check(src, sspan, "remap kernel: raw frame") || !fakecuda::check(dst, dspan, "remap kernel: level 0")) return true;
      auto px = [&](int x, int y) -> uint32_t {
        return ((unsigned)x < (unsigned)a.width && (unsigned)y < (unsigned)a.height) ? src[(size_t)y * a.src_pitch + x] : 0u;
      };
      for (int y = 0; y < a.height; ++y)
        for (int x = 0; x < a.width; ++x) {
          const size_t e = (size_t)y * a.map_pitch + x;
          const int sx = a.map1[e].x, sy = a.map1[e].y, fa = a.map2[e] & 31, fb = a.map2[e] >> 5;
          const uint32_t v = px(sx, sy) * (32 - fa) * (32 - fb) + px(sx + 1, sy) * fa * (32 - fb) + px(sx, sy + 1) * (32 - fa) * fb +
                             px(sx + 1, sy + 1) * fa * fb;
          dst[(size_t)y * a.dst_pitch + x] = (uint8_t)((v * 32 + (1u << 14)) >> 15);
        }
    }
    return true;
  });
}

}  // namespace plsvo
