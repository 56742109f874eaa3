// halfsample.cuh — vk::halfSample's truncating 2x2 mean on packed bytes, shared by pyramid_kernel.cu and the fused
// rectify + pyramid kernel of undistort_kernel.cu.
#pragma once
#include <stdint.h>

namespace plsvo {

// Truncating mean of the 2x2 blocks of two 4-byte row fragments: bytes (a0 a1 a2 a3) over (b0 b1 b2 b3)
// -> two output bytes ((a0+a1+b0+b1)/4, (a2+a3+b2+b3)/4) in the low half-word.  16-bit lanes hold the
// pair sums (<= 1020), exactly the integer arithmetic of vk::halfSample's scalar path.
__device__ __forceinline__ uint32_t half2x2(uint32_t top, uint32_t bot) {
  const uint32_t ht = (top & 0x00FF00FFu) + ((top >> 8) & 0x00FF00FFu);  // (a0+a1) | (a2+a3)<<16
  const uint32_t hb = (bot & 0x00FF00FFu) + ((bot >> 8) & 0x00FF00FFu);
  const uint32_t q = ((ht + hb) >> 2) & 0x00FF00FFu;                     // per-lane /4, truncating
  return (q & 0xFFu) | (q >> 8);                                          // pack the two bytes
}
// eight input bytes per row (two words) -> four output bytes
__device__ __forceinline__ uint32_t half2x2_word(uint32_t t0, uint32_t t1, uint32_t b0, uint32_t b1) {
  return half2x2(t0, b0) | (half2x2(t1, b1) << 16);
}

}  // namespace plsvo
