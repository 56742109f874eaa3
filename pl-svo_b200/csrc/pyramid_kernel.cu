// pyramid_kernel.cu — frame_utils::createImgPyramid (src/frame.cpp:171-180) = repeated vk::halfSample
// (rpg_vikit vision.cpp, scalar path: truncating mean of each 2x2 block) for a batch of frames.
// SURVEY.md §8f rank 2 ("next"): the producer of the alignment path's image input.
//
// One CTA owns a 64x64 tile of level 0: level 1 is formed in registers from two 16-byte row loads per
// thread (packed 16-bit-lane arithmetic), deeper levels from shared memory, all stores 4 or 8 bytes wide,
// so level 0 is read from HBM exactly once and each level is written once
// (traffic = 4/3 x the level-0 bytes; HBM-bound byte work, no tensor cores).  Tiles are aligned to
// 64 pixels, so the truncating 2x2 means are identical to the level-by-level computation.
#include <cuda_runtime.h>
#include <stdint.h>

#include "halfsample.cuh"
#include "internal.h"

namespace plsvo {
namespace {

constexpr int kTile = 64;
constexpr int kPyrThreads = 128;

__global__ void __launch_bounds__(kPyrThreads) pyramid_kernel(const PyramidArgs a) {
  __shared__ __align__(16) uint8_t t1[32 * 32];  // level-1 tile
  __shared__ __align__(16) uint8_t t2[16 * 16];  // level-2 tile, then reused alternately downwards
  __shared__ __align__(16) uint8_t t3[8 * 8];
  const int b = blockIdx.z;
  const int x0 = blockIdx.x * kTile, y0 = blockIdx.y * kTile;
  const uint8_t* src = a.level[0] + (size_t)b * a.stride[0];
  const int tid = threadIdx.x;
  // level 0 -> 1 straight from registers: thread = (row pair, 16-byte column segment); two 16-byte loads
  // (device rows are 16-byte pitched), eight output bytes, one 8-byte store to global and to shared memory.
  if (a.n_levels > 1) {
    const int rp = tid >> 2, cx = (tid & 3) * 16;
    const int y = y0 + 2 * rp;
    uint4 top = make_uint4(0, 0, 0, 0), bot = make_uint4(0, 0, 0, 0);
    if (x0 + cx < (int)a.pitch[0]) {
      if (y < a.height) top = __ldg(reinterpret_cast<const uint4*>(src + (size_t)y * a.pitch[0] + x0 + cx));
      if (y + 1 < a.height) bot = __ldg(reinterpret_cast<const uint4*>(src + (size_t)(y + 1) * a.pitch[0] + x0 + cx));
    }
    uint2 o;
    o.x = half2x2_word(top.x, top.y, bot.x, bot.y);
    o.y = half2x2_word(top.z, top.w, bot.z, bot.w);
    *reinterpret_cast<uint2*>(t1 + rp * 32 + (cx >> 1)) = o;
    const int W = a.width >> 1, H = a.height >> 1;
    const int ox = (x0 + cx) >> 1, oy = (y0 >> 1) + rp;
    if (oy < H && ox < W) {
      uint8_t* d = a.level[1] + (size_t)b * a.stride[1] + (size_t)oy * a.pitch[1] + ox;
      if (ox + 8 <= (int)a.pitch[1]) {
        *reinterpret_cast<uint2*>(d) = o;  // pitch is a multiple of 16 and ox of 8: aligned, inside the padded row
      } else {
        for (int k = 0; k < 8 && ox + k < W; ++k) d[k] = (uint8_t)((k < 4 ? o.x >> (8 * k) : o.y >> (8 * (k - 4))) & 0xFF);
      }
    }
  }
  __syncthreads();
  // levels 2.. from shared memory: thread = (output row, 4-byte output segment)
  const uint8_t* in = t1;
  int in_dim = 32;
  for (int l = 2; l < a.n_levels; ++l) {
    const int out_dim = in_dim >> 1;
    if (out_dim == 0) break;
    uint8_t* out = (l & 1) ? t3 : t2;
    const int W = a.width >> l, H = a.height >> l;
    const int ox0 = x0 >> l, oy0 = y0 >> l;
    uint8_t* dst = a.level[l] + (size_t)b * a.stride[l];
    if (out_dim >= 4) {
      const int segs = out_dim >> 2;
      if (tid < out_dim * segs) {
        const int oy = tid / segs, sx = (tid - oy * segs) * 4;
        const uint2 top = *reinterpret_cast<const uint2*>(in + (2 * oy) * in_dim + 2 * sx);
        const uint2 bot = *reinterpret_cast<const uint2*>(in + (2 * oy + 1) * in_dim + 2 * sx);
        const uint32_t o = half2x2_word(top.x, top.y, bot.x, bot.y);
        *reinterpret_cast<uint32_t*>(out + oy * out_dim + sx) = o;
        const int gx = ox0 + sx, gy = oy0 + oy;
        if (gy < H && gx < W) {
          uint8_t* d = dst + (size_t)gy * a.pitch[l] + gx;
          if (gx + 4 <= (int)a.pitch[l]) {
            *reinterpret_cast<uint32_t*>(d) = o;
          } else {
            for (int k = 0; k < 4 && gx + k < W; ++k) d[k] = (uint8_t)((o >> (8 * k)) & 0xFF);
          }
        }
      }
    } else {  // 2x2 and 1x1 tiles of the deepest levels: one byte per thread
      if (tid < out_dim * out_dim) {
        const int oy = tid / out_dim, ox = tid - oy * out_dim;
        const uint8_t* p = in + (2 * oy) * in_dim + 2 * ox;
        const uint8_t v = (uint8_t)(((int)p[0] + (int)p[1] + (int)p[in_dim] + (int)p[in_dim + 1]) / 4);
        out[tid] = v;
        if (ox0 + ox < W && oy0 + oy < H) dst[(size_t)(oy0 + oy) * a.pitch[l] + ox0 + ox] = v;
      }
    }
    __syncthreads();
    in = out;
    in_dim = out_dim;
  }
}

}  // namespace

cudaError_t pyramid_kernel_launch(const PyramidArgs& a, cudaStream_t s) {
  dim3 grid((a.width + kTile - 1) / kTile, (a.height + kTile - 1) / kTile, a.B);
  pyramid_kernel<<<grid, kPyrThreads, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace plsvo
