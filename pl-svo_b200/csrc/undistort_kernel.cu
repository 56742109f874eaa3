// undistort_kernel.cu — vk::PinholeCamera::undistortImage (rpg_vikit pinhole_camera.cpp) for a batch of frames:
// cv::initUndistortRectifyMap(cvK_, cvD_, I, cvK_, size, CV_16SC2) once per camera, cv::remap(raw, rect, map1, map2,
// INTER_LINEAR) per frame, both as OpenCV 3.4's scalar paths compute them (imgproc undistort.cpp, imgwarp.cpp) and
// restated in oracle/plsvo_oracle.cpp.  The rectified frame is written as pyramid level 0 in the 16-byte-pitched layout
// pyramid_kernel reads.  undistort_pyramid_kernel fuses the remap with pyramid_kernel's half-sampling for the raw-frame
// alignment calls, which need only a few coarse levels.
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include <algorithm>

#include "exact_math.cuh"
#include "halfsample.cuh"
#include "internal.h"

namespace plsvo {
namespace {

constexpr int kMapThreads = 64;
constexpr int kRemapRows = 16;  // tile: kRemapTileW x kRemapRows output pixels, four consecutive pixels per thread
constexpr int kRemapThreads = kRemapTileW / 4 * kRemapRows;
// 58 registers (ptxas, sm_90a): four CTAs per SM.  Forcing six or eight spills the gather offsets and weights.
constexpr int kRemapCtasPerSm = 4;
constexpr int kRawTile = 64;      // undistort_pyramid_kernel: 64x64 level-0 tiles, as pyramid_kernel
constexpr int kRawThreads = 512;  // thread = 2 rows x 4 columns of the tile's level 0
constexpr int kRawCtasPerSm = 2;

// cvRound: round half to even; out of int range (or NaN) converts to INT_MIN, as x86's cvtsd2si does on the host.
__device__ __forceinline__ int cv_round(double v) {
  const double r = rint(v);
  return (r >= -2147483648.0 && r <= 2147483647.0) ? __double2int_rn(r) : INT_MIN;
}

// One thread per map row: OpenCV walks each row by accumulating _x += ir[0] (and _y, _w) pixel after pixel, so a row
// is one sequential recurrence.  Every double operation is an explicit __d*_rn (no FMA contraction), in the order of
// the scalar loop; the map is built once per camera, so this kernel is off the per-frame path.
__global__ void __launch_bounds__(kMapThreads) undistort_map_kernel(const UndistortMapArgs a) {
  const int i = blockIdx.x * kMapThreads + threadIdx.x;
  if (i >= a.height) return;
  // iR = (K R).inv(DECOMP_LU) with R = I: OpenCV's closed-form 3x3 inverse (cofactors times 1/det3)
  const double m[3][3] = {{a.fx, 0.0, a.cx}, {0.0, a.fy, a.cy}, {0.0, 0.0, 1.0}};
  const double det = DA(DS(DM(m[0][0], DS(DM(m[1][1], m[2][2]), DM(m[1][2], m[2][1]))),
                           DM(m[0][1], DS(DM(m[1][0], m[2][2]), DM(m[1][2], m[2][0])))),
                        DM(m[0][2], DS(DM(m[1][0], m[2][1]), DM(m[1][1], m[2][0]))));
  const double d = DD(1.0, det);
  const double ir0 = DM(DS(DM(m[1][1], m[2][2]), DM(m[1][2], m[2][1])), d);
  const double ir1 = DM(DS(DM(m[0][2], m[2][1]), DM(m[0][1], m[2][2])), d);
  const double ir2 = DM(DS(DM(m[0][1], m[1][2]), DM(m[0][2], m[1][1])), d);
  const double ir3 = DM(DS(DM(m[1][2], m[2][0]), DM(m[1][0], m[2][2])), d);
  const double ir4 = DM(DS(DM(m[0][0], m[2][2]), DM(m[0][2], m[2][0])), d);
  const double ir5 = DM(DS(DM(m[0][2], m[1][0]), DM(m[0][0], m[1][2])), d);
  const double ir6 = DM(DS(DM(m[1][0], m[2][1]), DM(m[1][1], m[2][0])), d);
  const double ir7 = DM(DS(DM(m[0][1], m[2][0]), DM(m[0][0], m[2][1])), d);
  const double ir8 = DM(DS(DM(m[0][0], m[1][1]), DM(m[0][1], m[1][0])), d);
  const double di = (double)i;
  double _x = DA(DM(di, ir1), ir2), _y = DA(DM(di, ir4), ir5), _w = DA(DM(di, ir7), ir8);
  short2* m1 = a.map1 + (size_t)i * a.map_pitch;
  uint16_t* m2 = a.map2 + (size_t)i * a.map_pitch;
  for (int j = 0; j < a.width; ++j, _x = DA(_x, ir0), _y = DA(_y, ir3), _w = DA(_w, ir6)) {
    const double w = DD(1.0, _w), x = DM(_x, w), y = DM(_y, w);
    const double x2 = DM(x, x), y2 = DM(y, y);
    const double r2 = DA(x2, y2), _2xy = DM(DM(2.0, x), y);
    const double kr = DA(1.0, DM(DA(DM(DA(DM(a.k3, r2), a.k2), r2), a.k1), r2));
    const double u = DA(DM(a.fx, DA(DA(DM(x, kr), DM(a.p1, _2xy)), DM(a.p2, DA(r2, DM(2.0, x2))))), a.cx);
    const double v = DA(DM(a.fy, DA(DA(DM(y, kr), DM(a.p1, DA(r2, DM(2.0, y2)))), DM(a.p2, _2xy))), a.cy);
    const int iu = cv_round(DM(u, 32.0)), iv = cv_round(DM(v, 32.0));
    m1[j] = make_short2((short)(iu >> 5), (short)(iv >> 5));
    m2[j] = (uint16_t)((iv & 31) * 32 + (iu & 31));
  }
}

// One CTA owns a kRemapTileW x kRemapRows output tile and a run of frames.  The tile's map entries are read once and
// turned into per-pixel gather offsets, inside-the-frame masks and fixed-point weights, which stay in registers while
// the CTA loops over its frames: per frame a thread does 16 read-only byte gathers and one 4-byte store.
// OpenCV's remapBilinear for 8-bit images: out = (sum p*w + 2^14) >> 15 with the 32x32 table's weights, exact
// integers (32-a)(32-b)*32, a(32-b)*32, (32-a)b*32, ab*32 (a = map2 & 31, b = map2 >> 5); the one entry OpenCV
// saturates (32768 -> 32767 at a = b = 0) gives the same byte.  A neighbour outside the frame contributes 0
// (BORDER_CONSTANT, value 0).
__global__ void __launch_bounds__(kRemapThreads, kRemapCtasPerSm) undistort_remap_kernel(const RemapArgs a, int frames_per_cta) {
  const int tx = threadIdx.x % (kRemapTileW / 4), ty = threadIdx.x / (kRemapTileW / 4);
  const int x = blockIdx.x * kRemapTileW + 4 * tx, y = blockIdx.y * kRemapRows + ty;
  if (y >= a.height || x >= a.width) return;
  const size_t e = (size_t)y * a.map_pitch + x;  // x and map_pitch are multiples of 4: aligned vector loads
  const uint4 m1 = __ldg(reinterpret_cast<const uint4*>(a.map1 + e));
  const uint2 m2 = __ldg(reinterpret_cast<const uint2*>(a.map2 + e));
  const uint32_t m1w[4] = {m1.x, m1.y, m1.z, m1.w};
  const uint32_t m2w[4] = {m2.x & 0xFFFFu, m2.x >> 16, m2.y & 0xFFFFu, m2.y >> 16};
  int off[4];           // sy * src_pitch + sx
  uint32_t wlo[4], whi[4];  // weights of the top (lo) and bottom (hi) neighbour pairs, 16 bits each, 0 where outside
  const int W = a.width, H = a.height, P = (int)a.src_pitch;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int sx = (int)(short)(m1w[k] & 0xFFFFu), sy = (int)(short)(m1w[k] >> 16);
    const int fa = (int)(m2w[k] & 31u), fb = (int)(m2w[k] >> 5);
    const bool x0 = (unsigned)sx < (unsigned)W, x1 = (unsigned)(sx + 1) < (unsigned)W;
    const bool y0 = (unsigned)sy < (unsigned)H, y1 = (unsigned)(sy + 1) < (unsigned)H;
    // weights in units of 32 (the table's scale is 2^15 = 32 * 32 * 32): each fits 16 bits
    const uint32_t w00 = (x0 && y0) ? (32 - fa) * (32 - fb) : 0, w01 = (x1 && y0) ? fa * (32 - fb) : 0;
    const uint32_t w10 = (x0 && y1) ? (32 - fa) * fb : 0, w11 = (x1 && y1) ? fa * fb : 0;
    off[k] = sy * P + sx;
    wlo[k] = w00 | (w01 << 16);
    whi[k] = w10 | (w11 << 16);
  }
  const int b0 = blockIdx.z * frames_per_cta, b1 = min(a.B, b0 + frames_per_cta);
  const uint8_t* src = a.src + (size_t)b0 * a.src_stride;
  uint8_t* dst = a.dst + (size_t)b0 * a.dst_stride + (size_t)y * a.dst_pitch + x;
  for (int b = b0; b < b1; ++b, src += a.src_stride, dst += a.dst_stride) {
    uint32_t word = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint8_t* p = src + off[k];
      const uint32_t p00 = (wlo[k] & 0xFFFFu) ? __ldg(p) : 0u, p01 = (wlo[k] >> 16) ? __ldg(p + 1) : 0u;
      const uint32_t p10 = (whi[k] & 0xFFFFu) ? __ldg(p + P) : 0u, p11 = (whi[k] >> 16) ? __ldg(p + P + 1) : 0u;
      const uint32_t s = (p00 * (wlo[k] & 0xFFFFu) + p01 * (wlo[k] >> 16) + p10 * (whi[k] & 0xFFFFu) + p11 * (whi[k] >> 16)) * 32u;
      word |= ((s + (1u << 14)) >> 15) << (8 * k);
    }
    // dst_pitch is a multiple of 16 and x of 4: the word lies inside the padded row even past the last column
    *reinterpret_cast<uint32_t*>(dst) = word;
  }
}

// One output pixel of remapBilinear (the arithmetic of undistort_remap_kernel above) from its map entry: m1 = (x, y)
// source pixel as two shorts, m2 = (iv & 31) * 32 + (iu & 31).
__device__ __forceinline__ uint32_t remap_pixel(const uint8_t* src, uint32_t m1, uint32_t m2, int W, int H, size_t P) {
  const int sx = (int)(short)(m1 & 0xFFFFu), sy = (int)(short)(m1 >> 16);
  const uint32_t fa = m2 & 31u, fb = (m2 >> 5) & 31u;
  const bool x0 = (unsigned)sx < (unsigned)W, x1 = (unsigned)(sx + 1) < (unsigned)W;
  const bool y0 = (unsigned)sy < (unsigned)H, y1 = (unsigned)(sy + 1) < (unsigned)H;
  const uint32_t w00 = (x0 && y0) ? (32 - fa) * (32 - fb) : 0, w01 = (x1 && y0) ? fa * (32 - fb) : 0;
  const uint32_t w10 = (x0 && y1) ? (32 - fa) * fb : 0, w11 = (x1 && y1) ? fa * fb : 0;
  const uint8_t* p = src + ((long long)sy * (long long)P + sx);  // dereferenced only where a weight is non-zero
  const uint32_t p00 = w00 ? __ldg(p) : 0u, p01 = w01 ? __ldg(p + 1) : 0u;
  const uint32_t p10 = w10 ? __ldg(p + P) : 0u, p11 = w11 ? __ldg(p + P + 1) : 0u;
  return ((p00 * w00 + p01 * w01 + p10 * w10 + p11 * w11) * 32u + (1u << 14)) >> 15;
}

// Rectification and pyramid in one pass.  One CTA owns a 64x64 tile of rectified level 0 (as pyramid_kernel) and a run of
// frames.  A thread forms 2 rows x 4 columns of level 0 with remap_pixel, level 1 from those eight bytes in registers,
// and levels 2.. from shared memory as pyramid_kernel does.  The map entries are re-read for every frame (the map of a
// camera stays in L2); holding them across frames as the remap kernel does would cost 12 more registers and spill at two
// 512-thread CTAs per SM.  Level 0 is
// never read back from memory, and a level is stored only when level[l] is set: alignment at levels 4..2 writes about a
// 21st of the level-0 bytes.  Tiles are aligned to 64 pixels, so every level equals the level-by-level computation.
__global__ void __launch_bounds__(kRawThreads, kRawCtasPerSm) undistort_pyramid_kernel(const RawPyramidArgs a, int frames_per_cta) {
  __shared__ __align__(16) uint8_t t1[32 * 32];  // level-1 tile
  __shared__ __align__(16) uint8_t t2[16 * 16];  // level-2 tile, then reused alternately downwards
  __shared__ __align__(16) uint8_t t3[8 * 8];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int x0 = blockIdx.x * kRawTile, y0 = blockIdx.y * kRawTile;
  const int x = x0 + 4 * tx, y = y0 + 2 * ty;
  const int W = a.width, H = a.height;
  const int b0 = blockIdx.z * frames_per_cta, b1 = min(a.B, b0 + frames_per_cta);
  for (int b = b0; b < b1; ++b) {
    const uint8_t* src = a.src + (size_t)b * a.src_stride;
    uint32_t word[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      uint32_t w = 0;
      if (y + r < H) {
        if (a.map1) {  // x and map_pitch are multiples of 4: aligned vector loads, inside the padded map row
          const size_t e = (size_t)(y + r) * a.map_pitch + x;
          const uint4 m1 = __ldg(reinterpret_cast<const uint4*>(a.map1 + e));
          const uint2 m2 = __ldg(reinterpret_cast<const uint2*>(a.map2 + e));
          w = remap_pixel(src, m1.x, m2.x, W, H, a.src_pitch) | remap_pixel(src, m1.y, m2.x >> 16, W, H, a.src_pitch) << 8 |
              remap_pixel(src, m1.z, m2.y, W, H, a.src_pitch) << 16 | remap_pixel(src, m1.w, m2.y >> 16, W, H, a.src_pitch) << 24;
        } else {  // no distortion: level 0 is the raw frame
          const uint8_t* row = src + (size_t)(y + r) * a.src_pitch;
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (x + k < W) w |= (uint32_t)__ldg(row + x + k) << (8 * k);
        }
        // pitch is a multiple of 16 and x of 4: the word lies inside the padded row
        if (a.level[0] && x < (int)a.pitch[0])
          *reinterpret_cast<uint32_t*>(a.level[0] + (size_t)b * a.stride[0] + (size_t)(y + r) * a.pitch[0] + x) = w;
      }
      word[r] = w;
    }
    if (a.n_levels < 2) continue;
    // level 1 from registers: two output bytes per thread
    const uint32_t o1 = half2x2(word[0], word[1]) & 0xFFFFu;
    *reinterpret_cast<uint16_t*>(t1 + ty * 32 + 2 * tx) = (uint16_t)o1;
    if (a.level[1]) {
      const int ox = x >> 1, oy = y >> 1;  // ox is even and the pitch a multiple of 16: both bytes inside the padded row
      if (oy < (H >> 1) && ox < (W >> 1))
        *reinterpret_cast<uint16_t*>(a.level[1] + (size_t)b * a.stride[1] + (size_t)oy * a.pitch[1] + ox) = (uint16_t)o1;
    }
    __syncthreads();
    // levels 2.. from shared memory: thread = (output row, 4-byte output segment), as in pyramid_kernel
    const uint8_t* in = t1;
    int in_dim = 32;
    for (int l = 2; l < a.n_levels; ++l) {
      const int out_dim = in_dim >> 1;
      uint8_t* out = (l & 1) ? t3 : t2;
      const int Wl = W >> l, Hl = H >> l;
      const int ox0 = x0 >> l, oy0 = y0 >> l;
      uint8_t* dst = a.level[l] ? a.level[l] + (size_t)b * a.stride[l] : nullptr;
      if (out_dim >= 4) {
        const int segs = out_dim >> 2;
        if (tid < out_dim * segs) {
          const int oy = tid / segs, sx = (tid - oy * segs) * 4;
          const uint2 top = *reinterpret_cast<const uint2*>(in + (2 * oy) * in_dim + 2 * sx);
          const uint2 bot = *reinterpret_cast<const uint2*>(in + (2 * oy + 1) * in_dim + 2 * sx);
          const uint32_t o = half2x2_word(top.x, top.y, bot.x, bot.y);
          *reinterpret_cast<uint32_t*>(out + oy * out_dim + sx) = o;
          const int gx = ox0 + sx, gy = oy0 + oy;
          if (dst && gy < Hl && gx < Wl) {
            uint8_t* d = dst + (size_t)gy * a.pitch[l] + gx;
            if (gx + 4 <= (int)a.pitch[l]) {
              *reinterpret_cast<uint32_t*>(d) = o;
            } else {
              for (int k = 0; k < 4 && gx + k < Wl; ++k) d[k] = (uint8_t)((o >> (8 * k)) & 0xFF);
            }
          }
        }
      } else {  // 2x2 and 1x1 tiles of the deepest levels: one byte per thread
        if (tid < out_dim * out_dim) {
          const int oy = tid / out_dim, ox = tid - oy * out_dim;
          const uint8_t* p = in + (2 * oy) * in_dim + 2 * ox;
          const uint8_t v = (uint8_t)(((int)p[0] + (int)p[1] + (int)p[in_dim] + (int)p[in_dim + 1]) / 4);
          out[tid] = v;
          if (dst && ox0 + ox < Wl && oy0 + oy < Hl) dst[(size_t)(oy0 + oy) * a.pitch[l] + ox0 + ox] = v;
        }
      }
      __syncthreads();
      in = out;
      in_dim = out_dim;
    }
  }
}

// undistort_pyramid_kernel for the frames of several cameras (plsvo_*_raw_multicam_batch_run): the i-th frame of a run
// is visit[i].frame, rectified with visit[i]'s map, or copied when that is NULL.  The host lists the frames grouped by
// camera, so that the CTAs resident at one time (dispatched roughly in run order) read the map tiles of only a few
// cameras and those stay in L2.  The body is undistort_pyramid_kernel's with that choice at the top of the frame loop; it
// is spelled out again because extracting the shared body into an inlined device function changes the plain kernel's
// SASS (ptxas reorders its byte-store tail).
__global__ void __launch_bounds__(kRawThreads, kRawCtasPerSm) undistort_pyramid_multicam_kernel(const RawPyramidArgs a, int frames_per_cta,
                                                                                               const RawVisit* __restrict__ visit) {
  __shared__ __align__(16) uint8_t t1[32 * 32];  // level-1 tile
  __shared__ __align__(16) uint8_t t2[16 * 16];  // level-2 tile, then reused alternately downwards
  __shared__ __align__(16) uint8_t t3[8 * 8];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int x0 = blockIdx.x * kRawTile, y0 = blockIdx.y * kRawTile;
  const int x = x0 + 4 * tx, y = y0 + 2 * ty;
  const int i0 = blockIdx.z * frames_per_cta, i1 = min(a.B, i0 + frames_per_cta);
  for (int i = i0; i < i1; ++i) {
    // the frame, its camera's map and size: one record, the same for every thread of the CTA.  The grid covers the slot
    // (a.width x a.height); the frame is W x H in its top-left corner.
    const int b = __ldg(&visit[i].frame);
    const int W = __ldg(&visit[i].width), H = __ldg(&visit[i].height);
    if (x0 >= W || y0 >= H) continue;  // the tile lies wholly in the slot's padding: nothing of this frame to form
    const short2* map1 = visit[i].map1;
    const uint16_t* map2 = visit[i].map2;
    const uint8_t* src = a.src + (size_t)b * a.src_stride;
    uint32_t word[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      uint32_t w = 0;
      if (y + r < H) {
        if (map1) {  // x0 < W: the tile's 64 entries lie inside the camera's padded map row (map_pitch, a multiple of 64)
          const size_t e = (size_t)(y + r) * __ldg(&visit[i].map_pitch) + x;
          const uint4 m1 = __ldg(reinterpret_cast<const uint4*>(map1 + e));
          const uint2 m2 = __ldg(reinterpret_cast<const uint2*>(map2 + e));
          w = remap_pixel(src, m1.x, m2.x, W, H, a.src_pitch) | remap_pixel(src, m1.y, m2.x >> 16, W, H, a.src_pitch) << 8 |
              remap_pixel(src, m1.z, m2.y, W, H, a.src_pitch) << 16 | remap_pixel(src, m1.w, m2.y >> 16, W, H, a.src_pitch) << 24;
        } else {
          const uint8_t* row = src + (size_t)(y + r) * a.src_pitch;
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (x + k < W) w |= (uint32_t)__ldg(row + x + k) << (8 * k);
        }
        // the bytes right of the frame are 0 (the slot's padding stays as the host cleared it); pitch is a multiple of
        // 16 and x of 4: the word lies inside the padded row
        if (x + 4 > W) w = x < W ? w & (0xFFFFFFFFu >> (8 * (x + 4 - W))) : 0u;
        if (a.level[0] && x < (int)a.pitch[0])
          *reinterpret_cast<uint32_t*>(a.level[0] + (size_t)b * a.stride[0] + (size_t)(y + r) * a.pitch[0] + x) = w;
      }
      word[r] = w;
    }
    if (a.n_levels < 2) continue;
    // level 1 from registers: two output bytes per thread
    const uint32_t o1 = half2x2(word[0], word[1]) & 0xFFFFu;
    *reinterpret_cast<uint16_t*>(t1 + ty * 32 + 2 * tx) = (uint16_t)o1;
    if (a.level[1]) {
      const int ox = x >> 1, oy = y >> 1;  // ox is even: both bytes, or the last byte of the frame's row
      uint8_t* d = a.level[1] + (size_t)b * a.stride[1] + (size_t)oy * a.pitch[1] + ox;
      if (oy < (H >> 1) && ox + 1 < (W >> 1)) *reinterpret_cast<uint16_t*>(d) = (uint16_t)o1;
      else if (oy < (H >> 1) && ox < (W >> 1)) *d = (uint8_t)o1;
    }
    __syncthreads();
    // levels 2.. from shared memory: thread = (output row, 4-byte output segment), as in pyramid_kernel
    const uint8_t* in = t1;
    int in_dim = 32;
    for (int l = 2; l < a.n_levels; ++l) {
      const int out_dim = in_dim >> 1;
      uint8_t* out = (l & 1) ? t3 : t2;
      const int Wl = W >> l, Hl = H >> l;
      const int ox0 = x0 >> l, oy0 = y0 >> l;
      uint8_t* dst = a.level[l] ? a.level[l] + (size_t)b * a.stride[l] : nullptr;
      if (out_dim >= 4) {
        const int segs = out_dim >> 2;
        if (tid < out_dim * segs) {
          const int oy = tid / segs, sx = (tid - oy * segs) * 4;
          const uint2 top = *reinterpret_cast<const uint2*>(in + (2 * oy) * in_dim + 2 * sx);
          const uint2 bot = *reinterpret_cast<const uint2*>(in + (2 * oy + 1) * in_dim + 2 * sx);
          const uint32_t o = half2x2_word(top.x, top.y, bot.x, bot.y);
          *reinterpret_cast<uint32_t*>(out + oy * out_dim + sx) = o;
          const int gx = ox0 + sx, gy = oy0 + oy;
          if (dst && gy < Hl && gx < Wl) {
            uint8_t* d = dst + (size_t)gy * a.pitch[l] + gx;
            if (gx + 4 <= Wl) {
              *reinterpret_cast<uint32_t*>(d) = o;
            } else {
              for (int k = 0; k < 4 && gx + k < Wl; ++k) d[k] = (uint8_t)((o >> (8 * k)) & 0xFF);
            }
          }
        }
      } else {  // 2x2 and 1x1 tiles of the deepest levels: one byte per thread
        if (tid < out_dim * out_dim) {
          const int oy = tid / out_dim, ox = tid - oy * out_dim;
          const uint8_t* p = in + (2 * oy) * in_dim + 2 * ox;
          const uint8_t v = (uint8_t)(((int)p[0] + (int)p[1] + (int)p[in_dim] + (int)p[in_dim + 1]) / 4);
          out[tid] = v;
          if (dst && ox0 + ox < Wl && oy0 + oy < Hl) dst[(size_t)(oy0 + oy) * a.pitch[l] + ox0 + ox] = v;
        }
      }
      __syncthreads();
      in = out;
      in_dim = out_dim;
    }
  }
}


}  // namespace

namespace {
// Frame runs: each CTA loops over a run of frames of one tile.  Enough runs for about eight waves of resident CTAs keep
// the last wave short.
dim3 raw_pyramid_grid(const RawPyramidArgs& a, int num_sms, int* per_cta) {
  const int gx = (a.width + kRawTile - 1) / kRawTile, gy = (a.height + kRawTile - 1) / kRawTile;
  const long long want = (long long)(num_sms > 0 ? num_sms : 1) * kRawCtasPerSm * 8;
  long long runs = (want + gx * gy - 1) / (gx * gy);
  runs = runs < 1 ? 1 : (runs > a.B ? a.B : runs);
  int per = (int)((a.B + runs - 1) / runs);
  per = std::max(per, (a.B + 65534) / 65535);  // gridDim.z <= 65535
  runs = (a.B + per - 1) / per;
  *per_cta = per;
  return dim3(gx, gy, (unsigned)runs);
}
}  // namespace

cudaError_t undistort_pyramid_launch(const RawPyramidArgs& a, int num_sms, cudaStream_t s) {
  int per = 0;
  const dim3 grid = raw_pyramid_grid(a, num_sms, &per);
  undistort_pyramid_kernel<<<grid, kRawThreads, 0, s>>>(a, per);
  return cudaGetLastError();
}

cudaError_t undistort_pyramid_multicam_launch(const RawPyramidArgs& a, const RawVisit* visit, int num_sms, cudaStream_t s) {
  int per = 0;
  const dim3 grid = raw_pyramid_grid(a, num_sms, &per);
  undistort_pyramid_multicam_kernel<<<grid, kRawThreads, 0, s>>>(a, per, visit);
  return cudaGetLastError();
}

cudaError_t undistort_map_launch(const UndistortMapArgs& a, cudaStream_t s) {
  undistort_map_kernel<<<(a.height + kMapThreads - 1) / kMapThreads, kMapThreads, 0, s>>>(a);
  return cudaGetLastError();
}

cudaError_t undistort_remap_launch(const RemapArgs& a, int num_sms, cudaStream_t s) {
  const int gx = (a.width + kRemapTileW - 1) / kRemapTileW, gy = (a.height + kRemapRows - 1) / kRemapRows;
  // Enough frame runs to fill every SM once with resident CTAs; each CTA then loops over its run, so the map's per-tile
  // work is paid once per run instead of once per frame.
  const int want = (num_sms > 0 ? num_sms : 1) * kRemapCtasPerSm;
  int runs = (want + gx * gy - 1) / (gx * gy);
  runs = runs < 1 ? 1 : (runs > a.B ? a.B : runs);
  const int per = (a.B + runs - 1) / runs;
  runs = (a.B + per - 1) / per;
  undistort_remap_kernel<<<dim3(gx, gy, runs), kRemapThreads, 0, s>>>(a, per);
  return cudaGetLastError();
}

}  // namespace plsvo
