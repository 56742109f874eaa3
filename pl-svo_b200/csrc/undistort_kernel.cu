// undistort_kernel.cu — vk::PinholeCamera::undistortImage (rpg_vikit pinhole_camera.cpp) for a batch of frames:
// cv::initUndistortRectifyMap(cvK_, cvD_, I, cvK_, size, CV_16SC2) once per camera, cv::remap(raw, rect, map1, map2,
// INTER_LINEAR) per frame, both as OpenCV 3.4's scalar paths compute them (imgproc undistort.cpp, imgwarp.cpp) and
// restated in oracle/plsvo_oracle.cpp.  The rectified frame is written as pyramid level 0 in the 16-byte-pitched layout
// pyramid_kernel reads.
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include "exact_math.cuh"
#include "internal.h"

namespace plsvo {
namespace {

constexpr int kMapThreads = 64;
constexpr int kRemapRows = 16;  // tile: kRemapTileW x kRemapRows output pixels, four consecutive pixels per thread
constexpr int kRemapThreads = kRemapTileW / 4 * kRemapRows;
// 58 registers (ptxas, sm_90a): four CTAs per SM.  Forcing six or eight spills the gather offsets and weights.
constexpr int kRemapCtasPerSm = 4;

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

}  // namespace

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
