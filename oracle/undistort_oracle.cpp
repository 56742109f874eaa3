// undistort_oracle.cpp — CPU restatement of vk::PinholeCamera::undistortImage (rpg_vikit pinhole_camera.cpp).
// TEST INFRASTRUCTURE ONLY, like plsvo_oracle.cpp; built by oracle/undistort_oracle.py with the same flags
// (-ffp-contract=off: strict IEEE double arithmetic, no FMA contraction).
//
// The constructor sets distortion_ = fabs(d0) > 1e-7, builds cvK_ / cvD_ as Mat_<float> and calls
// cv::initUndistortRectifyMap(cvK_, cvD_, I, cvK_, size, CV_16SC2, map1, map2) once; undistortImage is
// cv::remap(raw, rect, map1, map2, INTER_LINEAR) (default BORDER_CONSTANT, 0), or raw.clone() without distortion_.
// Both OpenCV functions are restated from OpenCV 3.4's scalar paths (imgproc undistort.cpp, imgwarp.cpp).  The pyramid
// of the rectified frame is plsvo_oracle.cpp's createImgPyramid.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <thread>
#include <vector>

#include "../include/plsvo_b200.h"

namespace {

// cvRound: round half to even; a value outside int (or NaN) converts to INT_MIN as x86's cvtsd2si does.
inline int cv_round(double v) {
  const double r = std::rint(v);
  return (r >= -2147483648.0 && r <= 2147483647.0) ? (int)r : std::numeric_limits<int>::min();
}

// cv::remap, 8-bit, INTER_LINEAR, BORDER_CONSTANT 0 (remapBilinear with FixedPtCast<int, uchar, 15>): the weights of the
// 32x32 table are (32-a)(32-b)*32, a(32-b)*32, (32-a)b*32, ab*32 with a = map2 & 31, b = map2 >> 5 (the one saturated
// entry, 32768 -> 32767 at a = b = 0, rounds to the same byte); a neighbour outside the image contributes 0.
void remap_linear_u8(const uint8_t* src, size_t sp, int W, int H, const int16_t* map1, const uint16_t* map2, size_t map_pitch,
                     uint8_t* dst, size_t dp) {
  auto px = [&](int x, int y) -> int { return ((unsigned)x < (unsigned)W && (unsigned)y < (unsigned)H) ? src[(size_t)y * sp + x] : 0; };
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const size_t e = (size_t)y * map_pitch + x;
      const int sx = map1[2 * e], sy = map1[2 * e + 1], a = map2[e] & 31, b = map2[e] >> 5;
      const int s = px(sx, sy) * ((32 - a) * (32 - b) * 32) + px(sx + 1, sy) * (a * (32 - b) * 32) + px(sx, sy + 1) * ((32 - a) * b * 32) +
                    px(sx + 1, sy + 1) * (a * b * 32);
      dst[(size_t)y * dp + x] = (uint8_t)((s + (1 << 14)) >> 15);
    }
}

}  // namespace

extern "C" {

// cv::initUndistortRectifyMap, CV_16SC2 + CV_16UC1 maps (map1 [H][map_pitch][2], map2 [H][map_pitch]; map_pitch >= width).
// iR = (K*R).inv(DECOMP_LU), which for 3x3 is the closed form: cofactors times 1/det3.  Each row starts at
// _x = i*ir[1] + ir[2] (_y, _w alike) and adds ir[0] (ir[3], ir[6]) pixel by pixel; w = 1/_w, x = _x*w, y = _y*w;
// kr = 1 + ((k3 r2 + k2) r2 + k1) r2 (the rational and thin-prism terms are zero);
// u = fx*(x kr + p1 2xy + p2 (r2 + 2x^2)) + cx; iu = cvRound(u*32);
// map1 = ((short)(iu >> 5), (short)(iv >> 5)), map2 = (iv & 31)*32 + (iu & 31).
int plsvo_oracle_undistort_map(const plsvo_pinhole_camera* cam, int16_t* map1, uint16_t* map2, size_t map_pitch) {
  if (!cam || !map1 || !map2 || cam->width <= 0 || cam->height <= 0 || map_pitch < (size_t)cam->width) return PLSVO_ERR_INVALID;
  const double fx = (float)cam->fx, fy = (float)cam->fy, cx = (float)cam->cx, cy = (float)cam->cy;
  const double k1 = (float)cam->d[0], k2 = (float)cam->d[1], p1 = (float)cam->d[2], p2 = (float)cam->d[3], k3 = (float)cam->d[4];
  const double m[3][3] = {{fx, 0.0, cx}, {0.0, fy, cy}, {0.0, 0.0, 1.0}};
  double d = m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
             m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
  d = 1. / d;
  const double ir[9] = {(m[1][1] * m[2][2] - m[1][2] * m[2][1]) * d, (m[0][2] * m[2][1] - m[0][1] * m[2][2]) * d,
                        (m[0][1] * m[1][2] - m[0][2] * m[1][1]) * d, (m[1][2] * m[2][0] - m[1][0] * m[2][2]) * d,
                        (m[0][0] * m[2][2] - m[0][2] * m[2][0]) * d, (m[0][2] * m[1][0] - m[0][0] * m[1][2]) * d,
                        (m[1][0] * m[2][1] - m[1][1] * m[2][0]) * d, (m[0][1] * m[2][0] - m[0][0] * m[2][1]) * d,
                        (m[0][0] * m[1][1] - m[0][1] * m[1][0]) * d};
  for (int i = 0; i < cam->height; ++i) {
    int16_t* m1 = map1 + (size_t)i * map_pitch * 2;
    uint16_t* m2 = map2 + (size_t)i * map_pitch;
    double _x = i * ir[1] + ir[2], _y = i * ir[4] + ir[5], _w = i * ir[7] + ir[8];
    for (int j = 0; j < cam->width; ++j, _x += ir[0], _y += ir[3], _w += ir[6]) {
      const double w = 1. / _w, x = _x * w, y = _y * w;
      const double x2 = x * x, y2 = y * y;
      const double r2 = x2 + y2, _2xy = 2 * x * y;
      const double kr = 1 + ((k3 * r2 + k2) * r2 + k1) * r2;
      const double u = fx * (x * kr + p1 * _2xy + p2 * (r2 + 2 * x2)) + cx;
      const double v = fy * (y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy) + cy;
      const int iu = cv_round(u * 32), iv = cv_round(v * 32);
      m1[j * 2] = (int16_t)(iu >> 5);
      m1[j * 2 + 1] = (int16_t)(iv >> 5);
      m2[j] = (uint16_t)((iv & 31) * 32 + (iu & 31));
    }
  }
  return PLSVO_OK;
}

// undistortImage on each of the B frames of `in` into level 0 of `out`, with a map from plsvo_oracle_undistort_map
// (pitch = width; ignored when fabs(d0) <= 1e-7).  Frames are spread over n_threads threads.
int plsvo_oracle_undistort_frames(const plsvo_undistort_batch* in, const int16_t* map1, const uint16_t* map2,
                                  const plsvo_pyramid_result* out, int n_threads) {
  if (!in || !out || !in->img0 || !out->level[0] || in->batch < 0) return PLSVO_ERR_INVALID;
  const int W = in->cam.width, H = in->cam.height;
  const bool distortion = std::fabs(in->cam.d[0]) > 0.0000001;
  if (distortion && (!map1 || !map2)) return PLSVO_ERR_INVALID;
  std::atomic<int> next{0};
  auto work = [&] {
    for (int b; (b = next.fetch_add(1)) < in->batch;) {
      const uint8_t* raw = in->img0 + (size_t)b * in->stride0;
      uint8_t* rect = out->level[0] + (size_t)b * out->stride[0];
      if (distortion)
        remap_linear_u8(raw, in->pitch0, W, H, map1, map2, (size_t)W, rect, out->pitch[0]);
      else
        for (int y = 0; y < H; ++y) memcpy(rect + (size_t)y * out->pitch[0], raw + (size_t)y * in->pitch0, (size_t)W);
    }
  };
  std::vector<std::thread> pool;
  for (int t = 1; t < std::min(std::max(n_threads, 1), std::max(in->batch, 1)); ++t) pool.emplace_back(work);
  work();
  for (auto& th : pool) th.join();
  return PLSVO_OK;
}

}  // extern "C"
