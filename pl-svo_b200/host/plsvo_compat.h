// plsvo_compat.h — minimal stand-ins for the reference's data model, ONLY for building and testing
// the shim in an image without Eigen / Sophus / OpenCV / boost / vikit.  Member names and the few
// methods the shim touches match the reference headers:
//   Frame        include/plsvo/frame.h:52-71      (T_f_w_, Cov_, img_pyr_, pt_fts_, seg_fts_, cam_)
//   PointFeat    include/plsvo/feature.h:56-73    (px, f, level, feat3D)
//   LineFeat     include/plsvo/feature.h:76-104   (spx, epx, sf, ef, line, length, level, feat3D)
//   Point        include/plsvo/feature3D.h:103    (pos_)
//   LineSeg      include/plsvo/feature3D.h:149-150 (spos_, epos_)
//   FramePtr     include/plsvo/global.h:120       (boost::shared_ptr<Frame>; std::shared_ptr here)
// With the real headers available, compile the shim with -DPLSVO_SHIM_WITH_REFERENCE_HEADERS and this
// file is not used.
#pragma once
#include <cstddef>
#include <cstdint>
#include <list>
#include <memory>
#include <vector>

namespace Eigen {
template <int N>
struct VectorNd {
  double v[N];
  double& operator[](int i) { return v[i]; }
  const double& operator[](int i) const { return v[i]; }
};
typedef VectorNd<2> Vector2d;
typedef VectorNd<3> Vector3d;
struct Quaterniond {
  double x_, y_, z_, w_;
  Quaterniond() : x_(0), y_(0), z_(0), w_(1) {}
  Quaterniond(double w, double x, double y, double z) : x_(x), y_(y), z_(z), w_(w) {}
  double x() const { return x_; }
  double y() const { return y_; }
  double z() const { return z_; }
  double w() const { return w_; }
};
struct Matrix6d {
  double m[36];
  double& operator()(int r, int c) { return m[r * 6 + c]; }
  double operator()(int r, int c) const { return m[r * 6 + c]; }
};
}  // namespace Eigen

namespace Sophus {
struct SE3 {  // old non-templated Sophus API: unit_quaternion(), translation(), SE3(Quaterniond, Vector3d)
  Eigen::Quaterniond q_;
  Eigen::Vector3d t_;
  SE3() { t_[0] = t_[1] = t_[2] = 0; }
  SE3(const Eigen::Quaterniond& q, const Eigen::Vector3d& t) : q_(q), t_(t) {}
  const Eigen::Quaterniond& unit_quaternion() const { return q_; }
  const Eigen::Vector3d& translation() const { return t_; }
};
}  // namespace Sophus

namespace cv {
struct Mat {  // the shim reads data / step[0] / cols / rows of CV_8UC1 pyramid levels
  uint8_t* data = nullptr;
  size_t step[2] = {0, 1};
  int cols = 0, rows = 0;
};
}  // namespace cv

namespace vk {
class AbstractCamera {
 public:
  virtual ~AbstractCamera() {}
  virtual double errorMultiplier2() const = 0;
  int width() const { return width_; }
  int height() const { return height_; }
  int width_ = 0, height_ = 0;
};
class PinholeCamera : public AbstractCamera {  // undistorted model, as given to FrameHandlerMono
 public:
  PinholeCamera(int w, int h, double fx, double fy, double cx, double cy) : fx_(fx), fy_(fy), cx_(cx), cy_(cy) {
    width_ = w, height_ = h;
  }
  double errorMultiplier2() const override { return fx_ < 0 ? -fx_ : fx_; }
  double fx() const { return fx_; }
  double fy() const { return fy_; }
  double cx() const { return cx_; }
  double cy() const { return cy_; }

 private:
  double fx_, fy_, cx_, cy_;
};
// vk::ATANCamera (rpg_vikit atan_camera.h), the FOV model of cam_model ATAN: constructor with intrinsics normalised by
// the image size; the shim reads width/height and the members fx_, fy_, cx_, cy_, s_.
class ATANCamera : public AbstractCamera {
 public:
  ATANCamera(double w, double h, double fx, double fy, double cx, double cy, double d0)
      : fx_(w * fx), fy_(h * fy), cx_(cx * w - 0.5), cy_(cy * h - 0.5), s_(d0) {
    width_ = (int)w, height_ = (int)h;
  }
  double errorMultiplier2() const override { return fx_; }
  double fx_, fy_, cx_, cy_, s_;
};
}  // namespace vk

namespace plsvo {
using Eigen::Vector2d;
using Eigen::Vector3d;
using Sophus::SE3;
struct Point {
  Vector3d pos_;
};
struct LineSeg {
  Vector3d spos_, epos_;
};
struct PointFeat {
  Vector2d px;
  Vector3d f;
  int level = 0;
  Point* feat3D = nullptr;
};
struct LineFeat {
  Vector2d spx, epx;
  Vector3d sf, ef, line;
  double length = 0;
  int level = 0;
  LineSeg* feat3D = nullptr;
};
typedef std::vector<cv::Mat> ImgPyr;
class Frame {
 public:
  vk::AbstractCamera* cam_ = nullptr;
  Sophus::SE3 T_f_w_;
  Eigen::Matrix6d Cov_;
  ImgPyr img_pyr_;
  std::list<PointFeat*> pt_fts_;
  std::list<LineFeat*> seg_fts_;
};
typedef std::shared_ptr<Frame> FramePtr;
}  // namespace plsvo
