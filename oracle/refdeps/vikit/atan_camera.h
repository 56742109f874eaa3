// Stand-in for rpg_vikit vikit_common/atan_camera.{h,cpp} (vk::ATANCamera, the FOV model of Devernay & Faugeras) —
// TEST INFRASTRUCTURE.
//
// This is a RESTATEMENT, not a copy: rpg_vikit is not vendored with the reference, so the model is written down here
// from upstream vk::ATANCamera (github.com/uzh-rpg/rpg_vikit, vikit_common/src/atan_camera.cpp) as this project's
// contract states it (include/plsvo_b200.h, plsvo_atan_camera).  The constructor arguments are those
// app/run_pipeline.cpp passes: (width, height, fx, fy, cx, cy, d0), fx..cy normalised by the image size.  Whoever has
// an upstream copy at hand should check the formulas below against it; if they differ, this header and the contract in
// include/plsvo_b200.h change together.  It is the one statement of the model the C++ oracles use (atan_oracle.cpp and
// the reference's own translation units compiled against these stand-ins).
#ifndef PLSVO_REFDEPS_VIKIT_ATAN_CAMERA
#define PLSVO_REFDEPS_VIKIT_ATAN_CAMERA
#include <cmath>

#include <vikit/abstract_camera.h>
#include <vikit/math_utils.h>

namespace vk {

class ATANCamera : public AbstractCamera {
 public:
  double fx_, fy_, cx_, cy_;            // pixels: width fx, height fy, cx width - 0.5, cy height - 0.5
  double s_, s_inv_, tans_, tans_inv_;  // d0, 1/d0, 2 tan(d0/2), 1/tans_ (all zero when d0 == 0: no distortion)

  ATANCamera(double width, double height, double fx, double fy, double cx, double cy, double d0)
      : AbstractCamera((int)width, (int)height),
        fx_(width * fx), fy_(height * fy), cx_(cx * width - 0.5), cy_(cy * height - 0.5), s_(d0) {
    if (s_ != 0.0) {
      tans_ = 2.0 * std::tan(s_ / 2.0);
      tans_inv_ = 1.0 / tans_;
      s_inv_ = 1.0 / s_;
    } else {
      s_inv_ = 0.0, tans_ = 0.0, tans_inv_ = 0.0;
    }
  }

  // radial distortion factor of a point at distance r from the principal point on the unit plane
  inline double rtrans_factor(double r) const {
    if (r < 0.001 || s_ == 0.0) return 1.0;
    return s_inv_ * std::atan(r * tans_) / r;
  }
  // undistorted radius of a distorted one
  inline double invrtrans(double r) const {
    if (s_ == 0.0) return r;
    return std::tan(r * s_) * tans_inv_;
  }

  virtual Vector3d cam2world(const double& x, const double& y) const {
    const Vector2d dist_cam((x - cx_) / fx_, (y - cy_) / fy_);
    const double dist_r = dist_cam.norm();
    const double r = invrtrans(dist_r);
    const double factor = dist_r > 0.01 ? r / dist_r : 1.0;
    return unproject2d(Vector2d(factor * dist_cam)).normalized();
  }
  virtual Vector3d cam2world(const Vector2d& px) const { return cam2world(px[0], px[1]); }
  virtual Vector2d world2cam(const Vector3d& xyz_c) const { return world2cam(project2d(xyz_c)); }
  virtual Vector2d world2cam(const Vector2d& uv) const {
    const double r = uv.norm();
    const double factor = rtrans_factor(r);
    const Vector2d dist_cam = factor * uv;
    return Vector2d(cx_ + fx_ * dist_cam[0], cy_ + fy_ * dist_cam[1]);
  }
  virtual double errorMultiplier2() const { return fx_; }
  virtual double errorMultiplier() const { return 4.0 * fx_ * fy_; }
};

}  // namespace vk
#endif
