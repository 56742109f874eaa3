// plsvo_shim_next.h — reference-typed bindings of the "next" rows (SURVEY.md §8f) over the B200 C ABI: the per-feature
// loops either side of the hot path, each turned into ONE device call per frame while the reference keeps its list
// logic.  Reference-headers build only (-DPLSVO_SHIM_WITH_REFERENCE_HEADERS): everything here speaks the reference's
// own Point / LineSeg / Feature / Frame / PointSeed / LineSeed / DepthFilter types.
//
//   plsvo::b200::DirectMatcher    all Matcher::findMatchDirect calls of Reprojector::reprojectMap
//                                 (src/reprojector.cpp:186-207 -> :236-277 -> :278-387; src/matcher.cpp:159-275)
//   plsvo::b200::DepthFilterB200  DepthFilter with updateSeeds() batched on the device
//                                 (src/depth_filter.cpp:262-471; virtual in include/plsvo/depth_filter.h:214)
//   plsvo::b200::optimizeStructure is declared in plsvo_shim.h (src/frame_handler_base.cpp:202-237).
//
// INTEGRATION.md §6 shows the lines a maintainer changes in reprojector.cpp / frame_handler_mono.cpp.
#pragma once
#ifndef PLSVO_SHIM_WITH_REFERENCE_HEADERS
#error "plsvo_shim_next.h binds reference types: build with -DPLSVO_SHIM_WITH_REFERENCE_HEADERS"
#endif
#include <plsvo/depth_filter.h>
#include <plsvo/feature.h>
#include <plsvo/feature3D.h>
#include <plsvo/frame.h>
#include <plsvo/global.h>

#include <cstddef>
#include <cstdint>
#include <vector>

namespace plsvo {
namespace b200 {

/// Batched stand-in for the `Matcher matcher_` member of Reprojector (include/plsvo/reprojector.h:125).
///
/// Reprojector::reprojectMap first sorts every candidate into grid cells, then walks the cells and calls
/// matcher_.findMatchDirect(*pt, *frame, px_est) once per candidate until a cell has a match (:186-207, :236-277).
/// A candidate's outcome does not depend on any other candidate, so all of them can be evaluated at once:
///   0. reset(*frame) at the top of reprojectMap;
///   1. enqueue() every candidate after the grids are filled — this runs Point/LineSeg::getCloseViewObs (list logic,
///      stays on the host, src/feature3D.cpp:80-124) and records the reference observation;
///   2. run() — ONE plsvo_match_direct_batch_run for the frame (a segment is two rows), or, when the frame's cam_ is a
///      vk::ATANCamera, ONE plsvo_match_direct_atan_batch_run with that camera (its constructor arguments rebuilt from
///      the members fx_..cy_, s_; the keyframes are taken to share it, as in a reference pipeline);
///   3. the reference's own cell loops replay unchanged, with matcher_.findMatchDirect(...) replaced by
///      findMatchDirect(k, ...), which returns what Matcher::findMatchDirect would have returned for candidate k and
///      leaves search_level_ / ref_ftr_ / A_cur_ref_ as the Matcher members would be left (Reprojector::refine reads
///      them at :311-320 and :365).
/// Candidates the sequential loop would never have reached (their cell already matched, or maxFts() hit) are evaluated
/// too; that is extra parallel work, not a change of result.
class DirectMatcher {
 public:
  /// align_max_iter = Matcher::Options::align_max_iter (include/plsvo/matcher.h:85); the pyramid depth is Config::nPyrLevels()
  explicit DirectMatcher(int align_max_iter = 10);

  /// Forgets the previous frame's candidates and targets `cur_frame` (which must outlive run()).
  void reset(const Frame& cur_frame);
  /// Returns the candidate's index k (store it next to the candidate).  px_est as Reprojector::reproject computed it.
  size_t enqueue(Point* pt, const Vector2d& px_est);
  size_t enqueue(LineSeg* ls, const Vector2d& spx_est, const Vector2d& epx_est);
  size_t size() const { return cands_.size(); }

  /// One device call for everything enqueued.  Returns the C-ABI status (PLSVO_OK = 0); on failure every
  /// findMatchDirect(k, ...) below returns false and touches nothing.
  int run();

  /// Matcher::findMatchDirect(const Point&, const Frame&, Vector2d&) for candidate k (src/matcher.cpp:159-211)
  bool findMatchDirect(size_t k, Vector2d& px_cur);
  /// Matcher::findMatchDirect(const LineSeg&, const Frame&, Vector2d&, Vector2d&) for candidate k (:234-275)
  bool findMatchDirect(size_t k, Vector2d& spx_cur, Vector2d& epx_cur);

  // the Matcher members Reprojector::refine reads after a call (include/plsvo/matcher.h:91-99)
  Matrix2d A_cur_ref_;
  Feature* ref_ftr_;
  int search_level_;

 private:
  struct Cand {
    Feature* ref_ftr;   // what getCloseViewObs selected (NULL never: obs_ is non-empty for a map feature)
    bool close_view;    // its return value (:165-166 / :239-240)
    bool is_segment;
    int32_t row;        // first device row (-1: not sent — getCloseViewObs failed)
  };
  std::vector<Cand> cands_;
  // device rows, in enqueue order
  std::vector<Frame*> ref_frames_;
  std::vector<int32_t> ref_index_, ref_level_;
  std::vector<uint8_t> is_edgelet_;
  std::vector<double> ref_px_, ref_f_, ref_grad_, pos_, px_in_;
  // results
  std::vector<double> px_out_, A_out_;
  std::vector<uint8_t> success_;
  std::vector<int32_t> level_out_;
  const Frame* cur_;
  bool ran_;
  int align_max_iter_;
  int32_t add_row(Feature* ref, const Vector2d& px, const Vector3d& f, const Vector3d& pos, const Vector2d& px_est, bool edgelet,
                  const Vector2d& grad);
};

/// DepthFilter whose seed updates run on the device: same constructor, same callbacks, same seed lists.
/// `depth_filter_ = new DepthFilter(pt_detector, seg_detector, cb, cb_ls)` (src/frame_handler_mono.cpp:97) becomes
/// `depth_filter_ = new b200::DepthFilterB200(pt_detector, seg_detector, cb, cb_ls)`; nothing else changes
/// (updateSeeds is virtual, include/plsvo/depth_filter.h:214).
///
/// updateSeeds(frame) restates DepthFilter::updatePointSeeds / updateLineSeeds (src/depth_filter.cpp:270-365, :367-471):
/// seed ageing and erasing, the b++ of a failed search, the state write-back, setGridOccpuancy on keyframes, creating
/// the Point / LineSeg of a converged seed and handing it to seed_converged_cb_[ls_] — with the per-seed work
/// (visibility test, epipolar search, triangulation, computeTau, Gaussian x Beta update) of ALL live seeds in one
/// plsvo_seed_update_batch_run and one plsvo_line_seed_update_batch_run.  Seeds are independent of one another, so
/// the result is that of the sequential loop; (mu, sigma2, a, b) agree to libm round-off (acos / atan / exp on the
/// device vs glibc), everything else exactly.  seeds_updating_halt_ is honoured between the two calls and before the
/// first, not per seed.
class DepthFilterB200 : public DepthFilter {
 public:
  DepthFilterB200(feature_detection::DetectorPtr<PointFeat> pt_feature_detector, feature_detection::DetectorPtr<LineFeat> seg_feature_detector,
                  callback_t seed_converged_cb, callback_t_ls seed_converged_cb_ls);
  /// C-ABI status of the last updateSeeds (PLSVO_OK = 0).  On failure the seeds are left as they were.  Frames whose
  /// cam_ is a vk::ATANCamera are not supported (the seed updates have no ATAN path): updateSeeds then sets an error
  /// status and leaves every seed as it was.
  int last_status() const { return last_status_; }

 protected:
  void updateSeeds(FramePtr frame) override;

 private:
  int last_status_;
  int update_point_seeds(FramePtr frame);
  int update_line_seeds(FramePtr frame);
};

}  // namespace b200
}  // namespace plsvo
