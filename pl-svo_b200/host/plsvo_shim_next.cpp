// plsvo_shim_next.cpp — see plsvo_shim_next.h.  Packs the reference's own objects into the flat arrays of the C ABI
// (one device call per frame and per feature kind), then replays the reference's list logic over the results.
#include "plsvo_shim_next.h"

#include <plsvo/config.h>
#include <vikit/pinhole_camera.h>

#include <cmath>
#include <cstring>
#include <limits>
#include <list>

#include "../../include/plsvo_b200.h"
#include "plsvo_shim.h"

#include <vikit/atan_camera.h>
// A weak reference, as plsvo_shim.cpp's to the ATAN alignment call: the shim is also linked against implementations of
// the C ABI that answer only the pinhole calls; there DirectMatcher::run on ATAN frames returns PLSVO_ERR_CUDA.
#pragma weak plsvo_match_direct_atan_batch_run

namespace plsvo {
namespace b200 {
namespace {

void pose7_of(const Sophus::SE3& T, double* p) {
  const auto& q = T.unit_quaternion();
  const auto& t = T.translation();
  p[0] = q.x(), p[1] = q.y(), p[2] = q.z(), p[3] = q.w();
  p[4] = t[0], p[5] = t[1], p[6] = t[2];
}
bool camera_of(const Frame& f, plsvo_camera* cam) {
  const vk::PinholeCamera* pin = dynamic_cast<const vk::PinholeCamera*>(f.cam_);
  if (!pin) return false;  // the handler is given the undistorted pinhole model (app/run_pipeline.cpp:786-795)
  cam->width = pin->width(), cam->height = pin->height();
  cam->reserved0 = cam->reserved1 = 0;
  cam->fx = pin->fx(), cam->fy = pin->fy(), cam->cx = pin->cx(), cam->cy = pin->cy();
  return true;
}
// The frame's camera for DirectMatcher: the undistorted pinhole (returns 0) or vk::ATANCamera (returns 1; *atan receives the
// constructor arguments recovered from its members, fx = fx_ / width, cx = (cx_ + 0.5) / width, d0 = s_, as
// plsvo_shim.cpp's camera_of does, and cam its image size).  -1 for any other model.
int match_camera_of(const Frame& f, plsvo_camera* cam, plsvo_atan_camera* atan) {
  if (camera_of(f, cam)) return 0;
  const vk::ATANCamera* at = dynamic_cast<const vk::ATANCamera*>(f.cam_);
  if (!at) return -1;
  const double w = at->width(), h = at->height();
  std::memset(cam, 0, sizeof *cam);
  cam->width = at->width(), cam->height = at->height();
  atan->width = at->width(), atan->height = at->height();
  atan->fx = at->fx_ / w, atan->fy = at->fy_ / h, atan->cx = (at->cx_ + 0.5) / w, atan->cy = (at->cy_ + 0.5) / h;
  atan->d0 = at->s_;
  return 1;
}
template <class V>
void put(std::vector<double>& dst, const V& v, int n) {
  for (int i = 0; i < n; ++i) dst.push_back(v[i]);
}

// Everything a call sends to the device is packed into the shim's page-locked scratch (ShimSession::scratch_*), so that
// the library's copies are asynchronous DMA.  Sizes are summed first (Need), the scratch is reserved once, then carved.
struct Need {
  size_t bytes = 0;
  void add(size_t n) { bytes += (n + 255) / 256 * 256 + 256; }
};
template <class T>
const T* pinned_copy(ShimSession& ss, const std::vector<T>& v) {
  if (v.empty()) return nullptr;
  T* p = static_cast<T*>(ss.scratch_take(v.size() * sizeof(T)));
  if (p) std::memcpy(p, v.data(), v.size() * sizeof(T));
  return p;
}
template <class T>
T* pinned_out(ShimSession& ss, size_t n) {
  return static_cast<T*>(ss.scratch_take(std::max<size_t>(n, 1) * sizeof(T)));
}

// The reference observations of one call live in several keyframes, each with its own pyramid allocation; the ABI takes
// one block per level holding all of them ([n_frames][rows_l][cols_l], dense).  Only the levels some row refers to are
// packed (the kernels read a keyframe at the level of its feature only).
struct PackedPyramids {
  bool used[PLSVO_MAX_LEVELS];
  const uint8_t* img[PLSVO_MAX_LEVELS];
  size_t pitch[PLSVO_MAX_LEVELS], stride[PLSVO_MAX_LEVELS];
  size_t n_frames;
  bool plan(const std::vector<Frame*>& frames, const std::vector<int32_t>& level_of_row, int width, int height, Need& need) {
    n_frames = frames.size();
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) used[l] = false, img[l] = nullptr, pitch[l] = stride[l] = 0;
    for (int32_t l : level_of_row) {
      if (l < 0 || l >= PLSVO_MAX_LEVELS) return false;
      used[l] = true;
    }
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
      if (!used[l]) continue;
      pitch[l] = (size_t)(width >> l), stride[l] = pitch[l] * (size_t)(height >> l);
      need.add(stride[l] * n_frames);
    }
    return true;
  }
  bool pack(ShimSession& ss, const std::vector<Frame*>& frames, int width, int height) {
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
      if (!used[l]) continue;
      uint8_t* base = static_cast<uint8_t*>(ss.scratch_take(stride[l] * n_frames));
      if (!base) return false;
      img[l] = base;
      for (size_t r = 0; r < frames.size(); ++r) {
        if ((int)frames[r]->img_pyr_.size() <= l) return false;
        const cv::Mat& m = frames[r]->img_pyr_[l];
        if (m.rows != (height >> l) || m.cols != (width >> l) || !m.data) return false;
        uint8_t* d = base + r * stride[l];
        if (m.step[0] == pitch[l])
          std::memcpy(d, m.data, stride[l]);
        else
          for (int y = 0; y < m.rows; ++y) std::memcpy(d + (size_t)y * pitch[l], m.data + (size_t)y * m.step[0], (size_t)m.cols);
      }
    }
    return true;
  }
};

// the current frame: its levels 0 .. n_levels-1, copied densely into the scratch
struct CurPyramid {
  const uint8_t* img[PLSVO_MAX_LEVELS];
  size_t pitch[PLSVO_MAX_LEVELS], stride[PLSVO_MAX_LEVELS];
  bool plan(const Frame& f, int n_levels, int width, int height, Need& need) {
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
      img[l] = nullptr, pitch[l] = stride[l] = 0;
      if (l >= n_levels) continue;
      if ((int)f.img_pyr_.size() <= l) return false;
      const cv::Mat& m = f.img_pyr_[l];
      if (m.rows != (height >> l) || m.cols != (width >> l) || !m.data) return false;
      pitch[l] = (size_t)m.cols, stride[l] = pitch[l] * (size_t)m.rows;
      need.add(stride[l]);
    }
    return true;
  }
  bool pack(ShimSession& ss, const Frame& f, int n_levels) {
    for (int l = 0; l < n_levels && l < PLSVO_MAX_LEVELS; ++l) {
      const cv::Mat& m = f.img_pyr_[l];
      uint8_t* d = static_cast<uint8_t*>(ss.scratch_take(stride[l]));
      if (!d) return false;
      if (m.step[0] == pitch[l])
        std::memcpy(d, m.data, stride[l]);
      else
        for (int y = 0; y < m.rows; ++y) std::memcpy(d + (size_t)y * pitch[l], m.data + (size_t)y * m.step[0], (size_t)m.cols);
      img[l] = d;
    }
    return true;
  }
};

int32_t frame_index(std::vector<Frame*>& frames, Frame* f) {
  for (size_t k = 0; k < frames.size(); ++k)
    if (frames[k] == f) return (int32_t)k;
  frames.push_back(f);
  return (int32_t)(frames.size() - 1);
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------------
// DirectMatcher
// ------------------------------------------------------------------------------------------------------------------
DirectMatcher::DirectMatcher(int align_max_iter)
    : ref_ftr_(NULL), search_level_(0), cur_(NULL), ran_(false), align_max_iter_(align_max_iter) {
  A_cur_ref_.setZero();
}

void DirectMatcher::reset(const Frame& cur_frame) {
  cands_.clear(), ref_frames_.clear(), ref_index_.clear(), ref_level_.clear(), is_edgelet_.clear();
  ref_px_.clear(), ref_f_.clear(), ref_grad_.clear(), pos_.clear(), px_in_.clear();
  px_out_.clear(), A_out_.clear(), success_.clear(), level_out_.clear();
  cur_ = &cur_frame;
  ran_ = false;
}

int32_t DirectMatcher::add_row(Feature* ref, const Vector2d& px, const Vector3d& f, const Vector3d& pos, const Vector2d& px_est,
                               bool edgelet, const Vector2d& grad) {
  const int32_t row = (int32_t)ref_index_.size();
  ref_index_.push_back(frame_index(ref_frames_, ref->frame));
  ref_level_.push_back(ref->level);
  is_edgelet_.push_back(edgelet ? 1 : 0);
  put(ref_px_, px, 2), put(ref_f_, f, 3), put(ref_grad_, grad, 2), put(pos_, pos, 3), put(px_in_, px_est, 2);
  return row;
}

// list logic on the host: the closest-view observation of the candidate (matcher.cpp:165 / :239)
size_t DirectMatcher::enqueue(Point* pt, const Vector2d& px_est) {
  Cand c;
  c.ref_ftr = NULL, c.is_segment = false, c.row = -1;
  // a point without observations (deleted from the map) has nothing to match against; Reprojector::refine returns before the
  // matcher for TYPE_DELETED points (:280-281), and getCloseViewObs must not be run on an empty list
  c.close_view = cur_ && !pt->obs_.empty() && pt->getCloseViewObs(cur_->pos(), c.ref_ftr);
  if (c.close_view) {
    PointFeat* pf = static_cast<PointFeat*>(c.ref_ftr);
    const bool edgelet = pf->type == PointFeat::EDGELET;
    c.row = add_row(c.ref_ftr, pf->px, pf->f, pt->pos_, px_est, edgelet, edgelet ? pf->grad : Vector2d(0, 0));
  }
  cands_.push_back(c);
  ran_ = false;
  return cands_.size() - 1;
}

size_t DirectMatcher::enqueue(LineSeg* ls, const Vector2d& spx_est, const Vector2d& epx_est) {
  Cand c;
  c.ref_ftr = NULL, c.is_segment = true, c.row = -1;
  c.close_view = cur_ && !ls->obs_.empty() && ls->getCloseViewObs(cur_->pos(), c.ref_ftr);
  if (c.close_view) {
    LineFeat* lf = static_cast<LineFeat*>(c.ref_ftr);
    c.row = add_row(c.ref_ftr, lf->spx, lf->sf, ls->spos_, spx_est, false, Vector2d(0, 0));  // :251-260
    add_row(c.ref_ftr, lf->epx, lf->ef, ls->epos_, epx_est, false, Vector2d(0, 0));          // :261-271
  }
  cands_.push_back(c);
  ran_ = false;
  return cands_.size() - 1;
}

int DirectMatcher::run() {
  ran_ = false;
  if (!cur_) return PLSVO_ERR_INVALID;
  const Frame& cur_frame = *cur_;
  const size_t n = ref_index_.size();
  px_out_.assign(2 * n + 2, 0.0), A_out_.assign(4 * n + 4, 0.0), success_.assign(n + 1, 0), level_out_.assign(n + 1, -1);
  if (n == 0) {
    ran_ = true;
    return PLSVO_OK;
  }
  plsvo_match_batch b;
  std::memset(&b, 0, sizeof b);
  plsvo_atan_camera atan;
  const int model = match_camera_of(cur_frame, &b.cam, &atan);
  if (model < 0) return PLSVO_ERR_INVALID;
  if (model == 1 && !plsvo_match_direct_atan_batch_run) return PLSVO_ERR_CUDA;
  b.n_features = (int32_t)n, b.n_ref_images = (int32_t)ref_frames_.size(), b.n_cur_images = 1;
  b.n_pyr_levels = (int32_t)Config::nPyrLevels(), b.n_iter = align_max_iter_;
  std::vector<double> T_ref(7 * ref_frames_.size()), T_cur(7);
  for (size_t r = 0; r < ref_frames_.size(); ++r) pose7_of(ref_frames_[r]->T_f_w_, &T_ref[7 * r]);
  pose7_of(cur_frame.T_f_w_, T_cur.data());
  std::vector<int32_t> cur_index(n, 0);
  PackedPyramids refs;
  CurPyramid cur;
  Need need;
  if (!refs.plan(ref_frames_, ref_level_, b.cam.width, b.cam.height, need) ||
      !cur.plan(cur_frame, b.n_pyr_levels, b.cam.width, b.cam.height, need))
    return PLSVO_ERR_INVALID;
  for (size_t bytes : {T_ref.size() * 8, T_cur.size() * 8, n * 4, n * 4, n * 4, n, ref_px_.size() * 8, ref_f_.size() * 8, ref_grad_.size() * 8,
                       pos_.size() * 8, px_in_.size() * 8, /* outputs */ n * 16, n, n * 4, n * 32})
    need.add(bytes);
  ShimSession session;
  if (!session.ctx()) return PLSVO_ERR_NO_DEVICE;
  if (!session.scratch_reserve(need.bytes) || !refs.pack(session, ref_frames_, b.cam.width, b.cam.height) ||
      !cur.pack(session, cur_frame, b.n_pyr_levels))
    return session.fail(PLSVO_ERR_INVALID, "DirectMatcher::run (packing)");
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
    b.ref_img[l] = refs.img[l], b.ref_pitch[l] = refs.pitch[l], b.ref_stride[l] = refs.stride[l];
    b.cur_img[l] = cur.img[l], b.cur_pitch[l] = cur.pitch[l], b.cur_stride[l] = cur.stride[l];
  }
  b.T_ref_w = pinned_copy(session, T_ref), b.T_cur_w = pinned_copy(session, T_cur);
  b.ref_index = pinned_copy(session, ref_index_), b.cur_index = pinned_copy(session, cur_index);
  b.ref_px = pinned_copy(session, ref_px_), b.ref_f = pinned_copy(session, ref_f_), b.ref_level = pinned_copy(session, ref_level_);
  b.is_edgelet = pinned_copy(session, is_edgelet_), b.ref_grad = pinned_copy(session, ref_grad_);
  b.pos = pinned_copy(session, pos_), b.px_cur = pinned_copy(session, px_in_);
  plsvo_match_result r;
  std::memset(&r, 0, sizeof r);
  r.px_cur = pinned_out<double>(session, 2 * n), r.success = pinned_out<uint8_t>(session, n);
  r.search_level = pinned_out<int32_t>(session, n), r.A_cur_ref = pinned_out<double>(session, 4 * n);
  if (!b.T_ref_w || !b.T_cur_w || !b.ref_index || !b.cur_index || !b.ref_px || !b.ref_f || !b.ref_level || !b.is_edgelet || !b.ref_grad ||
      !b.pos || !b.px_cur || !r.px_cur || !r.success || !r.search_level || !r.A_cur_ref)
    return session.fail(PLSVO_ERR_INVALID, "DirectMatcher::run (scratch)");
  std::memset(r.A_cur_ref, 0, 4 * n * sizeof(double));  // rows the kernel leaves untouched come back as sent
  const int rc = model == 1 ? plsvo_match_direct_atan_batch_run(session.ctx(), &atan, &b, &r) : plsvo_match_direct_batch_run(session.ctx(), &b, &r);
  if (rc != PLSVO_OK) return session.fail(rc, "DirectMatcher::run");
  std::memcpy(px_out_.data(), r.px_cur, 2 * n * sizeof(double));
  std::memcpy(success_.data(), r.success, n);
  std::memcpy(level_out_.data(), r.search_level, n * sizeof(int32_t));
  std::memcpy(A_out_.data(), r.A_cur_ref, 4 * n * sizeof(double));
  ran_ = true;
  return PLSVO_OK;
}

bool DirectMatcher::findMatchDirect(size_t k, Vector2d& px_cur) {
  if (!ran_ || k >= cands_.size() || cands_[k].is_segment) return false;
  const Cand& c = cands_[k];
  ref_ftr_ = c.ref_ftr;                 // getCloseViewObs writes its pick even when it rejects it (feature3D.cpp:96-99)
  if (!c.close_view) return false;      // matcher.cpp:165-166
  const size_t row = (size_t)c.row;
  if (level_out_[row] < 0) return false;  // :168-170: reference patch too close to the border; nothing else touched
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) A_cur_ref_(i, j) = A_out_[4 * row + 2 * i + j];
  search_level_ = level_out_[row];
  px_cur[0] = px_out_[2 * row], px_cur[1] = px_out_[2 * row + 1];  // :209
  return success_[row] != 0;
}

bool DirectMatcher::findMatchDirect(size_t k, Vector2d& spx_cur, Vector2d& epx_cur) {
  if (!ran_ || k >= cands_.size() || !cands_[k].is_segment) return false;
  const Cand& c = cands_[k];
  ref_ftr_ = c.ref_ftr;
  if (!c.close_view) return false;  // :239-240
  const size_t rs = (size_t)c.row, re = rs + 1;
  if (level_out_[rs] < 0 || level_out_[re] < 0) return false;  // :244-248: either end point outside the reference image
  // start point (:251-260), then end point (:261-271): the members end up as the end point's call leaves them
  spx_cur[0] = px_out_[2 * rs], spx_cur[1] = px_out_[2 * rs + 1];
  epx_cur[0] = px_out_[2 * re], epx_cur[1] = px_out_[2 * re + 1];
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) A_cur_ref_(i, j) = A_out_[4 * re + 2 * i + j];
  search_level_ = level_out_[re];
  return success_[rs] != 0 && success_[re] != 0;
}

// ------------------------------------------------------------------------------------------------------------------
// DepthFilterB200
// ------------------------------------------------------------------------------------------------------------------
DepthFilterB200::DepthFilterB200(feature_detection::DetectorPtr<PointFeat> pt_feature_detector,
                                 feature_detection::DetectorPtr<LineFeat> seg_feature_detector, callback_t seed_converged_cb,
                                 callback_t_ls seed_converged_cb_ls)
    : DepthFilter(pt_feature_detector, seg_feature_detector, seed_converged_cb, seed_converged_cb_ls), last_status_(PLSVO_OK) {}

void DepthFilterB200::updateSeeds(FramePtr frame) {  // depth_filter.cpp:262-268
  last_status_ = update_point_seeds(frame);
  const int rc = update_line_seeds(frame);
  if (last_status_ == PLSVO_OK) last_status_ = rc;
}

namespace {
// the part of plsvo_seed_batch both seed kinds share
struct SeedPack {
  std::vector<Frame*> ref_frames;
  std::vector<int32_t> ref_index, ref_level, cur_index;
  std::vector<uint8_t> is_edgelet;
  std::vector<double> ref_px, ref_f, ref_grad, T_ref;
  std::vector<float> a, b, mu, z_range, sigma2;
  PackedPyramids refs;
  CurPyramid cur;
  void add(Feature* ftr, const Vector2d& px, const Vector3d& f, bool edgelet, const Vector2d& grad, float sa, float sb, float smu,
           float szr, float ssig) {
    ref_index.push_back(frame_index(ref_frames, ftr->frame));
    ref_level.push_back(ftr->level);
    cur_index.push_back(0);
    is_edgelet.push_back(edgelet ? 1 : 0);
    put(ref_px, px, 2), put(ref_f, f, 3), put(ref_grad, grad, 2);
    a.push_back(sa), b.push_back(sb), mu.push_back(smu), z_range.push_back(szr), sigma2.push_back(ssig);
  }
  // describe the batch and pack it into the session's page-locked scratch; `extra` = bytes the caller will take afterwards
  bool fill(ShimSession& ss, plsvo_seed_batch* sb, const Frame& frame, const Matcher::Options& mo, double convergence_thresh, size_t extra) {
    std::memset(sb, 0, sizeof *sb);
    if (!camera_of(frame, &sb->cam)) return false;
    const size_t n = ref_index.size();
    sb->n_seeds = (int32_t)n, sb->n_ref_images = (int32_t)ref_frames.size(), sb->n_cur_images = 1;
    sb->n_pyr_levels = (int32_t)Config::nPyrLevels();
    sb->n_iter = mo.align_max_iter, sb->max_epi_search_steps = (int32_t)mo.max_epi_search_steps;
    sb->align_1d = mo.align_1d, sb->subpix_refinement = mo.subpix_refinement;
    sb->epi_search_edgelet_filtering = mo.epi_search_edgelet_filtering;
    sb->epi_search_edgelet_max_angle = mo.epi_search_edgelet_max_angle;
    sb->seed_convergence_sigma2_thresh = convergence_thresh;
    T_ref.resize(7 * ref_frames.size());
    for (size_t r = 0; r < ref_frames.size(); ++r) pose7_of(ref_frames[r]->T_f_w_, &T_ref[7 * r]);
    std::vector<double> T_cur(7);
    pose7_of(frame.T_f_w_, T_cur.data());
    Need need;
    if (!refs.plan(ref_frames, ref_level, sb->cam.width, sb->cam.height, need) ||
        !cur.plan(frame, sb->n_pyr_levels, sb->cam.width, sb->cam.height, need))
      return false;
    for (size_t bytes : {T_ref.size() * 8, (size_t)56, n * 4, n * 4, n * 4, n, n * 16, n * 24, n * 16, n * 4, n * 4, n * 4, n * 4, n * 4}) need.add(bytes);
    need.bytes += extra;
    if (!ss.scratch_reserve(need.bytes) || !refs.pack(ss, ref_frames, sb->cam.width, sb->cam.height) || !cur.pack(ss, frame, sb->n_pyr_levels))
      return false;
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
      sb->ref_img[l] = refs.img[l], sb->ref_pitch[l] = refs.pitch[l], sb->ref_stride[l] = refs.stride[l];
      sb->cur_img[l] = cur.img[l], sb->cur_pitch[l] = cur.pitch[l], sb->cur_stride[l] = cur.stride[l];
    }
    sb->T_ref_w = pinned_copy(ss, T_ref), sb->T_cur_w = pinned_copy(ss, T_cur);
    sb->ref_index = pinned_copy(ss, ref_index), sb->cur_index = pinned_copy(ss, cur_index);
    sb->ref_px = pinned_copy(ss, ref_px), sb->ref_f = pinned_copy(ss, ref_f), sb->ref_level = pinned_copy(ss, ref_level);
    sb->is_edgelet = pinned_copy(ss, is_edgelet), sb->ref_grad = pinned_copy(ss, ref_grad);
    sb->a = pinned_copy(ss, a), sb->b = pinned_copy(ss, b), sb->mu = pinned_copy(ss, mu), sb->z_range = pinned_copy(ss, z_range);
    sb->sigma2 = pinned_copy(ss, sigma2);
    return sb->T_ref_w && sb->T_cur_w && sb->ref_index && sb->cur_index && sb->ref_px && sb->ref_f && sb->ref_level && sb->is_edgelet &&
           sb->ref_grad && sb->a && sb->b && sb->mu && sb->z_range && sb->sigma2;
  }
};
}  // namespace

int DepthFilterB200::update_point_seeds(FramePtr frame) {  // depth_filter.cpp:270-365
  lock_t lock(seeds_mut_);
  if (seeds_updating_halt_) return PLSVO_OK;
  // seed ageing (:290-293) first: it does not depend on the update
  for (auto it = pt_seeds_.begin(); it != pt_seeds_.end();) {
    if ((PointSeed::batch_counter - it->batch_id) > options_.max_n_kfs)
      it = pt_seeds_.erase(it);
    else
      ++it;
  }
  if (pt_seeds_.empty()) return PLSVO_OK;
  SeedPack pk;
  for (PointSeed& sd : pt_seeds_) {
    const bool edgelet = sd.ftr->type == PointFeat::EDGELET;
    pk.add(sd.ftr, sd.ftr->px, sd.ftr->f, edgelet, edgelet ? sd.ftr->grad : Vector2d(0, 0), sd.a, sd.b, sd.mu, sd.z_range, sd.sigma2);
  }
  const size_t n = pk.ref_index.size();
  std::vector<float> oa(n), ob(n), omu(n), osig(n);
  std::vector<int32_t> status(n);
  std::vector<double> px(2 * n);
  {
    ShimSession session;
    if (!session.ctx()) return PLSVO_ERR_NO_DEVICE;
    plsvo_seed_batch sb;
    if (!pk.fill(session, &sb, *frame, matcher_.options_, options_.seed_convergence_sigma2_thresh, 8 * (n * 16 + 512)))
      return session.fail(PLSVO_ERR_INVALID, "DepthFilterB200::updatePointSeeds (packing)");
    plsvo_seed_result sr;
    std::memset(&sr, 0, sizeof sr);
    sr.a = pinned_out<float>(session, n), sr.b = pinned_out<float>(session, n), sr.mu = pinned_out<float>(session, n);
    sr.sigma2 = pinned_out<float>(session, n), sr.status = pinned_out<int32_t>(session, n), sr.px_cur = pinned_out<double>(session, 2 * n);
    if (!sr.a || !sr.b || !sr.mu || !sr.sigma2 || !sr.status || !sr.px_cur)
      return session.fail(PLSVO_ERR_INVALID, "DepthFilterB200::updatePointSeeds (scratch)");
    const int rc = plsvo_seed_update_batch_run(session.ctx(), &sb, &sr);
    if (rc != PLSVO_OK) return session.fail(rc, "DepthFilterB200::updatePointSeeds");
    std::memcpy(oa.data(), sr.a, n * 4), std::memcpy(ob.data(), sr.b, n * 4), std::memcpy(omu.data(), sr.mu, n * 4);
    std::memcpy(osig.data(), sr.sigma2, n * 4), std::memcpy(status.data(), sr.status, n * 4), std::memcpy(px.data(), sr.px_cur, n * 16);
  }
  // ---- replay of the list logic, in list order ----
  size_t i = 0;
  for (auto it = pt_seeds_.begin(); it != pt_seeds_.end(); ++i) {
    if (!std::isnan(px[2 * i]) || !std::isnan(px[2 * i + 1]))  // Matcher::px_cur_ as this seed's search left it
      matcher_.px_cur_ = Vector2d(px[2 * i], px[2 * i + 1]);
    if (status[i] == PLSVO_SEED_NOT_VISIBLE) {  // :296-304
      ++it;
      continue;
    }
    if (status[i] == PLSVO_SEED_NO_MATCH) {  // :312-318
      it->b = ob[i];
      ++it;
      continue;
    }
    const float z_inv_min = it->mu + std::sqrt(it->sigma2);  // :307, of the state before the update
    it->a = oa[i], it->b = ob[i], it->mu = omu[i], it->sigma2 = osig[i];  // :325
    if (frame->isKeyframe()) pt_feature_detector_->setGridOccpuancy(PointFeat(matcher_.px_cur_));  // :328-332
    if (std::sqrt(it->sigma2) < it->z_range / options_.seed_convergence_sigma2_thresh) {  // :335-355
      Vector3d xyz_world(it->ftr->frame->T_f_w_.inverse() * (it->ftr->f * (1.0 / it->mu)));
      Point* point = new Point(xyz_world, it->ftr);
      it->ftr->feat3D = point;
      seed_converged_cb_(point, it->sigma2);
      it = pt_seeds_.erase(it);
    } else if (std::isnan(z_inv_min)) {  // :356-360
      it = pt_seeds_.erase(it);
    } else {
      ++it;
    }
  }
  return PLSVO_OK;
}

int DepthFilterB200::update_line_seeds(FramePtr frame) {  // depth_filter.cpp:367-471
  lock_t lock(seeds_mut_);
  if (seeds_updating_halt_) return PLSVO_OK;
  for (auto it = seg_seeds_.begin(); it != seg_seeds_.end();) {
    if ((LineSeed::batch_counter - it->batch_id) > options_.max_n_kfs)
      it = seg_seeds_.erase(it);
    else
      ++it;
  }
  if (seg_seeds_.empty()) return PLSVO_OK;
  SeedPack pk;
  std::vector<double> sf, ef;
  std::vector<float> mu_e, zr_e, sig_e;
  for (LineSeed& sd : seg_seeds_) {
    // both end-point searches warp around the segment feature's own px / f (base Feature fields, matcher.cpp:440-447)
    pk.add(sd.ftr, sd.ftr->px, sd.ftr->f, false, Vector2d(0, 0), sd.a, sd.b, sd.mu_s, sd.z_range_s, sd.sigma2_s);
    put(sf, sd.ftr->sf, 3), put(ef, sd.ftr->ef, 3);
    mu_e.push_back(sd.mu_e), zr_e.push_back(sd.z_range_e), sig_e.push_back(sd.sigma2_e);
  }
  const size_t n = pk.ref_index.size();
  std::vector<float> oa(n), ob(n), omu(n), osig(n), omu_e(n), osig_e(n);
  std::vector<int32_t> status(n);
  std::vector<double> pxe(2 * n);
  {
    ShimSession session;
    if (!session.ctx()) return PLSVO_ERR_NO_DEVICE;
    plsvo_line_seed_batch lb;
    std::memset(&lb, 0, sizeof lb);
    if (!pk.fill(session, &lb.seeds, *frame, matcherls_.options_, options_.seed_convergence_sigma2_thresh, 16 * (n * 24 + 512)))
      return session.fail(PLSVO_ERR_INVALID, "DepthFilterB200::updateLineSeeds (packing)");
    lb.seeds.is_edgelet = NULL, lb.seeds.ref_grad = NULL;
    lb.ref_sf = pinned_copy(session, sf), lb.ref_ef = pinned_copy(session, ef);
    lb.mu_e = pinned_copy(session, mu_e), lb.z_range_e = pinned_copy(session, zr_e), lb.sigma2_e = pinned_copy(session, sig_e);
    plsvo_line_seed_result lr;
    std::memset(&lr, 0, sizeof lr);
    lr.seeds.a = pinned_out<float>(session, n), lr.seeds.b = pinned_out<float>(session, n), lr.seeds.mu = pinned_out<float>(session, n);
    lr.seeds.sigma2 = pinned_out<float>(session, n), lr.seeds.status = pinned_out<int32_t>(session, n);
    lr.mu_e = pinned_out<float>(session, n), lr.sigma2_e = pinned_out<float>(session, n), lr.px_cur_e = pinned_out<double>(session, 2 * n);
    if (!lb.ref_sf || !lb.ref_ef || !lb.mu_e || !lb.z_range_e || !lb.sigma2_e || !lr.seeds.a || !lr.seeds.b || !lr.seeds.mu ||
        !lr.seeds.sigma2 || !lr.seeds.status || !lr.mu_e || !lr.sigma2_e || !lr.px_cur_e)
      return session.fail(PLSVO_ERR_INVALID, "DepthFilterB200::updateLineSeeds (scratch)");
    const int rc = plsvo_line_seed_update_batch_run(session.ctx(), &lb, &lr);
    if (rc != PLSVO_OK) return session.fail(rc, "DepthFilterB200::updateLineSeeds");
    std::memcpy(oa.data(), lr.seeds.a, n * 4), std::memcpy(ob.data(), lr.seeds.b, n * 4), std::memcpy(omu.data(), lr.seeds.mu, n * 4);
    std::memcpy(osig.data(), lr.seeds.sigma2, n * 4), std::memcpy(status.data(), lr.seeds.status, n * 4);
    std::memcpy(omu_e.data(), lr.mu_e, n * 4), std::memcpy(osig_e.data(), lr.sigma2_e, n * 4), std::memcpy(pxe.data(), lr.px_cur_e, n * 16);
  }
  size_t i = 0;
  for (auto it = seg_seeds_.begin(); it != seg_seeds_.end(); ++i) {
    if (status[i] == PLSVO_SEED_NOT_VISIBLE) {  // :393-401
      ++it;
      continue;
    }
    if (status[i] == PLSVO_SEED_NO_MATCH) {  // :410-416
      it->b = ob[i];
      ++it;
      continue;
    }
    const float z_inv_min_s = it->mu_s + std::sqrt(it->sigma2_s), z_inv_min_e = it->mu_e + std::sqrt(it->sigma2_e);  // :404-406
    it->a = oa[i], it->b = ob[i], it->mu_s = omu[i], it->sigma2_s = osig[i], it->mu_e = omu_e[i], it->sigma2_e = osig_e[i];  // :425
    if (frame->isKeyframe()) {  // :428-432: the POINT matcher's last position and the end-point search's, as the reference passes them
      matcherls_.px_cur_ = Vector2d(pxe[2 * i], pxe[2 * i + 1]);
      seg_feature_detector_->setGridOccpuancy(LineFeat(matcher_.px_cur_, matcherls_.px_cur_));
    }
    if (std::sqrt(it->sigma2_s) < it->z_range_s / options_.seed_convergence_sigma2_thresh &&
        std::sqrt(it->sigma2_e) < it->z_range_e / options_.seed_convergence_sigma2_thresh) {  // :435-460
      Vector3d xyz_world_s(it->ftr->frame->T_f_w_.inverse() * (it->ftr->sf * (1.0 / it->mu_s)));
      Vector3d xyz_world_e(it->ftr->frame->T_f_w_.inverse() * (it->ftr->ef * (1.0 / it->mu_e)));
      LineSeg* line = new LineSeg(xyz_world_s, xyz_world_e, it->ftr);
      it->ftr->feat3D = line;
      seed_converged_cb_ls_(line, it->sigma2_s, it->sigma2_e);
      it = seg_seeds_.erase(it);
    } else if (std::isnan(z_inv_min_s) || std::isnan(z_inv_min_e)) {  // :461-465
      it = seg_seeds_.erase(it);
    } else {
      ++it;
    }
  }
  return PLSVO_OK;
}

}  // namespace b200
}  // namespace plsvo
