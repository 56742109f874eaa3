// plsvo_shim.cpp — packs Frame / Feature lists into the flat arrays of the C ABI, calls B = 1, and
// writes results (pose, covariance, NULLed feat3D pointers) back.  Error behaviour follows the
// reference: no exceptions; run() returns 0 when there is nothing to track; the pose optimiser
// returns with its outputs untouched when there are no observations.
#include "plsvo_shim.h"

#include <cmath>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <deque>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/plsvo_b200.h"
#ifdef PLSVO_SHIM_WITH_REFERENCE_HEADERS
#include <vikit/atan_camera.h>
#endif
// A weak reference: the shim is also linked against implementations of the C ABI that answer only the pinhole calls
// (the CPU-oracle backend of the tests); there a frame with an ATAN camera fails like any other failed call.
#pragma weak plsvo_align_atan_batch_run

namespace plsvo {
namespace {

std::mutex g_mu;
plsvo_ctx* g_ctx = nullptr;
int g_device = 0;
std::string g_err;

plsvo_ctx* ctx() {
  if (!g_ctx) {
    if (plsvo_ctx_create(g_device, nullptr, &g_ctx) != PLSVO_OK) {
      g_err = plsvo_last_error(nullptr);
      std::fprintf(stderr, "[plsvo_b200] cannot create device context: %s\n", g_err.c_str());
      g_ctx = nullptr;
    }
  }
  return g_ctx;
}

void pose7_of(const Sophus::SE3& T, double* p) {
  const auto& q = T.unit_quaternion();
  const auto& t = T.translation();
  p[0] = q.x(), p[1] = q.y(), p[2] = q.z(), p[3] = q.w();
  p[4] = t[0], p[5] = t[1], p[6] = t[2];
}
Sophus::SE3 se3_of(const double* p) {
  Eigen::Vector3d t;
  t[0] = p[4], t[1] = p[5], t[2] = p[6];
  return Sophus::SE3(Eigen::Quaterniond(p[3], p[0], p[1], p[2]), t);  // Eigen ctor order: w, x, y, z
}
// The frame's camera model: the undistorted pinhole the handler is given for cam_model Pinhole (run_pipeline.cpp:786-795)
// or, for cam_model ATAN, vk::ATANCamera (:804-819), whose frames are aligned unrectified.  For ATAN, *atan receives the
// constructor arguments recovered from the camera's members (fx = fx_ / width, cx = (cx_ + 0.5) / width, d0 = s_; the
// library derives fx_ = width fx again, exact whenever fx_ / width is) and cam the image size the batch must carry.
enum CamModel { kNoCamera, kPinhole, kAtan };
CamModel camera_of(const Frame& f, plsvo_camera* cam, plsvo_atan_camera* atan) {
  std::memset(cam, 0, sizeof *cam);
  if (const vk::PinholeCamera* pin = dynamic_cast<const vk::PinholeCamera*>(f.cam_)) {
    cam->width = pin->width(), cam->height = pin->height();
    cam->fx = pin->fx(), cam->fy = pin->fy(), cam->cx = pin->cx(), cam->cy = pin->cy();
    return kPinhole;
  }
  if (const vk::ATANCamera* at = dynamic_cast<const vk::ATANCamera*>(f.cam_)) {
    const double w = at->width(), h = at->height();
    cam->width = at->width(), cam->height = at->height();
    atan->width = at->width(), atan->height = at->height();
    atan->fx = at->fx_ / w, atan->fy = at->fy_ / h, atan->cx = (at->cx_ + 0.5) / w, atan->cy = (at->cy_ + 0.5) / h;
    atan->d0 = at->s_;
    return kAtan;
  }
  return kNoCamera;
}
template <class V>
void put(std::vector<double>& dst, const V& v, int n) {
  for (int i = 0; i < n; ++i) dst.push_back(v[i]);
}

}  // namespace

int shim_set_device(int device) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_ctx) plsvo_ctx_destroy(g_ctx);
  g_ctx = nullptr;
  g_device = device;
  return ctx() ? 0 : -1;
}
const char* shim_last_error() { return g_err.c_str(); }

ShimSession::ShimSession() {
  g_mu.lock();
  ctx_ = plsvo::ctx();
}
ShimSession::~ShimSession() { g_mu.unlock(); }
namespace {
char* g_scratch = nullptr;
size_t g_scratch_cap = 0, g_scratch_off = 0;
}  // namespace
bool ShimSession::scratch_reserve(size_t bytes) {
  g_scratch_off = 0;
  if (bytes <= g_scratch_cap) return true;
  if (g_scratch) plsvo_host_free(g_scratch);
  g_scratch = nullptr, g_scratch_cap = 0;
  void* p = nullptr;
  const size_t cap = bytes + bytes / 4 + 4096;
  if (plsvo_host_alloc(&p, cap) != PLSVO_OK || !p) return false;
  g_scratch = static_cast<char*>(p), g_scratch_cap = cap;
  return true;
}
void* ShimSession::scratch_take(size_t bytes) {
  const size_t at = (g_scratch_off + 255) / 256 * 256;
  if (!g_scratch || at + bytes > g_scratch_cap) return nullptr;
  g_scratch_off = at + bytes;
  return g_scratch + at;
}
int ShimSession::fail(int rc, const char* what) {
  g_err = ctx_ ? plsvo_last_error(ctx_) : "no device context";
  std::fprintf(stderr, "[plsvo_b200] %s failed: %s\n", what, g_err.c_str());
  return rc;
}

SparseImgAlign::SparseImgAlign(int max_level, int min_level, int n_iter, Method method, bool display, bool verbose)
    : max_level_(max_level), min_level_(min_level), n_iter_(n_iter) {
  (void)method, (void)display, (void)verbose;
  std::memset(H_, 0, sizeof H_);
}

size_t SparseImgAlign::run(FramePtr ref_frame, FramePtr cur_frame) {
  if (ref_frame->pt_fts_.empty() && ref_frame->seg_fts_.empty()) return 0;  // sparse_img_align.cpp:58-62
  std::lock_guard<std::mutex> lk(g_mu);
  plsvo_ctx* c = ctx();
  if (!c) return 0;
  plsvo_align_batch b;
  std::memset(&b, 0, sizeof b);
  plsvo_atan_camera atan;
  const CamModel model = camera_of(*ref_frame, &b.cam, &atan);
  if (model == kNoCamera) return 0;
  if (model == kAtan && !plsvo_align_atan_batch_run) {
    g_err = "this C ABI implementation has no plsvo_align_atan_batch_run";
    std::fprintf(stderr, "[plsvo_b200] SparseImgAlign::run failed: %s\n", g_err.c_str());
    return 0;
  }
  b.batch = 1;
  b.n_pts = (int)ref_frame->pt_fts_.size();
  b.n_segs = (int)ref_frame->seg_fts_.size();
  for (int l = min_level_; l <= max_level_ && l < PLSVO_MAX_LEVELS; ++l) {
    const cv::Mat& r = ref_frame->img_pyr_.at(l);
    const cv::Mat& u = cur_frame->img_pyr_.at(l);
    b.ref_img[l] = r.data, b.cur_img[l] = u.data;
    b.img_pitch[l] = r.step[0];  // both frames come from createImgPyramid: same geometry
    b.img_stride[l] = r.step[0] * (size_t)r.rows;
    if (u.step[0] != r.step[0]) return 0;
  }
  double T_ref[7], T_cur[7];
  pose7_of(ref_frame->T_f_w_, T_ref);
  pose7_of(cur_frame->T_f_w_, T_cur);
  b.T_ref_w = T_ref, b.T_cur_w = T_cur;
  std::vector<double> px, f, pos, spx, epx, sf, ef, spos, epos, len;
  std::vector<uint8_t> pv, sv;
  for (PointFeat* p : ref_frame->pt_fts_) {
    put(px, p->px, 2), put(f, p->f, 3);
    pv.push_back(p->feat3D != NULL);
    if (p->feat3D) put(pos, p->feat3D->pos_, 3); else pos.insert(pos.end(), 3, 0.0);
  }
  std::vector<LineFeat*> segs;
  for (auto* s0 : ref_frame->seg_fts_) {
    LineFeat* s = static_cast<LineFeat*>(s0);
    segs.push_back(s);
    put(spx, s->spx, 2), put(epx, s->epx, 2), put(sf, s->sf, 3), put(ef, s->ef, 3);
    len.push_back(s->length);
    sv.push_back(s->feat3D != NULL);
    if (s->feat3D) put(spos, s->feat3D->spos_, 3), put(epos, s->feat3D->epos_, 3);
    else spos.insert(spos.end(), 3, 0.0), epos.insert(epos.end(), 3, 0.0);
  }
  b.pt_px = px.data(), b.pt_f = f.data(), b.pt_pos = pos.data(), b.pt_valid = pv.data();
  b.seg_spx = spx.data(), b.seg_epx = epx.data(), b.seg_sf = sf.data(), b.seg_ef = ef.data();
  b.seg_spos = spos.data(), b.seg_epos = epos.data(), b.seg_length = len.data(), b.seg_valid = sv.data();
  plsvo_align_params p = {max_level_, min_level_, n_iter_, 0, 0.000001};  // eps_ (:51)
  double T_out[7];
  int64_t n_tracked = 0;
  std::vector<uint8_t> killed(segs.size() + 1, 0);
  plsvo_align_result r;
  std::memset(&r, 0, sizeof r);
  r.T_cur_w = T_out, r.n_tracked = &n_tracked, r.H = H_, r.seg_killed = killed.data();
  const int rc = model == kAtan ? plsvo_align_atan_batch_run(c, &atan, &b, &p, &r) : plsvo_align_batch_run(c, &b, &p, &r);
  if (rc != PLSVO_OK) {
    g_err = plsvo_last_error(c);
    std::fprintf(stderr, "[plsvo_b200] SparseImgAlign::run failed: %s\n", g_err.c_str());
    return 0;
  }
  cur_frame->T_f_w_ = se3_of(T_out);  // :92
  for (size_t j = 0; j < segs.size(); ++j)
    if (killed[j]) segs[j]->feat3D = NULL;  // :687-688 (mutates the REFERENCE frame's features)
  return (size_t)n_tracked;
}

void SparseImgAlign::getFisherInformation(double out36[36]) const {
  const double sigma_i_sq = 5e-4 * 255 * 255;  // :99
  for (int i = 0; i < 36; ++i) out36[i] = H_[i] / sigma_i_sq;
}
#ifdef PLSVO_SHIM_WITH_REFERENCE_HEADERS
Eigen::Matrix<double, 6, 6> SparseImgAlign::getFisherInformation() {
  Eigen::Matrix<double, 6, 6> I;
  double tmp[36];
  static_cast<const SparseImgAlign*>(this)->getFisherInformation(tmp);
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) I(r, c) = tmp[r * 6 + c];
  return I;
}
#endif

namespace pose_optimizer {
namespace {
void run(double reproj_thresh, size_t n_iter, int n_iter_ref, FramePtr& frame, double& estimated_scale,
         double& error_init, double& error_final, size_t& num_obs_pt, size_t& num_obs_ls) {
  std::lock_guard<std::mutex> lk(g_mu);
  // The caller (frame_handler_mono.cpp:325-336) declares the observation counts uninitialised and then tests
  // `pt + ls < 10`.  The reference assigns num_obs_pt (= 0) before its "no observations" return (pose_optimizer.cpp:
  // 72,88-89); here every exit without a result — no device, a failed call, no observations — leaves both counts and
  // the errors at zero, so that test deterministically reports RESULT_FAILURE instead of reading garbage.
  num_obs_pt = 0, num_obs_ls = 0;
  error_init = 0.0, error_final = 0.0;
  plsvo_ctx* c = ctx();
  if (!c) return;
  plsvo_poseopt_batch b;
  std::memset(&b, 0, sizeof b);
  b.batch = 1;
  b.n_pts = (int)frame->pt_fts_.size();
  b.n_segs = (int)frame->seg_fts_.size();
  if (b.n_pts == 0 && b.n_segs == 0) return;
  b.fx = frame->cam_->errorMultiplier2();  // |fx| of the pinhole, fx_ of vk::ATANCamera: the optimiser's only camera read
  double T[7];
  pose7_of(frame->T_f_w_, T);
  b.T_f_w = T;
  std::vector<double> f, pos, line, spos, epos;
  std::vector<int32_t> pl, sl;
  std::vector<uint8_t> pv, sv;
  std::vector<PointFeat*> pts;
  std::vector<LineFeat*> segs;
  for (PointFeat* p : frame->pt_fts_) {
    pts.push_back(p);
    put(f, p->f, 3);
    pl.push_back(p->level);
    pv.push_back(p->feat3D != NULL);
    if (p->feat3D) put(pos, p->feat3D->pos_, 3); else pos.insert(pos.end(), 3, 0.0);
  }
  for (auto* s0 : frame->seg_fts_) {
    LineFeat* s = static_cast<LineFeat*>(s0);
    segs.push_back(s);
    put(line, s->line, 3);
    sl.push_back(s->level);
    sv.push_back(s->feat3D != NULL);
    if (s->feat3D) put(spos, s->feat3D->spos_, 3), put(epos, s->feat3D->epos_, 3);
    else spos.insert(spos.end(), 3, 0.0), epos.insert(epos.end(), 3, 0.0);
  }
  b.pt_f = f.data(), b.pt_pos = pos.data(), b.pt_level = pl.data(), b.pt_valid = pv.data();
  b.seg_line = line.data(), b.seg_spos = spos.data(), b.seg_epos = epos.data(), b.seg_level = sl.data();
  b.seg_valid = sv.data();
  plsvo_poseopt_params p = {reproj_thresh, (int32_t)n_iter, n_iter_ref};
  double T_out[7], cov[36], scale = 0, e0 = 0, e1 = 0;
  int64_t npt = 0, nls = 0;
  int32_t status = 0;
  std::vector<uint8_t> po(pts.size() + 1, 0), so(segs.size() + 1, 0);
  plsvo_poseopt_result r;
  std::memset(&r, 0, sizeof r);
  r.T_f_w = T_out, r.cov = cov, r.estimated_scale = &scale, r.error_init = &e0, r.error_final = &e1;
  r.num_obs_pt = &npt, r.num_obs_ls = &nls, r.pt_outlier = po.data(), r.seg_outlier = so.data(), r.status = &status;
  if (plsvo_poseopt_batch_run(c, &b, &p, &r) != PLSVO_OK) {
    g_err = plsvo_last_error(c);
    std::fprintf(stderr, "[plsvo_b200] pose_optimizer failed: %s\n", g_err.c_str());
    return;
  }
  if (status & 1) return;  // no observations: outputs untouched (pose_optimizer.cpp:88-89)
  frame->T_f_w_ = se3_of(T_out);
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) frame->Cov_(i, j) = cov[i * 6 + j];  // :199
  for (size_t i = 0; i < pts.size(); ++i)
    if (po[i]) pts[i]->feat3D = NULL;  // :218
  for (size_t j = 0; j < segs.size(); ++j)
    if (so[j]) segs[j]->feat3D = NULL;  // :239
  estimated_scale = scale, error_init = e0, error_final = e1;
  num_obs_pt = (size_t)npt, num_obs_ls = (size_t)nls;
}
}  // namespace

void optimizeGaussNewton(const double reproj_thresh, const size_t n_iter, const bool verbose, FramePtr& frame,
                         double& estimated_scale, double& error_init, double& error_final, size_t& num_obs_pt,
                         size_t& num_obs_ls) {
  (void)verbose;
  run(reproj_thresh, n_iter, -1, frame, estimated_scale, error_init, error_final, num_obs_pt, num_obs_ls);
}
void optimizeGaussNewton(const double reproj_thresh, const size_t n_iter, const size_t n_iter_ref, const bool verbose,
                         FramePtr& frame, double& estimated_scale, double& error_init, double& error_final,
                         size_t& num_obs_pt, size_t& num_obs_ls) {
  (void)verbose;
  run(reproj_thresh, n_iter, (int)n_iter_ref, frame, estimated_scale, error_init, error_final, num_obs_pt, num_obs_ls);
}
}  // namespace pose_optimizer

#ifdef PLSVO_SHIM_WITH_REFERENCE_HEADERS
namespace b200 {
int optimizeStructure(FramePtr frame, size_t max_n_pts, int max_iter, size_t max_n_segs, int max_iter_segs) {
  std::lock_guard<std::mutex> lk(g_mu);
  plsvo_ctx* c = ctx();
  if (!c) return PLSVO_ERR_NO_DEVICE;
  // selection: frame_handler_base.cpp:209-218 and :221-230, verbatim
  std::deque<Point*> pts;
  for (PointFeat* f : frame->pt_fts_)
    if (f->feat3D != NULL) pts.push_back(f->feat3D);
  max_n_pts = std::min(max_n_pts, pts.size());
  std::nth_element(pts.begin(), pts.begin() + max_n_pts, pts.end(),
                   [](Point* l, Point* r) { return l->last_structure_optim_ < r->last_structure_optim_; });
  std::deque<LineSeg*> segs;
  for (auto* f0 : frame->seg_fts_) {
    LineFeat* f = static_cast<LineFeat*>(f0);
    if (f->feat3D != NULL) segs.push_back(f->feat3D);
  }
  max_n_segs = std::min(max_n_segs, segs.size());
  std::nth_element(segs.begin(), segs.begin() + max_n_segs, segs.end(),
                   [](LineSeg* l, LineSeg* r) { return l->last_structure_optim_ < r->last_structure_optim_; });
  // observation lists -> CSR in obs_ order (the reference's summation order), keyframe poses de-duplicated
  std::vector<Frame*> frames;
  std::vector<double> T;
  auto frame_index = [&](Frame* f) {
    for (size_t k = 0; k < frames.size(); ++k)
      if (frames[k] == f) return (int32_t)k;
    frames.push_back(f);
    double p7[7];
    pose7_of(f->T_f_w_, p7);
    T.insert(T.end(), p7, p7 + 7);
    return (int32_t)(frames.size() - 1);
  };
  std::vector<int32_t> pb(1, 0), pfr, sb(1, 0), sfr;
  std::vector<double> pf, ppos, ssf, sef, sspos, sepos;
  for (size_t i = 0; i < max_n_pts; ++i) {
    for (PointFeat* o : pts[i]->obs_) {
      pfr.push_back(frame_index(o->frame));
      put(pf, o->f, 3);
    }
    pb.push_back((int32_t)pfr.size());
    put(ppos, pts[i]->pos_, 3);
  }
  for (size_t i = 0; i < max_n_segs; ++i) {
    for (LineFeat* o : segs[i]->obs_) {
      sfr.push_back(frame_index(o->frame));
      put(ssf, o->sf, 3);
      put(sef, o->ef, 3);
    }
    sb.push_back((int32_t)sfr.size());
    put(sspos, segs[i]->spos_, 3);
    put(sepos, segs[i]->epos_, 3);
  }
  if (max_n_pts == 0 && max_n_segs == 0) return PLSVO_OK;
  plsvo_structopt_batch b;
  std::memset(&b, 0, sizeof b);
  b.n_points = (int32_t)max_n_pts, b.n_segs = (int32_t)max_n_segs, b.n_frames = (int32_t)frames.size();
  b.n_iter_pts = max_iter, b.n_iter_segs = max_iter_segs;
  b.T_f_w = T.data();
  b.pt_obs_begin = pb.data(), b.pt_obs_frame = pfr.data(), b.pt_obs_f = pf.data(), b.pt_pos = ppos.data();
  b.seg_obs_begin = sb.data(), b.seg_obs_frame = sfr.data(), b.seg_obs_sf = ssf.data(), b.seg_obs_ef = sef.data();
  b.seg_spos = sspos.data(), b.seg_epos = sepos.data();
  std::vector<double> opos(3 * max_n_pts + 3), ospos(3 * max_n_segs + 3), oepos(3 * max_n_segs + 3);
  plsvo_structopt_result r;
  std::memset(&r, 0, sizeof r);
  r.pt_pos = opos.data(), r.seg_spos = ospos.data(), r.seg_epos = oepos.data();
  const int rc = plsvo_structopt_batch_run(c, &b, &r);
  if (rc != PLSVO_OK) {
    g_err = plsvo_last_error(c);
    std::fprintf(stderr, "[plsvo_b200] optimizeStructure failed: %s\n", g_err.c_str());
    return rc;
  }
  for (size_t i = 0; i < max_n_pts; ++i) {
    for (int k = 0; k < 3; ++k) pts[i]->pos_[k] = opos[3 * i + k];
    pts[i]->last_structure_optim_ = frame->id_;  // :217
  }
  for (size_t i = 0; i < max_n_segs; ++i) {
    for (int k = 0; k < 3; ++k) segs[i]->spos_[k] = ospos[3 * i + k], segs[i]->epos_[k] = oepos[3 * i + k];
    segs[i]->last_structure_optim_ = frame->id_;  // :229
  }
  return PLSVO_OK;
}
}  // namespace b200
#endif
}  // namespace plsvo
