// atan_match_ref_harness.cpp — the reference's OWN Matcher::findMatchDirect (src/matcher.cpp, compiled unmodified where it
// lies) with keyframes and current frames given the stand-in vk::ATANCamera (oracle/refdeps/vikit/atan_camera.h).
//
// TEST INFRASTRUCTURE, NOT THE PRODUCT.  Built by oracle_atan_match.build_ref() into oracle/_ref/libplsvo_atan_match_ref.so,
// with the reference's translation units and flags of oracle/Makefile's `ref` target, where the reference sources are
// present.  It includes atan_ref_harness.cpp (and through it ref_harness.cpp) unchanged and adds two entry points:
// ref_harness.cpp's plsvo_ref_match_direct_batch and plsvo_ref_match_scene with the frames' camera an ATANCamera.  The
// first is the checker of oracle/atan_match_oracle.cpp, the second of DirectMatcher on ATAN frames
// (oracle/atan_match_shimref_harness.cpp).
#include "atan_ref_harness.cpp"
#include "atan_next_scenes.h"

extern "C" int plsvo_ref_atan_match_direct_batch(const plsvo_atan_camera* C, const plsvo_match_batch* in, const plsvo_match_result* out) {
  if (!C || !in || !out) return PLSVO_ERR_INVALID;
  if (C->width != in->cam.width || C->height != in->cam.height) return PLSVO_ERR_INVALID;
  plsvo::Config::nPyrLevels() = (size_t)in->n_pyr_levels;
  vk::ATANCamera cam(C->width, C->height, C->fx, C->fy, C->cx, C->cy, C->d0);
  auto make_frames = [&](int n, const uint8_t* const* img, const size_t* pitch, const size_t* stride, const double* T) {
    std::vector<FramePtr> frames;
    for (int r = 0; r < n; ++r) {
      FramePtr f(new plsvo::Frame(&cam, cv::Mat(), 0.0));
      f->img_pyr_.resize(PLSVO_MAX_LEVELS);
      for (int l = 0; l < PLSVO_MAX_LEVELS; ++l)
        if (img[l])
          f->img_pyr_[l] = cv::Mat(in->cam.height >> l, in->cam.width >> l, CV_8U, const_cast<uint8_t*>(img[l] + (size_t)r * stride[l]), pitch[l]);
      f->T_f_w_ = pose_from7(T + 7 * (size_t)r);
      frames.push_back(f);
    }
    return frames;
  };
  std::vector<FramePtr> refs = make_frames(in->n_ref_images, in->ref_img, in->ref_pitch, in->ref_stride, in->T_ref_w);
  std::vector<FramePtr> curs = make_frames(in->n_cur_images, in->cur_img, in->cur_pitch, in->cur_stride, in->T_cur_w);
  for (int i = 0; i < in->n_features; ++i) {
    plsvo::Frame* rf = refs[in->ref_index[i]].get();
    plsvo::Point pt(v3(in->pos + 3 * (size_t)i));
    plsvo::PointFeat ftr(rf, &pt, v2(in->ref_px + 2 * (size_t)i), v3(in->ref_f + 3 * (size_t)i), in->ref_level[i]);
    if (in->is_edgelet && in->is_edgelet[i]) {
      ftr.type = plsvo::PointFeat::EDGELET;
      ftr.grad = v2(in->ref_grad + 2 * (size_t)i);
    }
    pt.addFrameRef(&ftr);
    plsvo::Matcher matcher{};
    matcher.search_level_ = -1;
    matcher.options_.align_max_iter = in->n_iter;
    Vector2d px(in->px_cur[2 * (size_t)i], in->px_cur[2 * (size_t)i + 1]);
    const bool ok = matcher.findMatchDirect(pt, *curs[in->cur_index[i]], px);
    out->px_cur[2 * (size_t)i] = px[0], out->px_cur[2 * (size_t)i + 1] = px[1];
    out->success[i] = ok ? 1 : 0;
    if (out->search_level) out->search_level[i] = matcher.search_level_;
    if (out->A_cur_ref && matcher.search_level_ >= 0)
      for (int r = 0; r < 2; ++r)
        for (int k = 0; k < 2; ++k) out->A_cur_ref[4 * (size_t)i + 2 * r + k] = matcher.A_cur_ref_(r, k);
  }
  return PLSVO_OK;
}

// Reprojector::refineBestCandidate -> refine (src/reprojector.cpp:236-387) on the multi-observation scene of
// atan_next_scenes.h: one reference Matcher answers every candidate of a frame in turn, as plsvo_ref_match_scene does.
extern "C" int plsvo_ref_atan_match_scene(const plsvo_atan_camera* C, const plsvo_match_batch* in, int n_obs, const plsvo_scene_match_out* out) {
  if (!C || !in || !out) return PLSVO_ERR_INVALID;
  if (C->width != in->cam.width || C->height != in->cam.height) return PLSVO_ERR_INVALID;
  plsvo::Config::nPyrLevels() = (size_t)in->n_pyr_levels;
  plsvo_scenes::AtanMatchScene sc(C, in, n_obs);
  plsvo::Matcher m{};
  m.search_level_ = -1, m.ref_ftr_ = NULL;
  m.A_cur_ref_.setZero();
  m.options_.align_max_iter = in->n_iter;
  struct Ask {
    plsvo::Matcher& m;
    plsvo_scenes::AtanMatchScene& sc;
    plsvo::Frame& cur;
    bool point(int i, Vector2d& px) { return m.findMatchDirect(*sc.points[i], cur, px); }
    bool segment(size_t j, Vector2d& spx, Vector2d& epx) { return m.findMatchDirect(*sc.segs[j], cur, spx, epx); }
  };
  for (int c = 0; c < in->n_cur_images; ++c) plsvo_scenes::record_scene_answers(m, sc, in, c, out, Ask{m, sc, *sc.curs[c]});
  return PLSVO_OK;
}
