// atan_next_scenes.h — next_scenes.h's multi-observation reprojector scene with every frame seen through the stand-in
// vk::ATANCamera (oracle/refdeps/vikit/atan_camera.h).  TEST INFRASTRUCTURE, NOT THE PRODUCT.
//
// The scene is MatchScene's: n map points, each observed in n_obs keyframes (the batch's own observation and its
// projections into the next keyframes, through the camera's world2cam / cam2world), and n/2 map segments made of
// consecutive rows.  Only the camera differs; the reference's own getCloseViewObs and findMatchDirect (reference side) or
// DirectMatcher (shim side) then run on these objects.  Include after next_scenes.h.
#pragma once

#include <vikit/atan_camera.h>

namespace plsvo_scenes {

inline std::vector<FramePtr> make_atan_frames(vk::ATANCamera* cam, int n, const uint8_t* const* img, const size_t* pitch,
                                              const size_t* stride, const double* T, int id0) {
  std::vector<FramePtr> frames;
  for (int r = 0; r < n; ++r) {
    FramePtr f(new plsvo::Frame(cam, cv::Mat(), 0.0));
    f->id_ = id0 + r;
    f->img_pyr_.resize(PLSVO_MAX_LEVELS);
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l)
      if (img[l])
        f->img_pyr_[l] = cv::Mat(cam->height() >> l, cam->width() >> l, CV_8U, const_cast<uint8_t*>(img[l] + (size_t)r * stride[l]), pitch[l]);
    f->T_f_w_ = pose_of7(T + 7 * (size_t)r);
    frames.push_back(f);
  }
  return frames;
}

struct AtanMatchScene {
  vk::ATANCamera cam;
  std::vector<FramePtr> refs, curs;
  std::vector<std::unique_ptr<plsvo::Point>> points;
  std::vector<std::unique_ptr<plsvo::LineSeg>> segs;  // [n/2]; NULL where rows 2j, 2j+1 belong to different current frames
  std::vector<std::unique_ptr<plsvo::PointFeat>> pt_obs;
  std::vector<std::unique_ptr<plsvo::LineFeat>> seg_obs;
  AtanMatchScene(const plsvo_atan_camera* C, const plsvo_match_batch* in, int n_obs)
      : cam(C->width, C->height, C->fx, C->fy, C->cx, C->cy, C->d0) {
    refs = make_atan_frames(&cam, in->n_ref_images, in->ref_img, in->ref_pitch, in->ref_stride, in->T_ref_w, 0);
    curs = make_atan_frames(&cam, in->n_cur_images, in->cur_img, in->cur_pitch, in->cur_stride, in->T_cur_w, 1000);
    n_obs = std::max(1, std::min(n_obs, in->n_ref_images));
    for (int i = 0; i < in->n_features; ++i) {
      const size_t I = (size_t)i;
      points.emplace_back(new plsvo::Point(vec3(in->pos + 3 * I)));
      plsvo::Point* pt = points.back().get();
      std::vector<plsvo::PointFeat*> obs;
      for (int k = 0; k < n_obs; ++k) {
        plsvo::Frame* kf = refs[(in->ref_index[i] + k) % in->n_ref_images].get();
        plsvo::PointFeat* f;
        if (k == 0) {
          f = new plsvo::PointFeat(kf, pt, vec2(in->ref_px + 2 * I), vec3(in->ref_f + 3 * I), in->ref_level[i]);
          if (in->is_edgelet && in->is_edgelet[i]) f->type = plsvo::PointFeat::EDGELET, f->grad = vec2(in->ref_grad + 2 * I);
        } else {
          const Vector2d px = kf->w2c(pt->pos_);
          f = new plsvo::PointFeat(kf, pt, px, kf->c2f(px), in->ref_level[i]);
        }
        pt_obs.emplace_back(f);
        obs.push_back(f);
      }
      if (i & 1) std::reverse(obs.begin(), obs.end());
      for (plsvo::PointFeat* f : obs) pt->addFrameRef(f);
    }
    for (int j = 0; j + 1 < in->n_features; j += 2) {
      segs.emplace_back();
      if (in->cur_index[j] != in->cur_index[j + 1]) continue;
      const size_t S = (size_t)j, E = (size_t)j + 1;
      segs.back().reset(new plsvo::LineSeg(vec3(in->pos + 3 * S), vec3(in->pos + 3 * E)));
      plsvo::LineSeg* ls = segs.back().get();
      for (int k = 0; k < n_obs; ++k) {
        plsvo::Frame* kf = refs[(in->ref_index[j] + k) % in->n_ref_images].get();
        const Vector2d spx = k == 0 ? vec2(in->ref_px + 2 * S) : Vector2d(kf->w2c(ls->spos_));
        const Vector3d sf = k == 0 ? vec3(in->ref_f + 3 * S) : Vector3d(kf->c2f(spx));
        const Vector2d epx = kf->w2c(ls->epos_);
        plsvo::LineFeat* f = new plsvo::LineFeat(kf, ls, spx, epx, sf, kf->c2f(epx), in->ref_level[j]);
        seg_obs.emplace_back(f);
        ls->addFrameRef(f);
      }
    }
  }
};

// Reprojector::refineBestCandidate -> refine over the scene, candidates of a frame in batch order: `Matcher` is the
// reference's plsvo::Matcher (answer: findMatchDirect(obj, frame, px...)) or the shim's DirectMatcher (answered through
// its own enqueue / run / findMatchDirect(k, ...) by the caller-supplied `ask`); what Reprojector::refine reads afterwards
// is recorded as plsvo_ref_match_scene records it.
template <class M, class Ask>
void record_scene_answers(M& m, const AtanMatchScene& sc, const plsvo_match_batch* in, int c, const plsvo_scene_match_out* out, Ask ask) {
  for (int i = 0; i < in->n_features; ++i) {
    if (in->cur_index[i] != c) continue;
    const size_t I = (size_t)i;
    Vector2d px(in->px_cur[2 * I], in->px_cur[2 * I + 1]);
    out->pt_found[i] = ask.point(i, px) ? 1 : 0;
    out->pt_px[2 * I] = px[0], out->pt_px[2 * I + 1] = px[1];
    out->pt_level[i] = m.search_level_;
    for (int r = 0; r < 2; ++r)
      for (int k = 0; k < 2; ++k) out->pt_A[4 * I + 2 * r + k] = m.A_cur_ref_(r, k);
    out->pt_ref[i] = m.ref_ftr_ ? frame_slot(sc.refs, m.ref_ftr_->frame) : -1;
  }
  for (size_t j = 0; j < sc.segs.size(); ++j) {
    if (!sc.segs[j] || in->cur_index[2 * j] != c) continue;
    Vector2d spx(in->px_cur[4 * j], in->px_cur[4 * j + 1]), epx(in->px_cur[4 * j + 2], in->px_cur[4 * j + 3]);
    out->seg_found[j] = ask.segment(j, spx, epx) ? 1 : 0;
    out->seg_spx[2 * j] = spx[0], out->seg_spx[2 * j + 1] = spx[1], out->seg_epx[2 * j] = epx[0], out->seg_epx[2 * j + 1] = epx[1];
    out->seg_level[j] = m.search_level_;
    for (int r = 0; r < 2; ++r)
      for (int k = 0; k < 2; ++k) out->seg_A[4 * j + 2 * r + k] = m.A_cur_ref_(r, k);
    out->seg_ref[j] = m.ref_ftr_ ? frame_slot(sc.refs, m.ref_ftr_->frame) : -1;
  }
}

}  // namespace plsvo_scenes
