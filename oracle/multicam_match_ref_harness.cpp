// multicam_match_ref_harness.cpp — the reference's OWN Matcher::findMatchDirect (src/matcher.cpp, compiled unmodified where
// it lies) with every keyframe and current frame holding its own camera object, a stand-in vk::PinholeCamera or
// vk::ATANCamera (oracle/refdeps/vikit).
//
// TEST INFRASTRUCTURE, NOT THE PRODUCT.  Built by oracle_multicam_match.build_ref() into
// oracle/_ref/libplsvo_multicam_match_ref.so, with the reference's translation units and flags of oracle/Makefile's `ref`
// target, where the reference sources are present.  It includes atan_ref_harness.cpp (and through it ref_harness.cpp)
// unchanged and adds one entry point: atan_match_ref_harness.cpp's plsvo_ref_atan_match_direct_batch with a camera per
// frame, the layout of plsvo_match_direct_multicam_batch_run.  Each frame's pyramid is a cv::Mat of its camera's size
// cut out of the slot, so findMatchDirect's in-frame test, warpAffine and align2D / align1D see the sizes the reference
// would.  It is the checker of oracle/multicam_match_oracle.cpp.
#include "atan_ref_harness.cpp"

extern "C" int plsvo_ref_match_direct_multicam_batch(const plsvo_match_camera* cams, int n_cams, const int32_t* cam_of_ref,
                                                     const int32_t* cam_of_cur, const plsvo_match_batch* in, const plsvo_match_result* out) {
  if (!cams || n_cams < 1 || !cam_of_ref || !cam_of_cur || !in || !out) return PLSVO_ERR_INVALID;
  plsvo::Config::nPyrLevels() = (size_t)in->n_pyr_levels;
  std::vector<std::unique_ptr<vk::AbstractCamera>> k;
  for (int j = 0; j < n_cams; ++j) {
    const plsvo_match_camera& m = cams[j];
    if (m.model == PLSVO_CAMERA_PINHOLE)
      k.emplace_back(new vk::PinholeCamera(m.pinhole.width, m.pinhole.height, m.pinhole.fx, m.pinhole.fy, m.pinhole.cx, m.pinhole.cy));
    else if (m.model == PLSVO_CAMERA_ATAN)
      k.emplace_back(new vk::ATANCamera(m.atan.width, m.atan.height, m.atan.fx, m.atan.fy, m.atan.cx, m.atan.cy, m.atan.d0));
    else
      return PLSVO_ERR_INVALID;
  }
  auto make_frames = [&](int n, const int32_t* cam_of, const uint8_t* const* img, const size_t* pitch, const size_t* stride,
                         const double* T) {
    std::vector<FramePtr> frames;
    for (int r = 0; r < n; ++r) {
      vk::AbstractCamera* cam = k.at((size_t)cam_of[r]).get();
      FramePtr f(new plsvo::Frame(cam, cv::Mat(), 0.0));
      f->img_pyr_.resize(PLSVO_MAX_LEVELS);
      for (int l = 0; l < PLSVO_MAX_LEVELS; ++l)
        if (img[l])
          f->img_pyr_[l] = cv::Mat(cam->height() >> l, cam->width() >> l, CV_8U, const_cast<uint8_t*>(img[l] + (size_t)r * stride[l]), pitch[l]);
      f->T_f_w_ = pose_from7(T + 7 * (size_t)r);
      frames.push_back(f);
    }
    return frames;
  };
  std::vector<FramePtr> refs = make_frames(in->n_ref_images, cam_of_ref, in->ref_img, in->ref_pitch, in->ref_stride, in->T_ref_w);
  std::vector<FramePtr> curs = make_frames(in->n_cur_images, cam_of_cur, in->cur_img, in->cur_pitch, in->cur_stride, in->T_cur_w);
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
        for (int c = 0; c < 2; ++c) out->A_cur_ref[4 * (size_t)i + 2 * r + c] = matcher.A_cur_ref_(r, c);
  }
  return PLSVO_OK;
}
