// atan_ref_harness.cpp — the reference's OWN SparseImgAlign (src/sparse_img_align.cpp, compiled unmodified where it lies)
// driven through the stand-in vk::ATANCamera (oracle/refdeps/vikit/atan_camera.h).
//
// TEST INFRASTRUCTURE, NOT THE PRODUCT.  Built by oracle_atan.build_ref() into oracle/_ref/libplsvo_atan_ref.so, with the
// reference's translation units and flags of oracle/Makefile's `ref` target, where the reference sources are present.
// It includes ref_harness.cpp unchanged (the out-of-line Frame members, AlignProbe, the pose helpers) and adds one
// entry point: ref_harness.cpp's align_one with the frames given an ATANCamera instead of a PinholeCamera, and bearings
// formed by that camera's cam2world where the batch carries none — as the feature constructors would (src/feature.cpp:42,
// 98-99).  It is the checker of oracle/atan_oracle.cpp.
#include "ref_harness.cpp"

#include <vikit/atan_camera.h>

namespace {

void atan_ref_align_one(const plsvo_atan_camera* C, const plsvo_align_batch* B, const plsvo_align_params* P,
                        const plsvo_align_result* out, int b) {
  const int np = B->pt_count ? B->pt_count[b] : B->n_pts;
  const int ns = B->seg_count ? B->seg_count[b] : B->n_segs;
  const size_t po = (size_t)b * B->n_pts, so = (size_t)b * B->n_segs;

  vk::ATANCamera cam(C->width, C->height, C->fx, C->fy, C->cx, C->cy, C->d0);
  FramePtr ref(new plsvo::Frame(&cam, cv::Mat(), 0.0));
  FramePtr cur(new plsvo::Frame(&cam, cv::Mat(), 1.0));
  ref->img_pyr_.resize(P->max_level + 1);
  cur->img_pyr_.resize(P->max_level + 1);
  for (int l = P->min_level; l <= P->max_level; ++l) {
    const int cols = B->cam.width >> l, rows = B->cam.height >> l;
    ref->img_pyr_[l] = cv::Mat(rows, cols, CV_8U, const_cast<uint8_t*>(B->ref_img[l] + (size_t)b * B->img_stride[l]), B->img_pitch[l]);
    cur->img_pyr_[l] = cv::Mat(rows, cols, CV_8U, const_cast<uint8_t*>(B->cur_img[l] + (size_t)b * B->img_stride[l]), B->img_pitch[l]);
  }
  ref->T_f_w_ = pose_from7(B->T_ref_w + 7 * (size_t)b);
  cur->T_f_w_ = pose_from7(B->T_cur_w + 7 * (size_t)b);

  auto bearing = [&](const double* f, const double* px) { return f ? v3(f) : cam.cam2world(px[0], px[1]); };
  std::vector<std::unique_ptr<plsvo::Point>> points;
  std::vector<std::unique_ptr<plsvo::LineSeg>> lines;
  for (int i = 0; i < np; ++i) {
    const bool valid = !B->pt_valid || B->pt_valid[po + i];
    plsvo::Point* p3 = NULL;
    if (valid) {
      points.emplace_back(new plsvo::Point(v3(B->pt_pos + 3 * (po + i))));
      p3 = points.back().get();
    }
    const double* px = B->pt_px + 2 * (po + i);
    ref->pt_fts_.push_back(new plsvo::PointFeat(ref.get(), p3, v2(px), bearing(B->pt_f ? B->pt_f + 3 * (po + i) : nullptr, px), 0));
  }
  std::vector<plsvo::LineFeat*> segs;
  for (int j = 0; j < ns; ++j) {
    const bool valid = !B->seg_valid || B->seg_valid[so + j];
    plsvo::LineSeg* l3 = NULL;
    if (valid) {
      lines.emplace_back(new plsvo::LineSeg(v3(B->seg_spos + 3 * (so + j)), v3(B->seg_epos + 3 * (so + j))));
      l3 = lines.back().get();
    }
    const double* spx = B->seg_spx + 2 * (so + j);
    const double* epx = B->seg_epx + 2 * (so + j);
    plsvo::LineFeat* f = new plsvo::LineFeat(ref.get(), l3, v2(spx), v2(epx), bearing(B->seg_sf ? B->seg_sf + 3 * (so + j) : nullptr, spx),
                                             bearing(B->seg_ef ? B->seg_ef + 3 * (so + j) : nullptr, epx), 0);
    f->length = B->seg_length[so + j];
    ref->seg_fts_.push_back(f);
    segs.push_back(f);
  }

  // src/frame_handler_mono.cpp:272-274
  AlignProbe img_align(P->max_level, P->min_level, P->n_iter);
  img_align.eps_ = P->eps;
  const bool empty = (np == 0 && ns == 0);
  const size_t n_tracked = img_align.run(ref, cur);

  if (out->T_cur_w) {
    if (empty)
      std::memcpy(out->T_cur_w + 7 * (size_t)b, B->T_cur_w + 7 * (size_t)b, 7 * sizeof(double));
    else
      pose_to7(cur->T_f_w_, out->T_cur_w + 7 * (size_t)b);
  }
  if (out->n_tracked) out->n_tracked[b] = (int64_t)n_tracked;
  if (out->H)
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) out->H[36 * (size_t)b + 6 * i + j] = empty ? 0.0 : img_align.H()(i, j);
  if (out->seg_killed) {
    for (int j = 0; j < B->n_segs; ++j) out->seg_killed[so + j] = 0;
    for (int j = 0; j < ns; ++j) {
      const bool valid = !B->seg_valid || B->seg_valid[so + j];
      out->seg_killed[so + j] = (valid && segs[j]->feat3D == NULL) ? 1 : 0;
    }
  }
  if (out->iters)
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) out->iters[(size_t)b * PLSVO_MAX_LEVELS + l] = img_align.iters[l];
  if (out->status) out->status[b] = (empty ? 1 : 0) | (img_align.stop_ ? 2 : 0);
  if (out->patch_iters) out->patch_iters[b] = 0;  // not observable from outside the reference class
  if (out->patch_levels) out->patch_levels[b] = 0;
}

}  // namespace

extern "C" int plsvo_ref_atan_align_batch(const plsvo_atan_camera* cam, const plsvo_align_batch* batch,
                                          const plsvo_align_params* params, const plsvo_align_result* out, int n_threads) {
  if (!cam || !batch || !params || !out) return PLSVO_ERR_INVALID;
  if (cam->width != batch->cam.width || cam->height != batch->cam.height) return PLSVO_ERR_INVALID;
  parallel_for(batch->batch, n_threads, [&](int b) { atan_ref_align_one(cam, batch, params, out, b); });
  return PLSVO_OK;
}
