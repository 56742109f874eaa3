// atan_shimref_harness.cpp — the reference's OWN Frame / Feature objects, their frames given a vk::ATANCamera, through the
// drop-in shim (pl-svo_b200/host/plsvo_shim.cpp in -DPLSVO_SHIM_WITH_REFERENCE_HEADERS mode) onto the device.
//
// TEST INFRASTRUCTURE, NOT THE PRODUCT.  Built by oracle_atan.build_shimref() into oracle/_ref/libplsvo_atan_shimref.so
// with the sources and flags of oracle/Makefile's `shimref` target, where the reference sources are present.  It
// includes shimref_harness.cpp unchanged and adds one entry point: its plsvo_shimref_align_batch with the frames'
// camera an ATANCamera, so SparseImgAlign::run must find the camera model through the frame and call the ATAN path.
#include "shimref_harness.cpp"

#include <vikit/atan_camera.h>

extern "C" int plsvo_shimref_atan_align_batch(const plsvo_atan_camera* C, const plsvo_align_batch* B, const plsvo_align_params* P,
                                              const plsvo_align_result* out) {
  if (!C || !B || !P || !out) return PLSVO_ERR_INVALID;
  for (int b = 0; b < B->batch; ++b) {
    const int np = B->pt_count ? B->pt_count[b] : B->n_pts;
    const int ns = B->seg_count ? B->seg_count[b] : B->n_segs;
    const size_t po = (size_t)b * B->n_pts, so = (size_t)b * B->n_segs;
    vk::ATANCamera cam(C->width, C->height, C->fx, C->fy, C->cx, C->cy, C->d0);
    FramePtr ref(new plsvo::Frame(&cam, cv::Mat(), 0.0)), cur(new plsvo::Frame(&cam, cv::Mat(), 1.0));
    ref->img_pyr_.resize(P->max_level + 1);
    cur->img_pyr_.resize(P->max_level + 1);
    for (int l = P->min_level; l <= P->max_level; ++l) {
      const int cols = B->cam.width >> l, rows = B->cam.height >> l;
      ref->img_pyr_[l] = cv::Mat(rows, cols, CV_8U, const_cast<uint8_t*>(B->ref_img[l] + (size_t)b * B->img_stride[l]), B->img_pitch[l]);
      cur->img_pyr_[l] = cv::Mat(rows, cols, CV_8U, const_cast<uint8_t*>(B->cur_img[l] + (size_t)b * B->img_stride[l]), B->img_pitch[l]);
    }
    ref->T_f_w_ = pose_from7(B->T_ref_w + 7 * (size_t)b);
    cur->T_f_w_ = pose_from7(B->T_cur_w + 7 * (size_t)b);
    std::vector<std::unique_ptr<plsvo::Point>> points;
    std::vector<std::unique_ptr<plsvo::LineSeg>> lines;
    std::vector<plsvo::LineFeat*> segs;
    for (int i = 0; i < np; ++i) {
      plsvo::Point* p3 = NULL;
      if (!B->pt_valid || B->pt_valid[po + i]) {
        points.emplace_back(new plsvo::Point(v3(B->pt_pos + 3 * (po + i))));
        p3 = points.back().get();
      }
      ref->pt_fts_.push_back(new plsvo::PointFeat(ref.get(), p3, v2(B->pt_px + 2 * (po + i)), v3(B->pt_f + 3 * (po + i)), 0));
    }
    for (int j = 0; j < ns; ++j) {
      plsvo::LineSeg* l3 = NULL;
      if (!B->seg_valid || B->seg_valid[so + j]) {
        lines.emplace_back(new plsvo::LineSeg(v3(B->seg_spos + 3 * (so + j)), v3(B->seg_epos + 3 * (so + j))));
        l3 = lines.back().get();
      }
      plsvo::LineFeat* f = new plsvo::LineFeat(ref.get(), l3, v2(B->seg_spx + 2 * (so + j)), v2(B->seg_epx + 2 * (so + j)),
                                               v3(B->seg_sf + 3 * (so + j)), v3(B->seg_ef + 3 * (so + j)), 0);
      f->length = B->seg_length[so + j];
      ref->seg_fts_.push_back(f);
      segs.push_back(f);
    }
    // src/frame_handler_mono.cpp:272-274, verbatim but for the Config:: constants
    plsvo::SparseImgAlign img_align(P->max_level, P->min_level, P->n_iter, plsvo::SparseImgAlign::GaussNewton, false, false);
    const size_t img_align_n_tracked = img_align.run(ref, cur);
    pose_to7(cur->T_f_w_, out->T_cur_w + 7 * (size_t)b);
    out->n_tracked[b] = (int64_t)img_align_n_tracked;
    if (out->seg_killed) {
      for (int j = 0; j < B->n_segs; ++j) out->seg_killed[so + j] = 0;
      for (int j = 0; j < ns; ++j)
        out->seg_killed[so + j] = ((!B->seg_valid || B->seg_valid[so + j]) && segs[j]->feat3D == NULL) ? 1 : 0;
    }
  }
  return PLSVO_OK;
}
