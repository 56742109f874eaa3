// atan_match_shimref_harness.cpp — the reprojector scene of atan_next_scenes.h (the reference's own Frame / Point / LineSeg
// objects, every frame given a vk::ATANCamera) answered by the drop-in plsvo::b200::DirectMatcher
// (pl-svo_b200/host/plsvo_shim_next.cpp in -DPLSVO_SHIM_WITH_REFERENCE_HEADERS mode).
//
// TEST INFRASTRUCTURE, NOT THE PRODUCT.  Built by oracle_atan_match.build_shimref() into
// oracle/_ref/libplsvo_atan_match_shimref.so (C ABI of the product library, on the GPU) and, with the C ABI answered by the
// CPU oracle (abi_on_oracle.cpp + atan_abi_on_oracle.cpp), into oracle/_ref/libplsvo_atan_match_shimref_cpu.so.  It
// includes atan_shimref_harness.cpp (and through it shimref_harness.cpp) unchanged and adds one entry point, the shim's
// counterpart of atan_match_ref_harness.cpp's plsvo_ref_atan_match_scene: DirectMatcher must find the ATAN camera through
// the frame and call plsvo_match_direct_atan_batch_run.
#include "atan_shimref_harness.cpp"
#include "atan_next_scenes.h"

extern "C" int plsvo_shimref_atan_match_scene(const plsvo_atan_camera* C, const plsvo_match_batch* in, int n_obs,
                                              const plsvo_scene_match_out* out) {
  if (!C || !in || !out) return PLSVO_ERR_INVALID;
  if (C->width != in->cam.width || C->height != in->cam.height) return PLSVO_ERR_INVALID;
  plsvo::Config::nPyrLevels() = (size_t)in->n_pyr_levels;
  plsvo_scenes::AtanMatchScene sc(C, in, n_obs);
  plsvo::b200::DirectMatcher m(in->n_iter);
  m.search_level_ = -1, m.ref_ftr_ = NULL;
  m.A_cur_ref_.setZero();
  struct Ask {
    plsvo::b200::DirectMatcher& m;
    const std::vector<size_t>& kp;
    const std::vector<size_t>& ks;
    bool point(int i, Vector2d& px) { return m.findMatchDirect(kp[i], px); }
    bool segment(size_t j, Vector2d& spx, Vector2d& epx) { return m.findMatchDirect(ks[j], spx, epx); }
  };
  for (int c = 0; c < in->n_cur_images; ++c) {
    m.reset(*sc.curs[c]);
    std::vector<size_t> kp(in->n_features, 0), ks(sc.segs.size(), 0);
    for (int i = 0; i < in->n_features; ++i)
      if (in->cur_index[i] == c) kp[i] = m.enqueue(sc.points[i].get(), Vector2d(in->px_cur[2 * (size_t)i], in->px_cur[2 * (size_t)i + 1]));
    for (size_t j = 0; j < sc.segs.size(); ++j)
      if (sc.segs[j] && in->cur_index[2 * j] == c)
        ks[j] = m.enqueue(sc.segs[j].get(), Vector2d(in->px_cur[4 * j], in->px_cur[4 * j + 1]), Vector2d(in->px_cur[4 * j + 2], in->px_cur[4 * j + 3]));
    const int rc = m.run();
    if (rc != PLSVO_OK) return rc;
    plsvo_scenes::record_scene_answers(m, sc, in, c, out, Ask{m, kp, ks});
  }
  return PLSVO_OK;
}
