// atan_oracle.cpp — the CPU oracle's SparseImgAlign restatement seen through vk::ATANCamera.
//
// TEST INFRASTRUCTURE, NOT THE PRODUCT (see the header of plsvo_oracle.cpp).  On the reference's ATAN path
// (app/run_pipeline.cpp, cam_model ATAN) frames are not rectified: SparseImgAlign projects every patch with the distorted
// cam_->world2cam (src/sparse_img_align.cpp:425,584), reads errorMultiplier2() = fx_ (:203,:279), and the feature
// constructors form bearings with its cam2world (src/feature.cpp:42,98-99).  Nothing else on the path reads the camera.
//
// This translation unit includes plsvo_oracle.cpp unchanged and derives from its SparseImgAlign: the passes that call
// world2cam (computePoints, computeSegments) are restated with the ATAN projection, and the solver loop that calls them
// (computeResiduals, optimize, run) is repeated so that it reaches them; precompute, sampling, patches, the SE3 algebra
// and the solver arithmetic are the included ones.  The experiments of the pinhole oracle (h_mode, chi2 in double,
// traces) are left out.  The camera model is the stand-in oracle/refdeps/vikit/atan_camera.h, the one statement of it.
// The pose optimiser needs no ATAN path: it is camera-free apart from errorMultiplier2, which its caller passes.
//
// Build: oracle_atan.py (same flags as oracle/Makefile: strict IEEE, no FMA contraction).
#include "plsvo_oracle.cpp"

#include <vikit/atan_camera.h>

namespace {

struct AtanSparseImgAlign : SparseImgAlign {
  const vk::ATANCamera* cam = nullptr;

  Vec3 world2cam_px(Vec3 p) const {  // vk::ATANCamera::world2cam(xyz) = world2cam(project2d(xyz))
    const Eigen::Vector2d px = cam->world2cam(Eigen::Vector3d(p.x, p.y, p.z));
    return {px[0], px[1], 0};
  }

  // sparse_img_align.cpp:380-502, as SparseImgAlign::computePoints
  void computePoints(const SE3& T_cur_from_ref, double H[36], double Jres[6], float& chi2) {
    Patch patch(level_image(B->cur_img, level_));
    const float scale = 1.0f / (1 << level_);
    chi2 = 0.0f;
    std::fill(H, H + 36, 0.0);
    std::fill(Jres, Jres + 6, 0.0);
    for (int i = 0; i < n_pts; ++i) {
      if (!pt_cache_.visible[i]) continue;
      const Vec3 pos{pt_pos[3 * i], pt_pos[3 * i + 1], pt_pos[3 * i + 2]};
      const double depth = norm(pos - ref_pos);
      const Vec3 xyz_ref = Vec3{pt_f[3 * i], pt_f[3 * i + 1], pt_f[3 * i + 2]} * depth;
      const Vec3 xyz_cur = se3_act(T_cur_from_ref, xyz_ref);
      const Vec3 uv = world2cam_px(xyz_cur);
      patch.setPosition(uv.x * scale, uv.y * scale);
      if (!patch.isInFrame(patch.halfsize)) continue;
      patch.computeInterpWeights();
      patch.setRoi();
      ++patch_iters;
      const float* cache_ptr = &pt_cache_.ref_patch[(size_t)16 * i];
      const double* Jc = &pt_cache_.jacobian[(size_t)6 * 16 * i];
      const int stride = patch.img.stride;
      for (int y = 0; y < 4; ++y) {
        const uint8_t* img_ptr = patch.roi + (size_t)y * stride;
        for (int x = 0; x < 4; ++x, ++img_ptr, ++cache_ptr, Jc += 6) {
          const float intensity_cur = patch.wTL * img_ptr[0] + patch.wTR * img_ptr[1] + patch.wBL * img_ptr[stride] +
                                      patch.wBR * img_ptr[stride + 1];
          const float res = intensity_cur - (*cache_ptr);
          float weight = 1.0;
          weight = 1.0 / (1.0 + fabsf(res));  // :479
          chi2 += res * res * weight;         // :484
          n_meas_++;
          for (int r = 0; r < 6; ++r) {
            for (int c = 0; c < 6; ++c) H[r * 6 + c] += Jc[r] * Jc[c] * weight;  // :491
            Jres[r] -= Jc[r] * res * weight;                                       // :492
          }
        }
      }
    }
  }

  // sparse_img_align.cpp:504-695, as SparseImgAlign::computeSegments
  void computeSegments(const SE3& T_cur_from_ref, double H[36], double Jres[6], float& chi2) {
    Patch patch(level_image(B->cur_img, level_));
    const float scale = 1.0f / (1 << level_);
    chi2 = 0.0f;
    std::fill(H, H + 36, 0.0);
    std::fill(Jres, Jres + 6, 0.0);
    std::vector<float> ls_res;
    for (int j = 0; j < n_segs; ++j) {
      if (!seg_alive[j]) continue;
      if (!seg_cache_.visible[j]) continue;
      size_t cache_idx = patch_offset[j];
      double inc2d[2];
      size_t N_samples = setup_sampling(patch.size, seg_spx + 2 * j, seg_epx + 2 * j, seg_length[j], inc2d);
      N_samples = 1 + (N_samples - 1) / (1 << level_);
      const Vec3 spos{seg_spos[3 * j], seg_spos[3 * j + 1], seg_spos[3 * j + 2]};
      const Vec3 epos{seg_epos[3 * j], seg_epos[3 * j + 1], seg_epos[3 * j + 2]};
      const double p_depth = norm(spos - ref_pos);
      const Vec3 p_ref = Vec3{seg_sf[3 * j], seg_sf[3 * j + 1], seg_sf[3 * j + 2]} * p_depth;
      const double q_depth = norm(epos - ref_pos);
      const Vec3 q_ref = Vec3{seg_ef[3 * j], seg_ef[3 * j + 1], seg_ef[3 * j + 2]} * q_depth;
      const double nm1 = (double)(N_samples - 1);
      const Vec3 d = q_ref - p_ref;
      const Vec3 inc3d{d.x / nm1, d.y / nm1, d.z / nm1};
      Vec3 xyz_ref = p_ref;
      double Hs[36] = {0}, Js[6] = {0};
      ls_res.clear();
      bool good_line = true;
      ensure_seg_capacity(cache_idx / 16 + N_samples + 1);
      for (unsigned sample = 0; sample < N_samples; ++sample, xyz_ref = xyz_ref + inc3d) {
        const Vec3 xyz_cur = se3_act(T_cur_from_ref, xyz_ref);
        const Vec3 uv = world2cam_px(xyz_cur);
        patch.setPosition(uv.x * scale, uv.y * scale);
        if (!patch.isInFrame(patch.halfsize)) {
          cache_idx += patch.size;
          good_line = false;
          sample = (unsigned)N_samples;
          continue;
        }
        patch.computeInterpWeights();
        patch.setRoi();
        ++patch_iters;
        const int stride = patch.img.stride;
        for (int y = 0; y < 4; ++y) {
          const uint8_t* img_ptr = patch.roi + (size_t)y * stride;
          for (int x = 0; x < 4; ++x, ++img_ptr, ++cache_idx) {
            const float intensity_cur = patch.wTL * img_ptr[0] + patch.wTR * img_ptr[1] +
                                        patch.wBL * img_ptr[stride] + patch.wBR * img_ptr[stride + 1];
            const float res = intensity_cur - seg_cache_.ref_patch[cache_idx];
            ls_res.push_back(res);
            const double* Jc = &seg_cache_.jacobian[6 * cache_idx];
            for (int r = 0; r < 6; ++r) {
              for (int c = 0; c < 6; ++c) Hs[r * 6 + c] += Jc[r] * Jc[c];  // :628
              Js[r] -= Jc[r] * res;                                          // :629
            }
          }
        }
      }
      float res_ = 0.0;
      for (float r : ls_res) res_ += fabsf(r);
      res_ = res_ / double(N_samples);  // :647
      if (good_line && res_ < 200.0) {
        float weight = 1.0;
        weight = 1.0 / (1.0 + res_);  // :675
        for (int k = 0; k < 36; ++k) H[k] += Hs[k] * weight / res_;  // :681
        for (int k = 0; k < 6; ++k) Jres[k] += Js[k] * weight;        // :682
        chi2 += res_ * res_ * weight;                                  // :683
        n_meas_++;
      } else {
        seg_alive[j] = 0;  // it->feat3D = NULL  (:688)
      }
    }
  }

  // sparse_img_align.cpp:112-193
  double computeResiduals(const SE3& T_cur_from_ref) {
    if (!have_ref_patch_cache_) {  // :126-127, :104-110
      precomputePoints();
      precomputeSegments();
      have_ref_patch_cache_ = true;
    }
    use_weights_ = true;  // :132
    double pt_H[36], pt_J[6], seg_H[36], seg_J[6];
    float pt_chi2, seg_chi2;
    computePoints(T_cur_from_ref, pt_H, pt_J, pt_chi2);
    computeSegments(T_cur_from_ref, seg_H, seg_J, seg_chi2);
    for (int k = 0; k < 36; ++k) H_[k] = pt_H[k] + seg_H[k];  // :167
    for (int k = 0; k < 6; ++k) Jres_[k] = pt_J[k] + seg_J[k];
    float chi2 = pt_chi2 + seg_chi2;  // :171
    return chi2 / n_meas_;            // :192  (float / size_t -> float)
  }

  // vk::NLLSSolver<6,SE3>::optimizeGaussNewton + SparseImgAlign::solve/update (:697-710)
  void optimize(SE3& model) {
    if (use_weights_) {  // pre-pass: computeResiduals(model, false, true), excluded from the patch accounting
      const uint32_t saved = patch_iters;
      computeResiduals(model);
      patch_iters = saved;
    }
    SE3 old_model = model;
    for (iter_ = 0; iter_ < n_iter_; ++iter_) {
      std::fill(H_, H_ + 36, 0.0);
      std::fill(Jres_, Jres_ + 6, 0.0);
      n_meas_ = 0;
      const double new_chi2 = computeResiduals(model);
      ++iters_at_level[level_];
      solve6(H_, Jres_, x_);  // :699
      if (std::isnan(x_[0])) stop_ = true;
      if ((iter_ > 0 && new_chi2 > chi2_) || stop_) {
        model = old_model;
        break;
      }
      double mx[6];
      for (int k = 0; k < 6; ++k) mx[k] = -x_[k];
      const SE3 new_model = se3_mul(model, se3_exp(mx));  // :709
      old_model = model;
      model = new_model;
      chi2_ = new_chi2;
      if (norm_max6(x_) <= eps_) break;
    }
  }

  // sparse_img_align.cpp:54-95.  Returns n_meas_/16; writes T_cur_w.
  size_t run(const plsvo_align_params& P, const SE3& T_ref_w, SE3& T_cur_w, int n_pts_list, int n_segs_list) {
    chi2_ = 1e10, n_meas_ = 0, iter_ = 0, stop_ = false;
    n_iter_ = n_iter_init_ = P.n_iter;
    eps_ = P.eps;
    max_level_ = P.max_level, min_level_ = P.min_level;
    std::fill(H_, H_ + 36, 0.0);
    if (n_pts_list == 0 && n_segs_list == 0) return 0;  // :58-62
    float total_length = 0;
    for (int j = 0; j < n_segs; ++j) total_length += seg_length[j];  // :69-73
    const int max_num_seg_samples = (int)std::ceil(total_length / 4);
    pt_cache_.ref_patch.assign((size_t)n_pts * 16, 0.f);
    pt_cache_.jacobian.assign((size_t)n_pts * 16 * 6, 0.0);
    pt_cache_.visible.assign(n_pts, 0);
    seg_cache_.ref_patch.assign((size_t)max_num_seg_samples * 16, 0.f);
    seg_cache_.jacobian.assign((size_t)max_num_seg_samples * 16 * 6, 0.0);
    seg_cache_.visible.assign(n_segs, 0);
    ref_pos = se3_inverse(T_ref_w).t;                              // Frame::pos(), frame.h:131
    SE3 T_cur_from_ref = se3_mul(T_cur_w, se3_inverse(T_ref_w));  // :80
    for (level_ = max_level_; level_ >= min_level_; --level_) {
      std::fill(pt_cache_.jacobian.begin(), pt_cache_.jacobian.end(), 0.0);   // :85
      std::fill(seg_cache_.jacobian.begin(), seg_cache_.jacobian.end(), 0.0); // :86
      have_ref_patch_cache_ = false;
      optimize(T_cur_from_ref);  // :90
    }
    T_cur_w = se3_mul(T_cur_from_ref, T_ref_w);  // :92
    return n_meas_ / 16;                         // :94
  }
};

// bearing of a pixel as the feature constructors form it (src/feature.cpp:42,98-99)
void atan_bearing(const vk::ATANCamera& cam, const double* px, double* f) {
  const Eigen::Vector3d v = cam.cam2world(px[0], px[1]);
  f[0] = v[0], f[1] = v[1], f[2] = v[2];
}

// as align_one of plsvo_oracle.cpp; NULL bearings are formed with the camera's cam2world
void atan_align_one(const plsvo_atan_camera* C, const plsvo_align_batch* B, const plsvo_align_params* P,
                    const plsvo_align_result* out, int b) {
  const vk::ATANCamera cam(C->width, C->height, C->fx, C->fy, C->cx, C->cy, C->d0);
  // the pinhole fields the included precompute reads (errorMultiplier2, image size) hold the ATAN camera's
  plsvo_align_batch Bd = *B;
  Bd.cam.fx = cam.fx_, Bd.cam.fy = cam.fy_, Bd.cam.cx = cam.cx_, Bd.cam.cy = cam.cy_;
  AtanSparseImgAlign s;
  s.cam = &cam;
  s.B = &Bd, s.b = b;
  const int np = B->pt_count ? B->pt_count[b] : B->n_pts;
  const int ns = B->seg_count ? B->seg_count[b] : B->n_segs;
  s.n_pts = np, s.n_segs = ns;
  const size_t po = (size_t)b * B->n_pts, so = (size_t)b * B->n_segs;
  std::vector<double> pt_f, seg_sf, seg_ef, pt_pos, seg_spos, seg_epos;
  s.pt_px = B->pt_px ? B->pt_px + 2 * po : nullptr;
  if (B->pt_f) {
    s.pt_f = B->pt_f + 3 * po;
  } else {
    pt_f.resize(3 * (size_t)np);
    for (int i = 0; i < np; ++i) atan_bearing(cam, s.pt_px + 2 * i, &pt_f[3 * i]);
    s.pt_f = pt_f.data();
  }
  s.pt_pos = B->pt_pos ? B->pt_pos + 3 * po : nullptr;
  s.pt_valid = B->pt_valid ? B->pt_valid + po : nullptr;
  s.seg_spx = B->seg_spx ? B->seg_spx + 2 * so : nullptr;
  s.seg_epx = B->seg_epx ? B->seg_epx + 2 * so : nullptr;
  if (B->seg_sf && B->seg_ef) {
    s.seg_sf = B->seg_sf + 3 * so, s.seg_ef = B->seg_ef + 3 * so;
  } else {
    seg_sf.resize(3 * (size_t)ns), seg_ef.resize(3 * (size_t)ns);
    for (int j = 0; j < ns; ++j) {
      atan_bearing(cam, s.seg_spx + 2 * j, &seg_sf[3 * j]);
      atan_bearing(cam, s.seg_epx + 2 * j, &seg_ef[3 * j]);
    }
    s.seg_sf = seg_sf.data(), s.seg_ef = seg_ef.data();
  }
  s.seg_spos = B->seg_spos ? B->seg_spos + 3 * so : nullptr;
  s.seg_epos = B->seg_epos ? B->seg_epos + 3 * so : nullptr;
  s.seg_length = B->seg_length ? B->seg_length + so : nullptr;
  s.seg_alive.assign(ns, 1);
  if (B->seg_valid)
    for (int j = 0; j < ns; ++j) s.seg_alive[j] = B->seg_valid[so + j] ? 1 : 0;
  std::vector<uint8_t> alive0 = s.seg_alive;

  const SE3 T_ref_w = se3_from_pose7(B->T_ref_w + 7 * (size_t)b);
  SE3 T_cur_w = se3_from_pose7(B->T_cur_w + 7 * (size_t)b);
  const bool empty = (np == 0 && ns == 0);
  const size_t n_tracked = s.run(*P, T_ref_w, T_cur_w, np, ns);

  if (out->T_cur_w) {
    if (empty)
      std::memcpy(out->T_cur_w + 7 * (size_t)b, B->T_cur_w + 7 * (size_t)b, 7 * sizeof(double));
    else
      se3_to_pose7(T_cur_w, out->T_cur_w + 7 * (size_t)b);
  }
  if (out->n_tracked) out->n_tracked[b] = (int64_t)n_tracked;
  if (out->H) std::memcpy(out->H + 36 * (size_t)b, s.H_, 36 * sizeof(double));
  if (out->seg_killed) {
    for (int j = 0; j < B->n_segs; ++j) out->seg_killed[so + j] = 0;
    for (int j = 0; j < ns; ++j) out->seg_killed[so + j] = (alive0[j] && !s.seg_alive[j]) ? 1 : 0;
  }
  if (out->iters)
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) out->iters[(size_t)b * PLSVO_MAX_LEVELS + l] = s.iters_at_level[l];
  if (out->status) out->status[b] = (empty ? 1 : 0) | (s.stop_ ? 2 : 0);
  if (out->patch_iters) out->patch_iters[b] = s.patch_iters;
  if (out->patch_levels) out->patch_levels[b] = s.patch_levels;
}

}  // namespace

extern "C" {

// SparseImgAlign::run for a batch of pairs seen through one vk::ATANCamera.  Images, poses and features as for
// plsvo_oracle_align_batch (pt_f / seg_sf / seg_ef may be NULL); batch->cam is ignored apart from its image size.
int plsvo_oracle_atan_align_batch(const plsvo_atan_camera* cam, const plsvo_align_batch* batch, const plsvo_align_params* params,
                                  const plsvo_align_result* out, int n_threads) {
  if (!cam || !batch || !params || !out) return PLSVO_ERR_INVALID;
  if (params->max_level < params->min_level || params->min_level < 0 || params->max_level >= PLSVO_MAX_LEVELS)
    return PLSVO_ERR_INVALID;
  if (cam->width != batch->cam.width || cam->height != batch->cam.height) return PLSVO_ERR_INVALID;
  parallel_for(batch->batch, n_threads, [&](int b) { atan_align_one(cam, batch, params, out, b); });
  return PLSVO_OK;
}

// the stand-in camera, for the checks of its NumPy restatement: n pixels -> bearings, n points -> pixels,
// and errorMultiplier2
void plsvo_oracle_atan_cam2world(const plsvo_atan_camera* c, const double* px, int n, double* f) {
  const vk::ATANCamera cam(c->width, c->height, c->fx, c->fy, c->cx, c->cy, c->d0);
  for (int i = 0; i < n; ++i) atan_bearing(cam, px + 2 * i, f + 3 * i);
}
void plsvo_oracle_atan_world2cam(const plsvo_atan_camera* c, const double* xyz, int n, double* px) {
  const vk::ATANCamera cam(c->width, c->height, c->fx, c->fy, c->cx, c->cy, c->d0);
  for (int i = 0; i < n; ++i) {
    const Eigen::Vector2d p = cam.world2cam(Eigen::Vector3d(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]));
    px[2 * i] = p[0], px[2 * i + 1] = p[1];
  }
}
double plsvo_oracle_atan_error_multiplier2(const plsvo_atan_camera* c) {
  return vk::ATANCamera(c->width, c->height, c->fx, c->fy, c->cx, c->cy, c->d0).errorMultiplier2();
}

}  // extern "C"
