// multicam_match_oracle.cpp — the CPU oracle's Matcher::findMatchDirect with a camera per image, pinhole or ATAN.
//
// TEST INFRASTRUCTURE, NOT THE PRODUCT (see the header of plsvo_oracle.cpp).  In the reference the cameras belong to the
// frames: findMatchDirect (src/matcher.cpp:159-211) tests the reference pixel against ref_ftr_->frame->cam_, and
// warp::getWarpMatrixAffine (:44-71) lifts with cam_ref.cam2world and projects with cam_cur.world2cam.  warpAffine and
// align2D / align1D are bounded by the images they read, so by the ref camera's and the current camera's sizes.
//
// This translation unit includes plsvo_oracle.cpp unchanged.  Its warp matrix takes two vk::AbstractCamera, the stand-in
// PinholeCamera and ATANCamera of oracle/refdeps/vikit (the one statement of each model), and runs the included
// getBestSearchLevel, warpAffine, align2D and align1D restatements downstream of it with per-image sizes.  The one-camera
// oracles (plsvo_oracle.cpp's pinhole matcher, atan_match_oracle.cpp) stay as they are: they check the one-camera calls,
// and the tests hold this oracle equal to them when every image shares one camera.  A second entry point takes A_cur_ref
// as an input: on the device atan / tan are not glibc's, so the GPU tests compare what follows A_cur_ref with what this
// code computes from the kernel's own A_cur_ref.
//
// Build: oracle_multicam_match.py (the flags of oracle/Makefile: strict IEEE, no FMA contraction).
#include "plsvo_oracle.cpp"

#include <memory>

#include <vikit/atan_camera.h>
#include <vikit/pinhole_camera.h>

namespace {

// warp::getWarpMatrixAffine (src/matcher.cpp:44-71) with cam_ref.cam2world and cam_cur.world2cam, in the operation order
// of plsvo_oracle.cpp's pinhole warp_matrix_affine
void warp_matrix_affine_2cam(const vk::AbstractCamera& cam_ref, const vk::AbstractCamera& cam_cur, const double* px_ref, Vec3 f_ref,
                             double depth_ref, const SE3& T_cur_ref, int level_ref, double A[2][2]) {
  const int halfpatch_size = 5;
  const Vec3 xyz_ref = f_ref * depth_ref;
  const double step = (double)halfpatch_size * (double)(1 << level_ref);
  const Eigen::Vector3d du = cam_ref.cam2world(px_ref[0] + step, px_ref[1] + 0.0 * (double)(1 << level_ref));
  const Eigen::Vector3d dv = cam_ref.cam2world(px_ref[0] + 0.0 * (double)(1 << level_ref), px_ref[1] + step);
  Vec3 xyz_du_ref{du[0], du[1], du[2]}, xyz_dv_ref{dv[0], dv[1], dv[2]};
  xyz_du_ref = xyz_du_ref * (xyz_ref.z / xyz_du_ref.z);
  xyz_dv_ref = xyz_dv_ref * (xyz_ref.z / xyz_dv_ref.z);
  auto w2c = [&](Vec3 p, double px[2]) {
    const Eigen::Vector2d q = cam_cur.world2cam(Eigen::Vector3d(p.x, p.y, p.z));
    px[0] = q[0], px[1] = q[1];
  };
  double px_cur[2], px_du[2], px_dv[2];
  w2c(se3_act(T_cur_ref, xyz_ref), px_cur);
  w2c(se3_act(T_cur_ref, xyz_du_ref), px_du);
  w2c(se3_act(T_cur_ref, xyz_dv_ref), px_dv);
  A[0][0] = (px_du[0] - px_cur[0]) / halfpatch_size;
  A[1][0] = (px_du[1] - px_cur[1]) / halfpatch_size;
  A[0][1] = (px_dv[0] - px_cur[0]) / halfpatch_size;
  A[1][1] = (px_dv[1] - px_cur[1]) / halfpatch_size;
}

// The stand-in camera of a plsvo_match_camera; nullptr for an unknown model
std::unique_ptr<vk::AbstractCamera> make_camera(const plsvo_match_camera& m) {
  if (m.model == PLSVO_CAMERA_PINHOLE)
    return std::make_unique<vk::PinholeCamera>(m.pinhole.width, m.pinhole.height, m.pinhole.fx, m.pinhole.fy, m.pinhole.cx, m.pinhole.cy);
  if (m.model == PLSVO_CAMERA_ATAN)
    return std::make_unique<vk::ATANCamera>(m.atan.width, m.atan.height, m.atan.fx, m.atan.fy, m.atan.cx, m.atan.cy, m.atan.d0);
  return nullptr;
}

plsvo_camera size_of(const vk::AbstractCamera& k) { return plsvo_camera{k.width(), k.height(), 0, 0, 0.0, 0.0, 0.0, 0.0}; }

// findMatchDirect for candidate i with its ref image seen through cam_ref and its current image through cam_cur; the warp
// matrix from the two cameras, or, when A_in is given, read from A_in[4 i .. 4 i + 3] (row-major)
void match_direct_one_2cam(const vk::AbstractCamera& cam_ref, const vk::AbstractCamera& cam_cur, const double* A_in,
                           const plsvo_match_batch* in, const plsvo_match_result* out, int i) {
  const plsvo_camera ref_size = size_of(cam_ref), cur_size = size_of(cam_cur);
  const int halfpatch_size_ = 4;
  const size_t I = (size_t)i;
  const double* px_ref = in->ref_px + 2 * I;
  const int level_ref = in->ref_level[i];
  out->px_cur[2 * I] = in->px_cur[2 * I], out->px_cur[2 * I + 1] = in->px_cur[2 * I + 1];
  out->success[i] = 0;
  if (out->search_level) out->search_level[i] = -1;
  {  // :169-171
    const int ox = (int)px_ref[0] / (1 << level_ref), oy = (int)px_ref[1] / (1 << level_ref);
    if (!cam_is_in_frame(ref_size, ox, oy, halfpatch_size_ + 2, level_ref)) return;
  }
  double A[2][2];
  if (!A_in) {
    const SE3 T_ref_w = se3_from_pose7(in->T_ref_w + 7 * (size_t)in->ref_index[i]);
    const SE3 T_cur_w = se3_from_pose7(in->T_cur_w + 7 * (size_t)in->cur_index[i]);
    const SE3 T_w_ref = se3_inverse(T_ref_w);
    const SE3 T_cur_ref = se3_mul(T_cur_w, T_w_ref);
    const Vec3 pos{in->pos[3 * I], in->pos[3 * I + 1], in->pos[3 * I + 2]};
    const Vec3 f_ref{in->ref_f[3 * I], in->ref_f[3 * I + 1], in->ref_f[3 * I + 2]};
    const double depth_ref = norm(T_w_ref.t - pos);
    warp_matrix_affine_2cam(cam_ref, cam_cur, px_ref, f_ref, depth_ref, T_cur_ref, level_ref, A);
  } else {
    A[0][0] = A_in[4 * I], A[0][1] = A_in[4 * I + 1], A[1][0] = A_in[4 * I + 2], A[1][1] = A_in[4 * I + 3];
  }
  const int search_level = best_search_level(A, in->n_pyr_levels - 1);
  if (out->search_level) out->search_level[i] = search_level;
  if (out->A_cur_ref) out->A_cur_ref[4 * I] = A[0][0], out->A_cur_ref[4 * I + 1] = A[0][1], out->A_cur_ref[4 * I + 2] = A[1][0], out->A_cur_ref[4 * I + 3] = A[1][1];
  uint8_t patch_with_border[100] = {0};
  uint8_t patch[64];
  warp_affine_patches(A, in->ref_img[level_ref] + (size_t)in->ref_index[i] * in->ref_stride[level_ref], (int)in->ref_pitch[level_ref],
                      ref_size.width >> level_ref, ref_size.height >> level_ref, px_ref, level_ref, search_level, patch_with_border, patch);
  const double scale = (double)(1 << search_level);
  double px_scaled[2] = {in->px_cur[2 * I] / scale, in->px_cur[2 * I + 1] / scale};
  const uint8_t* cur = in->cur_img[search_level] + (size_t)in->cur_index[i] * in->cur_stride[search_level];
  const int ccols = cur_size.width >> search_level, crows = cur_size.height >> search_level;
  int ok;
  if (in->is_edgelet && in->is_edgelet[i]) {
    const double g0 = in->ref_grad[2 * I], g1 = in->ref_grad[2 * I + 1];
    double d0 = A[0][0] * g0 + A[0][1] * g1, d1 = A[1][0] * g0 + A[1][1] * g1;
    const double n = std::sqrt(d0 * d0 + d1 * d1);
    d0 /= n, d1 /= n;
    const float dir[2] = {(float)d0, (float)d1};
    double h_inv;
    ok = align1d_one(cur, ccols, crows, in->cur_pitch[search_level], dir, patch_with_border, patch, in->n_iter, px_scaled, &h_inv,
                     DirectStats{nullptr});
  } else {
    ok = align2d_one(cur, ccols, crows, in->cur_pitch[search_level], patch_with_border, patch, in->n_iter, px_scaled, DirectStats{nullptr});
  }
  out->px_cur[2 * I] = px_scaled[0] * scale, out->px_cur[2 * I + 1] = px_scaled[1] * scale;
  out->success[i] = (uint8_t)ok;
}

int run(const plsvo_match_camera* cams, int n_cams, const int32_t* cam_of_ref, const int32_t* cam_of_cur, const double* A,
        const plsvo_match_batch* in, const plsvo_match_result* out, int n_threads) {
  if (!cams || n_cams < 1 || !cam_of_ref || !cam_of_cur || !in || !out) return PLSVO_ERR_INVALID;
  std::vector<std::unique_ptr<vk::AbstractCamera>> k;
  for (int j = 0; j < n_cams; ++j) {
    k.push_back(make_camera(cams[j]));
    if (!k.back()) return PLSVO_ERR_INVALID;
  }
  for (int r = 0; r < in->n_ref_images; ++r)
    if (cam_of_ref[r] < 0 || cam_of_ref[r] >= n_cams) return PLSVO_ERR_INVALID;
  for (int c = 0; c < in->n_cur_images; ++c)
    if (cam_of_cur[c] < 0 || cam_of_cur[c] >= n_cams) return PLSVO_ERR_INVALID;
  parallel_for(in->n_features, n_threads, [&](int i) {
    match_direct_one_2cam(*k[cam_of_ref[in->ref_index[i]]], *k[cam_of_cur[in->cur_index[i]]], A, in, out, i);
  });
  return PLSVO_OK;
}

}  // namespace

extern "C" {

// Matcher::findMatchDirect with ref image r seen through cams[cam_of_ref[r]] and current image c through
// cams[cam_of_cur[c]] (plsvo_match_direct_multicam_batch_run's layout; in->cam is the slot and is not read).
int plsvo_oracle_match_direct_multicam_batch(const plsvo_match_camera* cams, int n_cams, const int32_t* cam_of_ref,
                                             const int32_t* cam_of_cur, const plsvo_match_batch* in, const plsvo_match_result* out,
                                             int n_threads) {
  return run(cams, n_cams, cam_of_ref, cam_of_cur, nullptr, in, out, n_threads);
}

// Everything of that call downstream of the warp matrix, with A_cur_ref given per candidate (A [n][4], row-major): the
// in-frame test at the ref camera's size, getBestSearchLevel, warpAffine at the ref camera's size, the edgelet direction
// and align2D / align1D at the current camera's size.  No camera model is read.
int plsvo_oracle_match_direct_multicam_given_A(const plsvo_match_camera* cams, int n_cams, const int32_t* cam_of_ref,
                                               const int32_t* cam_of_cur, const double* A, const plsvo_match_batch* in,
                                               const plsvo_match_result* out, int n_threads) {
  if (!A) return PLSVO_ERR_INVALID;
  return run(cams, n_cams, cam_of_ref, cam_of_cur, A, in, out, n_threads);
}

// The same call with each camera given by its members, as the device kernel receives them: members [n_cams][8] =
// (model, width, height, fx, fy, cx, cy, d0), fx..cy in pixels (an ATAN camera's fx_..cy_), so that no normalisation round
// trip W * (fx_ / W) can move a member by an ulp.  Every image index and camera index is trusted.
int plsvo_oracle_match_direct_multicam_members(const double* members, int n_cams, const int32_t* cam_of_ref, const int32_t* cam_of_cur,
                                               const plsvo_match_batch* in, const plsvo_match_result* out, int n_threads) {
  if (!members || n_cams < 1 || !cam_of_ref || !cam_of_cur || !in || !out) return PLSVO_ERR_INVALID;
  std::vector<std::unique_ptr<vk::AbstractCamera>> k;
  for (int j = 0; j < n_cams; ++j) {
    const double* m = members + 8 * (size_t)j;
    const int w = (int)m[1], h = (int)m[2];
    if (m[0] == PLSVO_CAMERA_PINHOLE) {
      k.push_back(std::make_unique<vk::PinholeCamera>(w, h, m[3], m[4], m[5], m[6]));
    } else if (m[0] == PLSVO_CAMERA_ATAN) {
      auto a = std::make_unique<vk::ATANCamera>(w, h, 1.0, 1.0, 0.5, 0.5, m[7]);
      a->fx_ = m[3], a->fy_ = m[4], a->cx_ = m[5], a->cy_ = m[6];
      k.push_back(std::move(a));
    } else {
      return PLSVO_ERR_INVALID;
    }
  }
  parallel_for(in->n_features, n_threads, [&](int i) {
    match_direct_one_2cam(*k[cam_of_ref[in->ref_index[i]]], *k[cam_of_cur[in->cur_index[i]]], nullptr, in, out, i);
  });
  return PLSVO_OK;
}

}  // extern "C"
