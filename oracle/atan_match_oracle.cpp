// atan_match_oracle.cpp — the CPU oracle's Matcher::findMatchDirect seen through vk::ATANCamera.
//
// TEST INFRASTRUCTURE, NOT THE PRODUCT (see the header of plsvo_oracle.cpp).  In Matcher::findMatchDirect
// (src/matcher.cpp:159-211) the camera is read in two places only: the in-frame test, which depends on the image size
// alone, and warp::getWarpMatrixAffine (:44-71), two cam_ref.cam2world and three cam_cur.world2cam calls.  Everything
// after A_cur_ref (search level, warpAffine, the 8x8 patch, the edgelet direction A*grad, align2D / align1D) does not
// read the camera.
//
// This translation unit includes plsvo_oracle.cpp unchanged.  It restates the warp matrix with the stand-in camera's own
// cam2world / world2cam (oracle/refdeps/vikit/atan_camera.h, the one statement of the model) and runs the included
// getBestSearchLevel, warpAffine, align2D and align1D restatements downstream of it.  A second entry point takes
// A_cur_ref as an input and runs the same downstream code: on the device atan / tan are not glibc's, so the GPU tests
// compare the kernel's search level and refined position with what this code computes from the kernel's own A_cur_ref.
//
// Build: oracle_atan_match.py (the flags of oracle/Makefile: strict IEEE, no FMA contraction).
#include "plsvo_oracle.cpp"

#include <vikit/atan_camera.h>

namespace {

// warp::getWarpMatrixAffine (src/matcher.cpp:44-71) with cam_ref = cam_cur = the stand-in ATANCamera, in the operation
// order of plsvo_oracle.cpp's pinhole warp_matrix_affine
void atan_warp_matrix_affine(const vk::ATANCamera& cam, const double* px_ref, Vec3 f_ref, double depth_ref, const SE3& T_cur_ref,
                             int level_ref, double A[2][2]) {
  const int halfpatch_size = 5;
  const Vec3 xyz_ref = f_ref * depth_ref;
  const double step = (double)halfpatch_size * (double)(1 << level_ref);
  const Eigen::Vector3d du = cam.cam2world(px_ref[0] + step, px_ref[1] + 0.0 * (double)(1 << level_ref));
  const Eigen::Vector3d dv = cam.cam2world(px_ref[0] + 0.0 * (double)(1 << level_ref), px_ref[1] + step);
  Vec3 xyz_du_ref{du[0], du[1], du[2]}, xyz_dv_ref{dv[0], dv[1], dv[2]};
  xyz_du_ref = xyz_du_ref * (xyz_ref.z / xyz_du_ref.z);
  xyz_dv_ref = xyz_dv_ref * (xyz_ref.z / xyz_dv_ref.z);
  auto w2c = [&](Vec3 p, double px[2]) {
    const Eigen::Vector2d q = cam.world2cam(Eigen::Vector3d(p.x, p.y, p.z));
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

// match_direct_one of plsvo_oracle.cpp with the warp matrix of candidate i from `cam`, or, when cam is null, read from
// A_in[4 i .. 4 i + 3] (row-major, as plsvo_match_result::A_cur_ref)
void atan_match_direct_one(const vk::ATANCamera* cam, const double* A_in, const plsvo_match_batch* in, const plsvo_match_result* out,
                           int i) {
  const plsvo_camera& size = in->cam;  // the in-frame test and the level sizes read the image size only
  const int halfpatch_size_ = 4;
  const size_t I = (size_t)i;
  const double* px_ref = in->ref_px + 2 * I;
  const int level_ref = in->ref_level[i];
  out->px_cur[2 * I] = in->px_cur[2 * I], out->px_cur[2 * I + 1] = in->px_cur[2 * I + 1];
  out->success[i] = 0;
  if (out->search_level) out->search_level[i] = -1;
  {  // :169-171
    const int ox = (int)px_ref[0] / (1 << level_ref), oy = (int)px_ref[1] / (1 << level_ref);
    if (!cam_is_in_frame(size, ox, oy, halfpatch_size_ + 2, level_ref)) return;
  }
  double A[2][2];
  if (cam) {
    const SE3 T_ref_w = se3_from_pose7(in->T_ref_w + 7 * (size_t)in->ref_index[i]);
    const SE3 T_cur_w = se3_from_pose7(in->T_cur_w + 7 * (size_t)in->cur_index[i]);
    const SE3 T_w_ref = se3_inverse(T_ref_w);
    const SE3 T_cur_ref = se3_mul(T_cur_w, T_w_ref);
    const Vec3 pos{in->pos[3 * I], in->pos[3 * I + 1], in->pos[3 * I + 2]};
    const Vec3 f_ref{in->ref_f[3 * I], in->ref_f[3 * I + 1], in->ref_f[3 * I + 2]};
    const double depth_ref = norm(T_w_ref.t - pos);
    atan_warp_matrix_affine(*cam, px_ref, f_ref, depth_ref, T_cur_ref, level_ref, A);
  } else {
    A[0][0] = A_in[4 * I], A[0][1] = A_in[4 * I + 1], A[1][0] = A_in[4 * I + 2], A[1][1] = A_in[4 * I + 3];
  }
  const int search_level = best_search_level(A, in->n_pyr_levels - 1);
  if (out->search_level) out->search_level[i] = search_level;
  if (out->A_cur_ref) out->A_cur_ref[4 * I] = A[0][0], out->A_cur_ref[4 * I + 1] = A[0][1], out->A_cur_ref[4 * I + 2] = A[1][0], out->A_cur_ref[4 * I + 3] = A[1][1];
  uint8_t patch_with_border[100] = {0};
  uint8_t patch[64];
  warp_affine_patches(A, in->ref_img[level_ref] + (size_t)in->ref_index[i] * in->ref_stride[level_ref], (int)in->ref_pitch[level_ref],
                      size.width >> level_ref, size.height >> level_ref, px_ref, level_ref, search_level, patch_with_border, patch);
  const double scale = (double)(1 << search_level);
  double px_scaled[2] = {in->px_cur[2 * I] / scale, in->px_cur[2 * I + 1] / scale};
  const uint8_t* cur = in->cur_img[search_level] + (size_t)in->cur_index[i] * in->cur_stride[search_level];
  const int ccols = size.width >> search_level, crows = size.height >> search_level;
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

}  // namespace

extern "C" {

// Matcher::findMatchDirect for a batch of candidates whose keyframes and current frames are seen through one
// vk::ATANCamera(*cam).  in->cam supplies the image size only and must equal the camera's.
int plsvo_oracle_atan_match_direct_batch(const plsvo_atan_camera* cam, const plsvo_match_batch* in, const plsvo_match_result* out,
                                         int n_threads) {
  if (!cam || !in || !out) return PLSVO_ERR_INVALID;
  if (cam->width != in->cam.width || cam->height != in->cam.height) return PLSVO_ERR_INVALID;
  const vk::ATANCamera c(cam->width, cam->height, cam->fx, cam->fy, cam->cx, cam->cy, cam->d0);
  parallel_for(in->n_features, n_threads, [&](int i) { atan_match_direct_one(&c, nullptr, in, out, i); });
  return PLSVO_OK;
}

// The same, with the camera given by its members fx_, fy_, cx_, cy_ (pixels) and d0, as the device kernel receives it
// (MatchArgs), so that no normalisation round trip W * (fx_ / W) can move a member by an ulp.  in->cam supplies the size.
int plsvo_oracle_atan_match_direct_members(double fx_, double fy_, double cx_, double cy_, double d0, const plsvo_match_batch* in,
                                           const plsvo_match_result* out, int n_threads) {
  if (!in || !out) return PLSVO_ERR_INVALID;
  vk::ATANCamera c(in->cam.width, in->cam.height, 1.0, 1.0, 0.5, 0.5, d0);
  c.fx_ = fx_, c.fy_ = fy_, c.cx_ = cx_, c.cy_ = cy_;
  parallel_for(in->n_features, n_threads, [&](int i) { atan_match_direct_one(&c, nullptr, in, out, i); });
  return PLSVO_OK;
}

// Everything of findMatchDirect downstream of the warp matrix, with A_cur_ref given per candidate (A [n][4], row-major):
// the in-frame test, getBestSearchLevel, warpAffine, the edgelet direction and align2D / align1D.  No camera is read.
int plsvo_oracle_match_direct_given_A(const double* A, const plsvo_match_batch* in, const plsvo_match_result* out, int n_threads) {
  if (!A || !in || !out) return PLSVO_ERR_INVALID;
  parallel_for(in->n_features, n_threads, [&](int i) { atan_match_direct_one(nullptr, A, in, out, i); });
  return PLSVO_OK;
}

}  // extern "C"
