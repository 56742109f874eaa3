// plsvo_oracle.cpp — CPU restatement of PL-SVO's per-frame optimisation path.
//
// THIS IS TEST INFRASTRUCTURE, NOT THE PRODUCT.  Only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs may load this library; the product
// (pl-svo_b200/csrc) never links, loads or calls it.
//
// PARITY PINNED AGAINST THE REFERENCE RUN HERE.  The reference (rubengooj/pl-svo @ 5d4ca39) ships no
// tests, golden vectors or fixtures for this path, and its own build cannot run in this image (cmake +
// Eigen, Sophus, OpenCV C++, boost, rpg_vikit are absent; no network).  Its three translation units on the
// path — src/sparse_img_align.cpp, src/pose_optimizer.cpp, src/feature.cpp — are however compiled
// UNMODIFIED, where they lie under /root/reference, against the reference's own headers and small
// stand-in headers for the absent third-party libraries (oracle/refdeps/, oracle/ref_harness.cpp,
// `make -C oracle ref` -> oracle/_ref/libplsvo_ref.so).  tests/test_reference_tu_cpu.py requires this
// file to reproduce that library BIT FOR BIT (poses, H, n_tracked, killed segments, iteration counts,
// status; pose, covariance, scale, errors, counts, outlier flags) over the domain's edge cases, and
// tests/golden/*.npz are outputs of that library (tests/golden/make_golden.py).
// What remains a restatement on BOTH sides is the un-vendored third-party arithmetic the path calls
// (uzh-rpg/rpg_vikit vikit_common: NLLSSolver<6,SE3>, robust_cost, math_utils, PinholeCamera;
// strasdat/Sophus non-templated SE3/SO3; Eigen LDLT / inverse / quaternion), written from their
// published sources; the reference pins no version of them (CMakeLists.txt:40-41,57; SURVEY.md §8c).
// Those pieces are additionally checked against closed forms, an independent NumPy restatement
// (oracle/np_oracle.py) and analytic properties (tests/test_oracle_cpu.py).
// This file is a line-by-line restatement: each function cites the reference file:line it follows.
//
// Arithmetic follows the source text as strict IEEE-754 without FMA contraction (build with
// -ffp-contract=off): float where the reference uses float, double where it uses double.
//
// Build: see oracle/Makefile  (g++ -O3 -march=x86-64-v3 -ffp-contract=off -shared -fPIC).

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <thread>
#include <vector>

#include "../include/plsvo_b200.h"

namespace {

// ------------------------------------------------------------------------------------------------
// Sophus (old, non-templated) SO3/SE3 — restated from strasdat/Sophus sophus/so3.cpp, se3.cpp.
// Rotation is a unit quaternion (Eigen::Quaterniond), every product re-normalises.
// ------------------------------------------------------------------------------------------------
constexpr double kSmallEps = 1e-10;  // Sophus SMALL_EPS

struct Quat {
  double x, y, z, w;
};
struct Vec3 {
  double x, y, z;
};
inline Vec3 operator+(Vec3 a, Vec3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
inline Vec3 operator-(Vec3 a, Vec3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline Vec3 operator*(Vec3 a, double s) { return {a.x * s, a.y * s, a.z * s}; }
inline Vec3 cross(Vec3 a, Vec3 b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
inline double norm(Vec3 a) { return std::sqrt(a.x * a.x + a.y * a.y + a.z * a.z); }

inline Quat qnormalized(Quat q) {  // Eigen: coeffs() /= coeffs().norm()
  const double n = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  return {q.x / n, q.y / n, q.z / n, q.w / n};
}
inline Quat qmul(Quat a, Quat b) {  // Eigen quaternion product
  return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
          a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
          a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x,
          a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
inline Vec3 qrot(Quat q, Vec3 v) {  // Eigen QuaternionBase::_transformVector
  const Vec3 qv{q.x, q.y, q.z};
  Vec3 uv = cross(qv, v);
  uv = uv + uv;
  return v + uv * q.w + cross(qv, uv);
}

inline void quat_to_matrix(Quat q, double R[3][3]) {  // Eigen QuaternionBase::toRotationMatrix
  const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0][0] = 1 - (tyy + tzz), R[0][1] = txy - twz, R[0][2] = txz + twy;
  R[1][0] = txy + twz, R[1][1] = 1 - (txx + tzz), R[1][2] = tyz - twx;
  R[2][0] = txz - twy, R[2][1] = tyz + twx, R[2][2] = 1 - (txx + tyy);
}

struct SE3 {
  Quat q{0, 0, 0, 1};
  Vec3 t{0, 0, 0};
};
inline SE3 se3_from_pose7(const double* p) {
  SE3 T;
  T.q = qnormalized(Quat{p[0], p[1], p[2], p[3]});  // SO3(const Quaterniond&) normalises
  T.t = {p[4], p[5], p[6]};
  return T;
}
inline void se3_to_pose7(const SE3& T, double* p) {
  p[0] = T.q.x, p[1] = T.q.y, p[2] = T.q.z, p[3] = T.q.w;
  p[4] = T.t.x, p[5] = T.t.y, p[6] = T.t.z;
}
inline SE3 se3_mul(const SE3& a, const SE3& b) {  // SE3::operator*=
  SE3 r;
  r.t = a.t + qrot(a.q, b.t);
  r.q = qnormalized(qmul(a.q, b.q));
  return r;
}
inline SE3 se3_inverse(const SE3& a) {  // SE3::inverse
  SE3 r;
  r.q = qnormalized(Quat{-a.q.x, -a.q.y, -a.q.z, a.q.w});
  r.t = qrot(r.q, a.t * -1.0);
  return r;
}
inline Vec3 se3_act(const SE3& T, Vec3 p) { return qrot(T.q, p) + T.t; }

// SE3::exp( [upsilon, omega] ), SO3::expAndTheta
inline SE3 se3_exp(const double u[6]) {
  const Vec3 upsilon{u[0], u[1], u[2]};
  const Vec3 omega{u[3], u[4], u[5]};
  const double theta = norm(omega);
  const double half_theta = 0.5 * theta;
  double imag_factor;
  const double real_factor = std::cos(half_theta);
  if (theta < kSmallEps) {
    const double theta_sq = theta * theta;
    const double theta_po4 = theta_sq * theta_sq;
    imag_factor = 0.5 - 0.0208333 * theta_sq + 0.000260417 * theta_po4;
  } else {
    imag_factor = std::sin(half_theta) / theta;
  }
  SE3 r;
  r.q = qnormalized(Quat{imag_factor * omega.x, imag_factor * omega.y, imag_factor * omega.z, real_factor});
  // V = I + (1-cos)/theta^2 * Omega + (theta - sin)/theta^3 * Omega^2 ;  t = V * upsilon, formed as 3x3
  // matrices coefficient by coefficient exactly as Sophus writes it (se3.cpp, SE3::exp).
  const double Om[3][3] = {{0, -omega.z, omega.y}, {omega.z, 0, -omega.x}, {-omega.y, omega.x, 0}};
  double Om2[3][3], V[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) Om2[i][j] = (Om[i][0] * Om[0][j] + Om[i][1] * Om[1][j]) + Om[i][2] * Om[2][j];
  if (theta < kSmallEps) {
    quat_to_matrix(r.q, V);  // V = so3.matrix()
  } else {
    const double theta_sq = theta * theta;
    const double a = (1 - std::cos(theta)) / theta_sq;
    const double b = (theta - std::sin(theta)) / (theta_sq * theta);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) V[i][j] = ((i == j ? 1.0 : 0.0) + a * Om[i][j]) + b * Om2[i][j];
  }
  const double u3[3] = {upsilon.x, upsilon.y, upsilon.z};
  double t3[3];
  for (int i = 0; i < 3; ++i) t3[i] = (V[i][0] * u3[0] + V[i][1] * u3[1]) + V[i][2] * u3[2];
  r.t = {t3[0], t3[1], t3[2]};
  return r;
}

// ------------------------------------------------------------------------------------------------
// Eigen fixed-size 6x6 helpers — LDLT with diagonal pivoting (Eigen/src/Cholesky/LDLT.h,
// ldlt_inplace<Lower>::unblocked + _solve_impl) and inverse via partial-pivot LU.
// ------------------------------------------------------------------------------------------------
struct Ldlt6 {
  double m[6][6];  // lower: L (unit diag implied) + D on the diagonal
  int tr[6];       // transpositions
};
inline void ldlt6_compute(const double A[36], Ldlt6& f) {
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) f.m[i][j] = A[i * 6 + j];
  for (int k = 0; k < 6; ++k) {
    int piv = k;
    double big = std::fabs(f.m[k][k]);
    for (int i = k + 1; i < 6; ++i)
      if (std::fabs(f.m[i][i]) > big) big = std::fabs(f.m[i][i]), piv = i;
    f.tr[k] = piv;
    if (piv != k) {
      // symmetric swap of rows/cols k and piv restricted to the lower triangle
      for (int j = 0; j < k; ++j) std::swap(f.m[k][j], f.m[piv][j]);
      for (int i = piv + 1; i < 6; ++i) std::swap(f.m[i][k], f.m[i][piv]);
      std::swap(f.m[k][k], f.m[piv][piv]);
      for (int i = k + 1; i < piv; ++i) std::swap(f.m[i][k], f.m[piv][i]);
    }
    if (k > 0) {
      double temp[6];
      for (int j = 0; j < k; ++j) temp[j] = f.m[j][j] * f.m[k][j];
      double s = 0;
      for (int j = 0; j < k; ++j) s += f.m[k][j] * temp[j];
      f.m[k][k] -= s;
      for (int i = k + 1; i < 6; ++i) {
        double s2 = 0;
        for (int j = 0; j < k; ++j) s2 += f.m[i][j] * temp[j];
        f.m[i][k] -= s2;
      }
    }
    const double akk = f.m[k][k];
    const bool pivot_is_valid = std::fabs(akk) > 0.0;
    if (k == 0 && !pivot_is_valid) {
      for (int j = 0; j < 6; ++j) f.tr[j] = j;
      return;
    }
    if (pivot_is_valid)
      for (int i = k + 1; i < 6; ++i) f.m[i][k] /= akk;
  }
}
inline void ldlt6_solve(const Ldlt6& f, const double b[6], double x[6]) {
  for (int i = 0; i < 6; ++i) x[i] = b[i];
  for (int k = 0; k < 6; ++k) std::swap(x[k], x[f.tr[k]]);  // P b
  for (int i = 0; i < 6; ++i)                               // L^-1
    for (int j = 0; j < i; ++j) x[i] -= f.m[i][j] * x[j];
  const double tol = 1.0 / std::numeric_limits<double>::max();  // Eigen >= 3.3 pseudo-inverse of D
  for (int i = 0; i < 6; ++i) {
    if (std::fabs(f.m[i][i]) > tol)
      x[i] /= f.m[i][i];
    else
      x[i] = 0.0;
  }
  for (int i = 5; i >= 0; --i)  // L^-T
    for (int j = i + 1; j < 6; ++j) x[i] -= f.m[j][i] * x[j];
  for (int k = 5; k >= 0; --k) std::swap(x[k], x[f.tr[k]]);  // P^T
}
inline void solve6(const double A[36], const double b[6], double x[6]) {
  Ldlt6 f;
  ldlt6_compute(A, f);
  ldlt6_solve(f, b, x);
}
// Matrix6d::inverse(): Eigen uses PartialPivLU for fixed sizes > 4.
inline void inverse6(const double A[36], double out[36]) {
  double lu[6][6];
  int perm[6];
  for (int i = 0; i < 6; ++i) {
    perm[i] = i;
    for (int j = 0; j < 6; ++j) lu[i][j] = A[i * 6 + j];
  }
  for (int k = 0; k < 6; ++k) {
    int piv = k;
    double big = std::fabs(lu[k][k]);
    for (int i = k + 1; i < 6; ++i)
      if (std::fabs(lu[i][k]) > big) big = std::fabs(lu[i][k]), piv = i;
    if (piv != k) {
      for (int j = 0; j < 6; ++j) std::swap(lu[k][j], lu[piv][j]);
      std::swap(perm[k], perm[piv]);
    }
    for (int i = k + 1; i < 6; ++i) {
      lu[i][k] /= lu[k][k];
      for (int j = k + 1; j < 6; ++j) lu[i][j] -= lu[i][k] * lu[k][j];
    }
  }
  for (int c = 0; c < 6; ++c) {
    double y[6];
    for (int i = 0; i < 6; ++i) {
      y[i] = (perm[i] == c) ? 1.0 : 0.0;
      for (int j = 0; j < i; ++j) y[i] -= lu[i][j] * y[j];
    }
    for (int i = 5; i >= 0; --i) {
      for (int j = i + 1; j < 6; ++j) y[i] -= lu[i][j] * y[j];
      y[i] /= lu[i][i];
    }
    for (int i = 0; i < 6; ++i) out[i * 6 + c] = y[i];
  }
}

// ------------------------------------------------------------------------------------------------
// vikit_common pieces (math_utils.h, robust_cost.cpp)
// ------------------------------------------------------------------------------------------------
template <class T>
inline T get_median(std::vector<T>& v) {  // vk::getMedian: nth_element at floor(n/2)
  auto it = v.begin() + v.size() / 2;
  std::nth_element(v.begin(), it, v.end());
  return *it;
}
inline float mad_scale(std::vector<float>& errors) {  // MADScaleEstimator::compute, NORMALIZER=1.48f
  return 1.48f * get_median(errors);
}
inline float tukey_value(const float& x) {  // TukeyWeightFunction::value, b = 4.6851f
  const float b = 4.6851f;
  const float b_square = b * b;
  const float x_square = x * x;
  if (x_square <= b_square) {
    const float tmp = 1.0f - x_square / b_square;
    return tmp * tmp;
  }
  return 0.0f;
}
inline double norm_max6(const double x[6]) {  // vk::norm_max
  double m = 0;
  for (int i = 0; i < 6; ++i) m = std::max(m, std::fabs(x[i]));
  return m;
}

// Frame::jacobian_xyz2uv — include/plsvo/frame.h:138-160
inline void jacobian_xyz2uv(Vec3 p, double J[2][6]) {
  const double x = p.x, y = p.y;
  const double z_inv = 1. / p.z;
  const double z_inv_2 = z_inv * z_inv;
  J[0][0] = -z_inv;
  J[0][1] = 0.0;
  J[0][2] = x * z_inv_2;
  J[0][3] = y * J[0][2];
  J[0][4] = -(1.0 + x * J[0][2]);
  J[0][5] = y * z_inv;
  J[1][0] = 0.0;
  J[1][1] = -z_inv;
  J[1][2] = y * z_inv_2;
  J[1][3] = 1.0 + y * J[1][2];
  J[1][4] = -J[0][3];
  J[1][5] = -x * z_inv;
}

// ------------------------------------------------------------------------------------------------
// Patch — src/feature.cpp:175-218, include/plsvo/feature.h:107-147
// ------------------------------------------------------------------------------------------------
struct Image {
  const uint8_t* data;
  int cols, rows;
  int stride;
};
struct Patch {
  static constexpr int size = 4, halfsize = 2, area = 16;
  Image img;
  float u_ref, v_ref;
  int u_ref_i, v_ref_i;
  float wTL, wTR, wBL, wBR;
  const uint8_t* roi;  // top-left pixel of the 4x4 ROI
  explicit Patch(const Image& im) : img(im) {}
  void setPosition(double px0, double px1) {  // feature.cpp:189-197
    u_ref = (float)px0;
    v_ref = (float)px1;
    u_ref_i = (int)floorf(u_ref);
    v_ref_i = (int)floorf(v_ref);
  }
  void computeInterpWeights() {  // feature.cpp:199-208
    const float subpix_u_ref = u_ref - u_ref_i;
    const float subpix_v_ref = v_ref - v_ref_i;
    wTL = (float)((1.0 - subpix_u_ref) * (1.0 - subpix_v_ref));
    wTR = (float)(subpix_u_ref * (1.0 - subpix_v_ref));
    wBL = (float)((1.0 - subpix_u_ref) * subpix_v_ref);
    wBR = subpix_u_ref * subpix_v_ref;  // float*float in the source
  }
  void setRoi() {  // feature.cpp:210-218
    roi = img.data + (size_t)(v_ref_i - halfsize) * img.stride + (u_ref_i - halfsize);
  }
  bool isInFrame(int boundary) const {  // feature.h:139-144
    return !(u_ref_i < boundary || v_ref_i < boundary || u_ref_i >= img.cols - boundary ||
             v_ref_i >= img.rows - boundary);
  }
};

// vk::AbstractCamera::isInFrame(obs, boundary, level)
inline bool cam_is_in_frame(const plsvo_camera& cam, int ox, int oy, int boundary, int level) {
  return ox >= boundary && ox < cam.width / (1 << level) - boundary && oy >= boundary &&
         oy < cam.height / (1 << level) - boundary;
}

// LineFeat::setupSampling — src/feature.cpp:160-173
inline size_t setup_sampling(size_t patch_size, const double spx[2], const double epx[2], double length,
                             double dif[2]) {
  dif[0] = epx[0] - spx[0];
  dif[1] = epx[1] - spx[1];
  const double tan_dir = std::min(std::fabs(dif[0]), std::fabs(dif[1])) / std::max(std::fabs(dif[0]), std::fabs(dif[1]));
  const double sin_dir = tan_dir / std::sqrt(1.0 + tan_dir * tan_dir);
  const double correction = 2.0 * std::sqrt(1.0 + sin_dir * sin_dir);
  return (size_t)std::max(1.0, length / (2.0 * patch_size * correction));
}

// ------------------------------------------------------------------------------------------------
// SparseImgAlign (src/sparse_img_align.cpp) on top of vk::NLLSSolver<6,SE3>
// ------------------------------------------------------------------------------------------------
constexpr int kTraceStride = 64;  // doubles per trace record
// record: [0]=level [1]=iter [2]=new_chi2 [3]=n_meas [4]=accepted [5..40]=H [41..46]=Jres [47..52]=x [53..59]=T(model after)

struct AlignOptions {
  bool chi2_double = false;  // experiment switch: accumulate chi2 in double (NOT the reference behaviour)
  // experiment switch (NOT the reference behaviour): form the point-patch normal equations the way the CUDA
  // kernel does — five in-patch sums (1 = fp32 FMA chain, 2 = double) followed by a rank-2 update with the two
  // projection-Jacobian rows — while chi2 keeps the reference's sequential float order.  Used by
  // tools/emulate_kernel_sums.py to measure how often the accept/rollback decision can flip for that reason alone.
  int h_mode = 0;
};

struct SparseImgAlign {
  // inputs of one pair
  const plsvo_align_batch* B;
  int b;
  int n_pts, n_segs;
  const double *pt_px, *pt_f, *pt_pos;
  const uint8_t* pt_valid;
  const double *seg_spx, *seg_epx, *seg_sf, *seg_ef, *seg_spos, *seg_epos, *seg_length;
  std::vector<uint8_t> seg_alive;  // feat3D != NULL (mutated: sparse_img_align.cpp:687-688)
  AlignOptions opt;

  // solver state (vk::NLLSSolver members)
  int n_iter_, n_iter_init_;
  double eps_;
  bool stop_ = false, use_weights_ = false;
  double chi2_ = 1e10;
  size_t n_meas_ = 0;
  int iter_ = 0;
  double H_[36], Jres_[6], x_[6];
  int max_level_, min_level_, level_ = 0;
  bool have_ref_patch_cache_ = false;
  Vec3 ref_pos;

  struct Cache {
    std::vector<float> ref_patch;
    std::vector<double> jacobian;  // 6 x (N*16), column major
    std::vector<uint8_t> visible;
    std::vector<float> gdx, gdy;  // experiment (h_mode): float gradients per pixel
    std::vector<double> xyz;      // experiment (h_mode): X, Y, 1/Z per patch
  } pt_cache_, seg_cache_;
  std::vector<size_t> patch_offset;

  // accounting + trace
  int iters_at_level[PLSVO_MAX_LEVELS] = {0};
  uint32_t patch_iters = 0, patch_levels = 0;
  double* trace = nullptr;
  int trace_cap = 0, trace_n = 0;

  Image level_image(const uint8_t* const* imgs, int level) const {
    Image im;
    im.data = imgs[level] + (size_t)b * B->img_stride[level];
    im.cols = B->cam.width >> level;
    im.rows = B->cam.height >> level;
    im.stride = (int)B->img_pitch[level];
    return im;
  }
  Vec3 world2cam_px(Vec3 p) const {  // vk::PinholeCamera::world2cam(xyz) without distortion
    const double u = p.x / p.z, v = p.y / p.z;
    return {B->cam.fx * u + B->cam.cx, B->cam.fy * v + B->cam.cy, 0};
  }

  // sparse_img_align.cpp:195-268
  void precomputePoints() {
    Patch patch(level_image(B->ref_img, level_));
    const float scale = 1.0f / (1 << level_);
    const double focal_length = std::fabs(B->cam.fx);  // errorMultiplier2()
    for (int i = 0; i < n_pts; ++i) {
      if (pt_valid && !pt_valid[i]) continue;
      patch.setPosition(pt_px[2 * i] * scale, pt_px[2 * i + 1] * scale);
      if (!patch.isInFrame(patch.halfsize + 1)) continue;
      patch.computeInterpWeights();
      patch.setRoi();
      pt_cache_.visible[i] = 1;
      ++patch_levels;
      const Vec3 pos{pt_pos[3 * i], pt_pos[3 * i + 1], pt_pos[3 * i + 2]};
      const double depth = norm(pos - ref_pos);
      const Vec3 xyz_ref = Vec3{pt_f[3 * i], pt_f[3 * i + 1], pt_f[3 * i + 2]} * depth;
      double frame_jac[2][6];
      jacobian_xyz2uv(xyz_ref, frame_jac);
      if (opt.h_mode) {
        pt_cache_.gdx.resize((size_t)n_pts * 16), pt_cache_.gdy.resize((size_t)n_pts * 16), pt_cache_.xyz.resize((size_t)n_pts * 3);
        pt_cache_.xyz[3 * i] = xyz_ref.x, pt_cache_.xyz[3 * i + 1] = xyz_ref.y, pt_cache_.xyz[3 * i + 2] = 1. / xyz_ref.z;
      }
      fill_patch(patch, &pt_cache_.ref_patch[(size_t)16 * i], &pt_cache_.jacobian[(size_t)6 * 16 * i], frame_jac,
                 focal_length, opt.h_mode ? &pt_cache_.gdx[(size_t)16 * i] : nullptr,
                 opt.h_mode ? &pt_cache_.gdy[(size_t)16 * i] : nullptr);
    }
  }
  // the 16-pixel body shared by :243-264 and :354-375
  void fill_patch(const Patch& patch, float* cache_ptr, double* jac_cols, const double frame_jac[2][6],
                  double focal_length, float* gdx = nullptr, float* gdy = nullptr) const {
    const int stride = patch.img.stride;
    const double jscale = focal_length / (1 << level_);
    for (int y = 0; y < 4; ++y) {
      const uint8_t* img_ptr = patch.roi + (size_t)y * stride;
      for (int x = 0; x < 4; ++x, ++img_ptr, ++cache_ptr, jac_cols += 6) {
        *cache_ptr = patch.wTL * img_ptr[0] + patch.wTR * img_ptr[1] + patch.wBL * img_ptr[stride] +
                     patch.wBR * img_ptr[stride + 1];
        float dx = 0.5f * ((patch.wTL * img_ptr[1] + patch.wTR * img_ptr[2] + patch.wBL * img_ptr[stride + 1] +
                            patch.wBR * img_ptr[stride + 2]) -
                           (patch.wTL * img_ptr[-1] + patch.wTR * img_ptr[0] + patch.wBL * img_ptr[stride - 1] +
                            patch.wBR * img_ptr[stride]));
        float dy = 0.5f * ((patch.wTL * img_ptr[stride] + patch.wTR * img_ptr[1 + stride] +
                            patch.wBL * img_ptr[stride * 2] + patch.wBR * img_ptr[stride * 2 + 1]) -
                           (patch.wTL * img_ptr[-stride] + patch.wTR * img_ptr[1 - stride] + patch.wBL * img_ptr[0] +
                            patch.wBR * img_ptr[1]));
        for (int k = 0; k < 6; ++k) jac_cols[k] = (dx * frame_jac[0][k] + dy * frame_jac[1][k]) * jscale;
        if (gdx) *gdx++ = dx, *gdy++ = dy;
      }
    }
  }

  // sparse_img_align.cpp:270-378
  void precomputeSegments() {
    Patch patch(level_image(B->ref_img, level_));
    const float scale = 1.0f / (1 << level_);
    const double focal_length = std::fabs(B->cam.fx);
    patch_offset.assign(n_segs, 0);
    size_t cache_idx = 0;
    for (int j = 0; j < n_segs; ++j) {
      patch_offset[j] = cache_idx;
      if (!seg_alive[j]) continue;
      const double* spx = seg_spx + 2 * j;
      const double* epx = seg_epx + 2 * j;
      if (!cam_is_in_frame(B->cam, (int)(spx[0] * scale), (int)(spx[1] * scale), patch.halfsize + 1, level_) ||
          !cam_is_in_frame(B->cam, (int)(epx[0] * scale), (int)(epx[1] * scale), patch.halfsize + 1, level_))
        continue;
      seg_cache_.visible[j] = 1;
      double inc2d[2];
      size_t N_samples = setup_sampling(patch.size, spx, epx, seg_length[j], inc2d);
      N_samples = 1 + (N_samples - 1) / (1 << level_);
      inc2d[0] = inc2d[0] * scale / (N_samples - 1);
      inc2d[1] = inc2d[1] * scale / (N_samples - 1);
      double px_ref[2] = {spx[0] * scale, spx[1] * scale};
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
      ensure_seg_capacity(cache_idx / 16 + N_samples);
      for (unsigned sample = 0; sample < N_samples;
           ++sample, px_ref[0] += inc2d[0], px_ref[1] += inc2d[1], xyz_ref = xyz_ref + inc3d) {
        patch.setPosition(px_ref[0], px_ref[1]);
        patch.computeInterpWeights();
        patch.setRoi();
        double frame_jac[2][6];
        jacobian_xyz2uv(xyz_ref, frame_jac);
        fill_patch(patch, &seg_cache_.ref_patch[cache_idx], &seg_cache_.jacobian[6 * cache_idx], frame_jac,
                   focal_length);
        cache_idx += 16;
        ++patch_levels;
      }
    }
  }
  void ensure_seg_capacity(size_t n_patches) {
    // The reference sizes the cache as ceil(total_length/4) patches (sparse_img_align.cpp:69-78)
    // and never checks it; we grow instead of overflowing.
    if (seg_cache_.ref_patch.size() < n_patches * 16) {
      seg_cache_.ref_patch.resize(n_patches * 16, 0.f);
      seg_cache_.jacobian.resize(n_patches * 16 * 6, 0.0);
    }
  }

  // sparse_img_align.cpp:380-502  (linearize_system=true, compute_weight_scale=false, use_weights_=true)
  void computePoints(const SE3& T_cur_from_ref, double H[36], double Jres[6], float& chi2, double& chi2d) {
    Patch patch(level_image(B->cur_img, level_));
    const float scale = 1.0f / (1 << level_);
    chi2 = 0.0f;
    chi2d = 0.0;
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
      if (opt.h_mode) {  // experiment: kernel-style normal equations, reference-order chi2
        float Sf[5] = {0, 0, 0, 0, 0};
        double Sd[5] = {0, 0, 0, 0, 0};
        const float* gx = &pt_cache_.gdx[(size_t)16 * i];
        const float* gy = &pt_cache_.gdy[(size_t)16 * i];
        for (int y = 0; y < 4; ++y) {
          const uint8_t* img_ptr = patch.roi + (size_t)y * stride;
          for (int x = 0; x < 4; ++x, ++img_ptr, ++cache_ptr, ++gx, ++gy) {
            const float intensity_cur = patch.wTL * img_ptr[0] + patch.wTR * img_ptr[1] + patch.wBL * img_ptr[stride] +
                                        patch.wBR * img_ptr[stride + 1];
            const float res = intensity_cur - (*cache_ptr);
            const float weight = 1.0 / (1.0 + fabsf(res));
            chi2 += res * res * weight;
            chi2d += (double)(res * res * weight);
            n_meas_++;
            const float wdx = weight * *gx, wdy = weight * *gy;
            Sf[0] = fmaf(wdx, *gx, Sf[0]), Sf[1] = fmaf(wdx, *gy, Sf[1]), Sf[2] = fmaf(wdy, *gy, Sf[2]);
            Sf[3] = fmaf(wdx, res, Sf[3]), Sf[4] = fmaf(wdy, res, Sf[4]);
            const double dwdx = (double)weight * (double)*gx, dwdy = (double)weight * (double)*gy;
            Sd[0] += dwdx * (double)*gx, Sd[1] += dwdx * (double)*gy, Sd[2] += dwdy * (double)*gy;
            Sd[3] += dwdx * (double)res, Sd[4] += dwdy * (double)res;
          }
        }
        const double cJ = std::fabs(B->cam.fx) / (1 << level_), cJ2 = cJ * cJ;
        double S[5];
        for (int k = 0; k < 5; ++k) S[k] = (opt.h_mode == 1) ? (double)Sf[k] : Sd[k];
        double fj[2][6];
        const double X = pt_cache_.xyz[3 * i], Y = pt_cache_.xyz[3 * i + 1], zi = pt_cache_.xyz[3 * i + 2];
        jacobian_xyz2uv(Vec3{X, Y, 1.0 / zi}, fj);
        const double Sxx = S[0] * cJ2, Sxy = S[1] * cJ2, Syy = S[2] * cJ2, Sxr = S[3] * cJ, Syr = S[4] * cJ;
        for (int r = 0; r < 6; ++r) {
          const double pr = Sxx * fj[0][r] + Sxy * fj[1][r], qr = Sxy * fj[0][r] + Syy * fj[1][r];
          for (int c = 0; c < 6; ++c) H[r * 6 + c] += pr * fj[0][c] + qr * fj[1][c];
          Jres[r] -= Sxr * fj[0][r] + Syr * fj[1][r];
        }
        continue;
      }
      for (int y = 0; y < 4; ++y) {
        const uint8_t* img_ptr = patch.roi + (size_t)y * stride;
        for (int x = 0; x < 4; ++x, ++img_ptr, ++cache_ptr, Jc += 6) {
          const float intensity_cur = patch.wTL * img_ptr[0] + patch.wTR * img_ptr[1] + patch.wBL * img_ptr[stride] +
                                      patch.wBR * img_ptr[stride + 1];
          const float res = intensity_cur - (*cache_ptr);
          float weight = 1.0;
          weight = 1.0 / (1.0 + fabsf(res));  // :479
          chi2 += res * res * weight;         // :484
          chi2d += (double)(res * res * weight);
          n_meas_++;
          for (int r = 0; r < 6; ++r) {
            for (int c = 0; c < 6; ++c) H[r * 6 + c] += Jc[r] * Jc[c] * weight;  // :491
            Jres[r] -= Jc[r] * res * weight;                                       // :492
          }
        }
      }
    }
  }

  // sparse_img_align.cpp:504-695
  void computeSegments(const SE3& T_cur_from_ref, double H[36], double Jres[6], float& chi2, double& chi2d) {
    Patch patch(level_image(B->cur_img, level_));
    const float scale = 1.0f / (1 << level_);
    chi2 = 0.0f;
    chi2d = 0.0;
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
        chi2d += (double)(res_ * res_ * weight);
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
    double pt_chi2d, seg_chi2d;
    computePoints(T_cur_from_ref, pt_H, pt_J, pt_chi2, pt_chi2d);
    computeSegments(T_cur_from_ref, seg_H, seg_J, seg_chi2, seg_chi2d);
    for (int k = 0; k < 36; ++k) H_[k] = pt_H[k] + seg_H[k];  // :167
    for (int k = 0; k < 6; ++k) Jres_[k] = pt_J[k] + seg_J[k];
    if (opt.chi2_double) return (double)((float)(pt_chi2d + seg_chi2d) / (float)n_meas_);
    float chi2 = pt_chi2 + seg_chi2;  // :171
    return chi2 / n_meas_;            // :192  (float / size_t -> float)
  }

  // vk::NLLSSolver<6,SE3>::optimizeGaussNewton + SparseImgAlign::solve/update (:697-710)
  void optimize(SE3& model) {
    if (use_weights_) {  // pre-pass: computeResiduals(model, false, true)
      // (work executed by the reference but without observable effect beyond what iteration 0
      // repeats at the same model; excluded from the patch_iters accounting, which counts GN passes)
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
      const bool reject = (iter_ > 0 && new_chi2 > chi2_) || stop_;
      if (trace && trace_n < trace_cap) {
        double* r = trace + (size_t)trace_n * kTraceStride;
        std::fill(r, r + kTraceStride, 0.0);
        r[0] = level_, r[1] = iter_, r[2] = new_chi2, r[3] = (double)n_meas_, r[4] = reject ? 0 : 1;
        std::copy(H_, H_ + 36, r + 5);
        std::copy(Jres_, Jres_ + 6, r + 41);
        std::copy(x_, x_ + 6, r + 47);
      }
      if (reject) {
        model = old_model;
        if (trace && trace_n < trace_cap) se3_to_pose7(model, trace + (size_t)trace_n++ * kTraceStride + 53);
        break;
      }
      double mx[6];
      for (int k = 0; k < 6; ++k) mx[k] = -x_[k];
      const SE3 new_model = se3_mul(model, se3_exp(mx));  // :709
      old_model = model;
      model = new_model;
      chi2_ = new_chi2;
      if (trace && trace_n < trace_cap) se3_to_pose7(model, trace + (size_t)trace_n++ * kTraceStride + 53);
      if (norm_max6(x_) <= eps_) break;
    }
  }

  // sparse_img_align.cpp:54-95.  Returns n_meas_/16; writes T_cur_w.
  size_t run(const plsvo_align_params& P, const SE3& T_ref_w, SE3& T_cur_w, int n_pts_list, int n_segs_list) {
    // reset()
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

void align_one(const plsvo_align_batch* B, const plsvo_align_params* P, const plsvo_align_result* out, int b,
               const AlignOptions& opt, double* trace, int trace_cap, int* trace_n) {
  SparseImgAlign s;
  s.B = B, s.b = b, s.opt = opt;
  const int np = B->pt_count ? B->pt_count[b] : B->n_pts;
  const int ns = B->seg_count ? B->seg_count[b] : B->n_segs;
  s.n_pts = np, s.n_segs = ns;
  const size_t po = (size_t)b * B->n_pts, so = (size_t)b * B->n_segs;
  s.pt_px = B->pt_px ? B->pt_px + 2 * po : nullptr;
  s.pt_f = B->pt_f ? B->pt_f + 3 * po : nullptr;
  s.pt_pos = B->pt_pos ? B->pt_pos + 3 * po : nullptr;
  s.pt_valid = B->pt_valid ? B->pt_valid + po : nullptr;
  s.seg_spx = B->seg_spx ? B->seg_spx + 2 * so : nullptr;
  s.seg_epx = B->seg_epx ? B->seg_epx + 2 * so : nullptr;
  s.seg_sf = B->seg_sf ? B->seg_sf + 3 * so : nullptr;
  s.seg_ef = B->seg_ef ? B->seg_ef + 3 * so : nullptr;
  s.seg_spos = B->seg_spos ? B->seg_spos + 3 * so : nullptr;
  s.seg_epos = B->seg_epos ? B->seg_epos + 3 * so : nullptr;
  s.seg_length = B->seg_length ? B->seg_length + so : nullptr;
  s.seg_alive.assign(ns, 1);
  if (B->seg_valid)
    for (int j = 0; j < ns; ++j) s.seg_alive[j] = B->seg_valid[so + j] ? 1 : 0;
  std::vector<uint8_t> alive0 = s.seg_alive;
  s.trace = trace, s.trace_cap = trace_cap;

  const SE3 T_ref_w = se3_from_pose7(B->T_ref_w + 7 * (size_t)b);
  SE3 T_cur_w = se3_from_pose7(B->T_cur_w + 7 * (size_t)b);
  const bool empty = (np == 0 && ns == 0);
  const size_t n_tracked = s.run(*P, T_ref_w, T_cur_w, np, ns);
  if (trace_n) *trace_n = s.trace_n;

  if (out->T_cur_w) {
    if (empty)  // early-out leaves cur_frame->T_f_w_ untouched
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

// ------------------------------------------------------------------------------------------------
// pose_optimizer::optimizeGaussNewton — src/pose_optimizer.cpp:38-260 and :262-582
// ------------------------------------------------------------------------------------------------
inline void project2d(Vec3 p, double uv[2]) {  // vk::project2d
  uv[0] = p.x / p.z;
  uv[1] = p.y / p.z;
}

// One frame's record of plsvo_oracle_poseopt_stats (doubles), per loop l (0 main, 1 refinement) where marked [2]:
//   exit[2]           why the loop ended: kPoExit*
//   fallback[2]       1 if some solve's A has an unpivoted LDL^T pivot that is not > 1e-13 * max|diag A|
//   scale_pt, scale_ls  the two MAD scales (before the fx factor)
//   med_count[4], med_tie[4]  the MAD point, MAD segment, error_init and error_final medians: live count, and whether
//                     the key of rank floor(n/2) equals a neighbour in sorted order
//   out_margin_pt, out_margin_ls  smallest |e - thr| / thr of the outlier decisions (inf: none, or an infinite thr)
//   chi2_margin[2]    smallest |new_chi2 - chi2| / max(|new_chi2|, |chi2|) of the new_chi2 > chi2 decisions evaluated
//   eps_margin[2]     smallest |norm_max(dT) - EPS| / EPS of the convergence decisions evaluated
//   iter_margin[2][kPoStatIters]  the smaller of the two at each iteration (inf: no decision with a margin)
enum { kPoExitNone = 0, kPoExitChi2 = 1, kPoExitNan = 2, kPoExitEps = 3, kPoExitCap = 4 };
enum {
  kPoStatIters = 32,
  kPoSExit = 0, kPoSFallback = 2, kPoSScalePt = 4, kPoSScaleLs = 5, kPoSMedCount = 6, kPoSMedTie = 10, kPoSOutPt = 14,
  kPoSOutLs = 15, kPoSChi2 = 16, kPoSEps = 18, kPoSIter = 20, kPoStats = kPoSIter + 2 * kPoStatIters
};
inline void keep_min(double& slot, double m) {  // a NaN margin sticks
  if (std::isnan(slot)) return;
  if (std::isnan(m) || m < slot) slot = m;
}
inline double outlier_margin(double e, double thr) {  // an infinite threshold keeps every feature, whatever round-off
  return std::isinf(thr) ? std::numeric_limits<double>::infinity() : std::fabs(e - thr) / thr;
}
inline double rel_margin(double a, double b) {
  const double s = std::max(std::fabs(a), std::fabs(b));
  return s > 0.0 ? std::fabs(a - b) / s : 0.0;
}
// The register solve's acceptance rule, from its statement rather than its code: without pivoting, A = L D L^T must
// have every d_j = A_jj - sum_{k<j} L_jk^2 d_k above 1e-13 times the largest |A_ii|; otherwise the pivoted solve runs.
inline bool reg_rule_rejects(const double A[36]) {
  double dmax = 0.0;
  for (int i = 0; i < 6; ++i) dmax = std::max(dmax, std::fabs(A[i * 6 + i]));
  double L[6][6] = {}, d[6];
  for (int j = 0; j < 6; ++j) {
    double s = A[j * 6 + j];
    for (int k = 0; k < j; ++k) s -= L[j][k] * L[j][k] * d[k];
    if (!(s > 1e-13 * dmax)) return true;
    d[j] = s;
    for (int i = j + 1; i < 6; ++i) {
      double t = A[i * 6 + j];
      for (int k = 0; k < j; ++k) t -= L[i][k] * L[j][k] * d[k];
      L[i][j] = t / s;
    }
  }
  return false;
}
template <class T>
void median_stats(std::vector<T> v, double* st, int which) {  // on a copy: get_median reorders its argument
  const size_t n = v.size(), k = n / 2;
  st[kPoSMedCount + which] = (double)n;
  if (n == 0) return;
  std::sort(v.begin(), v.end());
  st[kPoSMedTie + which] = ((k > 0 && v[k - 1] == v[k]) || (k + 1 < n && v[k + 1] == v[k])) ? 1.0 : 0.0;
}

void poseopt_one(const plsvo_poseopt_batch* B, const plsvo_poseopt_params* P, const plsvo_poseopt_result* out, int b,
                 double* st = nullptr) {
  if (st) {
    const double inf = std::numeric_limits<double>::infinity();
    std::fill(st, st + kPoStats, 0.0);
    std::fill(st + kPoSOutPt, st + kPoStats, inf);  // every margin
  }
  const int np = B->pt_count ? B->pt_count[b] : B->n_pts;
  const int ns = B->seg_count ? B->seg_count[b] : B->n_segs;
  const size_t po = (size_t)b * B->n_pts, so = (size_t)b * B->n_segs;
  const double* pt_f = B->pt_f + 3 * po;
  const double* pt_pos = B->pt_pos + 3 * po;
  const int32_t* pt_level = B->pt_level + po;
  const double* seg_line = B->seg_line ? B->seg_line + 3 * so : nullptr;
  const double* seg_spos = B->seg_spos ? B->seg_spos + 3 * so : nullptr;
  const double* seg_epos = B->seg_epos ? B->seg_epos + 3 * so : nullptr;
  const int32_t* seg_level = B->seg_level ? B->seg_level + so : nullptr;
  std::vector<uint8_t> pt_alive(np, 1), seg_alive(ns, 1);
  if (B->pt_valid)
    for (int i = 0; i < np; ++i) pt_alive[i] = B->pt_valid[po + i] ? 1 : 0;
  if (B->seg_valid)
    for (int j = 0; j < ns; ++j) seg_alive[j] = B->seg_valid[so + j] ? 1 : 0;
  const std::vector<uint8_t> pt_alive0 = pt_alive, seg_alive0 = seg_alive;
  const double fx = B->fx;
  SE3 T = se3_from_pose7(B->T_f_w + 7 * (size_t)b);

  if (out->iters) out->iters[2 * (size_t)b] = out->iters[2 * (size_t)b + 1] = 0;
  if (out->pt_outlier) std::memset(out->pt_outlier + po, 0, B->n_pts);
  if (out->seg_outlier && B->n_segs) std::memset(out->seg_outlier + so, 0, B->n_segs);

  double chi2 = 0.0;
  std::vector<double> chi2_vec_init, chi2_vec_final;
  SE3 T_old = T;
  double A[36], bvec[6];

  // :58-71 MAD scale on point errors
  std::vector<float> errors;
  errors.reserve(np + ns);
  for (int i = 0; i < np; ++i) {
    if (!pt_alive[i]) continue;
    double uvf[2], uvp[2];
    project2d({pt_f[3 * i], pt_f[3 * i + 1], pt_f[3 * i + 2]}, uvf);
    project2d(se3_act(T, {pt_pos[3 * i], pt_pos[3 * i + 1], pt_pos[3 * i + 2]}), uvp);
    double e[2] = {uvf[0] - uvp[0], uvf[1] - uvp[1]};
    const double s = 1.0 / (1 << pt_level[i]);
    e[0] *= s, e[1] *= s;
    errors.push_back((float)std::sqrt(e[0] * e[0] + e[1] * e[1]));
  }
  // NOTE: the reference calls getMedian on an empty vector (UB) when there are no valid points but
  // there are lines; we define that case as scale 0 (the assert in vk::getMedian would fire).
  if (st) median_stats(errors, st, 0);
  double estimated_scale_pt = errors.empty() ? 0.0 : (double)mad_scale(errors);
  size_t num_obs_pt = errors.size();
  // :73-87
  std::vector<float> errors_ls;
  for (int j = 0; j < ns; ++j) {
    if (!seg_alive[j]) continue;
    double s2[2], e2[2];
    project2d(se3_act(T, {seg_spos[3 * j], seg_spos[3 * j + 1], seg_spos[3 * j + 2]}), s2);
    project2d(se3_act(T, {seg_epos[3 * j], seg_epos[3 * j + 1], seg_epos[3 * j + 2]}), e2);
    const double* l = seg_line + 3 * j;
    float es = (float)(l[0] * s2[0] + l[1] * s2[1] + l[2] * 1.0);
    float ee = (float)(l[0] * e2[0] + l[1] * e2[1] + l[2] * 1.0);
    errors.push_back(std::sqrt(es * es + ee * ee));
    errors_ls.push_back(std::sqrt(es * es + ee * ee));
  }
  if (errors.empty()) {  // :88-89: return with outputs untouched
    if (out->status) out->status[b] = 1;
    if (out->T_f_w) std::memcpy(out->T_f_w + 7 * (size_t)b, B->T_f_w + 7 * (size_t)b, 7 * sizeof(double));
    return;
  }
  if (out->status) out->status[b] = 0;
  size_t num_obs_ls = errors_ls.size();
  double estimated_scale_ls = 1.f;
  if (st) median_stats(errors_ls, st, 1);
  if (!errors_ls.empty()) estimated_scale_ls = mad_scale(errors_ls);
  double estimated_scale = estimated_scale_pt;
  const double scale_pt = estimated_scale_pt, scale_ls = estimated_scale_ls;
  if (st) st[kPoSScalePt] = scale_pt, st[kPoSScaleLs] = scale_ls;

  // one GN loop (:103-195 and, for the 10-arg overload, :473-563)
  auto gn_loop = [&](size_t n_iter, int which) {
    if (st) st[kPoSExit + which] = n_iter > 0 ? kPoExitCap : kPoExitNone;
    auto margin = [&](size_t iter, int slot, double m) {
      keep_min(st[slot + which], m);
      if (iter < (size_t)kPoStatIters) keep_min(st[kPoSIter + which * kPoStatIters + iter], m);
    };
    for (size_t iter = 0; iter < n_iter; iter++) {
      std::fill(A, A + 36, 0.0);
      std::fill(bvec, bvec + 6, 0.0);
      double new_chi2 = 0.0;
      for (int i = 0; i < np; ++i) {
        if (!pt_alive[i]) continue;
        double J[2][6];
        const Vec3 xyz_f = se3_act(T, {pt_pos[3 * i], pt_pos[3 * i + 1], pt_pos[3 * i + 2]});
        jacobian_xyz2uv(xyz_f, J);
        double uvf[2], uvp[2];
        project2d({pt_f[3 * i], pt_f[3 * i + 1], pt_f[3 * i + 2]}, uvf);
        project2d(xyz_f, uvp);
        double e[2] = {uvf[0] - uvp[0], uvf[1] - uvp[1]};
        const double sqrt_inv_cov = 1.0 / (1 << pt_level[i]);
        e[0] *= sqrt_inv_cov, e[1] *= sqrt_inv_cov;
        const double e_sq = e[0] * e[0] + e[1] * e[1];
        if (iter == 0) chi2_vec_init.push_back(e_sq);
        for (int k = 0; k < 6; ++k) J[0][k] *= sqrt_inv_cov, J[1][k] *= sqrt_inv_cov;
        const double weight = tukey_value((float)(std::sqrt(e_sq) / scale_pt));
        for (int r = 0; r < 6; ++r) {
          for (int c = 0; c < 6; ++c) A[r * 6 + c] += (J[0][r] * J[0][c] + J[1][r] * J[1][c]) * weight;
          bvec[r] -= (J[0][r] * e[0] + J[1][r] * e[1]) * weight;
        }
        new_chi2 += e_sq * weight;
      }
      for (int j = 0; j < ns; ++j) {
        if (!seg_alive[j]) continue;
        double J_s[2][6], J_e[2][6], J[2][6];
        const Vec3 xyz_f_s = se3_act(T, {seg_spos[3 * j], seg_spos[3 * j + 1], seg_spos[3 * j + 2]});
        const Vec3 xyz_f_e = se3_act(T, {seg_epos[3 * j], seg_epos[3 * j + 1], seg_epos[3 * j + 2]});
        jacobian_xyz2uv(xyz_f_s, J_s);
        jacobian_xyz2uv(xyz_f_e, J_e);
        double s2[2], e2[2];
        project2d(xyz_f_s, s2);
        project2d(xyz_f_e, e2);
        const double* l = seg_line + 3 * j;
        const float ds = (float)(l[0] * s2[0] + l[1] * s2[1] + l[2] * 1.0);
        const float de = (float)(l[0] * e2[0] + l[1] * e2[1] + l[2] * 1.0);
        double e[2] = {ds, de};
        const double sqrt_inv_cov = 1.0 / (1 << seg_level[j]);
        e[0] *= sqrt_inv_cov, e[1] *= sqrt_inv_cov;
        const double e_sq = e[0] * e[0] + e[1] * e[1];
        if (iter == 0) chi2_vec_init.push_back(e_sq);
        const double e_norm = std::sqrt(e_sq);
        const double js = sqrt_inv_cov * ds / e_norm;  // :157-158: ds for BOTH endpoints [sic]
        for (int k = 0; k < 6; ++k) {
          J_s[0][k] *= js, J_s[1][k] *= js;
          J_e[0][k] *= js, J_e[1][k] *= js;
        }
        for (int k = 0; k < 6; ++k) {
          J[0][k] = l[0] * J_s[0][k] + l[1] * J_s[1][k];
          J[1][k] = l[0] * J_e[0][k] + l[1] * J_e[1][k];
        }
        const double weight = tukey_value((float)(e_norm / scale_ls));
        for (int r = 0; r < 6; ++r) {
          for (int c = 0; c < 6; ++c) A[r * 6 + c] += (J[0][r] * J[0][c] + J[1][r] * J[1][c]) * weight;
          bvec[r] -= (J[0][r] * e[0] + J[1][r] * e[1]) * weight;
        }
        new_chi2 += e_sq * weight;
      }
      double dT[6];
      solve6(A, bvec, dT);
      if (out->iters) out->iters[2 * (size_t)b + which] += 1;
      if (st) {
        if (reg_rule_rejects(A)) st[kPoSFallback + which] = 1.0;
        if (iter > 0) margin(iter, kPoSChi2, rel_margin(new_chi2, chi2));
      }
      if ((iter > 0 && new_chi2 > chi2) || std::isnan(dT[0])) {
        if (st) st[kPoSExit + which] = (iter > 0 && new_chi2 > chi2) ? kPoExitChi2 : kPoExitNan;
        T = T_old;
        break;
      }
      const SE3 T_new = se3_mul(se3_exp(dT), T);
      T_old = T;
      T = T_new;
      chi2 = new_chi2;
      if (st) margin(iter, kPoSEps, std::fabs(norm_max6(dT) - 0.0000000001) / 0.0000000001);
      if (norm_max6(dT) <= 0.0000000001) {  // EPS, global.h:99
        if (st) st[kPoSExit + which] = kPoExitEps;
        break;
      }
    }
  };

  gn_loop((size_t)P->n_iter, 0);

  // :197-199 covariance from the last evaluated A
  double Afx[36], cov[36];
  const double fx2 = std::pow(fx, 2);
  for (int k = 0; k < 36; ++k) Afx[k] = A[k] * fx2;
  inverse6(Afx, cov);

  // :201-242 outlier removal at the final pose
  const double reproj_thresh_scaled_pt = P->reproj_thresh / fx;
  const double reproj_thresh_scaled_ls = reproj_thresh_scaled_pt * estimated_scale_ls / estimated_scale_pt;
  size_t n_deleted_refs_pt = 0, n_deleted_refs_ls = 0;
  for (int i = 0; i < np; ++i) {
    if (!pt_alive[i]) continue;
    double uvf[2], uvp[2];
    project2d({pt_f[3 * i], pt_f[3 * i + 1], pt_f[3 * i + 2]}, uvf);
    project2d(se3_act(T, {pt_pos[3 * i], pt_pos[3 * i + 1], pt_pos[3 * i + 2]}), uvp);
    double e[2] = {uvf[0] - uvp[0], uvf[1] - uvp[1]};
    const double s = 1.0 / (1 << pt_level[i]);
    e[0] *= s, e[1] *= s;
    const double e_sq = e[0] * e[0] + e[1] * e[1];
    chi2_vec_final.push_back(e_sq);
    if (st) keep_min(st[kPoSOutPt], outlier_margin(std::sqrt(e_sq), reproj_thresh_scaled_pt));
    if (std::sqrt(e_sq) > reproj_thresh_scaled_pt) {
      pt_alive[i] = 0;
      ++n_deleted_refs_pt;
    }
  }
  for (int j = 0; j < ns; ++j) {
    if (!seg_alive[j]) continue;
    double s2[2], e2[2];
    project2d(se3_act(T, {seg_spos[3 * j], seg_spos[3 * j + 1], seg_spos[3 * j + 2]}), s2);
    project2d(se3_act(T, {seg_epos[3 * j], seg_epos[3 * j + 1], seg_epos[3 * j + 2]}), e2);
    const double* l = seg_line + 3 * j;
    double e[2] = {l[0] * s2[0] + l[1] * s2[1] + l[2] * 1.0, l[0] * e2[0] + l[1] * e2[1] + l[2] * 1.0};
    const double s = 1.0 / (1 << seg_level[j]);
    e[0] *= s, e[1] *= s;
    const double e_sq = e[0] * e[0] + e[1] * e[1];
    chi2_vec_final.push_back(e_sq);
    if (st) keep_min(st[kPoSOutLs], outlier_margin(std::sqrt(e_sq), reproj_thresh_scaled_ls));
    if (std::sqrt(e_sq) > reproj_thresh_scaled_ls) {
      seg_alive[j] = 0;
      ++n_deleted_refs_ls;
    }
  }

  if (P->n_iter_ref >= 0) gn_loop((size_t)P->n_iter_ref, 1);  // :469-563 refinement with inliers

  if (st) median_stats(chi2_vec_init, st, 2), median_stats(chi2_vec_final, st, 3);
  double error_init = 0.0, error_final = 0.0;
  if (!chi2_vec_init.empty()) error_init = std::sqrt(get_median(chi2_vec_init)) * fx;
  if (!chi2_vec_final.empty()) error_final = std::sqrt(get_median(chi2_vec_final)) * fx;
  estimated_scale *= fx;
  num_obs_pt -= n_deleted_refs_pt;
  num_obs_ls -= n_deleted_refs_ls;

  if (out->T_f_w) se3_to_pose7(T, out->T_f_w + 7 * (size_t)b);
  if (out->cov) std::memcpy(out->cov + 36 * (size_t)b, cov, sizeof(cov));
  if (out->estimated_scale) out->estimated_scale[b] = estimated_scale;
  if (out->error_init) out->error_init[b] = error_init;
  if (out->error_final) out->error_final[b] = error_final;
  if (out->num_obs_pt) out->num_obs_pt[b] = (int64_t)num_obs_pt;
  if (out->num_obs_ls) out->num_obs_ls[b] = (int64_t)num_obs_ls;
  if (out->pt_outlier)
    for (int i = 0; i < np; ++i) out->pt_outlier[po + i] = (pt_alive0[i] && !pt_alive[i]) ? 1 : 0;
  if (out->seg_outlier)
    for (int j = 0; j < ns; ++j) out->seg_outlier[so + j] = (seg_alive0[j] && !seg_alive[j]) ? 1 : 0;
}

template <class F>
void parallel_for(int n, int n_threads, F f) {
  if (n_threads <= 1 || n <= 1) {
    for (int i = 0; i < n; ++i) f(i);
    return;
  }
  std::atomic<int> next{0};
  std::vector<std::thread> pool;
  const int nt = std::min(n_threads, n);
  for (int t = 0; t < nt; ++t)
    pool.emplace_back([&] {
      for (int i; (i = next.fetch_add(1)) < n;) f(i);
    });
  for (auto& th : pool) th.join();
}

}  // namespace

extern "C" {

// flags: bit0 = accumulate chi2 in double; bits 1-2 = AlignOptions::h_mode (experiments; NOT the reference behaviour)
int plsvo_oracle_align_batch(const plsvo_align_batch* batch, const plsvo_align_params* params,
                             const plsvo_align_result* out, int n_threads, int flags) {
  if (!batch || !params || !out) return PLSVO_ERR_INVALID;
  if (params->max_level < params->min_level || params->min_level < 0 || params->max_level >= PLSVO_MAX_LEVELS)
    return PLSVO_ERR_INVALID;
  AlignOptions opt;
  opt.chi2_double = (flags & 1) != 0;
  opt.h_mode = (flags >> 1) & 3;  // bits 1-2: kernel-style normal equations (experiment, see AlignOptions)
  parallel_for(batch->batch, n_threads, [&](int b) { align_one(batch, params, out, b, opt, nullptr, 0, nullptr); });
  return PLSVO_OK;
}

// Per-iteration trace of one pair: records of plsvo_oracle_trace_stride() doubles, laid out
// [level, iter, new_chi2, n_meas, accepted, H(36), Jres(6), x(6), T_cur_from_ref after the step(7)].
int plsvo_oracle_trace_stride(void) { return kTraceStride; }
int plsvo_oracle_align_trace(const plsvo_align_batch* batch, const plsvo_align_params* params, int pair,
                             double* records, int max_records, int* n_records) {
  if (!batch || !params || pair < 0 || pair >= batch->batch) return PLSVO_ERR_INVALID;
  plsvo_align_result out;
  std::memset(&out, 0, sizeof(out));
  align_one(batch, params, &out, pair, AlignOptions{}, records, max_records, n_records);
  return PLSVO_OK;
}

int plsvo_oracle_poseopt_batch(const plsvo_poseopt_batch* batch, const plsvo_poseopt_params* params,
                               const plsvo_poseopt_result* out, int n_threads) {
  if (!batch || !params || !out) return PLSVO_ERR_INVALID;
  parallel_for(batch->batch, n_threads, [&](int b) { poseopt_one(batch, params, out, b); });
  return PLSVO_OK;
}

// The same optimisation, also recording every frame's decisions: stats [batch][plsvo_oracle_poseopt_stats_stride()]
// doubles, laid out as described at poseopt_one (test infrastructure: which exits, ties and near-ties a test batch reaches).
int plsvo_oracle_poseopt_stats_stride(void) { return kPoStats; }
int plsvo_oracle_poseopt_stats(const plsvo_poseopt_batch* batch, const plsvo_poseopt_params* params,
                               const plsvo_poseopt_result* out, double* stats, int n_threads) {
  if (!batch || !params || !out || !stats) return PLSVO_ERR_INVALID;
  parallel_for(batch->batch, n_threads, [&](int b) { poseopt_one(batch, params, out, b, stats + (size_t)kPoStats * b); });
  return PLSVO_OK;
}

// SE3 helpers exposed so tests can pin the Sophus restatement against closed forms.
void plsvo_oracle_se3_exp(const double* xi6, double* pose7) { se3_to_pose7(se3_exp(xi6), pose7); }
void plsvo_oracle_se3_mul(const double* a7, const double* b7, double* out7) {
  se3_to_pose7(se3_mul(se3_from_pose7(a7), se3_from_pose7(b7)), out7);
}
void plsvo_oracle_se3_inverse(const double* a7, double* out7) { se3_to_pose7(se3_inverse(se3_from_pose7(a7)), out7); }
void plsvo_oracle_solve6(const double* A36, const double* b6, double* x6) { solve6(A36, b6, x6); }
void plsvo_oracle_inverse6(const double* A36, double* out36) { inverse6(A36, out36); }

// vk::halfSample, scalar path (rpg_vikit vision.cpp): out(i,j) = (in(2i,2j)+in(2i,2j+1)+in(2i+1,2j)+in(2i+1,2j+1))/4,
// integer division; called level by level from frame_utils::createImgPyramid (src/frame.cpp:171-180).
// in: rows x cols with row pitch in_pitch; out: (rows/2) x (cols/2), pitch out_pitch.
void plsvo_oracle_half_sample(const uint8_t* in, int cols, int rows, size_t in_pitch, uint8_t* out, size_t out_pitch) {
  const int oc = cols / 2, orows = rows / 2;
  for (int i = 0; i < orows; ++i) {
    const uint8_t* top = in + (size_t)(2 * i) * in_pitch;
    const uint8_t* bottom = top + in_pitch;
    uint8_t* p = out + (size_t)i * out_pitch;
    for (int j = 0; j < oc; ++j, top += 2, bottom += 2, ++p)
      *p = static_cast<uint8_t>((top[0] + top[1] + bottom[0] + bottom[1]) / 4);
  }
}

// One feature's record of plsvo_oracle_align2d_stats / _align1d_stats / _match_direct_stats (doubles; written, never
// read — test infrastructure: which exits, bounds and degenerate systems a test batch reaches):
//   [kDsExit]      how the Gauss-Newton loop ended: kExitNone (no iteration ran), kExitFrame (the patch left the frame),
//                  kExitConverged, kExitCap (n_iter iterations ran), kExitBackoff (align1D's new_chi2 > chi2)
//   [kDsIter]      the iteration it ended at (n_iter - 1 at the cap; -1 without an iteration)
//   [kDsSingular]  bit 0: det == 0; bit 1: an entry of Hinv is not finite; bit 2: align1D's h_inv is not finite
//   [kDsConvMargin], [kDsBackMargin]  smallest |a - b| / |b| of the convergence test (update^2 < min_update_squared) and
//                  of the back-off test (new_chi2 > chi2); inf without such a test
//   [kDsTie]       1 if a back-off test compared equal chi2 values
//   [kDsDist + k]  smallest distance of floor(u), floor(v) to the in-frame bounds over all iterations, k = left (u - 4),
//                  top (v - 4), right (cols - 5 - u), bottom (rows - 5 - v); negative = outside; inf without an iteration
//   [kDsBound]     the bounds the frame exit failed: 1 left, 2 top, 4 right, 8 bottom
//   [kDsOffset]    (floor(u) - 4) & 3 at the first iteration inside the frame (the byte offset of the window), else -1
// findMatchDirect only:
//   [kDsReject]    the candidate failed the reference in-frame test (isInFrame(px / 2^level, 6, level))
//   [kDsNanWarp]   the affine warp is NaN (warpAffine leaves the zeroed patch as it is)
//   [kDsClamped]   getBestSearchLevel stopped at n_pyr_levels - 1 with D > 3 still true
//   [kDsZeroed]    number of border-patch pixels set to 0 because they fall outside the reference image
//   [kDsNanDir]    an edgelet whose warped gradient direction is NaN;  [kDsEdgelet] aligned with align1D
//   [kDsOnBound]   number of border-patch samples exactly on the last column or row (q0 == cols - 1 or q1 == rows - 1),
//                  which `q >= cols - 1` zeroes and `q > cols - 1` would interpolate; the four corners, which no template
//                  gradient reads, are not counted
enum { kDsExit, kDsIter, kDsSingular, kDsConvMargin, kDsBackMargin, kDsTie, kDsDist, kDsBound = kDsDist + 4, kDsOffset, kDsReject,
       kDsNanWarp, kDsClamped, kDsZeroed, kDsNanDir, kDsEdgelet, kDsOnBound, kDsStride };
enum { kExitNone, kExitFrame, kExitConverged, kExitCap, kExitBackoff };
struct DirectStats {
  double* s;
  void begin() {
    if (!s) return;
    for (int k = 0; k < kDsStride; ++k) s[k] = 0;
    s[kDsIter] = -1, s[kDsOffset] = -1;
    s[kDsConvMargin] = s[kDsBackMargin] = INFINITY;
    for (int k = 0; k < 4; ++k) s[kDsDist + k] = INFINITY;
  }
  static double margin(double a, double b) { return std::fabs(a - b) / std::fabs(b); }
  void bounds(int iter, int ui, int vi, int cols, int rows) {
    if (!s) return;
    const double d[4] = {(double)ui - 4, (double)vi - 4, (double)cols - 5 - ui, (double)rows - 5 - vi};
    int mask = 0;
    for (int k = 0; k < 4; ++k) s[kDsDist + k] = std::min(s[kDsDist + k], d[k]), mask |= d[k] < 0 ? 1 << k : 0;
    if (mask) s[kDsBound] = mask, exit(kExitFrame, iter);
    else if (s[kDsOffset] < 0) s[kDsOffset] = (double)((ui - 4) & 3);
  }
  void converge_test(float q, float thr) {
    if (s) s[kDsConvMargin] = std::min(s[kDsConvMargin], margin(q, thr));
  }
  void backoff_test(float new_chi2, float chi2) {
    if (!s) return;
    s[kDsBackMargin] = std::min(s[kDsBackMargin], margin(new_chi2, chi2));
    if (new_chi2 == chi2) s[kDsTie] = 1;
  }
  void singular(double det, const float* hinv, int n) {
    if (!s) return;
    int f = det == 0 ? 1 : 0;
    for (int k = 0; k < n; ++k) f |= std::isfinite(hinv[k]) ? 0 : 2;
    s[kDsSingular] = f;
  }
  void exit(int kind, int iter) {
    if (s) s[kDsExit] = kind, s[kDsIter] = iter;
  }
  void end(int n_iter) {  // the loop ran out of iterations
    if (s && n_iter > 0 && s[kDsExit] == kExitNone) exit(kExitCap, n_iter - 1);
  }
};

// feature_alignment::align2D, scalar path — src/feature_alignment.cpp:160-290.  cur_img: cols x rows, row step
// cur_step; ref_patch_with_border 10x10, ref_patch 8x8; px = cur_px_estimate in/out.  Returns `converged`.
// Hinv = H.inverse() follows Eigen's fixed-size 3x3 inverse (cofactors of column 0, determinant, 1/det).
static int align2d_one(const uint8_t* cur_img, int cols, int rows, size_t cur_step_, const uint8_t* ref_patch_with_border,
                       const uint8_t* ref_patch, int n_iter, double* px, DirectStats st) {
  const int patch_size_ = 8;
  Image im{cur_img, cols, rows, (int)cur_step_};
  bool converged = false;
  float ref_patch_dx[64], ref_patch_dy[64];
  float H[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  const int ref_step = patch_size_ + 2;
  float* it_dx = ref_patch_dx;
  float* it_dy = ref_patch_dy;
  for (int y = 0; y < patch_size_; ++y) {
    const uint8_t* it = ref_patch_with_border + (y + 1) * ref_step + 1;
    for (int x = 0; x < patch_size_; ++x, ++it, ++it_dx, ++it_dy) {
      float J[3];
      J[0] = 0.5 * (it[1] - it[-1]);
      J[1] = 0.5 * (it[ref_step] - it[-ref_step]);
      J[2] = 1;
      *it_dx = J[0];
      *it_dy = J[1];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) H[r][c] += J[r] * J[c];
    }
  }
  float Hinv[3][3];
  {
    auto cof = [&](int i, int j) {
      const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
      return H[i1][j1] * H[i2][j2] - H[i1][j2] * H[i2][j1];
    };
    const float c0 = cof(0, 0), c1 = cof(1, 0), c2 = cof(2, 0);
    const float det = (c0 * H[0][0] + c1 * H[1][0]) + c2 * H[2][0];
    const float invdet = 1.0f / det;
    Hinv[0][0] = c0 * invdet, Hinv[0][1] = c1 * invdet, Hinv[0][2] = c2 * invdet;
    Hinv[1][0] = cof(0, 1) * invdet, Hinv[1][1] = cof(1, 1) * invdet, Hinv[1][2] = cof(2, 1) * invdet;
    Hinv[2][0] = cof(0, 2) * invdet, Hinv[2][1] = cof(1, 2) * invdet, Hinv[2][2] = cof(2, 2) * invdet;
    st.singular(det, &Hinv[0][0], 9);
  }
  float mean_diff = 0;
  float u = (float)px[0];
  float v = (float)px[1];
  const float min_update_squared = 0.03 * 0.03;
  const int cur_step = (int)cur_step_;
  float update[3] = {0, 0, 0};
  for (int iter = 0; iter < n_iter; ++iter) {
    Patch patch(im);
    patch.setPosition((double)u, (double)v);
    st.bounds(iter, patch.u_ref_i, patch.v_ref_i, cols, rows);
    if (!patch.isInFrame(4)) break;
    patch.computeInterpWeights();
    const uint8_t* roi = im.data + (size_t)(patch.v_ref_i - 4) * im.stride + (patch.u_ref_i - 4);
    const uint8_t* it_ref = ref_patch;
    float* it_ref_dx = ref_patch_dx;
    float* it_ref_dy = ref_patch_dy;
    float Jres[3] = {0, 0, 0};
    for (int y = 0; y < 8; ++y) {
      const uint8_t* ptr = roi + (size_t)y * im.stride;
      for (int x = 0; x < 8; ++x, ++ptr, ++it_ref, ++it_ref_dx, ++it_ref_dy) {
        float search_pixel = patch.wTL * ptr[0] + patch.wTR * ptr[1] + patch.wBL * ptr[cur_step] + patch.wBR * ptr[cur_step + 1];
        float res = search_pixel - *it_ref + mean_diff;
        Jres[0] -= res * (*it_ref_dx);
        Jres[1] -= res * (*it_ref_dy);
        Jres[2] -= res;
      }
    }
    for (int r = 0; r < 3; ++r) update[r] = (Hinv[r][0] * Jres[0] + Hinv[r][1] * Jres[1]) + Hinv[r][2] * Jres[2];
    u += update[0];
    v += update[1];
    mean_diff += update[2];
    const float update_squared = update[0] * update[0] + update[1] * update[1];
    st.converge_test(update_squared, min_update_squared);
    if (update_squared < min_update_squared) {
      converged = true;
      st.exit(kExitConverged, iter);
      break;
    }
  }
  st.end(n_iter);
  px[0] = u, px[1] = v;
  return converged ? 1 : 0;
}
int plsvo_oracle_align2d(const uint8_t* cur_img, int cols, int rows, size_t cur_step_, const uint8_t* ref_patch_with_border,
                         const uint8_t* ref_patch, int n_iter, double* px) {
  return align2d_one(cur_img, cols, rows, cur_step_, ref_patch_with_border, ref_patch, n_iter, px, DirectStats{nullptr});
}

// feature_alignment::align1D — src/feature_alignment.cpp:40-157.  dir = direction the patch may move in;
// returns `converged`, writes px (in/out) and h_inv.  Matrix2f::inverse() follows Eigen's 2x2 path
// (determinant, 1/det, adjugate * invdet).
static int align1d_one(const uint8_t* cur_img, int cols, int rows, size_t cur_step_, const float* dir, const uint8_t* ref_patch_with_border,
                       const uint8_t* ref_patch, int n_iter, double* px, double* h_inv, DirectStats st) {
  const int halfpatch_size_ = 4, patch_size = 8;
  bool converged = false;
  float ref_patch_dv[64];
  float H[2][2] = {{0, 0}, {0, 0}};
  const int ref_step = patch_size + 2;
  float* it_dv = ref_patch_dv;
  for (int y = 0; y < patch_size; ++y) {
    const uint8_t* it = ref_patch_with_border + (y + 1) * ref_step + 1;
    for (int x = 0; x < patch_size; ++x, ++it, ++it_dv) {
      float J[2];
      J[0] = 0.5 * (dir[0] * (it[1] - it[-1]) + dir[1] * (it[ref_step] - it[-ref_step]));
      J[1] = 1;
      *it_dv = J[0];
      for (int r = 0; r < 2; ++r)
        for (int c = 0; c < 2; ++c) H[r][c] += J[r] * J[c];
    }
  }
  *h_inv = 1.0 / H[0][0] * patch_size * patch_size;
  float Hinv[2][2];
  {
    const float det = H[0][0] * H[1][1] - H[1][0] * H[0][1];
    const float invdet = 1.0f / det;
    Hinv[0][0] = H[1][1] * invdet;
    Hinv[1][0] = -H[1][0] * invdet;
    Hinv[0][1] = -H[0][1] * invdet;
    Hinv[1][1] = H[0][0] * invdet;
    st.singular(det, &Hinv[0][0], 4);
    if (st.s && !std::isfinite(*h_inv)) st.s[kDsSingular] += 4;
  }
  float mean_diff = 0;
  float u = (float)px[0];
  float v = (float)px[1];
  const float min_update_squared = 0.03 * 0.03;
  const int cur_step = (int)cur_step_;
  float chi2 = 0;
  float update[2] = {0, 0};
  for (int iter = 0; iter < n_iter; ++iter) {
    // int u_r = floor(u): out-of-range / NaN conversions give INT_MIN on x86 and fail the bounds test,
    // so the isnan() early return at :94-95 is never reached.
    const double fu = std::floor((double)u), fv = std::floor((double)v);
    const int u_r = (fu >= -2147483648.0 && fu < 2147483648.0) ? (int)fu : INT32_MIN;
    const int v_r = (fv >= -2147483648.0 && fv < 2147483648.0) ? (int)fv : INT32_MIN;
    st.bounds(iter, u_r, v_r, cols, rows);
    if (u_r < halfpatch_size_ || v_r < halfpatch_size_ || u_r >= cols - halfpatch_size_ || v_r >= rows - halfpatch_size_) break;
    const float subpix_x = u - u_r;
    const float subpix_y = v - v_r;
    const float wTL = (float)((1.0 - subpix_x) * (1.0 - subpix_y));
    const float wTR = (float)(subpix_x * (1.0 - subpix_y));
    const float wBL = (float)((1.0 - subpix_x) * subpix_y);
    const float wBR = subpix_x * subpix_y;
    const uint8_t* it_ref = ref_patch;
    const float* it_ref_dv = ref_patch_dv;
    float new_chi2 = 0.0;
    float Jres[2] = {0, 0};
    for (int y = 0; y < patch_size; ++y) {
      const uint8_t* it = cur_img + (ptrdiff_t)(v_r + y - halfpatch_size_) * cur_step + u_r - halfpatch_size_;
      for (int x = 0; x < patch_size; ++x, ++it, ++it_ref, ++it_ref_dv) {
        const float search_pixel = wTL * it[0] + wTR * it[1] + wBL * it[cur_step] + wBR * it[cur_step + 1];
        const float res = search_pixel - *it_ref + mean_diff;
        Jres[0] -= res * (*it_ref_dv);
        Jres[1] -= res;
        new_chi2 += res * res;
      }
    }
    if (iter > 0) st.backoff_test(new_chi2, chi2);
    if (iter > 0 && new_chi2 > chi2) {
      u -= update[0];
      v -= update[1];
      st.exit(kExitBackoff, iter);
      break;
    }
    chi2 = new_chi2;
    const float up0 = Hinv[0][0] * Jres[0] + Hinv[0][1] * Jres[1];
    const float up1 = Hinv[1][0] * Jres[0] + Hinv[1][1] * Jres[1];
    update[0] = up0, update[1] = up1;
    u += update[0] * dir[0];
    v += update[0] * dir[1];
    mean_diff += update[1];
    const float update_squared = update[0] * update[0] + update[1] * update[1];
    st.converge_test(update_squared, min_update_squared);
    if (update_squared < min_update_squared) {
      converged = true;
      st.exit(kExitConverged, iter);
      break;
    }
  }
  st.end(n_iter);
  px[0] = u, px[1] = v;
  return converged ? 1 : 0;
}
int plsvo_oracle_align1d(const uint8_t* cur_img, int cols, int rows, size_t cur_step_, const float* dir,
                         const uint8_t* ref_patch_with_border, const uint8_t* ref_patch, int n_iter, double* px, double* h_inv) {
  return align1d_one(cur_img, cols, rows, cur_step_, dir, ref_patch_with_border, ref_patch, n_iter, px, h_inv, DirectStats{nullptr});
}

// ------------------------------------------------------------------------------------------------
// Matcher::findMatchDirect(const Point&, const Frame&, Vector2d&) — src/matcher.cpp:159-211, with
// warp::getWarpMatrixAffine (:42-71), getBestSearchLevel (:73-87), warpAffine (:89-133),
// createPatchFromPatchWithBorder (:148-157) and vk::interpolateMat_8u (rpg_vikit vision.h).
// ------------------------------------------------------------------------------------------------
static Vec3 pinhole_cam2world(const plsvo_camera& c, double u, double v) {  // PinholeCamera::cam2world, undistorted
  const Vec3 xyz{(u - c.cx) / c.fx, (v - c.cy) / c.fy, 1.0};
  const double n = std::sqrt((xyz.x * xyz.x + xyz.y * xyz.y) + xyz.z * xyz.z);
  return {xyz.x / n, xyz.y / n, xyz.z / n};
}
static void pinhole_world2cam(const plsvo_camera& c, Vec3 p, double px[2]) {  // world2cam(project2d(xyz))
  const double u = p.x / p.z, v = p.y / p.z;
  px[0] = c.fx * u + c.cx;
  px[1] = c.fy * v + c.cy;
}
static float interpolate_mat_8u(const uint8_t* data, int stride, float u, float v) {
  const int x = (int)std::floor(u);
  const int y = (int)std::floor(v);
  const float subpix_x = u - x;
  const float subpix_y = v - y;
  const float w00 = (1.0f - subpix_x) * (1.0f - subpix_y);
  const float w01 = (1.0f - subpix_x) * subpix_y;
  const float w10 = subpix_x * (1.0f - subpix_y);
  const float w11 = 1.0f - w00 - w01 - w10;
  const uint8_t* ptr = data + (ptrdiff_t)y * stride + x;
  return w00 * ptr[0] + w01 * ptr[stride] + w10 * ptr[1] + w11 * ptr[stride + 1];
}

// warp::getWarpMatrixAffine — src/matcher.cpp:42-71 (same undistorted pinhole for both frames)
static void warp_matrix_affine(const plsvo_camera& cam, const double* px_ref, Vec3 f_ref, double depth_ref, const SE3& T_cur_ref,
                               int level_ref, double A[2][2]) {
  const int halfpatch_size = 5;
  const Vec3 xyz_ref = f_ref * depth_ref;
  const double step = (double)halfpatch_size * (double)(1 << level_ref);
  Vec3 xyz_du_ref = pinhole_cam2world(cam, px_ref[0] + step, px_ref[1] + 0.0 * (double)(1 << level_ref));
  Vec3 xyz_dv_ref = pinhole_cam2world(cam, px_ref[0] + 0.0 * (double)(1 << level_ref), px_ref[1] + step);
  xyz_du_ref = xyz_du_ref * (xyz_ref.z / xyz_du_ref.z);
  xyz_dv_ref = xyz_dv_ref * (xyz_ref.z / xyz_dv_ref.z);
  double px_cur[2], px_du[2], px_dv[2];
  pinhole_world2cam(cam, se3_act(T_cur_ref, xyz_ref), px_cur);
  pinhole_world2cam(cam, se3_act(T_cur_ref, xyz_du_ref), px_du);
  pinhole_world2cam(cam, se3_act(T_cur_ref, xyz_dv_ref), px_dv);
  A[0][0] = (px_du[0] - px_cur[0]) / halfpatch_size;
  A[1][0] = (px_du[1] - px_cur[1]) / halfpatch_size;
  A[0][1] = (px_dv[0] - px_cur[0]) / halfpatch_size;
  A[1][1] = (px_dv[1] - px_cur[1]) / halfpatch_size;
}
// warp::getBestSearchLevel — :73-87
static int best_search_level(const double A[2][2], int max_level, bool* clamped = nullptr) {
  int search_level = 0;
  double D = A[0][0] * A[1][1] - A[1][0] * A[0][1];
  while (D > 3.0 && search_level < max_level) {
    search_level += 1;
    D *= 0.25;
  }
  if (clamped) *clamped = D > 3.0;
  return search_level;
}
// warp::warpAffine with halfpatch_size = 5 (:89-133) + createPatchFromPatchWithBorder (:148-157).
// patch_with_border must be zero-initialised by the caller (a NaN warp leaves it untouched).
static void warp_affine_patches(const double A[2][2], const uint8_t* img, int stride, int cols, int rows, const double* px_ref,
                                int level_ref, int search_level, uint8_t patch_with_border[100], uint8_t patch[64],
                                DirectStats st = DirectStats{nullptr}) {
  const int halfpatch_size = 5, patch_size = 10;
  const double det = A[0][0] * A[1][1] - A[1][0] * A[0][1];
  const double invdet = 1.0 / det;
  const float R00 = (float)(A[1][1] * invdet), R10 = (float)(-A[1][0] * invdet);
  const float R01 = (float)(-A[0][1] * invdet), R11 = (float)(A[0][0] * invdet);
  if (st.s && std::isnan(R00)) st.s[kDsNanWarp] = 1;
  if (!std::isnan(R00)) {
    const float pr0 = (float)px_ref[0] / (1 << level_ref), pr1 = (float)px_ref[1] / (1 << level_ref);
    uint8_t* patch_ptr = patch_with_border;
    for (int y = 0; y < patch_size; ++y)
      for (int x = 0; x < patch_size; ++x, ++patch_ptr) {
        float p0 = (float)(x - halfpatch_size), p1 = (float)(y - halfpatch_size);
        p0 *= (1 << search_level), p1 *= (1 << search_level);
        const float q0 = (R00 * p0 + R01 * p1) + pr0;
        const float q1 = (R10 * p0 + R11 * p1) + pr1;
        const bool corner = (x == 0 || x == 9) && (y == 0 || y == 9);  // no template gradient reads the corners
        if (st.s && !corner && (q0 == cols - 1 || q1 == rows - 1)) st.s[kDsOnBound] += 1;
        if (q0 < 0 || q1 < 0 || q0 >= cols - 1 || q1 >= rows - 1) {
          *patch_ptr = 0;
          if (st.s) st.s[kDsZeroed] += 1;
        } else
          *patch_ptr = (uint8_t)interpolate_mat_8u(img, stride, q0, q1);
      }
  }
  for (int y = 1; y < 9; ++y)
    for (int x = 0; x < 8; ++x) patch[(y - 1) * 8 + x] = patch_with_border[y * 10 + 1 + x];
}

static void match_direct_one(const plsvo_match_batch* in, const plsvo_match_result* out, int i, double* stats = nullptr) {
  const plsvo_camera& cam = in->cam;
  const int halfpatch_size_ = 4;
  const size_t I = (size_t)i;
  const double* px_ref = in->ref_px + 2 * I;
  const int level_ref = in->ref_level[i];
  DirectStats st{stats ? stats + (size_t)kDsStride * I : nullptr};
  st.begin();
  out->px_cur[2 * I] = in->px_cur[2 * I], out->px_cur[2 * I + 1] = in->px_cur[2 * I + 1];
  out->success[i] = 0;
  if (out->search_level) out->search_level[i] = -1;
  // :169-171  isInFrame(px.cast<int>()/(1<<level), halfpatch_size_+2, level)
  {
    const int ox = (int)px_ref[0] / (1 << level_ref), oy = (int)px_ref[1] / (1 << level_ref);
    if (!cam_is_in_frame(cam, ox, oy, halfpatch_size_ + 2, level_ref)) {
      if (st.s) st.s[kDsReject] = 1;
      return;
    }
  }
  const SE3 T_ref_w = se3_from_pose7(in->T_ref_w + 7 * (size_t)in->ref_index[i]);
  const SE3 T_cur_w = se3_from_pose7(in->T_cur_w + 7 * (size_t)in->cur_index[i]);
  const SE3 T_w_ref = se3_inverse(T_ref_w);
  const SE3 T_cur_ref = se3_mul(T_cur_w, T_w_ref);
  const Vec3 pos{in->pos[3 * I], in->pos[3 * I + 1], in->pos[3 * I + 2]};
  const Vec3 f_ref{in->ref_f[3 * I], in->ref_f[3 * I + 1], in->ref_f[3 * I + 2]};
  const double depth_ref = norm(T_w_ref.t - pos);  // (ref_ftr_->frame->pos() - pt.pos_).norm()
  double A[2][2];
  warp_matrix_affine(cam, px_ref, f_ref, depth_ref, T_cur_ref, level_ref, A);
  bool clamped;
  const int search_level = best_search_level(A, in->n_pyr_levels - 1, &clamped);
  if (st.s) st.s[kDsClamped] = clamped;
  if (out->search_level) out->search_level[i] = search_level;
  if (out->A_cur_ref) out->A_cur_ref[4 * I] = A[0][0], out->A_cur_ref[4 * I + 1] = A[0][1], out->A_cur_ref[4 * I + 2] = A[1][0], out->A_cur_ref[4 * I + 3] = A[1][1];
  uint8_t patch_with_border[100] = {0};
  uint8_t patch[64];
  warp_affine_patches(A, in->ref_img[level_ref] + (size_t)in->ref_index[i] * in->ref_stride[level_ref], (int)in->ref_pitch[level_ref],
                      cam.width >> level_ref, cam.height >> level_ref, px_ref, level_ref, search_level, patch_with_border, patch, st);
  // ---- align at the search level ----
  const double scale = (double)(1 << search_level);
  double px_scaled[2] = {in->px_cur[2 * I] / scale, in->px_cur[2 * I + 1] / scale};
  const uint8_t* cur = in->cur_img[search_level] + (size_t)in->cur_index[i] * in->cur_stride[search_level];
  const int ccols = cam.width >> search_level, crows = cam.height >> search_level;
  int ok;
  if (in->is_edgelet && in->is_edgelet[i]) {
    const double g0 = in->ref_grad[2 * I], g1 = in->ref_grad[2 * I + 1];
    double d0 = A[0][0] * g0 + A[0][1] * g1, d1 = A[1][0] * g0 + A[1][1] * g1;
    const double n = std::sqrt(d0 * d0 + d1 * d1);
    d0 /= n, d1 /= n;
    const float dir[2] = {(float)d0, (float)d1};
    if (st.s) st.s[kDsEdgelet] = 1, st.s[kDsNanDir] = std::isnan(dir[0]) || std::isnan(dir[1]);
    double h_inv;
    ok = align1d_one(cur, ccols, crows, in->cur_pitch[search_level], dir, patch_with_border, patch, in->n_iter, px_scaled, &h_inv, st);
  } else {
    ok = align2d_one(cur, ccols, crows, in->cur_pitch[search_level], patch_with_border, patch, in->n_iter, px_scaled, st);
  }
  out->px_cur[2 * I] = px_scaled[0] * scale, out->px_cur[2 * I + 1] = px_scaled[1] * scale;
  out->success[i] = (uint8_t)ok;
}

int plsvo_oracle_match_direct_batch(const plsvo_match_batch* in, const plsvo_match_result* out, int n_threads) {
  if (!in || !out) return PLSVO_ERR_INVALID;
  parallel_for(in->n_features, n_threads, [&](int i) { match_direct_one(in, out, i); });
  return PLSVO_OK;
}

// The stride of the records of the three *_stats entry points below (see DirectStats).
int plsvo_oracle_direct_stats_stride(void) { return kDsStride; }
// The same findMatchDirect, also recording every candidate's decisions: stats [n_features][kDsStride].
int plsvo_oracle_match_direct_stats(const plsvo_match_batch* in, const plsvo_match_result* out, double* stats, int n_threads) {
  if (!in || !out || !stats) return PLSVO_ERR_INVALID;
  parallel_for(in->n_features, n_threads, [&](int i) { match_direct_one(in, out, i, stats); });
  return PLSVO_OK;
}

// ------------------------------------------------------------------------------------------------
// Structure optimisation — Point::optimize (src/feature3D_impl.cpp:36-95), LineSeg::optimize (:97-174),
// Point::jacobian_xyz2uv (include/plsvo/feature3D.h:126-140), Eigen 3x3 LDLT (same unblocked pivoted
// algorithm as the 6x6 one above).
// ------------------------------------------------------------------------------------------------
struct Ldlt3 {
  double m[3][3];
  int tr[3];
  bool zero;  // the k == 0 early return ran: the whole diagonal of A is 0 (or NaN)
};
static void ldlt3_compute(const double A[3][3], Ldlt3& f) {
  const int n = 3;
  f.zero = false;
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) f.m[i][j] = A[i][j];
  for (int k = 0; k < n; ++k) {
    int piv = k;
    double big = std::fabs(f.m[k][k]);
    for (int i = k + 1; i < n; ++i)
      if (std::fabs(f.m[i][i]) > big) big = std::fabs(f.m[i][i]), piv = i;
    f.tr[k] = piv;
    if (piv != k) {
      for (int j = 0; j < k; ++j) std::swap(f.m[k][j], f.m[piv][j]);
      for (int i = piv + 1; i < n; ++i) std::swap(f.m[i][k], f.m[i][piv]);
      std::swap(f.m[k][k], f.m[piv][piv]);
      for (int i = k + 1; i < piv; ++i) std::swap(f.m[i][k], f.m[piv][i]);
    }
    if (k > 0) {
      double temp[3];
      for (int j = 0; j < k; ++j) temp[j] = f.m[j][j] * f.m[k][j];
      double s = 0;
      for (int j = 0; j < k; ++j) s += f.m[k][j] * temp[j];
      f.m[k][k] -= s;
      for (int i = k + 1; i < n; ++i) {
        double s2 = 0;
        for (int j = 0; j < k; ++j) s2 += f.m[i][j] * temp[j];
        f.m[i][k] -= s2;
      }
    }
    const double akk = f.m[k][k];
    const bool pivot_is_valid = std::fabs(akk) > 0.0;
    if (k == 0 && !pivot_is_valid) {
      for (int j = 0; j < n; ++j) f.tr[j] = j;
      f.zero = true;
      return;
    }
    if (pivot_is_valid)
      for (int i = k + 1; i < n; ++i) f.m[i][k] /= akk;
  }
}
static const double kLdlt3Tol = 1.0 / std::numeric_limits<double>::max();  // the pseudo-inverse's cut of D
static void ldlt3_solve(const Ldlt3& f, const double b[3], double x[3]) {
  const int n = 3;
  for (int i = 0; i < n; ++i) x[i] = b[i];
  for (int k = 0; k < n; ++k) std::swap(x[k], x[f.tr[k]]);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < i; ++j) x[i] -= f.m[i][j] * x[j];
  const double tol = kLdlt3Tol;
  for (int i = 0; i < n; ++i) {
    if (std::fabs(f.m[i][i]) > tol)
      x[i] /= f.m[i][i];
    else
      x[i] = 0.0;
  }
  for (int i = n - 1; i >= 0; --i)
    for (int j = i + 1; j < n; ++j) x[i] -= f.m[j][i] * x[j];
  for (int k = n - 1; k >= 0; --k) std::swap(x[k], x[f.tr[k]]);
}
// one observation's contribution: A += J^T J, b -= J^T e, chi2 += |e|^2   (feature3D_impl.cpp:49-59)
static void structopt_accumulate(const SE3& T, const double R[3][3], Vec3 pos, Vec3 f, double A[3][3], double b[3], double& chi2) {
  const Vec3 p = se3_act(T, pos);
  const double z_inv = 1.0 / p.z;
  const double z_inv_sq = z_inv * z_inv;
  // point_jac = -[[z_inv, 0, -x z_inv^2], [0, z_inv, -y z_inv^2]] * R_f_w
  const double P[2][3] = {{-(z_inv), -(0.0), -(-p.x * z_inv_sq)}, {-(0.0), -(z_inv), -(-p.y * z_inv_sq)}};
  double J[2][3];
  for (int r = 0; r < 2; ++r)
    for (int c = 0; c < 3; ++c) J[r][c] = (P[r][0] * R[0][c] + P[r][1] * R[1][c]) + P[r][2] * R[2][c];
  const double e0 = f.x / f.z - p.x / p.z, e1 = f.y / f.z - p.y / p.z;
  chi2 += e0 * e0 + e1 * e1;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) A[r][c] += J[0][r] * J[0][c] + J[1][r] * J[1][c];
  for (int r = 0; r < 3; ++r) b[r] -= J[0][r] * e0 + J[1][r] * e1;
}
static double norm_max3(const double x[3]) { return std::max(std::max(std::fabs(x[0]), std::fabs(x[1])), std::fabs(x[2])); }

// One point's or one segment end's record of plsvo_oracle_structopt_stats (doubles):
//   exit        why the loop ended: kSoExit* (a segment's two ends share it)
//   exit_it     the iteration it ended at (-1: n_iter = 0)
//   cause       what this end did at the exit: 1 chi2 rise (it > 0), 2 NaN step, 4 step within EPS (a segment exits when
//               either end asks; cause tells which did)
//   pivots      bitmask over the LDLTs factored: bit 2 * tr[0] + tr[1] - 1 for the transposition pair (tr[0], tr[1])
//   zero        1 if some LDLT took the k == 0 early return (the whole diagonal 0)
//   d_zeroed    1 if, in an LDLT without the early return, the pseudo-inverse tolerance zeroed a finite D entry
//   d_ratio     smallest min|D| / max|D| over the LDLTs factored (NaN sticks; 0 / 0 counts as 0)
//   A[9], b[3]  the first iteration's normal equations (0: n_iter = 0)
enum { kSoExitNone = 0, kSoExitChi2 = 1, kSoExitNan = 2, kSoExitEps = 3, kSoExitCap = 4 };
enum { kSoSExit = 0, kSoSIt = 1, kSoSCause = 2, kSoSPivots = 3, kSoSZero = 4, kSoSZeroed = 5, kSoSRatio = 6, kSoSA = 7, kSoSB = 16,
       kSoStats = 19 };
static void structopt_stat_ldlt(double* st, const Ldlt3& f) {
  if (!st) return;
  st[kSoSPivots] = (double)((int)st[kSoSPivots] | (1 << (2 * f.tr[0] + f.tr[1] - 1)));
  if (f.zero) {
    st[kSoSZero] = 1;
  } else {
    for (int i = 0; i < 3; ++i)
      if (std::fabs(f.m[i][i]) <= kLdlt3Tol) st[kSoSZeroed] = 1;
  }
  double lo = std::fabs(f.m[0][0]), hi = lo;
  for (int i = 1; i < 3; ++i) lo = std::min(lo, std::fabs(f.m[i][i])), hi = std::max(hi, std::fabs(f.m[i][i]));
  const bool nan = std::isnan(f.m[0][0]) || std::isnan(f.m[1][1]) || std::isnan(f.m[2][2]);
  keep_min(st[kSoSRatio], nan ? std::numeric_limits<double>::quiet_NaN() : hi > 0 ? lo / hi : 0.0);
}
static void structopt_stat_first(double* st, int it, const double A[3][3], const double b[3]) {
  if (!st || it != 0) return;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) st[kSoSA + 3 * r + c] = A[r][c];
    st[kSoSB + r] = b[r];
  }
}
static void structopt_stat_init(double* st) {
  if (!st) return;
  for (int k = 0; k < kSoStats; ++k) st[k] = 0;
  st[kSoSExit] = kSoExitNone, st[kSoSIt] = -1, st[kSoSRatio] = std::numeric_limits<double>::infinity();
}
static void structopt_stat_exit(double* st, int exit, int it, int cause) {
  if (st) st[kSoSExit] = exit, st[kSoSIt] = it, st[kSoSCause] = cause;
}

namespace {
struct StructOptFrames {
  std::vector<SE3> T;
  std::vector<double> R;
  explicit StructOptFrames(const plsvo_structopt_batch* in) : T(in->n_frames), R((size_t)in->n_frames * 9) {
    for (int k = 0; k < in->n_frames; ++k) {
      T[k] = se3_from_pose7(in->T_f_w + 7 * (size_t)k);
      quat_to_matrix(T[k].q, reinterpret_cast<double(*)[3]>(R.data() + 9 * (size_t)k));
    }
  }
  const double (*Rk(int k) const)[3] { return reinterpret_cast<const double(*)[3]>(R.data() + 9 * (size_t)k); }
};
const double kStructOptEps = 0.0000000001;  // plsvo::EPS, global.h:92
}  // namespace

// Point::optimize of point i; st: its record, or nullptr
static void structopt_point(const plsvo_structopt_batch* in, const StructOptFrames& F, const plsvo_structopt_result* out, int i, double* st) {
  structopt_stat_init(st);
  Vec3 pos{in->pt_pos[3 * (size_t)i], in->pt_pos[3 * (size_t)i + 1], in->pt_pos[3 * (size_t)i + 2]};
  Vec3 old_point = pos;
  double chi2 = 0.0;
  int iters = 0;
  for (int it = 0; it < in->n_iter_pts; ++it) {
    double A[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, b[3] = {0, 0, 0}, new_chi2 = 0.0;
    for (int o = in->pt_obs_begin[i]; o < in->pt_obs_begin[i + 1]; ++o) {
      const int k = in->pt_obs_frame[o];
      structopt_accumulate(F.T[k], F.Rk(k), pos, Vec3{in->pt_obs_f[3 * (size_t)o], in->pt_obs_f[3 * (size_t)o + 1], in->pt_obs_f[3 * (size_t)o + 2]},
                           A, b, new_chi2);
    }
    structopt_stat_first(st, it, A, b);
    Ldlt3 f;
    ldlt3_compute(A, f);
    structopt_stat_ldlt(st, f);
    double dp[3];
    ldlt3_solve(f, b, dp);
    ++iters;
    if ((it > 0 && new_chi2 > chi2) || std::isnan(dp[0])) {
      const bool rise = it > 0 && new_chi2 > chi2;
      structopt_stat_exit(st, rise ? kSoExitChi2 : kSoExitNan, it, (rise ? 1 : 0) | (std::isnan(dp[0]) ? 2 : 0));
      pos = old_point;
      break;
    }
    const Vec3 new_point{pos.x + dp[0], pos.y + dp[1], pos.z + dp[2]};
    old_point = pos;
    pos = new_point;
    chi2 = new_chi2;
    if (norm_max3(dp) <= kStructOptEps) {
      structopt_stat_exit(st, kSoExitEps, it, 4);
      break;
    }
    if (it + 1 == in->n_iter_pts) structopt_stat_exit(st, kSoExitCap, it, 0);
  }
  out->pt_pos[3 * (size_t)i] = pos.x, out->pt_pos[3 * (size_t)i + 1] = pos.y, out->pt_pos[3 * (size_t)i + 2] = pos.z;
  if (out->pt_iters) out->pt_iters[i] = iters;
}

// LineSeg::optimize of segment i; st: the records of its s and e ends, or nullptr
static void structopt_segment(const plsvo_structopt_batch* in, const StructOptFrames& F, const plsvo_structopt_result* out, int i, double* st) {
  double* ss = st;
  double* se = st ? st + kSoStats : nullptr;
  structopt_stat_init(ss);
  structopt_stat_init(se);
  const size_t I = (size_t)i;
  Vec3 sp{in->seg_spos[3 * I], in->seg_spos[3 * I + 1], in->seg_spos[3 * I + 2]};
  Vec3 ep{in->seg_epos[3 * I], in->seg_epos[3 * I + 1], in->seg_epos[3 * I + 2]};
  Vec3 old_s = sp, old_e = ep;
  double chi2s = 0.0, chi2e = 0.0;
  int iters = 0;
  for (int it = 0; it < in->n_iter_segs; ++it) {
    double As[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, Ae[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    double bs[3] = {0, 0, 0}, be[3] = {0, 0, 0}, ns = 0.0, ne = 0.0;
    for (int o = in->seg_obs_begin[i]; o < in->seg_obs_begin[i + 1]; ++o) {
      const int k = in->seg_obs_frame[o];
      const size_t O = (size_t)o;
      structopt_accumulate(F.T[k], F.Rk(k), sp, Vec3{in->seg_obs_sf[3 * O], in->seg_obs_sf[3 * O + 1], in->seg_obs_sf[3 * O + 2]}, As, bs, ns);
      structopt_accumulate(F.T[k], F.Rk(k), ep, Vec3{in->seg_obs_ef[3 * O], in->seg_obs_ef[3 * O + 1], in->seg_obs_ef[3 * O + 2]}, Ae, be, ne);
    }
    structopt_stat_first(ss, it, As, bs);
    structopt_stat_first(se, it, Ae, be);
    Ldlt3 fs, fe;
    ldlt3_compute(As, fs);
    ldlt3_compute(Ae, fe);
    structopt_stat_ldlt(ss, fs);
    structopt_stat_ldlt(se, fe);
    double dps[3], dpe[3];
    ldlt3_solve(fs, bs, dps);
    ldlt3_solve(fe, be, dpe);
    ++iters;
    if ((it > 0 && ns > chi2s) || std::isnan(dps[0]) || (it > 0 && ne > chi2e) || std::isnan(dpe[0])) {
      const int cs = (it > 0 && ns > chi2s ? 1 : 0) | (std::isnan(dps[0]) ? 2 : 0);
      const int ce = (it > 0 && ne > chi2e ? 1 : 0) | (std::isnan(dpe[0]) ? 2 : 0);
      const int exit = ((cs | ce) & 1) ? kSoExitChi2 : kSoExitNan;  // a rise at either end counts as a chi2 exit
      structopt_stat_exit(ss, exit, it, cs);
      structopt_stat_exit(se, exit, it, ce);
      sp = old_s, ep = old_e;
      break;
    }
    const Vec3 new_s{sp.x + dps[0], sp.y + dps[1], sp.z + dps[2]};
    old_s = sp, sp = new_s, chi2s = ns;
    const Vec3 new_e{ep.x + dpe[0], ep.y + dpe[1], ep.z + dpe[2]};
    old_e = ep, ep = new_e, chi2e = ne;
    if (norm_max3(dps) <= kStructOptEps || norm_max3(dpe) <= kStructOptEps) {
      structopt_stat_exit(ss, kSoExitEps, it, norm_max3(dps) <= kStructOptEps ? 4 : 0);
      structopt_stat_exit(se, kSoExitEps, it, norm_max3(dpe) <= kStructOptEps ? 4 : 0);
      break;
    }
    if (it + 1 == in->n_iter_segs) structopt_stat_exit(ss, kSoExitCap, it, 0), structopt_stat_exit(se, kSoExitCap, it, 0);
  }
  out->seg_spos[3 * I] = sp.x, out->seg_spos[3 * I + 1] = sp.y, out->seg_spos[3 * I + 2] = sp.z;
  out->seg_epos[3 * I] = ep.x, out->seg_epos[3 * I + 1] = ep.y, out->seg_epos[3 * I + 2] = ep.z;
  if (out->seg_iters) out->seg_iters[i] = iters;
}

int plsvo_oracle_structopt_batch(const plsvo_structopt_batch* in, const plsvo_structopt_result* out, int n_threads) {
  if (!in || !out) return PLSVO_ERR_INVALID;
  const StructOptFrames F(in);
  parallel_for(in->n_points, n_threads, [&](int i) { structopt_point(in, F, out, i, nullptr); });
  parallel_for(in->n_segs, n_threads, [&](int i) { structopt_segment(in, F, out, i, nullptr); });
  return PLSVO_OK;
}

// The same optimisation, also recording every feature's decisions (test infrastructure: which pivots, exits and degenerate
// systems a test batch reaches): pt_stats [n_points][stride], seg_stats [n_segs][2 (s, e)][stride] doubles, laid out as
// described above structopt_stat_ldlt.
int plsvo_oracle_structopt_stats_stride(void) { return kSoStats; }
int plsvo_oracle_structopt_stats(const plsvo_structopt_batch* in, const plsvo_structopt_result* out, double* pt_stats, double* seg_stats,
                                 int n_threads) {
  if (!in || !out || (in->n_points > 0 && !pt_stats) || (in->n_segs > 0 && !seg_stats)) return PLSVO_ERR_INVALID;
  const StructOptFrames F(in);
  parallel_for(in->n_points, n_threads, [&](int i) { structopt_point(in, F, out, i, pt_stats + (size_t)kSoStats * i); });
  parallel_for(in->n_segs, n_threads, [&](int i) { structopt_segment(in, F, out, i, seg_stats + (size_t)2 * kSoStats * i); });
  return PLSVO_OK;
}

// ------------------------------------------------------------------------------------------------
// Depth-filter point-seed update: DepthFilter::updatePointSeeds body (src/depth_filter.cpp:270-365),
// Matcher::findEpipolarMatchDirect (src/matcher.cpp:277-420), depthFromTriangulation (:135-146),
// vk::patch_score::ZMSSD<4> (rpg_vikit patch_score.h), DepthFilter::computeTau (:568-584),
// DepthFilter::updatePointSeed (:489-512), boost::math::pdf(normal_distribution<float>).
// ------------------------------------------------------------------------------------------------
static bool depth_from_triangulation(const SE3& T_search_ref, Vec3 f_ref, Vec3 f_cur, double& depth) {
  double R[3][3];
  quat_to_matrix(T_search_ref.q, R);
  const double fr[3] = {f_ref.x, f_ref.y, f_ref.z};
  double A[3][2];
  for (int i = 0; i < 3; ++i) A[i][0] = (R[i][0] * fr[0] + R[i][1] * fr[1]) + R[i][2] * fr[2];
  A[0][1] = f_cur.x, A[1][1] = f_cur.y, A[2][1] = f_cur.z;
  double AtA[2][2];
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) AtA[i][j] = (A[0][i] * A[0][j] + A[1][i] * A[1][j]) + A[2][i] * A[2][j];
  const double det = AtA[0][0] * AtA[1][1] - AtA[1][0] * AtA[0][1];
  if (det < 0.000001) return false;
  const double invdet = 1.0 / det;
  // M = -(AtA.inverse())
  const double M[2][2] = {{-(AtA[1][1] * invdet), -(-AtA[0][1] * invdet)}, {-(-AtA[1][0] * invdet), -(AtA[0][0] * invdet)}};
  // N = M * A^T (2x3), depth2 = N * t
  const double t[3] = {T_search_ref.t.x, T_search_ref.t.y, T_search_ref.t.z};
  double N0[3];
  for (int j = 0; j < 3; ++j) N0[j] = M[0][0] * A[j][0] + M[0][1] * A[j][1];
  const double d0 = (N0[0] * t[0] + N0[1] * t[1]) + N0[2] * t[2];
  depth = std::fabs(d0);
  return true;
}

struct EpiResult {
  int search_level = -1;
  double px_cur[2] = {std::numeric_limits<double>::quiet_NaN(), std::numeric_limits<double>::quiet_NaN()};
  // statistics of the ZMSSD search (plsvo_oracle_*seed_search_stats; written, never read): its step count n_steps + 1
  // (-1: the search was never reached), whether max_epi_search_steps rejected it, the first and the last step whose score
  // equals the final best (-1: none), whether no score beat PatchScore::threshold()
  int steps = -1, rejected = 0, first_best = -1, last_best = -1, no_win = 0;
};
// segment_endpoint = true restates Matcher::findEpipolarMatchDirectSegmentEndpoint (src/matcher.cpp:420-588): NaN depth
// range and NaN/inf epipolar length are rejected up front, no edgelet pre-selection, otherwise the same search.
static bool find_epipolar_match_direct(const plsvo_seed_batch* in, int i, double d_estimate, double d_min, double d_max, double& depth,
                                       EpiResult& er, bool segment_endpoint = false) {
  const plsvo_camera& cam = in->cam;
  const size_t I = (size_t)i;
  const int halfpatch_size_ = 4, patch_size_ = 8;
  const SE3 T_ref_w = se3_from_pose7(in->T_ref_w + 7 * (size_t)in->ref_index[i]);
  const SE3 T_cur_w = se3_from_pose7(in->T_cur_w + 7 * (size_t)in->cur_index[i]);
  const SE3 T_cur_ref = se3_mul(T_cur_w, se3_inverse(T_ref_w));
  const Vec3 f{in->ref_f[3 * I], in->ref_f[3 * I + 1], in->ref_f[3 * I + 2]};
  const double* px_ref = in->ref_px + 2 * I;
  const int level_ref = in->ref_level[i];
  int zmssd_best = 2000 * 64;  // PatchScore::threshold()
  double uv_best[2] = {0, 0};
  if (segment_endpoint && (std::isnan(d_min) || std::isnan(d_max))) return false;  // :434-438
  // start and end of the epipolar segment on the unit plane (:291-293)
  double A2[2], B2[2];
  project2d(se3_act(T_cur_ref, f * d_min), A2);
  project2d(se3_act(T_cur_ref, f * d_max), B2);
  const double epi_dir[2] = {A2[0] - B2[0], A2[1] - B2[1]};
  double A[2][2];
  warp_matrix_affine(cam, px_ref, f, d_estimate, T_cur_ref, level_ref, A);
  // feature pre-selection (:300-310)
  if (!segment_endpoint && in->is_edgelet && in->is_edgelet[i] && in->epi_search_edgelet_filtering) {
    const double g0 = in->ref_grad[2 * I], g1 = in->ref_grad[2 * I + 1];
    double c0 = A[0][0] * g0 + A[0][1] * g1, c1 = A[1][0] * g0 + A[1][1] * g1;
    const double nc = std::sqrt(c0 * c0 + c1 * c1);
    c0 /= nc, c1 /= nc;
    const double ne = std::sqrt(epi_dir[0] * epi_dir[0] + epi_dir[1] * epi_dir[1]);
    const double e0 = epi_dir[0] / ne, e1 = epi_dir[1] / ne;
    const double cosangle = std::fabs(c0 * e0 + c1 * e1);
    if (cosangle < in->epi_search_edgelet_max_angle) return false;  // reject_
  }
  const int search_level = best_search_level(A, in->n_pyr_levels - 1);
  er.search_level = search_level;
  // length of the search range (:315-317); world2cam(Vector2d uv) = (fx*u+cx, fy*v+cy)
  const double px_A[2] = {cam.fx * A2[0] + cam.cx, cam.fy * A2[1] + cam.cy};
  const double px_B[2] = {cam.fx * B2[0] + cam.cx, cam.fy * B2[1] + cam.cy};
  const double dAB[2] = {px_A[0] - px_B[0], px_A[1] - px_B[1]};
  const double epi_length = std::sqrt(dAB[0] * dAB[0] + dAB[1] * dAB[1]) / (1 << search_level);
  if (segment_endpoint && (std::isnan(epi_length) || std::isinf(epi_length))) return false;  // :481-485
  uint8_t patch_with_border[100] = {0};
  uint8_t patch[64];
  warp_affine_patches(A, in->ref_img[level_ref] + (size_t)in->ref_index[i] * in->ref_stride[level_ref], (int)in->ref_pitch[level_ref],
                      cam.width >> level_ref, cam.height >> level_ref, px_ref, level_ref, search_level, patch_with_border, patch);
  const uint8_t* cur = in->cur_img[search_level] + (size_t)in->cur_index[i] * in->cur_stride[search_level];
  const int ccols = cam.width >> search_level, crows = cam.height >> search_level;
  const size_t cpitch = in->cur_pitch[search_level];
  const double scale = (double)(1 << search_level);
  float dir1d[2];
  {  // (px_A-px_B).cast<float>().normalized()
    const float fx_ = (float)dAB[0], fy_ = (float)dAB[1];
    const float n = std::sqrt(fx_ * fx_ + fy_ * fy_);
    dir1d[0] = fx_ / n, dir1d[1] = fy_ / n;
  }
  auto refine_and_triangulate = [&](const double px_start[2]) -> bool {
    double px_scaled[2] = {px_start[0] / scale, px_start[1] / scale};
    int res;
    double h_inv;
    if (in->align_1d)
      res = plsvo_oracle_align1d(cur, ccols, crows, cpitch, dir1d, patch_with_border, patch, in->n_iter, px_scaled, &h_inv);
    else
      res = plsvo_oracle_align2d(cur, ccols, crows, cpitch, patch_with_border, patch, in->n_iter, px_scaled);
    if (res) {
      er.px_cur[0] = px_scaled[0] * scale, er.px_cur[1] = px_scaled[1] * scale;
      if (depth_from_triangulation(T_cur_ref, f, pinhole_cam2world(cam, er.px_cur[0], er.px_cur[1]), depth)) return true;
    }
    return false;
  };
  if (epi_length < 2.0 && (segment_endpoint || (!std::isnan(fabsf((float)epi_length)) && !std::isinf(fabsf((float)epi_length))))) {  // :324-343
    er.px_cur[0] = (px_A[0] + px_B[0]) / 2.0, er.px_cur[1] = (px_A[1] + px_B[1]) / 2.0;
    const double start[2] = {er.px_cur[0], er.px_cur[1]};
    return refine_and_triangulate(start);
  }
  size_t n_steps = (size_t)(epi_length / 0.7);  // one step per pixel (:345)
  const double step[2] = {epi_dir[0] / (double)n_steps, epi_dir[1] / (double)n_steps};
  er.steps = n_steps < (size_t)INT32_MAX ? (int)n_steps + 1 : INT32_MAX;
  er.rejected = n_steps > (size_t)in->max_epi_search_steps;
  if (n_steps > (size_t)in->max_epi_search_steps) return false;
  // ZMSSD of the warped reference patch (:354-356)
  int sumA = 0, sumAA = 0;
  for (int r = 0; r < 64; ++r) sumA += patch[r], sumAA += patch[r] * patch[r];
  double uv[2] = {B2[0] - step[0], B2[1] - step[1]};
  int last_checked[2] = {0, 0};
  ++n_steps;
  for (size_t k = 0; k < n_steps; ++k, uv[0] += step[0], uv[1] += step[1]) {
    const double px[2] = {cam.fx * uv[0] + cam.cx, cam.fy * uv[1] + cam.cy};
    const double qx = px[0] / (1 << search_level) + 0.5, qy = px[1] / (1 << search_level) + 0.5;
    // Vector2i(double, double): conversion toward zero (x86 gives INT_MIN outside the int range / for NaN)
    const int pxi0 = (qx >= -2147483648.0 && qx < 2147483648.0) ? (int)qx : INT32_MIN;
    const int pxi1 = (qy >= -2147483648.0 && qy < 2147483648.0) ? (int)qy : INT32_MIN;
    if (pxi0 == last_checked[0] && pxi1 == last_checked[1]) continue;
    last_checked[0] = pxi0, last_checked[1] = pxi1;
    if (!cam_is_in_frame(cam, pxi0, pxi1, patch_size_, search_level)) continue;
    // the reference strides the patch with Mat::cols (:380-382); images are dense (checked by the caller)
    const uint8_t* cur_patch_ptr = cur + (ptrdiff_t)(pxi1 - halfpatch_size_) * ccols + (pxi0 - halfpatch_size_);
    int sumB = 0, sumBB = 0, sumAB = 0;
    for (int y = 0, r = 0; y < patch_size_; ++y) {
      const uint8_t* p = cur_patch_ptr + (ptrdiff_t)y * ccols;
      for (int x = 0; x < patch_size_; ++x, ++r) {
        const int cur_px = p[x];
        sumB += cur_px, sumBB += cur_px * cur_px, sumAB += cur_px * patch[r];
      }
    }
    const int zmssd = sumAA - 2 * sumAB + sumBB - (sumA * sumA - 2 * sumA * sumB + sumB * sumB) / 64;
    if (zmssd < zmssd_best) zmssd_best = zmssd, uv_best[0] = uv[0], uv_best[1] = uv[1], er.first_best = (int)k;
    if (zmssd == zmssd_best && er.first_best >= 0) er.last_best = (int)k;
  }
  er.no_win = zmssd_best >= 2000 * 64;
  if (zmssd_best < 2000 * 64) {
    er.px_cur[0] = cam.fx * uv_best[0] + cam.cx, er.px_cur[1] = cam.fy * uv_best[1] + cam.cy;
    if (in->subpix_refinement) {
      const double start[2] = {er.px_cur[0], er.px_cur[1]};
      return refine_and_triangulate(start);
    }
    const Vec3 u3{uv_best[0], uv_best[1], 1.0};  // vk::unproject2d(uv_best).normalized()
    const double n = std::sqrt((u3.x * u3.x + u3.y * u3.y) + u3.z * u3.z);
    if (depth_from_triangulation(T_cur_ref, f, Vec3{u3.x / n, u3.y / n, u3.z / n}, depth)) return true;
  }
  return false;
}

static double compute_tau(const SE3& T_ref_cur, Vec3 f, double z, double px_error_angle) {  // depth_filter.cpp:568-584
  const Vec3 t = T_ref_cur.t;
  const Vec3 a = f * z - t;
  const double t_norm = norm(t), a_norm = norm(a);
  const double alpha = std::acos(((f.x * t.x + f.y * t.y) + f.z * t.z) / t_norm);
  const Vec3 mt{-t.x, -t.y, -t.z};
  const double beta = std::acos(((a.x * mt.x + a.y * mt.y) + a.z * mt.z) / (t_norm * a_norm));
  const double beta_plus = beta + px_error_angle;
  const double gamma_plus = 3.14159265 - alpha - beta_plus;  // plsvo::PI (global.h:93)
  const double z_plus = t_norm * std::sin(beta_plus) / std::sin(gamma_plus);
  return z_plus - z;
}
struct SeedState {
  float a, b, mu, z_range, sigma2;
};
static void update_point_seed(const float x, const float tau2, SeedState* seed) {  // depth_filter.cpp:489-512
  const float norm_scale = std::sqrt(seed->sigma2 + tau2);
  if (std::isnan(norm_scale)) return;
  float pdf;
  {  // boost::math::pdf(normal_distribution<float>(mu, norm_scale), x)
    float exponent = x - seed->mu;
    exponent *= -exponent;
    exponent /= 2 * norm_scale * norm_scale;
    pdf = std::exp(exponent);
    pdf /= norm_scale * std::sqrt(2 * static_cast<float>(3.141592653589793238462643383279502884L));
    if (std::isinf(x)) pdf = 0;
  }
  const float s2 = 1. / (1. / seed->sigma2 + 1. / tau2);
  const float m = s2 * (seed->mu / seed->sigma2 + x / tau2);
  float C1 = seed->a / (seed->a + seed->b) * pdf;
  float C2 = seed->b / (seed->a + seed->b) * 1. / seed->z_range;
  const float normalization_constant = C1 + C2;
  C1 /= normalization_constant;
  C2 /= normalization_constant;
  const float f = C1 * (seed->a + 1.) / (seed->a + seed->b + 1.) + C2 * seed->a / (seed->a + seed->b + 1.);
  const float e = C1 * (seed->a + 1.) * (seed->a + 2.) / ((seed->a + seed->b + 1.) * (seed->a + seed->b + 2.)) +
                  C2 * seed->a * (seed->a + 1.0f) / ((seed->a + seed->b + 1.0f) * (seed->a + seed->b + 2.0f));
  const float mu_new = C1 * m + C2 * seed->mu;
  seed->sigma2 = C1 * (s2 + m * m) + C2 * (seed->sigma2 + seed->mu * seed->mu) - mu_new * mu_new;
  seed->mu = mu_new;
  seed->a = (e - f) / (f - e / f);
  seed->b = seed->a * (1.0f - f) / f;
}

// one search's record of plsvo_oracle_*seed_search_stats: steps, rejected, search level, first best, last best, no win
enum { kSearchStats = 6 };
static void put_search_stats(const EpiResult& er, int32_t* s) {
  if (!s) return;
  s[0] = er.steps, s[1] = er.rejected, s[2] = er.search_level, s[3] = er.first_best, s[4] = er.last_best, s[5] = er.no_win;
}

static void seed_update_one(const plsvo_seed_batch* in, const plsvo_seed_result* out, int i, int32_t* stats = nullptr) {
  const plsvo_camera& cam = in->cam;
  const size_t I = (size_t)i;
  SeedState sd{in->a[i], in->b[i], in->mu[i], in->z_range[i], in->sigma2[i]};
  int status = PLSVO_SEED_NOT_VISIBLE;
  double z = std::numeric_limits<double>::quiet_NaN();
  EpiResult er;
  const SE3 T_ref_w = se3_from_pose7(in->T_ref_w + 7 * (size_t)in->ref_index[i]);
  const SE3 T_cur_w = se3_from_pose7(in->T_cur_w + 7 * (size_t)in->cur_index[i]);
  const Vec3 f{in->ref_f[3 * I], in->ref_f[3 * I + 1], in->ref_f[3 * I + 2]};
  const double focal_length = std::fabs(cam.fx);  // errorMultiplier2()
  const double px_noise = 1.0;
  const double px_error_angle = std::atan(px_noise / (2.0 * focal_length)) * 2.0;  // law of chord (:279-280)
  do {
    const SE3 T_ref_cur = se3_mul(T_ref_w, se3_inverse(T_cur_w));  // :291
    const Vec3 xyz_f = se3_act(se3_inverse(T_ref_cur), f * (1.0 / sd.mu));
    if (xyz_f.z < 0.0) break;  // behind the camera
    double pxc[2];
    pinhole_world2cam(cam, xyz_f, pxc);
    {
      const int ox = (pxc[0] >= -2147483648.0 && pxc[0] < 2147483648.0) ? (int)pxc[0] : INT32_MIN;
      const int oy = (pxc[1] >= -2147483648.0 && pxc[1] < 2147483648.0) ? (int)pxc[1] : INT32_MIN;
      if (!(ox >= 0 && ox < cam.width && oy >= 0 && oy < cam.height)) break;  // isInFrame(obs, 0)
    }
    const float z_inv_min = sd.mu + std::sqrt(sd.sigma2);
    const float z_inv_max = std::max(sd.mu - std::sqrt(sd.sigma2), 0.00000001f);
    if (!find_epipolar_match_direct(in, i, 1.0 / sd.mu, 1.0 / z_inv_min, 1.0 / z_inv_max, z, er)) {
      sd.b++;  // :314
      status = PLSVO_SEED_NO_MATCH;
      z = std::numeric_limits<double>::quiet_NaN();
      break;
    }
    const double tau = compute_tau(T_ref_cur, f, z, px_error_angle);
    const double tau_inverse = 0.5 * (1.0 / std::max(0.0000001, z - tau) - 1.0 / (z + tau));
    update_point_seed((float)(1. / z), (float)(tau_inverse * tau_inverse), &sd);
    status = PLSVO_SEED_UPDATED;
  } while (false);
  out->a[i] = sd.a, out->b[i] = sd.b, out->mu[i] = sd.mu, out->sigma2[i] = sd.sigma2;
  out->status[i] = status;
  if (out->converged)
    out->converged[i] = (status == PLSVO_SEED_UPDATED && std::sqrt(sd.sigma2) < sd.z_range / in->seed_convergence_sigma2_thresh) ? 1 : 0;
  if (out->depth) out->depth[i] = z;
  if (out->px_cur) out->px_cur[2 * I] = er.px_cur[0], out->px_cur[2 * I + 1] = er.px_cur[1];
  put_search_stats(er, stats ? stats + kSearchStats * I : nullptr);
}

int plsvo_oracle_seed_update_batch(const plsvo_seed_batch* in, const plsvo_seed_result* out, int n_threads) {
  if (!in || !out) return PLSVO_ERR_INVALID;
  parallel_for(in->n_seeds, n_threads, [&](int i) { seed_update_one(in, out, i); });
  return PLSVO_OK;
}

// The same update, also recording the epipolar search of every seed: stats [n_seeds][kSearchStats] (test infrastructure:
// which step counts, ties and winners a test batch exercises).
int plsvo_oracle_seed_search_stats(const plsvo_seed_batch* in, const plsvo_seed_result* out, int32_t* stats, int n_threads) {
  if (!in || !out || !stats) return PLSVO_ERR_INVALID;
  parallel_for(in->n_seeds, n_threads, [&](int i) { seed_update_one(in, out, i, stats); });
  return PLSVO_OK;
}

// One end point's share of DepthFilter::updateLineSeed (depth_filter.cpp:524-539 / :541-556): new mean and variance of the
// end point's Gaussian and the moments f, e of the Beta update — the same arithmetic as update_point_seed.
static void line_endpoint_update(float x, float tau2, float norm_scale, float a, float b, float z_range, float& mu, float& sigma2,
                                 float& f_out, float& e_out) {
  float pdf;
  {
    float exponent = x - mu;
    exponent *= -exponent;
    exponent /= 2 * norm_scale * norm_scale;
    pdf = std::exp(exponent);
    pdf /= norm_scale * std::sqrt(2 * static_cast<float>(3.141592653589793238462643383279502884L));
    if (std::isinf(x)) pdf = 0;
  }
  const float s2 = 1. / (1. / sigma2 + 1. / tau2);
  const float m = s2 * (mu / sigma2 + x / tau2);
  float C1 = a / (a + b) * pdf;
  float C2 = b / (a + b) * 1. / z_range;
  const float normalization_constant = C1 + C2;
  C1 /= normalization_constant;
  C2 /= normalization_constant;
  f_out = C1 * (a + 1.) / (a + b + 1.) + C2 * a / (a + b + 1.);
  e_out = C1 * (a + 1.) * (a + 2.) / ((a + b + 1.) * (a + b + 2.)) + C2 * a * (a + 1.0f) / ((a + b + 1.0f) * (a + b + 2.0f));
  const float mu_new = C1 * m + C2 * mu;
  sigma2 = C1 * (s2 + m * m) + C2 * (sigma2 + mu * mu) - mu_new * mu_new;
  mu = mu_new;
}

static void line_seed_update_one(const plsvo_line_seed_batch* inl, const plsvo_line_seed_result* outl, int i, int32_t* stats = nullptr) {
  const plsvo_seed_batch* in = &inl->seeds;
  const plsvo_seed_result* out = &outl->seeds;
  const plsvo_camera& cam = in->cam;
  const size_t I = (size_t)i;
  float a = in->a[i], b = in->b[i];
  float mu_s = in->mu[i], sig_s = in->sigma2[i], mu_e = inl->mu_e[i], sig_e = inl->sigma2_e[i];
  const float zr_s = in->z_range[i], zr_e = inl->z_range_e[i];
  int status = PLSVO_SEED_NOT_VISIBLE;
  const double nan = std::numeric_limits<double>::quiet_NaN();
  double z_s = nan, z_e = nan;
  EpiResult er_s, er_e;
  const SE3 T_ref_w = se3_from_pose7(in->T_ref_w + 7 * (size_t)in->ref_index[i]);
  const SE3 T_cur_w = se3_from_pose7(in->T_cur_w + 7 * (size_t)in->cur_index[i]);
  const Vec3 sf{inl->ref_sf[3 * I], inl->ref_sf[3 * I + 1], inl->ref_sf[3 * I + 2]};
  const Vec3 ef{inl->ref_ef[3 * I], inl->ref_ef[3 * I + 1], inl->ref_ef[3 * I + 2]};
  const double px_error_angle = std::atan(1.0 / (2.0 * std::fabs(cam.fx))) * 2.0;
  auto in_image = [&](Vec3 p) {
    double px[2];
    pinhole_world2cam(cam, p, px);
    const int ox = (px[0] >= -2147483648.0 && px[0] < 2147483648.0) ? (int)px[0] : INT32_MIN;
    const int oy = (px[1] >= -2147483648.0 && px[1] < 2147483648.0) ? (int)px[1] : INT32_MIN;
    return ox >= 0 && ox < cam.width && oy >= 0 && oy < cam.height;
  };
  do {
    const SE3 T_ref_cur = se3_mul(T_ref_w, se3_inverse(T_cur_w));  // :388
    const SE3 T_cur_ref_vis = se3_inverse(T_ref_cur);
    const Vec3 xyz_f_s = se3_act(T_cur_ref_vis, sf * (1.0 / mu_s));
    const Vec3 xyz_f_e = se3_act(T_cur_ref_vis, ef * (1.0 / mu_e));
    if (xyz_f_s.z < 0.0 || xyz_f_e.z < 0.0) break;
    if (!in_image(xyz_f_s) || !in_image(xyz_f_e)) break;
    const float z_inv_min_s = mu_s + std::sqrt(sig_s), z_inv_max_s = std::max(mu_s - std::sqrt(sig_s), 0.00000001f);
    const float z_inv_min_e = mu_e + std::sqrt(sig_e), z_inv_max_e = std::max(mu_e - std::sqrt(sig_e), 0.00000001f);
    if (!find_epipolar_match_direct(in, i, 1.0 / mu_s, 1.0 / z_inv_min_s, 1.0 / z_inv_max_s, z_s, er_s, true) ||
        !find_epipolar_match_direct(in, i, 1.0 / mu_e, 1.0 / z_inv_min_e, 1.0 / z_inv_max_e, z_e, er_e, true)) {
      b++;
      status = PLSVO_SEED_NO_MATCH;
      z_s = z_e = nan;
      break;
    }
    const double tau_s = compute_tau(T_ref_cur, sf, z_s, px_error_angle);
    const double tau_inverse_s = 0.5 * (1.0 / std::max(0.0000001, z_s - tau_s) - 1.0 / (z_s + tau_s));
    const double tau_e = compute_tau(T_ref_cur, ef, z_e, px_error_angle);
    const double tau_inverse_e = 0.5 * (1.0 / std::max(0.0000001, z_e - tau_e) - 1.0 / (z_e + tau_e));
    status = PLSVO_SEED_UPDATED;
    // updateLineSeed (:514-565)
    const float x_s = (float)(1. / z_s), tau2_s = (float)(tau_inverse_s * tau_inverse_s);
    const float x_e = (float)(1. / z_e), tau2_e = (float)(tau_inverse_e * tau_inverse_e);
    const float norm_scale_s = std::sqrt(sig_s + tau2_s), norm_scale_e = std::sqrt(sig_e + tau2_e);
    if (std::isnan(norm_scale_s) || std::isnan(norm_scale_e)) break;
    float f_s, e_s, f_e, e_e;
    line_endpoint_update(x_s, tau2_s, norm_scale_s, a, b, zr_s, mu_s, sig_s, f_s, e_s);
    line_endpoint_update(x_e, tau2_e, norm_scale_e, a, b, zr_e, mu_e, sig_e, f_e, e_e);
    const float a_s = (e_s - f_s) / (f_s - e_s / f_s), a_e = (e_e - f_e) / (f_e - e_e / f_e);
    const float b_s = a_s * (1.f - f_s) / f_s, b_e = a_e * (1.f - f_e) / f_e;
    a = std::max(a_s, a_e);
    b = std::min(b_s, b_e);
  } while (false);
  out->a[i] = a, out->b[i] = b, out->mu[i] = mu_s, out->sigma2[i] = sig_s;
  outl->mu_e[i] = mu_e, outl->sigma2_e[i] = sig_e;
  out->status[i] = status;
  if (out->converged)
    out->converged[i] = (status == PLSVO_SEED_UPDATED && std::sqrt(sig_s) < zr_s / in->seed_convergence_sigma2_thresh &&
                         std::sqrt(sig_e) < zr_e / in->seed_convergence_sigma2_thresh) ? 1 : 0;
  if (out->depth) out->depth[i] = z_s;
  if (outl->depth_e) outl->depth_e[i] = z_e;
  if (out->px_cur) out->px_cur[2 * I] = er_s.px_cur[0], out->px_cur[2 * I + 1] = er_s.px_cur[1];
  if (outl->px_cur_e) outl->px_cur_e[2 * I] = er_e.px_cur[0], outl->px_cur_e[2 * I + 1] = er_e.px_cur[1];
  put_search_stats(er_s, stats ? stats + kSearchStats * 2 * I : nullptr);
  put_search_stats(er_e, stats ? stats + kSearchStats * (2 * I + 1) : nullptr);
}

int plsvo_oracle_line_seed_update_batch(const plsvo_line_seed_batch* in, const plsvo_line_seed_result* out, int n_threads) {
  if (!in || !out) return PLSVO_ERR_INVALID;
  parallel_for(in->seeds.n_seeds, n_threads, [&](int i) { line_seed_update_one(in, out, i); });
  return PLSVO_OK;
}

// plsvo_oracle_seed_search_stats for line seeds: stats [n_seeds][2][kSearchStats], start point then end point (an end point
// whose start point did not match is never searched)
int plsvo_oracle_line_seed_search_stats(const plsvo_line_seed_batch* in, const plsvo_line_seed_result* out, int32_t* stats, int n_threads) {
  if (!in || !out || !stats) return PLSVO_ERR_INVALID;
  parallel_for(in->seeds.n_seeds, n_threads, [&](int i) { line_seed_update_one(in, out, i, stats); });
  return PLSVO_OK;
}

// Batch drivers over the ABI structs (CPU baseline of tools/bench_next.py): one call per feature, threads over features.
// (The *_stats variants also write each feature's DirectStats record to stats [n_features][kDsStride].)
static void align_batch_one(const plsvo_align2d_batch* in, const float* dir, double* o_px, uint8_t* o_conv, double* o_hinv, int i,
                            double* stats) {
  const int l = in->level[i];
  const uint8_t* img = in->img[l] + (size_t)in->image_index[i] * in->img_stride[l];
  double px[2] = {in->px[2 * (size_t)i], in->px[2 * (size_t)i + 1]};
  DirectStats st{stats ? stats + (size_t)kDsStride * i : nullptr};
  st.begin();
  const uint8_t* border = in->ref_patch_with_border + 100 * (size_t)i;
  const uint8_t* patch = in->ref_patch + 64 * (size_t)i;
  if (dir) {
    double h_inv = 0;
    o_conv[i] = (uint8_t)align1d_one(img, in->width >> l, in->height >> l, in->img_pitch[l], dir + 2 * (size_t)i, border, patch, in->n_iter,
                                     px, &h_inv, st);
    if (o_hinv) o_hinv[i] = h_inv;
  } else {
    o_conv[i] = (uint8_t)align2d_one(img, in->width >> l, in->height >> l, in->img_pitch[l], border, patch, in->n_iter, px, st);
  }
  o_px[2 * (size_t)i] = px[0], o_px[2 * (size_t)i + 1] = px[1];
}
int plsvo_oracle_align2d_batch(const plsvo_align2d_batch* in, const plsvo_align2d_result* out, int n_threads) {
  if (!in || !out) return PLSVO_ERR_INVALID;
  parallel_for(in->n_features, n_threads, [&](int i) { align_batch_one(in, nullptr, out->px, out->converged, nullptr, i, nullptr); });
  return PLSVO_OK;
}
int plsvo_oracle_align1d_batch(const plsvo_align1d_batch* in1, const plsvo_align1d_result* out, int n_threads) {
  if (!in1 || !out) return PLSVO_ERR_INVALID;
  parallel_for(in1->features.n_features, n_threads,
               [&](int i) { align_batch_one(&in1->features, in1->dir, out->px, out->converged, out->h_inv, i, nullptr); });
  return PLSVO_OK;
}
int plsvo_oracle_align2d_stats(const plsvo_align2d_batch* in, const plsvo_align2d_result* out, double* stats, int n_threads) {
  if (!in || !out || !stats) return PLSVO_ERR_INVALID;
  parallel_for(in->n_features, n_threads, [&](int i) { align_batch_one(in, nullptr, out->px, out->converged, nullptr, i, stats); });
  return PLSVO_OK;
}
int plsvo_oracle_align1d_stats(const plsvo_align1d_batch* in1, const plsvo_align1d_result* out, double* stats, int n_threads) {
  if (!in1 || !out || !stats) return PLSVO_ERR_INVALID;
  parallel_for(in1->features.n_features, n_threads,
               [&](int i) { align_batch_one(&in1->features, in1->dir, out->px, out->converged, out->h_inv, i, stats); });
  return PLSVO_OK;
}
int plsvo_oracle_pyramid_batch(const plsvo_pyramid_batch* in, const plsvo_pyramid_result* out, int n_threads) {
  if (!in || !out) return PLSVO_ERR_INVALID;
  parallel_for(in->batch, n_threads, [&](int b) {
    const uint8_t* prev = in->img0 + (size_t)b * in->stride0;
    size_t prev_pitch = in->pitch0;
    for (int l = 1; l < in->n_levels; ++l) {
      uint8_t* dst = out->level[l] + (size_t)b * out->stride[l];
      plsvo_oracle_half_sample(prev, in->width >> (l - 1), in->height >> (l - 1), prev_pitch, dst, out->pitch[l]);
      prev = dst, prev_pitch = out->pitch[l];
    }
  });
  return PLSVO_OK;
}

int plsvo_oracle_hardware_threads(void) { return (int)std::thread::hardware_concurrency(); }
}
