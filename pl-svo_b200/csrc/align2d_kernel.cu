// align2d_kernel.cu — feature_alignment::align2D (src/feature_alignment.cpp:160-290): 8x8 inverse-
// compositional Lucas-Kanade refinement of a feature position (2 DoF + mean intensity offset), the
// per-feature kernel of Matcher::findMatchDirect (src/matcher.cpp:201,257,268).  SURVEY.md §8f rank 1
// ("next"): the step between the two hot-path calls.
//
// One thread per feature keeps the reference's sequential fp32 accumulation order over the 64 pixels,
// so positions and convergence flags are bit-identical to the scalar reference code (the SSE2/NEON
// variants of the reference use fixed-point arithmetic and differ from its own scalar path).
// The 10x10 reference patch with border and the 8x8 reference patch of a feature live in shared
// memory; template gradients are recomputed from the border patch (two byte subtractions) instead
// of being cached.  Image bytes come straight from global memory / L2 (9x9 footprint per iteration).
#include <cuda_runtime.h>
#include <stdint.h>

#include "exact_math.cuh"
#include "internal.h"

namespace plsvo {
namespace {

constexpr int kA2Threads = 128;

// Exact u8 -> f32 and (u8 - u8) -> f32 without the conversion unit: 0x4B000000 | v is the float 2^23 + v, so one
// FADD gives v exactly; differences of two such values (|d| <= 255) and their halves are exact as well, i.e. the
// same numbers as the reference's int -> float / double conversions, produced on the FMA pipe instead of XU.
__device__ __forceinline__ float u8f(uint8_t v) { return __fsub_rn(__uint_as_float(0x4B000000u | (uint32_t)v), 8388608.0f); }
__device__ __forceinline__ float u8diff(uint8_t a, uint8_t b) {
  return __fsub_rn(__uint_as_float(0x4B000000u | (uint32_t)a), __uint_as_float(0x4B000000u | (uint32_t)b));
}

// Nine consecutive image bytes starting at an arbitrary address, as exact floats: three aligned 32-bit loads and
// two funnel shifts instead of nine byte loads (the image buffers are 256-byte aligned with 256 bytes of slack, so
// the aligned window never leaves the allocation).  Byte -> float through PRMT + FADD (see u8f).
__device__ __forceinline__ float bytef(uint32_t w, int k) {
  return __fsub_rn(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7440 | k)), 8388608.0f);
}
__device__ __forceinline__ void load_row9(const uint8_t* p, float f[9]) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~static_cast<uintptr_t>(3));
  const uint32_t sh = static_cast<uint32_t>(a & 3) * 8;
  const uint32_t w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2);
  const uint32_t lo = __funnelshift_r(w0, w1, sh), mid = __funnelshift_r(w1, w2, sh), hi = w2 >> sh;
#pragma unroll
  for (int k = 0; k < 4; ++k) f[k] = bytef(lo, k), f[4 + k] = bytef(mid, k);
  f[8] = bytef(hi, 0);
}

// align2D on one feature.  border = 10x10 reference patch with border, ref = 8x8 reference patch with row step
// ref_step (8 for a packed patch, 10 when it is the interior of `border`).  u,v in/out; returns `converged`.
__device__ __forceinline__ bool align2d_core(const uint8_t* border, const uint8_t* ref, const int ref_step, const uint8_t* img,
                                             const int cur_step, const int cols, const int rows, const int n_iter, float& u,
                                             float& v) {
  // ---- template Hessian (:183-201): J = (0.5*dx, 0.5*dy, 1), H = sum J J^T (exact in fp32) ----
  float H00 = 0, H01 = 0, H02 = 0, H11 = 0, H12 = 0, H22 = 0;
  for (int y = 0; y < 8; ++y) {
    const uint8_t* it = border + (y + 1) * 10 + 1;
    for (int x = 0; x < 8; ++x, ++it) {
      const float J0 = __fmul_rn(0.5f, u8diff(it[1], it[-1]));
      const float J1 = __fmul_rn(0.5f, u8diff(it[10], it[-10]));
      H00 = __fadd_rn(H00, __fmul_rn(J0, J0));
      H01 = __fadd_rn(H01, __fmul_rn(J0, J1));
      H02 = __fadd_rn(H02, J0);
      H11 = __fadd_rn(H11, __fmul_rn(J1, J1));
      H12 = __fadd_rn(H12, J1);
      H22 = __fadd_rn(H22, 1.0f);
    }
  }
  // ---- Hinv = H.inverse(): Eigen's fixed-size 3x3 path (cofactors of column 0, determinant, 1/det) ----
  const float m00 = H00, m01 = H01, m02 = H02, m10 = H01, m11 = H11, m12 = H12, m20 = H02, m21 = H12, m22 = H22;
#define COF(i1, j1, i2, j2, i3, j3, i4, j4) __fsub_rn(__fmul_rn(m##i1##j1, m##i2##j2), __fmul_rn(m##i3##j3, m##i4##j4))
  const float c00 = COF(1, 1, 2, 2, 1, 2, 2, 1);  // cofactor<0,0>
  const float c10 = COF(2, 1, 0, 2, 2, 2, 0, 1);  // cofactor<1,0>
  const float c20 = COF(0, 1, 1, 2, 0, 2, 1, 1);  // cofactor<2,0>
  const float det = __fadd_rn(__fadd_rn(__fmul_rn(c00, m00), __fmul_rn(c10, m10)), __fmul_rn(c20, m20));
  const float invdet = __fdiv_rn(1.0f, det);
  const float c01 = COF(1, 2, 2, 0, 1, 0, 2, 2);  // cofactor<0,1>
  const float c11 = COF(2, 2, 0, 0, 2, 0, 0, 2);  // cofactor<1,1>
  const float c21 = COF(0, 2, 1, 0, 0, 0, 1, 2);  // cofactor<2,1>
  const float c02 = COF(1, 0, 2, 1, 1, 1, 2, 0);  // cofactor<0,2>
  const float c12 = COF(2, 0, 0, 1, 2, 1, 0, 0);  // cofactor<1,2>
  const float c22 = COF(0, 0, 1, 1, 0, 1, 1, 0);  // cofactor<2,2>
#undef COF
  // result.row(0) = cofactors_col0 * invdet ; result(1,0)=c01*invdet ; (1,1)=c11 ; (1,2)=c21 ; (2,0)=c02 ; (2,1)=c12 ; (2,2)=c22
  const float I00 = __fmul_rn(c00, invdet), I01 = __fmul_rn(c10, invdet), I02 = __fmul_rn(c20, invdet);
  const float I10 = __fmul_rn(c01, invdet), I11 = __fmul_rn(c11, invdet), I12 = __fmul_rn(c21, invdet);
  const float I20 = __fmul_rn(c02, invdet), I21 = __fmul_rn(c12, invdet), I22 = __fmul_rn(c22, invdet);

  float mean_diff = 0.f;
  const float min_update_squared = (float)(0.03 * 0.03);
  bool converged = false;
  for (int iter = 0; iter < n_iter; ++iter) {
    // Patch::setPosition / isInFrame(halfsize=4) / computeInterpWeights (src/feature.cpp:189-208)
    const float fu = floorf(u), fv = floorf(v);
    const int ui = (int)fu, vi = (int)fv;
    if (ui < 4 || vi < 4 || ui >= cols - 4 || vi >= rows - 4) break;
    const float su = __fsub_rn(u, fu), sv = __fsub_rn(v, fv);
    const float wTL = (float)((1.0 - (double)su) * (1.0 - (double)sv));
    const float wTR = (float)((double)su * (1.0 - (double)sv));
    const float wBL = (float)((1.0 - (double)su) * (double)sv);
    const float wBR = __fmul_rn(su, sv);
    float J0 = 0.f, J1 = 0.f, J2 = 0.f;
    const uint8_t* row = img + (size_t)(vi - 4) * cur_step + (ui - 4);
    const uint8_t* ref_row = ref;
    float top[9], bot[9];
    load_row9(row, top);
#pragma unroll 1
    for (int y = 0; y < 8; ++y, ref_row += ref_step) {
      row += cur_step;
      load_row9(row, bot);
      const uint8_t* itb = border + (y + 1) * 10 + 1;
      const uint8_t* it_ref = ref_row;
#pragma unroll
      for (int x = 0; x < 8; ++x, ++it_ref, ++itb) {
        const float search_pixel =
            __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(wTL, top[x]), __fmul_rn(wTR, top[x + 1])), __fmul_rn(wBL, bot[x])),
                      __fmul_rn(wBR, bot[x + 1]));
        const float res = __fadd_rn(__fsub_rn(search_pixel, u8f(*it_ref)), mean_diff);
        const float dx = __fmul_rn(0.5f, u8diff(itb[1], itb[-1]));
        const float dy = __fmul_rn(0.5f, u8diff(itb[10], itb[-10]));
        J0 = __fsub_rn(J0, __fmul_rn(res, dx));
        J1 = __fsub_rn(J1, __fmul_rn(res, dy));
        J2 = __fsub_rn(J2, res);
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) top[k] = bot[k];
    }
    // update = Hinv * Jres
    const float up0 = __fadd_rn(__fadd_rn(__fmul_rn(I00, J0), __fmul_rn(I01, J1)), __fmul_rn(I02, J2));
    const float up1 = __fadd_rn(__fadd_rn(__fmul_rn(I10, J0), __fmul_rn(I11, J1)), __fmul_rn(I12, J2));
    const float up2 = __fadd_rn(__fadd_rn(__fmul_rn(I20, J0), __fmul_rn(I21, J1)), __fmul_rn(I22, J2));
    u = __fadd_rn(u, up0);
    v = __fadd_rn(v, up1);
    mean_diff = __fadd_rn(mean_diff, up2);
    if (__fadd_rn(__fmul_rn(up0, up0), __fmul_rn(up1, up1)) < min_update_squared) {
      converged = true;
      break;
    }
  }
  return converged;
}

// align1D on one feature (same conventions as align2d_core); d0,d1 = direction, h_inv out.
__device__ __forceinline__ bool align1d_core(const uint8_t* border, const uint8_t* ref, const int ref_step, const uint8_t* img,
                                             const int cur_step, const int cols, const int rows, const int n_iter, const float d0,
                                             const float d1, float& u, float& v, double& h_inv) {
  // directional template derivative (:63-66): J0 = 0.5*(dir0*(I[x+1]-I[x-1]) + dir1*(I[y+1]-I[y-1])) in float, J1 = 1
  auto dv_at = [&](const uint8_t* it) {
    const float gx = __fmul_rn(d0, u8diff(it[1], it[-1]));
    const float gy = __fmul_rn(d1, u8diff(it[10], it[-10]));
    return __fmul_rn(0.5f, __fadd_rn(gx, gy));
  };
  float H00 = 0, H01 = 0, H11 = 0;
  for (int y = 0; y < 8; ++y) {
    const uint8_t* it = border + (y + 1) * 10 + 1;
    for (int x = 0; x < 8; ++x, ++it) {
      const float J0 = dv_at(it);
      H00 = __fadd_rn(H00, __fmul_rn(J0, J0));
      H01 = __fadd_rn(H01, J0);
      H11 = __fadd_rn(H11, 1.0f);
    }
  }
  h_inv = 1.0 / (double)H00 * 8 * 8;  // :75
  // Matrix2f::inverse(): 1/det, (d, -c; -b, a) * invdet
  const float det = __fsub_rn(__fmul_rn(H00, H11), __fmul_rn(H01, H01));
  const float invdet = __fdiv_rn(1.0f, det);
  const float I00 = __fmul_rn(H11, invdet), I10 = __fmul_rn(-H01, invdet);
  const float I01 = __fmul_rn(-H01, invdet), I11 = __fmul_rn(H00, invdet);

  float mean_diff = 0.f;
  const float min_update_squared = (float)(0.03 * 0.03);
  float chi2 = 0.f, up0 = 0.f, up1 = 0.f;
  bool converged = false;
  for (int iter = 0; iter < n_iter; ++iter) {
    const float fu = floorf(u), fv = floorf(v);
    const int ui = (int)fu, vi = (int)fv;
    if (ui < 4 || vi < 4 || ui >= cols - 4 || vi >= rows - 4) break;  // NaN never passes this test (:87-92)
    const float su = __fsub_rn(u, fu), sv = __fsub_rn(v, fv);
    const float wTL = (float)((1.0 - (double)su) * (1.0 - (double)sv));
    const float wTR = (float)((double)su * (1.0 - (double)sv));
    const float wBL = (float)((1.0 - (double)su) * (double)sv);
    const float wBR = __fmul_rn(su, sv);
    float J0 = 0.f, J1 = 0.f, new_chi2 = 0.f;
    const uint8_t* row = img + (size_t)(vi - 4) * cur_step + (ui - 4);
    const uint8_t* ref_row = ref;
    float top[9], bot[9];
    load_row9(row, top);
#pragma unroll 1
    for (int y = 0; y < 8; ++y, ref_row += ref_step) {
      row += cur_step;
      load_row9(row, bot);
      const uint8_t* itb = border + (y + 1) * 10 + 1;
      const uint8_t* it_ref = ref_row;
#pragma unroll
      for (int x = 0; x < 8; ++x, ++it_ref, ++itb) {
        const float search_pixel =
            __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(wTL, top[x]), __fmul_rn(wTR, top[x + 1])), __fmul_rn(wBL, bot[x])),
                      __fmul_rn(wBR, bot[x + 1]));
        const float res = __fadd_rn(__fsub_rn(search_pixel, u8f(*it_ref)), mean_diff);
        J0 = __fsub_rn(J0, __fmul_rn(res, dv_at(itb)));
        J1 = __fsub_rn(J1, res);
        new_chi2 = __fadd_rn(new_chi2, __fmul_rn(res, res));
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) top[k] = bot[k];
    }
    if (iter > 0 && new_chi2 > chi2) {  // :124-132 (the back-off subtracts the raw update, as the reference does)
      u = __fsub_rn(u, up0);
      v = __fsub_rn(v, up1);
      break;
    }
    chi2 = new_chi2;
    up0 = __fadd_rn(__fmul_rn(I00, J0), __fmul_rn(I01, J1));
    up1 = __fadd_rn(__fmul_rn(I10, J0), __fmul_rn(I11, J1));
    u = __fadd_rn(u, __fmul_rn(up0, d0));
    v = __fadd_rn(v, __fmul_rn(up0, d1));
    mean_diff = __fadd_rn(mean_diff, up1);
    if (__fadd_rn(__fmul_rn(up0, up0), __fmul_rn(up1, up1)) < min_update_squared) {
      converged = true;
      break;
    }
  }
  return converged;
}

__global__ void __launch_bounds__(kA2Threads) align2d_kernel(const Align2DArgs a) {
  __shared__ __align__(4) uint8_t s_border[kA2Threads][108];  // 100 used; 27-word pitch (odd) keeps the threads of a warp on distinct banks
  __shared__ __align__(4) uint8_t s_ref[kA2Threads][68];  // 64 used; 17-word pitch (odd): no bank conflicts
  const int tid = threadIdx.x;
  const int i = blockIdx.x * kA2Threads + tid;
  const bool active = i < a.n;
  if (active) {
    const uint32_t* gb = reinterpret_cast<const uint32_t*>(a.ref_patch_with_border + (size_t)i * 100);
    const uint32_t* gr = reinterpret_cast<const uint32_t*>(a.ref_patch + (size_t)i * 64);
    uint32_t* sb = reinterpret_cast<uint32_t*>(s_border[tid]);
    uint32_t* sr = reinterpret_cast<uint32_t*>(s_ref[tid]);
#pragma unroll
    for (int k = 0; k < 25; ++k) sb[k] = gb[k];
#pragma unroll
    for (int k = 0; k < 16; ++k) sr[k] = gr[k];
  }
  if (!active) return;
  const uint8_t* border = s_border[tid];
  const uint8_t* ref = s_ref[tid];
  const int level = a.level[i];
  const int cols = a.width >> level, rows = a.height >> level;
  const int cur_step = (int)a.pitch[level];
  const uint8_t* img = a.img[level] + (size_t)a.image_index[i] * a.stride[level];

  float u = (float)a.px[2 * (size_t)i], v = (float)a.px[2 * (size_t)i + 1];
  const bool converged = align2d_core(border, ref, 8, img, cur_step, cols, rows, a.n_iter, u, v);
  a.out_px[2 * (size_t)i] = (double)u;
  a.out_px[2 * (size_t)i + 1] = (double)v;
  a.out_converged[i] = converged ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------
// feature_alignment::align1D (src/feature_alignment.cpp:40-157): the patch moves along `dir` only
// (edgelets), 1 DoF + mean intensity offset, with the reference's chi2 back-off.  Same layout and
// the same bit-exact fp32 sequencing as align2d_kernel.
__global__ void __launch_bounds__(kA2Threads) align1d_kernel(const Align2DArgs a) {
  __shared__ __align__(4) uint8_t s_border[kA2Threads][108];  // 100 used; 27-word pitch (odd) keeps the threads of a warp on distinct banks
  __shared__ __align__(4) uint8_t s_ref[kA2Threads][68];  // 64 used; 17-word pitch (odd): no bank conflicts
  const int tid = threadIdx.x;
  const int i = blockIdx.x * kA2Threads + tid;
  if (i >= a.n) return;
  {
    const uint32_t* gb = reinterpret_cast<const uint32_t*>(a.ref_patch_with_border + (size_t)i * 100);
    const uint32_t* gr = reinterpret_cast<const uint32_t*>(a.ref_patch + (size_t)i * 64);
    uint32_t* sb = reinterpret_cast<uint32_t*>(s_border[tid]);
    uint32_t* sr = reinterpret_cast<uint32_t*>(s_ref[tid]);
#pragma unroll
    for (int k = 0; k < 25; ++k) sb[k] = gb[k];
#pragma unroll
    for (int k = 0; k < 16; ++k) sr[k] = gr[k];
  }
  const uint8_t* border = s_border[tid];
  const uint8_t* ref = s_ref[tid];
  const int level = a.level[i];
  const int cols = a.width >> level, rows = a.height >> level;
  const int cur_step = (int)a.pitch[level];
  const uint8_t* img = a.img[level] + (size_t)a.image_index[i] * a.stride[level];
  const float d0 = a.dir[2 * (size_t)i], d1 = a.dir[2 * (size_t)i + 1];

  float u = (float)a.px[2 * (size_t)i], v = (float)a.px[2 * (size_t)i + 1];
  double h_inv;
  const bool converged = align1d_core(border, ref, 8, img, cur_step, cols, rows, a.n_iter, d0, d1, u, v, h_inv);
  a.out_h_inv[i] = h_inv;
  a.out_px[2 * (size_t)i] = (double)u;
  a.out_px[2 * (size_t)i + 1] = (double)v;
  a.out_converged[i] = converged ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------
// Shared pieces of Matcher::findMatchDirect and Matcher::findEpipolarMatchDirect.  The double-precision geometry
// is written with explicit round-to-nearest intrinsics (exact_math.cuh) so that the compiler cannot contract a*b+c
// into an FMA: A_cur_ref, the search level and every byte of the warped patch are bit-identical to the scalar code.
struct CamP {
  double fx, fy, cx, cy;
  int width, height;
};
__device__ __forceinline__ V3 cam2world(const CamP& c, double u, double v) {  // PinholeCamera::cam2world, undistorted, normalized()
  const V3 xyz{DD(DS(u, c.cx), c.fx), DD(DS(v, c.cy), c.fy), 1.0};
  const double n = v_norm(xyz);
  return V3{DD(xyz.x, n), DD(xyz.y, n), DD(xyz.z, n)};
}
__device__ __forceinline__ void world2cam(const CamP& c, V3 p, double& u, double& v) {  // world2cam(project2d(xyz))
  u = DA(DM(c.fx, DD(p.x, p.z)), c.cx);
  v = DA(DM(c.fy, DD(p.y, p.z)), c.cy);
}
__device__ __forceinline__ bool cam_in_frame(const CamP& c, int ox, int oy, int b, int level) {  // AbstractCamera::isInFrame(obs, b, level)
  return ox >= b && ox < c.width / (1 << level) - b && oy >= b && oy < c.height / (1 << level) - b;
}
// double -> int as the x86 cvttsd2si the reference compiles to: out-of-range and NaN give INT_MIN
__device__ __forceinline__ int d2i_x86(double q) { return (q >= -2147483648.0 && q < 2147483648.0) ? (int)q : (-2147483647 - 1); }

// warp::getWarpMatrixAffine (src/matcher.cpp:42-71)
__device__ __forceinline__ void warp_matrix_affine(const CamP& cam, double px_ref0, double px_ref1, V3 f_ref, double depth_ref,
                                                   const Pose& T_cur_ref, int level_ref, double& A00, double& A01, double& A10,
                                                   double& A11) {
  const V3 xyz_ref = v_scale(f_ref, depth_ref);
  const double scale_ref = (double)(1 << level_ref);
  const double step = DM(5.0, scale_ref), zero = DM(0.0, scale_ref);
  V3 xyz_du = cam2world(cam, DA(px_ref0, step), DA(px_ref1, zero));
  V3 xyz_dv = cam2world(cam, DA(px_ref0, zero), DA(px_ref1, step));
  xyz_du = v_scale(xyz_du, DD(xyz_ref.z, xyz_du.z));
  xyz_dv = v_scale(xyz_dv, DD(xyz_ref.z, xyz_dv.z));
  double pc0, pc1, pu0, pu1, pv0, pv1;
  world2cam(cam, pose_act(T_cur_ref, xyz_ref), pc0, pc1);
  world2cam(cam, pose_act(T_cur_ref, xyz_du), pu0, pu1);
  world2cam(cam, pose_act(T_cur_ref, xyz_dv), pv0, pv1);
  A00 = DD(DS(pu0, pc0), 5.0), A10 = DD(DS(pu1, pc1), 5.0);
  A01 = DD(DS(pv0, pc0), 5.0), A11 = DD(DS(pv1, pc1), 5.0);
}
// warp::getBestSearchLevel (:73-87)
__device__ __forceinline__ int best_search_level(double det, int max_level) {
  int search_level = 0;
  double D = det;
  while (D > 3.0 && search_level < max_level) {
    search_level += 1;
    D = DM(D, 0.25);
  }
  return search_level;
}
// warp::warpAffine with halfpatch_size 5 (:89-133, vk::interpolateMat_8u) into a 10x10 patch with border
__device__ __forceinline__ void warp_affine_patch(double A00, double A01, double A10, double A11, double det, const uint8_t* img,
                                                  int stride, int cols, int rows, double px_ref0, double px_ref1, int level_ref,
                                                  int search_level, uint8_t* border) {
  const double invdet = DD(1.0, det);
  const float R00 = (float)DM(A11, invdet), R10 = (float)DM(-A10, invdet);
  const float R01 = (float)DM(-A01, invdet), R11 = (float)DM(A00, invdet);
  const bool bad = isnan(R00);  // "Affine warp is NaN": the reference leaves the (zeroed) patch untouched
  const float fs = (float)(1 << level_ref);
  const float pr0 = __fdiv_rn((float)px_ref0, fs), pr1 = __fdiv_rn((float)px_ref1, fs);
  const float ss = (float)(1 << search_level);
  const float xmax = (float)(cols - 1), ymax = (float)(rows - 1);
  for (int y = 0; y < 10; ++y) {
    const float p1 = __fmul_rn((float)(y - 5), ss);
    for (int x = 0; x < 10; ++x) {
      uint8_t val = 0;
      if (!bad) {
        const float p0 = __fmul_rn((float)(x - 5), ss);
        const float q0 = __fadd_rn(__fadd_rn(__fmul_rn(R00, p0), __fmul_rn(R01, p1)), pr0);
        const float q1 = __fadd_rn(__fadd_rn(__fmul_rn(R10, p0), __fmul_rn(R11, p1)), pr1);
        if (!(q0 < 0 || q1 < 0 || q0 >= xmax || q1 >= ymax)) {
          const float fx = floorf(q0), fy = floorf(q1);
          const int ix = (int)fx, iy = (int)fy;
          const float sx = __fsub_rn(q0, fx), sy = __fsub_rn(q1, fy);
          const float w00 = __fmul_rn(__fsub_rn(1.0f, sx), __fsub_rn(1.0f, sy));
          const float w01 = __fmul_rn(__fsub_rn(1.0f, sx), sy);
          const float w10 = __fmul_rn(sx, __fsub_rn(1.0f, sy));
          const float w11 = __fsub_rn(__fsub_rn(__fsub_rn(1.0f, w00), w01), w10);
          const uint8_t* ptr = img + (size_t)iy * stride + ix;
          const float I = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w00, u8f(ptr[0])), __fmul_rn(w01, u8f(ptr[stride]))),
                                              __fmul_rn(w10, u8f(ptr[1]))),
                                    __fmul_rn(w11, u8f(ptr[stride + 1])));
          val = (uint8_t)I;
        }
      }
      border[y * 10 + x] = val;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Matcher::findMatchDirect(const Point&, const Frame&, Vector2d&) after getCloseViewObs (src/matcher.cpp:159-211):
// in-frame test, affine warp, search level, warped patch, align2D / align1D at the search level.  One thread per
// candidate; the refined position is bit-identical to the reference's scalar code.
__global__ void __launch_bounds__(kA2Threads) match_direct_kernel(const MatchArgs a) {
  __shared__ __align__(4) uint8_t s_border[kA2Threads][108];  // 100 used; 27-word pitch (odd) keeps the threads of a warp on distinct banks
  const int tid = threadIdx.x;
  const int i = blockIdx.x * kA2Threads + tid;
  if (i >= a.n) return;
  const size_t I = (size_t)i;
  const CamP cam{a.fx, a.fy, a.cx, a.cy, a.width, a.height};
  const double px_ref0 = a.ref_px[2 * I], px_ref1 = a.ref_px[2 * I + 1];
  const int level_ref = a.ref_level[i];
  const int r = a.ref_index[i], c = a.cur_index[i];
  a.out_px[2 * I] = a.px_cur[2 * I];
  a.out_px[2 * I + 1] = a.px_cur[2 * I + 1];
  a.out_success[i] = 0;
  a.out_level[i] = -1;
  // :169-171  cam.isInFrame(px.cast<int>() / (1 << level), halfpatch_size_ + 2, level)
  if (!cam_in_frame(cam, (int)px_ref0 / (1 << level_ref), (int)px_ref1 / (1 << level_ref), 6, level_ref)) return;
  const Pose T_w_ref = pose_inverse(pose_load(a.T_ref_w + 7 * (size_t)r));
  const Pose T_cur_ref = pose_mul(pose_load(a.T_cur_w + 7 * (size_t)c), T_w_ref);
  const V3 pos{a.pos[3 * I], a.pos[3 * I + 1], a.pos[3 * I + 2]};
  const V3 f_ref{a.ref_f[3 * I], a.ref_f[3 * I + 1], a.ref_f[3 * I + 2]};
  const double depth_ref = v_norm(v_sub(T_w_ref.t, pos));
  double A00, A01, A10, A11;
  warp_matrix_affine(cam, px_ref0, px_ref1, f_ref, depth_ref, T_cur_ref, level_ref, A00, A01, A10, A11);
  const double det = DS(DM(A00, A11), DM(A10, A01));
  const int search_level = best_search_level(det, a.n_pyr_levels - 1);
  a.out_level[i] = search_level;
  if (a.out_A) a.out_A[4 * I] = A00, a.out_A[4 * I + 1] = A01, a.out_A[4 * I + 2] = A10, a.out_A[4 * I + 3] = A11;
  uint8_t* border = s_border[tid];
  warp_affine_patch(A00, A01, A10, A11, det, a.ref_img[level_ref] + (size_t)r * a.ref_stride[level_ref], (int)a.ref_pitch[level_ref],
                    a.width >> level_ref, a.height >> level_ref, px_ref0, px_ref1, level_ref, search_level, border);
  // ---- align at the search level; the 8x8 reference patch is the interior of the border patch ----
  const double scale = (double)(1 << search_level);
  float u = (float)DD(a.px_cur[2 * I], scale), v = (float)DD(a.px_cur[2 * I + 1], scale);
  const uint8_t* cur = a.cur_img[search_level] + (size_t)c * a.cur_stride[search_level];
  const int ccols = a.width >> search_level, crows = a.height >> search_level;
  const int cur_step = (int)a.cur_pitch[search_level];
  const uint8_t* ref = border + 11;
  bool ok;
  if (a.is_edgelet && a.is_edgelet[i]) {
    const double g0 = a.ref_grad[2 * I], g1 = a.ref_grad[2 * I + 1];
    double d0 = DA(DM(A00, g0), DM(A01, g1)), d1 = DA(DM(A10, g0), DM(A11, g1));
    const double n = __dsqrt_rn(DA(DM(d0, d0), DM(d1, d1)));
    d0 = DD(d0, n), d1 = DD(d1, n);
    double h_inv;
    ok = align1d_core(border, ref, 10, cur, cur_step, ccols, crows, a.n_iter, (float)d0, (float)d1, u, v, h_inv);
  } else {
    ok = align2d_core(border, ref, 10, cur, cur_step, ccols, crows, a.n_iter, u, v);
  }
  a.out_px[2 * I] = DM((double)u, scale);
  a.out_px[2 * I + 1] = DM((double)v, scale);
  a.out_success[i] = ok ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------
// Depth-filter point-seed update: the body of DepthFilter::updatePointSeeds (src/depth_filter.cpp:270-365) with
// Matcher::findEpipolarMatchDirect (src/matcher.cpp:277-420), depthFromTriangulation (:135-146), the ZMSSD patch score
// (rpg_vikit patch_score.h; packed-byte dot products, exact integer arithmetic), DepthFilter::computeTau (:568-584)
// and DepthFilter::updatePointSeed (:489-512).  One thread per seed.  Everything up to and including the
// triangulated depth z is bit-identical to the scalar code; computeTau and the Gaussian pdf go through
// acos/sin/atan/expf, whose last bit differs between libm implementations, so the updated seed agrees to float
// round-off (tests/test_depth_filter.py states the tolerance).
__device__ __forceinline__ bool depth_from_triangulation(const Pose& T, V3 f_ref, V3 f_cur, double& depth) {
  double R[3][3];
  q_to_matrix(T.q, R);
  double A0[3], A1[3] = {f_cur.x, f_cur.y, f_cur.z};
#pragma unroll
  for (int i = 0; i < 3; ++i) A0[i] = DA(DA(DM(R[i][0], f_ref.x), DM(R[i][1], f_ref.y)), DM(R[i][2], f_ref.z));
  const double a00 = DA(DA(DM(A0[0], A0[0]), DM(A0[1], A0[1])), DM(A0[2], A0[2]));
  const double a01 = DA(DA(DM(A0[0], A1[0]), DM(A0[1], A1[1])), DM(A0[2], A1[2]));
  const double a10 = DA(DA(DM(A1[0], A0[0]), DM(A1[1], A0[1])), DM(A1[2], A0[2]));
  const double a11 = DA(DA(DM(A1[0], A1[0]), DM(A1[1], A1[1])), DM(A1[2], A1[2]));
  const double det = DS(DM(a00, a11), DM(a10, a01));
  if (det < 0.000001) return false;
  const double invdet = DD(1.0, det);
  const double M00 = -DM(a11, invdet), M01 = -DM(-a01, invdet);  // -(AtA.inverse()), first row
  const double N0 = DA(DM(M00, A0[0]), DM(M01, A1[0])), N1 = DA(DM(M00, A0[1]), DM(M01, A1[1])), N2 = DA(DM(M00, A0[2]), DM(M01, A1[2]));
  depth = fabs(DA(DA(DM(N0, T.t.x), DM(N1, T.t.y)), DM(N2, T.t.z)));
  return true;
}

// Matcher::findEpipolarMatchDirect (src/matcher.cpp:277-420) for one seed; segment_endpoint = true gives
// Matcher::findEpipolarMatchDirectSegmentEndpoint (:420-588): NaN depth ranges and NaN / infinite epipolar lengths are
// rejected up front and there is no edgelet pre-selection.  Returns false where the reference returns false; on success z is
// the triangulated depth and (pxc0, pxc1) the matched position (also set, as Matcher::px_cur_, on some failure paths).
//
// The match runs in three phases so that the one long loop in it — up to max_epi_search_steps ZMSSD evaluations along the
// epipolar line, whose count differs from seed to seed by orders of magnitude — is not walked by one thread while the 31
// other lanes of its warp wait for the longest line among them:
//   epi_begin   (per thread)   everything up to the search: epipolar segment, affine warp, edgelet gate, warped patch, the
//                              short-segment shortcut (direct alignment); hands out the search description;
//   warp_epipolar_search (all 32 lanes, one seed at a time)  32 consecutive steps per pass, one per lane;
//   epi_end     (per thread)   sub-pixel refinement at the best step and triangulation.
// The search is bit-identical to the sequential loop: uv is advanced by repeated addition exactly as the loop does (lane j
// applies j additions to the pass's first value), the "same pixel as the previous step" test is a comparison with the
// neighbouring lane, scores are integers, and ties go to the lowest step as `zmssd < zmssd_best` does.
struct EpiCtx {
  double scale, uv0, uv1, step0, step1, uvb0, uvb1;
  const uint8_t* cur;
  int ccols, crows, cur_step, search_level, zmssd_best;
  unsigned int n_iters;
  float dir0, dir1;
  uint32_t refw[16], sumA, sumAA;
};
enum { EPI_FALSE = 0, EPI_TRUE = 1, EPI_SEARCH = 2 };

// sub-pixel refinement at the search level followed by triangulation (matcher.cpp:326-342, :396-413)
__device__ __forceinline__ bool epi_refine(const SeedArgs& a, const CamP& cam, const EpiCtx& E, const uint8_t* border, const Pose& T_cur_ref,
                                           const V3 f, const double start0, const double start1, double& z, double& pxc0, double& pxc1) {
  float u = (float)DD(start0, E.scale), v = (float)DD(start1, E.scale);
  const uint8_t* ref = border + 11;
  bool res;
  if (a.align_1d) {
    double h_inv;
    res = align1d_core(border, ref, 10, E.cur, E.cur_step, E.ccols, E.crows, a.n_iter, E.dir0, E.dir1, u, v, h_inv);
  } else {
    res = align2d_core(border, ref, 10, E.cur, E.cur_step, E.ccols, E.crows, a.n_iter, u, v);
  }
  if (!res) return false;
  pxc0 = DM((double)u, E.scale), pxc1 = DM((double)v, E.scale);
  return depth_from_triangulation(T_cur_ref, f, cam2world(cam, pxc0, pxc1), z);
}

__device__ __forceinline__ int epi_begin(const SeedArgs& a, const CamP& cam, const int i, const int r, const int c, const Pose& T_cur_ref,
                                         const double px_ref0, const double px_ref1, const V3 f, const int level_ref, const double d_estimate,
                                         const double d_min, const double d_max, const bool segment_endpoint, uint8_t* border, EpiCtx& E,
                                         double& z, double& pxc0, double& pxc1) {
  const size_t I = (size_t)i;
  if (segment_endpoint && (isnan(d_min) || isnan(d_max))) return EPI_FALSE;  // matcher.cpp:434-438
  const V3 pa = pose_act(T_cur_ref, v_scale(f, d_min)), pb = pose_act(T_cur_ref, v_scale(f, d_max));
  const double Au = DD(pa.x, pa.z), Av = DD(pa.y, pa.z), Bu = DD(pb.x, pb.z), Bv = DD(pb.y, pb.z);
  const double epi0 = DS(Au, Bu), epi1 = DS(Av, Bv);
  double A00, A01, A10, A11;
  warp_matrix_affine(cam, px_ref0, px_ref1, f, d_estimate, T_cur_ref, level_ref, A00, A01, A10, A11);
  if (!segment_endpoint && a.is_edgelet && a.is_edgelet[i] && a.edgelet_filtering) {  // :300-310
    const double g0 = a.ref_grad[2 * I], g1 = a.ref_grad[2 * I + 1];
    double c0 = DA(DM(A00, g0), DM(A01, g1)), c1 = DA(DM(A10, g0), DM(A11, g1));
    const double nc = __dsqrt_rn(DA(DM(c0, c0), DM(c1, c1)));
    c0 = DD(c0, nc), c1 = DD(c1, nc);
    const double ne = __dsqrt_rn(DA(DM(epi0, epi0), DM(epi1, epi1)));
    const double cosangle = fabs(DA(DM(c0, DD(epi0, ne)), DM(c1, DD(epi1, ne))));
    if (cosangle < a.edgelet_max_angle) return EPI_FALSE;
  }
  const double det = DS(DM(A00, A11), DM(A10, A01));
  const int search_level = best_search_level(det, a.n_pyr_levels - 1);
  const double pxA0 = DA(DM(cam.fx, Au), cam.cx), pxA1 = DA(DM(cam.fy, Av), cam.cy);
  const double pxB0 = DA(DM(cam.fx, Bu), cam.cx), pxB1 = DA(DM(cam.fy, Bv), cam.cy);
  const double dAB0 = DS(pxA0, pxB0), dAB1 = DS(pxA1, pxB1);
  const double scale = (double)(1 << search_level);
  const double epi_length = DD(__dsqrt_rn(DA(DM(dAB0, dAB0), DM(dAB1, dAB1))), scale);
  if (segment_endpoint && (isnan(epi_length) || isinf(epi_length))) return EPI_FALSE;  // matcher.cpp:481-485
  warp_affine_patch(A00, A01, A10, A11, det, a.ref_img[level_ref] + (size_t)r * a.ref_stride[level_ref], (int)a.ref_pitch[level_ref],
                    a.width >> level_ref, a.height >> level_ref, px_ref0, px_ref1, level_ref, search_level, border);
  E.scale = scale, E.search_level = search_level;
  E.cur = a.cur_img[search_level] + (size_t)c * a.cur_stride[search_level];
  E.ccols = a.width >> search_level, E.crows = a.height >> search_level;
  E.cur_step = (int)a.cur_pitch[search_level];
  {  // (px_A - px_B).cast<float>().normalized()
    const float fx_ = (float)dAB0, fy_ = (float)dAB1;
    const float n = __fsqrt_rn(__fadd_rn(__fmul_rn(fx_, fx_), __fmul_rn(fy_, fy_)));
    E.dir0 = __fdiv_rn(fx_, n), E.dir1 = __fdiv_rn(fy_, n);
  }
  const float elf = fabsf((float)epi_length);
  if (epi_length < 2.0 && (segment_endpoint || (!isnan(elf) && !isinf(elf)))) {
    pxc0 = DD(DA(pxA0, pxB0), 2.0), pxc1 = DD(DA(pxA1, pxB1), 2.0);
    return epi_refine(a, cam, E, border, T_cur_ref, f, pxc0, pxc1, z, pxc0, pxc1) ? EPI_TRUE : EPI_FALSE;
  }
  const double qsteps = DD(epi_length, 0.7);
  if (!(qsteps < 9.0e18)) return EPI_FALSE;  // NaN / beyond size_t: the x86 conversion yields 2^63, i.e. "too many steps"
  const unsigned long long n_steps = (unsigned long long)qsteps;
  if (n_steps > (unsigned long long)a.max_epi_search_steps) return EPI_FALSE;
  E.step0 = DD(epi0, (double)n_steps), E.step1 = DD(epi1, (double)n_steps);
  // ZMSSD of the warped 8x8 patch against the integer-pixel patches along the epipolar line (:354-391)
  const uint8_t* ref = border + 11;
  uint32_t sumA = 0, sumAA = 0;
#pragma unroll
  for (int y = 0; y < 8; ++y) {
    const uint8_t* p = ref + y * 10;
    const uint32_t w0 = p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24);
    const uint32_t w1 = p[4] | (p[5] << 8) | (p[6] << 16) | ((uint32_t)p[7] << 24);
    E.refw[2 * y] = w0, E.refw[2 * y + 1] = w1;
    sumA = __dp4a(w0, 0x01010101u, sumA), sumA = __dp4a(w1, 0x01010101u, sumA);
    sumAA = __dp4a(w0, w0, sumAA), sumAA = __dp4a(w1, w1, sumAA);
  }
  E.sumA = sumA, E.sumAA = sumAA;
  E.uv0 = DS(Bu, E.step0), E.uv1 = DS(Bv, E.step1);
  E.n_iters = (unsigned int)n_steps + 1u;
  E.zmssd_best = 2000 * 64, E.uvb0 = 0.0, E.uvb1 = 0.0;
  return EPI_SEARCH;
}

// ZMSSD of the reference words against the 8x8 patch whose top-left pixel is p (any alignment)
__device__ __forceinline__ int zmssd_at(const uint8_t* p, const int cur_step, const uint32_t (&refw)[16], const uint32_t sumA, const uint32_t sumAA) {
  const uintptr_t addr = reinterpret_cast<uintptr_t>(p);
  const uint32_t sh = static_cast<uint32_t>(addr & 3) * 8;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(addr & ~static_cast<uintptr_t>(3));
  uint32_t sumB = 0, sumBB = 0, sumAB = 0;
#pragma unroll
  for (int y = 0; y < 8; ++y) {
    const uint32_t* wr = w + (size_t)y * (cur_step >> 2);
    const uint32_t x0 = __ldg(wr), x1 = __ldg(wr + 1), x2 = __ldg(wr + 2);
    const uint32_t c0 = __funnelshift_r(x0, x1, sh), c1 = __funnelshift_r(x1, x2, sh);
    sumB = __dp4a(c0, 0x01010101u, sumB), sumB = __dp4a(c1, 0x01010101u, sumB);
    sumBB = __dp4a(c0, c0, sumBB), sumBB = __dp4a(c1, c1, sumBB);
    sumAB = __dp4a(c0, refw[2 * y], sumAB), sumAB = __dp4a(c1, refw[2 * y + 1], sumAB);
  }
  const int iA = (int)sumA, iAA = (int)sumAA, iB = (int)sumB, iBB = (int)sumBB, iAB = (int)sumAB;
  return iAA - 2 * iAB + iBB - (iA * iA - 2 * iA * iB + iB * iB) / 64;
}

#ifdef PLSVO_SERIAL_EPI_SEARCH
// A/B build: the search of a seed walked by its own thread, step by step (the scalar loop of matcher.cpp:354-391)
__device__ __forceinline__ void warp_epipolar_search(const CamP& cam, const bool mine, EpiCtx& E, const unsigned int) {
  if (!mine) return;
  double uv0 = E.uv0, uv1 = E.uv1;
  int last0 = 0, last1 = 0;
  for (unsigned int k = 0; k < E.n_iters; ++k, uv0 = DA(uv0, E.step0), uv1 = DA(uv1, E.step1)) {
    const double px0 = DA(DM(cam.fx, uv0), cam.cx), px1 = DA(DM(cam.fy, uv1), cam.cy);
    const int pxi0 = d2i_x86(DA(DD(px0, E.scale), 0.5)), pxi1 = d2i_x86(DA(DD(px1, E.scale), 0.5));
    if (pxi0 == last0 && pxi1 == last1) continue;
    last0 = pxi0, last1 = pxi1;
    if (!cam_in_frame(cam, pxi0, pxi1, 8, E.search_level)) continue;
    const int zmssd = zmssd_at(E.cur + (size_t)(pxi1 - 4) * E.cur_step + (pxi0 - 4), E.cur_step, E.refw, E.sumA, E.sumAA);
    if (zmssd < E.zmssd_best) E.zmssd_best = zmssd, E.uvb0 = uv0, E.uvb1 = uv1;
  }
}
#else
__device__ __forceinline__ double shfl_d(const double v, const int src) { return __shfl_sync(0xffffffffu, v, src); }
// Every lane of the warp calls this; `mine` says whether the lane's own seed needs a search (described by its E).
// Hybrid schedule: the first `serial_steps` steps of every search are walked by the seed's own thread (all lanes busy side
// by side: most epipolar segments are that short), what lies beyond is taken over by the whole warp, 32 steps per pass,
// seed after seed — so a warp never waits for one long line with 31 lanes idle.  serial_steps = 0 when a warp holds few seeds.
__device__ __forceinline__ void warp_epipolar_search(const CamP& cam, const bool mine, EpiCtx& E, const unsigned int serial_steps) {
  const int lane = threadIdx.x & 31;
  // ---- own thread: steps [0, min(n, serial_steps)) ----
  double uv0 = E.uv0, uv1 = E.uv1;
  int last0 = 0, last1 = 0;  // `last_checked_pxi` starts at (0, 0)
  unsigned int k_done = 0;
  if (mine) {
    const unsigned int n_own = E.n_iters < serial_steps ? E.n_iters : serial_steps;
    for (; k_done < n_own; ++k_done, uv0 = DA(uv0, E.step0), uv1 = DA(uv1, E.step1)) {
      const double px0 = DA(DM(cam.fx, uv0), cam.cx), px1 = DA(DM(cam.fy, uv1), cam.cy);
      const int pxi0 = d2i_x86(DA(DD(px0, E.scale), 0.5)), pxi1 = d2i_x86(DA(DD(px1, E.scale), 0.5));
      if (pxi0 == last0 && pxi1 == last1) continue;
      last0 = pxi0, last1 = pxi1;
      if (!cam_in_frame(cam, pxi0, pxi1, 8, E.search_level)) continue;
      const int zmssd = zmssd_at(E.cur + (size_t)(pxi1 - 4) * E.cur_step + (pxi0 - 4), E.cur_step, E.refw, E.sumA, E.sumAA);
      if (zmssd < E.zmssd_best) E.zmssd_best = zmssd, E.uvb0 = uv0, E.uvb1 = uv1;
    }
  }
  // ---- whole warp: the steps beyond, one seed at a time ----
  unsigned int todo = __ballot_sync(0xffffffffu, mine && k_done < E.n_iters);
  while (todo) {
    const int s = __ffs(todo) - 1;
    todo &= todo - 1;
    // the owner's search state, broadcast
    const double st0 = shfl_d(E.step0, s), st1 = shfl_d(E.step1, s), scale = shfl_d(E.scale, s);
    double base0 = shfl_d(uv0, s), base1 = shfl_d(uv1, s);
    const unsigned int n = __shfl_sync(0xffffffffu, E.n_iters, s), k_first = __shfl_sync(0xffffffffu, k_done, s);
    const int cur_step = __shfl_sync(0xffffffffu, E.cur_step, s), level = __shfl_sync(0xffffffffu, E.search_level, s);
    const uint8_t* cur = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(E.cur), s));
    const uint32_t sumA = __shfl_sync(0xffffffffu, E.sumA, s), sumAA = __shfl_sync(0xffffffffu, E.sumAA, s);
    uint32_t rw[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) rw[j] = __shfl_sync(0xffffffffu, E.refw[j], s);
    int best = __shfl_sync(0xffffffffu, E.zmssd_best, s);
    int prev0 = __shfl_sync(0xffffffffu, last0, s), prev1 = __shfl_sync(0xffffffffu, last1, s);
    double bu0 = shfl_d(E.uvb0, s), bu1 = shfl_d(E.uvb1, s);
    for (unsigned int k0 = k_first; k0 < n; k0 += 32) {
      // uv of step k0 + lane: the pass's first value advanced `lane` times, one rounded addition at a time
      double u0 = base0, u1 = base1;
#pragma unroll 1
      for (int t = 0; t < 31; ++t)
        if (t < lane) u0 = DA(u0, st0), u1 = DA(u1, st1);
      base0 = DA(shfl_d(u0, 31), st0), base1 = DA(shfl_d(u1, 31), st1);
      const double px0 = DA(DM(cam.fx, u0), cam.cx), px1 = DA(DM(cam.fy, u1), cam.cy);
      const int pxi0 = d2i_x86(DA(DD(px0, scale), 0.5)), pxi1 = d2i_x86(DA(DD(px1, scale), 0.5));
      int q0 = __shfl_up_sync(0xffffffffu, pxi0, 1), q1 = __shfl_up_sync(0xffffffffu, pxi1, 1);
      if (lane == 0) q0 = prev0, q1 = prev1;
      prev0 = __shfl_sync(0xffffffffu, pxi0, 31), prev1 = __shfl_sync(0xffffffffu, pxi1, 31);
      const bool eval = (k0 + (unsigned int)lane < n) && !(pxi0 == q0 && pxi1 == q1) && cam_in_frame(cam, pxi0, pxi1, 8, level);
      int zm = 0x7fffffff;
      if (eval) zm = zmssd_at(cur + (size_t)(pxi1 - 4) * cur_step + (pxi0 - 4), cur_step, rw, sumA, sumAA);
      // lowest score of the pass, ties to the lowest lane (= the lowest step, as `zmssd < zmssd_best` keeps the first)
      int zmin = zm, lmin = lane;
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) {
        const int oz = __shfl_xor_sync(0xffffffffu, zmin, d), ol = __shfl_xor_sync(0xffffffffu, lmin, d);
        if (oz < zmin || (oz == zmin && ol < lmin)) zmin = oz, lmin = ol;
      }
      if (zmin < best) best = zmin, bu0 = shfl_d(u0, lmin), bu1 = shfl_d(u1, lmin);
    }
    if (lane == s) E.zmssd_best = best, E.uvb0 = bu0, E.uvb1 = bu1;
  }
}
#endif

// after the search (matcher.cpp:393-413)
__device__ __forceinline__ bool epi_end(const SeedArgs& a, const CamP& cam, const EpiCtx& E, const uint8_t* border, const Pose& T_cur_ref,
                                        const V3 f, double& z, double& pxc0, double& pxc1) {
  if (E.zmssd_best < 2000 * 64) {
    pxc0 = DA(DM(cam.fx, E.uvb0), cam.cx), pxc1 = DA(DM(cam.fy, E.uvb1), cam.cy);
    if (a.subpix_refinement) {
      return epi_refine(a, cam, E, border, T_cur_ref, f, pxc0, pxc1, z, pxc0, pxc1);
    } else {
      const V3 u3{E.uvb0, E.uvb1, 1.0};
      const double n = v_norm(u3);
      return depth_from_triangulation(T_cur_ref, f, V3{DD(u3.x, n), DD(u3.y, n), DD(u3.z, n)}, z);
    }
  }
  return false;
}

// computeTau (src/depth_filter.cpp:568-584) and the measurement (x = 1/z, tau2) handed to the Bayesian update (:319-323).
// acos / sin / atan are libm calls: the result agrees with the scalar code to double round-off, not bit for bit.
__device__ __forceinline__ void seed_measurement(const CamP& cam, const Pose& T_ref_cur, const V3 f, const double z, float& x, float& tau2) {
  const double px_error_angle = atan(1.0 / (2.0 * fabs(cam.fx))) * 2.0;
  const V3 t = T_ref_cur.t;
  const V3 av = v_sub(v_scale(f, z), t);
  const double t_norm = v_norm(t), a_norm = v_norm(av);
  const double alpha = acos(DD(DA(DA(DM(f.x, t.x), DM(f.y, t.y)), DM(f.z, t.z)), t_norm));
  const double beta = acos(DD(DA(DA(DM(av.x, -t.x), DM(av.y, -t.y)), DM(av.z, -t.z)), DM(t_norm, a_norm)));
  const double beta_plus = DA(beta, px_error_angle);
  const double gamma_plus = DS(DS(3.14159265, alpha), beta_plus);  // plsvo::PI
  const double z_plus = DD(DM(t_norm, sin(beta_plus)), sin(gamma_plus));
  const double tau = DS(z_plus, z);
  const double zmt = DS(z, tau);
  const double lo = (0.0000001 < zmt) ? zmt : 0.0000001;  // std::max(0.0000001, z - tau)
  const double tau_inverse = DM(0.5, DS(DD(1.0, lo), DD(1.0, DA(z, tau))));
  x = (float)DD(1.0, z);
  tau2 = (float)DM(tau_inverse, tau_inverse);
}
// One inverse-depth Gaussian's share of DepthFilter::updatePointSeed / updateLineSeed (src/depth_filter.cpp:489-512,
// :524-556): the new mean and variance and the moments f, e of the Beta update, with the reference's float / double mixing.
__device__ __forceinline__ void gaussian_beta_update(const float x, const float tau2, const float norm_scale, const float sa, const float sb,
                                                     const float z_range, float& smu, float& ssig, float& fq, float& eq) {
  float ex = __fsub_rn(x, smu);
  ex = __fmul_rn(ex, -ex);
  ex = __fdiv_rn(ex, __fmul_rn(__fmul_rn(2.0f, norm_scale), norm_scale));
  float pdf = expf(ex);
  pdf = __fdiv_rn(pdf, __fmul_rn(norm_scale, __fsqrt_rn(__fmul_rn(2.0f, 3.14159274101257324f))));
  if (isinf(x)) pdf = 0.0f;
  const float s2 = (float)DD(1.0, DA(DD(1.0, (double)ssig), DD(1.0, (double)tau2)));
  const float m = __fmul_rn(s2, __fadd_rn(__fdiv_rn(smu, ssig), __fdiv_rn(x, tau2)));
  const float ab = __fadd_rn(sa, sb);
  float C1 = __fmul_rn(__fdiv_rn(sa, ab), pdf);
  float C2 = (float)DD(DM((double)__fdiv_rn(sb, ab), 1.0), (double)z_range);
  const float nc = __fadd_rn(C1, C2);
  C1 = __fdiv_rn(C1, nc), C2 = __fdiv_rn(C2, nc);
  const double ab1 = DA((double)ab, 1.0), ab2 = DA((double)ab, 2.0);
  fq = (float)DA(DD(DM((double)C1, DA((double)sa, 1.0)), ab1), DD((double)__fmul_rn(C2, sa), ab1));
  const float abf1 = __fadd_rn(ab, 1.0f), abf2 = __fadd_rn(ab, 2.0f);
  eq = (float)DA(DD(DM(DM((double)C1, DA((double)sa, 1.0)), DA((double)sa, 2.0)), DM(ab1, ab2)),
                 (double)__fdiv_rn(__fmul_rn(__fmul_rn(C2, sa), __fadd_rn(sa, 1.0f)), __fmul_rn(abf1, abf2)));
  const float mu_new = __fadd_rn(__fmul_rn(C1, m), __fmul_rn(C2, smu));
  ssig = __fsub_rn(__fadd_rn(__fmul_rn(C1, __fadd_rn(s2, __fmul_rn(m, m))), __fmul_rn(C2, __fadd_rn(ssig, __fmul_rn(smu, smu)))),
                   __fmul_rn(mu_new, mu_new));
  smu = mu_new;
}
// visibility of a seed hypothesis in the current frame (depth_filter.cpp:291-304)
__device__ __forceinline__ bool seed_visible(const CamP& cam, const Pose& T_cur_ref_vis, const V3 f, const float mu) {
  const V3 xyz_f = pose_act(T_cur_ref_vis, v_scale(f, DD(1.0, (double)mu)));
  if (xyz_f.z < 0.0) return false;
  double u, v;
  world2cam(cam, xyz_f, u, v);
  const int ox = d2i_x86(u), oy = d2i_x86(v);
  return ox >= 0 && ox < cam.width && oy >= 0 && oy < cam.height;
}
// inverse-depth search range of a Gaussian (depth_filter.cpp:307-311)
__device__ __forceinline__ void depth_range(const float mu, const float sigma2, double& d_estimate, double& d_min, double& d_max) {
  const float sq = __fsqrt_rn(sigma2);
  const float z_inv_min = __fadd_rn(mu, sq);
  const float dmin = __fsub_rn(mu, sq);
  const float z_inv_max = (dmin < 0.00000001f) ? 0.00000001f : dmin;  // std::max(dmin, 1e-8f)
  d_estimate = DD(1.0, (double)mu), d_min = DD(1.0, (double)z_inv_min), d_max = DD(1.0, (double)z_inv_max);
}

// a.spw seeds per warp (lanes >= spw idle outside the search): 32 when the batch fills the GPU, fewer for the few hundred
// seeds of one frame, so that their searches run side by side instead of one after the other inside a warp
__global__ void __launch_bounds__(kA2Threads) seed_update_kernel(const SeedArgs a) {
  __shared__ __align__(4) uint8_t s_border[kA2Threads][108];
  const int tid = threadIdx.x, lane = tid & 31;
  const int i = (blockIdx.x * (kA2Threads / 32) + (tid >> 5)) * a.spw + lane;
  const bool live = lane < a.spw && i < a.n;
  const size_t I = (size_t)(live ? i : 0);
  const CamP cam{a.fx, a.fy, a.cx, a.cy, a.width, a.height};
  float sa = 0.f, sb = 0.f, smu = 1.f, ssig = 1.f, z_range = 1.f;
  int status = 0, code = EPI_FALSE;
  const double kNaN = __longlong_as_double(0x7ff8000000000000LL);
  double z = kNaN, pxc0 = kNaN, pxc1 = kNaN;
  Pose T_ref_cur, T_cur_ref;
  V3 f{0.0, 0.0, 1.0};
  EpiCtx E;
  E.n_iters = 0;
  if (live) {
    sa = a.a[i], sb = a.b[i], smu = a.mu[i], ssig = a.sigma2[i], z_range = a.z_range[i];
    const int r = a.ref_index[i], c = a.cur_index[i];
    const Pose T_ref_w = pose_load(a.T_ref_w + 7 * (size_t)r), T_cur_w = pose_load(a.T_cur_w + 7 * (size_t)c);
    f = V3{a.ref_f[3 * I], a.ref_f[3 * I + 1], a.ref_f[3 * I + 2]};
    T_ref_cur = pose_mul(T_ref_w, pose_inverse(T_cur_w));  // depth_filter.cpp:291
    if (seed_visible(cam, pose_inverse(T_ref_cur), f, smu)) {
      double d_estimate, d_min, d_max;
      depth_range(smu, ssig, d_estimate, d_min, d_max);
      T_cur_ref = pose_mul(T_cur_w, pose_inverse(T_ref_w));
      code = epi_begin(a, cam, i, r, c, T_cur_ref, a.ref_px[2 * I], a.ref_px[2 * I + 1], f, a.ref_level[i], d_estimate, d_min, d_max, false,
                       s_border[tid], E, z, pxc0, pxc1);
      status = 1;  // visible: failed unless the match below succeeds
    }
  }
  warp_epipolar_search(cam, code == EPI_SEARCH, E, (unsigned int)a.serial_steps);
  if (!live) return;
  if (code == EPI_SEARCH) code = epi_end(a, cam, E, s_border[tid], T_cur_ref, f, z, pxc0, pxc1) ? EPI_TRUE : EPI_FALSE;
  if (status == 1 && code == EPI_TRUE) status = 2;
  if (status == 2) {  // computeTau (:568-584) and updatePointSeed (:489-512)
    float x, tau2, fq, eq;
    seed_measurement(cam, T_ref_cur, f, z, x, tau2);
    const float norm_scale = __fsqrt_rn(__fadd_rn(ssig, tau2));
    if (!isnan(norm_scale)) {
      gaussian_beta_update(x, tau2, norm_scale, sa, sb, z_range, smu, ssig, fq, eq);
      sa = __fdiv_rn(__fsub_rn(eq, fq), __fsub_rn(fq, __fdiv_rn(eq, fq)));
      sb = __fdiv_rn(__fmul_rn(sa, __fsub_rn(1.0f, fq)), fq);
    }
  }
  if (status == 1) {
    sb = __fadd_rn(sb, 1.0f);  // :314
    z = kNaN;
  }
  a.out_a[i] = sa, a.out_b[i] = sb, a.out_mu[i] = smu, a.out_sigma2[i] = ssig;
  a.out_status[i] = status;
  a.out_converged[i] = (status == 2 && (double)__fsqrt_rn(ssig) < DD((double)z_range, a.convergence_thresh)) ? 1 : 0;
  a.out_depth[i] = z;
  a.out_px_cur[2 * I] = pxc0, a.out_px_cur[2 * I + 1] = pxc1;
}

// Line seeds: the body of DepthFilter::updateLineSeeds (src/depth_filter.cpp:367-471).  Both end points are searched around
// the segment feature's own px / f (as the reference does) with their own depth hypotheses; computeTau uses sf / ef; the
// shared Beta takes a = max(a_s, a_e), b = min(b_s, b_e) (updateLineSeed, :514-565).
__global__ void __launch_bounds__(kA2Threads) line_seed_update_kernel(const SeedArgs a) {
  __shared__ __align__(4) uint8_t s_border[kA2Threads][108];
  const int tid = threadIdx.x, lane = tid & 31;
  const int i = (blockIdx.x * (kA2Threads / 32) + (tid >> 5)) * a.spw + lane;
  const bool live = lane < a.spw && i < a.n;
  const size_t I = (size_t)(live ? i : 0);
  const CamP cam{a.fx, a.fy, a.cx, a.cy, a.width, a.height};
  float sa = 0.f, sb = 0.f, mu_s = 1.f, sig_s = 1.f, mu_e = 1.f, sig_e = 1.f, zr_s = 1.f, zr_e = 1.f;
  int status = 0;
  const double kNaN = __longlong_as_double(0x7ff8000000000000LL);
  double z_s = kNaN, z_e = kNaN, pxc0 = kNaN, pxc1 = kNaN, pxe0 = kNaN, pxe1 = kNaN;
  Pose T_ref_cur, T_cur_ref;
  V3 f{0.0, 0.0, 1.0}, sf{0.0, 0.0, 1.0}, ef{0.0, 0.0, 1.0};
  double px0 = 0.0, px1 = 0.0;
  int r = 0, c = 0, level_ref = 0;
  bool visible = false;
  if (live) {
    sa = a.a[i], sb = a.b[i];
    mu_s = a.mu[i], sig_s = a.sigma2[i], mu_e = a.mu_e[i], sig_e = a.sigma2_e[i];
    zr_s = a.z_range[i], zr_e = a.z_range_e[i];
    r = a.ref_index[i], c = a.cur_index[i];
    const Pose T_ref_w = pose_load(a.T_ref_w + 7 * (size_t)r), T_cur_w = pose_load(a.T_cur_w + 7 * (size_t)c);
    f = V3{a.ref_f[3 * I], a.ref_f[3 * I + 1], a.ref_f[3 * I + 2]};
    sf = V3{a.ref_sf[3 * I], a.ref_sf[3 * I + 1], a.ref_sf[3 * I + 2]}, ef = V3{a.ref_ef[3 * I], a.ref_ef[3 * I + 1], a.ref_ef[3 * I + 2]};
    T_ref_cur = pose_mul(T_ref_w, pose_inverse(T_cur_w));  // :388
    const Pose T_vis = pose_inverse(T_ref_cur);
    // :389-400: both hypotheses in front of the camera, then both inside the image
    {
      const V3 ps = pose_act(T_vis, v_scale(sf, DD(1.0, (double)mu_s))), pe = pose_act(T_vis, v_scale(ef, DD(1.0, (double)mu_e)));
      visible = !(ps.z < 0.0 || pe.z < 0.0);
      if (visible) {
        double u, v;
        world2cam(cam, ps, u, v);
        int ox = d2i_x86(u), oy = d2i_x86(v);
        visible = ox >= 0 && ox < cam.width && oy >= 0 && oy < cam.height;
        if (visible) {
          world2cam(cam, pe, u, v);
          ox = d2i_x86(u), oy = d2i_x86(v);
          visible = ox >= 0 && ox < cam.width && oy >= 0 && oy < cam.height;
        }
      }
    }
    if (visible) {
      T_cur_ref = pose_mul(T_cur_w, pose_inverse(T_ref_w));
      px0 = a.ref_px[2 * I], px1 = a.ref_px[2 * I + 1];
      level_ref = a.ref_level[i];
    }
  }
  bool ok = visible;
#pragma unroll 1
  for (int e = 0; e < 2; ++e) {  // start point, then (only if it matched) end point; the search is shared by the warp
    EpiCtx E;
    E.n_iters = 0;
    int code = EPI_FALSE;
    double zz = kNaN, q0 = kNaN, q1 = kNaN;
    if (ok) {
      double de, dmin, dmax;
      depth_range(e ? mu_e : mu_s, e ? sig_e : sig_s, de, dmin, dmax);
      code = epi_begin(a, cam, i, r, c, T_cur_ref, px0, px1, f, level_ref, de, dmin, dmax, true, s_border[tid], E, zz, q0, q1);
    }
    warp_epipolar_search(cam, code == EPI_SEARCH, E, (unsigned int)a.serial_steps);
    if (ok) {
      if (code == EPI_SEARCH) code = epi_end(a, cam, E, s_border[tid], T_cur_ref, f, zz, q0, q1) ? EPI_TRUE : EPI_FALSE;
      ok = code == EPI_TRUE;
      if (e == 0)
        z_s = zz, pxc0 = q0, pxc1 = q1;
      else
        z_e = zz, pxe0 = q0, pxe1 = q1;
    }
  }
  if (!live) return;
  if (visible) status = ok ? 2 : 1;
  if (status == 2) {
    float x_s, tau2_s, x_e, tau2_e;
    seed_measurement(cam, T_ref_cur, sf, z_s, x_s, tau2_s);
    seed_measurement(cam, T_ref_cur, ef, z_e, x_e, tau2_e);
    const float ns_s = __fsqrt_rn(__fadd_rn(sig_s, tau2_s)), ns_e = __fsqrt_rn(__fadd_rn(sig_e, tau2_e));
    if (!(isnan(ns_s) || isnan(ns_e))) {
      float f_s, e_s, f_e, e_e;
      gaussian_beta_update(x_s, tau2_s, ns_s, sa, sb, zr_s, mu_s, sig_s, f_s, e_s);
      gaussian_beta_update(x_e, tau2_e, ns_e, sa, sb, zr_e, mu_e, sig_e, f_e, e_e);
      const float a_s = __fdiv_rn(__fsub_rn(e_s, f_s), __fsub_rn(f_s, __fdiv_rn(e_s, f_s)));
      const float a_e = __fdiv_rn(__fsub_rn(e_e, f_e), __fsub_rn(f_e, __fdiv_rn(e_e, f_e)));
      const float b_s = __fdiv_rn(__fmul_rn(a_s, __fsub_rn(1.0f, f_s)), f_s), b_e = __fdiv_rn(__fmul_rn(a_e, __fsub_rn(1.0f, f_e)), f_e);
      sa = (a_s < a_e) ? a_e : a_s;  // std::max(a_s, a_e)
      sb = (b_e < b_s) ? b_e : b_s;  // std::min(b_s, b_e)
    }
  }
  if (status == 1) {
    sb = __fadd_rn(sb, 1.0f);  // :410
    z_s = z_e = kNaN;
  }
  a.out_a[i] = sa, a.out_b[i] = sb, a.out_mu[i] = mu_s, a.out_sigma2[i] = sig_s;
  a.out_mu_e[i] = mu_e, a.out_sigma2_e[i] = sig_e;
  a.out_status[i] = status;
  a.out_converged[i] = (status == 2 && (double)__fsqrt_rn(sig_s) < DD((double)zr_s, a.convergence_thresh) &&
                        (double)__fsqrt_rn(sig_e) < DD((double)zr_e, a.convergence_thresh))
                           ? 1
                           : 0;
  a.out_depth[i] = z_s, a.out_depth_e[i] = z_e;
  a.out_px_cur[2 * I] = pxc0, a.out_px_cur[2 * I + 1] = pxc1;
  a.out_px_cur_e[2 * I] = pxe0, a.out_px_cur_e[2 * I + 1] = pxe1;
}

}  // namespace

cudaError_t match_direct_kernel_launch(const MatchArgs& a, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  match_direct_kernel<<<(a.n + kA2Threads - 1) / kA2Threads, kA2Threads, 0, s>>>(a);
  return cudaGetLastError();
}

// seeds per warp: as many as keeps ~8 warps on every SM (a power of two between 1 and 32)
static int seeds_per_warp(int n) {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  int spw = 1;
  while (spw < 32 && (long long)n > (long long)spw * sms * 8) spw <<= 1;
  return spw;
}
// steps of a search its own thread walks before the warp takes over: worth it only when most lanes hold a seed
static int own_thread_steps(int spw) { return spw >= 16 ? 16 : 0; }

// the schedule of a launch: the caller's forced values (PLSVO_SEEDS_PER_WARP / PLSVO_EPI_SERIAL_STEPS, validated by the host
// code) where set, the automatic choice elsewhere
static SeedArgs seed_schedule(const SeedArgs& a0) {
  SeedArgs a = a0;
  if (a.spw < 1) a.spw = seeds_per_warp(a.n);
  if (a.serial_steps < 0) a.serial_steps = own_thread_steps(a.spw);
  return a;
}

cudaError_t line_seed_update_kernel_launch(const SeedArgs& a0, cudaStream_t s) {
  if (a0.n <= 0) return cudaSuccess;
  const SeedArgs a = seed_schedule(a0);
  const int per_cta = a.spw * (kA2Threads / 32);
  line_seed_update_kernel<<<(a.n + per_cta - 1) / per_cta, kA2Threads, 0, s>>>(a);
  return cudaGetLastError();
}

cudaError_t seed_update_kernel_launch(const SeedArgs& a0, cudaStream_t s) {
  if (a0.n <= 0) return cudaSuccess;
  const SeedArgs a = seed_schedule(a0);
  const int per_cta = a.spw * (kA2Threads / 32);
  seed_update_kernel<<<(a.n + per_cta - 1) / per_cta, kA2Threads, 0, s>>>(a);
  return cudaGetLastError();
}

cudaError_t align1d_kernel_launch(const Align2DArgs& a, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  align1d_kernel<<<(a.n + kA2Threads - 1) / kA2Threads, kA2Threads, 0, s>>>(a);
  return cudaGetLastError();
}

cudaError_t align2d_kernel_launch(const Align2DArgs& a, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  align2d_kernel<<<(a.n + kA2Threads - 1) / kA2Threads, kA2Threads, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace plsvo
