// device_math.cuh — small fixed-size double-precision helpers shared by the kernels:
// Sophus-style quaternion SE3 (what plsvo::Frame::T_f_w_ stores, include/plsvo/frame.h:62),
// 6x6 pivoted LDLT solve (Eigen's ldlt().solve used at src/sparse_img_align.cpp:699 and
// src/pose_optimizer.cpp:170) and 6x6 inverse (src/pose_optimizer.cpp:199).
// Written for one thread operating on registers / shared memory; no dynamic indexing into
// register arrays after unrolling.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace plsvo {

struct Quat {
  double x, y, z, w;
};
struct Vec3 {
  double x, y, z;
};
struct SE3q {
  Quat q;
  Vec3 t;
};

__device__ __forceinline__ Vec3 v3(double x, double y, double z) {
  Vec3 r;
  r.x = x, r.y = y, r.z = z;
  return r;
}
__device__ __forceinline__ Vec3 vadd(Vec3 a, Vec3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ Vec3 vsub(Vec3 a, Vec3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ Vec3 vscale(Vec3 a, double s) { return v3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ Vec3 vcross(Vec3 a, Vec3 b) {
  return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
__device__ __forceinline__ double vnorm(Vec3 a) { return sqrt(a.x * a.x + a.y * a.y + a.z * a.z); }

// q / |q| (Eigen: coeffs() /= coeffs().norm()).  One reciprocal square root (refined to full double
// accuracy) and four multiplies instead of a square root and four divisions: this sits on the serial
// solver path of every Gauss-Newton pass; the result differs from the divide form by <= 1 ulp.
__device__ __forceinline__ Quat qnormalized(Quat q) {
  const double s = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
  double r = rsqrt(s);
  r = r * (1.5 - 0.5 * s * r * r);
  Quat o;
  o.x = q.x * r, o.y = q.y * r, o.z = q.z * r, o.w = q.w * r;
  return o;
}
__device__ __forceinline__ Quat qmul(Quat a, Quat b) {
  Quat r;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
  r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  return r;
}
// rotate v by unit quaternion q (same operation order as Eigen's _transformVector)
__device__ __forceinline__ Vec3 qrot(Quat q, Vec3 v) {
  const Vec3 qv = v3(q.x, q.y, q.z);
  Vec3 uv = vcross(qv, v);
  uv = vadd(uv, uv);
  return vadd(vadd(v, vscale(uv, q.w)), vcross(qv, uv));
}
__device__ __forceinline__ SE3q se3_load(const double* p) {
  SE3q T;
  Quat q;
  q.x = p[0], q.y = p[1], q.z = p[2], q.w = p[3];
  T.q = qnormalized(q);
  T.t = v3(p[4], p[5], p[6]);
  return T;
}
__device__ __forceinline__ void se3_store(const SE3q& T, double* p) {
  p[0] = T.q.x, p[1] = T.q.y, p[2] = T.q.z, p[3] = T.q.w;
  p[4] = T.t.x, p[5] = T.t.y, p[6] = T.t.z;
}
__device__ __forceinline__ SE3q se3_mul(const SE3q& a, const SE3q& b) {
  SE3q r;
  r.t = vadd(a.t, qrot(a.q, b.t));
  r.q = qnormalized(qmul(a.q, b.q));
  return r;
}
__device__ __forceinline__ SE3q se3_inverse(const SE3q& a) {
  SE3q r;
  Quat c;
  c.x = -a.q.x, c.y = -a.q.y, c.z = -a.q.z, c.w = a.q.w;
  r.q = qnormalized(c);
  r.t = qrot(r.q, vscale(a.t, -1.0));
  return r;
}
__device__ __forceinline__ Vec3 se3_act(const SE3q& T, Vec3 p) { return vadd(qrot(T.q, p), T.t); }

// SE3::exp([upsilon, omega]) — Sophus (non-templated) se3.cpp / so3.cpp.
// For |omega|^2 < 0.25 (every Gauss-Newton step of a converging run) the four scalar functions of theta
// that Sophus evaluates with sqrt, sin, cos and three divisions —
//   sin(theta/2)/theta, cos(theta/2), (1-cos theta)/theta^2, (theta-sin theta)/theta^3 —
// are even in theta and are evaluated as short polynomials in theta^2 (truncation < 1e-20): no square
// root, no division, no cancellation on the serial solver path.  They agree with the closed forms to
// double rounding (and are more accurate than `theta - sin(theta)` for small theta).  Larger rotations
// take the closed forms.
__device__ __forceinline__ SE3q se3_exp(const double* u) {
  const Vec3 upsilon = v3(u[0], u[1], u[2]);
  const Vec3 omega = v3(u[3], u[4], u[5]);
  const double t2 = omega.x * omega.x + omega.y * omega.y + omega.z * omega.z;
  double imag_factor, real_factor, a, b;
  if (t2 < 0.25) {
    const double h2 = 0.25 * t2;  // (theta/2)^2
    double ps = 1.0 / 355687428096000.0;  // sin(h)/h = 1 - h2/3! + h2^2/5! - ...
    ps = ps * h2 - 1.0 / 1307674368000.0;
    ps = ps * h2 + 1.0 / 6227020800.0;
    ps = ps * h2 - 1.0 / 39916800.0;
    ps = ps * h2 + 1.0 / 362880.0;
    ps = ps * h2 - 1.0 / 5040.0;
    ps = ps * h2 + 1.0 / 120.0;
    ps = ps * h2 - 1.0 / 6.0;
    ps = ps * h2 + 1.0;
    imag_factor = 0.5 * ps;  // sin(theta/2)/theta
    double pc = 1.0 / 20922789888000.0;  // cos(h) = 1 - h2/2! + h2^2/4! - ...
    pc = pc * h2 - 1.0 / 87178291200.0;
    pc = pc * h2 + 1.0 / 479001600.0;
    pc = pc * h2 - 1.0 / 3628800.0;
    pc = pc * h2 + 1.0 / 40320.0;
    pc = pc * h2 - 1.0 / 720.0;
    pc = pc * h2 + 1.0 / 24.0;
    pc = pc * h2 - 0.5;
    real_factor = pc * h2 + 1.0;
    double pa = 1.0 / 6402373705728000.0;  // (1-cos t)/t^2 = 1/2! - t2/4! + t2^2/6! - ...
    pa = pa * t2 - 1.0 / 20922789888000.0;
    pa = pa * t2 + 1.0 / 87178291200.0;
    pa = pa * t2 - 1.0 / 479001600.0;
    pa = pa * t2 + 1.0 / 3628800.0;
    pa = pa * t2 - 1.0 / 40320.0;
    pa = pa * t2 + 1.0 / 720.0;
    pa = pa * t2 - 1.0 / 24.0;
    a = pa * t2 + 0.5;
    double pb = 1.0 / 121645100408832000.0;  // (t-sin t)/t^3 = 1/3! - t2/5! + t2^2/7! - ...
    pb = pb * t2 - 1.0 / 355687428096000.0;
    pb = pb * t2 + 1.0 / 1307674368000.0;
    pb = pb * t2 - 1.0 / 6227020800.0;
    pb = pb * t2 + 1.0 / 39916800.0;
    pb = pb * t2 - 1.0 / 362880.0;
    pb = pb * t2 + 1.0 / 5040.0;
    pb = pb * t2 - 1.0 / 120.0;
    b = pb * t2 + 1.0 / 6.0;
  } else {
    const double theta = sqrt(t2);
    double s_half, c_half, sn, cs;
    sincos(0.5 * theta, &s_half, &c_half);
    sincos(theta, &sn, &cs);
    imag_factor = s_half / theta;
    real_factor = c_half;
    a = (1 - cs) / t2;
    b = (theta - sn) / (t2 * theta);
  }
  SE3q r;
  Quat q;
  q.x = imag_factor * omega.x, q.y = imag_factor * omega.y, q.z = imag_factor * omega.z, q.w = real_factor;
  r.q = qnormalized(q);
  // t = V*upsilon, V = I + a*Omega + b*Omega^2 (for theta -> 0 this tends to upsilon, as Sophus' small-angle branch)
  const Vec3 wu = vcross(omega, upsilon);
  const Vec3 wwu = vcross(omega, wu);
  r.t = vadd(vadd(upsilon, vscale(wu, a)), vscale(wwu, b));
  return r;
}
// rotation matrix of a unit quaternion (Eigen toRotationMatrix), row-major R[9]
__device__ __forceinline__ void quat_to_R(Quat q, double* R) {
  const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0] = 1 - (tyy + tzz), R[1] = txy - twz, R[2] = txz + twy;
  R[3] = txy + twz, R[4] = 1 - (txx + tzz), R[5] = tyz - twx;
  R[6] = txz - twy, R[7] = tyz + twx, R[8] = 1 - (txx + tyy);
}

// ---- 6x6 LDLT with diagonal pivoting, same algorithm as Eigen's ldlt_inplace<Lower>::unblocked +
// solve (pseudo-inverse of D with tolerance 1/highest).  m is a 6x6 row-major scratch in memory
// (shared or local); A is the full symmetric matrix. ----
static __device__ __noinline__ void ldlt6_solve(const double* A, const double* b, double* x, double* m /*[36]*/) {
  int tr[6];
#pragma unroll 1
  for (int i = 0; i < 36; ++i) m[i] = A[i];
#pragma unroll 1
  for (int k = 0; k < 6; ++k) {
    int piv = k;
    double big = fabs(m[k * 6 + k]);
    for (int i = k + 1; i < 6; ++i) {
      const double v = fabs(m[i * 6 + i]);
      if (v > big) big = v, piv = i;
    }
    tr[k] = piv;
    if (piv != k) {
      for (int j = 0; j < k; ++j) {
        const double t = m[k * 6 + j];
        m[k * 6 + j] = m[piv * 6 + j];
        m[piv * 6 + j] = t;
      }
      for (int i = piv + 1; i < 6; ++i) {
        const double t = m[i * 6 + k];
        m[i * 6 + k] = m[i * 6 + piv];
        m[i * 6 + piv] = t;
      }
      {
        const double t = m[k * 6 + k];
        m[k * 6 + k] = m[piv * 6 + piv];
        m[piv * 6 + piv] = t;
      }
      for (int i = k + 1; i < piv; ++i) {
        const double t = m[i * 6 + k];
        m[i * 6 + k] = m[piv * 6 + i];
        m[piv * 6 + i] = t;
      }
    }
    if (k > 0) {
      double temp[6];
      double s = 0;
      for (int j = 0; j < k; ++j) {
        temp[j] = m[j * 6 + j] * m[k * 6 + j];
        s += m[k * 6 + j] * temp[j];
      }
      m[k * 6 + k] -= s;
      for (int i = k + 1; i < 6; ++i) {
        double s2 = 0;
        for (int j = 0; j < k; ++j) s2 += m[i * 6 + j] * temp[j];
        m[i * 6 + k] -= s2;
      }
    }
    const double akk = m[k * 6 + k];
    const bool valid = fabs(akk) > 0.0;
    if (k == 0 && !valid) {
      for (int j = 0; j < 6; ++j) tr[j] = j;
      break;
    }
    if (valid)
      for (int i = k + 1; i < 6; ++i) m[i * 6 + k] /= akk;
  }
  double y[6];
  for (int i = 0; i < 6; ++i) y[i] = b[i];
#pragma unroll 1
  for (int k = 0; k < 6; ++k) {
    const double t = y[k];
    y[k] = y[tr[k]];
    y[tr[k]] = t;
  }
#pragma unroll 1
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < i; ++j) y[i] -= m[i * 6 + j] * y[j];
  const double tol = 1.0 / 1.7976931348623157e308;
#pragma unroll 1
  for (int i = 0; i < 6; ++i) y[i] = (fabs(m[i * 6 + i]) > tol) ? y[i] / m[i * 6 + i] : 0.0;
#pragma unroll 1
  for (int i = 5; i >= 0; --i)
    for (int j = i + 1; j < 6; ++j) y[i] -= m[j * 6 + i] * y[j];
#pragma unroll 1
  for (int k = 5; k >= 0; --k) {
    const double t = y[k];
    y[k] = y[tr[k]];
    y[tr[k]] = t;
  }
  for (int i = 0; i < 6; ++i) x[i] = y[i];
}

// 6x6 inverse by partial-pivot LU (Eigen: PartialPivLU for fixed sizes > 4).  lu: 36-double scratch.
static __device__ __noinline__ void inverse6(const double* A, double* out, double* lu) {
  int perm[6];
#pragma unroll 1
  for (int i = 0; i < 36; ++i) lu[i] = A[i];
  for (int i = 0; i < 6; ++i) perm[i] = i;
#pragma unroll 1
  for (int k = 0; k < 6; ++k) {
    int piv = k;
    double big = fabs(lu[k * 6 + k]);
    for (int i = k + 1; i < 6; ++i) {
      const double v = fabs(lu[i * 6 + k]);
      if (v > big) big = v, piv = i;
    }
    if (piv != k) {
      for (int j = 0; j < 6; ++j) {
        const double t = lu[k * 6 + j];
        lu[k * 6 + j] = lu[piv * 6 + j];
        lu[piv * 6 + j] = t;
      }
      const int t = perm[k];
      perm[k] = perm[piv];
      perm[piv] = t;
    }
    for (int i = k + 1; i < 6; ++i) {
      lu[i * 6 + k] /= lu[k * 6 + k];
      for (int j = k + 1; j < 6; ++j) lu[i * 6 + j] -= lu[i * 6 + k] * lu[k * 6 + j];
    }
  }
#pragma unroll 1
  for (int c = 0; c < 6; ++c) {
    double y[6];
    for (int i = 0; i < 6; ++i) {
      y[i] = (perm[i] == c) ? 1.0 : 0.0;
      for (int j = 0; j < i; ++j) y[i] -= lu[i * 6 + j] * y[j];
    }
    for (int i = 5; i >= 0; --i) {
      for (int j = i + 1; j < 6; ++j) y[i] -= lu[i * 6 + j] * y[j];
      y[i] /= lu[i * 6 + i];
    }
    for (int i = 0; i < 6; ++i) out[i * 6 + c] = y[i];
  }
}


// ---- register-resident, fully unrolled LDL^T solve of the symmetric 6x6 system (no pivoting).
// H is a sum of weighted outer products (SPD unless degenerate); when a pivot is not safely
// positive the caller falls back to the pivoted Eigen-style routine above, which also defines
// the zero / NaN behaviour.  Hu = upper triangle, row-major (21 values).
__device__ __forceinline__ bool ldlt6_reg(const double* Hu, const double* g, double* x) {
  double A[6][6];
  {
    int idx = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int j = i; j < 6; ++j) A[j][i] = Hu[idx++];  // lower triangle
  }
  double dmax = 0.0;
#pragma unroll
  for (int i = 0; i < 6; ++i) dmax = fmax(dmax, fabs(A[i][i]));
  const double tiny = 1e-13 * dmax;
  double L[6][6], dinv[6], T[6][6];  // T[j][k] = L[j][k]*d[k]
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    double s = A[j][j];
#pragma unroll
    for (int k = 0; k < j; ++k) s -= L[j][k] * T[j][k];

    ok = ok && (s > tiny);
    dinv[j] = __drcp_rn(s);
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      double t = A[i][j];
#pragma unroll
      for (int k = 0; k < j; ++k) t -= L[i][k] * T[j][k];
      T[i][j] = t;
      L[i][j] = t * dinv[j];
    }
  }
  double z[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    double t = g[i];
#pragma unroll
    for (int k = 0; k < i; ++k) t -= L[i][k] * z[k];
    z[i] = t;
  }
#pragma unroll
  for (int i = 5; i >= 0; --i) {
    double t = z[i] * dinv[i];
#pragma unroll
    for (int k = i + 1; k < 6; ++k) t -= L[k][i] * x[k];
    x[i] = t;
  }
  return ok;
}

// RN_float(1/(1+a)) for a >= 0 without leaving fp32: the reference evaluates
// `1.0/(1.0+fabsf(res))` in double and narrows (sparse_img_align.cpp:479).  1+a is split exactly
// into sh+sl (TwoSum), q0 = RN(1/sh), one Newton step with the exact residual.  Equal to the
// double-then-narrow result except when the true quotient lies within ~2^-48 relative of a
// rounding boundary (checked exhaustively by plsvo_selftest_weight).
__device__ __forceinline__ float weight_rcp(float a) {
  const float sh = __fadd_rn(1.0f, a);
  const float bb = __fsub_rn(sh, 1.0f);
  const float sl = __fadd_rn(__fsub_rn(1.0f, __fsub_rn(sh, bb)), __fsub_rn(a, bb));
  float q0;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(q0) : "f"(sh));  // MUFU.RCP; refined below
  float e = __fmaf_rn(-sh, q0, 1.0f);
  e = __fmaf_rn(-sl, q0, e);
  return __fmaf_rn(e, q0, q0);
}

// byte k of w as float, via PRMT + FADD (keeps the XU conversion pipe free): 0x4B0000bb = 2^23 + bb
__device__ __forceinline__ float byte_to_float(uint32_t w, int k) {
  return __fsub_rn(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7440u | (uint32_t)k)), 8388608.0f);
}

// Frame::jacobian_xyz2uv rows (include/plsvo/frame.h:138-160)
__device__ __forceinline__ void jacobian_rows(double x, double y, double z, double* r0, double* r1) {
  const double z_inv = 1. / z;
  const double z_inv_2 = z_inv * z_inv;
  r0[0] = -z_inv;
  r0[1] = 0.0;
  r0[2] = x * z_inv_2;
  r0[3] = y * r0[2];
  r0[4] = -(1.0 + x * r0[2]);
  r0[5] = y * z_inv;
  r1[0] = 0.0;
  r1[1] = -z_inv;
  r1[2] = y * z_inv_2;
  r1[3] = 1.0 + y * r1[2];
  r1[4] = -r0[3];
  r1[5] = -x * z_inv;
}

__device__ __forceinline__ void jacobian_rows_zinv(double x, double y, double z_inv, double* r0, double* r1) {
  const double z_inv_2 = z_inv * z_inv;
  r0[0] = -z_inv;
  r0[1] = 0.0;
  r0[2] = x * z_inv_2;
  r0[3] = y * r0[2];
  r0[4] = -(1.0 + x * r0[2]);
  r0[5] = y * z_inv;
  r1[0] = 0.0;
  r1[1] = -z_inv;
  r1[2] = y * z_inv_2;
  r1[3] = 1.0 + y * r1[2];
  r1[4] = -r0[3];
  r1[5] = -x * z_inv;
}

// ---- shared-memory address + mbarrier + bulk async copy (TMA engine, SASS UBLKCP) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// global -> shared bulk copy, completion signalled on the mbarrier (bytes % 16 == 0, 16B aligned)
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

__device__ __forceinline__ void fence_mbarrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// one butterfly step of warp_reduce32.  S is a template argument so that every index into v is a constant after
// unrolling: a loop whose trip count depends on the step leaves v indexed at run time, and that puts v in local memory.
template <int S>
__device__ __forceinline__ void warp_reduce_step(double* v, int lane) {
  const bool upper = (lane & S) != 0;
#pragma unroll
  for (int i = 0; i < S; ++i) {
    const double send = upper ? v[i] : v[i + S];
    const double keep = upper ? v[i + S] : v[i];
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, S);
  }
}

// register-halving warp reduction of 32 doubles: afterwards lane L holds the warp-wide sum of v[L]
// (fixed summation order -> bitwise reproducible).
__device__ __forceinline__ double warp_reduce32(double* v, int lane) {
  warp_reduce_step<16>(v, lane);
  warp_reduce_step<8>(v, lane);
  warp_reduce_step<4>(v, lane);
  warp_reduce_step<2>(v, lane);
  warp_reduce_step<1>(v, lane);
  return v[0];
}

}  // namespace plsvo
