// poseopt_kernel.cu — plsvo::pose_optimizer::optimizeGaussNewton (src/pose_optimizer.cpp:38-260 and
// :262-582) as one sm_90a kernel: a CTA owns one frame for the whole optimisation — MAD scale
// pre-pass, Gauss-Newton loop with Tukey weights, covariance, outlier pass, optional refinement
// loop and the two reporting medians — with no host round trips.
//
// Mapping: thread per feature (points then line segments), 21+6+1 double accumulators per thread,
// register-halving warp reduction + fixed-order cross-warp sum (deterministic), thread 0 does the
// 6x6 LDLT solve and the SE3 update.  Medians use vk::getMedian's convention (element of rank
// floor(n/2)) via rank counting on shared-memory keys, dead features carrying +inf keys.
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include "device_math.cuh"
#include "internal.h"

namespace plsvo {

namespace {

#ifndef PLSVO_PO_THREADS
#define PLSVO_PO_THREADS 128
#endif
constexpr int kPoThreads = PLSVO_PO_THREADS;
constexpr int kPoWarps = kPoThreads / 32;

struct PoCtl {
  double R[9];
  double t[3];
  double T[7];
  double T_old[7];
  double A[36];
  double b[6];
  double dT[6];
  double scratch[36];
  double cov_in[36];
  double chi2;
  unsigned long long sel[2];
  int hist[256];
  int flag;
  int iter;
  int count;
};

// TukeyWeightFunction::value (vikit robust_cost.cpp), b = 4.6851f, all in float
__device__ __forceinline__ float tukey(float x) {
  const float b = 4.6851f;
  const float b_square = __fmul_rn(b, b);
  const float x_square = __fmul_rn(x, x);
  if (x_square <= b_square) {
    const float tmp = __fsub_rn(1.0f, __fdiv_rn(x_square, b_square));
    return __fmul_rn(tmp, tmp);
  }
  return 0.0f;
}

__device__ __forceinline__ void accumulate(double* acc, const double* J0, const double* J1, double e0, double e1,
                                           double e_sq, double w) {
  int idx = 0;
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = i; j < 6; ++j) acc[idx++] += (J0[i] * J0[j] + J1[i] * J1[j]) * w;  // :126
#pragma unroll
  for (int i = 0; i < 6; ++i) acc[21 + i] -= (J0[i] * e0 + J1[i] * e1) * w;  // :127
  acc[27] += e_sq * w;                                                        // :128
}

// element of rank k (0-based) among the non-negative keys[0..n) — vk::getMedian's nth_element at
// floor(n/2) — by MSB-first radix select on the IEEE bit patterns (monotone for keys >= 0, +inf last):
// 8 bits per pass, shared-memory histogram, warp 0 locates the bin holding rank k.
__device__ __forceinline__ double block_kth(const double* keys, int n, int k, int* hist, unsigned long long* sel,
                                            int tid) {
  const int lane = tid & 31;
  if (tid == 0) {
    sel[0] = 0ull;                    // bits decided so far
    sel[1] = (unsigned long long)k;   // rank inside the surviving set
  }
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += kPoThreads) hist[i] = 0;
    __syncthreads();
    const unsigned long long prefix = sel[0];
    const unsigned long long hi_mask = (shift == 56) ? 0ull : (~0ull << (shift + 8));
    for (int i = tid; i < n; i += kPoThreads) {
      const unsigned long long key = (unsigned long long)__double_as_longlong(keys[i]);
      if ((key & hi_mask) == prefix) atomicAdd(&hist[(int)((key >> shift) & 255ull)], 1);
    }
    __syncthreads();
    if (tid < 32) {
      int c[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c[j] = hist[lane * 8 + j];
        sum += c[j];
      }
      int incl = sum;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += v;
      }
      const int kk = (int)sel[1];
      __syncwarp();  // every lane has read the rank before the owning lane overwrites it
      const int before = incl - sum;
      if (kk >= before && kk < incl) {  // exactly one lane
        int acc = before, bin = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (kk >= acc && kk < acc + c[j]) bin = j, sel[1] = (unsigned long long)(kk - acc);
          acc += c[j];
        }
        sel[0] = prefix | ((unsigned long long)(lane * 8 + bin) << shift);
      }
    }
    __syncthreads();
  }
  const double r = __longlong_as_double((long long)sel[0]);
  __syncthreads();
  return r;
}

struct Feat {  // per-frame feature arrays
  const double *pt_f, *pt_pos, *seg_line, *seg_spos, *seg_epos;
  const int32_t *pt_level, *seg_level;
  int np, ns;
};

__device__ __forceinline__ void load_T(const PoCtl* ctl, double* R, double* t) {
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = ctl->R[i];
  t[0] = ctl->t[0], t[1] = ctl->t[1], t[2] = ctl->t[2];
}
__device__ __forceinline__ void xform(const double* R, const double* t, const double* p, double& x, double& y,
                                      double& z) {
  x = R[0] * p[0] + R[1] * p[1] + R[2] * p[2] + t[0];
  y = R[3] * p[0] + R[4] * p[1] + R[5] * p[2] + t[1];
  z = R[6] * p[0] + R[7] * p[1] + R[8] * p[2] + t[2];
}
__device__ __forceinline__ void set_T(PoCtl* ctl, const SE3q& T) {
  se3_store(T, ctl->T);
  quat_to_R(T.q, ctl->R);
  ctl->t[0] = T.t.x, ctl->t[1] = T.t.y, ctl->t[2] = T.t.z;
}
__device__ __forceinline__ SE3q get_T(const double* p) {
  SE3q T;
  T.q.x = p[0], T.q.y = p[1], T.q.z = p[2], T.q.w = p[3];
  T.t = v3(p[4], p[5], p[6]);
  return T;
}

// point residual on the unit plane, scaled by 1/2^level (:65-67, :116-120, :211-213)
__device__ __forceinline__ void point_error(const double* R, const double* t, const double* f, const double* pos,
                                            int level, double& x, double& y, double& z, double& e0, double& e1,
                                            double& sic) {
  xform(R, t, pos, x, y, z);
  sic = 1.0 / (double)(1 << level);
  e0 = (f[0] / f[2] - x / z) * sic;
  e1 = (f[1] / f[2] - y / z) * sic;
}
// line endpoint-to-line distances (:80-84, :144-148, :229-232), in double
__device__ __forceinline__ void line_dists(const double* R, const double* t, const double* l, const double* sp,
                                           const double* ep, double* xs, double* xe, double& ds, double& de) {
  xform(R, t, sp, xs[0], xs[1], xs[2]);
  xform(R, t, ep, xe[0], xe[1], xe[2]);
  ds = __dadd_rn(__dadd_rn(__dmul_rn(l[0], xs[0] / xs[2]), __dmul_rn(l[1], xs[1] / xs[2])), l[2]);
  de = __dadd_rn(__dadd_rn(__dmul_rn(l[0], xe[0] / xe[2]), __dmul_rn(l[1], xe[1] / xe[2])), l[2]);
}

// One Gauss-Newton loop (:103-195 / :473-563).  `which` = 0 main loop, 1 refinement.
__device__ __forceinline__ void gn_loop(const PoseOptArgs& a, const Feat& F, PoCtl* ctl, double* red, double* tot,
                                        uint8_t* pt_alive, uint8_t* seg_alive, double* keys_init, int init_off,
                                        double scale_pt, double scale_ls, int n_iter, int* iters_out, int tid) {
  const int lane = tid & 31, warp = tid >> 5;
  if (tid == 0) ctl->iter = 0;
  __syncthreads();
  if (n_iter <= 0) return;
  for (;;) {
    double acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.0;
    double R[9], t[3];
    load_T(ctl, R, t);
    const bool first = (ctl->iter == 0);
    for (int i = tid; i < F.np; i += kPoThreads) {
      if (!pt_alive[i]) continue;
      double x, y, z, e0, e1, sic;
      point_error(R, t, F.pt_f + 3 * i, F.pt_pos + 3 * i, F.pt_level[i], x, y, z, e0, e1, sic);
      double J0[6], J1[6];
      jacobian_rows(x, y, z, J0, J1);
      const double e_sq = e0 * e0 + e1 * e1;
      if (first) keys_init[init_off + i] = e_sq;  // chi2_vec_init (:121-122)
#pragma unroll
      for (int k = 0; k < 6; ++k) J0[k] *= sic, J1[k] *= sic;
      const double w = (double)tukey((float)(sqrt(e_sq) / scale_pt));  // :124
      accumulate(acc, J0, J1, e0, e1, e_sq, w);
    }
    for (int j = tid; j < F.ns; j += kPoThreads) {
      if (!seg_alive[j]) continue;
      const double* l = F.seg_line + 3 * j;
      double xs[3], xe[3], dsd, ded;
      line_dists(R, t, l, F.seg_spos + 3 * j, F.seg_epos + 3 * j, xs, xe, dsd, ded);
      const float ds = (float)dsd, de = (float)ded;  // :147-148 float truncation
      const double sic = 1.0 / (double)(1 << F.seg_level[j]);
      const double e0 = (double)ds * sic, e1 = (double)de * sic;
      const double e_sq = e0 * e0 + e1 * e1;
      if (first) keys_init[init_off + F.np + j] = e_sq;
      const double e_norm = sqrt(e_sq);
      const double js = sic * (double)ds / e_norm;  // :157-158 (ds for both endpoints, as in the reference)
      double Js0[6], Js1[6], Je0[6], Je1[6], J0[6], J1[6];
      jacobian_rows(xs[0], xs[1], xs[2], Js0, Js1);
      jacobian_rows(xe[0], xe[1], xe[2], Je0, Je1);
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        J0[k] = l[0] * (Js0[k] * js) + l[1] * (Js1[k] * js);  // :159
        J1[k] = l[0] * (Je0[k] * js) + l[1] * (Je1[k] * js);  // :160
      }
      const double w = (double)tukey((float)(e_norm / scale_ls));  // :162
      accumulate(acc, J0, J1, e0, e1, e_sq, w);
    }
    const double mine = warp_reduce32(acc, lane);
    red[warp * 32 + lane] = mine;
    __syncthreads();
    if (warp == 0) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < kPoWarps; ++w) s += red[w * 32 + lane];
      tot[lane] = s;
      __syncwarp();
      if (lane == 0) {
        // A (for Cov_ = (A*fx^2)^-1, :199, and for the pivoted fallback) is only unpacked where it is read: on the last
        // evaluated pass and on a degenerate system — not on every pass of this serial section
        auto unpack_A = [&]() {
          int idx = 0;
          for (int i = 0; i < 6; ++i)
            for (int j = i; j < 6; ++j) {
              ctl->A[i * 6 + j] = tot[idx];
              ctl->A[j * 6 + i] = tot[idx];
              ++idx;
            }
          for (int i = 0; i < 6; ++i) ctl->b[i] = tot[21 + i];
        };
        const double new_chi2 = tot[27];
        {  // :170 — register LDL^T; the pivoted Eigen-style routine handles degenerate systems
          double Hu[21], gg[6], xx[6];
#pragma unroll
          for (int i = 0; i < 21; ++i) Hu[i] = tot[i];
#pragma unroll
          for (int i = 0; i < 6; ++i) gg[i] = tot[21 + i];
          if (ldlt6_reg(Hu, gg, xx)) {
#pragma unroll
            for (int i = 0; i < 6; ++i) ctl->dT[i] = xx[i];
          } else {
            unpack_A();
            ldlt6_solve(ctl->A, ctl->b, ctl->dT, ctl->scratch);
          }
        }
        *iters_out += 1;
        int flag = 0;
        if ((ctl->iter > 0 && new_chi2 > ctl->chi2) || isnan(ctl->dT[0])) {  // :173-180
          const SE3q To = get_T(ctl->T_old);
          set_T(ctl, To);
          flag = 1;
        } else {
          const SE3q T = get_T(ctl->T);
          const SE3q Tn = se3_mul(se3_exp(ctl->dT), T);  // :183
          for (int i = 0; i < 7; ++i) ctl->T_old[i] = ctl->T[i];
          set_T(ctl, Tn);
          ctl->chi2 = new_chi2;
          double nm = 0.0;
          for (int i = 0; i < 6; ++i) nm = fmax(nm, fabs(ctl->dT[i]));
          if (nm <= 0.0000000001) flag = 1;  // EPS (global.h:99)
        }
        ctl->iter += 1;
        if (ctl->iter >= n_iter) flag = 1;
        if (flag) unpack_A();
        ctl->flag = flag;
      }
    }
    __syncthreads();
    if (ctl->flag) break;
  }
}

#ifndef PLSVO_PO_MINB
#define PLSVO_PO_MINB 3  // resident CTAs per SM the register budget is compiled for (168 registers fit three)
#endif
// The whole kernel.  kPerFrameFx: frame b's errorMultiplier2 is a.fx_frame[b] (the multicam entry points) instead of
// a.fx; it is the only difference between the two __global__ entry points below.
template <bool kPerFrameFx>
__device__ __forceinline__ void optimize_frames(const PoseOptArgs& a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x;
  const int n_tot = a.n_pts + a.n_segs;
  PoCtl* ctl = reinterpret_cast<PoCtl*>(smem);
  double* red = reinterpret_cast<double*>(smem + ((sizeof(PoCtl) + 15) / 16) * 16);
  double* tot = red + kPoWarps * 32;
  double* keys_init = tot + 32;              // [2*n_tot]
  double* keys_final = keys_init + 2 * n_tot;  // [n_tot]
  uint8_t* pt_alive = reinterpret_cast<uint8_t*>(keys_final + n_tot);
  uint8_t* seg_alive = pt_alive + a.n_pts;

  for (int b = blockIdx.x; b < a.B; b += gridDim.x) {
    __syncthreads();
    Feat F;
    // validated on upload; the clamp keeps a corrupted count from indexing shared memory out of bounds
    F.np = min(max(a.pt_count ? a.pt_count[b] : a.n_pts, 0), a.n_pts);
    F.ns = min(max(a.seg_count ? a.seg_count[b] : a.n_segs, 0), a.n_segs);
    const size_t po = (size_t)b * a.n_pts, so = (size_t)b * a.n_segs;
    F.pt_f = a.pt_f + 3 * po;
    F.pt_pos = a.pt_pos + 3 * po;
    F.pt_level = a.pt_level + po;
    F.seg_line = a.seg_line + 3 * so;
    F.seg_spos = a.seg_spos + 3 * so;
    F.seg_epos = a.seg_epos + 3 * so;
    F.seg_level = a.seg_level + so;
    const double fx = kPerFrameFx ? a.fx_frame[b] : a.fx;

    if (tid == 0) {
      const SE3q T = se3_load(a.T_f_w + (size_t)b * 7);
      set_T(ctl, T);
      for (int i = 0; i < 7; ++i) ctl->T_old[i] = ctl->T[i];
      ctl->chi2 = 0.0;
      for (int i = 0; i < 36; ++i) ctl->A[i] = 0.0;
      a.out_iters[2 * (size_t)b] = 0;
      a.out_iters[2 * (size_t)b + 1] = 0;
    }
    for (int i = tid; i < a.n_pts; i += kPoThreads) {
      pt_alive[i] = (i < F.np) && (a.pt_valid ? a.pt_valid[po + i] != 0 : true);
      a.out_pt_outlier[po + i] = 0;
    }
    for (int j = tid; j < a.n_segs; j += kPoThreads) {
      seg_alive[j] = (j < F.ns) && (a.seg_valid ? a.seg_valid[so + j] != 0 : true);
      a.out_seg_outlier[so + j] = 0;
    }
    for (int i = tid; i < 2 * n_tot; i += kPoThreads) keys_init[i] = CUDART_INF;
    for (int i = tid; i < n_tot; i += kPoThreads) keys_final[i] = CUDART_INF;
    __syncthreads();

    // ---- MAD scale pre-pass (:58-96): float error norms at the initial pose ----
    double R[9], t[3];
    load_T(ctl, R, t);
    int my_pt = 0, my_ls = 0;
    double* keys = keys_final;  // reuse as scratch: [0,n_pts) point errors, [n_pts,n_tot) line errors
    for (int i = tid; i < F.np; i += kPoThreads) {
      if (!pt_alive[i]) continue;
      double x, y, z, e0, e1, sic;
      point_error(R, t, F.pt_f + 3 * i, F.pt_pos + 3 * i, F.pt_level[i], x, y, z, e0, e1, sic);
      keys[i] = (double)(float)sqrt(e0 * e0 + e1 * e1);  // errors.push_back(e.norm()) -> float
      ++my_pt;
    }
    for (int j = tid; j < F.ns; j += kPoThreads) {
      if (!seg_alive[j]) continue;
      double xs[3], xe[3], dsd, ded;
      line_dists(R, t, F.seg_line + 3 * j, F.seg_spos + 3 * j, F.seg_epos + 3 * j, xs, xe, dsd, ded);
      const float es = (float)dsd, ee = (float)ded;
      keys[a.n_pts + j] = (double)__fsqrt_rn(__fadd_rn(__fmul_rn(es, es), __fmul_rn(ee, ee)));  // :85-86
      ++my_ls;
    }
    // counts (each thread handles a disjoint subset)
    for (int d = 16; d >= 1; d >>= 1) {
      my_pt += __shfl_xor_sync(0xffffffffu, my_pt, d);
      my_ls += __shfl_xor_sync(0xffffffffu, my_ls, d);
    }
    if ((tid & 31) == 0) {
      red[tid >> 5] = (double)my_pt;
      red[kPoWarps + (tid >> 5)] = (double)my_ls;
    }
    __syncthreads();
    int n_pt = 0, n_ls = 0;
    for (int w = 0; w < kPoWarps; ++w) {
      n_pt += (int)red[w];
      n_ls += (int)red[kPoWarps + w];
    }
    __syncthreads();
    if (n_pt + n_ls == 0) {  // :88-89 — outputs untouched
      if (tid == 0) {
        for (int i = 0; i < 7; ++i) a.out_T[(size_t)b * 7 + i] = a.T_f_w[(size_t)b * 7 + i];
        a.out_status[b] = 1;
      }
      continue;
    }
    double estimated_scale_pt = 0.0;  // reference: getMedian on an empty vector is UB; defined as 0 here
    if (n_pt > 0) estimated_scale_pt = (double)__fmul_rn(1.48f, (float)block_kth(keys, a.n_pts, n_pt / 2, ctl->hist, ctl->sel, tid));
    double estimated_scale_ls = 1.0;
    if (n_ls > 0)
      estimated_scale_ls = (double)__fmul_rn(1.48f, (float)block_kth(keys + a.n_pts, a.n_segs, n_ls / 2, ctl->hist, ctl->sel, tid));
    __syncthreads();
    for (int i = tid; i < n_tot; i += kPoThreads) keys_final[i] = CUDART_INF;
    __syncthreads();

    // ---- main GN loop ----
    gn_loop(a, F, ctl, red, tot, pt_alive, seg_alive, keys_init, 0, estimated_scale_pt, estimated_scale_ls, a.n_iter,
            &a.out_iters[2 * (size_t)b], tid);

    // ---- covariance (:197-199): (A * fx^2)^-1 from the last evaluated A ----
    if (tid == 0) {
      const double fx2 = fx * fx;
      for (int i = 0; i < 36; ++i) ctl->cov_in[i] = ctl->A[i] * fx2;
      inverse6(ctl->cov_in, a.out_cov + (size_t)b * 36, ctl->scratch);
    }

    // ---- outlier pass at the final pose (:201-242) ----
    load_T(ctl, R, t);
    const double thr_pt = a.reproj_thresh / fx;
    const double thr_ls = thr_pt * estimated_scale_ls / estimated_scale_pt;
    int del_pt = 0, del_ls = 0;
    for (int i = tid; i < F.np; i += kPoThreads) {
      if (!pt_alive[i]) continue;
      double x, y, z, e0, e1, sic;
      point_error(R, t, F.pt_f + 3 * i, F.pt_pos + 3 * i, F.pt_level[i], x, y, z, e0, e1, sic);
      const double e_sq = e0 * e0 + e1 * e1;
      keys_final[i] = e_sq;
      if (sqrt(e_sq) > thr_pt) {
        pt_alive[i] = 0;
        a.out_pt_outlier[po + i] = 1;
        ++del_pt;
      }
    }
    for (int j = tid; j < F.ns; j += kPoThreads) {
      if (!seg_alive[j]) continue;
      double xs[3], xe[3], dsd, ded;
      line_dists(R, t, F.seg_line + 3 * j, F.seg_spos + 3 * j, F.seg_epos + 3 * j, xs, xe, dsd, ded);
      const double sic = 1.0 / (double)(1 << F.seg_level[j]);
      const double e0 = dsd * sic, e1 = ded * sic;
      const double e_sq = e0 * e0 + e1 * e1;
      keys_final[a.n_pts + j] = e_sq;
      if (sqrt(e_sq) > thr_ls) {
        seg_alive[j] = 0;
        a.out_seg_outlier[so + j] = 1;
        ++del_ls;
      }
    }
    for (int d = 16; d >= 1; d >>= 1) {
      del_pt += __shfl_xor_sync(0xffffffffu, del_pt, d);
      del_ls += __shfl_xor_sync(0xffffffffu, del_ls, d);
    }
    __syncthreads();
    if ((tid & 31) == 0) {
      red[tid >> 5] = (double)del_pt;
      red[kPoWarps + (tid >> 5)] = (double)del_ls;
    }
    __syncthreads();
    int n_del_pt = 0, n_del_ls = 0;
    for (int w = 0; w < kPoWarps; ++w) {
      n_del_pt += (int)red[w];
      n_del_ls += (int)red[kPoWarps + w];
    }
    __syncthreads();

    // ---- refinement loop of the 10-argument overload (:469-563) ----
    int n_init = (a.n_iter > 0) ? (n_pt + n_ls) : 0;
    if (a.n_iter_ref >= 0) {
      gn_loop(a, F, ctl, red, tot, pt_alive, seg_alive, keys_init, n_tot, estimated_scale_pt, estimated_scale_ls,
              a.n_iter_ref, &a.out_iters[2 * (size_t)b + 1], tid);
      if (a.n_iter_ref > 0) n_init += (n_pt - n_del_pt) + (n_ls - n_del_ls);
    }

    // ---- reporting medians (:244-251) ----
    const int n_final = n_pt + n_ls;
    const double med_init = (n_init > 0) ? block_kth(keys_init, 2 * n_tot, n_init / 2, ctl->hist, ctl->sel, tid) : 0.0;
    const double med_final = block_kth(keys_final, n_tot, n_final / 2, ctl->hist, ctl->sel, tid);
    if (tid == 0) {
      for (int i = 0; i < 7; ++i) a.out_T[(size_t)b * 7 + i] = ctl->T[i];
      a.out_scale[b] = estimated_scale_pt * fx;
      a.out_err_init[b] = (n_init > 0) ? sqrt(med_init) * fx : 0.0;
      a.out_err_final[b] = sqrt(med_final) * fx;
      a.out_num_pt[b] = (long long)(n_pt - n_del_pt);
      a.out_num_ls[b] = (long long)(n_ls - n_del_ls);
      a.out_status[b] = 0;
    }
  }
}

__global__ void __launch_bounds__(kPoThreads, PLSVO_PO_MINB) pose_optimizer_kernel(const PoseOptArgs a) {
  optimize_frames<false>(a);
}

__global__ void __launch_bounds__(kPoThreads, PLSVO_PO_MINB) pose_optimizer_multicam_kernel(const PoseOptArgs a) {
  optimize_frames<true>(a);
}

}  // namespace

size_t poseopt_smem_bytes(int n_pts, int n_segs) {
  const size_t n_tot = (size_t)n_pts + n_segs;
  size_t s = ((sizeof(PoCtl) + 15) / 16) * 16;
  s += (kPoWarps * 32 + 32) * sizeof(double);
  s += 3 * n_tot * sizeof(double);
  s += n_tot + 16;
  return s;
}

namespace {
// one launch of either entry point: at most 16 CTAs per SM, each walking its frames with a grid stride
cudaError_t launch_frames(void (*kernel)(const PoseOptArgs), const PoseOptArgs& a, size_t smem_bytes, cudaStream_t s) {
  static int max_grid = 0;
  if (max_grid == 0) {
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    max_grid = sms * 16;
  }
  cudaError_t e = cudaSuccess;
  if (smem_bytes > 48 * 1024)
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
  if (e != cudaSuccess) return e;
  const int grid = a.B < max_grid ? a.B : max_grid;
  kernel<<<grid, kPoThreads, smem_bytes, s>>>(a);
  return cudaGetLastError();
}
}  // namespace

cudaError_t poseopt_kernel_launch(const PoseOptArgs& a, size_t smem_bytes, cudaStream_t s) {
  return launch_frames(pose_optimizer_kernel, a, smem_bytes, s);
}

cudaError_t poseopt_multicam_kernel_launch(const PoseOptArgs& a, size_t smem_bytes, cudaStream_t s) {
  return launch_frames(pose_optimizer_multicam_kernel, a, smem_bytes, s);
}

}  // namespace plsvo
