// fake_atan_match.cpp — model kernel of the ATAN findMatchDirect call (plsvo_match_direct_atan_batch_run) for the
// host-pipeline model.  TEST INFRASTRUCTURE ONLY (see fake_cuda.h).
//
// tests/test_atan_match_host_cpu.py and tools/preflight_gpu_tests.py link it into a model library of their own, next to
// the stock model kernels (fake_kernels.cpp), which lack this launcher; plsvo_abi.cu reaches it through a weak reference.
//
//   digest mode       : every byte the real kernel reads or writes is bounds-checked against the live device blocks — the
//                       per-candidate arrays, the pose of every referenced keyframe and current frame, the reference level
//                       of every candidate's keyframe and every level below n_pyr_levels of its current frame, the
//                       outputs — and MatchArgs must carry the distortion terms vk::ATANCamera derives from s_.  The
//                       outputs are written as for a candidate that failed the in-frame test (px_cur copied, success 0,
//                       search level -1, A_cur_ref untouched).
//   PLSVO_FAKE_ORACLE : the kernel is answered by plsvo_oracle_atan_match_direct_members (oracle/atan_match_oracle.cpp) with
//                       the members fx_..cy_ and d0 it receives, looked up in the oracle library or, when that is the plain
//                       oracle, in libplsvo_atan_match_oracle.so next to it.
#include <dlfcn.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <thread>

#include "../../pl-svo_b200/csrc/internal.h"
#include "fake_cuda.h"

namespace {

using MatchMembersFn = int (*)(double, double, double, double, double, const plsvo_match_batch*, const plsvo_match_result*, int);

MatchMembersFn oracle_match() {
  static MatchMembersFn fn = nullptr;
  static bool looked = false;
  if (!looked) {
    looked = true;
    const char* path = getenv("PLSVO_FAKE_ORACLE");
    if (path && *path) {
      const char* sym = "plsvo_oracle_atan_match_direct_members";
      if (void* h = dlopen(path, RTLD_NOW | RTLD_LOCAL)) fn = reinterpret_cast<MatchMembersFn>(dlsym(h, sym));
      if (!fn) {
        std::string sib(path);
        sib = sib.substr(0, sib.find_last_of('/') + 1) + "libplsvo_atan_match_oracle.so";
        if (void* h = dlopen(sib.c_str(), RTLD_NOW | RTLD_LOCAL)) fn = reinterpret_cast<MatchMembersFn>(dlsym(h, sym));
      }
      if (!fn) fakecuda::error(std::string("PLSVO_FAKE_ORACLE: no ATAN matcher next to ") + path +
                               " (build oracle/libplsvo_atan_match_oracle.so)");
    }
  }
  return fn;
}

int host_threads() { return (int)std::max(1u, std::thread::hardware_concurrency()); }

// the distortion terms vk::ATANCamera's constructor derives from s_ (oracle/refdeps/vikit/atan_camera.h)
bool terms_of_s(const plsvo::MatchArgs& a) {
  if (a.atan_s == 0.0) return a.atan_s_inv == 0.0 && a.atan_tans == 0.0 && a.atan_tans_inv == 0.0;
  const double tans = 2.0 * tan(a.atan_s / 2.0);
  return a.atan_tans == tans && a.atan_tans_inv == 1.0 / tans && a.atan_s_inv == 1.0 / a.atan_s;
}

// bounds of everything the kernel touches; false (and a recorded model error) on the first violation
bool check_reads(const plsvo::MatchArgs& a) {
  using fakecuda::check;
  const size_t n = (size_t)a.n;
  if (!check(a.ref_index, n * 4, "ATAN match kernel: ref_index") || !check(a.cur_index, n * 4, "ATAN match kernel: cur_index") ||
      !check(a.ref_level, n * 4, "ATAN match kernel: ref_level") || !check(a.ref_px, n * 16, "ATAN match kernel: ref_px") ||
      !check(a.ref_f, n * 24, "ATAN match kernel: ref_f") || !check(a.pos, n * 24, "ATAN match kernel: pos") ||
      !check(a.px_cur, n * 16, "ATAN match kernel: px_cur") || !check(a.out_px, n * 16, "ATAN match kernel: out_px") ||
      !check(a.out_success, n, "ATAN match kernel: out_success") || !check(a.out_level, n * 4, "ATAN match kernel: out_level"))
    return false;
  if (a.is_edgelet && (!check(a.is_edgelet, n, "ATAN match kernel: is_edgelet") || !check(a.ref_grad, n * 16, "ATAN match kernel: ref_grad")))
    return false;
  if (a.out_A && !check(a.out_A, n * 32, "ATAN match kernel: out_A")) return false;
  for (size_t i = 0; i < n; ++i) {
    const int r = a.ref_index[i], c = a.cur_index[i], l = a.ref_level[i];
    if (r < 0 || c < 0 || l < 0 || l >= PLSVO_MAX_LEVELS) {
      fakecuda::error("ATAN match kernel: a candidate refers to a negative frame or a level out of range");
      return false;
    }
    if (!check(a.T_ref_w + 7 * (size_t)r, 56, "ATAN match kernel: keyframe pose") ||
        !check(a.T_cur_w + 7 * (size_t)c, 56, "ATAN match kernel: current-frame pose") ||
        !check(a.ref_img[l] + (size_t)r * a.ref_stride[l], (size_t)(a.height >> l) * a.ref_pitch[l], "ATAN match kernel: keyframe level"))
      return false;
    for (int s = 0; s < a.n_pyr_levels; ++s)
      if (!check(a.cur_img[s] + (size_t)c * a.cur_stride[s], (size_t)(a.height >> s) * a.cur_pitch[s], "ATAN match kernel: current level"))
        return false;
  }
  return true;
}

}  // namespace

namespace plsvo {

cudaError_t match_direct_atan_kernel_launch(const MatchArgs& a0, cudaStream_t s) {
  if (a0.n <= 0) return cudaSuccess;
  const MatchMembersFn orc = oracle_match();
  const char* path = getenv("PLSVO_FAKE_ORACLE");
  if (path && *path && !orc) return cudaErrorNotSupported;
  const MatchArgs a = a0;
  return fakecuda::enqueue(s, [a, orc]() {
    if (!terms_of_s(a)) fakecuda::error("ATAN match kernel: distortion terms are not those vk::ATANCamera derives from s_");
    if (!check_reads(a)) return true;
    const size_t n = (size_t)a.n;
    if (!orc) {
      memcpy(a.out_px, a.px_cur, n * 16), memset(a.out_success, 0, n);
      std::fill(a.out_level, a.out_level + n, -1);
      return true;
    }
    plsvo_match_batch b;
    memset(&b, 0, sizeof b);
    b.n_features = a.n, b.n_ref_images = 1 << 30, b.n_cur_images = 1 << 30, b.n_pyr_levels = a.n_pyr_levels, b.n_iter = a.n_iter;
    b.cam.width = a.width, b.cam.height = a.height;
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
      b.ref_img[l] = a.ref_img[l], b.ref_pitch[l] = a.ref_pitch[l], b.ref_stride[l] = a.ref_stride[l];
      b.cur_img[l] = a.cur_img[l], b.cur_pitch[l] = a.cur_pitch[l], b.cur_stride[l] = a.cur_stride[l];
    }
    b.T_ref_w = a.T_ref_w, b.T_cur_w = a.T_cur_w, b.ref_index = a.ref_index, b.cur_index = a.cur_index, b.ref_px = a.ref_px;
    b.ref_f = a.ref_f, b.ref_level = a.ref_level, b.is_edgelet = a.is_edgelet, b.ref_grad = a.ref_grad, b.pos = a.pos, b.px_cur = a.px_cur;
    memset(a.out_px, 0, n * 16), memset(a.out_success, 0, n), memset(a.out_level, 0, n * 4);
    plsvo_match_result r{a.out_px, a.out_success, a.out_level, a.out_A};
    if (orc(a.fx, a.fy, a.cx, a.cy, a.atan_s, &b, &r, host_threads()) != PLSVO_OK)
      fakecuda::error("the oracle refused the ATAN match batch the host code built");
    return true;
  });
}

}  // namespace plsvo
