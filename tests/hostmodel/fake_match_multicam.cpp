// fake_match_multicam.cpp — model kernel of the per-image-camera findMatchDirect call
// (plsvo_match_direct_multicam_batch_run) for the host-pipeline model.  TEST INFRASTRUCTURE ONLY (see fake_cuda.h).
//
// tests/test_match_multicam_host_cpu.py and tools/preflight_gpu_tests.py link it into a model library of their own, next
// to the stock model kernels and the ATAN matching kernel's model (fake_atan_match.cpp); plsvo_abi.cu reaches it through a
// weak reference.
//
//   digest mode       : every byte the real kernel reads or writes is bounds-checked against the live device blocks — the
//                       per-candidate arrays, the camera index of every referenced image and the camera record it names,
//                       the pose of every referenced keyframe and current frame, the keyframe's reference level and every
//                       level below n_pyr_levels of the current frame, each only inside its camera's region — and every
//                       record must carry the terms its model derives (an ATAN camera's those of vk::ATANCamera from s_, a
//                       pinhole's zero).  The outputs are written as for a candidate that failed the in-frame test.
//   PLSVO_FAKE_ORACLE : the kernel is answered by plsvo_oracle_match_direct_multicam_members
//                       (oracle/multicam_match_oracle.cpp) with the records it receives, looked up in the oracle library
//                       or, when that is the plain oracle, in libplsvo_multicam_match_oracle.so next to it.
#include <dlfcn.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <thread>
#include <vector>

#include "../../pl-svo_b200/csrc/internal.h"
#include "fake_cuda.h"

namespace {

using MembersFn = int (*)(const double*, int, const int32_t*, const int32_t*, const plsvo_match_batch*, const plsvo_match_result*, int);

MembersFn oracle_match() {
  static MembersFn fn = nullptr;
  static bool looked = false;
  if (!looked) {
    looked = true;
    const char* path = getenv("PLSVO_FAKE_ORACLE");
    if (path && *path) {
      const char* sym = "plsvo_oracle_match_direct_multicam_members";
      if (void* h = dlopen(path, RTLD_NOW | RTLD_LOCAL)) fn = reinterpret_cast<MembersFn>(dlsym(h, sym));
      if (!fn) {
        std::string sib(path);
        sib = sib.substr(0, sib.find_last_of('/') + 1) + "libplsvo_multicam_match_oracle.so";
        if (void* h = dlopen(sib.c_str(), RTLD_NOW | RTLD_LOCAL)) fn = reinterpret_cast<MembersFn>(dlsym(h, sym));
      }
      if (!fn) fakecuda::error(std::string("PLSVO_FAKE_ORACLE: no per-image matcher next to ") + path +
                               " (build oracle/libplsvo_multicam_match_oracle.so)");
    }
  }
  return fn;
}

int host_threads() { return (int)std::max(1u, std::thread::hardware_concurrency()); }

// the terms a record's model derives: vk::ATANCamera's constructor from s_ (oracle/refdeps/vikit/atan_camera.h), none for a pinhole
bool terms_of_model(const plsvo::MatchCamRecord& m) {
  if (m.model == PLSVO_CAMERA_PINHOLE || m.s == 0.0) return m.s == 0.0 && m.s_inv == 0.0 && m.tans == 0.0 && m.tans_inv == 0.0;
  const double tans = 2.0 * tan(m.s / 2.0);
  return m.model == PLSVO_CAMERA_ATAN && m.tans == tans && m.tans_inv == 1.0 / tans && m.s_inv == 1.0 / m.s;
}

// bytes of level l of an image seen through m: the camera's rows and columns at the slot's pitch
size_t region(const plsvo::MatchCamRecord& m, int l, uint32_t pitch) {
  const int w = m.width >> l, h = m.height >> l;
  return (w <= 0 || h <= 0) ? 1 : (size_t)(h - 1) * pitch + (size_t)w;
}

// bounds of everything the kernel touches; false (and a recorded model error) on the first violation.  *n_cams, *n_ref
// and *n_cur are one past the largest camera, keyframe and current frame a candidate refers to.
bool check_reads(const plsvo::MatchArgs& a, int* n_cams, int* n_ref, int* n_cur) {
  using fakecuda::check;
  const size_t n = (size_t)a.n;
  const char* K = "multicam match kernel: ";
  auto chk = [&](const void* p, size_t bytes, const char* what) { return check(p, bytes, (std::string(K) + what).c_str()); };
  if (!chk(a.ref_index, n * 4, "ref_index") || !chk(a.cur_index, n * 4, "cur_index") || !chk(a.ref_level, n * 4, "ref_level") ||
      !chk(a.ref_px, n * 16, "ref_px") || !chk(a.ref_f, n * 24, "ref_f") || !chk(a.pos, n * 24, "pos") || !chk(a.px_cur, n * 16, "px_cur") ||
      !chk(a.out_px, n * 16, "out_px") || !chk(a.out_success, n, "out_success") || !chk(a.out_level, n * 4, "out_level"))
    return false;
  if (a.is_edgelet && (!chk(a.is_edgelet, n, "is_edgelet") || !chk(a.ref_grad, n * 16, "ref_grad"))) return false;
  if (a.out_A && !chk(a.out_A, n * 32, "out_A")) return false;
  *n_cams = *n_ref = *n_cur = 0;
  for (size_t i = 0; i < n; ++i) {
    const int r = a.ref_index[i], c = a.cur_index[i], l = a.ref_level[i];
    if (r < 0 || c < 0 || l < 0 || l >= PLSVO_MAX_LEVELS) {
      fakecuda::error(std::string(K) + "a candidate refers to a negative frame or a level out of range");
      return false;
    }
    if (!chk(a.cam_of_ref + r, 4, "cam_of_ref") || !chk(a.cam_of_cur + c, 4, "cam_of_cur")) return false;
    const int kr = a.cam_of_ref[r], kc = a.cam_of_cur[c];
    if (kr < 0 || kc < 0 || !chk(a.cams + kr, sizeof(plsvo::MatchCamRecord), "camera record of a keyframe") ||
        !chk(a.cams + kc, sizeof(plsvo::MatchCamRecord), "camera record of a current frame"))
      return false;
    const plsvo::MatchCamRecord &mr = a.cams[kr], &mc = a.cams[kc];
    if (!terms_of_model(mr) || !terms_of_model(mc)) {
      fakecuda::error(std::string(K) + "a camera record does not carry the terms its model derives");
      return false;
    }
    if (mr.width > a.width || mr.height > a.height || mc.width > a.width || mc.height > a.height) {
      fakecuda::error(std::string(K) + "a camera record is larger than the slot");
      return false;
    }
    if (!chk(a.T_ref_w + 7 * (size_t)r, 56, "keyframe pose") || !chk(a.T_cur_w + 7 * (size_t)c, 56, "current-frame pose") ||
        !chk(a.ref_img[l] + (size_t)r * a.ref_stride[l], region(mr, l, a.ref_pitch[l]), "keyframe level inside its camera"))
      return false;
    for (int s = 0; s < a.n_pyr_levels; ++s)
      if (!chk(a.cur_img[s] + (size_t)c * a.cur_stride[s], region(mc, s, a.cur_pitch[s]), "current level inside its camera")) return false;
    *n_cams = std::max(*n_cams, std::max(kr, kc) + 1), *n_ref = std::max(*n_ref, r + 1), *n_cur = std::max(*n_cur, c + 1);
  }
  return true;
}

}  // namespace

namespace plsvo {

cudaError_t match_direct_multicam_kernel_launch(const MatchArgs& a0, cudaStream_t s) {
  if (a0.n <= 0) return cudaSuccess;
  const MembersFn orc = oracle_match();
  const char* path = getenv("PLSVO_FAKE_ORACLE");
  if (path && *path && !orc) return cudaErrorNotSupported;
  const MatchArgs a = a0;
  return fakecuda::enqueue(s, [a, orc]() {
    int n_cams, n_ref, n_cur;
    if (!check_reads(a, &n_cams, &n_ref, &n_cur)) return true;
    const size_t n = (size_t)a.n;
    if (!orc) {
      memcpy(a.out_px, a.px_cur, n * 16), memset(a.out_success, 0, n);
      std::fill(a.out_level, a.out_level + n, -1);
      return true;
    }
    std::vector<double> members(8 * (size_t)n_cams);
    for (int k = 0; k < n_cams; ++k) {
      const MatchCamRecord& m = a.cams[k];
      const double row[8] = {(double)m.model, (double)m.width, (double)m.height, m.fx, m.fy, m.cx, m.cy, m.s};
      std::copy(row, row + 8, members.begin() + 8 * k);
    }
    plsvo_match_batch b;
    memset(&b, 0, sizeof b);
    b.n_features = a.n, b.n_ref_images = n_ref, b.n_cur_images = n_cur, b.n_pyr_levels = a.n_pyr_levels, b.n_iter = a.n_iter;
    b.cam.width = a.width, b.cam.height = a.height;
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
      b.ref_img[l] = a.ref_img[l], b.ref_pitch[l] = a.ref_pitch[l], b.ref_stride[l] = a.ref_stride[l];
      b.cur_img[l] = a.cur_img[l], b.cur_pitch[l] = a.cur_pitch[l], b.cur_stride[l] = a.cur_stride[l];
    }
    b.T_ref_w = a.T_ref_w, b.T_cur_w = a.T_cur_w, b.ref_index = a.ref_index, b.cur_index = a.cur_index, b.ref_px = a.ref_px;
    b.ref_f = a.ref_f, b.ref_level = a.ref_level, b.is_edgelet = a.is_edgelet, b.ref_grad = a.ref_grad, b.pos = a.pos, b.px_cur = a.px_cur;
    memset(a.out_px, 0, n * 16), memset(a.out_success, 0, n), memset(a.out_level, 0, n * 4);
    plsvo_match_result r{a.out_px, a.out_success, a.out_level, a.out_A};
    if (orc(members.data(), n_cams, a.cam_of_ref, a.cam_of_cur, &b, &r, host_threads()) != PLSVO_OK)
      fakecuda::error("the oracle refused the per-image match batch the host code built");
    return true;
  });
}

}  // namespace plsvo
