// fake_kernels.cpp — model kernels for the host-pipeline tests.  TEST INFRASTRUCTURE ONLY (see fake_cuda.h).
//
// The launch entry points of pl-svo_b200/csrc/internal.h, implemented on the host: each "kernel" is queued on its stream
// in the model runtime and, when it runs, checks that every byte the real kernel would read lies inside a device block
// and folds those bytes into a digest per work item.  The digest comes back through the ordinary output arrays, so a test
// sees — through the unchanged C ABI and Python mirror — exactly which bytes the host code presented to the kernel:
//
//   alignment : out_n_tracked[b] = digest of pair b, as (h >> 1) | 1 (image levels min..max of both frames, poses, counts, every feature
//               array that was shipped); out_H[b][2*(l-min_level)+{0,1}] = digest of the ref / cur level l alone (top 52
//               bits, exact in a double); out_T[b] = T_cur_w[b]; out_patch_iters/levels = the pair's feature counts.
//               Levels that the real kernel derives itself (AlignArgs::derive_from) are derived here the same way; the
//               arrival gate is honoured pair by pair, advancing the other streams only as far as the gate requires.
//   pyramid   : the real computation (truncating 2x2 mean), it is the producer of derived levels.
//               The ATAN kernels (align_atan_kernel_*) are the same model: the camera model changes no byte they read.
//   pose-opt  : out_num_pt[b] = digest of frame b's inputs; out_T[b] = T_f_w[b].
//   the next-row kernels exist in the oracle-backed mode only (below); otherwise they report cudaErrorNotSupported.
//
// The same digest is restated in NumPy in tests/hostmodel/scenarios.py, from the caller's arrays.
//
// Second mode, PLSVO_FAKE_ORACLE=<path of oracle/libplsvo_oracle.so>: every "kernel" hands its
// device-layout arguments to the CPU oracle instead of digesting them, so that the GPU tier's own test files can be run
// here against the unchanged host code (a pre-flight of those files and of the host paths they take, never a parity
// statement: oracle is compared with oracle).  Inputs the oracle cannot take (depth-only features, bearings not shipped)
// are refused with cudaErrorNotSupported.  The ATAN kernels are answered by the oracle's ATAN path
// (plsvo_oracle_atan_align_batch_members, oracle/atan_oracle.cpp), looked up in the same library or, when that is the plain
// oracle, in libplsvo_atan_oracle.so next to it; it forms NULL bearings itself, as the ATAN kernels do.
#include <dlfcn.h>
#include <string.h>

#include <thread>
#include <vector>

#include <memory>

#include "../../pl-svo_b200/csrc/internal.h"
#include "fake_cuda.h"

namespace {

constexpr uint64_t K = 0x9E3779B97F4A7C15ull;

// position- and value-sensitive, vectorisable: sum over i of (byte_i + 1) * ((i + 1) * K)   (mod 2^64)
uint64_t dig_bytes(const void* p, size_t n, uint64_t first_index = 0) {
  const uint8_t* b = static_cast<const uint8_t*>(p);
  uint64_t h = 0;
  for (size_t i = 0; i < n; ++i) h += (uint64_t)(b[i] + 1u) * ((first_index + i + 1) * K);
  return h;
}

uint64_t mix(uint64_t h, uint64_t v) {
  h ^= v + K + (h << 6) + (h >> 2);
  return h;
}

// rows x cols bytes of a pitched image, indexed row-major over the visible pixels only
uint64_t dig_image(const uint8_t* img, int rows, int cols, size_t pitch) {
  uint64_t h = 0;
  for (int y = 0; y < rows; ++y) h += dig_bytes(img + (size_t)y * pitch, (size_t)cols, (uint64_t)y * cols);
  return h;
}

void half_sample(const uint8_t* src, size_t pin, uint8_t* dst, size_t pout, int rows, int cols) {
  for (int y = 0; y < rows; ++y) {
    const uint8_t* r0 = src + (size_t)(2 * y) * pin;
    for (int x = 0; x < cols; ++x)
      dst[(size_t)y * pout + x] = (uint8_t)(((int)r0[2 * x] + (int)r0[2 * x + 1] + (int)r0[pin + 2 * x] + (int)r0[pin + 2 * x + 1]) >> 2);
  }
}

template <class T>
uint64_t dig_array(uint64_t h, const T* base, size_t first, size_t count, const char* what) {
  if (!base) return mix(h, 0x5151);  // array not shipped
  const T* p = base + first;
  if (!fakecuda::check(p, count * sizeof(T), what)) return mix(h, 0xDEAD);
  return mix(h, dig_bytes(p, count * sizeof(T)));
}

struct AlignRun {
  plsvo::AlignArgs a;
  cudaStream_t stream;
  int next = 0;
};

// device-side level derivation of pair b (what the real kernel does before it touches the pair)
void derive_pair_levels(const plsvo::AlignArgs& a, int b) {
  if (a.derive_from < 0) return;
  for (int l = a.derive_from + 1; l <= a.max_level; ++l) {
    const int cols = a.width >> l, rows = a.height >> l;
    for (int which = 0; which < 2; ++which) {
      const uint8_t* src = (which ? a.cur_img[l - 1] : a.ref_img[l - 1]) + (size_t)b * a.stride[l - 1];
      uint8_t* dst = const_cast<uint8_t*>(which ? a.cur_img[l] : a.ref_img[l]) + (size_t)b * a.stride[l];
      if (!fakecuda::check(src, a.stride[l - 1], "align kernel: source level of a derived level") ||
          !fakecuda::check(dst, a.stride[l], "align kernel: derived level"))
        return;
      half_sample(src, a.pitch[l - 1], dst, a.pitch[l], rows, cols);
    }
  }
}

bool align_pair(const plsvo::AlignArgs& a, int b) {
  using fakecuda::check;
  bool ok = true;
  derive_pair_levels(a, b);  // levels the kernel forms itself from the finest shipped one (gated host pipeline)
  uint64_t h = 0;
  for (int i = 0; i < 36; ++i) a.out_H[(size_t)b * 36 + i] = 0.0;
  for (int l = a.min_level; l <= a.max_level; ++l) {
    const int cols = a.width >> l, rows = a.height >> l;
    if (!a.ref_img[l] || !a.cur_img[l] || !a.pitch[l]) {
      fakecuda::error("align kernel: a level in [min_level, max_level] has no image");
      return false;
    }
    if (a.pitch[l] % 4 != 0 || a.stride[l] % 16 != 0) fakecuda::error("align kernel: level pitch / stride not word / 16-byte aligned");
    const uint8_t* r = a.ref_img[l] + (size_t)b * a.stride[l];
    const uint8_t* c = a.cur_img[l] + (size_t)b * a.stride[l];
    ok &= check(r, a.stride[l], "align kernel: reference image level");
    ok &= check(c, a.stride[l], "align kernel: current image level");
    if (!ok) return false;
    const uint64_t hr = dig_image(r, rows, cols, a.pitch[l]), hc = dig_image(c, rows, cols, a.pitch[l]);
    h = mix(mix(h, hr), hc);
    const int k = 2 * (l - a.min_level);
    if (k + 1 < 36) a.out_H[(size_t)b * 36 + k] = (double)(hr >> 12), a.out_H[(size_t)b * 36 + k + 1] = (double)(hc >> 12);
  }
  const size_t np_ = (size_t)a.n_pts, ns_ = (size_t)a.n_segs;
  const int np = a.pt_count ? a.pt_count[b] : a.n_pts, ns = a.seg_count ? a.seg_count[b] : a.n_segs;
  if (np < 0 || np > a.n_pts || ns < 0 || ns > a.n_segs) {
    fakecuda::error("align kernel: feature count outside [0, n]");
    return false;
  }
  h = dig_array(h, a.T_ref_w, (size_t)b * 7, 7, "T_ref_w");
  h = dig_array(h, a.T_cur_w, (size_t)b * 7, 7, "T_cur_w");
  h = mix(h, (uint64_t)np * 65536u + (uint64_t)ns);
  h = dig_array(h, a.pt_px, b * np_ * 2, (size_t)np * 2, "pt_px");
  h = dig_array(h, a.pt_f, b * np_ * 3, (size_t)np * 3, "pt_f");
  h = dig_array(h, a.pt_pos, b * np_ * 3, (size_t)np * 3, "pt_pos");
  h = dig_array(h, a.pt_depth, b * np_, (size_t)np, "pt_depth");
  h = dig_array(h, a.pt_valid, b * np_, (size_t)np, "pt_valid");
  h = dig_array(h, a.seg_spx, b * ns_ * 2, (size_t)ns * 2, "seg_spx");
  h = dig_array(h, a.seg_epx, b * ns_ * 2, (size_t)ns * 2, "seg_epx");
  h = dig_array(h, a.seg_sf, b * ns_ * 3, (size_t)ns * 3, "seg_sf");
  h = dig_array(h, a.seg_ef, b * ns_ * 3, (size_t)ns * 3, "seg_ef");
  h = dig_array(h, a.seg_spos, b * ns_ * 3, (size_t)ns * 3, "seg_spos");
  h = dig_array(h, a.seg_epos, b * ns_ * 3, (size_t)ns * 3, "seg_epos");
  h = dig_array(h, a.seg_sdepth, b * ns_, (size_t)ns, "seg_sdepth");
  h = dig_array(h, a.seg_edepth, b * ns_, (size_t)ns, "seg_edepth");
  h = dig_array(h, a.seg_length, b * ns_, (size_t)ns, "seg_length");
  h = dig_array(h, a.seg_valid, b * ns_, (size_t)ns, "seg_valid");
  // outputs, every one of them range-checked like an input
  ok &= check(a.out_T + (size_t)b * 7, 56, "out_T") && check(a.out_n_tracked + b, 8, "out_n_tracked") &&
        check(a.out_H + (size_t)b * 36, 288, "out_H") && check(a.out_iters + (size_t)b * PLSVO_MAX_LEVELS, 4 * PLSVO_MAX_LEVELS, "out_iters") &&
        check(a.out_status + b, 4, "out_status") && check(a.out_patch_iters + b, 4, "out_patch_iters") &&
        check(a.out_patch_levels + b, 4, "out_patch_levels");
  if (a.n_segs > 0) ok &= check(a.out_seg_killed + b * ns_, ns_, "out_seg_killed");
  if (!ok) return false;
  for (int i = 0; i < 7; ++i) a.out_T[(size_t)b * 7 + i] = a.T_cur_w ? a.T_cur_w[(size_t)b * 7 + i] : 0.0;
  a.out_n_tracked[b] = (long long)((h >> 1) | 1u);  // positive, like a count of tracked patches
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) a.out_iters[(size_t)b * PLSVO_MAX_LEVELS + l] = (l >= a.min_level && l <= a.max_level) ? 1 : 0;
  a.out_status[b] = 0;
  a.out_patch_iters[b] = (uint32_t)np;
  a.out_patch_levels[b] = (uint32_t)ns;
  for (int j = 0; j < a.n_segs; ++j) a.out_seg_killed[b * ns_ + j] = 0;
  return true;
}

// ---- PLSVO_FAKE_ORACLE: the CPU oracle behind the launch entry points ----
struct OracleApi {
  int (*align)(const plsvo_align_batch*, const plsvo_align_params*, const plsvo_align_result*, int, int) = nullptr;
  int (*poseopt)(const plsvo_poseopt_batch*, const plsvo_poseopt_params*, const plsvo_poseopt_result*, int) = nullptr;
  int (*align2d)(const plsvo_align2d_batch*, const plsvo_align2d_result*, int) = nullptr;
  int (*align1d)(const plsvo_align1d_batch*, const plsvo_align1d_result*, int) = nullptr;
  int (*match)(const plsvo_match_batch*, const plsvo_match_result*, int) = nullptr;
  int (*structopt)(const plsvo_structopt_batch*, const plsvo_structopt_result*, int) = nullptr;
  int (*seed)(const plsvo_seed_batch*, const plsvo_seed_result*, int) = nullptr;
  int (*line_seed)(const plsvo_line_seed_batch*, const plsvo_line_seed_result*, int) = nullptr;
  // optional: the ATAN alignment, camera given by its members fx_, fy_, cx_, cy_ and d0
  int (*atan_align)(double, double, double, double, double, const plsvo_align_batch*, const plsvo_align_params*,
                    const plsvo_align_result*, int) = nullptr;
};

const OracleApi* oracle() {
  static OracleApi api;
  static int state = 0;  // 0: not looked up, 1: loaded, -1: digest mode
  if (state == 0) {
    state = -1;
    const char* path = getenv("PLSVO_FAKE_ORACLE");
    if (path && *path) {
      void* h = dlopen(path, RTLD_NOW | RTLD_LOCAL);
      if (h) {
        api.align = reinterpret_cast<decltype(api.align)>(dlsym(h, "plsvo_oracle_align_batch"));
        api.poseopt = reinterpret_cast<decltype(api.poseopt)>(dlsym(h, "plsvo_oracle_poseopt_batch"));
        api.align2d = reinterpret_cast<decltype(api.align2d)>(dlsym(h, "plsvo_oracle_align2d_batch"));
        api.align1d = reinterpret_cast<decltype(api.align1d)>(dlsym(h, "plsvo_oracle_align1d_batch"));
        api.match = reinterpret_cast<decltype(api.match)>(dlsym(h, "plsvo_oracle_match_direct_batch"));
        api.structopt = reinterpret_cast<decltype(api.structopt)>(dlsym(h, "plsvo_oracle_structopt_batch"));
        api.seed = reinterpret_cast<decltype(api.seed)>(dlsym(h, "plsvo_oracle_seed_update_batch"));
        api.line_seed = reinterpret_cast<decltype(api.line_seed)>(dlsym(h, "plsvo_oracle_line_seed_update_batch"));
        const char* atan_sym = "plsvo_oracle_atan_align_batch_members";
        api.atan_align = reinterpret_cast<decltype(api.atan_align)>(dlsym(h, atan_sym));
        if (!api.atan_align) {
          std::string sib(path);
          sib = sib.substr(0, sib.find_last_of('/') + 1) + "libplsvo_atan_oracle.so";
          if (void* ha = dlopen(sib.c_str(), RTLD_NOW | RTLD_LOCAL))
            api.atan_align = reinterpret_cast<decltype(api.atan_align)>(dlsym(ha, atan_sym));
        }
      }
      if (api.align && api.poseopt && api.align2d && api.align1d && api.match && api.structopt && api.seed && api.line_seed) state = 1;
      else fakecuda::error(std::string("PLSVO_FAKE_ORACLE: cannot load the oracle from ") + path);
    }
  }
  return state == 1 ? &api : nullptr;
}

int host_threads() { return (int)std::max(1u, std::thread::hardware_concurrency()); }

void align_by_oracle(const OracleApi* o, const plsvo::AlignArgs& a, bool atan) {
  plsvo_align_batch b;
  memset(&b, 0, sizeof b);
  b.batch = a.B, b.n_pts = a.n_pts, b.n_segs = a.n_segs;
  b.cam.width = a.width, b.cam.height = a.height, b.cam.fx = a.fx, b.cam.fy = a.fy, b.cam.cx = a.cx, b.cam.cy = a.cy;
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
    if (!a.pitch[l] || !a.ref_img[l] || !a.cur_img[l]) continue;
    b.ref_img[l] = a.ref_img[l], b.cur_img[l] = a.cur_img[l], b.img_pitch[l] = a.pitch[l], b.img_stride[l] = a.stride[l];
  }
  b.T_ref_w = a.T_ref_w, b.T_cur_w = a.T_cur_w;
  b.pt_count = a.pt_count, b.pt_px = a.pt_px, b.pt_f = a.pt_f, b.pt_pos = a.pt_pos, b.pt_valid = a.pt_valid;
  b.seg_count = a.seg_count, b.seg_spx = a.seg_spx, b.seg_epx = a.seg_epx, b.seg_sf = a.seg_sf, b.seg_ef = a.seg_ef;
  b.seg_spos = a.seg_spos, b.seg_epos = a.seg_epos, b.seg_length = a.seg_length, b.seg_valid = a.seg_valid;
  plsvo_align_params p;
  memset(&p, 0, sizeof p);
  p.max_level = a.max_level, p.min_level = a.min_level, p.n_iter = a.n_iter, p.eps = a.eps;
  plsvo_align_result r;
  memset(&r, 0, sizeof r);
  r.T_cur_w = a.out_T, r.n_tracked = reinterpret_cast<int64_t*>(a.out_n_tracked), r.H = a.out_H;
  r.seg_killed = a.n_segs > 0 ? a.out_seg_killed : nullptr, r.iters = a.out_iters, r.status = a.out_status;
  r.patch_iters = a.out_patch_iters, r.patch_levels = a.out_patch_levels;
  const size_t B = (size_t)a.B;
  // the oracle's callers hand it zeroed outputs (abi.AlignOut)
  memset(a.out_T, 0, B * 56), memset(a.out_n_tracked, 0, B * 8), memset(a.out_H, 0, B * 288);
  memset(a.out_iters, 0, B * 4 * PLSVO_MAX_LEVELS), memset(a.out_status, 0, B * 4);
  memset(a.out_patch_iters, 0, B * 4), memset(a.out_patch_levels, 0, B * 4);
  if (a.n_segs > 0) memset(a.out_seg_killed, 0, B * (size_t)a.n_segs);
  const int rc = atan ? o->atan_align(a.fx, a.fy, a.cx, a.cy, a.atan_s, &b, &p, &r, host_threads()) : o->align(&b, &p, &r, host_threads(), 0);
  if (rc != PLSVO_OK) fakecuda::error("the oracle refused the alignment batch the host code built");
}

void poseopt_by_oracle(const OracleApi* o, const plsvo::PoseOptArgs& a) {
  plsvo_poseopt_batch b;
  memset(&b, 0, sizeof b);
  b.batch = a.B, b.n_pts = a.n_pts, b.n_segs = a.n_segs, b.fx = a.fx;
  b.T_f_w = a.T_f_w, b.pt_count = a.pt_count, b.pt_f = a.pt_f, b.pt_pos = a.pt_pos, b.pt_level = a.pt_level, b.pt_valid = a.pt_valid;
  b.seg_count = a.seg_count, b.seg_line = a.seg_line, b.seg_spos = a.seg_spos, b.seg_epos = a.seg_epos, b.seg_level = a.seg_level;
  b.seg_valid = a.seg_valid;
  plsvo_poseopt_params p;
  memset(&p, 0, sizeof p);
  p.reproj_thresh = a.reproj_thresh, p.n_iter = a.n_iter, p.n_iter_ref = a.n_iter_ref;
  plsvo_poseopt_result r;
  memset(&r, 0, sizeof r);
  r.T_f_w = a.out_T, r.cov = a.out_cov, r.estimated_scale = a.out_scale, r.error_init = a.out_err_init, r.error_final = a.out_err_final;
  r.num_obs_pt = reinterpret_cast<int64_t*>(a.out_num_pt), r.num_obs_ls = reinterpret_cast<int64_t*>(a.out_num_ls);
  r.pt_outlier = a.out_pt_outlier, r.seg_outlier = a.n_segs > 0 ? a.out_seg_outlier : nullptr, r.iters = a.out_iters, r.status = a.out_status;
  const size_t B = (size_t)a.B;
  // what the real kernel always writes and the oracle may leave alone: start from zeros (abi.PoseOptOut) and the input pose
  memcpy(a.out_T, a.T_f_w, B * 56);
  memset(a.out_pt_outlier, 0, B * (size_t)std::max(1, a.n_pts)), memset(a.out_seg_outlier, 0, B * (size_t)std::max(1, a.n_segs));
  memset(a.out_iters, 0, B * 8), memset(a.out_status, 0, B * 4);
  const int rc = o->poseopt(&b, &p, &r, host_threads());
  if (rc != PLSVO_OK) fakecuda::error("the oracle refused the pose-optimiser batch the host code built");
}

}  // namespace

namespace plsvo {

// Same structure as make_layout() in align_kernel.cu (which is device code and cannot be compiled here); only the plan's
// decisions depend on it (variant choice, image staging), none of which the digest kernel looks at.
size_t align_smem_bytes(int n_pts, int n_segs, int max_patches, int max_seg_slots, int img_bytes, int threads) {
  const size_t nw = (size_t)threads / 32, chunks = ((size_t)n_pts + 31) / 32, rounds = ((size_t)n_pts + threads - 1) / threads;
  size_t o = 1024;                                   // control block
  o += nw * 256 + 256 + 8 * (rounds * nw + 1);       // reduction scratch, chunk totals
  o += 256 * (chunks + 1) + 4 * (chunks + 1) + 512;  // chi2 items
  o += 64 * (size_t)align_opq_cap(n_pts);            // opaque patches
  o += 21 * (size_t)n_segs + 2 * (size_t)max_seg_slots + (size_t)n_pts;
  o += 24 * (size_t)max_patches + 64 * (size_t)threads;
  o = (o + 127) / 128 * 128;
  return o + (size_t)img_bytes + 16;
}

cudaError_t align_kernel_prepare(int threads, int min_blocks, size_t smem_bytes, int* ctas_per_sm) {
  (void)threads;
  *ctas_per_sm = (int)std::min<size_t>((size_t)min_blocks, (232448 + 1024) / (smem_bytes + 1024));
  return cudaSuccess;
}

cudaError_t weight_selftest_launch(uint32_t, uint32_t, unsigned long long* d_mismatch, cudaStream_t s) {
  return fakecuda::enqueue(s, [d_mismatch]() {
    if (fakecuda::check(d_mismatch, 8, "selftest counter")) *d_mismatch = 0;
    return true;
  });
}

// the pinhole and the ATAN kernels (atan: AlignArgs::fx..cy hold the members fx_..cy_, atan_s is d0)
static cudaError_t launch_align(const AlignArgs& a, int grid, int threads, int min_blocks, size_t smem_bytes, cudaStream_t s, bool atan) {
  if (grid < 1 || threads < 32 || min_blocks < 1 || smem_bytes > 232448) {
    fakecuda::error("align_kernel_launch: launch configuration out of range");
    return cudaErrorInvalidConfiguration;
  }
  const OracleApi* orc = oracle();
  if (orc && atan && !orc->atan_align) {
    fakecuda::error("oracle-backed model kernel: the oracle library has no ATAN path (build oracle/libplsvo_atan_oracle.so)");
    return cudaErrorNotSupported;
  }
  // the ATAN oracle forms NULL bearings with the camera's cam2world, as the ATAN kernels do; the pinhole oracle cannot
  const bool no_bearings = !atan && ((a.n_pts > 0 && !a.pt_f) || (a.n_segs > 0 && (!a.seg_sf || !a.seg_ef)));
  if (orc && (no_bearings || (a.n_pts > 0 && !a.pt_pos) || (a.n_segs > 0 && (!a.seg_spos || !a.seg_epos)))) {
    // depth-only features / bearings not shipped are outside the oracle's inputs: refused, unless the caller asked for the
    // digest kernel on such batches (the bench pre-flight, whose end-to-end legs ship lean inputs)
    if (!getenv("PLSVO_FAKE_LEAN_DIGEST")) {
      fakecuda::error("oracle-backed model kernel: depth-only features / bearings not shipped are outside the oracle's inputs");
      return cudaErrorNotSupported;
    }
    orc = nullptr;
  }
  auto run = std::make_shared<AlignRun>();
  run->a = a, run->stream = s;
  return fakecuda::enqueue(s, [run, orc, atan]() {
    const AlignArgs& a = run->a;
    if (run->next == 0) {
      if (!fakecuda::check(a.work_counter, 4, "work counter")) return true;
      if (*a.work_counter != 0) fakecuda::error("align kernel: work counter not cleared before the launch");
    }
    while (run->next < a.B) {
      const int b = run->next;
      if (a.gate_chunk > 0) {
        if (!fakecuda::check(a.arrived, 4, "arrival counter")) return true;
        const unsigned need = (unsigned)(b / a.gate_chunk) + 1u;
        while (*a.arrived < need)
          if (!fakecuda::advance_others(run->stream)) return false;  // blocked: this pair's chunk is still in flight
      }
      if (orc) derive_pair_levels(a, b);
      else align_pair(a, b);
      run->next = b + 1;
      *a.work_counter = (unsigned)run->next;
    }
    if (orc) align_by_oracle(orc, a, atan);
    return true;
  });
}

cudaError_t align_kernel_launch(const AlignArgs& a, int grid, int threads, int min_blocks, size_t smem_bytes, cudaStream_t s) {
  return launch_align(a, grid, threads, min_blocks, smem_bytes, s, false);
}

cudaError_t align_atan_kernel_prepare(int threads, int min_blocks, size_t smem_bytes, int* ctas_per_sm) {
  return align_kernel_prepare(threads, min_blocks, smem_bytes, ctas_per_sm);
}

cudaError_t align_atan_kernel_launch(const AlignArgs& a, int grid, int threads, int min_blocks, size_t smem_bytes, cudaStream_t s) {
  return launch_align(a, grid, threads, min_blocks, smem_bytes, s, true);
}

size_t poseopt_smem_bytes(int n_pts, int n_segs) { return 4096 + 24 * ((size_t)n_pts + (size_t)n_segs); }

cudaError_t poseopt_kernel_launch(const PoseOptArgs& a0, size_t, cudaStream_t s) {
  const PoseOptArgs a = a0;
  if (const OracleApi* orc = oracle())
    return fakecuda::enqueue(s, [a, orc]() {
      poseopt_by_oracle(orc, a);
      return true;
    });
  return fakecuda::enqueue(s, [a]() {
    const size_t np_ = (size_t)a.n_pts, ns_ = (size_t)a.n_segs;
    for (int b = 0; b < a.B; ++b) {
      const int np = a.pt_count ? a.pt_count[b] : a.n_pts, ns = a.seg_count ? a.seg_count[b] : a.n_segs;
      uint64_t h = dig_array<double>(0, a.T_f_w, (size_t)b * 7, 7, "T_f_w");
      h = mix(h, (uint64_t)np * 65536u + (uint64_t)ns);
      h = dig_array(h, a.pt_f, b * np_ * 3, (size_t)np * 3, "pt_f");
      h = dig_array(h, a.pt_pos, b * np_ * 3, (size_t)np * 3, "pt_pos");
      h = dig_array(h, a.pt_level, b * np_, (size_t)np, "pt_level");
      h = dig_array(h, a.pt_valid, b * np_, (size_t)np, "pt_valid");
      h = dig_array(h, a.seg_line, b * ns_ * 3, (size_t)ns * 3, "seg_line");
      h = dig_array(h, a.seg_spos, b * ns_ * 3, (size_t)ns * 3, "seg_spos");
      h = dig_array(h, a.seg_epos, b * ns_ * 3, (size_t)ns * 3, "seg_epos");
      h = dig_array(h, a.seg_level, b * ns_, (size_t)ns, "seg_level");
      h = dig_array(h, a.seg_valid, b * ns_, (size_t)ns, "seg_valid");
      if (!fakecuda::check(a.out_T + (size_t)b * 7, 56, "poseopt out_T") || !fakecuda::check(a.out_num_pt + b, 8, "poseopt out_num_pt") ||
          !fakecuda::check(a.out_status + b, 4, "poseopt out_status"))
        return true;
      for (int i = 0; i < 7; ++i) a.out_T[(size_t)b * 7 + i] = a.T_f_w[(size_t)b * 7 + i];
      a.out_num_pt[b] = (long long)((h >> 1) | 1u);
      a.out_status[b] = 0;
    }
    return true;
  });
}

cudaError_t pyramid_kernel_launch(const PyramidArgs& a0, cudaStream_t s) {
  const PyramidArgs a = a0;
  // what the real kernel cannot run: one 64x64 level-0 tile per CTA holds levels 0..6 (level 7 would be left unwritten),
  // and the frames sit on gridDim.z (at most 65535)
  if (a.n_levels < 1 || a.n_levels > 7) {
    fakecuda::error("pyramid kernel: n_levels " + std::to_string(a.n_levels) + " outside [1,7]");
    return cudaErrorInvalidValue;
  }
  if (a.B < 1 || a.B > 65535) {
    fakecuda::error("pyramid kernel: B " + std::to_string(a.B) + " outside [1,65535] (gridDim.z)");
    return cudaErrorInvalidConfiguration;
  }
  // level 0 is read with 16-byte loads up to its pitch, levels 1.. are written with 8- and 4-byte stores: every level's
  // base, pitch and frame stride must be a multiple of 16
  for (int l = 0; l < a.n_levels; ++l)
    if (reinterpret_cast<uintptr_t>(a.level[l]) % 16 != 0 || a.pitch[l] % 16 != 0 || a.stride[l] % 16 != 0) {
      fakecuda::error("pyramid kernel: level " + std::to_string(l) + " base, pitch or stride is not a multiple of 16");
      return cudaErrorMisalignedAddress;
    }
  return fakecuda::enqueue(s, [a]() {
    for (int b = 0; b < a.B; ++b)
      for (int l = 1; l < a.n_levels; ++l) {
        const int cols = a.width >> l, rows = a.height >> l;
        const uint8_t* src = a.level[l - 1] + (size_t)b * a.stride[l - 1];
        uint8_t* dst = a.level[l] + (size_t)b * a.stride[l];
        const size_t sspan = (size_t)(2 * rows - 1) * a.pitch[l - 1] + 2 * (size_t)cols;
        const size_t dspan = (size_t)(rows - 1) * a.pitch[l] + (size_t)cols;
        if (rows <= 0 || cols <= 0) continue;
        if (!fakecuda::check(src, sspan, "pyramid kernel: source level") || !fakecuda::check(dst, dspan, "pyramid kernel: destination level"))
          return true;
        half_sample(src, a.pitch[l - 1], dst, a.pitch[l], rows, cols);
      }
    return true;
  });
}

// ---- the next-row kernels: oracle-backed only (their host code is plain upload -> launch -> download) ----
static void fill_align2d(const Align2DArgs& a, plsvo_align2d_batch* b) {
  memset(b, 0, sizeof *b);
  b->n_features = a.n, b->n_images = 1 << 30, b->width = a.width, b->height = a.height, b->n_iter = a.n_iter;
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) b->img[l] = a.img[l], b->img_pitch[l] = a.pitch[l], b->img_stride[l] = a.stride[l];
  b->image_index = a.image_index, b->level = a.level, b->ref_patch_with_border = a.ref_patch_with_border, b->ref_patch = a.ref_patch;
  b->px = a.px;
}

cudaError_t align2d_kernel_launch(const Align2DArgs& a0, cudaStream_t s) {
  const OracleApi* o = oracle();
  if (!o) return cudaErrorNotSupported;
  const Align2DArgs a = a0;
  return fakecuda::enqueue(s, [a, o]() {
    plsvo_align2d_batch b;
    fill_align2d(a, &b);
    memset(a.out_px, 0, (size_t)a.n * 16), memset(a.out_converged, 0, (size_t)a.n);
    plsvo_align2d_result r{a.out_px, a.out_converged};
    if (o->align2d(&b, &r, host_threads()) != PLSVO_OK) fakecuda::error("the oracle refused the align2D batch the host code built");
    return true;
  });
}

cudaError_t align1d_kernel_launch(const Align2DArgs& a0, cudaStream_t s) {
  const OracleApi* o = oracle();
  if (!o) return cudaErrorNotSupported;
  const Align2DArgs a = a0;
  return fakecuda::enqueue(s, [a, o]() {
    plsvo_align1d_batch b;
    memset(&b, 0, sizeof b);
    fill_align2d(a, &b.features);
    b.dir = a.dir;
    memset(a.out_px, 0, (size_t)a.n * 16), memset(a.out_converged, 0, (size_t)a.n), memset(a.out_h_inv, 0, (size_t)a.n * 8);
    plsvo_align1d_result r{a.out_px, a.out_converged, a.out_h_inv};
    if (o->align1d(&b, &r, host_threads()) != PLSVO_OK) fakecuda::error("the oracle refused the align1D batch the host code built");
    return true;
  });
}

cudaError_t match_direct_kernel_launch(const MatchArgs& a0, cudaStream_t s) {
  const OracleApi* o = oracle();
  if (!o) return cudaErrorNotSupported;
  const MatchArgs a = a0;
  return fakecuda::enqueue(s, [a, o]() {
    plsvo_match_batch b;
    memset(&b, 0, sizeof b);
    b.n_features = a.n, b.n_ref_images = 1 << 30, b.n_cur_images = 1 << 30, b.n_pyr_levels = a.n_pyr_levels, b.n_iter = a.n_iter;
    b.cam.width = a.width, b.cam.height = a.height, b.cam.fx = a.fx, b.cam.fy = a.fy, b.cam.cx = a.cx, b.cam.cy = a.cy;
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
      b.ref_img[l] = a.ref_img[l], b.ref_pitch[l] = a.ref_pitch[l], b.ref_stride[l] = a.ref_stride[l];
      b.cur_img[l] = a.cur_img[l], b.cur_pitch[l] = a.cur_pitch[l], b.cur_stride[l] = a.cur_stride[l];
    }
    b.T_ref_w = a.T_ref_w, b.T_cur_w = a.T_cur_w, b.ref_index = a.ref_index, b.cur_index = a.cur_index, b.ref_px = a.ref_px;
    b.ref_f = a.ref_f, b.ref_level = a.ref_level, b.is_edgelet = a.is_edgelet, b.ref_grad = a.ref_grad, b.pos = a.pos, b.px_cur = a.px_cur;
    memset(a.out_px, 0, (size_t)a.n * 16), memset(a.out_success, 0, (size_t)a.n), memset(a.out_level, 0, (size_t)a.n * 4);
    plsvo_match_result r{a.out_px, a.out_success, a.out_level, a.out_A};
    if (o->match(&b, &r, host_threads()) != PLSVO_OK) fakecuda::error("the oracle refused the match batch the host code built");
    return true;
  });
}

// The oracle's epipolar ZMSSD search strides the current image with its width, as the reference does with Mat::cols
// (src/matcher.cpp:380-382; "images are dense"), while the device layout pads rows to 16 bytes: levels whose pitch is not
// their width are handed over as dense copies.
static void densify_cur_levels(const SeedArgs& a, plsvo_seed_batch* b, std::vector<std::vector<uint8_t>>* keep) {
  int n_cur = 0;
  for (int i = 0; i < a.n; ++i) n_cur = std::max(n_cur, a.cur_index[i] + 1);
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
    const int cols = a.width >> l, rows = a.height >> l;
    if (!a.cur_img[l] || cols <= 0 || rows <= 0 || a.cur_pitch[l] == (uint32_t)cols) continue;
    if (!fakecuda::check(a.cur_img[l], (size_t)n_cur * a.cur_stride[l], "seed kernel: current image level")) continue;
    keep->emplace_back((size_t)n_cur * rows * cols);
    uint8_t* d = keep->back().data();
    for (int f = 0; f < n_cur; ++f)
      for (int y = 0; y < rows; ++y)
        memcpy(d + ((size_t)f * rows + y) * cols, a.cur_img[l] + (size_t)f * a.cur_stride[l] + (size_t)y * a.cur_pitch[l], (size_t)cols);
    b->cur_img[l] = d, b->cur_pitch[l] = (size_t)cols, b->cur_stride[l] = (size_t)rows * cols;
  }
}

static void fill_seed(const SeedArgs& a, plsvo_seed_batch* b, plsvo_seed_result* r) {
  memset(b, 0, sizeof *b);
  b->n_seeds = a.n, b->n_ref_images = 1 << 30, b->n_cur_images = 1 << 30, b->n_pyr_levels = a.n_pyr_levels, b->n_iter = a.n_iter;
  b->max_epi_search_steps = a.max_epi_search_steps, b->align_1d = (uint8_t)a.align_1d, b->subpix_refinement = (uint8_t)a.subpix_refinement;
  b->epi_search_edgelet_filtering = (uint8_t)a.edgelet_filtering, b->epi_search_edgelet_max_angle = a.edgelet_max_angle;
  b->seed_convergence_sigma2_thresh = a.convergence_thresh;
  b->cam.width = a.width, b->cam.height = a.height, b->cam.fx = a.fx, b->cam.fy = a.fy, b->cam.cx = a.cx, b->cam.cy = a.cy;
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
    b->ref_img[l] = a.ref_img[l], b->ref_pitch[l] = a.ref_pitch[l], b->ref_stride[l] = a.ref_stride[l];
    b->cur_img[l] = a.cur_img[l], b->cur_pitch[l] = a.cur_pitch[l], b->cur_stride[l] = a.cur_stride[l];
  }
  b->T_ref_w = a.T_ref_w, b->T_cur_w = a.T_cur_w, b->ref_index = a.ref_index, b->cur_index = a.cur_index, b->ref_px = a.ref_px;
  b->ref_f = a.ref_f, b->ref_level = a.ref_level, b->is_edgelet = a.is_edgelet, b->ref_grad = a.ref_grad;
  b->a = a.a, b->b = a.b, b->mu = a.mu, b->z_range = a.z_range, b->sigma2 = a.sigma2;
  const size_t n = (size_t)a.n;
  memset(a.out_a, 0, n * 4), memset(a.out_b, 0, n * 4), memset(a.out_mu, 0, n * 4), memset(a.out_sigma2, 0, n * 4);
  memset(a.out_status, 0, n * 4), memset(a.out_converged, 0, n), memset(a.out_depth, 0, n * 8), memset(a.out_px_cur, 0, n * 16);
  *r = plsvo_seed_result{a.out_a, a.out_b, a.out_mu, a.out_sigma2, a.out_status, a.out_converged, a.out_depth, a.out_px_cur};
}

cudaError_t seed_update_kernel_launch(const SeedArgs& a0, cudaStream_t s) {
  const OracleApi* o = oracle();
  if (!o) return cudaErrorNotSupported;
  const SeedArgs a = a0;
  return fakecuda::enqueue(s, [a, o]() {
    plsvo_seed_batch b;
    plsvo_seed_result r;
    std::vector<std::vector<uint8_t>> dense;
    fill_seed(a, &b, &r);
    densify_cur_levels(a, &b, &dense);
    if (o->seed(&b, &r, host_threads()) != PLSVO_OK) fakecuda::error("the oracle refused the seed batch the host code built");
    return true;
  });
}

cudaError_t line_seed_update_kernel_launch(const SeedArgs& a0, cudaStream_t s) {
  const OracleApi* o = oracle();
  if (!o) return cudaErrorNotSupported;
  const SeedArgs a = a0;
  return fakecuda::enqueue(s, [a, o]() {
    plsvo_line_seed_batch b;
    plsvo_line_seed_result r;
    memset(&b, 0, sizeof b), memset(&r, 0, sizeof r);
    std::vector<std::vector<uint8_t>> dense;
    fill_seed(a, &b.seeds, &r.seeds);
    densify_cur_levels(a, &b.seeds, &dense);
    b.ref_sf = a.ref_sf, b.ref_ef = a.ref_ef, b.mu_e = a.mu_e, b.z_range_e = a.z_range_e, b.sigma2_e = a.sigma2_e;
    const size_t n = (size_t)a.n;
    memset(a.out_mu_e, 0, n * 4), memset(a.out_sigma2_e, 0, n * 4), memset(a.out_depth_e, 0, n * 8), memset(a.out_px_cur_e, 0, n * 16);
    r.mu_e = a.out_mu_e, r.sigma2_e = a.out_sigma2_e, r.depth_e = a.out_depth_e, r.px_cur_e = a.out_px_cur_e;
    if (o->line_seed(&b, &r, host_threads()) != PLSVO_OK) fakecuda::error("the oracle refused the line-seed batch the host code built");
    return true;
  });
}

cudaError_t structopt_kernel_launch(const StructOptArgs& a0, cudaStream_t s) {
  const OracleApi* o = oracle();
  if (!o) return cudaErrorNotSupported;
  const StructOptArgs a = a0;
  return fakecuda::enqueue(s, [a, o]() {
    plsvo_structopt_batch b;
    memset(&b, 0, sizeof b);
    b.n_points = a.n_points, b.n_segs = a.n_segs, b.n_iter_pts = a.n_iter_pts, b.n_iter_segs = a.n_iter_segs;
    int n_frames = 0;  // not part of the kernel arguments: the highest frame any observation names
    const int npo = a.n_points ? a.pt_obs_begin[a.n_points] : 0, nso = a.n_segs ? a.seg_obs_begin[a.n_segs] : 0;
    for (int i = 0; i < npo; ++i) n_frames = std::max(n_frames, a.pt_obs_frame[i] + 1);
    for (int i = 0; i < nso; ++i) n_frames = std::max(n_frames, a.seg_obs_frame[i] + 1);
    b.n_frames = n_frames;
    b.T_f_w = a.T_f_w, b.pt_obs_begin = a.pt_obs_begin, b.pt_obs_frame = a.pt_obs_frame, b.pt_obs_f = a.pt_obs_f, b.pt_pos = a.pt_pos;
    b.seg_obs_begin = a.seg_obs_begin, b.seg_obs_frame = a.seg_obs_frame, b.seg_obs_sf = a.seg_obs_sf, b.seg_obs_ef = a.seg_obs_ef;
    b.seg_spos = a.seg_spos, b.seg_epos = a.seg_epos;
    plsvo_structopt_result r{a.out_pt_pos, a.out_seg_spos, a.out_seg_epos, a.out_pt_iters, a.out_seg_iters};
    if (o->structopt(&b, &r, host_threads()) != PLSVO_OK) fakecuda::error("the oracle refused the structure-optimisation batch the host code built");
    return true;
  });
}

}  // namespace plsvo
