// plsvo_abi.cu — the C ABI of include/plsvo_b200.h: context, host<->device staging, launches.
// Host-side only; the kernels are in align_kernel.cu and poseopt_kernel.cu.
#include <cuda_runtime.h>
#include <chrono>
#include <errno.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <string>
#include <thread>
#include <vector>

#include "internal.h"

using namespace plsvo;

namespace {

thread_local std::string g_create_error;

// A device allocation that grows on demand (ensure) and is freed with its owner.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() {
    if (p) cudaFree(p);
  }
};

struct plsvo_ctx_impl {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  cudaStream_t copy_stream = nullptr;  // copy stream of the arrival-gated host path
  cudaEvent_t start_ev = nullptr;
  cudaEvent_t k_ev[2] = {nullptr, nullptr};  // around the kernel of the last pyramid / align2D / align1D call
  unsigned int* h_flags = nullptr;  // pinned arrival values of the gated pipeline
  char* h_out = nullptr;            // pinned staging of the alignment outputs (one D2H per download)
  size_t h_out_cap = 0, out_bytes = 0;
  size_t oo_T = 0, oo_H = 0, oo_ntr = 0, oo_iters = 0, oo_status = 0, oo_pi = 0, oo_pl = 0, oo_killed = 0;
  int h_flags_cap = 0;
  int num_sms = 0;
  int smem_optin = 0;
  std::string err;
  long long launches = 0;

  // ---- alignment state ----
  bool align_ready = false;
  AlignArgs aa;
  plsvo_camera cam;
  int a_max_seg_patches_l0 = 0;  // bound at level 0 (levels >= 0 never need more)
  std::vector<int> seg_patch_bound;  // per level: max over pairs of the number of segment samples
  std::vector<int> seg_slot_bound;   // per level: max over pairs of the lane slots of the segment groups
  std::vector<int> seg_maxN;         // per level: most samples of any one segment
  DevBuf d_ref_der, d_cur_der;       // pyramid levels derived on the device (vk::halfSample) instead of uploaded
  int der_src = -1, der_top = -1;    // derived levels are (der_src, der_top], built from uploaded level der_src
  bool lvl_uploaded[PLSVO_MAX_LEVELS] = {false};
  bool chain = false;              // PLSVO_ALIGN_FRAME_CHAIN: one stack of B+1 frames, cur(b) = frame b+1 = ref(b+1)
  bool atan = false;               // the uploaded batch is seen through a vk::ATANCamera (the ATAN kernel variants)
  DevBuf d_feat;                     // every per-pair input array of the batch, at 256-byte-aligned offsets
  size_t feat_bytes = 0;
  char* h_po_out = nullptr;          // pinned staging of the pose-optimiser outputs (one D2H per download)
  size_t h_po_out_cap = 0, po_out_bytes = 0, po_zero_off = 0, po_zero_bytes = 0;
  DevBuf p_in;                       // every input array of a pose-optimiser batch, at 256-byte-aligned offsets
  char* h_in = nullptr;              // pinned staging of the small-batch upload
  size_t h_in_cap = 0, img_total = 0;
  cudaEvent_t h_in_ev = nullptr;     // the staged copies of the previous small upload
  DevBuf d_ref_img, d_cur_img;
  DevBuf d_out_T, d_counter, d_ws_cache, d_ws_segpx, d_ws_rec, d_stage;  // d_out_T: every output, one block
  size_t level_off[PLSVO_MAX_LEVELS];

  // ---- pose-opt state ----
  bool po_ready = false;
  PoseOptArgs pa;
  DevBuf y_img;  // pyramid levels
  DevBuf f_img, f_idx, f_lvl, f_border, f_ref, f_px, f_opx, f_oconv, f_dir, f_ohinv;  // align2D / align1D
  DevBuf m_ref_img, m_cur_img, m_T_ref, m_T_cur, m_ridx, m_cidx, m_px, m_f, m_lvl, m_edge, m_grad, m_pos, m_pxc, m_opx, m_osucc,
      m_olvl, m_oA;  // findMatchDirect
  DevBuf d_sa, d_sb, d_smu, d_szr, d_ssig, d_smu_e, d_szr_e, d_ssig_e, d_sout;  // depth-filter seeds
  DevBuf s_T, s_pb, s_pf, s_pof, s_pp, s_sb, s_sf, s_ssf, s_sef, s_sp, s_ep, s_out;  // structure optimisation
  // undistortion: raw frames, and the map of the camera in u_cam (valid when u_map_ok), built on the device
  DevBuf u_raw, u_map1, u_map2;
  plsvo_pinhole_camera u_cam;
  int u_map_pitch = 0;
  bool u_map_ok = false;
  bool u_map_built = false;  // the last undistort call built the map (timed by u_map_ev)
  cudaEvent_t u_map_ev[2] = {nullptr, nullptr};
  DevBuf p_out_T;  // every pose-optimiser output, one block
};

#define CTX(c) reinterpret_cast<plsvo_ctx_impl*>(c)

int fail(plsvo_ctx_impl* c, int code, const char* what, cudaError_t e = cudaSuccess) {
  char buf[512];
  if (e != cudaSuccess)
    snprintf(buf, sizeof buf, "%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
  else
    snprintf(buf, sizeof buf, "%s", what);
  if (c)
    c->err = buf;
  else
    g_create_error = buf;
  return code;
}

#define CK(call)                                                        \
  do {                                                                  \
    cudaError_t e_ = (call);                                            \
    if (e_ != cudaSuccess) return fail(c, PLSVO_ERR_CUDA, #call, e_);   \
  } while (0)

// Records a timing event, creating it on first use.
cudaError_t record_event(cudaEvent_t& ev, cudaStream_t s) {
  if (!ev) {
    cudaError_t e = cudaEventCreate(&ev);
    if (e != cudaSuccess) return e;
  }
  return cudaEventRecord(ev, s);
}

// Records one of the two timing events around the kernel of a host-in/host-out entry point.
cudaError_t kernel_timer(plsvo_ctx_impl* c, int which, cudaStream_t s) { return record_event(c->k_ev[which], s); }

cudaError_t ensure(DevBuf& b, size_t bytes) {
  if (bytes <= b.cap && b.p) return cudaSuccess;
  if (b.p) cudaFree(b.p);
  b.p = nullptr;
  b.cap = 0;
  const size_t want = std::max<size_t>(bytes, 256);
  cudaError_t e = cudaMalloc(&b.p, want);
  if (e == cudaSuccess) b.cap = want;
  return e;
}

// upload a host array (or leave the device pointer NULL when the host pointer is NULL)
template <class T>
cudaError_t up(DevBuf& b, const T* host, size_t count, cudaStream_t s, const T** dev) {
  if (!host || count == 0) {
    *dev = nullptr;
    return cudaSuccess;
  }
  cudaError_t e = ensure(b, count * sizeof(T));
  if (e != cudaSuccess) return e;
  *dev = static_cast<const T*>(b.p);
  return cudaMemcpyAsync(b.p, host, count * sizeof(T), cudaMemcpyHostToDevice, s);
}

// LineFeat::setupSampling + per-level decimation on the host, to size the segment-sample slots
// (reference: src/feature.cpp:160-173, src/sparse_img_align.cpp:318-320)
int host_seg_samples(const double* spx, const double* epx, double length, int level) {
  const double d0 = fabs(epx[0] - spx[0]), d1 = fabs(epx[1] - spx[1]);
  const double tan_dir = std::min(d0, d1) / std::max(d0, d1);
  const double sin_dir = tan_dir / sqrt(1.0 + tan_dir * tan_dir);
  const double correction = 2.0 * sqrt(1.0 + sin_dir * sin_dir);
  double nd = length / (2.0 * 4 * correction);
  if (!(nd >= 1.0)) nd = 1.0;  // also catches NaN
  if (nd > 1e6) nd = 1e6;
  const unsigned long long n0 = (unsigned long long)nd;
  return (int)(1 + (n0 - 1) / (unsigned long long)(1 << level));
}

// The host-in/host-out entry points (plsvo_*_batch_run) promise that the caller's arrays are not read once they have
// returned — also when they return an error after copies have been queued (a level that can neither be found nor derived, a
// count out of range found by the sizing pass, ...).  Every such entry point passes its result through here: a non-OK
// result first drains every stream of the context (tests/test_host_pipeline_cpu.py counts pending host reads).
int settled(plsvo_ctx_impl* c, int rc) {
  if (rc == PLSVO_OK || !c) return rc;
  if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
  cudaStreamSynchronize(c->stream);
  return rc;
}

}  // namespace

extern "C" {

const char* plsvo_version(void) { return "plsvo_b200 0.1.0 sm_90a"; }

int plsvo_ctx_create(int device, void* stream, plsvo_ctx** out) {
  if (!out) return PLSVO_ERR_INVALID;
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    return fail(nullptr, PLSVO_ERR_NO_DEVICE, "no CUDA device available (there is no CPU fallback)", e);
  if (device < 0 || device >= n) return fail(nullptr, PLSVO_ERR_INVALID, "device ordinal out of range");
  e = cudaSetDevice(device);
  if (e != cudaSuccess) return fail(nullptr, PLSVO_ERR_CUDA, "cudaSetDevice", e);
  plsvo_ctx_impl* c = new plsvo_ctx_impl();
  c->device = device;
  cudaDeviceGetAttribute(&c->num_sms, cudaDevAttrMultiProcessorCount, device);
  cudaDeviceGetAttribute(&c->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
  if (stream) {
    c->stream = static_cast<cudaStream_t>(stream);
  } else {
    e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) {
      delete c;
      return fail(nullptr, PLSVO_ERR_CUDA, "cudaStreamCreate", e);
    }
    c->own_stream = true;
  }
  memset(&c->aa, 0, sizeof c->aa);
  memset(&c->pa, 0, sizeof c->pa);
  *out = reinterpret_cast<plsvo_ctx*>(c);
  return PLSVO_OK;
}

void plsvo_ctx_destroy(plsvo_ctx* ctx) {
  if (!ctx) return;
  plsvo_ctx_impl* c = CTX(ctx);
  cudaSetDevice(c->device);
  // nothing may still be writing into the buffers freed below (the device buffers go with `delete c`): the copy stream
  // first, then the main stream
  if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
  cudaStreamSynchronize(c->stream);
  if (c->h_flags) cudaFreeHost(c->h_flags);
  if (c->h_out) cudaFreeHost(c->h_out);
  if (c->h_in) cudaFreeHost(c->h_in);
  if (c->h_po_out) cudaFreeHost(c->h_po_out);
  if (c->h_in_ev) cudaEventDestroy(c->h_in_ev);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  if (c->start_ev) cudaEventDestroy(c->start_ev);
  for (auto& e : c->k_ev)
    if (e) cudaEventDestroy(e);
  for (auto& e : c->u_map_ev)
    if (e) cudaEventDestroy(e);
  if (c->own_stream) cudaStreamDestroy(c->stream);
  delete c;
}

const char* plsvo_last_error(const plsvo_ctx* ctx) {
  if (!ctx) return g_create_error.c_str();
  return reinterpret_cast<const plsvo_ctx_impl*>(ctx)->err.c_str();
}

void* plsvo_ctx_stream(plsvo_ctx* ctx) { return ctx ? (void*)CTX(ctx)->stream : nullptr; }

int plsvo_sync(plsvo_ctx* ctx) {
  if (!ctx) return PLSVO_ERR_INVALID;
  plsvo_ctx_impl* c = CTX(ctx);
  CK(cudaStreamSynchronize(c->stream));
  return PLSVO_OK;
}

int plsvo_host_alloc(void** ptr, size_t bytes) {
  if (!ptr) return PLSVO_ERR_INVALID;
  cudaError_t e = cudaHostAlloc(ptr, bytes, cudaHostAllocDefault);
  if (e != cudaSuccess) {
    *ptr = nullptr;
    return fail(nullptr, e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver ? PLSVO_ERR_NO_DEVICE : PLSVO_ERR_CUDA,
                "cudaHostAlloc", e);
  }
  return PLSVO_OK;
}
int plsvo_host_free(void* ptr) {
  if (!ptr) return PLSVO_OK;
  return cudaFreeHost(ptr) == cudaSuccess ? PLSVO_OK : PLSVO_ERR_CUDA;
}

int plsvo_last_kernel_ms(plsvo_ctx* ctx, float* ms) {
  if (!ctx || !ms) return PLSVO_ERR_INVALID;
  plsvo_ctx_impl* c = CTX(ctx);
  if (!c->k_ev[0] || !c->k_ev[1]) return fail(c, PLSVO_ERR_STATE, "no timed kernel has run on this context");
  CK(cudaEventSynchronize(c->k_ev[1]));
  CK(cudaEventElapsedTime(ms, c->k_ev[0], c->k_ev[1]));
  return PLSVO_OK;
}

int64_t plsvo_launch_count(const plsvo_ctx* ctx) {
  return ctx ? reinterpret_cast<const plsvo_ctx_impl*>(ctx)->launches : 0;
}

int plsvo_selftest_weight(plsvo_ctx* ctx, uint32_t n, uint32_t seed, uint64_t* mismatches) {
  if (!ctx || !mismatches) return PLSVO_ERR_INVALID;
  plsvo_ctx_impl* c = CTX(ctx);
  CK(cudaSetDevice(c->device));
  CK(ensure(c->d_counter, 256));
  unsigned long long* d = reinterpret_cast<unsigned long long*>(static_cast<char*>(c->d_counter.p) + 64);
  CK(cudaMemsetAsync(d, 0, sizeof(unsigned long long), c->stream));
  CK(weight_selftest_launch(n, seed, d, c->stream));
  c->launches += 1;
  unsigned long long h = 0;
  CK(cudaMemcpyAsync(&h, d, sizeof h, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  *mismatches = h;
  return PLSVO_OK;
}

// ------------------------------------------------------------------------------------------------
// alignment
// ------------------------------------------------------------------------------------------------
}  // extern "C" (helpers below use templates)

namespace {

// The per-pair input arrays of an alignment batch, each listed once: host array, the AlignArgs field that receives its
// device address, and its bytes for the whole batch.  An array is sent when host != NULL and bytes > 0.  Depths replace
// positions: pt_pos is not sent when pt_depth is, nor seg_spos / seg_epos when the segment depths are.
struct PairArray {
  const void* host;
  const void** dev;
  size_t bytes;
  bool sent() const { return host && bytes; }
};

std::array<PairArray, 19> pair_arrays(const plsvo_align_batch* h, AlignArgs& a) {
  const size_t B = (size_t)h->batch, np = (size_t)h->n_pts, ns = (size_t)h->n_segs;
  return {{
      {h->T_ref_w, (const void**)&a.T_ref_w, B * 7 * 8},
      {h->T_cur_w, (const void**)&a.T_cur_w, B * 7 * 8},
      {h->pt_count, (const void**)&a.pt_count, B * 4},
      {h->pt_px, (const void**)&a.pt_px, B * np * 16},
      {h->pt_f, (const void**)&a.pt_f, B * np * 24},
      {h->pt_depth ? nullptr : h->pt_pos, (const void**)&a.pt_pos, B * np * 24},
      {h->pt_depth, (const void**)&a.pt_depth, B * np * 8},
      {h->pt_valid, (const void**)&a.pt_valid, B * np},
      {h->seg_count, (const void**)&a.seg_count, B * 4},
      {h->seg_spx, (const void**)&a.seg_spx, B * ns * 16},
      {h->seg_epx, (const void**)&a.seg_epx, B * ns * 16},
      {h->seg_sf, (const void**)&a.seg_sf, B * ns * 24},
      {h->seg_ef, (const void**)&a.seg_ef, B * ns * 24},
      {h->seg_sdepth ? nullptr : h->seg_spos, (const void**)&a.seg_spos, B * ns * 24},
      {h->seg_edepth ? nullptr : h->seg_epos, (const void**)&a.seg_epos, B * ns * 24},
      {h->seg_sdepth, (const void**)&a.seg_sdepth, B * ns * 8},
      {h->seg_edepth, (const void**)&a.seg_edepth, B * ns * 8},
      {h->seg_length, (const void**)&a.seg_length, B * ns * 8},
      {h->seg_valid, (const void**)&a.seg_valid, B * ns},
  }};
}

// Validates the batch and lays it out on the device, copying nothing: every provided image level packed as
// [frames][rows][pitch] at level_off[l] of d_ref_img / d_cur_img, the staging area of the repack path, and every sent
// per-pair array at a 256-byte-aligned offset of d_feat.
int align_layout(plsvo_ctx_impl* c, const plsvo_align_batch* h) {
  AlignArgs& a = c->aa;
  c->align_ready = false;
  if (h->batch <= 0 || h->n_pts < 0 || h->n_segs < 0 || h->n_segs > 32767)
    return fail(c, PLSVO_ERR_INVALID, "batch/n_pts/n_segs out of range");
  if (!h->T_ref_w || !h->T_cur_w) return fail(c, PLSVO_ERR_INVALID, "T_ref_w/T_cur_w missing");
  if (h->n_pts > 0 && (!h->pt_px || (!h->pt_pos && !h->pt_depth)))
    return fail(c, PLSVO_ERR_INVALID, "point arrays missing");
  if (h->n_segs > 0 && (!h->seg_spx || !h->seg_epx || (!h->seg_spos && !h->seg_sdepth) ||
                        (!h->seg_epos && !h->seg_edepth) || !h->seg_length))
    return fail(c, PLSVO_ERR_INVALID, "segment arrays missing");
  if (h->cam.width <= 0 || h->cam.height <= 0) return fail(c, PLSVO_ERR_INVALID, "camera size");
  if (h->flags & ~PLSVO_ALIGN_FRAME_CHAIN) return fail(c, PLSVO_ERR_INVALID, "unknown bits in plsvo_align_batch.flags");
  CK(cudaSetDevice(c->device));
  // frame chain: ref_img[l] is one stack of B+1 frames and the current image of pair b is frame b+1 — the kernel's
  // `cur_img[l] + b*stride` then simply starts one frame further into the same stack
  c->chain = (h->flags & PLSVO_ALIGN_FRAME_CHAIN) != 0;
  c->atan = false;  // the ATAN entry points set it after the upload
  a.B = h->batch, a.n_pts = h->n_pts, a.n_segs = h->n_segs;
  a.width = h->cam.width, a.height = h->cam.height;
  a.fx = h->cam.fx, a.fy = h->cam.fy, a.cx = h->cam.cx, a.cy = h->cam.cy;
  c->cam = h->cam;
  c->der_src = c->der_top = -1;
  // images: every provided level packed as [frames][rows][pitch]; a level whose host layout the device does not keep
  // passes through the staging area d_stage
  {
    const size_t B = (size_t)h->batch;
    const size_t n_frames = B + (c->chain ? 1 : 0);
    size_t total = 0;
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
      a.ref_img[l] = a.cur_img[l] = nullptr;
      a.pitch[l] = 0, a.stride[l] = 0;
      c->level_off[l] = 0;
      c->lvl_uploaded[l] = false;
      if (!h->ref_img[l] || (!c->chain && !h->cur_img[l])) continue;
      c->lvl_uploaded[l] = true;
      const int cols = h->cam.width >> l, rows = h->cam.height >> l;
      if (cols <= 0 || rows <= 0) return fail(c, PLSVO_ERR_INVALID, "pyramid level smaller than one pixel");
      if (h->img_pitch[l] < (size_t)cols) return fail(c, PLSVO_ERR_INVALID, "img_pitch smaller than the level width");
      // device pitch: the host layout is kept when rows are word aligned and images 16-byte aligned
      // (what the aligned-word loads and the bulk copy need) — then a level moves with one linear copy;
      // otherwise rows are padded to 16 bytes and repacked on the device.
      uint32_t pitch = (uint32_t)((cols + 15) / 16 * 16);
      const bool uniform = h->img_stride[l] == (size_t)rows * h->img_pitch[l];
      if (uniform && h->img_pitch[l] % 4 == 0 && h->img_stride[l] % 16 == 0 && h->img_pitch[l] < (1u << 20))
        pitch = (uint32_t)h->img_pitch[l];
      a.pitch[l] = pitch;
      a.stride[l] = (size_t)rows * pitch;
      total = (total + 255) / 256 * 256;
      c->level_off[l] = total;
      total += a.stride[l] * n_frames;
    }
    CK(ensure(c->d_ref_img, total + 256));
    if (!c->chain) CK(ensure(c->d_cur_img, total + 256));
    c->img_total = total;
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
      if (!c->lvl_uploaded[l]) continue;
      a.ref_img[l] = static_cast<uint8_t*>(c->d_ref_img.p) + c->level_off[l];
      a.cur_img[l] = c->chain ? a.ref_img[l] + a.stride[l] : static_cast<uint8_t*>(c->d_cur_img.p) + c->level_off[l];
    }
    size_t stage = 0;
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l)
      if (a.pitch[l] && h->img_pitch[l] != a.pitch[l]) stage = std::max(stage, 2 * h->img_stride[l] * n_frames);
    if (stage) CK(ensure(c->d_stage, stage));
  }
  const auto arrays = pair_arrays(h, a);
  size_t off = 0;
  for (const PairArray& p : arrays)
    if (p.sent()) off += (p.bytes + 255) / 256 * 256;
  CK(ensure(c->d_feat, off + 256));
  c->feat_bytes = off;
  off = 0;
  for (const PairArray& p : arrays) {
    *p.dev = p.sent() ? static_cast<char*>(c->d_feat.p) + off : nullptr;
    if (p.sent()) off += (p.bytes + 255) / 256 * 256;
  }
  return PLSVO_OK;
}

// One host->device copy per sent per-pair array, into its place in d_feat.
int align_copy_features(plsvo_ctx_impl* c, const plsvo_align_batch* h, cudaStream_t s) {
  for (const PairArray& p : pair_arrays(h, c->aa))
    if (p.sent()) CK(cudaMemcpyAsync(const_cast<void*>(*p.dev), p.host, p.bytes, cudaMemcpyHostToDevice, s));
  return PLSVO_OK;
}

// The image levels of pairs [b0,b1): one linear copy per stack where the device keeps the host layout; a uniformly pitched
// stack with another pitch goes linearly into staging and is repacked on the device; any other stack moves frame by frame.
int align_copy_images(plsvo_ctx_impl* c, const plsvo_align_batch* h, size_t b0, size_t b1, cudaStream_t s) {
  const AlignArgs& a = c->aa;
  const size_t nb = b1 - b0;
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
    if (!c->lvl_uploaded[l]) continue;
    const int cols = h->cam.width >> l, rows = h->cam.height >> l;
    uint8_t* dr = static_cast<uint8_t*>(c->d_ref_img.p) + c->level_off[l];
    const bool uniform = h->img_stride[l] == (size_t)rows * h->img_pitch[l];
    if (c->chain) {
      // pairs [b0,b1) read frames [b0, b1]: frame b0 came with the previous range (or is frame 0 of the first one)
      const size_t f0 = b0 ? b0 + 1 : 0, nf = b1 + 1 - f0;
      const uint8_t* hf = h->ref_img[l] + f0 * h->img_stride[l];
      uint8_t* df = dr + f0 * a.stride[l];
      if (uniform && h->img_pitch[l] == a.pitch[l]) {
        CK(cudaMemcpyAsync(df, hf, a.stride[l] * nf, cudaMemcpyHostToDevice, s));
      } else if (uniform) {
        uint8_t* st = static_cast<uint8_t*>(c->d_stage.p) + h->img_stride[l] * f0;
        CK(cudaMemcpyAsync(st, hf, h->img_stride[l] * nf, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpy2DAsync(df, a.pitch[l], st, h->img_pitch[l], cols, (size_t)rows * nf, cudaMemcpyDeviceToDevice, s));
      } else {
        for (size_t k = 0; k < nf; ++k)
          CK(cudaMemcpy2DAsync(df + k * a.stride[l], a.pitch[l], hf + k * h->img_stride[l], h->img_pitch[l], cols, rows,
                               cudaMemcpyHostToDevice, s));
      }
      continue;
    }
    uint8_t* dc = static_cast<uint8_t*>(c->d_cur_img.p) + c->level_off[l] + b0 * a.stride[l];
    dr += b0 * a.stride[l];
    const uint8_t* hr = h->ref_img[l] + b0 * h->img_stride[l];
    const uint8_t* hc = h->cur_img[l] + b0 * h->img_stride[l];
    if (uniform && h->img_pitch[l] == a.pitch[l]) {
      // host stack already has the device layout: one linear copy per frame set
      CK(cudaMemcpyAsync(dr, hr, a.stride[l] * nb, cudaMemcpyHostToDevice, s));
      CK(cudaMemcpyAsync(dc, hc, a.stride[l] * nb, cudaMemcpyHostToDevice, s));
    } else if (uniform) {
      // uniformly pitched stack with a different pitch: linear H2D into staging (PCIe-friendly), then a
      // device-side 2D repack into the 16-byte-pitched layout (row-granular DMA over PCIe is slow)
      const size_t off = 2 * h->img_stride[l] * b0, bytes = h->img_stride[l] * nb;
      uint8_t* st = static_cast<uint8_t*>(c->d_stage.p) + off;
      CK(cudaMemcpyAsync(st, hr, bytes, cudaMemcpyHostToDevice, s));
      CK(cudaMemcpyAsync(st + bytes, hc, bytes, cudaMemcpyHostToDevice, s));
      CK(cudaMemcpy2DAsync(dr, a.pitch[l], st, h->img_pitch[l], cols, (size_t)rows * nb, cudaMemcpyDeviceToDevice, s));
      CK(cudaMemcpy2DAsync(dc, a.pitch[l], st + bytes, h->img_pitch[l], cols, (size_t)rows * nb, cudaMemcpyDeviceToDevice, s));
    } else {
      for (size_t b = 0; b < nb; ++b) {
        CK(cudaMemcpy2DAsync(dr + b * a.stride[l], a.pitch[l], hr + b * h->img_stride[l], h->img_pitch[l], cols, rows,
                             cudaMemcpyHostToDevice, s));
        CK(cudaMemcpy2DAsync(dc + b * a.stride[l], a.pitch[l], hc + b * h->img_stride[l], h->img_pitch[l], cols, rows,
                             cudaMemcpyHostToDevice, s));
      }
    }
  }
  return PLSVO_OK;
}

// Small batches (the reference's own call is B = 1, frame_handler_mono.cpp:272): every input is packed into one pinned
// staging block and moves with three copies (reference images, current images, all per-pair arrays) instead of ~20
// separate copies from pageable memory, each of which costs more than the kernel of a single pair.  The block holds the
// images in their device layout, so every level must come in the layout the device keeps.
bool align_small_block_fits(const plsvo_ctx_impl* c, const plsvo_align_batch* h) {
  if (getenv("PLSVO_NO_SMALL_UPLOAD") || 2 * c->img_total + c->feat_bytes > (size_t)4 << 20) return false;
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
    const int rows = h->cam.height >> l;
    if (c->lvl_uploaded[l] && !(h->img_stride[l] == (size_t)rows * h->img_pitch[l] && h->img_pitch[l] == c->aa.pitch[l]))
      return false;  // needs the repack path
  }
  return true;
}

int align_copy_small_block(plsvo_ctx_impl* c, const plsvo_align_batch* h) {
  const AlignArgs& a = c->aa;
  const size_t B = (size_t)h->batch;
  const size_t need = 2 * c->img_total + c->feat_bytes + 256;
  if (c->h_in_cap < need) {
    if (c->h_in_ev) CK(cudaEventSynchronize(c->h_in_ev));  // a copy out of the old block may still be queued
    if (c->h_in) cudaFreeHost(c->h_in);
    c->h_in = nullptr, c->h_in_cap = 0;
    CK(cudaHostAlloc((void**)&c->h_in, need, cudaHostAllocDefault));
    c->h_in_cap = need;
  }
  if (!c->h_in_ev) CK(cudaEventCreateWithFlags(&c->h_in_ev, cudaEventDisableTiming));
  else CK(cudaEventSynchronize(c->h_in_ev));  // the previous upload's copies have left the staging block
  char* hr = c->h_in;
  char* hc = c->h_in + c->img_total;
  char* hf = c->h_in + 2 * c->img_total;
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
    if (!c->lvl_uploaded[l]) continue;
    memcpy(hr + c->level_off[l], h->ref_img[l], a.stride[l] * (B + (c->chain ? 1 : 0)));
    if (!c->chain) memcpy(hc + c->level_off[l], h->cur_img[l], a.stride[l] * B);
  }
  const char* feat = static_cast<const char*>(c->d_feat.p);
  for (const PairArray& p : pair_arrays(h, c->aa))
    if (p.sent()) memcpy(hf + (static_cast<const char*>(*p.dev) - feat), p.host, p.bytes);
  if (c->img_total) {
    CK(cudaMemcpyAsync(c->d_ref_img.p, hr, c->img_total, cudaMemcpyHostToDevice, c->stream));
    if (!c->chain) CK(cudaMemcpyAsync(c->d_cur_img.p, hc, c->img_total, cudaMemcpyHostToDevice, c->stream));
  }
  if (c->feat_bytes) CK(cudaMemcpyAsync(c->d_feat.p, hf, c->feat_bytes, cudaMemcpyHostToDevice, c->stream));
  CK(cudaEventRecord(c->h_in_ev, c->stream));
  return PLSVO_OK;
}

// Host-side sizing of the laid-out batch (the host arrays are still valid here) and its output block.  size_level >= 0:
// the sizing is wanted for that pyramid level only and may be a cheap upper bound (it sits on the launch path of the
// streamed host call).
int align_size(plsvo_ctx_impl* c, const plsvo_align_batch* h, int size_level) {
  AlignArgs& a = c->aa;
  const size_t B = (size_t)h->batch;
  // per-pair feature counts index shared memory and the feature arrays in the kernels: reject anything outside
  // [0, n_pts] / [0, n_segs] here (every other index array of the ABI is range-checked on the host as well)
  for (size_t b = 0; b < B; ++b) {
    if (h->pt_count && (h->pt_count[b] < 0 || h->pt_count[b] > h->n_pts))
      return fail(c, PLSVO_ERR_INVALID, "pt_count[b] outside [0, n_pts]");
    if (h->seg_count && (h->seg_count[b] < 0 || h->seg_count[b] > h->n_segs))
      return fail(c, PLSVO_ERR_INVALID, "seg_count[b] outside [0, n_segs]");
  }
  // per-level bounds on the segment samples of a pair: sample slots, lane slots of the segment groups (a segment
  // with N samples owns 2^k >= min(N,32) lanes) and the longest segment
  c->seg_patch_bound.assign(PLSVO_MAX_LEVELS, 0);
  c->seg_slot_bound.assign(PLSVO_MAX_LEVELS, 0);
  c->seg_maxN.assign(PLSVO_MAX_LEVELS, 0);
  if (h->n_segs > 0) {
    // a few host threads: the sizing sits between the enqueued copies and the kernel launch of the host-buffer path
    struct Bounds {
      int patches[PLSVO_MAX_LEVELS], slots[PLSVO_MAX_LEVELS], maxN[PLSVO_MAX_LEVELS];
    };
    const bool fast = size_level >= 0 && size_level < PLSVO_MAX_LEVELS;
    const int nt = fast ? (int)std::max<size_t>(1, std::min<size_t>(4, B * (size_t)h->n_segs / 262144))
                        : (int)std::max<size_t>(1, std::min<size_t>(8, B * (size_t)h->n_segs / 8192));
    std::vector<Bounds> part(nt);
    auto work = [&](int t) {
      Bounds bd;
      memset(&bd, 0, sizeof bd);
      if (fast) {
        // Upper bound without the square roots and divisions of setupSampling: correction = 2 sqrt(1 + sin^2) >= 2, so the
        // sample count length / (2 * 4 * correction) is at most length / 16 (NaN or tiny lengths give 1, as on the device).
        const int l = size_level;
        int best_sum = 0, best_slots = 0, best_N = 0;
        for (size_t b = B * t / nt; b < B * (t + 1) / nt; ++b) {
          const int nsb = h->seg_count ? h->seg_count[b] : h->n_segs;
          const double* len = h->seg_length + b * (size_t)h->n_segs;
          int sum = 0, slots = 0;
          for (int j = 0; j < nsb; ++j) {
            double nd = len[j] * 0.0625;
            nd = nd >= 1.0 ? nd : 1.0;  // also catches NaN
            nd = nd > 1e6 ? 1e6 : nd;
            const int N = 1 + (((int)nd - 1) >> l);
            const int g = 2 * N - 1;  // the group of a segment has 2^k >= min(N, 32) lanes: at most min(2N - 1, 32)
            sum += N, slots += g < 32 ? g : 32;
            best_N = N > best_N ? N : best_N;
          }
          best_sum = std::max(best_sum, sum), best_slots = std::max(best_slots, slots);
        }
        bd.patches[l] = best_sum, bd.slots[l] = best_slots, bd.maxN[l] = best_N;
        part[t] = bd;
        return;
      }
      for (size_t b = B * t / nt; b < B * (t + 1) / nt; ++b) {
        const int nsb = h->seg_count ? h->seg_count[b] : h->n_segs;
        int sum[PLSVO_MAX_LEVELS] = {0}, slots[PLSVO_MAX_LEVELS] = {0};
        for (int j = 0; j < nsb; ++j) {
          const size_t k = b * h->n_segs + j;
          const int n0 = host_seg_samples(h->seg_spx + 2 * k, h->seg_epx + 2 * k, h->seg_length[k], 0);
          for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
            const int N = 1 + ((n0 - 1) >> l);
            int g = 1;
            while (g < N && g < 32) g <<= 1;
            sum[l] += N;
            slots[l] += g;
            bd.maxN[l] = std::max(bd.maxN[l], N);
          }
        }
        for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
          bd.patches[l] = std::max(bd.patches[l], sum[l]);
          bd.slots[l] = std::max(bd.slots[l], slots[l]);
        }
      }
      part[t] = bd;
    };
    if (nt == 1) {
      work(0);
    } else {
      std::vector<std::thread> pool;
      for (int t = 1; t < nt; ++t) pool.emplace_back(work, t);
      work(0);
      for (auto& th : pool) th.join();
    }
    for (const Bounds& bd : part)
      for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
        c->seg_patch_bound[l] = std::max(c->seg_patch_bound[l], bd.patches[l]);
        c->seg_slot_bound[l] = std::max(c->seg_slot_bound[l], bd.slots[l]);
        c->seg_maxN[l] = std::max(c->seg_maxN[l], bd.maxN[l]);
      }
  }
  // all outputs live in one device block so that the download is a single D2H into pinned staging
  {
    const size_t nsg = (size_t)std::max(1, h->n_segs);
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o = (o + bytes + 255) / 256 * 256; return at; };
    c->oo_T = take(B * 7 * sizeof(double));
    c->oo_H = take(B * 36 * sizeof(double));
    c->oo_ntr = take(B * sizeof(long long));
    c->oo_iters = take(B * PLSVO_MAX_LEVELS * sizeof(int32_t));
    c->oo_status = take(B * sizeof(int32_t));
    c->oo_pi = take(B * sizeof(uint32_t));
    c->oo_pl = take(B * sizeof(uint32_t));
    c->oo_killed = take(B * nsg);
    c->out_bytes = o;
    CK(ensure(c->d_out_T, o));
    if (c->h_out_cap < o) {
      if (c->h_out) cudaFreeHost(c->h_out);
      c->h_out = nullptr, c->h_out_cap = 0;
      CK(cudaHostAlloc((void**)&c->h_out, o, cudaHostAllocDefault));
      c->h_out_cap = o;
    }
    char* base = static_cast<char*>(c->d_out_T.p);
    a.out_T = reinterpret_cast<double*>(base + c->oo_T);
    a.out_H = reinterpret_cast<double*>(base + c->oo_H);
    a.out_n_tracked = reinterpret_cast<long long*>(base + c->oo_ntr);
    a.out_iters = reinterpret_cast<int32_t*>(base + c->oo_iters);
    a.out_status = reinterpret_cast<int32_t*>(base + c->oo_status);
    a.out_patch_iters = reinterpret_cast<uint32_t*>(base + c->oo_pi);
    a.out_patch_levels = reinterpret_cast<uint32_t*>(base + c->oo_pl);
    a.out_seg_killed = reinterpret_cast<uint8_t*>(base + c->oo_killed);
  }
  CK(ensure(c->d_counter, 256));
  a.work_counter = static_cast<unsigned int*>(c->d_counter.p);
  c->align_ready = true;
  return PLSVO_OK;
}

// The launch limits of pyramid_kernel, for every caller.  One CTA forms levels 1..6 of a 64x64 level-0 tile, so a launch
// makes at most 7 levels; a deeper pyramid continues with a second launch whose level 0 is the last level of the first.
// That level was written by the kernel, so its pitch, stride and base are 16-byte multiples, as the kernel's row loads
// need.  The frames sit on gridDim.z (at most 65535), so a launch takes at most kPyramidFramesPerLaunch of them.
constexpr int kPyramidLevelsPerLaunch = 7;
constexpr int kPyramidFramesPerLaunch = 32768;

int pyramid_launch(plsvo_ctx_impl* c, const PyramidArgs& a, cudaStream_t s) {
  for (int l0 = 0; l0 + 1 < a.n_levels; l0 += kPyramidLevelsPerLaunch - 1) {
    PyramidArgs p;
    memset(&p, 0, sizeof p);
    p.n_levels = std::min(kPyramidLevelsPerLaunch, a.n_levels - l0);
    p.width = a.width >> l0, p.height = a.height >> l0;
    for (int k = 0; k < p.n_levels; ++k) p.pitch[k] = a.pitch[l0 + k], p.stride[k] = a.stride[l0 + k];
    for (int z0 = 0; z0 < a.B; z0 += kPyramidFramesPerLaunch) {
      p.B = std::min(kPyramidFramesPerLaunch, a.B - z0);
      for (int k = 0; k < p.n_levels; ++k) p.level[k] = a.level[l0 + k] + (size_t)z0 * a.stride[l0 + k];
      CK(pyramid_kernel_launch(p, s));
      c->launches += 1;
    }
  }
  return PLSVO_OK;
}

// Pyramid levels that were not uploaded are derived on the device from the highest uploaded level below them by
// repeated vk::halfSample (pyramid_kernel.cu; bit-identical to frame_utils::createImgPyramid).  The device layout of the
// derived levels is made once per upload and kept while later launches need no other levels.
int align_derive_levels(plsvo_ctx_impl* c, int min_level, int max_level, cudaStream_t s, bool in_kernel = false) {
  AlignArgs& a = c->aa;
  a.derive_from = -1;
  int first_missing = -1;
  for (int l = min_level; l <= max_level; ++l)
    if (!c->lvl_uploaded[l]) {
      first_missing = l;
      break;
    }
  if (first_missing < 0) return PLSVO_OK;
  int src = -1;
  for (int l = first_missing - 1; l >= 0; --l)
    if (c->lvl_uploaded[l]) {
      src = l;
      break;
    }
  if (src < 0) return fail(c, PLSVO_ERR_INVALID, "a pyramid level in [min_level,max_level] was not uploaded and no lower level is there to derive it from");
  for (int l = first_missing; l <= max_level; ++l)
    if (c->lvl_uploaded[l]) return fail(c, PLSVO_ERR_INVALID, "derived pyramid levels must be contiguous above the uploaded ones");
  // the pyramid kernel reads 16-byte rows; a source level whose host layout was kept with a pitch that is only word aligned
  // (e.g. 188-byte rows: level 2 of a 752-pixel-wide camera) is halfSampled by the alignment kernel itself, pair by pair,
  // byte by byte — the same code the arrival-gated stream uses
  if (a.pitch[src] % 16 != 0 || a.stride[src] % 16 != 0) in_kernel = true;
  const size_t B = (size_t)a.B, n_frames = B + (c->chain ? 1 : 0);
  if (c->der_src != src || c->der_top < max_level) {
    size_t total = 0, off[PLSVO_MAX_LEVELS] = {0};
    for (int l = src + 1; l <= max_level; ++l) {
      const int cols = a.width >> l, rows = a.height >> l;
      if (cols <= 0 || rows <= 0) return fail(c, PLSVO_ERR_INVALID, "pyramid level smaller than one pixel");
      a.pitch[l] = (uint32_t)((cols + 15) / 16 * 16);
      a.stride[l] = (size_t)rows * a.pitch[l];
      off[l] = total;
      total += (a.stride[l] * n_frames + 255) / 256 * 256;
    }
    CK(ensure(c->d_ref_der, total + 256));
    if (!c->chain) CK(ensure(c->d_cur_der, total + 256));
    for (int l = src + 1; l <= max_level; ++l) {
      a.ref_img[l] = static_cast<uint8_t*>(c->d_ref_der.p) + off[l];
      a.cur_img[l] = c->chain ? a.ref_img[l] + a.stride[l] : static_cast<uint8_t*>(c->d_cur_der.p) + off[l];
    }
    c->der_src = src, c->der_top = max_level;
  }
  if (in_kernel) {  // the persistent alignment kernel derives the levels pair by pair
    a.derive_from = src;
    return PLSVO_OK;
  }
  // frame chain: the one stack of B+1 frames
  for (int which = 0; which < (c->chain ? 1 : 2); ++which) {
    PyramidArgs pa;
    memset(&pa, 0, sizeof pa);
    pa.B = (int)n_frames, pa.width = a.width >> src, pa.height = a.height >> src, pa.n_levels = max_level - src + 1;
    for (int l = src; l <= max_level; ++l) {
      pa.level[l - src] = const_cast<uint8_t*>(which ? a.cur_img[l] : a.ref_img[l]);
      pa.pitch[l - src] = a.pitch[l];
      pa.stride[l - src] = a.stride[l];
    }
    const int rc = pyramid_launch(c, pa, s);
    if (rc != PLSVO_OK) return rc;
  }
  return PLSVO_OK;
}

// launch plan of the alignment kernel for the uploaded batch (shared memory, CTA size, grid)
struct AlignPlan {
  int threads, min_blocks, ctas_per_sm;
  size_t smem;
};

// kernel variants (threads per CTA, resident CTAs per SM the register budget is compiled for), see align_kernel.cu
static const int kAlignVariants[][2] = {{128, 4}, {128, 5}, {96, 5}, {96, 7}, {64, 8}, {160, 3}, {192, 2}, {256, 2}};

int align_plan(plsvo_ctx_impl* c, const plsvo_align_params* p, AlignPlan* plan, bool streamed = false) {
  if (!c->align_ready) return fail(c, PLSVO_ERR_STATE, "plsvo_align_launch before plsvo_align_upload");
  if (p->min_level < 0 || p->max_level < p->min_level || p->max_level >= PLSVO_MAX_LEVELS || p->n_iter < 1)
    return fail(c, PLSVO_ERR_INVALID, "level range / n_iter");
  AlignArgs& a = c->aa;
  for (int l = p->min_level; l <= p->max_level; ++l)
    if (!a.pitch[l] || !a.ref_img[l])
      return fail(c, PLSVO_ERR_INVALID, "a pyramid level in [min_level,max_level] was neither uploaded nor derived");
  CK(cudaSetDevice(c->device));
  a.max_level = p->max_level, a.min_level = p->min_level, a.n_iter = p->n_iter, a.eps = p->eps;
  a.max_seg_patches = std::max(c->seg_patch_bound[p->min_level], 1);
  a.max_seg_slots = (c->seg_slot_bound[p->min_level] + 31) / 32 * 32 + 32;
  if (a.max_seg_slots > 65504) return fail(c, PLSVO_ERR_INVALID, "segment samples exceed the lane-slot plan");
  a.max_patches = (a.n_pts + a.max_seg_patches + 3) / 4 * 4;
  if (a.max_patches == 0) a.max_patches = 4;
  const int maxN = std::max(c->seg_maxN[p->min_level], 1);

  // Kernel variant.  Default: 128-thread CTAs with the register budget of four resident pairs per SM; small
  // batches (at most one pair per SM) take 256-thread CTAs to cut the latency of a pair.
  // PLSVO_VARIANT="threads,ctas" selects another compiled variant (tuning, A/B runs, tests).  A selected variant is the
  // only one tried: a batch it cannot run is an error, so whoever selected it knows which kernel ran.
  int want_t = 128, want_b = 4;
  if (a.B <= c->num_sms) want_t = 256, want_b = 2;
  // streamed host path: pairs trickle in at the rate of the host link, so fewer are in flight than the grid has room for
  // and the call ends one pair-latency after the last chunk lands — bigger CTAs shorten that tail (tools/e2e_trace.py)
  else if (streamed) want_t = 192, want_b = 2;
  const char* forced = getenv("PLSVO_VARIANT");
  if (forced && !*forced) forced = nullptr;
  if (forced) {
    int t = 0, mb = 0;
    if (sscanf(forced, "%d,%d", &t, &mb) != 2) return fail(c, PLSVO_ERR_INVALID, "PLSVO_VARIANT is not of the form \"threads,ctas\"");
    bool known = false;
    for (auto& kv : kAlignVariants) known |= (kv[0] == t && kv[1] == mb);
    if (!known) return fail(c, PLSVO_ERR_INVALID, "PLSVO_VARIANT names a variant that is not compiled");
    want_t = t, want_b = mb;
  }
  const int limit = c->smem_optin;  // 227 KB on sm_90a
  // try the wanted variant first, then bigger CTAs (more patches per round, fewer records per thread)
  const int order[][2] = {{want_t, want_b}, {128, 4}, {256, 2}};
  int rc_last = PLSVO_ERR_INVALID;
  for (int i = 0; i < (forced ? 1 : 3); ++i) {
    const int threads = order[i][0], min_blocks = order[i][1];
    // parked in-patch sums of a segment longer than a warp (one record per thread and 32-sample trip)
    const int rec_cap = std::max(1, (maxN + 31) / 32);
    if (rec_cap > 32) {
      rc_last = fail(c, PLSVO_ERR_INVALID, "a segment has more than 1024 samples");
      continue;
    }
    // shared-memory plan: stage the current image level when the CTA still fits min_blocks times per SM next to
    // the per-pair state; bigger levels are read through L2 with the same aligned-word loads.
    const int other = (int)align_smem_bytes(a.n_pts, a.n_segs, a.max_patches, a.max_seg_slots, 0, threads);
    int img_budget = (limit + 1024) / min_blocks - 1024 - other;
    if (img_budget < 0) img_budget = 0;
    img_budget = std::min(img_budget, 96 * 1024);
    if (const char* e = getenv("PLSVO_IMG_SMEM")) img_budget = atoi(e) ? 96 * 1024 : 0;
    int img_bytes = 0;
    for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) a.img_in_smem[l] = 0;
    for (int l = p->min_level; l <= p->max_level; ++l) {
      const size_t bytes = a.stride[l];
      a.img_in_smem[l] = (bytes <= (size_t)img_budget && bytes < (1u << 20) && bytes % 16 == 0) ? 1 : 0;
      if (a.img_in_smem[l]) img_bytes = std::max(img_bytes, (int)bytes);
    }
    size_t smem = align_smem_bytes(a.n_pts, a.n_segs, a.max_patches, a.max_seg_slots, img_bytes, threads);
    if (smem > (size_t)limit) {  // drop image staging as a last resort
      for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) a.img_in_smem[l] = 0;
      img_bytes = 0;
      smem = align_smem_bytes(a.n_pts, a.n_segs, a.max_patches, a.max_seg_slots, 0, threads);
      if (smem > (size_t)limit) {
        rc_last = fail(c, PLSVO_ERR_INVALID, "feature counts exceed the shared-memory plan");
        continue;
      }
    }
    a.smem_img_bytes = img_bytes;
    a.rec_cap = rec_cap;
    int ctas_per_sm = 0;
    CK(c->atan ? align_atan_kernel_prepare(threads, min_blocks, smem, &ctas_per_sm)
               : align_kernel_prepare(threads, min_blocks, smem, &ctas_per_sm));
    if (ctas_per_sm < 1) {
      rc_last = fail(c, PLSVO_ERR_INVALID, "kernel does not fit on an SM");
      continue;
    }
    const char* cap = getenv("PLSVO_CTAS_PER_SM");
    if (cap && atoi(cap) > 0) ctas_per_sm = std::min(ctas_per_sm, atoi(cap));
    // per-CTA workspaces: reference-patch cache, patch geometry, segment sample centres, pass records
    const size_t grid_max = (size_t)std::min(a.B, c->num_sms * ctas_per_sm);
    CK(ensure(c->d_ws_cache, grid_max * kCacheRows * a.max_patches * sizeof(float4)));
    CK(ensure(c->d_ws_segpx, grid_max * 2 * a.max_seg_patches * sizeof(double)));
    CK(ensure(c->d_ws_rec, grid_max * 5 * (size_t)rec_cap * threads * sizeof(double)));
    a.ws_cache = static_cast<float4*>(c->d_ws_cache.p);
    a.ws_segpx = static_cast<double*>(c->d_ws_segpx.p);
    a.ws_rec = static_cast<double*>(c->d_ws_rec.p);
    plan->threads = threads, plan->min_blocks = min_blocks, plan->ctas_per_sm = ctas_per_sm, plan->smem = smem;
    return PLSVO_OK;
  }
  if (forced) {
    const std::string why = c->err;
    char msg[128];
    snprintf(msg, sizeof msg, "PLSVO_VARIANT=%d,%d cannot run this batch: ", want_t, want_b);
    return fail(c, rc_last, (msg + why).c_str());
  }
  return rc_last;
}

// one kernel over the uploaded batch; gate_chunk > 0: a pair is handed out only once its chunk of gate_chunk pairs has
// arrived (the arrival counter sits 32 words behind the work counter)
int align_launch_kernel(plsvo_ctx_impl* c, const AlignPlan& plan, cudaStream_t s, int gate_chunk = 0) {
  AlignArgs a = c->aa;
  a.arrived = gate_chunk > 0 ? a.work_counter + 32 : nullptr;
  a.gate_chunk = gate_chunk;
  const int grid = std::min(a.B, c->num_sms * plan.ctas_per_sm);
  CK(cudaMemsetAsync(a.work_counter, 0, sizeof(unsigned int), s));
  CK(c->atan ? align_atan_kernel_launch(a, grid, plan.threads, plan.min_blocks, plan.smem, s)
             : align_kernel_launch(a, grid, plan.threads, plan.min_blocks, plan.smem, s));
  c->launches += 1;
  return PLSVO_OK;
}

}  // namespace

extern "C" {

int plsvo_align_upload(plsvo_ctx* ctx, const plsvo_align_batch* h) {
  if (!ctx || !h) return PLSVO_ERR_INVALID;
  plsvo_ctx_impl* c = CTX(ctx);
  int rc = align_layout(c, h);
  if (rc != PLSVO_OK) return rc;
  if (align_small_block_fits(c, h)) {
    rc = align_copy_small_block(c, h);
  } else {
    rc = align_copy_images(c, h, 0, (size_t)h->batch, c->stream);
    if (rc == PLSVO_OK) rc = align_copy_features(c, h, c->stream);
  }
  if (rc != PLSVO_OK) return rc;
  return align_size(c, h, -1);
}

int plsvo_align_launch(plsvo_ctx* ctx, const plsvo_align_params* p) {
  if (!ctx || !p) return PLSVO_ERR_INVALID;
  plsvo_ctx_impl* c = CTX(ctx);
  if (!c->align_ready) return fail(c, PLSVO_ERR_STATE, "plsvo_align_launch before plsvo_align_upload");
  if (p->min_level < 0 || p->max_level < p->min_level || p->max_level >= PLSVO_MAX_LEVELS)
    return fail(c, PLSVO_ERR_INVALID, "level range / n_iter");
  AlignPlan plan;
  int rc = align_derive_levels(c, p->min_level, p->max_level, c->stream);
  if (rc != PLSVO_OK) return rc;
  rc = align_plan(c, p, &plan);
  if (rc != PLSVO_OK) return rc;
  return align_launch_kernel(c, plan, c->stream);
}

int plsvo_align_download(plsvo_ctx* ctx, const plsvo_align_result* o) {
  if (!ctx || !o) return PLSVO_ERR_INVALID;
  plsvo_ctx_impl* c = CTX(ctx);
  if (!c->align_ready) return fail(c, PLSVO_ERR_STATE, "plsvo_align_download before plsvo_align_upload");
  CK(cudaSetDevice(c->device));
  const AlignArgs& a = c->aa;
  const size_t B = (size_t)a.B;
  cudaStream_t s = c->stream;
  // one D2H of the whole output block into pinned staging, then plain copies into the caller's arrays
  // (which are usually pageable: eight separate device->pageable copies cost several times more)
  CK(cudaMemcpyAsync(c->h_out, c->d_out_T.p, c->out_bytes, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  const char* hb = c->h_out;
  if (o->T_cur_w) memcpy(o->T_cur_w, hb + c->oo_T, B * 7 * sizeof(double));
  if (o->n_tracked) memcpy(o->n_tracked, hb + c->oo_ntr, B * sizeof(int64_t));
  if (o->H) memcpy(o->H, hb + c->oo_H, B * 36 * sizeof(double));
  if (o->seg_killed && a.n_segs > 0) memcpy(o->seg_killed, hb + c->oo_killed, B * a.n_segs);
  if (o->iters) memcpy(o->iters, hb + c->oo_iters, B * PLSVO_MAX_LEVELS * sizeof(int32_t));
  if (o->status) memcpy(o->status, hb + c->oo_status, B * sizeof(int32_t));
  if (o->patch_iters) memcpy(o->patch_iters, hb + c->oo_pi, B * sizeof(uint32_t));
  if (o->patch_levels) memcpy(o->patch_levels, hb + c->oo_pl, B * sizeof(uint32_t));
  return PLSVO_OK;
}

static int align_batch_run_body(plsvo_ctx* ctx, const plsvo_align_batch* b, const plsvo_align_params* p,
                                const plsvo_align_result* o) {
  plsvo_ctx_impl* c = CTX(ctx);
  // Host-buffer pipeline.  Default for large batches: ONE persistent kernel over the whole batch is
  // launched immediately while a second stream copies the batch to the device in chunks of 256 pairs
  // and bumps an arrival counter after each chunk; the kernel's work queue hands a pair out only once
  // its chunk has landed (arrival gate), so the PCIe leg and the compute leg overlap without cutting
  // the batch into under-filled kernels.  Chunks of 128 pairs keep every array's chunk boundary
  // 128-byte aligned (no cache line shared between an arrived and an in-flight chunk).
  // Smaller batches and layouts the gate cannot take run the plain upload -> launch -> download sequence.
  bool gated = b->batch >= 256;
  if (gated) {
    for (int l = p->min_level; l <= p->max_level && l < PLSVO_MAX_LEVELS && l >= 0; ++l) {
      const int rows = b->cam.height >> l;
      if (!b->ref_img[l] && l > p->min_level) continue;  // derived on the device after each chunk has landed
      const bool direct = b->ref_img[l] && b->img_stride[l] == (size_t)rows * b->img_pitch[l] && b->img_pitch[l] % 4 == 0 &&
                          b->img_stride[l] % 16 == 0;
      if (!direct) gated = false;  // padded layouts need a device-side repack kernel: not under the gate
      // frame chain: the last frame of an arrived chunk and the first frame of the chunk in flight are neighbours in one
      // stack — they must not share a 128-byte line
      if ((b->flags & PLSVO_ALIGN_FRAME_CHAIN) && b->img_stride[l] % 128 != 0) gated = false;
    }
  }
  if (!gated) {
    int rc = plsvo_align_upload(ctx, b);
    if (rc != PLSVO_OK) return rc;
    rc = plsvo_align_launch(ctx, p);
    if (rc != PLSVO_OK) return rc;
    return plsvo_align_download(ctx, o);
  }
  CK(cudaSetDevice(c->device));
  if (!c->copy_stream) {
    CK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&c->start_ev, cudaEventDisableTiming));
  }
  const size_t B = (size_t)b->batch;
  int chunk = 256;  // multiple of 128 pairs: every array's chunk boundary stays 128-byte aligned (tools/tune_e2e.py)
  const char* genv = getenv("PLSVO_GATE_CHUNK");
  if (genv && atoi(genv) >= 128) chunk = atoi(genv) / 128 * 128;
  const int n_chunks = (int)((B + chunk - 1) / chunk);
  if (!c->h_flags || c->h_flags_cap < n_chunks) {
    if (c->h_flags) cudaFreeHost(c->h_flags);
    c->h_flags = nullptr;
    CK(cudaHostAlloc((void**)&c->h_flags, sizeof(unsigned int) * (size_t)n_chunks, cudaHostAllocDefault));
    c->h_flags_cap = n_chunks;
  }
  for (int k = 0; k < n_chunks; ++k) c->h_flags[k] = (unsigned int)(k + 1);
  // the copy stream must not overtake work already queued on the main stream; the arrival counter is
  // cleared on the main stream before the copy stream may bump it
  CK(ensure(c->d_counter, 256));
  unsigned int* d_arrived = static_cast<unsigned int*>(c->d_counter.p) + 32;
  CK(cudaMemsetAsync(d_arrived, 0, sizeof(unsigned int), c->stream));
  // PLSVO_TRACE_E2E=1: timeline of this call on stderr (chunk arrival times, kernel end, download end) — measurement aid
  const bool trace = getenv("PLSVO_TRACE_E2E") != nullptr;
  cudaEvent_t tr_start = nullptr, tr_chunk[64] = {nullptr}, tr_kernel = nullptr;
  const auto t_host0 = std::chrono::steady_clock::now();
  if (trace) {
    cudaEventCreate(&tr_start), cudaEventCreate(&tr_kernel);
    for (int k = 0; k < n_chunks && k < 64; ++k) cudaEventCreate(&tr_chunk[k]);
    cudaEventRecord(tr_start, c->stream);
  }
  CK(cudaEventRecord(c->start_ev, c->stream));
  CK(cudaStreamWaitEvent(c->copy_stream, c->start_ev, 0));
  // enqueue every copy first (asynchronous from pinned memory): the host-side sizing below and the kernel launch then
  // overlap with the DMA.  Every per-pair array of the whole batch first (a dozen large copies, ~a quarter of the bytes),
  // then the images chunk by chunk (two copies per chunk and level): few, large transfers keep the link near its peak
  // rate and the arrival flags then track the image stream alone.  On an error return settled() drains the copies.
  int rc = align_layout(c, b);
  if (rc == PLSVO_OK) rc = align_copy_features(c, b, c->copy_stream);
  // coarser levels that were not shipped: the persistent kernel halfSamples them pair by pair (a pyramid kernel behind
  // a chunk's copies could not become resident next to the grid that waits for it)
  if (rc == PLSVO_OK) rc = align_derive_levels(c, p->min_level, p->max_level, c->copy_stream, /*in_kernel=*/true);
  if (rc != PLSVO_OK) return rc;
  for (int k = 0; k < n_chunks; ++k) {
    const size_t b0 = (size_t)k * chunk, b1 = std::min<size_t>(b0 + chunk, B);
    rc = align_copy_images(c, b, b0, b1, c->copy_stream);
    if (rc != PLSVO_OK) return rc;
    CK(cudaMemcpyAsync(d_arrived, &c->h_flags[k], sizeof(unsigned int), cudaMemcpyHostToDevice, c->copy_stream));
    if (trace && k < 64) cudaEventRecord(tr_chunk[k], c->copy_stream);
  }
  const auto t_host1 = std::chrono::steady_clock::now();
  // host-side sizing (segment-sample bound of the finest level, outputs): on the launch path, so the cheap bound
  rc = align_size(c, b, p->min_level);
  AlignPlan plan;
  if (rc == PLSVO_OK) rc = align_plan(c, p, &plan, /*streamed=*/true);
  if (rc != PLSVO_OK) return rc;
  const auto t_host2 = std::chrono::steady_clock::now();
  rc = align_launch_kernel(c, plan, c->stream, chunk);  // gated on arrivals
  if (rc != PLSVO_OK) return rc;
  if (trace) cudaEventRecord(tr_kernel, c->stream);
  const auto t_host3 = std::chrono::steady_clock::now();
  rc = plsvo_align_download(ctx, o);
  if (trace) {
    const auto t_host4 = std::chrono::steady_clock::now();
    auto ms = [&](std::chrono::steady_clock::time_point t) { return std::chrono::duration<double, std::milli>(t - t_host0).count(); };
    std::fprintf(stderr, "[plsvo e2e trace] host: copies enqueued %.3f, sized+planned %.3f, launched %.3f, returned %.3f ms | device:", ms(t_host1),
                 ms(t_host2), ms(t_host3), ms(t_host4));
    for (int k = 0; k < n_chunks && k < 64; ++k) {
      float t = 0;
      cudaEventElapsedTime(&t, tr_start, tr_chunk[k]);
      std::fprintf(stderr, " chunk%d %.3f", k, t);
      cudaEventDestroy(tr_chunk[k]);
    }
    float t = 0;
    cudaEventElapsedTime(&t, tr_start, tr_kernel);
    std::fprintf(stderr, " kernel_end %.3f ms\n", t);
    cudaEventDestroy(tr_start), cudaEventDestroy(tr_kernel);
  }
  return rc;
}

int plsvo_align_batch_run(plsvo_ctx* ctx, const plsvo_align_batch* b, const plsvo_align_params* p,
                          const plsvo_align_result* o) {
  if (!ctx || !b || !p || !o) return PLSVO_ERR_INVALID;
  return settled(CTX(ctx), align_batch_run_body(ctx, b, p, o));
}

// ------------------------------------------------------------------------------------------------
// pose optimiser
// ------------------------------------------------------------------------------------------------
}  // extern "C"

namespace {
// device_T: poses already on the device (the chained call), instead of h->T_f_w
int poseopt_upload_impl(plsvo_ctx_impl* c, const plsvo_poseopt_batch* h, const double* device_T) {
  c->po_ready = false;
  if (h->batch <= 0 || h->n_pts < 0 || h->n_segs < 0) return fail(c, PLSVO_ERR_INVALID, "batch/n_pts/n_segs out of range");
  if (!h->T_f_w && !device_T) return fail(c, PLSVO_ERR_INVALID, "T_f_w missing");
  for (int b = 0; b < h->batch; ++b) {  // the counts index shared memory in the kernel
    if (h->pt_count && (h->pt_count[b] < 0 || h->pt_count[b] > h->n_pts)) return fail(c, PLSVO_ERR_INVALID, "pt_count[b] outside [0, n_pts]");
    if (h->seg_count && (h->seg_count[b] < 0 || h->seg_count[b] > h->n_segs))
      return fail(c, PLSVO_ERR_INVALID, "seg_count[b] outside [0, n_segs]");
  }
  if (h->n_pts > 0 && (!h->pt_f || !h->pt_pos || !h->pt_level)) return fail(c, PLSVO_ERR_INVALID, "point arrays missing");
  if (h->n_segs > 0 && (!h->seg_line || !h->seg_spos || !h->seg_epos || !h->seg_level))
    return fail(c, PLSVO_ERR_INVALID, "segment arrays missing");
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  PoseOptArgs& a = c->pa;
  const size_t B = (size_t)h->batch;
  a.B = h->batch, a.n_pts = h->n_pts, a.n_segs = h->n_segs, a.fx = h->fx;
  {
    const size_t np_ = (size_t)h->n_pts, ns_ = (size_t)h->n_segs;
    struct Item {
      const void* host;
      size_t bytes;
      const void** dev;
    };
    const Item items[] = {
        {device_T ? nullptr : h->T_f_w, B * 7 * 8, (const void**)&a.T_f_w},
        {h->pt_count, B * 4, (const void**)&a.pt_count},
        {h->pt_f, B * np_ * 24, (const void**)&a.pt_f},
        {h->pt_pos, B * np_ * 24, (const void**)&a.pt_pos},
        {h->pt_level, B * np_ * 4, (const void**)&a.pt_level},
        {h->pt_valid, B * np_, (const void**)&a.pt_valid},
        {h->seg_count, B * 4, (const void**)&a.seg_count},
        {h->seg_line, B * ns_ * 24, (const void**)&a.seg_line},
        {h->seg_spos, B * ns_ * 24, (const void**)&a.seg_spos},
        {h->seg_epos, B * ns_ * 24, (const void**)&a.seg_epos},
        {h->seg_level, B * ns_ * 4, (const void**)&a.seg_level},
        {h->seg_valid, B * ns_, (const void**)&a.seg_valid},
    };
    // every sent array at a 256-byte-aligned offset of p_in
    size_t total = 0;
    for (const Item& it : items)
      if (it.host && it.bytes) total += (it.bytes + 255) / 256 * 256;
    CK(ensure(c->p_in, total + 256));
    size_t off = 0;
    for (const Item& it : items) {
      *it.dev = it.host && it.bytes ? static_cast<char*>(c->p_in.p) + off : nullptr;
      if (it.host && it.bytes) off += (it.bytes + 255) / 256 * 256;
    }
    if (device_T) a.T_f_w = device_T;
    // small batches (the reference's own call is one frame, frame_handler_mono.cpp:327-329): every input packed into one
    // pinned block and moved with ONE copy instead of a dozen staged pageable ones
    const bool small = total > 0 && total <= ((size_t)4 << 20) && !getenv("PLSVO_NO_SMALL_UPLOAD");
    if (small) {
      if (c->h_in_cap < total + 256) {
        if (c->h_in_ev) CK(cudaEventSynchronize(c->h_in_ev));
        if (c->h_in) cudaFreeHost(c->h_in);
        c->h_in = nullptr, c->h_in_cap = 0;
        CK(cudaHostAlloc((void**)&c->h_in, total + 256, cudaHostAllocDefault));
        c->h_in_cap = total + 256;
      }
      if (!c->h_in_ev) CK(cudaEventCreateWithFlags(&c->h_in_ev, cudaEventDisableTiming));
      else CK(cudaEventSynchronize(c->h_in_ev));  // the previous packed upload has left the staging block
      for (const Item& it : items)
        if (it.host && it.bytes) memcpy(c->h_in + (static_cast<const char*>(*it.dev) - static_cast<char*>(c->p_in.p)), it.host, it.bytes);
      CK(cudaMemcpyAsync(c->p_in.p, c->h_in, total, cudaMemcpyHostToDevice, s));
      CK(cudaEventRecord(c->h_in_ev, s));
    } else {
      for (const Item& it : items)
        if (it.host && it.bytes) CK(cudaMemcpyAsync(const_cast<void*>(*it.dev), it.host, it.bytes, cudaMemcpyHostToDevice, s));
    }
  }
  // all outputs live in one device block: cleared with one memset where the kernel may leave them untouched, and brought
  // back with a single D2H into pinned staging
  {
    size_t o = 0;
    auto take = [&](size_t bytes) {
      const size_t at = o;
      o = (o + bytes + 255) / 256 * 256;
      return at;
    };
    const size_t oT = take(B * 7 * sizeof(double));
    const size_t ocov = take(B * 36 * sizeof(double)), oscale = take(B * sizeof(double)), oei = take(B * sizeof(double));
    const size_t oef = take(B * sizeof(double)), onpt = take(B * sizeof(long long)), onls = take(B * sizeof(long long));
    const size_t zero_end = o;
    const size_t opto = take(B * (size_t)std::max(1, h->n_pts)), osgo = take(B * (size_t)std::max(1, h->n_segs));
    const size_t oit = take(B * 2 * sizeof(int32_t)), ost = take(B * sizeof(int32_t));
    c->po_out_bytes = o, c->po_zero_off = ocov, c->po_zero_bytes = zero_end - ocov;
    CK(ensure(c->p_out_T, o));
    if (c->h_po_out_cap < o) {
      if (c->h_po_out) cudaFreeHost(c->h_po_out);
      c->h_po_out = nullptr, c->h_po_out_cap = 0;
      CK(cudaHostAlloc((void**)&c->h_po_out, o, cudaHostAllocDefault));
      c->h_po_out_cap = o;
    }
    char* base = static_cast<char*>(c->p_out_T.p);
    a.out_T = reinterpret_cast<double*>(base + oT);
    a.out_cov = reinterpret_cast<double*>(base + ocov);
    a.out_scale = reinterpret_cast<double*>(base + oscale);
    a.out_err_init = reinterpret_cast<double*>(base + oei);
    a.out_err_final = reinterpret_cast<double*>(base + oef);
    a.out_num_pt = reinterpret_cast<long long*>(base + onpt);
    a.out_num_ls = reinterpret_cast<long long*>(base + onls);
    a.out_pt_outlier = reinterpret_cast<uint8_t*>(base + opto);
    a.out_seg_outlier = reinterpret_cast<uint8_t*>(base + osgo);
    a.out_iters = reinterpret_cast<int32_t*>(base + oit);
    a.out_status = reinterpret_cast<int32_t*>(base + ost);
  }
  c->po_ready = true;
  return PLSVO_OK;
}
}  // namespace

extern "C" {

int plsvo_poseopt_upload(plsvo_ctx* ctx, const plsvo_poseopt_batch* h) {
  if (!ctx || !h) return PLSVO_ERR_INVALID;
  return poseopt_upload_impl(CTX(ctx), h, nullptr);
}

int plsvo_poseopt_launch(plsvo_ctx* ctx, const plsvo_poseopt_params* p) {
  if (!ctx || !p) return PLSVO_ERR_INVALID;
  plsvo_ctx_impl* c = CTX(ctx);
  if (!c->po_ready) return fail(c, PLSVO_ERR_STATE, "plsvo_poseopt_launch before plsvo_poseopt_upload");
  if (p->n_iter < 0) return fail(c, PLSVO_ERR_INVALID, "n_iter");
  CK(cudaSetDevice(c->device));
  PoseOptArgs& a = c->pa;
  a.reproj_thresh = p->reproj_thresh, a.n_iter = p->n_iter, a.n_iter_ref = p->n_iter_ref;
  const size_t smem = poseopt_smem_bytes(a.n_pts, a.n_segs);
  if (smem > (size_t)c->smem_optin) return fail(c, PLSVO_ERR_INVALID, "feature counts exceed shared memory");
  // outputs of frames that return early keep their previous contents: clear the ones we always report
  CK(cudaMemsetAsync(static_cast<char*>(c->p_out_T.p) + c->po_zero_off, 0, c->po_zero_bytes, c->stream));
  CK(poseopt_kernel_launch(a, smem, c->stream));
  c->launches += 1;
  return PLSVO_OK;
}

int plsvo_poseopt_download(plsvo_ctx* ctx, const plsvo_poseopt_result* o) {
  if (!ctx || !o) return PLSVO_ERR_INVALID;
  plsvo_ctx_impl* c = CTX(ctx);
  if (!c->po_ready) return fail(c, PLSVO_ERR_STATE, "plsvo_poseopt_download before plsvo_poseopt_upload");
  CK(cudaSetDevice(c->device));
  const PoseOptArgs& a = c->pa;
  const size_t B = (size_t)a.B;
  cudaStream_t s = c->stream;
  CK(cudaMemcpyAsync(c->h_po_out, c->p_out_T.p, c->po_out_bytes, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  {
    const char* dbase = static_cast<const char*>(c->p_out_T.p);
    auto host_of = [&](const void* dev) { return c->h_po_out + (static_cast<const char*>(dev) - dbase); };
    if (o->T_f_w) memcpy(o->T_f_w, host_of(a.out_T), B * 7 * sizeof(double));
    if (o->cov) memcpy(o->cov, host_of(a.out_cov), B * 36 * sizeof(double));
    if (o->estimated_scale) memcpy(o->estimated_scale, host_of(a.out_scale), B * sizeof(double));
    if (o->error_init) memcpy(o->error_init, host_of(a.out_err_init), B * sizeof(double));
    if (o->error_final) memcpy(o->error_final, host_of(a.out_err_final), B * sizeof(double));
    if (o->num_obs_pt) memcpy(o->num_obs_pt, host_of(a.out_num_pt), B * sizeof(int64_t));
    if (o->num_obs_ls) memcpy(o->num_obs_ls, host_of(a.out_num_ls), B * sizeof(int64_t));
    if (o->pt_outlier && a.n_pts > 0) memcpy(o->pt_outlier, host_of(a.out_pt_outlier), B * (size_t)a.n_pts);
    if (o->seg_outlier && a.n_segs > 0) memcpy(o->seg_outlier, host_of(a.out_seg_outlier), B * (size_t)a.n_segs);
    if (o->iters) memcpy(o->iters, host_of(a.out_iters), B * 2 * sizeof(int32_t));
    if (o->status) memcpy(o->status, host_of(a.out_status), B * sizeof(int32_t));
  }
  return PLSVO_OK;
}

// FrameHandlerMono::processFrame's two hot-path calls back to back (src/frame_handler_mono.cpp:272-274 and :327-329) for
// a batch of frames, without the pose leaving the device: sparse image alignment of (ref, cur), then the pose optimiser
// on cur's matched features starting from the aligned pose.  pb->T_f_w may be NULL (the usual case): frame b of the
// pose-optimiser batch then starts from the alignment result of pair b, read on the device.
int plsvo_track_upload(plsvo_ctx* ctx, const plsvo_align_batch* ab, const plsvo_poseopt_batch* pb) {
  if (!ctx || !ab || !pb) return PLSVO_ERR_INVALID;
  plsvo_ctx_impl* c = CTX(ctx);
  if (pb->batch != ab->batch) return fail(c, PLSVO_ERR_INVALID, "alignment and pose-optimiser batches differ in size");
  int rc = plsvo_align_upload(ctx, ab);
  if (rc != PLSVO_OK) return rc;
  // the pose optimiser reads the aligned poses where the alignment kernel leaves them (unless poses are given)
  return poseopt_upload_impl(c, pb, pb->T_f_w ? nullptr : c->aa.out_T);
}

int plsvo_track_launch(plsvo_ctx* ctx, const plsvo_align_params* ap, const plsvo_poseopt_params* pp) {
  if (!ctx || !ap || !pp) return PLSVO_ERR_INVALID;
  int rc = plsvo_align_launch(ctx, ap);  // the two kernels back to back on the context's stream
  if (rc != PLSVO_OK) return rc;
  return plsvo_poseopt_launch(ctx, pp);
}

int plsvo_track_batch_run(plsvo_ctx* ctx, const plsvo_align_batch* ab, const plsvo_align_params* ap,
                          const plsvo_poseopt_batch* pb, const plsvo_poseopt_params* pp, const plsvo_align_result* ao,
                          const plsvo_poseopt_result* po) {
  if (!ctx || !ab || !ap || !pb || !pp || !po) return PLSVO_ERR_INVALID;
  int rc = plsvo_track_upload(ctx, ab, pb);
  if (rc == PLSVO_OK) rc = plsvo_track_launch(ctx, ap, pp);
  if (rc == PLSVO_OK && ao) rc = plsvo_align_download(ctx, ao);
  if (rc == PLSVO_OK) rc = plsvo_poseopt_download(ctx, po);
  return settled(CTX(ctx), rc);
}

int plsvo_poseopt_batch_run(plsvo_ctx* ctx, const plsvo_poseopt_batch* b, const plsvo_poseopt_params* p,
                            const plsvo_poseopt_result* o) {
  if (!ctx || !b || !p || !o) return PLSVO_ERR_INVALID;
  int rc = plsvo_poseopt_upload(ctx, b);
  if (rc == PLSVO_OK) rc = plsvo_poseopt_launch(ctx, p);
  if (rc == PLSVO_OK) rc = plsvo_poseopt_download(ctx, o);
  return settled(CTX(ctx), rc);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// ATAN (FOV) camera: vk::ATANCamera instead of the undistorted pinhole
// ------------------------------------------------------------------------------------------------
namespace {

// Validates the camera against the batch and returns in *derived the batch with cam.fx / fy / cx / cy replaced by the
// ATANCamera members fx_, fy_, cx_, cy_ (what the kernels read as fx, fy, cx, cy).  Nothing is queued here.
int atan_batch(plsvo_ctx_impl* c, const plsvo_atan_camera* cam, const plsvo_align_batch* b, plsvo_align_batch* derived) {
  if (cam->width != b->cam.width || cam->height != b->cam.height)
    return fail(c, PLSVO_ERR_INVALID, "plsvo_atan_camera size differs from batch->cam");
  if (!std::isfinite(cam->fx) || !std::isfinite(cam->fy) || !std::isfinite(cam->cx) || !std::isfinite(cam->cy) ||
      !std::isfinite(cam->d0))
    return fail(c, PLSVO_ERR_INVALID, "plsvo_atan_camera has a non-finite parameter");
  if (!(cam->fx > 0.0) || !(cam->fy > 0.0)) return fail(c, PLSVO_ERR_INVALID, "plsvo_atan_camera fx and fy must be positive");
  *derived = *b;
  derived->cam.fx = (double)cam->width * cam->fx;
  derived->cam.fy = (double)cam->height * cam->fy;
  derived->cam.cx = cam->cx * (double)cam->width - 0.5;
  derived->cam.cy = cam->cy * (double)cam->height - 0.5;
  if (!std::isfinite(derived->cam.fx) || !std::isfinite(derived->cam.fy) || !(derived->cam.fx > 0.0) || !(derived->cam.fy > 0.0))
    return fail(c, PLSVO_ERR_INVALID, "plsvo_atan_camera focal length out of range");
  if (!align_atan_kernel_prepare || !align_atan_kernel_launch)
    return fail(c, PLSVO_ERR_CUDA, "this library was built without the ATAN alignment kernels");
  return PLSVO_OK;
}

// after the upload of the derived batch: select the ATAN kernels and give them the distortion terms of the constructor
void atan_select(plsvo_ctx_impl* c, const plsvo_atan_camera* cam) {
  AlignArgs& a = c->aa;
  c->atan = true;
  a.atan_s = cam->d0;
  a.atan_s_inv = a.atan_tans = a.atan_tans_inv = 0.0;
  if (cam->d0 != 0.0) {
    a.atan_tans = 2.0 * tan(cam->d0 / 2.0);
    a.atan_tans_inv = 1.0 / a.atan_tans;
    a.atan_s_inv = 1.0 / cam->d0;
  }
}

}  // namespace

extern "C" {

static int align_atan_body(plsvo_ctx* ctx, const plsvo_atan_camera* cam, const plsvo_align_batch* b, const plsvo_align_params* p,
                           const plsvo_align_result* o) {
  plsvo_ctx_impl* c = CTX(ctx);
  plsvo_align_batch d;
  int rc = atan_batch(c, cam, b, &d);
  if (rc == PLSVO_OK) rc = plsvo_align_upload(ctx, &d);
  if (rc != PLSVO_OK) return rc;
  atan_select(c, cam);
  rc = plsvo_align_launch(ctx, p);
  if (rc == PLSVO_OK) rc = plsvo_align_download(ctx, o);
  return rc;
}

int plsvo_align_atan_batch_run(plsvo_ctx* ctx, const plsvo_atan_camera* cam, const plsvo_align_batch* b,
                               const plsvo_align_params* p, const plsvo_align_result* o) {
  if (!ctx || !cam || !b || !p || !o) return PLSVO_ERR_INVALID;
  return settled(CTX(ctx), align_atan_body(ctx, cam, b, p, o));
}

static int track_atan_body(plsvo_ctx* ctx, const plsvo_atan_camera* cam, const plsvo_align_batch* ab, const plsvo_align_params* ap,
                           const plsvo_poseopt_batch* pb, const plsvo_poseopt_params* pp, const plsvo_align_result* ao,
                           const plsvo_poseopt_result* po) {
  plsvo_ctx_impl* c = CTX(ctx);
  plsvo_align_batch d;
  int rc = atan_batch(c, cam, ab, &d);
  if (rc == PLSVO_OK) rc = plsvo_track_upload(ctx, &d, pb);
  if (rc != PLSVO_OK) return rc;
  atan_select(c, cam);
  rc = plsvo_track_launch(ctx, ap, pp);
  if (rc == PLSVO_OK && ao) rc = plsvo_align_download(ctx, ao);
  if (rc == PLSVO_OK) rc = plsvo_poseopt_download(ctx, po);
  return rc;
}

int plsvo_track_atan_batch_run(plsvo_ctx* ctx, const plsvo_atan_camera* cam, const plsvo_align_batch* ab,
                               const plsvo_align_params* ap, const plsvo_poseopt_batch* pb, const plsvo_poseopt_params* pp,
                               const plsvo_align_result* ao, const plsvo_poseopt_result* po) {
  if (!ctx || !cam || !ab || !ap || !pb || !pp || !po) return PLSVO_ERR_INVALID;
  return settled(CTX(ctx), track_atan_body(ctx, cam, ab, ap, pb, pp, ao, po));
}

}  // extern "C"

static int pyramid_batch_run_body(plsvo_ctx* ctx, const plsvo_pyramid_batch* in, const plsvo_pyramid_result* out) {
  plsvo_ctx_impl* c = CTX(ctx);
  if (in->batch <= 0 || in->width <= 0 || in->height <= 0 || in->n_levels < 1 || in->n_levels > 7 || !in->img0 ||
      in->pitch0 < (size_t)in->width)
    return fail(c, PLSVO_ERR_INVALID, "pyramid batch description");
  CK(cudaSetDevice(c->device));
  PyramidArgs a;
  memset(&a, 0, sizeof a);
  a.B = in->batch, a.width = in->width, a.height = in->height, a.n_levels = in->n_levels;
  const size_t B = (size_t)in->batch;
  size_t total = 0, off[PLSVO_MAX_LEVELS] = {0};
  for (int l = 0; l < in->n_levels; ++l) {
    const int cols = in->width >> l, rows = in->height >> l;
    if (cols <= 0 || rows <= 0) return fail(c, PLSVO_ERR_INVALID, "pyramid level smaller than one pixel");
    if (l > 0 && !out->level[l]) return fail(c, PLSVO_ERR_INVALID, "output level missing");
    a.pitch[l] = (uint32_t)((cols + 15) / 16 * 16);
    a.stride[l] = (size_t)rows * a.pitch[l];
    total = (total + 255) / 256 * 256;
    off[l] = total;
    total += a.stride[l] * B;
  }
  CK(ensure(c->y_img, total + 256));
  for (int l = 0; l < in->n_levels; ++l) a.level[l] = static_cast<uint8_t*>(c->y_img.p) + off[l];
  cudaStream_t s = c->stream;
  if (in->stride0 == (size_t)in->height * in->pitch0) {
    CK(cudaMemcpy2DAsync(a.level[0], a.pitch[0], in->img0, in->pitch0, in->width, (size_t)in->height * B, cudaMemcpyHostToDevice, s));
  } else {
    for (size_t b = 0; b < B; ++b)
      CK(cudaMemcpy2DAsync(a.level[0] + b * a.stride[0], a.pitch[0], in->img0 + b * in->stride0, in->pitch0, in->width,
                           in->height, cudaMemcpyHostToDevice, s));
  }
  CK(kernel_timer(c, 0, s));
  const int rc = pyramid_launch(c, a, s);
  if (rc != PLSVO_OK) return rc;
  CK(kernel_timer(c, 1, s));
  for (int l = 1; l < in->n_levels; ++l) {
    const int cols = in->width >> l, rows = in->height >> l;
    if (out->pitch[l] < (size_t)cols) return fail(c, PLSVO_ERR_INVALID, "output pitch smaller than the level width");
    if (out->stride[l] == (size_t)rows * out->pitch[l]) {
      CK(cudaMemcpy2DAsync(out->level[l], out->pitch[l], a.level[l], a.pitch[l], cols, (size_t)rows * B, cudaMemcpyDeviceToHost, s));
    } else {
      for (size_t b = 0; b < B; ++b)
        CK(cudaMemcpy2DAsync(out->level[l] + b * out->stride[l], out->pitch[l], a.level[l] + b * a.stride[l], a.pitch[l], cols,
                             rows, cudaMemcpyDeviceToHost, s));
    }
  }
  CK(cudaStreamSynchronize(s));
  return PLSVO_OK;
}

namespace {
// align2D (dir == nullptr) and align1D (dir != nullptr) share staging and launch.
int feature_align_run(plsvo_ctx_impl* c, const plsvo_align2d_batch* in, const float* dir, double* o_px, uint8_t* o_conv,
                      double* o_hinv) {
  if (in->n_features < 0 || in->n_images <= 0 || in->width <= 0 || in->height <= 0 || in->n_iter < 0)
    return fail(c, PLSVO_ERR_INVALID, "align2d batch description");
  if (in->n_features == 0) return PLSVO_OK;
  if (!in->image_index || !in->level || !in->ref_patch_with_border || !in->ref_patch || !in->px || !o_px || !o_conv)
    return fail(c, PLSVO_ERR_INVALID, "align2d arrays missing");
  const size_t n = (size_t)in->n_features, B = (size_t)in->n_images;
  for (size_t i = 0; i < n; ++i) {
    const int l = in->level[i];
    if (l < 0 || l >= PLSVO_MAX_LEVELS || !in->img[l] || in->image_index[i] < 0 || in->image_index[i] >= in->n_images)
      return fail(c, PLSVO_ERR_INVALID, "align2d feature refers to a missing level or frame");
  }
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Align2DArgs a;
  memset(&a, 0, sizeof a);
  a.n = in->n_features, a.n_iter = in->n_iter, a.width = in->width, a.height = in->height;
  size_t total = 0, off[PLSVO_MAX_LEVELS] = {0};
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
    if (!in->img[l]) continue;
    const int cols = in->width >> l, rows = in->height >> l;
    if (cols <= 0 || rows <= 0 || in->img_pitch[l] < (size_t)cols) return fail(c, PLSVO_ERR_INVALID, "align2d level geometry");
    a.pitch[l] = (uint32_t)((cols + 15) / 16 * 16);
    a.stride[l] = (size_t)rows * a.pitch[l];
    total = (total + 255) / 256 * 256;
    off[l] = total;
    total += a.stride[l] * B;
  }
  CK(ensure(c->f_img, total + 256));
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
    if (!in->img[l]) continue;
    const int cols = in->width >> l, rows = in->height >> l;
    uint8_t* d = static_cast<uint8_t*>(c->f_img.p) + off[l];
    a.img[l] = d;
    if (in->img_stride[l] == (size_t)rows * in->img_pitch[l]) {
      CK(cudaMemcpy2DAsync(d, a.pitch[l], in->img[l], in->img_pitch[l], cols, (size_t)rows * B, cudaMemcpyHostToDevice, s));
    } else {
      for (size_t b = 0; b < B; ++b)
        CK(cudaMemcpy2DAsync(d + b * a.stride[l], a.pitch[l], in->img[l] + b * in->img_stride[l], in->img_pitch[l], cols, rows,
                             cudaMemcpyHostToDevice, s));
    }
  }
  CK(up(c->f_idx, in->image_index, n, s, &a.image_index));
  CK(up(c->f_lvl, in->level, n, s, &a.level));
  CK(up(c->f_border, in->ref_patch_with_border, n * 100, s, &a.ref_patch_with_border));
  CK(up(c->f_ref, in->ref_patch, n * 64, s, &a.ref_patch));
  CK(up(c->f_px, in->px, n * 2, s, &a.px));
  CK(ensure(c->f_opx, n * 2 * sizeof(double)));
  CK(ensure(c->f_oconv, n));
  a.out_px = static_cast<double*>(c->f_opx.p);
  a.out_converged = static_cast<uint8_t*>(c->f_oconv.p);
  if (dir) {
    CK(up(c->f_dir, dir, n * 2, s, &a.dir));
    CK(ensure(c->f_ohinv, n * sizeof(double)));
    a.out_h_inv = static_cast<double*>(c->f_ohinv.p);
  }
  CK(kernel_timer(c, 0, s));
  CK(dir ? align1d_kernel_launch(a, s) : align2d_kernel_launch(a, s));
  CK(kernel_timer(c, 1, s));
  c->launches += 1;
  CK(cudaMemcpyAsync(o_px, a.out_px, n * 2 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(o_conv, a.out_converged, n, cudaMemcpyDeviceToHost, s));
  if (dir && o_hinv) CK(cudaMemcpyAsync(o_hinv, a.out_h_inv, n * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return PLSVO_OK;
}
}  // namespace

extern "C" int plsvo_align2d_batch_run(plsvo_ctx* ctx, const plsvo_align2d_batch* in, const plsvo_align2d_result* out) {
  if (!ctx || !in || !out) return PLSVO_ERR_INVALID;
  return settled(CTX(ctx), feature_align_run(CTX(ctx), in, nullptr, out->px, out->converged, nullptr));
}

extern "C" int plsvo_align1d_batch_run(plsvo_ctx* ctx, const plsvo_align1d_batch* in, const plsvo_align1d_result* out) {
  if (!ctx || !in || !out) return PLSVO_ERR_INVALID;
  if (in->features.n_features > 0 && !in->dir) return fail(CTX(ctx), PLSVO_ERR_INVALID, "align1d directions missing");
  return settled(CTX(ctx), feature_align_run(CTX(ctx), &in->features, in->dir, out->px, out->converged, out->h_inv));
}

namespace {
// Copies the given pyramid levels of n_images frames to the device with 16-byte row pitch.
int stage_pyramid(plsvo_ctx_impl* c, DevBuf& buf, const uint8_t* const* img, const size_t* pitch, const size_t* stride, int n_images,
                  int width, int height, cudaStream_t s, const uint8_t** d_img, uint32_t* d_pitch, size_t* d_stride) {
  size_t total = 0, off[PLSVO_MAX_LEVELS] = {0};
  const size_t B = (size_t)n_images;
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
    d_img[l] = nullptr, d_pitch[l] = 0, d_stride[l] = 0;
    if (!img[l]) continue;
    const int cols = width >> l, rows = height >> l;
    if (cols <= 0 || rows <= 0 || pitch[l] < (size_t)cols) return fail(c, PLSVO_ERR_INVALID, "pyramid level geometry");
    d_pitch[l] = (uint32_t)((cols + 15) / 16 * 16);
    d_stride[l] = (size_t)rows * d_pitch[l];
    total = (total + 255) / 256 * 256;
    off[l] = total;
    total += d_stride[l] * B;
  }
  CK(ensure(buf, total + 256));
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
    if (!img[l]) continue;
    const int cols = width >> l, rows = height >> l;
    uint8_t* d = static_cast<uint8_t*>(buf.p) + off[l];
    d_img[l] = d;
    if (stride[l] == (size_t)rows * pitch[l]) {
      CK(cudaMemcpy2DAsync(d, d_pitch[l], img[l], pitch[l], cols, (size_t)rows * B, cudaMemcpyHostToDevice, s));
    } else {
      for (size_t b = 0; b < B; ++b)
        CK(cudaMemcpy2DAsync(d + b * d_stride[l], d_pitch[l], img[l] + b * stride[l], pitch[l], cols, rows, cudaMemcpyHostToDevice, s));
    }
  }
  return PLSVO_OK;
}
}  // namespace

static int match_direct_batch_run_body(plsvo_ctx* ctx, const plsvo_match_batch* in, const plsvo_match_result* out) {
  plsvo_ctx_impl* c = CTX(ctx);
  if (in->n_features < 0 || in->n_ref_images <= 0 || in->n_cur_images <= 0 || in->cam.width <= 0 || in->cam.height <= 0 ||
      in->n_iter < 0 || in->n_pyr_levels < 1 || in->n_pyr_levels > PLSVO_MAX_LEVELS)
    return fail(c, PLSVO_ERR_INVALID, "match batch description");
  if (in->n_features == 0) return PLSVO_OK;
  if (!in->T_ref_w || !in->T_cur_w || !in->ref_index || !in->cur_index || !in->ref_px || !in->ref_f || !in->ref_level || !in->pos ||
      !in->px_cur || !out->px_cur || !out->success)
    return fail(c, PLSVO_ERR_INVALID, "match arrays missing");
  if (in->is_edgelet && !in->ref_grad) return fail(c, PLSVO_ERR_INVALID, "edgelets need ref_grad");
  const size_t n = (size_t)in->n_features;
  for (int l = 0; l < in->n_pyr_levels; ++l)
    if (!in->cur_img[l]) return fail(c, PLSVO_ERR_INVALID, "current pyramid level missing below n_pyr_levels");
  for (size_t i = 0; i < n; ++i) {
    const int l = in->ref_level[i];
    if (l < 0 || l >= PLSVO_MAX_LEVELS || !in->ref_img[l] || in->ref_index[i] < 0 || in->ref_index[i] >= in->n_ref_images ||
        in->cur_index[i] < 0 || in->cur_index[i] >= in->n_cur_images)
      return fail(c, PLSVO_ERR_INVALID, "match candidate refers to a missing level or frame");
  }
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  MatchArgs a;
  memset(&a, 0, sizeof a);
  a.n = in->n_features, a.n_iter = in->n_iter, a.n_pyr_levels = in->n_pyr_levels;
  a.width = in->cam.width, a.height = in->cam.height;
  a.fx = in->cam.fx, a.fy = in->cam.fy, a.cx = in->cam.cx, a.cy = in->cam.cy;
  int rc = stage_pyramid(c, c->m_ref_img, in->ref_img, in->ref_pitch, in->ref_stride, in->n_ref_images, a.width, a.height, s, a.ref_img,
                         a.ref_pitch, a.ref_stride);
  if (rc != PLSVO_OK) return rc;
  rc = stage_pyramid(c, c->m_cur_img, in->cur_img, in->cur_pitch, in->cur_stride, in->n_cur_images, a.width, a.height, s, a.cur_img,
                     a.cur_pitch, a.cur_stride);
  if (rc != PLSVO_OK) return rc;
  CK(up(c->m_T_ref, in->T_ref_w, (size_t)in->n_ref_images * 7, s, &a.T_ref_w));
  CK(up(c->m_T_cur, in->T_cur_w, (size_t)in->n_cur_images * 7, s, &a.T_cur_w));
  CK(up(c->m_ridx, in->ref_index, n, s, &a.ref_index));
  CK(up(c->m_cidx, in->cur_index, n, s, &a.cur_index));
  CK(up(c->m_px, in->ref_px, n * 2, s, &a.ref_px));
  CK(up(c->m_f, in->ref_f, n * 3, s, &a.ref_f));
  CK(up(c->m_lvl, in->ref_level, n, s, &a.ref_level));
  CK(up(c->m_edge, in->is_edgelet, n, s, &a.is_edgelet));
  CK(up(c->m_grad, in->is_edgelet ? in->ref_grad : nullptr, n * 2, s, &a.ref_grad));
  CK(up(c->m_pos, in->pos, n * 3, s, &a.pos));
  CK(up(c->m_pxc, in->px_cur, n * 2, s, &a.px_cur));
  CK(ensure(c->m_opx, n * 2 * sizeof(double)));
  CK(ensure(c->m_osucc, n));
  CK(ensure(c->m_olvl, n * sizeof(int32_t)));
  a.out_px = static_cast<double*>(c->m_opx.p);
  a.out_success = static_cast<uint8_t*>(c->m_osucc.p);
  a.out_level = static_cast<int32_t*>(c->m_olvl.p);
  if (out->A_cur_ref) {
    CK(ensure(c->m_oA, n * 4 * sizeof(double)));
    a.out_A = static_cast<double*>(c->m_oA.p);
    // rows the kernel leaves untouched (in-frame test failed) must come back as the caller passed them
    CK(cudaMemcpyAsync(a.out_A, out->A_cur_ref, n * 4 * sizeof(double), cudaMemcpyHostToDevice, s));
  }
  CK(kernel_timer(c, 0, s));
  CK(match_direct_kernel_launch(a, s));
  CK(kernel_timer(c, 1, s));
  c->launches += 1;
  CK(cudaMemcpyAsync(out->px_cur, a.out_px, n * 2 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(out->success, a.out_success, n, cudaMemcpyDeviceToHost, s));
  if (out->search_level) CK(cudaMemcpyAsync(out->search_level, a.out_level, n * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  if (out->A_cur_ref) CK(cudaMemcpyAsync(out->A_cur_ref, a.out_A, n * 4 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return PLSVO_OK;
}

static int structopt_batch_run_body(plsvo_ctx* ctx, const plsvo_structopt_batch* in, const plsvo_structopt_result* out) {
  plsvo_ctx_impl* c = CTX(ctx);
  if (in->n_points < 0 || in->n_segs < 0 || in->n_frames <= 0 || in->n_iter_pts < 0 || in->n_iter_segs < 0 || !in->T_f_w)
    return fail(c, PLSVO_ERR_INVALID, "structopt batch description");
  if (in->n_points + in->n_segs == 0) return PLSVO_OK;
  if (in->n_points > 0 && (!in->pt_obs_begin || !in->pt_pos || !out->pt_pos)) return fail(c, PLSVO_ERR_INVALID, "structopt point arrays missing");
  if (in->n_segs > 0 && (!in->seg_obs_begin || !in->seg_spos || !in->seg_epos || !out->seg_spos || !out->seg_epos))
    return fail(c, PLSVO_ERR_INVALID, "structopt segment arrays missing");
  const size_t np = (size_t)in->n_points, ns = (size_t)in->n_segs;
  const size_t npo = np ? (size_t)in->pt_obs_begin[np] : 0, nso = ns ? (size_t)in->seg_obs_begin[ns] : 0;
  // observation lists: monotone offsets, frame indices in range
  for (size_t i = 0; i < np; ++i)
    if (in->pt_obs_begin[i] > in->pt_obs_begin[i + 1] || in->pt_obs_begin[i] < 0) return fail(c, PLSVO_ERR_INVALID, "pt_obs_begin not monotone");
  for (size_t i = 0; i < ns; ++i)
    if (in->seg_obs_begin[i] > in->seg_obs_begin[i + 1] || in->seg_obs_begin[i] < 0) return fail(c, PLSVO_ERR_INVALID, "seg_obs_begin not monotone");
  if ((npo && (!in->pt_obs_frame || !in->pt_obs_f)) || (nso && (!in->seg_obs_frame || !in->seg_obs_sf || !in->seg_obs_ef)))
    return fail(c, PLSVO_ERR_INVALID, "structopt observation arrays missing");
  for (size_t o = 0; o < npo; ++o)
    if (in->pt_obs_frame[o] < 0 || in->pt_obs_frame[o] >= in->n_frames) return fail(c, PLSVO_ERR_INVALID, "observation refers to a missing frame");
  for (size_t o = 0; o < nso; ++o)
    if (in->seg_obs_frame[o] < 0 || in->seg_obs_frame[o] >= in->n_frames) return fail(c, PLSVO_ERR_INVALID, "observation refers to a missing frame");
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  StructOptArgs a;
  memset(&a, 0, sizeof a);
  a.n_points = in->n_points, a.n_segs = in->n_segs, a.n_iter_pts = in->n_iter_pts, a.n_iter_segs = in->n_iter_segs;
  CK(up(c->s_T, in->T_f_w, (size_t)in->n_frames * 7, s, &a.T_f_w));
  CK(up(c->s_pb, in->pt_obs_begin, np ? np + 1 : 0, s, &a.pt_obs_begin));
  CK(up(c->s_pf, in->pt_obs_frame, npo, s, &a.pt_obs_frame));
  CK(up(c->s_pof, in->pt_obs_f, npo * 3, s, &a.pt_obs_f));
  CK(up(c->s_pp, in->pt_pos, np * 3, s, &a.pt_pos));
  CK(up(c->s_sb, in->seg_obs_begin, ns ? ns + 1 : 0, s, &a.seg_obs_begin));
  CK(up(c->s_sf, in->seg_obs_frame, nso, s, &a.seg_obs_frame));
  CK(up(c->s_ssf, in->seg_obs_sf, nso * 3, s, &a.seg_obs_sf));
  CK(up(c->s_sef, in->seg_obs_ef, nso * 3, s, &a.seg_obs_ef));
  CK(up(c->s_sp, in->seg_spos, ns * 3, s, &a.seg_spos));
  CK(up(c->s_ep, in->seg_epos, ns * 3, s, &a.seg_epos));
  CK(ensure(c->s_out, (np * 3 + ns * 6) * sizeof(double) + (np + ns) * sizeof(int32_t) + 64));
  a.out_pt_pos = static_cast<double*>(c->s_out.p);
  a.out_seg_spos = a.out_pt_pos + np * 3;
  a.out_seg_epos = a.out_seg_spos + ns * 3;
  a.out_pt_iters = reinterpret_cast<int32_t*>(a.out_seg_epos + ns * 3);
  a.out_seg_iters = a.out_pt_iters + np;
  CK(kernel_timer(c, 0, s));
  CK(structopt_kernel_launch(a, s));
  CK(kernel_timer(c, 1, s));
  c->launches += 1;
  if (np) CK(cudaMemcpyAsync(out->pt_pos, a.out_pt_pos, np * 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (ns) {
    CK(cudaMemcpyAsync(out->seg_spos, a.out_seg_spos, ns * 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(out->seg_epos, a.out_seg_epos, ns * 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
  }
  if (np && out->pt_iters) CK(cudaMemcpyAsync(out->pt_iters, a.out_pt_iters, np * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  if (ns && out->seg_iters) CK(cudaMemcpyAsync(out->seg_iters, a.out_seg_iters, ns * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return PLSVO_OK;
}

namespace {
// PLSVO_SEEDS_PER_WARP and PLSVO_EPI_SERIAL_STEPS force the search schedule of the seed kernels (tests, A/B runs).  Unset
// or empty means automatic (*v = -1).  Any other value must be a whole number in [lo, hi]: a switch that is set but not
// honoured would leave whoever set it measuring the automatic schedule without knowing.
int schedule_override(plsvo_ctx_impl* c, const char* name, int lo, int hi, int* v) {
  *v = -1;
  const char* e = getenv(name);
  if (!e || !*e) return PLSVO_OK;
  char* end = nullptr;
  errno = 0;
  const long x = strtol(e, &end, 10);
  if (end == e || *end || errno || x < lo || x > hi) {
    char msg[160];
    snprintf(msg, sizeof msg, "%s=\"%.40s\" is not a whole number in [%d, %d]", name, e, lo, hi);
    return fail(c, PLSVO_ERR_INVALID, msg);
  }
  *v = (int)x;
  return PLSVO_OK;
}

// point seeds (lin == nullptr) and line seeds share staging; the line variant adds the end-point arrays
int seed_update_run(plsvo_ctx_impl* c, const plsvo_seed_batch* in, const plsvo_seed_result* out, const plsvo_line_seed_batch* lin,
                    const plsvo_line_seed_result* lout) {
  if (in->n_seeds < 0 || in->n_ref_images <= 0 || in->n_cur_images <= 0 || in->cam.width <= 0 || in->cam.height <= 0 ||
      in->n_iter < 0 || in->n_pyr_levels < 1 || in->n_pyr_levels > PLSVO_MAX_LEVELS || in->max_epi_search_steps < 0)
    return fail(c, PLSVO_ERR_INVALID, "seed batch description");
  int spw = -1, serial_steps = -1;
  int rc = schedule_override(c, "PLSVO_SEEDS_PER_WARP", 1, 32, &spw);
  if (rc == PLSVO_OK) rc = schedule_override(c, "PLSVO_EPI_SERIAL_STEPS", 0, 100000, &serial_steps);
  if (rc != PLSVO_OK) return rc;
  if (in->n_seeds == 0) return PLSVO_OK;
  if (!in->T_ref_w || !in->T_cur_w || !in->ref_index || !in->cur_index || !in->ref_px || !in->ref_f || !in->ref_level || !in->a ||
      !in->b || !in->mu || !in->z_range || !in->sigma2 || !out->a || !out->b || !out->mu || !out->sigma2 || !out->status)
    return fail(c, PLSVO_ERR_INVALID, "seed arrays missing");
  if (!lin && in->is_edgelet && !in->ref_grad) return fail(c, PLSVO_ERR_INVALID, "edgelets need ref_grad");
  if (lin && (!lin->ref_sf || !lin->ref_ef || !lin->mu_e || !lin->z_range_e || !lin->sigma2_e || !lout->mu_e || !lout->sigma2_e))
    return fail(c, PLSVO_ERR_INVALID, "line-seed end-point arrays missing");
  const size_t n = (size_t)in->n_seeds;
  for (int l = 0; l < in->n_pyr_levels; ++l) {
    if (!in->cur_img[l]) return fail(c, PLSVO_ERR_INVALID, "current pyramid level missing below n_pyr_levels");
    // the reference strides the ZMSSD patch with Mat::cols (matcher.cpp:380-382): only dense images mean the same thing
    if (in->cur_pitch[l] != (size_t)(in->cam.width >> l)) return fail(c, PLSVO_ERR_INVALID, "current images must be dense (pitch == level width)");
  }
  for (size_t i = 0; i < n; ++i) {
    const int l = in->ref_level[i];
    if (l < 0 || l >= PLSVO_MAX_LEVELS || !in->ref_img[l] || in->ref_index[i] < 0 || in->ref_index[i] >= in->n_ref_images ||
        in->cur_index[i] < 0 || in->cur_index[i] >= in->n_cur_images)
      return fail(c, PLSVO_ERR_INVALID, "seed refers to a missing level or frame");
  }
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  SeedArgs a;
  memset(&a, 0, sizeof a);
  a.n = in->n_seeds, a.n_iter = in->n_iter, a.n_pyr_levels = in->n_pyr_levels, a.max_epi_search_steps = in->max_epi_search_steps;
  a.spw = spw, a.serial_steps = serial_steps;
  a.align_1d = in->align_1d, a.subpix_refinement = in->subpix_refinement, a.edgelet_filtering = in->epi_search_edgelet_filtering;
  a.edgelet_max_angle = in->epi_search_edgelet_max_angle, a.convergence_thresh = in->seed_convergence_sigma2_thresh;
  a.width = in->cam.width, a.height = in->cam.height;
  a.fx = in->cam.fx, a.fy = in->cam.fy, a.cx = in->cam.cx, a.cy = in->cam.cy;
  rc = stage_pyramid(c, c->m_ref_img, in->ref_img, in->ref_pitch, in->ref_stride, in->n_ref_images, a.width, a.height, s, a.ref_img,
                         a.ref_pitch, a.ref_stride);
  if (rc != PLSVO_OK) return rc;
  rc = stage_pyramid(c, c->m_cur_img, in->cur_img, in->cur_pitch, in->cur_stride, in->n_cur_images, a.width, a.height, s, a.cur_img,
                     a.cur_pitch, a.cur_stride);
  if (rc != PLSVO_OK) return rc;
  CK(up(c->m_T_ref, in->T_ref_w, (size_t)in->n_ref_images * 7, s, &a.T_ref_w));
  CK(up(c->m_T_cur, in->T_cur_w, (size_t)in->n_cur_images * 7, s, &a.T_cur_w));
  CK(up(c->m_ridx, in->ref_index, n, s, &a.ref_index));
  CK(up(c->m_cidx, in->cur_index, n, s, &a.cur_index));
  CK(up(c->m_px, in->ref_px, n * 2, s, &a.ref_px));
  CK(up(c->m_f, in->ref_f, n * 3, s, &a.ref_f));
  CK(up(c->m_lvl, in->ref_level, n, s, &a.ref_level));
  CK(up(c->m_edge, lin ? nullptr : in->is_edgelet, n, s, &a.is_edgelet));
  CK(up(c->m_grad, (!lin && in->is_edgelet) ? in->ref_grad : nullptr, n * 2, s, &a.ref_grad));
  if (lin) {
    CK(up(c->m_pos, lin->ref_sf, n * 3, s, &a.ref_sf));
    CK(up(c->m_pxc, lin->ref_ef, n * 3, s, &a.ref_ef));
    CK(up(c->d_smu_e, lin->mu_e, n, s, &a.mu_e));
    CK(up(c->d_szr_e, lin->z_range_e, n, s, &a.z_range_e));
    CK(up(c->d_ssig_e, lin->sigma2_e, n, s, &a.sigma2_e));
  }
  CK(up(c->d_sa, in->a, n, s, &a.a));
  CK(up(c->d_sb, in->b, n, s, &a.b));
  CK(up(c->d_smu, in->mu, n, s, &a.mu));
  CK(up(c->d_szr, in->z_range, n, s, &a.z_range));
  CK(up(c->d_ssig, in->sigma2, n, s, &a.sigma2));
  // outputs: [px_cur_e 2n f64][px_cur 2n f64][depth n f64][depth_e n f64][a b mu sigma2 mu_e sigma2_e n f32 each][status n i32][converged n u8]
  CK(ensure(c->d_sout, n * (16 + 16 + 8 + 8 + 24 + 4 + 1) + 64));
  a.out_px_cur_e = static_cast<double*>(c->d_sout.p);
  a.out_px_cur = a.out_px_cur_e + 2 * n;
  a.out_depth = a.out_px_cur + 2 * n;
  a.out_depth_e = a.out_depth + n;
  a.out_a = reinterpret_cast<float*>(a.out_depth_e + n);
  a.out_b = a.out_a + n, a.out_mu = a.out_b + n, a.out_sigma2 = a.out_mu + n;
  a.out_mu_e = a.out_sigma2 + n, a.out_sigma2_e = a.out_mu_e + n;
  a.out_status = reinterpret_cast<int32_t*>(a.out_sigma2_e + n);
  a.out_converged = reinterpret_cast<uint8_t*>(a.out_status + n);
  CK(kernel_timer(c, 0, s));
  CK(lin ? line_seed_update_kernel_launch(a, s) : seed_update_kernel_launch(a, s));
  CK(kernel_timer(c, 1, s));
  c->launches += 1;
  CK(cudaMemcpyAsync(out->a, a.out_a, n * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(out->b, a.out_b, n * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(out->mu, a.out_mu, n * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(out->sigma2, a.out_sigma2, n * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(out->status, a.out_status, n * 4, cudaMemcpyDeviceToHost, s));
  if (out->converged) CK(cudaMemcpyAsync(out->converged, a.out_converged, n, cudaMemcpyDeviceToHost, s));
  if (out->depth) CK(cudaMemcpyAsync(out->depth, a.out_depth, n * 8, cudaMemcpyDeviceToHost, s));
  if (out->px_cur) CK(cudaMemcpyAsync(out->px_cur, a.out_px_cur, n * 16, cudaMemcpyDeviceToHost, s));
  if (lin) {
    CK(cudaMemcpyAsync(lout->mu_e, a.out_mu_e, n * 4, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(lout->sigma2_e, a.out_sigma2_e, n * 4, cudaMemcpyDeviceToHost, s));
    if (lout->depth_e) CK(cudaMemcpyAsync(lout->depth_e, a.out_depth_e, n * 8, cudaMemcpyDeviceToHost, s));
    if (lout->px_cur_e) CK(cudaMemcpyAsync(lout->px_cur_e, a.out_px_cur_e, n * 16, cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  return PLSVO_OK;
}
}  // namespace

extern "C" int plsvo_seed_update_batch_run(plsvo_ctx* ctx, const plsvo_seed_batch* in, const plsvo_seed_result* out) {
  if (!ctx || !in || !out) return PLSVO_ERR_INVALID;
  return settled(CTX(ctx), seed_update_run(CTX(ctx), in, out, nullptr, nullptr));
}

extern "C" int plsvo_line_seed_update_batch_run(plsvo_ctx* ctx, const plsvo_line_seed_batch* in, const plsvo_line_seed_result* out) {
  if (!ctx || !in || !out) return PLSVO_ERR_INVALID;
  return settled(CTX(ctx), seed_update_run(CTX(ctx), &in->seeds, &out->seeds, in, out));
}

// exported forms of the three bodies above (see settled())
extern "C" int plsvo_pyramid_batch_run(plsvo_ctx* ctx, const plsvo_pyramid_batch* in, const plsvo_pyramid_result* out) {
  if (!ctx || !in || !out) return PLSVO_ERR_INVALID;
  return settled(CTX(ctx), pyramid_batch_run_body(ctx, in, out));
}

namespace {
// The CV_16SC2 map of a distorted camera, built on the device when the context's cached map is of another camera (or
// image size).  Sets u_map_built when it builds one (plsvo_last_map_build_ms).
int undistort_map_ensure(plsvo_ctx_impl* c, const plsvo_pinhole_camera& cam, cudaStream_t s) {
  if (c->u_map_ok && memcmp(&c->u_cam, &cam, sizeof cam) == 0) return PLSVO_OK;
  const int W = cam.width, H = cam.height;
  c->u_map_ok = false;
  const int mp = (W + kRemapTileW - 1) / kRemapTileW * kRemapTileW;
  const size_t n = (size_t)H * mp;
  CK(ensure(c->u_map1, n * sizeof(short2)));
  CK(ensure(c->u_map2, n * sizeof(uint16_t)));
  CK(cudaMemsetAsync(c->u_map1.p, 0, n * sizeof(short2), s));  // the row padding: read by whole-tile loads, never used
  CK(cudaMemsetAsync(c->u_map2.p, 0, n * sizeof(uint16_t), s));
  UndistortMapArgs m;
  m.width = W, m.height = H, m.map_pitch = mp;
  m.fx = (float)cam.fx, m.fy = (float)cam.fy, m.cx = (float)cam.cx, m.cy = (float)cam.cy;
  m.k1 = (float)cam.d[0], m.k2 = (float)cam.d[1], m.p1 = (float)cam.d[2], m.p2 = (float)cam.d[3], m.k3 = (float)cam.d[4];
  m.map1 = static_cast<short2*>(c->u_map1.p);
  m.map2 = static_cast<uint16_t*>(c->u_map2.p);
  CK(record_event(c->u_map_ev[0], s));
  CK(undistort_map_launch(m, s));
  CK(record_event(c->u_map_ev[1], s));
  c->launches += 1;
  c->u_cam = cam, c->u_map_pitch = mp, c->u_map_ok = true, c->u_map_built = true;
  return PLSVO_OK;
}

// vikit hands the parameters to OpenCV as Mat_<float>: they must stay finite, and fx, fy non-zero, after that rounding
int check_pinhole_params(plsvo_ctx_impl* c, const plsvo_pinhole_camera& cam, const char* who) {
  const double par[9] = {cam.fx, cam.fy, cam.cx, cam.cy, cam.d[0], cam.d[1], cam.d[2], cam.d[3], cam.d[4]};
  for (double p : par)
    if (!isfinite(p) || !isfinite((float)p)) return fail(c, PLSVO_ERR_INVALID, (std::string(who) + ": a parameter is not finite in float").c_str());
  if ((float)cam.fx == 0.f || (float)cam.fy == 0.f) return fail(c, PLSVO_ERR_INVALID, (std::string(who) + ": fx and fy must be non-zero").c_str());
  return PLSVO_OK;
}
}  // namespace

// vk::PinholeCamera::undistortImage + createImgPyramid for B frames: raw frames up, map (built once per camera), remap
// into level 0, pyramid kernel for levels 1.., every level down.
static int undistort_batch_run_body(plsvo_ctx* ctx, const plsvo_undistort_batch* in, const plsvo_pyramid_result* out) {
  plsvo_ctx_impl* c = CTX(ctx);
  c->u_map_built = false;
  const plsvo_pinhole_camera& cam = in->cam;
  const int W = cam.width, H = cam.height;
  if (in->batch <= 0 || W <= 0 || H <= 0) return fail(c, PLSVO_ERR_INVALID, "undistort batch: batch, width and height must be positive");
  if (in->n_levels < 1 || in->n_levels > 7) return fail(c, PLSVO_ERR_INVALID, "undistort batch: n_levels must be in [1,7]");
  if (!in->img0) return fail(c, PLSVO_ERR_INVALID, "undistort batch: raw frames missing (img0 is NULL)");
  if (in->pitch0 < (size_t)W) return fail(c, PLSVO_ERR_INVALID, "undistort batch: pitch0 smaller than the image width");
  if (check_pinhole_params(c, cam, "undistort camera") != PLSVO_OK) return PLSVO_ERR_INVALID;
  for (int l = 0; l < in->n_levels; ++l) {
    const int cols = W >> l, rows = H >> l;
    if (cols <= 0 || rows <= 0) return fail(c, PLSVO_ERR_INVALID, "pyramid level smaller than one pixel");
    if (!out->level[l]) return fail(c, PLSVO_ERR_INVALID, "output level missing (level 0 receives the rectified frame)");
    if (out->pitch[l] < (size_t)cols) return fail(c, PLSVO_ERR_INVALID, "output pitch smaller than the level width");
  }
  // PinholeCamera's distortion_ flag: without it undistortImage is a copy, so the raw frames go straight to level 0
  const bool distortion = fabs(cam.d[0]) > 0.0000001;
  if (distortion && (!undistort_map_launch || !undistort_remap_launch))
    return fail(c, PLSVO_ERR_CUDA, "undistort kernels are not linked into this library", cudaErrorNotSupported);
  CK(cudaSetDevice(c->device));
  PyramidArgs a;
  memset(&a, 0, sizeof a);
  a.B = in->batch, a.width = W, a.height = H, a.n_levels = in->n_levels;
  const size_t B = (size_t)in->batch;
  size_t total = 0, off[PLSVO_MAX_LEVELS] = {0};
  for (int l = 0; l < in->n_levels; ++l) {
    a.pitch[l] = (uint32_t)(((W >> l) + 15) / 16 * 16);
    a.stride[l] = (size_t)(H >> l) * a.pitch[l];
    total = (total + 255) / 256 * 256;
    off[l] = total;
    total += a.stride[l] * B;
  }
  CK(ensure(c->y_img, total + 256));
  for (int l = 0; l < in->n_levels; ++l) a.level[l] = static_cast<uint8_t*>(c->y_img.p) + off[l];
  cudaStream_t s = c->stream;
  uint8_t* raw = a.level[0];
  if (distortion) {
    CK(ensure(c->u_raw, a.stride[0] * B));
    raw = static_cast<uint8_t*>(c->u_raw.p);
  }
  if (in->stride0 == (size_t)H * in->pitch0) {
    CK(cudaMemcpy2DAsync(raw, a.pitch[0], in->img0, in->pitch0, W, (size_t)H * B, cudaMemcpyHostToDevice, s));
  } else {
    for (size_t b = 0; b < B; ++b)
      CK(cudaMemcpy2DAsync(raw + b * a.stride[0], a.pitch[0], in->img0 + b * in->stride0, in->pitch0, W, H, cudaMemcpyHostToDevice, s));
  }
  if (distortion) {
    const int rc = undistort_map_ensure(c, cam, s);
    if (rc != PLSVO_OK) return rc;
  }
  CK(kernel_timer(c, 0, s));
  if (distortion) {
    RemapArgs r;
    r.B = in->batch, r.width = W, r.height = H, r.map_pitch = c->u_map_pitch;
    r.map1 = static_cast<const short2*>(c->u_map1.p), r.map2 = static_cast<const uint16_t*>(c->u_map2.p);
    r.src = raw, r.src_pitch = a.pitch[0], r.src_stride = a.stride[0];
    r.dst = a.level[0], r.dst_pitch = a.pitch[0], r.dst_stride = a.stride[0];
    CK(undistort_remap_launch(r, c->num_sms, s));
    c->launches += 1;
  }
  const int rc = pyramid_launch(c, a, s);
  if (rc != PLSVO_OK) return rc;
  CK(kernel_timer(c, 1, s));
  for (int l = 0; l < in->n_levels; ++l) {
    const int cols = W >> l, rows = H >> l;
    if (out->stride[l] == (size_t)rows * out->pitch[l]) {
      CK(cudaMemcpy2DAsync(out->level[l], out->pitch[l], a.level[l], a.pitch[l], cols, (size_t)rows * B, cudaMemcpyDeviceToHost, s));
    } else {
      for (size_t b = 0; b < B; ++b)
        CK(cudaMemcpy2DAsync(out->level[l] + b * out->stride[l], out->pitch[l], a.level[l] + b * a.stride[l], a.pitch[l], cols, rows,
                             cudaMemcpyDeviceToHost, s));
    }
  }
  CK(cudaStreamSynchronize(s));
  return PLSVO_OK;
}

extern "C" int plsvo_undistort_batch_run(plsvo_ctx* ctx, const plsvo_undistort_batch* in, const plsvo_pyramid_result* out) {
  if (!ctx || !in || !out) return PLSVO_ERR_INVALID;
  return settled(CTX(ctx), undistort_batch_run_body(ctx, in, out));
}

extern "C" int plsvo_last_map_build_ms(plsvo_ctx* ctx, float* ms) {
  if (!ctx || !ms) return PLSVO_ERR_INVALID;
  plsvo_ctx_impl* c = CTX(ctx);
  if (!c->u_map_built) {
    *ms = -1.f;
    return PLSVO_OK;
  }
  CK(cudaEventSynchronize(c->u_map_ev[1]));
  CK(cudaEventElapsedTime(ms, c->u_map_ev[0], c->u_map_ev[1]));
  return PLSVO_OK;
}

// plsvo_align_raw_batch_run / plsvo_track_raw_batch_run (pb == NULL: alignment only): raw frames up, the camera's map
// (cached), one undistort_pyramid_kernel over every frame storing the levels alignment reads and those rect_out asks for,
// straight into the device layout of the alignment batch, then the alignment (and pose-optimiser) kernels as the plain
// upload -> launch -> download sequence runs them.  The arrival-gated streamed path is not taken.
static int raw_run_body(plsvo_ctx* ctx, const plsvo_raw_frames* raw, const plsvo_align_batch* ab, const plsvo_align_params* ap,
                        const plsvo_poseopt_batch* pb, const plsvo_poseopt_params* pp, const plsvo_align_result* ao,
                        const plsvo_poseopt_result* po, const plsvo_pyramid_result* rect) {
  plsvo_ctx_impl* c = CTX(ctx);
  c->u_map_built = false;
  const plsvo_pinhole_camera& cam = raw->cam;
  const int W = cam.width, H = cam.height;
  if (W <= 0 || H <= 0) return fail(c, PLSVO_ERR_INVALID, "raw frames: width and height must be positive");
  if (check_pinhole_params(c, cam, "raw-frame camera") != PLSVO_OK) return PLSVO_ERR_INVALID;
  if (ab->cam.width != W || ab->cam.height != H || ab->cam.fx != cam.fx || ab->cam.fy != cam.fy || ab->cam.cx != cam.cx ||
      ab->cam.cy != cam.cy)
    return fail(c, PLSVO_ERR_INVALID, "raw frames: batch->cam and raw->cam differ in width, height, fx, fy, cx or cy");
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l)
    if (ab->ref_img[l] || ab->cur_img[l])
      return fail(c, PLSVO_ERR_INVALID, "raw frames: image pointers in the alignment batch (the images come from the raw frames only)");
  const bool chain = (ab->flags & PLSVO_ALIGN_FRAME_CHAIN) != 0;
  if (!raw->ref_raw || (!chain && !raw->cur_raw)) return fail(c, PLSVO_ERR_INVALID, "raw frames missing (a raw stack is NULL)");
  if (chain && raw->cur_raw) return fail(c, PLSVO_ERR_INVALID, "raw frames: cur_raw must be NULL with PLSVO_ALIGN_FRAME_CHAIN");
  if (raw->pitch < (size_t)W) return fail(c, PLSVO_ERR_INVALID, "raw frames: pitch smaller than the image width");
  if (ap->min_level < 0 || ap->max_level < ap->min_level || ap->n_iter < 1) return fail(c, PLSVO_ERR_INVALID, "level range / n_iter");
  if (ap->max_level > 6) return fail(c, PLSVO_ERR_INVALID, "raw frames: max_level > 6 (one 64x64 level-0 tile holds levels 0..6)");
  if (pb && pb->batch != ab->batch) return fail(c, PLSVO_ERR_INVALID, "alignment and pose-optimiser batches differ in size");
  // the levels the kernel stores: [min_level, max_level] for alignment, and every level rect_out asks for
  bool want[PLSVO_MAX_LEVELS] = {false};
  int top = ap->max_level;
  for (int l = 0; l < PLSVO_MAX_LEVELS; ++l) {
    const bool out = rect && rect->level[l];
    want[l] = out || (l >= ap->min_level && l <= ap->max_level);
    if (!want[l]) continue;
    if (l > 6) return fail(c, PLSVO_ERR_INVALID, "rect_out: level above 6 (one 64x64 level-0 tile holds levels 0..6)");
    if ((W >> l) <= 0 || (H >> l) <= 0) return fail(c, PLSVO_ERR_INVALID, "pyramid level smaller than one pixel");
    if (out && rect->pitch[l] < (size_t)(W >> l)) return fail(c, PLSVO_ERR_INVALID, "rect_out: pitch smaller than the level width");
    top = std::max(top, l);
  }
  // PinholeCamera's distortion_ flag: without it level 0 is the raw frame itself
  const bool distortion = fabs(cam.d[0]) > 0.0000001;
  if (!undistort_pyramid_launch || (distortion && !undistort_map_launch))
    return fail(c, PLSVO_ERR_CUDA, "raw-frame rectification kernels are not linked into this library", cudaErrorNotSupported);
  // features, poses, outputs and the host-side sizing of the alignment batch (no image is shipped)
  int rc = plsvo_align_upload(ctx, ab);
  if (rc != PLSVO_OK) return rc;
  const size_t B = (size_t)ab->batch;
  if (pb) {
    rc = poseopt_upload_impl(c, pb, pb->T_f_w ? nullptr : c->aa.out_T);
    if (rc != PLSVO_OK) return rc;
  }
  cudaStream_t s = c->stream;
  AlignArgs& a = c->aa;
  // every frame in one stack per level: the B+1 frames of a chain, or the B reference frames followed by the B current ones
  const size_t n_frames = chain ? B + 1 : 2 * B;
  RawPyramidArgs r;
  memset(&r, 0, sizeof r);
  r.B = (int)n_frames, r.width = W, r.height = H, r.n_levels = top + 1;
  size_t total = 0, off[PLSVO_MAX_LEVELS] = {0};
  for (int l = 0; l <= top; ++l) {
    if (!want[l]) continue;
    r.pitch[l] = (uint32_t)(((W >> l) + 15) / 16 * 16);
    r.stride[l] = (size_t)(H >> l) * r.pitch[l];
    total = (total + 255) / 256 * 256;
    off[l] = total;
    total += r.stride[l] * n_frames;
  }
  CK(ensure(c->d_ref_img, total + 256));
  for (int l = 0; l <= top; ++l) {
    if (!want[l]) continue;
    r.level[l] = static_cast<uint8_t*>(c->d_ref_img.p) + off[l];
    a.ref_img[l] = r.level[l];
    a.cur_img[l] = r.level[l] + (chain ? 1 : B) * r.stride[l];
    a.pitch[l] = r.pitch[l], a.stride[l] = r.stride[l];
    c->lvl_uploaded[l] = true;  // present: align_derive_levels derives nothing
  }
  // raw frames: one linear copy per stack when the host layout is uniform (kept on the device), else frame by frame
  const bool uniform = raw->stride == (size_t)H * raw->pitch;
  r.src_pitch = uniform ? raw->pitch : (size_t)W;
  r.src_stride = uniform ? raw->stride : (size_t)H * W;
  CK(ensure(c->u_raw, r.src_stride * n_frames));
  uint8_t* d_raw = static_cast<uint8_t*>(c->u_raw.p);
  r.src = d_raw;
  const uint8_t* stacks[2] = {raw->ref_raw, chain ? nullptr : raw->cur_raw};
  const size_t per_stack = chain ? B + 1 : B;
  for (int k = 0; k < 2 && stacks[k]; ++k) {
    uint8_t* dst = d_raw + k * per_stack * r.src_stride;
    if (uniform) {
      // the last row of the last frame needs only W of its pitch bytes
      CK(cudaMemcpyAsync(dst, stacks[k], per_stack * r.src_stride - (raw->pitch - W), cudaMemcpyHostToDevice, s));
    } else {
      for (size_t f = 0; f < per_stack; ++f)
        CK(cudaMemcpy2DAsync(dst + f * r.src_stride, r.src_pitch, stacks[k] + f * raw->stride, raw->pitch, W, H, cudaMemcpyHostToDevice, s));
    }
  }
  if (distortion) {
    rc = undistort_map_ensure(c, cam, s);
    if (rc != PLSVO_OK) return rc;
    r.map_pitch = c->u_map_pitch;
    r.map1 = static_cast<const short2*>(c->u_map1.p), r.map2 = static_cast<const uint16_t*>(c->u_map2.p);
  }
  rc = align_derive_levels(c, ap->min_level, ap->max_level, s);
  if (rc != PLSVO_OK) return rc;
  AlignPlan plan;
  rc = align_plan(c, ap, &plan);
  if (rc != PLSVO_OK) return rc;
  CK(kernel_timer(c, 0, s));
  CK(undistort_pyramid_launch(r, c->num_sms, s));
  c->launches += 1;
  rc = align_launch_kernel(c, plan, s);
  if (rc == PLSVO_OK && pb) rc = plsvo_poseopt_launch(ctx, pp);
  if (rc != PLSVO_OK) return rc;
  CK(kernel_timer(c, 1, s));
  for (int l = 0; l <= top; ++l) {
    if (!rect || !rect->level[l]) continue;
    const int cols = W >> l, rows = H >> l;
    if (rect->stride[l] == (size_t)rows * rect->pitch[l]) {
      CK(cudaMemcpy2DAsync(rect->level[l], rect->pitch[l], r.level[l], r.pitch[l], cols, (size_t)rows * n_frames, cudaMemcpyDeviceToHost, s));
    } else {
      for (size_t f = 0; f < n_frames; ++f)
        CK(cudaMemcpy2DAsync(rect->level[l] + f * rect->stride[l], rect->pitch[l], r.level[l] + f * r.stride[l], r.pitch[l], cols, rows,
                             cudaMemcpyDeviceToHost, s));
    }
  }
  if (ao) {
    rc = plsvo_align_download(ctx, ao);
    if (rc != PLSVO_OK) return rc;
  }
  if (pb) return plsvo_poseopt_download(ctx, po);
  CK(cudaStreamSynchronize(s));
  return PLSVO_OK;
}

extern "C" int plsvo_align_raw_batch_run(plsvo_ctx* ctx, const plsvo_raw_frames* raw, const plsvo_align_batch* b,
                                         const plsvo_align_params* p, const plsvo_align_result* o, const plsvo_pyramid_result* rect_out) {
  if (!ctx || !raw || !b || !p || !o) return PLSVO_ERR_INVALID;
  return settled(CTX(ctx), raw_run_body(ctx, raw, b, p, nullptr, nullptr, o, nullptr, rect_out));
}

extern "C" int plsvo_track_raw_batch_run(plsvo_ctx* ctx, const plsvo_raw_frames* raw, const plsvo_align_batch* ab,
                                         const plsvo_align_params* ap, const plsvo_poseopt_batch* pb, const plsvo_poseopt_params* pp,
                                         const plsvo_align_result* ao, const plsvo_poseopt_result* po,
                                         const plsvo_pyramid_result* rect_out) {
  if (!ctx || !raw || !ab || !ap || !pb || !pp || !po) return PLSVO_ERR_INVALID;
  return settled(CTX(ctx), raw_run_body(ctx, raw, ab, ap, pb, pp, ao, po, rect_out));
}

extern "C" int plsvo_match_direct_batch_run(plsvo_ctx* ctx, const plsvo_match_batch* in, const plsvo_match_result* out) {
  if (!ctx || !in || !out) return PLSVO_ERR_INVALID;
  return settled(CTX(ctx), match_direct_batch_run_body(ctx, in, out));
}

extern "C" int plsvo_structopt_batch_run(plsvo_ctx* ctx, const plsvo_structopt_batch* in, const plsvo_structopt_result* out) {
  if (!ctx || !in || !out) return PLSVO_ERR_INVALID;
  return settled(CTX(ctx), structopt_batch_run_body(ctx, in, out));
}
