// dfk_api.cu -- C ABI of libdfk.so (see include/dfk.h): argument validation, host-side SE3
// algebra (relative pose + Jacobians, as the reference does on the host in
// cu_sfmaligner.cpp:164-166), launch planning, scratch ownership, error reporting.
//
// This unit: the handle, its parameters and profiling, dense RunStep (single, batch, host batch, stream), EvaluateError,
// the SE3 step, warp and tracker, UpdateDepth, the image helpers and DepthAligner.  The sparse factors are in
// dfk_api_sparse.cu, the keyframe window in dfk_api_window.cu, what they share in dfk_host.h.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "dfk.h"
#include "dfk_host.h"
#include "dfk_internal.h"
#include "dfk_se3.cuh"

using namespace dfk;

// pipelined host -> device -> host evaluation (dfk_sfm_stream_*)
struct DfkSfmStream {
  int device = 0, code_size = 0, max_items = 0, depth = 0;
  size_t max_bytes = 0;
  cudaStream_t copy_stream = nullptr;
  struct Slot {
    DeviceBuf<unsigned char> dev;   // staged inputs (+ valid0 / decoded-depth scratch)
    DeviceBuf<float> rec_dev;
    PinnedBuf<float> rec_host;
    cudaEvent_t uploaded = nullptr, done = nullptr;
    int n = 0;
    uint64_t ticket = 0;
    bool busy = false;
  };
  std::vector<Slot> slots;
  std::vector<DfkSfmWorkItem> dev_items;  // scratch of submit()
  uint64_t next_ticket = 0, next_wait = 0;
};

namespace {

// ---------------------------------------------------------------------------- SE3 algebra (fp32): dfk_se3.cuh
using se3f::relative_pose;

bool aligned(const void* p, size_t a) { return reinterpret_cast<uintptr_t>(p) % a == 0; }

// the inlier count a kernel stores as the bits of a float
uint32_t bits_of(float f)
{
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}

// a record [JtJ (nh) | Jtr (np) | residual | inliers] into the caller's outputs
void unpack_record(const float* rec, size_t nh, size_t np, float* JtJ, float* Jtr, float* residual, uint64_t* inliers)
{
  std::copy_n(rec, nh, JtJ);
  std::copy_n(rec + nh, np, Jtr);
  *residual = rec[nh + np];
  *inliers = bits_of(rec[nh + np + 1]);
}

bool track_level_ok(const DfkTrackLevel& L)
{
  const uint32_t W = L.img0.width, H = L.img0.height;
  return L.iterations >= 0 && W != 0 && H != 0 && img_ok(&L.img0, W, H, 1) && img_ok(&L.img1, W, H, 1) &&
         img_ok(&L.dpt0, W, H, 1) && img_ok(&L.grad1, W, H, 2) && cam_ok(&L.cam, W, H);
}

// One Se3TrackDesc: pose (used by RunStep; tracking reads the problem's device pose), border 1 and min_dpt 0
// (lucas_kanade_se3.h:52 defaults)
inline void set_se3_desc(Se3TrackDesc& d, const float pose[7], const DfkCamera& cam, const DfkImage& img0,
                         const DfkImage& img1, const DfkImage& dpt0, const DfkImage& grad1)
{
  d.pc = make_pixel_cam(pose, &cam, 1, 0.0f);
  d.img0 = view_of(&img0); d.img1 = view_of(&img1); d.dpt0 = view_of(&dpt0); d.grad1 = view_of(&grad1);
  d.width = (int)img0.width;
  d.height = (int)img0.height;
  d.nblocks = grid_for(d.width * d.height);
  d.grad_aligned = aligned(d.grad1.ptr, 8) && d.grad1.pitch % 2 == 0;
}

// an image, and its gradient view or none, as one pyramid level of the Sobel / blur-down kernels
PyrLevelDev pyr_level(const DfkImage* img, const DfkImage* grad)
{
  return PyrLevelDev{static_cast<float*>(img->ptr), (uint32_t)(img->pitch_bytes / 4), (int)img->width,
                     (int)img->height, grad ? static_cast<float*>(grad->ptr) : nullptr,
                     grad ? (uint32_t)(grad->pitch_bytes / 4) : 0u};
}

// one tracking problem's outputs from its last evaluated system (29 floats).  camera_tracker.cpp:65-69: inliers_ / error_
// are recorded at the LAST ITERATION OF LEVEL 0 only; with no level-0 iteration the reference keeps its previous values,
// so the outputs are left untouched then.  (Levels run coarse to fine, so the last evaluated system is level 0's last
// iteration whenever level 0 iterates at all.)
void track_outputs(const float* sys, const DfkTrackLevel& level0, float* inlier_fraction, float* error, float* last_system)
{
  if (level0.iterations > 0) {
    const uint32_t inl = bits_of(sys[28]), area = level0.img0.width * level0.img0.height;
    if (inlier_fraction) *inlier_fraction = area ? (float)inl / (float)area : 0.0f;
    if (error) *error = inl != 0 ? sys[27] / (float)inl : INFINITY;
  }
  if (last_system) memcpy(last_system, sys, sizeof(float) * 29);
}

uint32_t gcd_u32(uint32_t a, uint32_t b)
{
  while (b) {
    const uint32_t t = a % b;
    a = b;
    b = t;
  }
  return a;
}

// stride for the in-item tile permutation: ~golden-ratio of the tile count, coprime with it
uint32_t perm_multiplier(uint32_t n)
{
  if (n <= 2 || n > 65535u) return 1;  // keeps k * perm_mul below 2^32 on the device
  uint32_t m = (uint32_t)((double)n * 0.6180339887498949);
  if (m < 1) m = 1;
  while (gcd_u32(m, n) != 1) ++m;
  return m % n == 0 ? 1 : m;
}

constexpr size_t kMaxEventPairs = 8192;

// drains recorded event pairs into the accumulators (synchronizes the stream)
DfkStatus drain_events(DfkHandle h)
{
  if (h->ev_used == 0) return DFK_OK;
  DFK_CUDA(h, cudaStreamSynchronize(h->stream), "profiling: stream synchronize failed");
  for (size_t k = 0; k < h->ev_used; ++k) {
    float ms = 0.f;
    DFK_CUDA(h, cudaEventElapsedTime(&ms, h->ev_pool[2 * k], h->ev_pool[2 * k + 1]), "profiling: event read failed");
    h->ev_ms_accum += ms;
  }
  h->ev_count_accum += h->ev_used;
  h->ev_used = 0;
  return DFK_OK;
}

DfkStatus profile_events(DfkHandle h, cudaEvent_t* e0, cudaEvent_t* e1)
{
  if (h->ev_used == kMaxEventPairs) DFK_TRY(drain_events(h));
  while (h->ev_pool.size() < 2 * (h->ev_used + 1)) {
    cudaEvent_t e;
    DFK_CUDA(h, cudaEventCreate(&e), "profiling: event creation failed");
    h->ev_pool.push_back(e);
  }
  *e0 = h->ev_pool[2 * h->ev_used];
  *e1 = h->ev_pool[2 * h->ev_used + 1];
  h->ev_used += 1;
  return DFK_OK;
}

}  // namespace

DfkStatus build_items(DfkHandle h, const DfkSfmWorkItem* items, int n, int code_size, int tile_px, int max_ctas,
                      const float* codes_dev, SfmItemDev* out, SfmLaunchPlan* plan)
{
  const DfkDenseSfmParams& sp = h->params.sfmparams;
  for (int i = 0; i < n; ++i) {
    const DfkSfmWorkItem& w = items[i];
    SfmItemDev& d = out[i];
    const uint32_t W = w.img0.width, H = w.img0.height;
    if (W == 0 || H == 0) return fail(h, DFK_ERR_INVALID_ARG, "[SfmAligner::RunStep] empty image");
    if (!img_ok(&w.img0, W, H, 1) || !img_ok(&w.img1, W, H, 1) || !img_ok(&w.dpt0, W, H, 1) ||
        !img_ok(&w.valid0, W, H, 1) || !img_ok(&w.prx0_jac, W, H, code_size) || !img_ok(&w.grad1, W, H, 2))
      return fail(h, DFK_ERR_INVALID_ARG,
                  "[SfmAligner::RunStep] inconsistent image views (size, pitch or null pointer) in work item " +
                      std::to_string(i));
    if (!cam_ok(&w.cam, W, H))
      return fail(h, DFK_ERR_INVALID_ARG,
                  "[SfmAligner::RunStep] camera viewport larger than the image views in work item " + std::to_string(i));
    set_relative_pose(d, w.pose1, w.pose0, w.cam);
    d.border = (float)sp.valid_border;
    d.ulim = w.cam.width - (float)sp.valid_border;
    d.vlim = w.cam.height - (float)sp.valid_border;
    d.min_dpt = sp.min_dpt; d.avg_dpt = sp.avg_dpt; d.huber_delta = sp.huber_delta;
    d.img0 = (const float*)w.img0.ptr; d.img1 = (const float*)w.img1.ptr; d.dpt0 = (const float*)w.dpt0.ptr;
    d.valid0 = (float*)w.valid0.ptr; d.jac = (const float*)w.prx0_jac.ptr; d.grad1 = (const float*)w.grad1.ptr;
    d.img0_pitch = (uint32_t)(w.img0.pitch_bytes / 4); d.img1_pitch = (uint32_t)(w.img1.pitch_bytes / 4);
    d.dpt0_pitch = (uint32_t)(w.dpt0.pitch_bytes / 4); d.valid0_pitch = (uint32_t)(w.valid0.pitch_bytes / 4);
    d.jac_pitch = (uint32_t)(w.prx0_jac.pitch_bytes / 4); d.grad1_pitch = (uint32_t)(w.grad1.pitch_bytes / 4);
    d.dpt_out = nullptr; d.dpt_out_pitch = 0; d.code = nullptr;
    const bool fused = (w.code != nullptr);
    if (fused) {
      // UpdateDepth + RunStep in one pass: the tile loader stages prx_orig where it would stage dpt0, the front-end
      // decodes the depth (bit for bit what dfk_update_depth computes) and writes it to dpt0
      if (!img_ok(&w.prx_orig, W, H, 1))
        return fail(h, DFK_ERR_INVALID_ARG,
                    "[SfmAligner::RunStep] fused depth decode: inconsistent prx_orig view in work item " + std::to_string(i));
      d.dpt_out = (float*)w.dpt0.ptr;
      d.dpt_out_pitch = d.dpt0_pitch;
      d.dpt0 = (const float*)w.prx_orig.ptr;
      d.dpt0_pitch = (uint32_t)(w.prx_orig.pitch_bytes / 4);
      d.code = codes_dev + (size_t)i * code_size;
    }
    d.width = W; d.height = H; d.num_pixels = W * H;
    d.num_tiles = (d.num_pixels + tile_px - 1) / tile_px;
    d.perm_mul = perm_multiplier(d.num_tiles);
    d.mag_tiles = (uint32_t)((1ull << 32) / d.num_tiles);
    d.mag_width = (uint32_t)((1ull << 32) / W);
    d.flags = 0;
    const bool bulk = (W % 4 == 0) && aligned(d.img0, 16) && aligned(d.dpt0, 16) && aligned(d.jac, 16) &&
                      (d.img0_pitch % 4 == 0) && (d.dpt0_pitch % 4 == 0) && (d.jac_pitch % 4 == 0) &&
                      (code_size % 4 == 0);
    if (bulk) d.flags |= ITEM_FLAG_BULK;
    if (aligned(d.grad1, 8) && d.grad1_pitch % 2 == 0) d.flags |= ITEM_FLAG_GRAD_ALIGNED;
    if (fused) d.flags |= ITEM_FLAG_FUSED_DEPTH;
  }
  plan_tiles(out, n, max_ctas, plan);
  return DFK_OK;
}

// the tile plan of items whose num_tiles are set: their global tile ranges back to back, and which CTAs (and partial
// slots) each one's tiles fall to when CTA c of the grid owns global tiles [c T / G, (c + 1) T / G)
void plan_tiles(SfmItemDev* items, int n, int max_ctas, SfmLaunchPlan* plan)
{
  uint32_t tile_cursor = 0;
  for (int i = 0; i < n; ++i) {
    items[i].tile_begin = tile_cursor;
    tile_cursor += items[i].num_tiles;
  }
  const int T = (int)tile_cursor;
  int G = std::min(max_ctas, T);
  if (G < 1) G = 1;
  plan->num_items = n;
  plan->num_tiles = T;
  plan->num_ctas = G;
  // which CTAs touch which item (CTA c owns global tiles [c*T/G, (c+1)*T/G))
  uint32_t partial_cursor = 0;
  int c = 0;
  for (int i = 0; i < n; ++i) {
    SfmItemDev& d = items[i];
    const long long tb = d.tile_begin, te = tb + d.num_tiles;
    while ((long long)(c + 1) * T / G <= tb) ++c;  // first CTA whose range ends after tb
    int first = c, last = c;
    while ((long long)(last + 1) * T / G < te) ++last;
    d.first_cta = (uint32_t)first;
    d.num_ctas = (uint32_t)(last - first + 1);
    d.partial_begin = partial_cursor;
    partial_cursor += d.num_ctas;
  }
  plan->num_partials = (int)partial_cursor;
}

DfkStatus choose_step_kernel(DfkHandle h, const DfkSfmWorkItem* items, int n, int code_size, StepKernel* k)
{
  const bool wide = sfm_wide_supported(code_size);
  if (!sfm_fp32_supported(code_size) && !wide)
    return fail(h, DFK_ERR_UNSUPPORTED,
                "[SfmAligner::RunStep] no kernel instantiated for code size " + std::to_string(code_size));
  const bool tc_ok = sfm_tc_supported(code_size);
  bool tc = (h->gram_mode == DFK_GRAM_TF32X3) || (h->gram_mode == DFK_GRAM_AUTO && tc_ok);
  if (tc) {
    // the tensor-core kernels gather grad1 with 8-byte loads; odd layouts go to the fp32 / wide kernel (AUTO) or fail
    // (forced)
    bool grads_ok = true;
    for (int i = 0; i < n && grads_ok; ++i)
      grads_ok = items[i].grad1.ptr && aligned(items[i].grad1.ptr, 8) && (items[i].grad1.pitch_bytes % 8 == 0);
    if (!grads_ok) {
      if (h->gram_mode == DFK_GRAM_TF32X3)
        return fail(h, DFK_ERR_UNSUPPORTED, "[SfmAligner::RunStep] tensor-core path needs 8-byte aligned grad1 rows");
      tc = false;
    }
  }
  if (tc && !tc_ok)
    return fail(h, DFK_ERR_UNSUPPORTED,
                "[SfmAligner::RunStep] tensor-core Gram path is not instantiated for code size " +
                    std::to_string(code_size));
  k->tc = tc;
  k->wide = wide;
  k->tile_px = tc ? kSfmTcTilePixels : (wide ? sfm_wide_tile_pixels(code_size) : kTilePixels);
  const int ctas_per_sm = tc ? sfm_tc_ctas_per_sm(code_size) : (wide ? 1 : sfm_fp32_ctas_per_sm(code_size));
  const int sms = (h->sm_limit > 0 && h->sm_limit < h->num_sms) ? h->sm_limit : h->num_sms;
  k->max_ctas = ctas_per_sm * sms;
  k->pfloats = (tc && sfm_tc_writes_d(code_size)) ? sfm_tc_partial_floats(code_size) : sfm_partial_floats(code_size);
  return DFK_OK;
}

// the step kernel and the finalize of a planned, uploaded work list
DfkStatus launch_step(DfkHandle h, const StepKernel& k, int code_size, const SfmItemDev* items_dev, int n,
                      const SfmLaunchPlan& plan, float* partials_dev, float* records_dev)
{
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  if (h->profiling) DFK_TRY(profile_events(h, &ev0, &ev1));
  if (k.tc) {
    DFK_CUDA(h, launch_sfm_tc(code_size, items_dev, plan, partials_dev, h->stream, ev0, ev1),
             "[SfmAligner::RunStep] kernel launch failed");
  } else if (k.wide) {
    DFK_CUDA(h, launch_sfm_wide(code_size, items_dev, plan, partials_dev, h->stream, ev0, ev1),
             "[SfmAligner::RunStep] kernel launch failed");
  } else {
    DFK_CUDA(h, launch_sfm_fp32(code_size, items_dev, plan, partials_dev, h->stream, ev0, ev1),
             "[SfmAligner::RunStep] kernel launch failed");
  }
  DFK_CUDA(h, launch_sfm_finalize(code_size, k.tc, items_dev, n, partials_dev, records_dev, h->stream),
           "[SfmAligner::RunStep] kernel launch failed");
  h->launches += 2;  // step kernel + finalize kernel
  return DFK_OK;
}

namespace {

// Points every item at the ray table of its camera level in the handle's cache, filing the levels the cache has not
// seen; h->ray_pending lists the tables that are not built yet.
DfkStatus cache_ray_tables(DfkHandle h, SfmItemDev* items, int n)
{
  h->ray_pending.clear();
  // a caller cycling through more camera levels than the cache holds: start over (cudaFree synchronises).  Only here,
  // between calls, so that no item of a call is left pointing at a freed table
  if (h->ray_flush) {
    h->ray_cache.clear();
    h->ray_flush = false;
  }
  for (int i = 0; i < n; ++i) {
    SfmItemDev& d = items[i];
    const uint32_t W = d.width, H = d.height;
    size_t rt = 0;
    for (const auto& r : h->ray_cache) {
      if (r.fx == d.fx && r.fy == d.fy && r.u0 == d.u0 && r.v0 == d.v0 && r.w == W && r.h == H) break;
      ++rt;
    }
    if (rt == h->ray_cache.size()) {
      if (rt >= 256) h->ray_flush = true;
      DfkContext::RayTab r{d.fx, d.fy, d.u0, d.v0, W, H, {}, false};
      if (r.dev.ensure((size_t)W + H) != cudaSuccess)
        return fail(h, DFK_ERR_CUDA, "[SfmAligner::RunStep] scratch allocation failed");
      h->ray_cache.push_back(std::move(r));
    }
    d.ray_tab = h->ray_cache[rt].dev.ptr;
    if (!h->ray_cache[rt].built) h->ray_pending.push_back(rt);
  }
  return DFK_OK;
}

DfkStatus run_batch(DfkHandle h, const DfkSfmWorkItem* items, int n, int code_size, float* records_dev)
{
  if (!items || n <= 0 || !records_dev) return fail(h, DFK_ERR_INVALID_ARG, "[SfmAligner::RunStep] null/empty batch");
  StepKernel k;
  DFK_TRY(choose_step_kernel(h, items, n, code_size, &k));
  DeviceGuard guard(h->device);
  SfmLaunchPlan plan;
  bool any_fused = false;
  for (int i = 0; i < n; ++i) any_fused = any_fused || items[i].code != nullptr;
  if (any_fused)
    DFK_CUDA(h, h->codes_dev.ensure((size_t)n * code_size), "[SfmAligner::RunStep] scratch allocation failed");
  h->items_host.resize(n);
  DFK_TRY(build_items(h, items, n, code_size, k.tile_px, k.max_ctas, h->codes_dev.ptr, h->items_host.data(), &plan));
  DFK_TRY(cache_ray_tables(h, h->items_host.data(), n));
  if (any_fused) {
    h->codes_host.assign((size_t)n * code_size, 0.0f);
    for (int i = 0; i < n; ++i)
      if (items[i].code)
        memcpy(h->codes_host.data() + (size_t)i * code_size, items[i].code, sizeof(float) * code_size);
    DFK_CUDA(h, cudaMemcpyAsync(h->codes_dev.ptr, h->codes_host.data(), sizeof(float) * (size_t)n * code_size,
                                cudaMemcpyHostToDevice, h->stream),
             "[SfmAligner::RunStep] code upload failed");
  }
  DFK_CUDA(h, h->items_dev.ensure((size_t)n), "[SfmAligner::RunStep] scratch allocation failed");
  DFK_CUDA(h, h->partials_dev.ensure((size_t)plan.num_partials * k.pfloats), "[SfmAligner::RunStep] scratch allocation failed");
  SfmItemDev* items_dev = h->items_dev.ptr;
  DFK_CUDA(h, cudaMemcpyAsync(items_dev, h->items_host.data(), sizeof(SfmItemDev) * n, cudaMemcpyHostToDevice, h->stream),
           "[SfmAligner::RunStep] work list upload failed");
  if (!h->ray_pending.empty()) {  // the work list names a camera level the handle has no built table for yet
    DFK_CUDA(h, launch_sfm_ray_tables(items_dev, n, h->stream), "[SfmAligner::RunStep] kernel launch failed");
    for (size_t rt : h->ray_pending) h->ray_cache[rt].built = true;  // on the stream ahead of every later reader
    h->launches += 1;
  }
  return launch_step(h, k, code_size, items_dev, n, plan, h->partials_dev.ptr, records_dev);
}

}  // namespace

// ================================================================================== C ABI
extern "C" {

int dfk_version(void) { return DFK_VERSION; }

const char* dfk_status_string(DfkStatus s)
{
  switch (s) {
    case DFK_OK: return "ok";
    case DFK_ERR_INVALID_ARG: return "invalid argument";
    case DFK_ERR_CUDA: return "CUDA error";
    case DFK_ERR_UNSUPPORTED: return "unsupported";
    case DFK_ERR_NOMEM: return "out of memory";
  }
  return "unknown";
}

int dfk_sfm_supports_code_size(int code_size)
{
  return (sfm_fp32_supported(code_size) || sfm_wide_supported(code_size)) ? 1 : 0;
}

DfkStatus dfk_create(int device, DfkHandle* out)
{
  try {
    if (!out) return DFK_ERR_INVALID_ARG;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) return DFK_ERR_CUDA;
    if (device < 0) {
      if (cudaGetDevice(&device) != cudaSuccess) return DFK_ERR_CUDA;
    }
    if (device >= count) return DFK_ERR_INVALID_ARG;
    DfkContext* h = new (std::nothrow) DfkContext();
    if (!h) return DFK_ERR_NOMEM;
    h->device = device;
    h->params.sfmparams = DfkDenseSfmParams{0.1f, 1000.f, 2.0f, 0.0f, 2};
    h->params.step_threads = 32; h->params.step_blocks = 11; h->params.eval_threads = 224; h->params.eval_blocks = 66;
    DeviceGuard guard(device);
    bool ok = true;
    ok = ok && cudaDeviceGetAttribute(&h->num_sms, cudaDevAttrMultiProcessorCount, device) == cudaSuccess;
    ok = ok && cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking) == cudaSuccess;
    h->stream = h->own_stream;
    ok = ok && h->simple_scratch.ensure(kSimpleScratchFloats) == cudaSuccess;
    ok = ok && h->counter.ensure(1) == cudaSuccess;
    ok = ok && h->out_dev.ensure(32) == cudaSuccess;
    ok = ok && h->code_dev.ensure(256) == cudaSuccess;
    ok = ok && h->out_host.ensure(32) == cudaSuccess;
    ok = ok && cudaMemset(h->counter.ptr, 0, sizeof(unsigned int)) == cudaSuccess;
    if (!ok) {
      dfk_destroy(h);
      return DFK_ERR_CUDA;
    }
    *out = h;
    return DFK_OK;
  } catch (...) {
    return DFK_ERR_NOMEM;
  }
}

DfkStatus dfk_destroy(DfkHandle h)
{
  if (!h) return DFK_OK;
  DeviceGuard guard(h->device);
  if (h->own_stream) cudaStreamSynchronize(h->own_stream);
  delete h;
  return DFK_OK;
}

DfkStatus dfk_set_stream(DfkHandle h, void* cuda_stream)
{
  return guarded(h, [&] {
    h->stream = static_cast<cudaStream_t>(cuda_stream);
    return DFK_OK;
  });
}

DfkStatus dfk_use_own_stream(DfkHandle h)
{
  return guarded(h, [&] {
    h->stream = h->own_stream;
    return DFK_OK;
  });
}

DfkStatus dfk_set_sm_limit(DfkHandle h, int num_sms)
{
  return guarded(h, [&] {
    if (num_sms < 0) return fail(h, DFK_ERR_INVALID_ARG, "[dfk_set_sm_limit] num_sms < 0");
    h->sm_limit = num_sms;
    return DFK_OK;
  });
}

void* dfk_get_stream(DfkHandle h) { return h ? h->stream : nullptr; }

DfkStatus dfk_synchronize(DfkHandle h)
{
  return guarded(h, [&] {
    DeviceGuard guard(h->device);
    DFK_CUDA(h, cudaStreamSynchronize(h->stream), "stream synchronize failed");
    return DFK_OK;
  });
}

const char* dfk_last_error(DfkHandle h) { return h ? h->err.c_str() : "null handle"; }

DfkStatus dfk_set_profiling(DfkHandle h, int enabled)
{
  return guarded(h, [&] {
    h->profiling = enabled != 0;
    return DFK_OK;
  });
}

DfkStatus dfk_get_profile(DfkHandle h, double* main_kernel_ms, uint64_t* main_kernel_launches,
                          uint64_t* total_kernel_launches)
{
  return guarded(h, [&] {
    DeviceGuard guard(h->device);
    DFK_TRY(drain_events(h));
    if (main_kernel_ms) *main_kernel_ms = h->ev_ms_accum;
    if (main_kernel_launches) *main_kernel_launches = h->ev_count_accum;
    if (total_kernel_launches) *total_kernel_launches = h->launches;
    h->ev_ms_accum = 0.0;
    h->ev_count_accum = 0;
    h->launches = 0;
    return DFK_OK;
  });
}

DfkStatus dfk_sfm_set_params(DfkHandle h, const DfkSfmAlignerParams* p)
{
  return guarded(h, [&] {
    if (!p) return DFK_ERR_INVALID_ARG;
    // CHECK_EQ(threads % 32, 0), CHECK_LE(blocks, max_blocks) (cu_sfmaligner.cpp:187-203)
    if (p->step_threads % 32 != 0 || p->eval_threads % 32 != 0)
      return fail(h, DFK_ERR_INVALID_ARG, "threads must be a multiple of 32!");
    if (p->step_blocks > 1024 || p->eval_blocks > 1024) return fail(h, DFK_ERR_INVALID_ARG, "blocks must be less than 1024");
    if (p->sfmparams.valid_border < 1)
      return fail(h, DFK_ERR_INVALID_ARG, "valid_border must be >= 1 (bilinear sampling reads ix+1, iy+1)");
    h->params = *p;
    return DFK_OK;
  });
}

DfkStatus dfk_sfm_get_params(DfkHandle h, DfkSfmAlignerParams* p)
{
  return guarded(h, [&] {
    if (!p) return DFK_ERR_INVALID_ARG;
    *p = h->params;
    return DFK_OK;
  });
}

DfkStatus dfk_sfm_set_gram_mode(DfkHandle h, DfkGramMode m)
{
  return guarded(h, [&] {
    if (m != DFK_GRAM_AUTO && m != DFK_GRAM_FP32 && m != DFK_GRAM_TF32X3)
      return fail(h, DFK_ERR_INVALID_ARG, "unknown gram mode");
    h->gram_mode = m;
    return DFK_OK;
  });
}

DfkStatus dfk_se3_set_huber_delta(DfkHandle h, float v)
{
  return guarded(h, [&] {
    h->se3_huber_delta = v;
    return DFK_OK;
  });
}

DfkStatus dfk_sfm_run_step_batch(DfkHandle h, const DfkSfmWorkItem* items, int n, int code_size, float* records_dev)
{
  return guarded(h, [&] { return run_batch(h, items, n, code_size, records_dev); });
}

DfkStatus dfk_sfm_run_step_batch_host(DfkHandle h, const DfkSfmWorkItem* items, int n, int code_size,
                                      float* records_host)
{
  return guarded(h, [&] {
    if (!records_host || n <= 0) return fail(h, DFK_ERR_INVALID_ARG, "[SfmAligner::RunStep] null/empty batch");
    if (!dfk_sfm_supports_code_size(code_size))
      return fail(h, DFK_ERR_UNSUPPORTED,
                  "[SfmAligner::RunStep] no kernel instantiated for code size " + std::to_string(code_size));
    DeviceGuard guard(h->device);
    const size_t rec = (size_t)DFK_SFM_RECORD_FLOATS(code_size);
    DFK_CUDA(h, h->records_dev.ensure(rec * n), "[SfmAligner::RunStep] scratch allocation failed");
    DFK_CUDA(h, h->records_host.ensure(rec * n), "[SfmAligner::RunStep] pinned allocation failed");
    DFK_TRY(run_batch(h, items, n, code_size, h->records_dev.ptr));
    DFK_TRY(download(h, h->records_host.ptr, h->records_dev.ptr, rec * n * sizeof(float),
                     "[SfmAligner::RunStep] result download failed", "[SfmAligner::RunStep] kernel launch failed"));
    memcpy(records_host, h->records_host.ptr, rec * n * sizeof(float));
    return DFK_OK;
  });
}

DfkStatus dfk_sfm_run_step(DfkHandle h, const float pose0[7], const float pose1[7], const float* /*code0*/,
                           int code_size, const DfkCamera* cam, const DfkImage* img0, const DfkImage* img1,
                           const DfkImage* dpt0, const DfkImage* /*std0*/, const DfkImage* valid0,
                           const DfkImage* prx0_jac, const DfkImage* grad1, float* JtJ, float* Jtr, float* residual,
                           uint64_t* inliers)
{
  return guarded(h, [&] {
    if (!pose0 || !pose1 || !cam || !img0 || !img1 || !dpt0 || !valid0 || !prx0_jac || !grad1 || !JtJ || !Jtr ||
        !residual || !inliers)
      return fail(h, DFK_ERR_INVALID_ARG, "[SfmAligner::RunStep] null argument");
    DfkSfmWorkItem w{};  // no fused depth decode: code = NULL
    memcpy(w.pose0, pose0, sizeof(w.pose0));
    memcpy(w.pose1, pose1, sizeof(w.pose1));
    w.cam = *cam;
    w.img0 = *img0; w.img1 = *img1; w.dpt0 = *dpt0; w.valid0 = *valid0; w.prx0_jac = *prx0_jac; w.grad1 = *grad1;
    const int NP = 12 + code_size;
    const int NH = NP * (NP + 1) / 2;
    std::vector<float> rec((size_t)DFK_SFM_RECORD_FLOATS(code_size));
    DFK_TRY(dfk_sfm_run_step_batch_host(h, &w, 1, code_size, rec.data()));
    unpack_record(rec.data(), NH, NP, JtJ, Jtr, residual, inliers);
    return DFK_OK;
  });
}

static DfkStatus fetch_out(DfkHandle h, int nfloats, const char* what)
{
  h->launches += 1;
  return download(h, h->out_host.ptr, h->out_dev.ptr, sizeof(float) * nfloats, what, what);
}

DfkStatus dfk_sfm_evaluate_error(DfkHandle h, const float pose0[7], const float pose1[7], const DfkCamera* cam,
                                 const DfkImage* img0, const DfkImage* img1, const DfkImage* dpt0,
                                 const DfkImage* /*std0*/, const DfkImage* /*grad1*/, float* residual,
                                 uint64_t* inliers)
{
  return guarded(h, [&] {
    if (!pose0 || !pose1 || !cam || !img0 || !img1 || !dpt0 || !residual || !inliers)
      return fail(h, DFK_ERR_INVALID_ARG, "[SfmAligner::EvaluateError] null argument");
    const uint32_t W = img0->width, H = img0->height;
    if (W == 0 || H == 0 || !img_ok(img0, W, H, 1) || !img_ok(img1, W, H, 1) || !img_ok(dpt0, W, H, 1))
      return fail(h, DFK_ERR_INVALID_ARG, "[SfmAligner::EvaluateError] inconsistent image views");
    if (!cam_ok(cam, W, H)) return fail(h, DFK_ERR_INVALID_ARG, "[SfmAligner::EvaluateError] camera viewport larger than the image views");
    DeviceGuard guard(h->device);
    float p10[7];
    relative_pose(pose1, pose0, p10, nullptr, nullptr);  // cu_sfmaligner.cpp:131
    EvalErrorDesc d;
    int rows = 0, max_blocks = 1;
    set_eval_error_desc(d, *cam, p10, *img0, *img1, *dpt0, &rows, &max_blocks);
    DFK_CUDA(h, launch_eval_error(d, h->params.sfmparams.huber_delta, h->simple_scratch.ptr, h->counter.ptr,
                                  h->out_dev.ptr, h->stream),
             "[SfmAligner::EvaluateError] kernel launch failed");
    DFK_TRY(fetch_out(h, 2, "[SfmAligner::EvaluateError] kernel launch failed"));
    unpack_record(h->out_host.ptr, 0, 0, nullptr, nullptr, residual, inliers);
    return DFK_OK;
  });
}

DfkStatus dfk_sfm_evaluate_error_batch(DfkHandle h, const DfkSfmWorkItem* items, int n, float* out_dev)
{
  return guarded(h, [&] {
    if (!items || !out_dev || n < 1 || n > 65535)  // blockIdx.y of the kernel is the item
      return fail(h, DFK_ERR_INVALID_ARG,
                  "[SfmAligner::EvaluateError batch] null argument / number of items not in [1, 65535]");
    Staging s(h->staging);
    const Part<EvalErrorDesc> descs = s.add<EvalErrorDesc>(n);
    int max_blocks = 1, rows = 0;
    for (int i = 0; i < n; ++i) {
      const DfkSfmWorkItem& w = items[i];
      const std::string at = " in work item " + std::to_string(i);
      if (w.code)
        return fail(h, DFK_ERR_INVALID_ARG,
                    "[SfmAligner::EvaluateError batch] no fused depth decode: the depth is read from dpt0" + at);
      const uint32_t W = w.img0.width, H = w.img0.height;
      if (W == 0 || H == 0 || !img_ok(&w.img0, W, H, 1) || !img_ok(&w.img1, W, H, 1) || !img_ok(&w.dpt0, W, H, 1))
        return fail(h, DFK_ERR_INVALID_ARG, "[SfmAligner::EvaluateError batch] inconsistent image views" + at);
      if (!cam_ok(&w.cam, W, H))
        return fail(h, DFK_ERR_INVALID_ARG,
                    "[SfmAligner::EvaluateError batch] camera viewport larger than the image views" + at);
      float p10[7];
      relative_pose(w.pose1, w.pose0, p10, nullptr, nullptr);
      set_eval_error_desc(descs.at(s.host())[i], w.cam, p10, w.img0, w.img1, w.dpt0, &rows, &max_blocks);
    }
    DeviceGuard guard(h->device);
    DFK_CUDA(h, h->eval_partials.ensure((size_t)rows * 32), "[SfmAligner::EvaluateError batch] scratch allocation failed");
    DFK_TRY(ensure_tickets(h, h->eval_counters, (size_t)n, "[SfmAligner::EvaluateError batch] scratch allocation failed",
                           "[SfmAligner::EvaluateError batch] memset failed"));
    DFK_TRY(s.upload(h, h->eval_descs, "[SfmAligner::EvaluateError batch] "));
    DFK_CUDA(h, launch_eval_error(descs.at(s.dev), n, max_blocks, h->params.sfmparams.huber_delta, h->eval_partials.ptr,
                                  h->eval_counters.ptr, out_dev, h->stream),
             "[SfmAligner::EvaluateError batch] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_se3_run_step(DfkHandle h, const float se3[7], const DfkCamera* cam, const DfkImage* img0,
                           const DfkImage* img1, const DfkImage* dpt0, const DfkImage* grad1, float* JtJ, float* Jtr,
                           float* residual, uint64_t* inliers)
{
  return guarded(h, [&] {
    if (!se3 || !cam || !img0 || !img1 || !dpt0 || !grad1 || !JtJ || !Jtr || !residual || !inliers)
      return fail(h, DFK_ERR_INVALID_ARG, "[SE3Aligner::RunStep] null argument");
    const uint32_t W = img0->width, H = img0->height;
    if (W == 0 || H == 0 || !img_ok(img0, W, H, 1) || !img_ok(img1, W, H, 1) || !img_ok(dpt0, W, H, 1) ||
        !img_ok(grad1, W, H, 2))
      return fail(h, DFK_ERR_INVALID_ARG, "[SE3Aligner::RunStep] inconsistent image views");
    if (!cam_ok(cam, W, H)) return fail(h, DFK_ERR_INVALID_ARG, "[SE3Aligner::RunStep] camera viewport larger than the image views");
    DeviceGuard guard(h->device);
    Se3TrackDesc d;
    set_se3_desc(d, se3, *cam, *img0, *img1, *dpt0, *grad1);
    DFK_CUDA(h, launch_se3_step(d, h->se3_huber_delta, h->simple_scratch.ptr, h->counter.ptr, h->out_dev.ptr, nullptr,
                                nullptr, h->stream),
             "[SE3Aligner::RunStep] Kernel launch failed");
    DFK_TRY(fetch_out(h, 29, "[SE3Aligner::RunStep] Kernel launch failed"));
    unpack_record(h->out_host.ptr, 21, 6, JtJ, Jtr, residual, inliers);
    return DFK_OK;
  });
}

// N tracking problems of L levels each (levels[n L + l]), advanced in lockstep: one launch per iteration for all of
// them.  One problem (dfk_se3_track) may record its per-iteration history; a batch's messages name the problem.
static DfkStatus track(DfkHandle h, const std::string& what, bool batch, int N, int L, float* poses_ck,
                       const DfkTrackLevel* levels, float* inlier_fraction, float* error, float* last_systems,
                       float* history, int history_capacity)
{
  std::vector<Se3TrackDesc> descs((size_t)L * N);  // level-major: a launch reads the N descriptors of its level
  std::vector<int> level_blocks(L, 0);             // grid width of a level: its largest problem
  int stride = 1;                                  // partial rows per problem
  for (int n = 0; n < N; ++n) {
    for (int l = 0; l < L; ++l) {
      const DfkTrackLevel& T = levels[(size_t)n * L + l];
      if (!track_level_ok(T))
        return fail(h, DFK_ERR_INVALID_ARG,
                    what + "inconsistent image views / camera larger than them / negative iteration count at " +
                        (batch ? "problem " + std::to_string(n) + " level " : "level ") + std::to_string(l));
      if (T.iterations != levels[l].iterations)
        return fail(h, DFK_ERR_INVALID_ARG,
                    what + "problem " + std::to_string(n) + " has " + std::to_string(T.iterations) +
                        " iterations at level " + std::to_string(l) + ", problem 0 has " +
                        std::to_string(levels[l].iterations));
      Se3TrackDesc& d = descs[(size_t)l * N + n];
      set_se3_desc(d, poses_ck + 7 * (size_t)n, T.cam, T.img0, T.img1, T.dpt0, T.grad1);  // q/t: the device pose's
      level_blocks[l] = std::max(level_blocks[l], d.nblocks);
      stride = std::max(stride, d.nblocks);
    }
  }
  int total_iters = 0;
  for (int l = 0; l < L; ++l) total_iters += levels[l].iterations;
  if (history && history_capacity < total_iters) return fail(h, DFK_ERR_INVALID_ARG, what + "history buffer too small");
  DeviceGuard guard(h->device);
  Layout B;
  const size_t ndesc = N > 1 ? descs.size() : 0;  // a single problem passes its descriptor with the launch instead
  const Part<Se3TrackDesc> descs_at = B.add<Se3TrackDesc>(ndesc);
  const Part<float> poses_at = B.add<float>(8 * (size_t)N), outs_at = B.add<float>(32 * (size_t)N);
  const Part<float> history_at = B.add<float>(history ? 36 * (size_t)total_iters : 0);
  DFK_CUDA(h, h->batch_dev.ensure(B.bytes), (what + "scratch allocation failed").c_str());
  DFK_CUDA(h, h->batch_partials.ensure((size_t)N * stride * 32), (what + "scratch allocation failed").c_str());
  DFK_TRY(ensure_tickets(h, h->batch_counters, (size_t)N, (what + "scratch allocation failed").c_str(),
                         (what + "memset failed").c_str()));
  DFK_CUDA(h, h->batch_host.ensure(B.bytes), (what + "pinned allocation failed").c_str());
  // one upload: every level's descriptors and the start poses
  memcpy(descs_at.at(h->batch_host.ptr), descs.data(), ndesc * sizeof(Se3TrackDesc));
  float* host_poses = poses_at.at(h->batch_host.ptr);
  for (int n = 0; n < N; ++n) {
    memcpy(host_poses + 8 * (size_t)n, poses_ck + 7 * (size_t)n, sizeof(float) * 7);
    host_poses[8 * (size_t)n + 7] = 0.0f;
  }
  DFK_CUDA(h, cudaMemcpyAsync(h->batch_dev.ptr, h->batch_host.ptr, outs_at.off, cudaMemcpyHostToDevice, h->stream),
           (what + (batch ? "upload failed" : "pose upload failed")).c_str());
  float* poses_dev = poses_at.at(h->batch_dev.ptr);
  float* outs_dev = outs_at.at(h->batch_dev.ptr);
  DFK_CUDA(h, cudaMemsetAsync(outs_dev, 0, history_at.off - outs_at.off, h->stream), (what + "memset failed").c_str());
  int it = 0;
  for (int l = L - 1; l >= 0; --l) {  // coarse to fine (camera_tracker.cpp:48)
    for (int k = 0; k < levels[l].iterations; ++k, ++it) {
      DFK_CUDA(h,
               N == 1 ? launch_se3_step(descs[l], h->se3_huber_delta, h->batch_partials.ptr, h->batch_counters.ptr,
                                        outs_dev, poses_dev,
                                        history ? history_at.at(h->batch_dev.ptr) + 36 * (size_t)it : nullptr, h->stream)
                      : launch_se3_step(descs_at.at(h->batch_dev.ptr) + (size_t)l * N, N, level_blocks[l],
                                        h->se3_huber_delta, h->batch_partials.ptr, stride, h->batch_counters.ptr,
                                        outs_dev, poses_dev, h->stream),
               (what + "kernel launch failed").c_str());
      h->launches += 1;
    }
  }
  // one read-back: final poses, last evaluated systems and the history
  DFK_TRY(download(h, host_poses, poses_dev, B.bytes - poses_at.off, (what + "read-back failed").c_str(),
                   (what + "stream synchronize failed").c_str()));
  const float* host_outs = outs_at.at(h->batch_host.ptr);
  for (int n = 0; n < N; ++n) {
    memcpy(poses_ck + 7 * (size_t)n, host_poses + 8 * (size_t)n, sizeof(float) * 7);
    track_outputs(host_outs + 32 * (size_t)n, levels[(size_t)n * L], inlier_fraction ? inlier_fraction + n : nullptr,
                  error ? error + n : nullptr, last_systems ? last_systems + 29 * (size_t)n : nullptr);
  }
  if (history) memcpy(history, history_at.at(h->batch_host.ptr), sizeof(float) * 36 * (size_t)total_iters);
  return DFK_OK;
}

DfkStatus dfk_se3_track(DfkHandle h, float pose_ck[7], const DfkTrackLevel* levels, int num_levels,
                        float* inlier_fraction, float* error, float* last_system, float* history, int history_capacity)
{
  return guarded(h, [&] {
    if (!pose_ck || !levels || num_levels <= 0)
      return fail(h, DFK_ERR_INVALID_ARG, "[CameraTracker::TrackFrame] null argument / no pyramid levels");
    return track(h, "[CameraTracker::TrackFrame] ", false, 1, num_levels, pose_ck, levels, inlier_fraction, error,
                 last_system, history, history_capacity);
  });
}

DfkStatus dfk_se3_track_batch(DfkHandle h, int num_problems, int num_levels, float* poses_ck,
                              const DfkTrackLevel* levels, float* inlier_fraction, float* error, float* last_systems)
{
  return guarded(h, [&] {
    if (!poses_ck || !levels || num_levels <= 0)
      return fail(h, DFK_ERR_INVALID_ARG, "[CameraTracker::TrackFrame batch] null argument / no pyramid levels");
    if (num_problems < 1 || num_problems > 65535)  // blockIdx.y of the step kernel is the problem
      return fail(h, DFK_ERR_INVALID_ARG, "[CameraTracker::TrackFrame batch] number of problems must be in [1, 65535]");
    return track(h, "[CameraTracker::TrackFrame batch] ", true, num_problems, num_levels, poses_ck, levels,
                 inlier_fraction, error, last_systems, nullptr, 0);
  });
}

DfkStatus dfk_se3_warp(DfkHandle h, const float se3[7], const DfkCamera* cam, const DfkImage* img0,
                       const DfkImage* img1, const DfkImage* dpt0, const DfkImage* img2, float* residual,
                       uint64_t* inliers)
{
  return guarded(h, [&] {
    if (!se3 || !cam || !img0 || !img1 || !dpt0 || !img2 || !residual || !inliers)
      return fail(h, DFK_ERR_INVALID_ARG, "[SE3Aligner::Warp] null argument");
    const uint32_t W = img0->width, H = img0->height;
    if (W == 0 || H == 0 || !img_ok(img0, W, H, 1) || !img_ok(img1, W, H, 1) || !img_ok(dpt0, W, H, 1) ||
        !img_ok(img2, W, H, 1))
      return fail(h, DFK_ERR_INVALID_ARG, "[SE3Aligner::Warp] inconsistent image views");
    if (!cam_ok(cam, W, H)) return fail(h, DFK_ERR_INVALID_ARG, "[SE3Aligner::Warp] camera viewport larger than the image views");
    DeviceGuard guard(h->device);
    // depth <= 0 -> skip ; PixelValid(pix1, 1) (cu_se3aligner.cpp:89-97)
    const PixelCam pc = make_pixel_cam(se3, cam, 1, 0.0f);
    DFK_CUDA(h, launch_warp(pc, (int)W, (int)H, view_of(img0), view_of(img1), view_of(dpt0), (float*)img2->ptr,
                            (uint32_t)(img2->pitch_bytes / 4), h->simple_scratch.ptr, h->counter.ptr, h->out_dev.ptr,
                            h->stream),
             "[SE3Aligner::Warp] Kernel launch failed (kernel_warp_calculate)");
    DFK_TRY(fetch_out(h, 2, "[SE3Aligner::Warp] Kernel launch failed (kernel_finalize_reduction)"));
    unpack_record(h->out_host.ptr, 0, 0, nullptr, nullptr, residual, inliers);
    return DFK_OK;
  });
}

DfkStatus dfk_update_depth(DfkHandle h, const float* code, int code_size, const DfkImage* prx_orig,
                           const DfkImage* prx_jac, float avg_dpt, const DfkImage* dpt_out)
{
  return guarded(h, [&] {
    if (!code || !prx_orig || !prx_jac || !dpt_out) return fail(h, DFK_ERR_INVALID_ARG, "[UpdateDepth] null argument");
    if (code_size < 1 || code_size > 256) return fail(h, DFK_ERR_UNSUPPORTED, "[UpdateDepth] code size out of range");
    const uint32_t W = dpt_out->width, H = dpt_out->height;
    if (W == 0 || H == 0 || !img_ok(prx_orig, W, H, 1) || !img_ok(prx_jac, W, H, code_size) || !img_ok(dpt_out, W, H, 1))
      return fail(h, DFK_ERR_INVALID_ARG, "[UpdateDepth] inconsistent image views");
    DeviceGuard guard(h->device);
    DFK_CUDA(h, cudaMemcpyAsync(h->code_dev.ptr, code, sizeof(float) * code_size, cudaMemcpyHostToDevice, h->stream),
             "[UpdateDepth] code upload failed");
    DepthDecodeDesc d;
    int max_blocks = 1;
    set_depth_decode_desc(d, DfkDepthDecodeItem{*prx_orig, *prx_jac, *dpt_out, code}, code_size, h->code_dev.ptr,
                          static_cast<float*>(dpt_out->ptr), (uint32_t)(dpt_out->pitch_bytes / 4), &max_blocks);
    DFK_CUDA(h, launch_update_depth(code_size, d, avg_dpt, h->stream), "[UpdateDepth] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_update_depth_batch(DfkHandle h, const DfkDepthDecodeItem* items, int n, int code_size)
{
  return guarded(h, [&] {
    if (!items || n < 1 || n > 65535)  // blockIdx.y of the kernel is the item
      return fail(h, DFK_ERR_INVALID_ARG, "[UpdateDepth batch] null argument / number of items not in [1, 65535]");
    if (code_size < 1 || code_size > 256) return fail(h, DFK_ERR_UNSUPPORTED, "[UpdateDepth batch] code size out of range");
    for (int i = 0; i < n; ++i) {
      const DfkDepthDecodeItem& it = items[i];
      const uint32_t W = it.dpt.width, H = it.dpt.height;
      if (!it.code || W == 0 || H == 0 || !img_ok(&it.prx_orig, W, H, 1) || !img_ok(&it.prx_jac, W, H, code_size) ||
          !img_ok(&it.dpt, W, H, 1))
        return fail(h, DFK_ERR_INVALID_ARG,
                    "[UpdateDepth batch] null code or inconsistent image views in item " + std::to_string(i));
    }
    DeviceGuard guard(h->device);
    Staging s(h->staging);
    const Part<DepthDecodeDesc> descs = s.add<DepthDecodeDesc>(n);
    const Part<float> codes = s.add<float>((size_t)n * code_size);
    DFK_TRY(s.grow(h, h->depth_dev, "[UpdateDepth batch] "));
    int max_blocks = 1;
    for (int i = 0; i < n; ++i) {
      const DfkDepthDecodeItem& it = items[i];
      set_depth_decode_desc(descs.at(s.host())[i], it, code_size, codes.at(s.dev) + (size_t)i * code_size,
                            static_cast<float*>(it.dpt.ptr), (uint32_t)(it.dpt.pitch_bytes / 4), &max_blocks);
      memcpy(codes.at(s.host()) + (size_t)i * code_size, it.code, sizeof(float) * code_size);
    }
    DFK_TRY(s.upload(h, h->depth_dev, "[UpdateDepth batch] "));
    DFK_CUDA(h, launch_update_depth(code_size, descs.at(s.dev), n, max_blocks, h->params.sfmparams.avg_dpt, h->stream),
             "[UpdateDepth batch] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_sobel_gradients(DfkHandle h, const DfkImage* img, const DfkImage* grad)
{
  return guarded(h, [&] {
    if (!img || !grad) return fail(h, DFK_ERR_INVALID_ARG, "[SobelGradients] null argument");
    const uint32_t W = img->width, H = img->height;
    if (W == 0 || H == 0 || !img_ok(img, W, H, 1) || !img_ok(grad, W, H, 2))
      return fail(h, DFK_ERR_INVALID_ARG, "[SobelGradients] inconsistent image views");
    DeviceGuard guard(h->device);
    DFK_CUDA(h, launch_sobel(pyr_level(img, grad), h->stream),
             "Kernel launch failed (kernel_sobel_gradients)");
    h->launches += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_gaussian_blur_down(DfkHandle h, const DfkImage* in, const DfkImage* out)
{
  return guarded(h, [&] {
    if (!in || !out) return fail(h, DFK_ERR_INVALID_ARG, "[GaussianBlurDown] null argument");
    if (in->width == 0 || in->height == 0 || out->width == 0 || out->height == 0 ||
        !img_ok(in, in->width, in->height, 1) || !img_ok(out, out->width, out->height, 1))
      return fail(h, DFK_ERR_INVALID_ARG, "[GaussianBlurDown] inconsistent image views");
    DeviceGuard guard(h->device);
    DFK_CUDA(h, launch_blur_down(pyr_level(in, nullptr), pyr_level(out, nullptr), h->stream),
             "Kernel launch failed (kernel_gaussian_blur_down)");
    h->launches += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_build_image_pyramid(DfkHandle h, const DfkImage* imgs, const DfkImage* grads, int levels)
{
  return guarded(h, [&] {
    if (!imgs || levels <= 0) return fail(h, DFK_ERR_INVALID_ARG, "[BuildImagePyramid] null argument / no levels");
    for (int l = 1; l < levels; ++l) DFK_TRY(dfk_gaussian_blur_down(h, &imgs[l - 1], &imgs[l]));
    if (grads)
      for (int l = 0; l < levels; ++l) DFK_TRY(dfk_sobel_gradients(h, &imgs[l], &grads[l]));
    return DFK_OK;
  });
}

DfkStatus dfk_squared_error(DfkHandle h, const DfkImage* a, const DfkImage* b, float* out)
{
  return guarded(h, [&] {
    if (!a || !b || !out) return fail(h, DFK_ERR_INVALID_ARG, "[SquaredError] null argument");
    const uint32_t W = a->width, H = a->height;
    if (W == 0 || H == 0 || !img_ok(a, W, H, 1) || !img_ok(b, W, H, 1))
      return fail(h, DFK_ERR_INVALID_ARG, "[SquaredError] inconsistent image views");
    DeviceGuard guard(h->device);
    DFK_CUDA(h, launch_squared_error((int)W, (int)H, view_of(a), view_of(b), h->simple_scratch.ptr, h->counter.ptr,
                                     h->out_dev.ptr, h->stream),
             "[SquaredError] kernel launch failed");
    DFK_TRY(fetch_out(h, 1, "[SquaredError] kernel launch failed"));
    *out = h->out_host.ptr[0];
    return DFK_OK;
  });
}

static bool pp_cam_ok(const DfkCamera& c)
{
  return std::isfinite(c.fx) && std::isfinite(c.fy) && std::isfinite(c.u0) && std::isfinite(c.v0) && c.fx != 0.0f &&
         c.fy != 0.0f;
}

// a uint8 view of w x h pixels with `channels` bytes each
static bool pp_u8_ok(const DfkImage& im, uint32_t w, uint32_t h, uint32_t channels)
{
  return im.ptr && im.width == w && im.height == h && im.pitch_bytes >= (size_t)w * channels;
}

DfkStatus dfk_preprocess_batch(DfkHandle h, const DfkPreprocessItem* items, int n, int num_levels, double* stats_dev)
{
  return guarded(h, [&] {
    const std::string w = "[PreprocessImage batch] ";
    if (!items || n < 1 || n > 65535)  // gridDim.y / gridDim.z of the kernels is the item
      return fail(h, DFK_ERR_INVALID_ARG, w + "null argument / number of items not in [1, 65535]");
    if (num_levels < 0 || num_levels > DFK_PREPROCESS_MAX_LEVELS)
      return fail(h, DFK_ERR_INVALID_ARG, w + "number of levels not in [0, DFK_PREPROCESS_MAX_LEVELS]");
    if ((uintptr_t)stats_dev & 7) return fail(h, DFK_ERR_INVALID_ARG, w + "stats_dev must be 8-byte aligned");
    const int L = num_levels;
    // [item descriptors n | level descriptors L x n (level-major)]
    Staging up(h->staging);
    const Part<PpItemDev> pp_at = up.add<PpItemDev>(n);
    const Part<PyrLevelDev> lv_at = up.add<PyrLevelDev>((size_t)L * n);
    std::vector<int> max_w((size_t)L, 0), max_h((size_t)L, 0);
    long long partials = 0;
    int max_tiles = 0;
    bool any_norm = false, any_grad = false;
    for (int i = 0; i < n; ++i) {
      const DfkPreprocessItem& it = items[i];
      const std::string at = " in item " + std::to_string(i);
      const DfkImage& s = it.src;
      if (!s.ptr || s.width < 1 || s.height < 1 || s.width > DFK_ORB_MAX_SIDE || s.height > DFK_ORB_MAX_SIDE ||
          s.pitch_bytes < 3 * (size_t)s.width)
        return fail(h, DFK_ERR_INVALID_ARG, w + "source needs a pointer, width and height in [1, DFK_ORB_MAX_SIDE] and "
                                                "pitch_bytes >= 3 width" + at);
      if (!pp_cam_ok(it.src_cam) || !pp_cam_ok(it.out_cam))
        return fail(h, DFK_ERR_INVALID_ARG, w + "camera intrinsics must be finite, with fx and fy != 0" + at);
      const float cw = it.out_cam.width, ch = it.out_cam.height;
      if (!(cw >= 1.0f && ch >= 1.0f && cw <= (float)DFK_ORB_MAX_SIDE && ch <= (float)DFK_ORB_MAX_SIDE) ||
          cw != std::floor(cw) || ch != std::floor(ch))
        return fail(h, DFK_ERR_INVALID_ARG, w + "output camera size must be whole numbers in [1, DFK_ORB_MAX_SIDE]" + at);
      const uint32_t W = (uint32_t)cw, H = (uint32_t)ch;
      if (it.color.ptr && !pp_u8_ok(it.color, W, H, 3))
        return fail(h, DFK_ERR_INVALID_ARG, w + "color view is not W_o x H_o with pitch_bytes >= 3 W_o" + at);
      if (it.gray.ptr && !pp_u8_ok(it.gray, W, H, 1))
        return fail(h, DFK_ERR_INVALID_ARG, w + "gray view is not W_o x H_o with pitch_bytes >= W_o" + at);
      if (it.normalize != 0 && it.normalize != 1) return fail(h, DFK_ERR_INVALID_ARG, w + "normalize not 0 or 1" + at);
      if (L > 0 && !it.levels) return fail(h, DFK_ERR_INVALID_ARG, w + "null levels" + at);
      uint32_t lw = W, lh = H;
      for (int l = 0; l < L; ++l) {
        if (l > 0) {
          lw /= 2;
          lh /= 2;
        }
        const std::string atl = " at level " + std::to_string(l) + at;
        if (lw < 1 || lh < 1) return fail(h, DFK_ERR_INVALID_ARG, w + "level smaller than 1 x 1" + atl);
        if (!img_ok(&it.levels[l], lw, lh, 1))
          return fail(h, DFK_ERR_INVALID_ARG, w + "level view is not the halved size or not a float view" + atl);
        if (it.grads && !img_ok(&it.grads[l], lw, lh, 2))
          return fail(h, DFK_ERR_INVALID_ARG, w + "gradient view does not match its level" + atl);
        lv_at.at(up.host())[(size_t)l * n + i] = pyr_level(&it.levels[l], it.grads ? &it.grads[l] : nullptr);
        max_w[l] = std::max(max_w[l], (int)lw);
        max_h[l] = std::max(max_h[l], (int)lh);
      }
      any_grad = any_grad || (L > 0 && it.grads);
      PpItemDev& d = pp_at.at(up.host())[i];
      dfk_pm_map_init(&d.map, it.src_cam.fx, it.src_cam.fy, it.src_cam.u0, it.src_cam.v0, it.out_cam.fx,
                      it.out_cam.fy, it.out_cam.u0, it.out_cam.v0);
      d.src = static_cast<const uint8_t*>(s.ptr);
      d.src_pitch = s.pitch_bytes;
      d.sw = (int)s.width;
      d.sh = (int)s.height;
      d.w = (int)W;
      d.h = (int)H;
      d.tiles_x = (int)((W + DFK_PM_TILE_W - 1) / DFK_PM_TILE_W);
      d.tiles = d.tiles_x * (int)((H + DFK_PM_TILE_H - 1) / DFK_PM_TILE_H);
      d.color = static_cast<uint8_t*>(it.color.ptr);
      d.color_pitch = it.color.pitch_bytes;
      d.gray = static_cast<uint8_t*>(it.gray.ptr);
      d.gray_pitch = it.gray.pitch_bytes;
      d.level0 = L > 0 ? static_cast<float*>(it.levels[0].ptr) : nullptr;
      d.level0_pitch = L > 0 ? (uint32_t)(it.levels[0].pitch_bytes / 4) : 0u;
      d.normalize = it.normalize;
      d.partial_begin = (int)std::min(partials, (long long)INT32_MAX);
      d.stats = (it.normalize && stats_dev) ? stats_dev + 2 * (size_t)i : nullptr;
      if (it.normalize) partials += d.tiles;
      any_norm = any_norm || it.normalize;
      max_tiles = std::max(max_tiles, d.tiles);
    }
    if (partials > INT32_MAX)
      return fail(h, DFK_ERR_INVALID_ARG, w + "more than 2^31 - 1 tiles of normalising items in one call");
    DeviceGuard guard(h->device);
    // [tile partials 2 each | moments 2 per item]
    DFK_CUDA(h, h->pp_partials.ensure(2 * (size_t)partials + 2 * (size_t)n),
             "[PreprocessImage batch] scratch allocation failed");
    for (int i = 0; i < n; ++i) pp_at.at(up.host())[i].moments = h->pp_partials.ptr + 2 * ((size_t)partials + i);
    DFK_TRY(up.upload(h, h->pp_dev, w));
    const PyrLevelDev* lv_dev = lv_at.at(up.dev);
    DFK_CUDA(h, launch_preprocess(pp_at.at(up.dev), n, max_tiles, any_norm, h->pp_partials.ptr, h->stream),
             "[PreprocessImage batch] kernel launch failed");
    h->launches += any_norm ? 3 : 1;
    for (int l = 1; l < L; ++l) {
      DFK_CUDA(h, launch_blur_down(lv_dev + (size_t)(l - 1) * n, lv_dev + (size_t)l * n, n, max_w[l], max_h[l],
                                         h->stream),
               "Kernel launch failed (kernel_gaussian_blur_down)");
      h->launches += 1;
    }
    if (any_grad) {
      for (int l = 0; l < L; ++l) {
        DFK_CUDA(h, launch_sobel(lv_dev + (size_t)l * n, n, max_w[l], max_h[l], h->stream),
                 "Kernel launch failed (kernel_sobel_gradients)");
        h->launches += 1;
      }
    }
    return DFK_OK;
  });
}

// the checks of one keyframe of dfk_keyframe_mesh_batch; the failure text (naming the field), or null
static const char* mesh_item_error(const DfkKeyframeMeshItem& it, int code_size, bool colors, DfkStatus* status)
{
  *status = DFK_ERR_INVALID_ARG;
  const float cw = it.cam.width, ch = it.cam.height;
  if (!pp_cam_ok(it.cam)) return "cam: intrinsics must be finite, with fx and fy != 0";
  if (!(cw >= 1.0f && ch >= 1.0f && cw <= (float)DFK_ORB_MAX_SIDE && ch <= (float)DFK_ORB_MAX_SIDE) ||
      cw != std::floor(cw) || ch != std::floor(ch))
    return "cam: width and height must be whole numbers in [1, DFK_ORB_MAX_SIDE]";
  const uint32_t W = (uint32_t)cw, H = (uint32_t)ch;
  if (it.dpt.ptr) {
    if (it.prx_orig.ptr || it.prx_jac.ptr || it.code) return "dpt: set either dpt or (prx_orig, prx_jac, code), not both";
    if (!img_ok(&it.dpt, W, H, 1)) return "dpt: not a W x H float view";
  } else {
    if (!it.code) return "dpt: no dpt and no code to decode";
    if (code_size < 1 || code_size > 256) {
      *status = DFK_ERR_UNSUPPORTED;
      return "code_size: out of range for a decode";
    }
    if (!img_ok(&it.prx_orig, W, H, 1)) return "prx_orig: not a W x H float view";
    if (!img_ok(&it.prx_jac, W, H, (uint32_t)code_size)) return "prx_jac: not a W x H view of code_size floats";
  }
  if (it.std.ptr && !img_ok(&it.std, W, H, 1)) return "std: not a W x H float view";
  if (it.valid.ptr && !img_ok(&it.valid, W, H, 1)) return "valid: not a W x H float view";
  if (it.color.ptr && !pp_u8_ok(it.color, W, H, 3)) return "color: not W x H with pitch_bytes >= 3 W";
  if (colors && !it.color.ptr) return "color: colors_dev is given but the item has no color view";
  const DfkImage& u = it.depth_u16;
  if (u.ptr && (u.width != W || u.height != H || (u.pitch_bytes & 1) || u.pitch_bytes < 2 * (size_t)W))
    return "depth_u16: not W x H with an even pitch_bytes >= 2 W";
  for (int k = 0; k < 7; ++k)
    if (!std::isfinite(it.pose_wk[k])) return "pose_wk: not finite";
  if (it.vertex_capacity < 0 || it.triangle_capacity < 0) return "capacity: negative";
  return nullptr;
}

DfkStatus dfk_keyframe_mesh_batch(DfkHandle h, const DfkKeyframeMeshItem* items, int n, int code_size,
                                  const DfkKeyframeMeshParams* params, float* positions_dev, float* normals_dev,
                                  uint8_t* colors_dev, int32_t* pixels_dev, int32_t* triangles_dev, int32_t* counts_dev)
{
  return guarded(h, [&] {
    const std::string w = "[KeyframeMesh batch] ";
    if (!items || !params || n < 1 || n > 65535)  // gridDim.y of the tile kernels is the item
      return fail(h, DFK_ERR_INVALID_ARG, w + "null argument / number of items not in [1, 65535]");
    if (!positions_dev || !counts_dev) return fail(h, DFK_ERR_INVALID_ARG, w + "null positions or counts output");
    if (((uintptr_t)positions_dev & 3) || ((uintptr_t)normals_dev & 3) || ((uintptr_t)pixels_dev & 3) ||
        ((uintptr_t)triangles_dev & 3) || ((uintptr_t)counts_dev & 3))
      return fail(h, DFK_ERR_INVALID_ARG, w + "float and int32 outputs must be 4-byte aligned");
    const DfkKeyframeMeshParams& prm = *params;
    if (!std::isfinite(prm.stdev_thresh) || !std::isfinite(prm.slt_thresh))
      return fail(h, DFK_ERR_INVALID_ARG, w + "params: stdev_thresh and slt_thresh must be finite");
    if (prm.crop_pix < 0) return fail(h, DFK_ERR_INVALID_ARG, w + "params: crop_pix < 0");
    if (prm.draw_noisy_pixels != 0 && prm.draw_noisy_pixels != 1)
      return fail(h, DFK_ERR_INVALID_ARG, w + "params: draw_noisy_pixels not 0 or 1");
    // sizes: segments and decoded pixels before each item, output rows
    std::vector<long long> seg_at((size_t)n), dec_at((size_t)n);
    long long segs = 0, dec_px = 0, vrows = 0, trows = 0;
    int decodes = 0, max_tiles = 1;
    for (int i = 0; i < n; ++i) {
      const DfkKeyframeMeshItem& it = items[i];
      DfkStatus st;
      if (const char* e = mesh_item_error(it, code_size, colors_dev != nullptr, &st))
        return fail(h, st, w + "item " + std::to_string(i) + ": " + e);
      const long long W = (long long)it.cam.width, H = (long long)it.cam.height;
      const long long tx = (W + kMeshTileW - 1) / kMeshTileW, ty = (H + kMeshTileH - 1) / kMeshTileH;
      seg_at[(size_t)i] = segs;
      dec_at[(size_t)i] = dec_px;
      segs += H * tx;
      if (!it.dpt.ptr) {
        dec_px += (W * H + 3) & ~3LL;  // 16-byte aligned depths
        decodes += 1;
      }
      vrows += it.vertex_capacity;
      trows += it.triangle_capacity;
      max_tiles = std::max(max_tiles, (int)(tx * ty));
    }
    if (vrows > INT32_MAX || trows > INT32_MAX)
      return fail(h, DFK_ERR_INVALID_ARG, w + "capacity: more than 2^31 - 1 vertex or triangle rows in one call");
    DeviceGuard guard(h->device);
    // scratch [segment masks | segment bases | decoded depths]
    Layout S;
    const Part<uint3> masks_at = S.add<uint3>((size_t)segs);
    const Part<int2> bases_at = S.add<int2>((size_t)segs);
    const Part<float> decoded_at = S.add<float>((size_t)dec_px);
    DFK_CUDA(h, h->mesh_scratch.ensure(S.bytes), "[KeyframeMesh batch] scratch allocation failed");
    // descriptors [items | decode descriptors | codes], one upload
    Staging s(h->staging);
    const Part<MeshItemDev> items_at = s.add<MeshItemDev>(n);
    const Part<DepthDecodeDesc> descs_at = s.add<DepthDecodeDesc>(decodes);
    const Part<float> codes_at = s.add<float>((size_t)decodes * (size_t)std::max(code_size, 0));
    DFK_TRY(s.grow(h, h->mesh_dev, w));
    int dec = 0, max_blocks = 1;
    long long v_begin = 0, t_begin = 0;
    for (int i = 0; i < n; ++i) {
      const DfkKeyframeMeshItem& it = items[i];
      MeshItemDev& d = items_at.at(s.host())[i];
      d.w = (int)it.cam.width;
      d.h = (int)it.cam.height;
      if (it.dpt.ptr) {
        d.dpt = view_of(&it.dpt);
      } else {
        float* out = decoded_at.at(h->mesh_scratch.ptr) + dec_at[(size_t)i];
        DfkDepthDecodeItem di{it.prx_orig, it.prx_jac, DfkImage{out, sizeof(float) * (size_t)d.w, (uint32_t)d.w,
                                                                 (uint32_t)d.h}, it.code};
        set_depth_decode_desc(descs_at.at(s.host())[dec], di, code_size, codes_at.at(s.dev) + (size_t)dec * code_size,
                              out, (uint32_t)d.w, &max_blocks);
        memcpy(codes_at.at(s.host()) + (size_t)dec * code_size, it.code, sizeof(float) * code_size);
        dec += 1;
        d.dpt = View{out, (uint32_t)d.w};
      }
      d.std = it.std.ptr ? view_of(&it.std) : View{nullptr, 0};
      d.vld = it.valid.ptr ? view_of(&it.valid) : View{nullptr, 0};
      d.color = static_cast<const uint8_t*>(it.color.ptr);
      d.color_pitch = it.color.pitch_bytes;
      d.depth_u16 = static_cast<uint16_t*>(it.depth_u16.ptr);
      d.u16_pitch = it.depth_u16.pitch_bytes;
      d.fx = it.cam.fx; d.fy = it.cam.fy; d.u0 = it.cam.u0; d.v0 = it.cam.v0;
      for (int k = 0; k < 4; ++k) d.q[k] = it.pose_wk[k];
      for (int k = 0; k < 3; ++k) d.t[k] = it.pose_wk[4 + k];
      d.tiles_x = (d.w + kMeshTileW - 1) / kMeshTileW;
      d.tiles = d.tiles_x * ((d.h + kMeshTileH - 1) / kMeshTileH);
      d.seg_begin = seg_at[(size_t)i];
      d.v_begin = v_begin;
      d.t_begin = t_begin;
      d.v_cap = it.vertex_capacity;
      d.t_cap = it.triangle_capacity;
      v_begin += it.vertex_capacity;
      t_begin += it.triangle_capacity;
    }
    DFK_TRY(s.upload(h, h->mesh_dev, w));
    if (decodes > 0) {
      DFK_CUDA(h, launch_update_depth(code_size, descs_at.at(s.dev), decodes, max_blocks,
                                            h->params.sfmparams.avg_dpt, h->stream),
               "[KeyframeMesh batch] depth decode launch failed");
      h->launches += 1;
    }
    MeshParamsDev p;
    p.tau = prm.stdev_thresh > 0.0f ? std::log((double)prm.stdev_thresh / std::sqrt(2.0)) : -INFINITY;
    p.slt = prm.slt_thresh;
    p.crop = prm.crop_pix;
    p.draw_noisy = prm.draw_noisy_pixels;
    const MeshOutDev o{positions_dev, normals_dev, colors_dev, pixels_dev, triangles_dev, counts_dev};
    DFK_CUDA(h, launch_keyframe_mesh(items_at.at(s.dev), n, max_tiles, p, o, masks_at.at(h->mesh_scratch.ptr),
                                     bases_at.at(h->mesh_scratch.ptr), h->stream),
             "[KeyframeMesh batch] kernel launch failed");
    h->launches += 3;
    return DFK_OK;
  });
}

// ---------------------------------------------------------------------------------------------- streaming from host
DfkStatus dfk_sfm_stream_create(DfkHandle h, int code_size, int max_items, size_t max_bytes, int depth, DfkSfmStream** out)
{
  return guarded(h, [&] {
    if (!out || max_items <= 0 || max_bytes == 0 || depth < 1 || depth > 16)
      return fail(h, DFK_ERR_INVALID_ARG, "[SfmStream] bad argument (1 <= depth <= 16, max_items > 0, max_bytes > 0)");
    *out = nullptr;
    if (!dfk_sfm_supports_code_size(code_size))
      return fail(h, DFK_ERR_UNSUPPORTED, "[SfmStream] no RunStep kernel for code size " + std::to_string(code_size));
    DeviceGuard guard(h->device);
    DfkSfmStream* s = new (std::nothrow) DfkSfmStream();
    if (!s) return oom(h);
    s->device = h->device; s->code_size = code_size; s->max_items = max_items; s->depth = depth;
    // initial slot size (a hint): staged images are padded to a 256-byte row pitch and offset, scratch images (valid0,
    // decoded depth) ride along; a submission that needs more grows its slot
    s->max_bytes = max_bytes + max_bytes / 4 + (size_t)max_items * 8 * 4096;
    s->slots.resize(depth);
    s->dev_items.resize(max_items);
    const size_t rec = (size_t)DFK_SFM_RECORD_FLOATS(code_size) * max_items;
    cudaError_t e = cudaStreamCreateWithFlags(&s->copy_stream, cudaStreamNonBlocking);
    for (int k = 0; k < depth && e == cudaSuccess; ++k) {
      DfkSfmStream::Slot& sl = s->slots[k];
      e = sl.dev.ensure(s->max_bytes);
      if (e == cudaSuccess) e = sl.rec_dev.ensure(rec);
      if (e == cudaSuccess) e = sl.rec_host.ensure(rec);
      if (e == cudaSuccess) e = cudaEventCreateWithFlags(&sl.uploaded, cudaEventDisableTiming);
      if (e == cudaSuccess) e = cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming);
    }
    if (e != cudaSuccess) {
      dfk_sfm_stream_destroy(h, s);
      return cuda_fail(h, e, "[SfmStream] allocation failed");
    }
    *out = s;
    return DFK_OK;
  });
}

DfkStatus dfk_sfm_stream_destroy(DfkHandle /*h*/, DfkSfmStream* s)
{
  if (!s) return DFK_OK;
  DeviceGuard guard(s->device);
  if (s->copy_stream) cudaStreamSynchronize(s->copy_stream);
  for (auto& sl : s->slots) {
    if (sl.done) { cudaEventSynchronize(sl.done); cudaEventDestroy(sl.done); }
    if (sl.uploaded) cudaEventDestroy(sl.uploaded);
  }
  if (s->copy_stream) cudaStreamDestroy(s->copy_stream);
  delete s;
  return DFK_OK;
}

DfkStatus dfk_sfm_stream_submit(DfkHandle h, DfkSfmStream* s, const DfkSfmWorkItem* items, int n, uint64_t* ticket)
{
  return guarded(h, [&] {
    if (!s || !items || !ticket || n <= 0) return fail(h, DFK_ERR_INVALID_ARG, "[SfmStream] null argument / empty submission");
    if (n > s->max_items) return fail(h, DFK_ERR_INVALID_ARG, "[SfmStream] more work items than the stream was created for");
    if (s->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[SfmStream] stream and handle live on different devices");
    DfkSfmStream::Slot& sl = s->slots[s->next_ticket % (uint64_t)s->depth];
    if (sl.busy)
      return fail(h, DFK_ERR_INVALID_ARG,
                  "[SfmStream] " + std::to_string(s->depth) + " submissions outstanding: wait for ticket " +
                      std::to_string(sl.ticket) + " first");
    DeviceGuard guard(h->device);
    cudaError_t err = cudaSuccess;
    // one image: host view -> 256-byte aligned, 256-byte pitched device view inside the slot.  upload == false: device
    // scratch.  Two passes over the items: sizes first (the slot grows if it has to), then the copies.
    for (int pass = 0; pass < 2; ++pass) {
      size_t cursor = 0;
      auto stage = [&](const DfkImage& src, uint32_t floats_per_px, bool upload) -> DfkImage {
        DfkImage d{};
        const size_t row = (size_t)src.width * floats_per_px * sizeof(float);
        // rows that are already 16-byte multiples stay dense on the device (what the bulk-copy loaders of the kernels
        // need), so a dense host image travels as ONE linear copy: per-row DMA descriptors cost ~30 % of the PCIe rate on
        // the small pyramid levels; odd widths get a 256-byte pitch and a 2-D copy
        const size_t pitch = (row % 16 == 0) ? row : ((row + 255) & ~(size_t)255);
        cursor = (cursor + 255) & ~(size_t)255;
        d.ptr = sl.dev.ptr + cursor;
        d.pitch_bytes = pitch;
        d.width = src.width;
        d.height = src.height;
        cursor += pitch * src.height;
        if (pass == 1 && upload && err == cudaSuccess) {
          if (pitch == row && src.pitch_bytes == row)
            err = cudaMemcpyAsync(d.ptr, src.ptr, row * src.height, cudaMemcpyHostToDevice, s->copy_stream);
          else
            err = cudaMemcpy2DAsync(d.ptr, pitch, src.ptr, src.pitch_bytes, row, src.height, cudaMemcpyHostToDevice,
                                    s->copy_stream);
        }
        return d;
      };
      for (int i = 0; i < n; ++i) {
        const DfkSfmWorkItem& w = items[i];
        const uint32_t W = w.img0.width, H = w.img0.height;
        const bool fused = w.code != nullptr;
        if (pass == 0 && (W == 0 || H == 0 || !img_ok(&w.img0, W, H, 1) || !img_ok(&w.img1, W, H, 1) ||
                          !img_ok(&w.prx0_jac, W, H, s->code_size) || !img_ok(&w.grad1, W, H, 2) ||
                          (fused ? !img_ok(&w.prx_orig, W, H, 1) : !img_ok(&w.dpt0, W, H, 1))))
          return fail(h, DFK_ERR_INVALID_ARG, "[SfmStream] inconsistent host image views in work item " + std::to_string(i));
        DfkSfmWorkItem& d = s->dev_items[i];
        d = w;
        d.img0 = stage(w.img0, 1, true);
        d.img1 = stage(w.img1, 1, true);
        d.prx0_jac = stage(w.prx0_jac, (uint32_t)s->code_size, true);
        d.grad1 = stage(w.grad1, 2, true);
        const DfkImage scalar = w.img0;  // geometry of a scalar scratch image
        d.valid0 = stage(scalar, 1, false);
        if (fused) {
          d.prx_orig = stage(w.prx_orig, 1, true);
          d.dpt0 = stage(scalar, 1, false);  // the decoded depth stays on the device
        } else {
          d.dpt0 = stage(w.dpt0, 1, true);
        }
      }
      if (pass == 0 && cursor > sl.dev.cap) {  // the slot is idle (not busy): its memory can be replaced
        sl.dev.release();  // so that it grows to exactly what this submission needs
        DFK_CUDA(h, sl.dev.ensure(cursor), "[SfmStream] slot allocation failed");
      }
    }
    if (err != cudaSuccess) return cuda_fail(h, err, "[SfmStream] upload failed");
    DFK_CUDA(h, cudaEventRecord(sl.uploaded, s->copy_stream), "[SfmStream] event record failed");
    DFK_CUDA(h, cudaStreamWaitEvent(h->stream, sl.uploaded, 0), "[SfmStream] stream wait failed");
    DFK_TRY(run_batch(h, s->dev_items.data(), n, s->code_size, sl.rec_dev.ptr));
    DFK_CUDA(h, cudaMemcpyAsync(sl.rec_host.ptr, sl.rec_dev.ptr,
                                (size_t)DFK_SFM_RECORD_FLOATS(s->code_size) * n * sizeof(float), cudaMemcpyDeviceToHost,
                                h->stream),
             "[SfmStream] result download failed");
    DFK_CUDA(h, cudaEventRecord(sl.done, h->stream), "[SfmStream] event record failed");
    // the NEXT use of this slot's staging memory (depth submissions later) is host-ordered behind wait(ticket); the copy
    // stream itself must not run ahead of the evaluation that still reads the slot it is about to overwrite
    sl.busy = true;
    sl.n = n;
    sl.ticket = s->next_ticket;
    *ticket = s->next_ticket++;
    return DFK_OK;
  });
}

DfkStatus dfk_sfm_stream_wait(DfkHandle h, DfkSfmStream* s, uint64_t ticket, float* records_host)
{
  return guarded(h, [&] {
    if (!s || !records_host) return fail(h, DFK_ERR_INVALID_ARG, "[SfmStream] null argument");
    DfkSfmStream::Slot& sl = s->slots[ticket % (uint64_t)s->depth];
    if (!sl.busy || sl.ticket != ticket || ticket != s->next_wait)
      return fail(h, DFK_ERR_INVALID_ARG, "[SfmStream] tickets must be waited for once, in submission order");
    DeviceGuard guard(h->device);
    DFK_CUDA(h, cudaEventSynchronize(sl.done), "[SfmStream] kernel launch failed");
    memcpy(records_host, sl.rec_host.ptr, (size_t)DFK_SFM_RECORD_FLOATS(s->code_size) * sl.n * sizeof(float));
    sl.busy = false;
    s->next_wait += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_depth_run_step(DfkHandle h, const float* code, int code_size, const DfkImage* target_dpt,
                             const DfkImage* prx_orig, const DfkImage* prx_jac, float* JtJ, float* Jtr, float* residual,
                             uint64_t* inliers)
{
  return guarded(h, [&] {
    if (!code || !target_dpt || !prx_orig || !prx_jac || !JtJ || !Jtr || !residual || !inliers)
      return fail(h, DFK_ERR_INVALID_ARG, "[DepthAligner::RunStep] null argument");
    // CHECK_EQ(codesize, CS) (cu_depthaligner.cpp:90-91): the code size must be one this build instantiates
    if (!depth_supported(code_size))
      return fail(h, DFK_ERR_UNSUPPORTED,
                  "DepthAligner used with a different code size than it was compiled for: " + std::to_string(code_size));
    const uint32_t W = target_dpt->width, H = target_dpt->height;
    if (W == 0 || H == 0 || !img_ok(target_dpt, W, H, 1) || !img_ok(prx_orig, W, H, 1) || !img_ok(prx_jac, W, H, code_size))
      return fail(h, DFK_ERR_INVALID_ARG, "[DepthAligner::RunStep] inconsistent image views");
    DeviceGuard guard(h->device);
    const int area = (int)(W * H);
    const int blocks = std::max(1, std::min(2 * h->num_sms, (area + 63) / 64));
    const size_t NH = (size_t)code_size * (code_size + 1) / 2, REC = NH + code_size + 2;
    DFK_CUDA(h, h->partials_dev.ensure((size_t)blocks * depth_partial_floats(code_size)),
             "[DepthAligner::RunStep] scratch allocation failed");
    DFK_CUDA(h, h->records_dev.ensure(REC), "[DepthAligner::RunStep] scratch allocation failed");
    DFK_CUDA(h, h->records_host.ensure(REC), "[DepthAligner::RunStep] pinned allocation failed");
    DFK_CUDA(h, cudaMemcpyAsync(h->code_dev.ptr, code, sizeof(float) * code_size, cudaMemcpyHostToDevice, h->stream),
             "[DepthAligner::RunStep] code upload failed");
    DFK_CUDA(h, launch_depth_step(h->code_dev.ptr, code_size, (int)W, (int)H, view_of(target_dpt), view_of(prx_orig),
                                  view_of(prx_jac), h->params.sfmparams.avg_dpt, h->partials_dev.ptr, h->counter.ptr,
                                  h->records_dev.ptr, blocks, h->stream),
             "[DepthAligner::RunStep] kernel launch failed");
    h->launches += 1;
    DFK_TRY(download(h, h->records_host.ptr, h->records_dev.ptr, REC * sizeof(float),
                     "[DepthAligner::RunStep] kernel launch failed", "[DepthAligner::RunStep] kernel launch failed"));
    unpack_record(h->records_host.ptr, NH, code_size, JtJ, Jtr, residual, inliers);
    return DFK_OK;
  });
}

namespace {

DfkStatus depth_prior_batch(DfkHandle h, const char* what, const DfkDepthPriorItem* items, int n, int code_size,
                            float* out_dev, bool gram)
{
  if (!out_dev) return fail(h, DFK_ERR_INVALID_ARG, std::string(what) + "null argument");
  DeviceGuard guard(h->device);
  DepthPriorStaged st;
  DFK_TRY(stage_depth_prior(h, what, items, n, code_size, true, h->staging, h->depth_prior_dev, &st));
  DFK_CUDA(h, h->depth_prior_partials.ensure((size_t)st.rows * depth_prior_partial_floats(code_size, gram)),
           (std::string(what) + "scratch allocation failed").c_str());
  DFK_CUDA(h, launch_depth_prior_batch(code_size, st.descs.at(h->depth_prior_dev.ptr), n, st.max_parts,
                                       h->params.sfmparams.avg_dpt, h->depth_prior_partials.ptr, out_dev, gram,
                                       h->stream),
           (std::string(what) + "kernel launch failed").c_str());
  h->launches += 2;
  return DFK_OK;
}

}  // namespace

DfkStatus dfk_depth_prior_linearize_batch(DfkHandle h, const DfkDepthPriorItem* items, int n, int code_size,
                                          float* records_dev)
{
  return guarded(h, [&] {
    return depth_prior_batch(h, "[DepthPriorFactor::linearize batch] ", items, n, code_size, records_dev, true);
  });
}

DfkStatus dfk_depth_prior_error_batch(DfkHandle h, const DfkDepthPriorItem* items, int n, int code_size, float* out_dev)
{
  return guarded(h, [&] {
    return depth_prior_batch(h, "[DepthPriorFactor::error batch] ", items, n, code_size, out_dev, false);
  });
}

}  // extern "C"
