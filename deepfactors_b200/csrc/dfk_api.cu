// dfk_api.cu -- C ABI of libdfk.so (see include/dfk.h): argument validation, host-side SE3
// algebra (relative pose + Jacobians, as the reference does on the host in
// cu_sfmaligner.cpp:164-166), launch planning, scratch ownership, error reporting.
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
#include "dfk_internal.h"
#include "dfk_levels.h"
#include "dfk_lm.h"
#include "dfk_orb_model.h"
#include "dfk_se3.cuh"

using namespace dfk;

namespace {

// Grow-only scratch that owns its memory: device memory (cudaMalloc) or pinned host memory (cudaMallocHost).
template <typename T, bool Pinned>
struct Scratch {
  T* ptr = nullptr;
  size_t cap = 0;  // elements

  Scratch() = default;
  Scratch(Scratch&& o) noexcept : ptr(o.ptr), cap(o.cap) { o.ptr = nullptr; o.cap = 0; }
  ~Scratch() { release(); }

  void release()
  {
    if constexpr (Pinned) cudaFreeHost(ptr);
    else cudaFree(ptr);
    ptr = nullptr;
    cap = 0;
  }
  // At least `need` elements, twice the old capacity if that is more.  The old memory is freed first: cudaFree and
  // cudaFreeHost synchronise the device, so work still running on the stream has finished with it.  A failed allocation
  // leaves capacity 0.
  cudaError_t ensure(size_t need)
  {
    if (cap >= need) return cudaSuccess;
    const size_t n = std::max(need, cap * 2);
    release();
    void* p = nullptr;
    const cudaError_t e = Pinned ? cudaMallocHost(&p, n * sizeof(T)) : cudaMalloc(&p, n * sizeof(T));
    if (e != cudaSuccess) return e;
    ptr = static_cast<T*>(p);
    cap = n;
    return e;
  }
};
template <typename T>
using DeviceBuf = Scratch<T, false>;
template <typename T>
using PinnedBuf = Scratch<T, true>;

}  // namespace

struct DfkContext {
  int device = 0;
  int num_sms = 1;
  int sm_limit = 0;  // dfk_set_sm_limit: SMs the persistent step kernels may occupy (0 = all)
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;
  std::string err;
  DfkSfmAlignerParams params;
  DfkGramMode gram_mode = DFK_GRAM_AUTO;
  float se3_huber_delta = 0.1f;  // cu_se3aligner.h:85

  DeviceBuf<float> simple_scratch;       // kSimpleScratchFloats
  DeviceBuf<unsigned int> counter;       // 1 (self-resetting ticket)
  DeviceBuf<float> out_dev;              // 32 floats
  PinnedBuf<float> out_host;             // 32 floats
  DeviceBuf<float> code_dev;             // 256 floats
  DeviceBuf<float> track_dev;            // dfk_se3_track: [pose 8 | per-iteration history 36 each]
  PinnedBuf<float> track_host;           // mirror of track_dev + the last system (32)
  // dfk_se3_track_batch, apart from the single-problem buffers above so neither path disturbs the other:
  //   batch_dev  [descriptors L x N (level-major) | poses 8 N | last systems 32 N]  (bytes; one H2D, one D2H per call)
  //   batch_partials  N x stride x 32 floats,  batch_counters  N self-resetting tickets (zeroed on allocation)
  DeviceBuf<unsigned char> batch_dev;
  PinnedBuf<unsigned char> batch_host;   // mirror of batch_dev
  DeviceBuf<float> batch_partials;
  DeviceBuf<unsigned int> batch_counters;
  // dfk_sfm_evaluate_error_batch, apart from the single-call buffers: the descriptors (one H2D per call), the partials
  // (one 32-float row per block of every item) and one self-resetting ticket per item (zeroed on allocation)
  DeviceBuf<EvalErrorDesc> eval_descs;
  std::vector<EvalErrorDesc> eval_host;
  DeviceBuf<float> eval_partials;
  DeviceBuf<unsigned int> eval_counters;
  // dfk_update_depth_batch: [descriptors | codes] (bytes), one H2D per call from depth_host
  DeviceBuf<unsigned char> depth_dev;
  std::vector<unsigned char> depth_host;

  // dfk_reprojection_linearize / dfk_sparse_geometric_linearize: [one item's staging block | rows (| err2)]
  DeviceBuf<unsigned char> sparse_dev;
  PinnedBuf<unsigned char> sparse_host;  // mirror
  // dfk_reprojection_linearize_batch: [descriptors | codes | query | train] (bytes), one H2D per call from rep_host
  DeviceBuf<unsigned char> rep_dev;
  std::vector<unsigned char> rep_host;
  // dfk_sparse_geometric_linearize_batch: [descriptors | codes | points] (bytes), one H2D per call from geo_host; apart
  // from rep_dev so that batches of the two kinds enqueued back to back keep their own staging
  DeviceBuf<unsigned char> geo_dev;
  std::vector<unsigned char> geo_host;
  DeviceBuf<SfmItemDev> items_dev;
  DeviceBuf<float> partials_dev;
  // dfk_hamming_match_batch / dfk_reprojection_match_batch: the item descriptors (one H2D per call) and the RANSAC
  // scratch [matches (int2 per query) | hypothesis counts | selections (int3 per item)] (bytes)
  DeviceBuf<MatchItemDev> match_items;
  std::vector<MatchItemDev> match_host;
  DeviceBuf<unsigned char> match_scratch;
  // dfk_orb_detect_batch: the item descriptors (one H2D per call) and the detector's scratch (see the call)
  DeviceBuf<OrbItemDev> orb_items;
  std::vector<OrbItemDev> orb_host;
  DeviceBuf<unsigned char> orb_scratch;
  // dfk_window_marginalize_frames / dfk_window_add_priors: the call's index lists (one pageable H2D per call)
  DeviceBuf<int> window_lists;
  // dfk_window_marginalize_keyframe: the call's lists [refs | tile rows / cols | member locations | update tasks] (one
  // pageable H2D per call), the code of m, and the local system's workspace (tiles, rhs, f)
  DeviceBuf<int> marg_lists;
  DeviceBuf<double> marg_code;
  DeviceBuf<double> marg_dev;
  // normalised ray tables of the RunStep kernels: they depend on (fx, u0, width, fy, v0, height) only, so they are
  // built once per camera level and reused by every later call (one launch less per evaluation in steady state)
  struct RayTab {
    float fx, fy, u0, v0;
    uint32_t w, h;
    DeviceBuf<float> dev;
    bool built;  // the table kernel has been enqueued for it (an entry whose call failed before that stays false)
  };
  std::vector<RayTab> ray_cache;
  std::vector<size_t> ray_pending;  // entries the current call uses that are not built yet: run the table kernel
  bool ray_flush = false;           // a call missed on a full cache: empty it when the next call starts
  DeviceBuf<float> codes_dev;  // fused depth decode: code_size floats per work item
  std::vector<float> codes_host;
  DeviceBuf<float> records_dev;
  PinnedBuf<float> records_host;
  std::vector<SfmItemDev> items_host;

  // measurement hooks (dfk_set_profiling / dfk_get_profile)
  bool profiling = false;
  std::vector<cudaEvent_t> ev_pool;  // pairs: [2k] start, [2k+1] stop
  size_t ev_used = 0;                // number of pairs recorded since the last read
  double ev_ms_accum = 0.0;          // time of pairs already drained
  uint64_t ev_count_accum = 0;
  uint64_t launches = 0;

  // the scratch buffers free themselves after this
  ~DfkContext()
  {
    for (cudaEvent_t e : ev_pool) cudaEventDestroy(e);
    if (own_stream) cudaStreamDestroy(own_stream);
  }
};

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

// CSR adjacency of a keyframe window on the device (dfk_window_create)
struct DfkWindow {
  int device = 0;
  WindowDev dev{};
  // one allocation: kf0_ptr | kf0_items | kf1_ptr | kf1_items | pair_ptr | pair_items | lk0_ptr | lk0_links |
  // lk1_ptr | lk1_links
  DeviceBuf<int> ints;
  DeviceBuf<float> areas;
  size_t floats = 0;
  // host copy of the structure, for dfk_window_solver_create and dfk_window_marginalize_keyframe
  std::vector<int> pair_k0, pair_k1, link_k0, link_k1, item_pair;
  // keyframe priors (dfk_window_create_priors): members prior_kf[prior_ptr[q] .. prior_ptr[q + 1]), the prior blocks
  // (blk_i < blk_j) and their device lists (KfPriorDev)
  std::vector<int> prior_ptr{0}, prior_kf, blk_i, blk_j;
  std::vector<long long> prior_off;  // doubles: start of prior q in a priors buffer; back() = the buffer's size
  DeviceBuf<int> kp_ints;
  DeviceBuf<long long> kp_off;
  KfPriorDev kp{};
};

// damped block-sparse Cholesky of one window (dfk_window_solver_create)
struct DfkWindowSolver {
  int device = 0;
  int num_vars = 0, code_size = 0, num_keyframes = 0;
  WindowSolverDev* dev = nullptr;
  ~DfkWindowSolver() { window_solver_destroy(dev); }
};

namespace {

DfkStatus fail(DfkHandle h, DfkStatus s, const std::string& msg)
{
  if (h) h->err = msg;
  return s;
}

// out-of-memory exit of an extern "C" entry point (never throws itself)
DfkStatus oom(DfkHandle h) noexcept
{
  if (h) {
    try {
      h->err = "out of host memory";
    } catch (...) {
    }
  }
  return DFK_ERR_NOMEM;
}

// Every entry point that takes a handle runs its body through this: a null handle is an argument error, and no C++
// exception (std::bad_alloc / std::length_error from host containers) may cross the C ABI.
template <class F>
DfkStatus guarded(DfkHandle h, F&& body) noexcept
{
  if (!h) return DFK_ERR_INVALID_ARG;
  try {
    return body();
  } catch (...) {
    return oom(h);
  }
}

DfkStatus cuda_fail(DfkHandle h, cudaError_t e, const char* what)
{
  // message format of vc::CUDAException thrown from CudaCheckLastError (launch_utils.h:26-32)
  std::string m = std::string(what) + ": " + cudaGetErrorString(e);
  cudaGetLastError();  // clear sticky-less errors
  return fail(h, DFK_ERR_CUDA, m);
}

#define DFK_CUDA(h, call, what)                            \
  do {                                                     \
    cudaError_t e__ = (call);                              \
    if (e__ != cudaSuccess) return cuda_fail(h, e__, what); \
  } while (0)

// passes on the failure of a helper or of a nested entry point
#define DFK_TRY(call)                      \
  do {                                     \
    const DfkStatus s__ = (call);          \
    if (s__ != DFK_OK) return s__;         \
  } while (0)

// results to the host: one copy on the handle's stream, then the host waits for it
DfkStatus download(DfkHandle h, void* host, const void* dev, size_t bytes, const char* copy_what, const char* sync_what)
{
  DFK_CUDA(h, cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, h->stream), copy_what);
  DFK_CUDA(h, cudaStreamSynchronize(h->stream), sync_what);
  return DFK_OK;
}

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev)
  {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard()
  {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// ---------------------------------------------------------------------------- SE3 algebra (fp32): dfk_se3.cuh
using se3f::relative_pose;

// ---------------------------------------------------------------------------- validation helpers
bool img_ok(const DfkImage* im, uint32_t w, uint32_t h, uint32_t floats_per_px)
{
  return im && im->ptr && im->width == w && im->height == h && (im->pitch_bytes % 4 == 0) &&
         im->pitch_bytes >= (size_t)w * floats_per_px * 4;
}

// The validity window comes from the camera (PixelValid: u < cam.width - border, pinhole_camera_impl.h:102-108) while the
// bilinear taps index the images: a camera larger than the level it is used with (e.g. a level-0 camera with level-1
// buffers) would read outside them.  The reference has no such check (it would read out of bounds); here it is an
// argument error.
bool cam_ok(const DfkCamera* cam, uint32_t w, uint32_t h)
{
  return cam && cam->width <= (float)w && cam->height <= (float)h && cam->width >= 0.0f && cam->height >= 0.0f;
}

View view_of(const DfkImage* im) { return View{static_cast<const float*>(im->ptr), (uint32_t)(im->pitch_bytes / 4)}; }

bool aligned(const void* p, size_t a) { return reinterpret_cast<uintptr_t>(p) % a == 0; }

PixelCam make_pixel_cam(const float pose[7], const DfkCamera* cam, int border, float min_dpt)
{
  PixelCam pc;
  for (int i = 0; i < 4; ++i) pc.q[i] = pose[i];
  for (int i = 0; i < 3; ++i) pc.t[i] = pose[4 + i];
  pc.fx = cam->fx; pc.fy = cam->fy; pc.u0 = cam->u0; pc.v0 = cam->v0;
  pc.border = (float)border;
  pc.ulim = cam->width - (float)border;   // PixelValid: x < width_ - border (pinhole_camera_impl.h:107)
  pc.vlim = cam->height - (float)border;
  pc.min_dpt = min_dpt;
  return pc;
}

// RelativePose(pose1, pose0, J_pose1, J_pose0): q, t and R of pose_10 = pose1^-1 * pose0, both 6x6 Jacobians, and the
// intrinsics, into an SfmItemDev or a SparsePose
template <class D>
void set_relative_pose(D& d, const float pose1[7], const float pose0[7], const DfkCamera& cam)
{
  se3f::set_relative_pose_only(d, pose1, pose0);
  d.fx = cam.fx; d.fy = cam.fy; d.u0 = cam.u0; d.v0 = cam.v0;
}

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
  static const bool no_perm = []() { const char* e = getenv("DFK_NO_PERM"); return e && e[0] == '1'; }();
  if (no_perm) return 1;
  if (n <= 2 || n > 65535u) return 1;  // keeps k * perm_mul below 2^32 on the device
  uint32_t m = (uint32_t)((double)n * 0.6180339887498949);
  if (m < 1) m = 1;
  while (gcd_u32(m, n) != 1) ++m;
  return m % n == 0 ? 1 : m;
}

void plan_tiles(SfmItemDev* items, int n, int max_ctas, SfmLaunchPlan* plan);

DfkStatus build_items(DfkHandle h, const DfkSfmWorkItem* items, int n, int code_size, int tile_px, int max_ctas,
                      const float* codes_dev, SfmLaunchPlan* plan)
{
  h->ray_pending.clear();
  // a caller cycling through more camera levels than the cache holds: start over (cudaFree synchronises).  Only here,
  // between calls, so that no item of a call is left pointing at a freed table
  if (h->ray_flush) {
    h->ray_cache.clear();
    h->ray_flush = false;
  }
  const DfkDenseSfmParams& sp = h->params.sfmparams;
  h->items_host.resize(n);
  for (int i = 0; i < n; ++i) {
    const DfkSfmWorkItem& w = items[i];
    SfmItemDev& d = h->items_host[i];
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
      memcpy(h->codes_host.data() + (size_t)i * code_size, w.code, sizeof(float) * code_size);
    }
    d.width = W; d.height = H; d.num_pixels = W * H;
    d.num_tiles = (d.num_pixels + tile_px - 1) / tile_px;
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
  plan_tiles(h->items_host.data(), n, max_ctas, plan);
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

// The RunStep kernel a batch runs on (the Gram mode, the code size and the grad1 layout decide) and its launch shape
struct StepKernel {
  bool tc = false, wide = false;
  int tile_px = 0, max_ctas = 0;
  size_t pfloats = 0;  // floats per partial
};

DfkStatus choose_step_kernel(DfkHandle h, const DfkSfmWorkItem* items, int n, int code_size, StepKernel* k)
{
  const bool wide = sfm_wide_supported(code_size);
  if (!sfm_fp32_supported(code_size) && !wide)
    return fail(h, DFK_ERR_UNSUPPORTED,
                "[SfmAligner::RunStep] no kernel instantiated for code size " + std::to_string(code_size));
  const bool tc_ok = sfm_tc_supported(code_size) || sfm_tc_wide_supported(code_size);
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
  k->tile_px = tc ? sfm_tc_tile_pixels(code_size) : (wide ? sfm_wide_tile_pixels(code_size) : kTilePixels);
  const int ctas_per_sm = tc ? sfm_tc_ctas_per_sm(code_size) : (wide ? 1 : sfm_fp32_ctas_per_sm(code_size));
  const int sms = (h->sm_limit > 0 && h->sm_limit < h->num_sms) ? h->sm_limit : h->num_sms;
  k->max_ctas = ctas_per_sm * sms;
  k->pfloats = tc ? sfm_tc_partial_floats(code_size) : sfm_partial_floats(code_size);
  return DFK_OK;
}

// the step kernel and the finalize of a planned, uploaded work list
DfkStatus launch_step(DfkHandle h, const StepKernel& k, int code_size, const SfmItemDev* items_dev, int n,
                      const SfmLaunchPlan& plan, float* partials_dev, float* records_dev)
{
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  if (h->profiling) DFK_TRY(profile_events(h, &ev0, &ev1));
  if (k.tc && k.wide) {
    DFK_CUDA(h, launch_sfm_tc_wide(code_size, items_dev, plan, partials_dev, h->stream, ev0, ev1),
             "[SfmAligner::RunStep] kernel launch failed");
  } else if (k.tc) {
    DFK_CUDA(h, launch_sfm_tc(items_dev, plan, partials_dev, h->stream, ev0, ev1),
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

DfkStatus run_batch(DfkHandle h, const DfkSfmWorkItem* items, int n, int code_size, float* records_dev)
{
  if (!items || n <= 0 || !records_dev) return fail(h, DFK_ERR_INVALID_ARG, "[SfmAligner::RunStep] null/empty batch");
  StepKernel k;
  DFK_TRY(choose_step_kernel(h, items, n, code_size, &k));
  DeviceGuard guard(h->device);
  SfmLaunchPlan plan;
  bool any_fused = false;
  for (int i = 0; i < n; ++i) any_fused = any_fused || items[i].code != nullptr;
  if (any_fused) {
    DFK_CUDA(h, h->codes_dev.ensure((size_t)n * code_size), "[SfmAligner::RunStep] scratch allocation failed");
    h->codes_host.assign((size_t)n * code_size, 0.0f);
  }
  DFK_TRY(build_items(h, items, n, code_size, k.tile_px, k.max_ctas, h->codes_dev.ptr, &plan));
  if (any_fused)
    DFK_CUDA(h, cudaMemcpyAsync(h->codes_dev.ptr, h->codes_host.data(), sizeof(float) * (size_t)n * code_size,
                                cudaMemcpyHostToDevice, h->stream),
             "[SfmAligner::RunStep] code upload failed");
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

// ---------------------------------------------------------------------------- sparse factors
// A single call is a batch of one: the same checks, descriptors and staging.  Sparse<Item> is what the two factor kinds
// stage differently: the argument check (the failure text, or null), the matches / points of a factor and the bytes each
// takes, the codes per factor, and one factor's descriptor, codes and payload.
template <class Item>
struct Sparse;

template <>
struct Sparse<DfkReprojectionItem> {
  using Dev = ReprojItemDev;
  static constexpr int codes = 1;
  static constexpr size_t unit_bytes = 4 * sizeof(float);  // payload: query 2 total | train 2 total
  static constexpr const char* units = "matches";
  static size_t count(const DfkReprojectionItem& it) { return (size_t)it.num_matches; }
  static const char* error(const DfkReprojectionItem& it, int code_size)
  {
    if (!it.code || !it.query_xy || !it.train_xy) return "null argument";
    if (it.num_matches < 1 || !(it.sigma > 0.0f)) return "no matches / non-positive sigma";
    const uint32_t W = it.prx_orig.width, H = it.prx_orig.height;
    if (W == 0 || H == 0 || !img_ok(&it.prx_orig, W, H, 1) || !img_ok(&it.prx_jac, W, H, code_size))
      return "inconsistent image views";
    return nullptr;
  }
  // begin: the factor's first match, total: the matches of the block
  static void pack(const DfkReprojectionItem& it, int code_size, size_t begin, size_t total, Dev& d, float* code,
                   const float* code_dev, unsigned char* payload)
  {
    d = Dev{{}, view_of(&it.prx_orig), view_of(&it.prx_jac), code_dev, (int)it.prx_orig.width, (int)it.prx_orig.height,
            it.num_matches, (int)begin, it.cauchy_delta, it.sigma};
    set_relative_pose(d.sp, it.pose1, it.pose0, it.cam);  // pose10_J_pose1, pose10_J_pose0 (:189-190)
    memcpy(code, it.code, sizeof(float) * code_size);
    float* query = reinterpret_cast<float*>(payload);
    memcpy(query + 2 * begin, it.query_xy, sizeof(float) * 2 * it.num_matches);
    memcpy(query + 2 * (total + begin), it.train_xy, sizeof(float) * 2 * it.num_matches);
  }
};

template <>
struct Sparse<DfkSparseGeometricItem> {
  using Dev = GeoItemDev;
  static constexpr int codes = 2;  // code0, code1
  static constexpr size_t unit_bytes = 2 * sizeof(int32_t);  // payload: points 2 total
  static constexpr const char* units = "points";
  static size_t count(const DfkSparseGeometricItem& it) { return (size_t)it.num_points; }
  static const char* error(const DfkSparseGeometricItem& it, int code_size)
  {
    if (!it.code0 || !it.code1 || !it.points_xy) return "null argument";
    if (it.num_points < 1 || !(it.huber_delta > 0.0f)) return "no points / non-positive huber delta";
    const uint32_t W = it.prx0_orig.width, H = it.prx0_orig.height;
    if (W == 0 || H == 0 || !img_ok(&it.prx0_orig, W, H, 1) || !img_ok(&it.prx0_jac, W, H, code_size) ||
        !img_ok(&it.prx1_orig, W, H, 1) || !img_ok(&it.prx1_jac, W, H, code_size) || !img_ok(&it.dpt_grad1, W, H, 2))
      return "inconsistent image views";
    // the nearest-neighbour lookups in keyframe 1 index with the camera's validity window
    if (!cam_ok(&it.cam, W, H)) return "camera larger than the image views";
    return nullptr;
  }
  static void pack(const DfkSparseGeometricItem& it, int code_size, size_t begin, size_t /*total*/, Dev& d, float* code,
                   const float* code_dev, unsigned char* payload)
  {
    d = Dev{{}, view_of(&it.prx0_orig), view_of(&it.prx0_jac), view_of(&it.prx1_orig), view_of(&it.prx1_jac),
            view_of(&it.dpt_grad1), code_dev, code_dev + code_size, it.cam.width, it.cam.height, (int)it.prx0_orig.width,
            (int)it.prx0_orig.height, it.num_points, (int)begin, it.huber_delta};
    set_relative_pose(d.sp, it.pose1, it.pose0, it.cam);  // pose10_J_pose1, pose10_J_pose0 (:176-178)
    memcpy(code, it.code0, sizeof(float) * code_size);
    memcpy(code + code_size, it.code1, sizeof(float) * code_size);
    memcpy(reinterpret_cast<int32_t*>(payload) + 2 * begin, it.points_xy, sizeof(int32_t) * 2 * it.num_points);
  }
};

// Host staging: the batches stage in pageable memory (cudaMemcpyAsync has read it when it returns, so the next batch may
// refill it while the copy is still queued); the synchronous single calls in pinned memory, into which their rows return.
cudaError_t host_block(std::vector<unsigned char>& v, size_t bytes, unsigned char** p)
{
  v.assign(bytes, 0);
  *p = v.data();
  return cudaSuccess;
}
cudaError_t host_block(PinnedBuf<unsigned char>& b, size_t bytes, unsigned char** p)
{
  const cudaError_t e = b.ensure(bytes);
  *p = b.ptr;
  return e;
}

struct Staged {
  size_t bytes = 0;               // of the uploaded block; the caller's outputs may follow it
  size_t total = 0;               // matches / points
  const unsigned char* payload = nullptr;  // device address of the matches / points
};

// Checks the code size and items[0, n) (messages begin with `what`, a batch's name the item), then stages the factors in
// one upload: [descriptors n | codes n x codes C | payload], packed in `host` and copied to `dev`, both grown by
// out_bytes for the caller's outputs.
template <class Item, class HostBuf>
DfkStatus stage(DfkHandle h, const std::string& what, bool batch, const Item* items, int n, int code_size,
                size_t out_bytes, HostBuf& host, DeviceBuf<unsigned char>& dev, Staged* st)
{
  using S = Sparse<Item>;
  if (!sparse_supported(code_size))
    return fail(h, DFK_ERR_UNSUPPORTED, what + "code size not instantiated: " + std::to_string(code_size));
  for (int i = 0; i < n; ++i) {
    if (const char* e = S::error(items[i], code_size))
      return fail(h, DFK_ERR_INVALID_ARG, what + (batch ? "item " + std::to_string(i) + ": " : "") + e);
    st->total += S::count(items[i]);
  }
  if (st->total > (size_t)INT32_MAX)
    return fail(h, DFK_ERR_INVALID_ARG, what + "more than 2^31 - 1 " + S::units + " in one call");
  const size_t desc_bytes = (sizeof(typename S::Dev) * (size_t)n + 15) & ~(size_t)15;
  const size_t code_floats = (size_t)S::codes * code_size, payload = desc_bytes + sizeof(float) * n * code_floats;
  st->bytes = payload + S::unit_bytes * st->total;
  DFK_CUDA(h, dev.ensure(st->bytes + out_bytes), (what + "scratch allocation failed").c_str());
  unsigned char* hb = nullptr;
  DFK_CUDA(h, host_block(host, st->bytes + out_bytes, &hb), (what + "pinned allocation failed").c_str());
  const float* codes_dev = reinterpret_cast<const float*>(dev.ptr + desc_bytes);
  for (size_t i = 0, begin = 0; i < (size_t)n; begin += S::count(items[i]), ++i)
    S::pack(items[i], code_size, begin, st->total, reinterpret_cast<typename S::Dev*>(hb)[i],
            reinterpret_cast<float*>(hb + desc_bytes) + i * code_floats, codes_dev + i * code_floats, hb + payload);
  DFK_CUDA(h, cudaMemcpyAsync(dev.ptr, hb, st->bytes, cudaMemcpyHostToDevice, h->stream), (what + "upload failed").c_str());
  st->payload = dev.ptr + payload;
  return DFK_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------------- window problem
// One window's every work item, planned and uploaded once (dfk_window_problem_create); the loop kernels of
// dfk_window_lm.cu re-pose them from the device state.  Everything the items point at that is not the caller's (code
// slots, ray tables, depth scratch of the error path) belongs to the problem.
struct DfkWindowProblem {
  int device = 0;
  const DfkWindow* w = nullptr;
  int K = 0, F = 0, C = 0, B = 0;
  float avg_dpt = 2.0f, huber_delta = 0.1f;  // the handle's sfmparams at create, like the dense items' (SfmItemDev)
  int nd = 0, nr = 0, ng = 0, ndep = 0, ne = 0, mf = 0, nkm = 0;  // items of each kind, frame priors, kf-prior members
  size_t S = 0;  // doubles of one state: (K + F) 7 + K C
  StepKernel step;
  SfmLaunchPlan plan;
  DeviceBuf<SfmItemDev> dense;
  DeviceBuf<float> dense_codes;
  std::vector<DeviceBuf<float>> rays;
  DeviceBuf<unsigned char> rep, geo;  // the sparse batches' staged blocks [descriptors | codes | payload]
  std::vector<unsigned char> rep_host, geo_host;
  const unsigned char* rep_payload = nullptr;
  const unsigned char* geo_payload = nullptr;
  size_t rep_total = 0;
  DeviceBuf<EvalErrorDesc> err;
  int err_max_blocks = 1, err_rows = 0;
  DeviceBuf<unsigned char> depth;  // [descriptors | codes]
  int depth_max_blocks = 1;
  DeviceBuf<float> depth_scratch;
  DeviceBuf<int4> slots;           // dense | error | reproj | geo | depth
  DeviceBuf<double> areas;         // W * H of each error item
  DeviceBuf<float> err_out;        // (ne + nr + ng) x 2
  DeviceBuf<double> state;         // two states: [cur] the problem's, [1 - cur] an LM candidate
  int cur = 0;
  DeviceBuf<double> frows, kfrows, x0, delta;  // prior rows, frozen points (frame priors, then kf members), deltas
  DeviceBuf<int> delta_kf;         // keyframe of every delta row
  DeviceBuf<int> fp_lists;         // dfk_window_add_priors' CSR: ptr[K + 1] | prior indices
  float* records = nullptr;
  float* geo_records = nullptr;
  WindowSolverDev* solver[2] = {nullptr, nullptr};  // [fix_first_pose]
  DeviceBuf<float> bufs;           // the LM's accepted and candidate window buffers
  int acc = 0;
  DeviceBuf<double> dx;
  DeviceBuf<unsigned char> small;  // [energy 8 doubles | info int32]
  PinnedBuf<unsigned char> small_host;
  // active subsets (dfk_window_problem_set_active): the create-time dense and error items with their slots and areas
  // are the templates a mask selects from; the selected items go to arrays of their own, so the full arrays stay as
  // create planned them and an all-active mask runs exactly the create-time launches
  std::vector<SfmItemDev> dense_tmpl;
  std::vector<EvalErrorDesc> err_tmpl;
  std::vector<int4> slots_tmpl;      // dense | error
  std::vector<double> areas_tmpl;
  bool sub_dense = false, sub_err = false;
  int nda = 0, nea = 0;              // active dense / error items while sub_dense / sub_err
  SfmLaunchPlan sub_plan;
  DeviceBuf<SfmItemDev> dense_sub;
  DeviceBuf<EvalErrorDesc> err_sub;
  DeviceBuf<int4> sub_slots;         // dense [0, nd) | error [nd, nd + ne)
  DeviceBuf<double> areas_sub;
  DeviceBuf<int> rec_src;            // record slot i <- subset record rec_src[i], -1: zeros
  DeviceBuf<float> sub_records;
  ~DfkWindowProblem()
  {
    window_solver_destroy(solver[0]);
    window_solver_destroy(solver[1]);
  }
  double* st(int i) const { return state.ptr + (size_t)i * S; }
  double* energy() const { return reinterpret_cast<double*>(small.ptr); }
  int32_t* info() const { return reinterpret_cast<int32_t*>(small.ptr + 8 * sizeof(double)); }
};

namespace {

WindowReposeDev repose_args(const DfkWindowProblem* p, const double* state)
{
  const int4* sl = p->slots.ptr;
  WindowReposeDev a{};
  a.code_size = p->C;
  a.num_poses = p->K + p->F;
  a.state = state;
  a.dense = p->dense.ptr; a.dense_slots = sl; a.num_dense = p->nd;
  a.error = p->err.ptr; a.error_slots = sl + p->nd; a.num_error = p->ne;
  if (p->sub_dense) {
    a.dense = p->dense_sub.ptr; a.dense_slots = p->sub_slots.ptr; a.num_dense = p->nda;
  }
  if (p->sub_err) {
    a.error = p->err_sub.ptr; a.error_slots = p->sub_slots.ptr + p->nd; a.num_error = p->nea;
  }
  a.rep = reinterpret_cast<ReprojItemDev*>(p->rep.ptr); a.rep_slots = sl + p->nd + p->ne; a.num_rep = p->nr;
  a.geo = reinterpret_cast<GeoItemDev*>(p->geo.ptr); a.geo_slots = sl + p->nd + p->ne + p->nr; a.num_geo = p->ng;
  a.depth = reinterpret_cast<DepthDecodeDesc*>(p->depth.ptr); a.depth_slots = sl + p->nd + p->ne + p->nr + p->ng;
  a.num_depth = p->ndep;
  return a;
}

DfkStatus problem_deltas(DfkHandle h, const DfkWindowProblem* p, const double* state)
{
  DFK_CUDA(h, launch_window_deltas(state, p->K + p->F, p->C, p->mf + p->nkm, p->delta_kf.ptr, p->x0.ptr, p->delta.ptr,
                                   h->stream),
           "[WindowProblem] kernel launch failed");
  h->launches += (p->mf + p->nkm) > 0;
  return DFK_OK;
}

// the window buffer at state `state` into buf (dfk_window_problem_linearize)
DfkStatus problem_linearize(DfkHandle h, DfkWindowProblem* p, const double* state, float* buf)
{
  const char* what = "[WindowProblem::linearize] kernel launch failed";
  DFK_CUDA(h, launch_window_repose(repose_args(p, state), h->stream), what);
  h->launches += 1;
  const float avg = p->avg_dpt;
  if (p->sub_dense) {  // the active items only, then every record slot from the subset's records or zeros
    if (p->nda > 0) {
      DFK_CUDA(h, h->partials_dev.ensure((size_t)p->sub_plan.num_partials * p->step.pfloats),
               "[WindowProblem::linearize] scratch allocation failed");
      DFK_TRY(launch_step(h, p->step, p->C, p->dense_sub.ptr, p->nda, p->sub_plan, h->partials_dev.ptr,
                          p->sub_records.ptr));
    }
    DFK_CUDA(h, launch_window_scatter_records(p->sub_records.ptr, p->rec_src.ptr, p->nd, DFK_SFM_RECORD_FLOATS(p->C),
                                              p->records, h->stream),
             what);
    h->launches += 1;
  } else if (p->nd > 0) {
    DFK_CUDA(h, h->partials_dev.ensure((size_t)p->plan.num_partials * p->step.pfloats),
             "[WindowProblem::linearize] scratch allocation failed");
    DFK_TRY(launch_step(h, p->step, p->C, p->dense.ptr, p->nd, p->plan, h->partials_dev.ptr, p->records));
  }
  if (p->nr > 0) {
    const float2* q = reinterpret_cast<const float2*>(p->rep_payload);
    DFK_CUDA(h, launch_reprojection_records(p->C, reinterpret_cast<const ReprojItemDev*>(p->rep.ptr), p->nr, q,
                                            q + p->rep_total, avg, p->records + (size_t)p->nd * DFK_SFM_RECORD_FLOATS(p->C),
                                            h->stream),
             what);
    h->launches += 1;
  }
  if (p->ng > 0) {
    DFK_CUDA(h, launch_sparse_geometric_records(p->C, reinterpret_cast<const GeoItemDev*>(p->geo.ptr), p->ng,
                                                reinterpret_cast<const int2*>(p->geo_payload), avg, p->geo_records,
                                                h->stream),
             what);
    h->launches += 1;
  }
  const DfkWindow* w = p->w;
  DFK_CUDA(h, launch_window_assemble(w->dev, p->records, p->ng > 0 ? p->geo_records : nullptr, buf, h->stream), what);
  h->launches += 1;
  if (w->kp.num_blocks > 0)
    DFK_CUDA(h, cudaMemsetAsync(buf + w->kp.block_off, 0, (w->floats - w->kp.block_off) * sizeof(float), h->stream), what);
  DFK_TRY(problem_deltas(h, p, state));
  if (p->mf > 0) {
    DFK_CUDA(h, launch_window_add_priors(w->dev, p->mf, p->fp_lists.ptr, p->fp_lists.ptr + p->K + 1, p->frows.ptr,
                                         p->delta.ptr, buf, h->stream),
             what);
    h->launches += 1;
  }
  if (w->kp.num_priors > 0) {
    DFK_CUDA(h, launch_window_add_keyframe_priors(w->dev, w->kp, p->kfrows.ptr, p->delta.ptr + (size_t)p->mf * p->B, buf,
                                                  h->stream),
             what);
    h->launches += 1;
  }
  return DFK_OK;
}

WindowEnergyDev energy_args(const DfkWindowProblem* p, const double* state, double w)
{
  WindowEnergyDev a{};
  a.B = p->B;
  a.err_out = reinterpret_cast<const float2*>(p->err_out.ptr);
  a.areas = p->sub_err ? p->areas_sub.ptr : p->areas.ptr;
  a.num_error = p->sub_err ? p->nea : p->ne; a.num_rep = p->nr; a.num_geo = p->ng;
  a.num_frame_priors = p->mf; a.frame_rows = p->frows.ptr; a.frame_delta = p->delta.ptr;
  a.num_kf_priors = p->w->kp.num_priors; a.kf_rows = p->kfrows.ptr; a.kf_row_off = p->w->kp.off;
  a.kf_mem_ptr = p->w->kp.mem_ptr; a.kf_delta = p->delta.ptr + (size_t)p->mf * p->B;
  a.codes = state + (size_t)(p->K + p->F) * 7;
  a.num_codes = p->K * p->C;
  a.code_prior_weight = w;
  a.out = p->energy();
  return a;
}

// the energy at `state` without linearising into p->energy() (E + 1/2 w |c|^2 in slot 7)
DfkStatus problem_error(DfkHandle h, DfkWindowProblem* p, const double* state, double w)
{
  const char* what = "[WindowProblem::error] kernel launch failed";
  DFK_CUDA(h, launch_window_repose(repose_args(p, state), h->stream), what);
  h->launches += 1;
  const float avg = p->avg_dpt;
  if (p->ndep > 0) {
    DFK_CUDA(h, launch_update_depth_batch(p->C, reinterpret_cast<const DepthDecodeDesc*>(p->depth.ptr), p->ndep,
                                          p->depth_max_blocks, avg, h->stream),
             what);
    h->launches += 1;
  }
  float* out = p->err_out.ptr;
  // with an active subset only its items are evaluated, and their rows come first (energy_args reads as many)
  const int ne = p->sub_err ? p->nea : p->ne;
  if (ne > 0) {
    const char* sw = "[WindowProblem::error] scratch allocation failed";
    DFK_CUDA(h, h->eval_partials.ensure((size_t)p->err_rows * 32), sw);
    if (h->eval_counters.cap < (size_t)p->ne) {
      DFK_CUDA(h, h->eval_counters.ensure((size_t)p->ne), sw);
      DFK_CUDA(h, cudaMemsetAsync(h->eval_counters.ptr, 0, sizeof(unsigned int) * h->eval_counters.cap, h->stream), sw);
    }
    DFK_CUDA(h, launch_eval_error_batch(p->sub_err ? p->err_sub.ptr : p->err.ptr, ne, p->err_max_blocks,
                                        p->huber_delta, h->eval_partials.ptr, h->eval_counters.ptr, out, h->stream),
             what);
    h->launches += 1;
  }
  if (p->nr > 0) {
    const float2* q = reinterpret_cast<const float2*>(p->rep_payload);
    DFK_CUDA(h, launch_reprojection_error(p->C, reinterpret_cast<const ReprojItemDev*>(p->rep.ptr), p->nr, q,
                                          q + p->rep_total, avg, out + 2 * (size_t)ne, h->stream),
             what);
    h->launches += 1;
  }
  if (p->ng > 0) {
    DFK_CUDA(h, launch_sparse_geometric_error(p->C, reinterpret_cast<const GeoItemDev*>(p->geo.ptr), p->ng,
                                              reinterpret_cast<const int2*>(p->geo_payload), avg,
                                              out + 2 * (size_t)(ne + p->nr), h->stream),
             what);
    h->launches += 1;
  }
  DFK_TRY(problem_deltas(h, p, state));
  DFK_CUDA(h, launch_window_energy(energy_args(p, state, w), h->stream), what);
  h->launches += 1;
  return DFK_OK;
}

// the active subsets of a validated mask (em: one byte per error item): the selected templates, their slots and the
// subset's tile plan, uploaded on the stream behind every launch still reading the previous ones.  The subset arrays
// are allocated once at full size, so no later mask reallocates an array a queued launch reads
DfkStatus problem_set_active(DfkHandle h, DfkWindowProblem* p, const uint8_t* dm, const uint8_t* em)
{
  const char* amsg = "[WindowProblem::set_active] allocation failed";
  const char* umsg = "[WindowProblem::set_active] upload failed";
  const int nd = p->nd, ne = p->ne;
  const bool all_d = std::all_of(dm, dm + nd, [](uint8_t v) { return v != 0; });
  const bool all_e = std::all_of(em, em + ne, [](uint8_t v) { return v != 0; });
  if (!all_d || !all_e) {
    DFK_CUDA(h, p->sub_slots.ensure((size_t)std::max(nd + ne, 1)), amsg);
    if (!all_d) {
      DFK_CUDA(h, p->dense_sub.ensure((size_t)std::max(nd, 1)), amsg);
      DFK_CUDA(h, p->rec_src.ensure((size_t)nd), amsg);
      DFK_CUDA(h, p->sub_records.ensure((size_t)nd * DFK_SFM_RECORD_FLOATS(p->C)), amsg);
    }
    if (!all_e) {
      DFK_CUDA(h, p->err_sub.ensure((size_t)std::max(ne, 1)), amsg);
      DFK_CUDA(h, p->areas_sub.ensure((size_t)std::max(ne, 1)), amsg);
    }
  }
  if (!all_d) {
    std::vector<SfmItemDev> items;
    std::vector<int4> sl;
    std::vector<int> src(nd, -1);
    for (int i = 0; i < nd; ++i)
      if (dm[i]) {
        src[i] = (int)items.size();
        items.push_back(p->dense_tmpl[i]);
        sl.push_back(p->slots_tmpl[i]);
      }
    plan_tiles(items.data(), (int)items.size(), p->step.max_ctas, &p->sub_plan);
    if (!items.empty()) {
      DFK_CUDA(h, cudaMemcpyAsync(p->dense_sub.ptr, items.data(), sizeof(SfmItemDev) * items.size(),
                                  cudaMemcpyHostToDevice, h->stream),
               umsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->sub_slots.ptr, sl.data(), sizeof(int4) * sl.size(), cudaMemcpyHostToDevice,
                                  h->stream),
               umsg);
    }
    DFK_CUDA(h, cudaMemcpyAsync(p->rec_src.ptr, src.data(), sizeof(int) * nd, cudaMemcpyHostToDevice, h->stream), umsg);
    p->nda = (int)items.size();
  }
  if (!all_e) {
    std::vector<EvalErrorDesc> items;
    std::vector<int4> sl;
    std::vector<double> areas;
    for (int i = 0; i < ne; ++i)
      if (em[i]) {
        items.push_back(p->err_tmpl[i]);
        sl.push_back(p->slots_tmpl[nd + i]);
        areas.push_back(p->areas_tmpl[i]);
      }
    if (!items.empty()) {
      DFK_CUDA(h, cudaMemcpyAsync(p->err_sub.ptr, items.data(), sizeof(EvalErrorDesc) * items.size(),
                                  cudaMemcpyHostToDevice, h->stream),
               umsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->sub_slots.ptr + nd, sl.data(), sizeof(int4) * sl.size(), cudaMemcpyHostToDevice,
                                  h->stream),
               umsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->areas_sub.ptr, areas.data(), sizeof(double) * areas.size(),
                                  cudaMemcpyHostToDevice, h->stream),
               umsg);
    }
    p->nea = (int)items.size();
  }
  p->sub_dense = !all_d;
  p->sub_err = !all_e;
  return DFK_OK;
}

// dfk_window_lm's device half (the Ops of dfk_lm.h / dfk_levels.h): the state, buffers and solve of a problem
struct ProblemLMOps {
  DfkHandle h;
  DfkWindowProblem* p;
  const DfkLMParams* prm;
  WindowSolverDev* solver;
  size_t nf, f_off;
  double w;
  int cand() const { return 1 - p->cur; }
  float* buf(bool c) const { return p->bufs.ptr + (size_t)(c ? 1 - p->acc : p->acc) * nf; }
  DfkStatus linearize(bool c) { return problem_linearize(h, p, p->st(c ? cand() : p->cur), buf(c)); }
  DfkStatus energy(bool c, double* f)
  {
    const double* s = p->st(c ? cand() : p->cur);
    if (prm->use_error) {
      DFK_TRY(problem_error(h, p, s, w));
    } else {
      WindowEnergyDev a = energy_args(p, s, w);
      a.buf_f = buf(c) + f_off;
      a.num_frame_priors = a.num_kf_priors = 0;
      DFK_CUDA(h, launch_window_energy(a, h->stream), "[WindowLM] kernel launch failed");
      h->launches += 1;
    }
    DFK_TRY(download(h, p->small_host.ptr, p->energy(), 8 * sizeof(double), "[WindowLM] read-back failed",
                     "[WindowLM] kernel failed"));
    *f = reinterpret_cast<const double*>(p->small_host.ptr)[7];
    return DFK_OK;
  }
  DfkStatus solve(double lam, int* info)
  {
    DFK_CUDA(h, launch_window_solve(solver, buf(false), lam, w, p->st(p->cur) + (size_t)(p->K + p->F) * 7, p->dx.ptr,
                                    p->info(), h->stream, &h->launches, true),
             "[WindowLM] solve launch failed");
    DFK_TRY(download(h, p->small_host.ptr, p->info(), sizeof(int32_t), "[WindowLM] read-back failed",
                     "[WindowLM] solve failed"));
    *info = *reinterpret_cast<const int32_t*>(p->small_host.ptr);
    return DFK_OK;
  }
  DfkStatus retract()
  {
    DFK_CUDA(h, launch_window_retract(p->st(p->cur), p->st(cand()), p->dx.ptr, p->K, p->F, p->C, h->stream),
             "[WindowLM] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  }
  void accept()
  {
    p->cur = cand();
    p->acc = 1 - p->acc;
  }
};

// dfk_window_lm's checks of the parameters and trace, and the solver, buffers and Ops of a run
DfkStatus lm_setup(DfkHandle h, DfkWindowProblem* p, const DfkLMParams* prm, DfkLMTrace* tr, const char* name,
                   ProblemLMOps* ops)
{
  const std::string what = std::string("[") + name + "] ";
  if (!p || !prm || !tr || !tr->energy || (prm->iterations > 0 && (!tr->lambda || !tr->accepted)))
    return fail(h, DFK_ERR_INVALID_ARG, what + "null argument");
  if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, what + "problem and handle live on different devices");
  if (prm->iterations < 0 || !(std::isfinite(prm->lambda_init) && prm->lambda_init >= 0.0) ||
      !(std::isfinite(prm->code_prior_weight) && prm->code_prior_weight >= 0.0))
    return fail(h, DFK_ERR_INVALID_ARG, what + "iterations < 0, or lambda_init / code_prior_weight not finite and >= 0");
  if (!(std::isfinite(prm->lambda_up) && prm->lambda_up > 0.0) ||
      !(std::isfinite(prm->lambda_down) && prm->lambda_down > 0.0) || std::isnan(prm->lambda_max))
    return fail(h, DFK_ERR_INVALID_ARG, what + "lambda_up / lambda_down must be finite and > 0, lambda_max a number");
  const int fix = prm->fix_first_pose ? 1 : 0;
  const std::string amsg = what + "allocation failed";
  if (!p->solver[fix])
    DFK_CUDA(h, window_solver_create(p->K, p->C, p->F, p->w->pair_k0, p->w->pair_k1, p->w->link_k0, p->w->link_k1,
                                     p->w->blk_i, p->w->blk_j, p->w->kp.block_off, std::vector<int>(), &p->solver[0]),
             amsg.c_str());
  const size_t nf = p->w->floats, f_off = (size_t)p->K * p->B * (p->B + 1) + (size_t)p->w->dev.num_pairs * 6 * p->B;
  DFK_CUDA(h, p->bufs.ensure(2 * nf), amsg.c_str());
  DFK_CUDA(h, p->dx.ensure((size_t)p->K * p->B + 6 * (size_t)p->F), amsg.c_str());
  *ops = ProblemLMOps{h, p, prm, p->solver[fix], nf, f_off, prm->code_prior_weight};
  return DFK_OK;
}

bool slot_ok(int s, int lo, int hi) { return s >= lo && s < hi; }

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
    // DenseSfm_EvaluateError uses FindCorrespondence defaults: border 1, min_dpt 0 (dense_sfm.h:91)
    const PixelCam pc = make_pixel_cam(p10, cam, 1, 0.0f);
    DFK_CUDA(h, launch_eval_error(pc, h->params.sfmparams.huber_delta, (int)W, (int)H, view_of(img0), view_of(img1),
                                  view_of(dpt0), h->simple_scratch.ptr, h->counter.ptr, h->out_dev.ptr, h->stream),
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
    h->eval_host.resize(n);
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
      EvalErrorDesc& d = h->eval_host[i];
      float p10[7];
      relative_pose(w.pose1, w.pose0, p10, nullptr, nullptr);
      d.pc = make_pixel_cam(p10, &w.cam, 1, 0.0f);  // as dfk_sfm_evaluate_error: border 1, min_dpt 0 (dense_sfm.h:91)
      d.img0 = view_of(&w.img0); d.img1 = view_of(&w.img1); d.dpt0 = view_of(&w.dpt0);
      d.width = (int)W;
      d.height = (int)H;
      d.nblocks = eval_error_blocks(d.width, d.height);
      d.scratch_row = rows;
      rows += d.nblocks;
      max_blocks = std::max(max_blocks, d.nblocks);
    }
    DeviceGuard guard(h->device);
    DFK_CUDA(h, h->eval_descs.ensure((size_t)n), "[SfmAligner::EvaluateError batch] scratch allocation failed");
    DFK_CUDA(h, h->eval_partials.ensure((size_t)rows * 32), "[SfmAligner::EvaluateError batch] scratch allocation failed");
    if (h->eval_counters.cap < (size_t)n) {
      DFK_CUDA(h, h->eval_counters.ensure((size_t)n), "[SfmAligner::EvaluateError batch] scratch allocation failed");
      DFK_CUDA(h, cudaMemsetAsync(h->eval_counters.ptr, 0, sizeof(unsigned int) * h->eval_counters.cap, h->stream),
               "[SfmAligner::EvaluateError batch] memset failed");
    }
    DFK_CUDA(h, cudaMemcpyAsync(h->eval_descs.ptr, h->eval_host.data(), sizeof(EvalErrorDesc) * n,
                                cudaMemcpyHostToDevice, h->stream),
             "[SfmAligner::EvaluateError batch] upload failed");
    DFK_CUDA(h, launch_eval_error_batch(h->eval_descs.ptr, n, max_blocks, h->params.sfmparams.huber_delta,
                                        h->eval_partials.ptr, h->eval_counters.ptr, out_dev, h->stream),
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
    const PixelCam pc = make_pixel_cam(se3, cam, 1, 0.0f);  // lucas_kanade_se3.h:52 defaults
    const View g = view_of(grad1);
    const bool galigned = aligned(g.ptr, 8) && g.pitch % 2 == 0;
    DFK_CUDA(h, launch_se3_step(pc, h->se3_huber_delta, (int)W, (int)H, view_of(img0), view_of(img1), view_of(dpt0), g,
                                galigned, h->simple_scratch.ptr, h->counter.ptr, h->out_dev.ptr, h->stream),
             "[SE3Aligner::RunStep] Kernel launch failed");
    DFK_TRY(fetch_out(h, 29, "[SE3Aligner::RunStep] Kernel launch failed"));
    unpack_record(h->out_host.ptr, 21, 6, JtJ, Jtr, residual, inliers);
    return DFK_OK;
  });
}

DfkStatus dfk_se3_track(DfkHandle h, float pose_ck[7], const DfkTrackLevel* levels, int num_levels,
                        float* inlier_fraction, float* error, float* last_system, float* history, int history_capacity)
{
  return guarded(h, [&] {
    if (!pose_ck || !levels || num_levels <= 0)
      return fail(h, DFK_ERR_INVALID_ARG, "[CameraTracker::TrackFrame] null argument / no pyramid levels");
    int total_iters = 0;
    for (int l = 0; l < num_levels; ++l) {
      if (!track_level_ok(levels[l]))
        return fail(h, DFK_ERR_INVALID_ARG,
                    "[CameraTracker::TrackFrame] inconsistent image views / camera larger than them / negative iteration count at level " +
                        std::to_string(l));
      total_iters += levels[l].iterations;
    }
    if (history && history_capacity < total_iters)
      return fail(h, DFK_ERR_INVALID_ARG, "[CameraTracker::TrackFrame] history buffer too small");
    DeviceGuard guard(h->device);
    const size_t nfloat = 8 + 36 * (size_t)std::max(total_iters, 1);
    DFK_CUDA(h, h->track_dev.ensure(nfloat), "[CameraTracker::TrackFrame] scratch allocation failed");
    DFK_CUDA(h, h->track_host.ensure(nfloat + 32), "[CameraTracker::TrackFrame] pinned allocation failed");
    float* track_dev = h->track_dev.ptr;
    float* track_host = h->track_host.ptr;
    // the pose goes to the device once; every iteration reads it there and its last block writes the update
    memcpy(track_host, pose_ck, sizeof(float) * 7);
    DFK_CUDA(h, cudaMemcpyAsync(track_dev, track_host, sizeof(float) * 7, cudaMemcpyHostToDevice, h->stream),
             "[CameraTracker::TrackFrame] pose upload failed");
    DFK_CUDA(h, cudaMemsetAsync(h->out_dev.ptr, 0, sizeof(float) * 32, h->stream), "[CameraTracker::TrackFrame] memset failed");
    int it = 0;
    for (int l = num_levels - 1; l >= 0; --l) {  // coarse to fine (camera_tracker.cpp:48)
      const DfkTrackLevel& L = levels[l];
      const PixelCam pc = make_pixel_cam(pose_ck, &L.cam, 1, 0.0f);  // q/t are overridden by the device pose
      const View g = view_of(&L.grad1);
      const bool galigned = aligned(g.ptr, 8) && g.pitch % 2 == 0;
      for (int k = 0; k < L.iterations; ++k, ++it) {
        DFK_CUDA(h, launch_se3_step(pc, h->se3_huber_delta, (int)L.img0.width, (int)L.img0.height, view_of(&L.img0),
                                    view_of(&L.img1), view_of(&L.dpt0), g, galigned, h->simple_scratch.ptr,
                                    h->counter.ptr, h->out_dev.ptr, h->stream, track_dev, track_dev + 8 + 36 * (size_t)it),
                 "[CameraTracker::TrackFrame] kernel launch failed");
        h->launches += 1;
      }
    }
    // one read-back: final pose, the last evaluated system, the per-iteration history
    float* host_sys = track_host + nfloat;
    DFK_CUDA(h, cudaMemcpyAsync(track_host, track_dev, sizeof(float) * (8 + 36 * (size_t)total_iters),
                                cudaMemcpyDeviceToHost, h->stream),
             "[CameraTracker::TrackFrame] read-back failed");
    DFK_TRY(download(h, host_sys, h->out_dev.ptr, sizeof(float) * 29, "[CameraTracker::TrackFrame] read-back failed",
                     "[CameraTracker::TrackFrame] stream synchronize failed"));
    memcpy(pose_ck, track_host, sizeof(float) * 7);
    track_outputs(host_sys, levels[0], inlier_fraction, error, last_system);
    if (history) memcpy(history, track_host + 8, sizeof(float) * 36 * (size_t)total_iters);
    return DFK_OK;
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
    const int N = num_problems, L = num_levels;
    std::vector<Se3TrackDesc> descs((size_t)L * N);  // level-major: a launch reads the N descriptors of its level
    std::vector<int> level_blocks(L, 0);             // grid width of a level: its largest problem
    int stride = 1;                                  // partial rows per problem
    for (int n = 0; n < N; ++n) {
      for (int l = 0; l < L; ++l) {
        const DfkTrackLevel& T = levels[(size_t)n * L + l];
        if (!track_level_ok(T))
          return fail(h, DFK_ERR_INVALID_ARG,
                      "[CameraTracker::TrackFrame batch] inconsistent image views / camera larger than them / "
                      "negative iteration count at problem " + std::to_string(n) + " level " + std::to_string(l));
        // the problems advance in lockstep, one launch per iteration for all of them
        if (T.iterations != levels[l].iterations)
          return fail(h, DFK_ERR_INVALID_ARG,
                      "[CameraTracker::TrackFrame batch] problem " + std::to_string(n) + " has " +
                          std::to_string(T.iterations) + " iterations at level " + std::to_string(l) +
                          ", problem 0 has " + std::to_string(levels[l].iterations));
        Se3TrackDesc& d = descs[(size_t)l * N + n];
        d.pc = make_pixel_cam(poses_ck + 7 * (size_t)n, &T.cam, 1, 0.0f);  // q/t are overridden by the device pose
        d.img0 = view_of(&T.img0); d.img1 = view_of(&T.img1); d.dpt0 = view_of(&T.dpt0); d.grad1 = view_of(&T.grad1);
        d.width = (int)T.img0.width;
        d.height = (int)T.img0.height;
        d.nblocks = se3_step_blocks(d.width, d.height);
        d.grad_aligned = aligned(d.grad1.ptr, 8) && d.grad1.pitch % 2 == 0;
        level_blocks[l] = std::max(level_blocks[l], d.nblocks);
        stride = std::max(stride, d.nblocks);
      }
    }
    DeviceGuard guard(h->device);
    const size_t desc_bytes = (descs.size() * sizeof(Se3TrackDesc) + 15) & ~(size_t)15;
    const size_t pose_bytes = sizeof(float) * 8 * (size_t)N, out_bytes = sizeof(float) * 32 * (size_t)N;
    const size_t total = desc_bytes + pose_bytes + out_bytes;
    DFK_CUDA(h, h->batch_dev.ensure(total), "[CameraTracker::TrackFrame batch] scratch allocation failed");
    DFK_CUDA(h, h->batch_partials.ensure((size_t)N * stride * 32),
             "[CameraTracker::TrackFrame batch] scratch allocation failed");
    if (h->batch_counters.cap < (size_t)N) {
      DFK_CUDA(h, h->batch_counters.ensure((size_t)N), "[CameraTracker::TrackFrame batch] scratch allocation failed");
      DFK_CUDA(h, cudaMemsetAsync(h->batch_counters.ptr, 0, sizeof(unsigned int) * h->batch_counters.cap, h->stream),
               "[CameraTracker::TrackFrame batch] memset failed");
    }
    DFK_CUDA(h, h->batch_host.ensure(total), "[CameraTracker::TrackFrame batch] pinned allocation failed");
    // one upload: every level's descriptors and the start poses
    memcpy(h->batch_host.ptr, descs.data(), descs.size() * sizeof(Se3TrackDesc));
    float* host_poses = reinterpret_cast<float*>(h->batch_host.ptr + desc_bytes);
    const float* host_outs = host_poses + 8 * (size_t)N;
    for (int n = 0; n < N; ++n) {
      memcpy(host_poses + 8 * (size_t)n, poses_ck + 7 * (size_t)n, sizeof(float) * 7);
      host_poses[8 * (size_t)n + 7] = 0.0f;
    }
    DFK_CUDA(h, cudaMemcpyAsync(h->batch_dev.ptr, h->batch_host.ptr, desc_bytes + pose_bytes, cudaMemcpyHostToDevice,
                                h->stream),
             "[CameraTracker::TrackFrame batch] upload failed");
    const Se3TrackDesc* descs_dev = reinterpret_cast<const Se3TrackDesc*>(h->batch_dev.ptr);
    float* poses_dev = reinterpret_cast<float*>(h->batch_dev.ptr + desc_bytes);
    float* outs_dev = poses_dev + 8 * (size_t)N;
    DFK_CUDA(h, cudaMemsetAsync(outs_dev, 0, out_bytes, h->stream), "[CameraTracker::TrackFrame batch] memset failed");
    for (int l = L - 1; l >= 0; --l) {  // coarse to fine (camera_tracker.cpp:48)
      for (int k = 0; k < levels[l].iterations; ++k) {
        DFK_CUDA(h, launch_se3_track_batch(descs_dev + (size_t)l * N, N, level_blocks[l], h->se3_huber_delta,
                                           h->batch_partials.ptr, stride, h->batch_counters.ptr, outs_dev, poses_dev,
                                           h->stream),
                 "[CameraTracker::TrackFrame batch] kernel launch failed");
        h->launches += 1;
      }
    }
    // one read-back: final poses and last evaluated systems
    DFK_TRY(download(h, host_poses, poses_dev, pose_bytes + out_bytes, "[CameraTracker::TrackFrame batch] read-back failed",
                     "[CameraTracker::TrackFrame batch] stream synchronize failed"));
    for (int n = 0; n < N; ++n) {
      memcpy(poses_ck + 7 * (size_t)n, host_poses + 8 * (size_t)n, sizeof(float) * 7);
      track_outputs(host_outs + 32 * (size_t)n, levels[(size_t)n * L], inlier_fraction ? inlier_fraction + n : nullptr,
                    error ? error + n : nullptr, last_systems ? last_systems + 29 * (size_t)n : nullptr);
    }
    return DFK_OK;
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
    DFK_CUDA(h, launch_update_depth(h->code_dev.ptr, code_size, (int)W, (int)H, view_of(prx_orig), view_of(prx_jac),
                                    avg_dpt, (float*)dpt_out->ptr, (uint32_t)(dpt_out->pitch_bytes / 4), h->stream),
             "[UpdateDepth] kernel launch failed");
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
    const size_t desc_bytes = (sizeof(DepthDecodeDesc) * (size_t)n + 15) & ~(size_t)15;
    const size_t total = desc_bytes + sizeof(float) * (size_t)n * code_size;
    DFK_CUDA(h, h->depth_dev.ensure(total), "[UpdateDepth batch] scratch allocation failed");
    h->depth_host.assign(total, 0);
    DepthDecodeDesc* descs = reinterpret_cast<DepthDecodeDesc*>(h->depth_host.data());
    float* codes = reinterpret_cast<float*>(h->depth_host.data() + desc_bytes);
    const float* codes_dev = reinterpret_cast<const float*>(h->depth_dev.ptr + desc_bytes);
    int max_blocks = 1;
    for (int i = 0; i < n; ++i) {
      const DfkDepthDecodeItem& it = items[i];
      DepthDecodeDesc& d = descs[i];
      d.prx = view_of(&it.prx_orig);
      d.jac = view_of(&it.prx_jac);
      d.dpt = static_cast<float*>(it.dpt.ptr);
      d.dpt_pitch = (uint32_t)(it.dpt.pitch_bytes / 4);
      d.code = codes_dev + (size_t)i * code_size;
      memcpy(codes + (size_t)i * code_size, it.code, sizeof(float) * code_size);
      d.width = (int)it.dpt.width;
      d.height = (int)it.dpt.height;
      d.nblocks = update_depth_blocks(d.width, d.height);
      d.vector = update_depth_vector(code_size, d.code, d.jac) ? 1 : 0;
      max_blocks = std::max(max_blocks, d.nblocks);
    }
    DFK_CUDA(h, cudaMemcpyAsync(h->depth_dev.ptr, h->depth_host.data(), total, cudaMemcpyHostToDevice, h->stream),
             "[UpdateDepth batch] upload failed");
    DFK_CUDA(h, launch_update_depth_batch(code_size, reinterpret_cast<const DepthDecodeDesc*>(h->depth_dev.ptr), n,
                                          max_blocks, h->params.sfmparams.avg_dpt, h->stream),
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
    DFK_CUDA(h, launch_sobel((int)W, (int)H, view_of(img), (float*)grad->ptr, (uint32_t)(grad->pitch_bytes / 4),
                             h->stream),
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
    DFK_CUDA(h, launch_blur_down((int)in->width, (int)in->height, view_of(in), (int)out->width, (int)out->height,
                                 (float*)out->ptr, (uint32_t)(out->pitch_bytes / 4), h->stream),
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

DfkStatus dfk_window_create(DfkHandle h, const DfkWindowDesc* d, DfkWindow** out)
{
  return dfk_window_create_geometric(h, d, 0, nullptr, nullptr, out);
}

DfkStatus dfk_window_create_geometric(DfkHandle h, const DfkWindowDesc* d, int L, const int32_t* link_k0,
                                      const int32_t* link_k1, DfkWindow** out)
{
  return dfk_window_create_frames(h, d, L, link_k0, link_k1, 0, out);
}

DfkStatus dfk_window_create_frames(DfkHandle h, const DfkWindowDesc* d, int L, const int32_t* link_k0,
                                   const int32_t* link_k1, int F, DfkWindow** out)
{
  return dfk_window_create_priors(h, d, L, link_k0, link_k1, F, 0, nullptr, nullptr, out);
}

DfkStatus dfk_window_create_priors(DfkHandle h, const DfkWindowDesc* d, int L, const int32_t* link_k0,
                                   const int32_t* link_k1, int F, int Q, const int32_t* prior_ptr,
                                   const int32_t* prior_kf, DfkWindow** out)
{
  return guarded(h, [&] {
    if (!d || !out || L < 0 || F < 0 || (L > 0 && (!link_k0 || !link_k1)) || Q < 0 ||
        (Q > 0 && (!prior_ptr || !prior_kf)))
      return fail(h, DFK_ERR_INVALID_ARG, "[Window] null argument");
    *out = nullptr;
    const int K = d->num_keyframes, P = d->num_pairs, n = d->num_items;
    if (K <= 0 || P <= 0 || n <= 0 || !d->pair_k0 || !d->pair_k1 || !d->item_pair || !d->item_width || !d->item_height)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window] empty window / null index array");
    if (!dfk_sfm_supports_code_size(d->code_size))
      return fail(h, DFK_ERR_UNSUPPORTED, "[Window] no RunStep kernel for code size " + std::to_string(d->code_size));
    // pair_k1 in [K, K + F): frame pair_k1 - K, which must be k1 of exactly this one pair
    std::vector<int> frame_pair(F, -1);
    for (int p = 0; p < P; ++p) {
      if (d->pair_k0[p] < 0 || d->pair_k0[p] >= K || d->pair_k1[p] < 0 || d->pair_k1[p] >= K + F)
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] pair " + std::to_string(p) + " names a keyframe outside the window");
      if (d->pair_k1[p] >= K) {
        if (frame_pair[d->pair_k1[p] - K] >= 0)
          return fail(h, DFK_ERR_INVALID_ARG, "[Window] frame " + std::to_string(d->pair_k1[p] - K) +
                                                  " is k1 of more than one pair");
        frame_pair[d->pair_k1[p] - K] = p;
      }
    }
    for (int f = 0; f < F; ++f)
      if (frame_pair[f] < 0)
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] frame " + std::to_string(f) + " is k1 of no pair");
    for (int i = 0; i < n; ++i)
      // a record is scaled (W, H > 0: photometric) or unscaled (0, 0: reprojection)
      if (d->item_pair[i] < 0 || d->item_pair[i] >= P ||
          !((d->item_width[i] > 0 && d->item_height[i] > 0) || (d->item_width[i] == 0 && d->item_height[i] == 0)))
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] record " + std::to_string(i) + " names a pair outside the window");
    for (int i = 0; i < n; ++i)
      if (d->pair_k1[d->item_pair[i]] >= K && d->item_width[i] == 0)
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] record " + std::to_string(i) + " of a frame pair is unscaled");
    for (int l = 0; l < L; ++l) {
      if (link_k0[l] < 0 || link_k0[l] >= K || link_k1[l] < 0 || link_k1[l] >= K)
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] link " + std::to_string(l) + " names a keyframe outside the window");
      if (link_k0[l] == link_k1[l])
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] link " + std::to_string(l) + " ties a keyframe to itself");
    }
    // keyframe priors: non-empty ascending lists of distinct keyframes of the window
    if (Q > 0 && prior_ptr[0] != 0) return fail(h, DFK_ERR_INVALID_ARG, "[Window] prior_ptr[0] must be 0");
    for (int q = 0; q < Q; ++q) {
      if (prior_ptr[q + 1] <= prior_ptr[q])
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] keyframe prior " + std::to_string(q) + " has no keyframe");
      for (int a = prior_ptr[q]; a < prior_ptr[q + 1]; ++a)
        if (prior_kf[a] < 0 || prior_kf[a] >= K || (a > prior_ptr[q] && prior_kf[a] <= prior_kf[a - 1]))
          return fail(h, DFK_ERR_INVALID_ARG, "[Window] keyframe prior " + std::to_string(q) +
                                                  " is not an ascending list of distinct keyframes of the window");
    }
    const int M = Q > 0 ? prior_ptr[Q] : 0;  // members of all priors
    // prior blocks: the distinct (i < j) of every prior, ascending; the entries of each keyframe and each block in
    // prior order
    std::vector<std::pair<int, int>> blocks;
    for (int q = 0; q < Q; ++q)
      for (int a = prior_ptr[q]; a < prior_ptr[q + 1]; ++a)
        for (int c = a + 1; c < prior_ptr[q + 1]; ++c) blocks.push_back({prior_kf[a], prior_kf[c]});
    std::sort(blocks.begin(), blocks.end());
    blocks.erase(std::unique(blocks.begin(), blocks.end()), blocks.end());
    const int NB = (int)blocks.size();
    std::vector<std::vector<int>> kf_ent(K), blk_ent(NB);
    for (int q = 0; q < Q; ++q)
      for (int a = prior_ptr[q]; a < prior_ptr[q + 1]; ++a) {
        kf_ent[prior_kf[a]].insert(kf_ent[prior_kf[a]].end(), {q, a - prior_ptr[q]});
        for (int c = a + 1; c < prior_ptr[q + 1]; ++c) {
          const int b = (int)(std::lower_bound(blocks.begin(), blocks.end(), std::make_pair(prior_kf[a], prior_kf[c])) -
                              blocks.begin());
          blk_ent[b].insert(blk_ent[b].end(), {q, a - prior_ptr[q], c - prior_ptr[q]});
        }
      }
    std::vector<int> kp_blob(Q + 1, 0);  // mem_ptr
    for (int q = 0; q < Q; ++q) kp_blob[q + 1] = prior_ptr[q + 1];
    const size_t o_kfp = kp_blob.size();
    kp_blob.push_back(0);
    for (int k = 0; k < K; ++k) kp_blob.push_back(kp_blob[o_kfp + k] + (int)kf_ent[k].size() / 2);
    const size_t o_bp = kp_blob.size();
    kp_blob.push_back(0);
    for (int b = 0; b < NB; ++b) kp_blob.push_back(kp_blob[o_bp + b] + (int)blk_ent[b].size() / 3);
    kp_blob.resize((kp_blob.size() + 3) & ~(size_t)3, 0);  // int2 / int3 entries 16-byte aligned
    const size_t o_ke = kp_blob.size();
    for (int k = 0; k < K; ++k) kp_blob.insert(kp_blob.end(), kf_ent[k].begin(), kf_ent[k].end());
    kp_blob.resize((kp_blob.size() + 3) & ~(size_t)3, 0);
    const size_t o_be = kp_blob.size();
    for (int b = 0; b < NB; ++b) kp_blob.insert(kp_blob.end(), blk_ent[b].begin(), blk_ent[b].end());
    std::vector<long long> poff(Q + 1, 0);
    for (int q = 0; q < Q; ++q)
      poff[q + 1] = poff[q] + (long long)DFK_KF_PRIOR_DOUBLES(d->code_size, prior_ptr[q + 1] - prior_ptr[q]);
    // one CSR list per key kind (keyframe k0, frame k1, pair): ptr[keys + 1], then the items of each key in item order
    // (the summation order of the gather kernel); an item whose key is outside [0, keys) is in no list.  Returns where
    // the list starts in blob
    std::vector<int> blob;
    auto add_csr = [&](int keys, int n, auto key_of) {
      const size_t o = blob.size();
      blob.resize(o + keys + 1 + n, 0);
      int* ptr = blob.data() + o;
      for (int i = 0; i < n; ++i)
        if (key_of(i) < keys) ptr[key_of(i) + 1] += 1;
      for (int k = 0; k < keys; ++k) ptr[k + 1] += ptr[k];
      std::vector<int> next(ptr, ptr + keys);
      for (int i = 0; i < n; ++i)
        if (key_of(i) < keys) ptr[keys + 1 + next[key_of(i)]++] = i;
      return o;
    };
    const size_t o_kf0 = add_csr(K, n, [&](int i) { return d->pair_k0[d->item_pair[i]]; });
    // a frame pair's pose1 is the frame's: its items go to the frame's block, not to a keyframe's
    const size_t o_kf1 = add_csr(K, n, [&](int i) { return d->pair_k1[d->item_pair[i]]; });
    const size_t o_pair = add_csr(P, n, [&](int i) { return d->item_pair[i]; });
    const size_t o_lk0 = add_csr(K, L, [&](int l) { return link_k0[l]; });
    const size_t o_lk1 = add_csr(K, L, [&](int l) { return link_k1[l]; });
    const size_t o_fr = blob.size();
    blob.insert(blob.end(), frame_pair.begin(), frame_pair.end());
    std::vector<float> areas(n);
    for (int i = 0; i < n; ++i) areas[i] = (float)d->item_width[i] * (float)d->item_height[i];

    DeviceGuard guard(h->device);
    std::unique_ptr<DfkWindow> w(new (std::nothrow) DfkWindow());  // freed under the guard if the upload fails
    if (!w) return oom(h);
    w->device = h->device;
    const char* upload_failed = "[Window] index upload failed";
    DFK_CUDA(h, w->ints.ensure(blob.size()), upload_failed);
    DFK_CUDA(h, w->areas.ensure(areas.size()), upload_failed);
    DFK_CUDA(h, cudaMemcpy(w->ints.ptr, blob.data(), blob.size() * sizeof(int), cudaMemcpyHostToDevice), upload_failed);
    DFK_CUDA(h, cudaMemcpy(w->areas.ptr, areas.data(), areas.size() * sizeof(float), cudaMemcpyHostToDevice), upload_failed);
    const int* ints = w->ints.ptr;
    w->dev.num_keyframes = K; w->dev.num_pairs = P; w->dev.num_items = n; w->dev.code_size = d->code_size;
    w->dev.kf0_ptr = ints + o_kf0; w->dev.kf0_items = ints + o_kf0 + K + 1;
    w->dev.kf1_ptr = ints + o_kf1; w->dev.kf1_items = ints + o_kf1 + K + 1;
    w->dev.pair_ptr = ints + o_pair; w->dev.pair_items = ints + o_pair + P + 1;
    w->dev.item_area = w->areas.ptr;
    w->dev.num_links = L;
    w->dev.lk0_ptr = ints + o_lk0; w->dev.lk0_links = ints + o_lk0 + K + 1;
    w->dev.lk1_ptr = ints + o_lk1; w->dev.lk1_links = ints + o_lk1 + K + 1;
    w->dev.num_frames = F;
    w->dev.frame_pair = ints + o_fr;
    const size_t B = 6 + (size_t)d->code_size;
    const size_t block_off = (size_t)K * (B * B + B) + (size_t)P * 6 * B + 2 + (size_t)L * B * B + (size_t)F * 42;
    w->floats = block_off + (size_t)NB * B * B;
    w->pair_k0.assign(d->pair_k0, d->pair_k0 + P);
    w->pair_k1.assign(d->pair_k1, d->pair_k1 + P);
    w->link_k0.assign(link_k0, link_k0 + L);
    w->link_k1.assign(link_k1, link_k1 + L);
    w->item_pair.assign(d->item_pair, d->item_pair + n);
    if (Q > 0) {
      w->prior_ptr.assign(prior_ptr, prior_ptr + Q + 1);
      w->prior_kf.assign(prior_kf, prior_kf + M);
      for (const auto& b : blocks) {
        w->blk_i.push_back(b.first);
        w->blk_j.push_back(b.second);
      }
      w->prior_off = poff;
      DFK_CUDA(h, w->kp_ints.ensure(kp_blob.size()), upload_failed);
      DFK_CUDA(h, w->kp_off.ensure(poff.size()), upload_failed);
      DFK_CUDA(h, cudaMemcpy(w->kp_ints.ptr, kp_blob.data(), kp_blob.size() * sizeof(int), cudaMemcpyHostToDevice),
               upload_failed);
      DFK_CUDA(h, cudaMemcpy(w->kp_off.ptr, poff.data(), poff.size() * sizeof(long long), cudaMemcpyHostToDevice),
               upload_failed);
      const int* kpi = w->kp_ints.ptr;
      w->kp.num_priors = Q; w->kp.num_blocks = NB; w->kp.block_off = block_off;
      w->kp.mem_ptr = kpi; w->kp.off = w->kp_off.ptr;
      w->kp.kf_ptr = kpi + o_kfp; w->kp.kf_ent = reinterpret_cast<const int2*>(kpi + o_ke);
      w->kp.blk_ptr = kpi + o_bp; w->kp.blk_ent = reinterpret_cast<const int3*>(kpi + o_be);
    }
    *out = w.release();
    return DFK_OK;
  });
}

DfkStatus dfk_window_destroy(DfkHandle /*h*/, DfkWindow* w)
{
  if (!w) return DFK_OK;
  DeviceGuard guard(w->device);
  delete w;
  return DFK_OK;
}

size_t dfk_window_floats(const DfkWindow* w) { return w ? w->floats : 0; }

DfkStatus dfk_window_assemble(DfkHandle h, const DfkWindow* w, const float* records_dev, float* window_dev)
{
  return guarded(h, [&] {
    if (!w || !records_dev || !window_dev) return fail(h, DFK_ERR_INVALID_ARG, "[Window] null argument");
    if (w->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[Window] window and handle live on different devices");
    if (w->dev.num_links > 0)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window] window has geometric links: assemble it with dfk_window_assemble_geometric");
    DeviceGuard guard(h->device);
    DFK_CUDA(h, launch_window_assemble(w->dev, records_dev, nullptr, window_dev, h->stream), "[Window] kernel launch failed");
    h->launches += 1;
    if (w->kp.num_blocks > 0)
      DFK_CUDA(h, cudaMemsetAsync(window_dev + w->kp.block_off, 0, (w->floats - w->kp.block_off) * sizeof(float),
                                  h->stream),
               "[Window] kernel launch failed");
    return DFK_OK;
  });
}

DfkStatus dfk_window_assemble_geometric(DfkHandle h, const DfkWindow* w, const float* records_dev,
                                        const float* geo_records_dev, float* window_dev)
{
  return guarded(h, [&] {
    if (!w || !records_dev || !window_dev) return fail(h, DFK_ERR_INVALID_ARG, "[Window] null argument");
    if (w->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[Window] window and handle live on different devices");
    if (w->dev.num_links > 0 && !geo_records_dev)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window] window has geometric links but no geometric records");
    DeviceGuard guard(h->device);
    DFK_CUDA(h, launch_window_assemble(w->dev, records_dev, geo_records_dev, window_dev, h->stream),
             "[Window] kernel launch failed");
    h->launches += 1;
    if (w->kp.num_blocks > 0)  // the prior blocks start at zero: dfk_window_add_keyframe_priors fills them
      DFK_CUDA(h, cudaMemsetAsync(window_dev + w->kp.block_off, 0, (w->floats - w->kp.block_off) * sizeof(float),
                                  h->stream),
               "[Window] kernel launch failed");
    return DFK_OK;
  });
}

DfkStatus dfk_window_marginalize_frames(DfkHandle h, const DfkWindow* w, const float* records_dev, int n,
                                        const int32_t* frames_host, double* priors_dev, int32_t* info_dev)
{
  return guarded(h, [&] {
    if (!w || !records_dev || n < 0 || (n > 0 && (!frames_host || !priors_dev || !info_dev)))
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::MarginalizeFrames] null argument");
    if (w->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::MarginalizeFrames] window and handle live on different devices");
    for (int i = 0; i < n; ++i)
      if (frames_host[i] < 0 || frames_host[i] >= w->dev.num_frames)
        return fail(h, DFK_ERR_INVALID_ARG, "[Window::MarginalizeFrames] frame " + std::to_string(frames_host[i]) +
                                                " is not a frame of the window");
    if (n == 0) return DFK_OK;
    DeviceGuard guard(h->device);
    const char* what = "[Window::MarginalizeFrames] index upload failed";
    DFK_CUDA(h, h->window_lists.ensure(n), what);
    // pageable source: staged before the call returns
    DFK_CUDA(h, cudaMemcpyAsync(h->window_lists.ptr, frames_host, sizeof(int) * n, cudaMemcpyHostToDevice, h->stream),
             what);
    DFK_CUDA(h, launch_window_marginalize_frames(w->dev, records_dev, n, h->window_lists.ptr, priors_dev, info_dev,
                                                 h->stream),
             "[Window::MarginalizeFrames] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_window_add_priors(DfkHandle h, const DfkWindow* w, int m, const int32_t* prior_kf_host,
                                const double* priors_dev, const double* delta_dev, float* window_dev)
{
  return guarded(h, [&] {
    if (!w || !window_dev || m < 0 || (m > 0 && (!prior_kf_host || !priors_dev || !delta_dev)))
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddPriors] null argument");
    if (w->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddPriors] window and handle live on different devices");
    const int K = w->dev.num_keyframes;
    for (int i = 0; i < m; ++i)
      if (prior_kf_host[i] < 0 || prior_kf_host[i] >= K)
        return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddPriors] prior " + std::to_string(i) +
                                                " names a keyframe outside the window");
    if (m == 0) return DFK_OK;
    // CSR of the priors per keyframe, in list order: ptr[K + 1] | indices[m]
    std::vector<int> lists(K + 1 + m, 0);
    for (int i = 0; i < m; ++i) lists[prior_kf_host[i] + 1] += 1;
    for (int k = 0; k < K; ++k) lists[k + 1] += lists[k];
    std::vector<int> next(lists.begin(), lists.begin() + K);
    for (int i = 0; i < m; ++i) lists[K + 1 + next[prior_kf_host[i]]++] = i;
    DeviceGuard guard(h->device);
    const char* what = "[Window::AddPriors] index upload failed";
    DFK_CUDA(h, h->window_lists.ensure(lists.size()), what);
    DFK_CUDA(h, cudaMemcpyAsync(h->window_lists.ptr, lists.data(), sizeof(int) * lists.size(), cudaMemcpyHostToDevice,
                                h->stream),
             what);
    DFK_CUDA(h, launch_window_add_priors(w->dev, m, h->window_lists.ptr, h->window_lists.ptr + K + 1, priors_dev,
                                         delta_dev, window_dev, h->stream),
             "[Window::AddPriors] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_window_add_keyframe_priors(DfkHandle h, const DfkWindow* w, const double* priors_dev,
                                         const double* delta_dev, float* window_dev)
{
  return guarded(h, [&] {
    if (!w || !window_dev) return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddKeyframePriors] null argument");
    if (w->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddKeyframePriors] window and handle live on different devices");
    if (w->kp.num_priors == 0) return DFK_OK;
    if (!priors_dev || !delta_dev) return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddKeyframePriors] null argument");
    DeviceGuard guard(h->device);
    DFK_CUDA(h, launch_window_add_keyframe_priors(w->dev, w->kp, priors_dev, delta_dev, window_dev, h->stream),
             "[Window::AddKeyframePriors] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

namespace {

// N(m): the keyframes that share a pair, a link or a keyframe prior with m, ascending
std::vector<int> window_blanket(const DfkWindow* w, int m)
{
  const int K = w->dev.num_keyframes;
  std::vector<char> in(K, 0);
  auto tie = [&](int a, int b) {
    if (a < K && b < K && (a == m || b == m)) in[a] = in[b] = 1;
  };
  for (size_t p = 0; p < w->pair_k0.size(); ++p) tie(w->pair_k0[p], w->pair_k1[p]);
  for (size_t l = 0; l < w->link_k0.size(); ++l) tie(w->link_k0[l], w->link_k1[l]);
  for (size_t q = 0; q + 1 < w->prior_ptr.size(); ++q) {
    const auto b = w->prior_kf.begin() + w->prior_ptr[q], e = w->prior_kf.begin() + w->prior_ptr[q + 1];
    if (std::find(b, e, m) != e)
      for (auto it = b; it != e; ++it) in[*it] = 1;
  }
  in[m] = 0;
  std::vector<int> out;
  for (int k = 0; k < K; ++k)
    if (in[k]) out.push_back(k);
  return out;
}

bool prior_contains(const DfkWindow* w, int q, int m)
{
  const auto b = w->prior_kf.begin() + w->prior_ptr[q], e = w->prior_kf.begin() + w->prior_ptr[q + 1];
  return std::find(b, e, m) != e;
}

}  // namespace

DfkStatus dfk_window_blanket(DfkHandle h, const DfkWindow* w, int m, int32_t* kf_out, int32_t* n)
{
  return guarded(h, [&] {
    if (!w || !kf_out || !n) return fail(h, DFK_ERR_INVALID_ARG, "[Window::Blanket] null argument");
    if (m < 0 || m >= w->dev.num_keyframes)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::Blanket] keyframe " + std::to_string(m) + " is not in the window");
    const std::vector<int> nb = window_blanket(w, m);
    std::copy(nb.begin(), nb.end(), kf_out);
    *n = (int32_t)nb.size();
    return DFK_OK;
  });
}

DfkStatus dfk_window_marginalize_keyframe(DfkHandle h, const DfkWindow* w, const float* records_dev,
                                          const float* geo_records_dev, int m, int num_frame_priors,
                                          const double* frame_priors_dev, const double* frame_delta_dev,
                                          const double* kf_priors_dev, const double* kf_delta_dev,
                                          double code_prior_weight, const double* code_m_host, double* prior_dev,
                                          int32_t* info_dev)
{
  return guarded(h, [&] {
    const char* what = "[Window::MarginalizeKeyframe] ";
    auto bad = [&](DfkStatus s, const std::string& msg) { return fail(h, s, what + msg); };
    if (!w || !records_dev || !prior_dev || !info_dev || num_frame_priors < 0 ||
        (num_frame_priors > 0 && (!frame_priors_dev || !frame_delta_dev)))
      return bad(DFK_ERR_INVALID_ARG, "null argument");
    if (w->device != h->device) return bad(DFK_ERR_INVALID_ARG, "window and handle live on different devices");
    const int K = w->dev.num_keyframes, C = w->dev.code_size, B = 6 + C;
    if (m < 0 || m >= K) return bad(DFK_ERR_INVALID_ARG, "keyframe " + std::to_string(m) + " is not in the window");
    if (w->dev.num_links > 0 && !geo_records_dev)
      return bad(DFK_ERR_INVALID_ARG, "window has geometric links but no geometric records");
    if (!(std::isfinite(code_prior_weight) && code_prior_weight >= 0.0))
      return bad(DFK_ERR_INVALID_ARG, "code_prior_weight must be finite and >= 0");
    if (code_prior_weight > 0.0 && !code_m_host) return bad(DFK_ERR_INVALID_ARG, "code_prior_weight > 0 needs m's code");
    for (size_t p = 0; p < w->pair_k0.size(); ++p)
      if (w->pair_k0[p] == m && w->pair_k1[p] >= K)
        return bad(DFK_ERR_INVALID_ARG, "keyframe " + std::to_string(m) + " still has tracked frames: marginalise them first");
    const int Q = w->kp.num_priors;
    std::vector<int> kq;  // the keyframe priors that contain m
    for (int q = 0; q < Q; ++q)
      if (prior_contains(w, q, m)) kq.push_back(q);
    if (!kq.empty() && (!kf_priors_dev || !kf_delta_dev))
      return bad(DFK_ERR_INVALID_ARG, "keyframe priors contain m but none were given");
    const std::vector<int> nb = window_blanket(w, m);
    const int n = (int)nb.size();
    if (n == 0) return bad(DFK_ERR_INVALID_ARG, "keyframe " + std::to_string(m) + " shares no factor with another");
    if (n > DFK_MAX_BLANKET)
      return bad(DFK_ERR_UNSUPPORTED, "blanket of " + std::to_string(n) + " keyframes (at most " +
                                          std::to_string(DFK_MAX_BLANKET) + ")");
    std::vector<int> loc(K, -1);
    loc[m] = 0;
    for (int i = 0; i < n; ++i) loc[nb[i]] = 1 + i;
    // [refs | tile_row | tile_col | mem_loc | pad | update tasks]
    std::vector<int> lists;
    for (size_t i = 0; i < w->item_pair.size(); ++i) {
      const int k0 = w->pair_k0[w->item_pair[i]], k1 = w->pair_k1[w->item_pair[i]];
      if (k1 < K && (k0 == m || k1 == m)) lists.insert(lists.end(), {0, (int)i, loc[k0], loc[k1]});
    }
    for (size_t l = 0; l < w->link_k0.size(); ++l)
      if (w->link_k0[l] == m || w->link_k1[l] == m)
        lists.insert(lists.end(), {1, (int)l, loc[w->link_k0[l]], loc[w->link_k1[l]]});
    for (int i = 0; i < num_frame_priors; ++i) lists.insert(lists.end(), {2, i, 0, 0});
    for (int q : kq) lists.insert(lists.end(), {3, q, 0, 0});
    const int num_refs = (int)lists.size() / 4;
    const int T = n + 1 + n * (n + 1) / 2;
    const size_t o_tr = lists.size();
    for (int t = 0; t <= n; ++t) lists.push_back(t);
    for (int I = 1; I <= n; ++I)
      for (int J = 1; J <= I; ++J) lists.push_back(I);
    const size_t o_tc = lists.size();
    for (int t = 0; t <= n; ++t) lists.push_back(0);
    for (int I = 1; I <= n; ++I)
      for (int J = 1; J <= I; ++J) lists.push_back(J);
    const size_t o_ml = lists.size();
    for (int kf : w->prior_kf) lists.push_back(loc[kf]);
    lists.resize((lists.size() + 3) & ~(size_t)3, 0);
    const size_t o_tk = lists.size();
    std::vector<int> tasks;
    window_eliminate_first_tasks(n, tasks);
    lists.insert(lists.end(), tasks.begin(), tasks.end());
    const size_t ws = (size_t)(T + 1) * B * B + (size_t)(n + 1) * B + 1;

    DeviceGuard guard(h->device);
    const char* alloc = "[Window::MarginalizeKeyframe] scratch allocation failed";
    DFK_CUDA(h, h->marg_lists.ensure(lists.size()), alloc);
    DFK_CUDA(h, h->marg_dev.ensure(ws), alloc);
    DFK_CUDA(h, h->marg_code.ensure(C), alloc);
    // pageable sources: staged before the call returns
    DFK_CUDA(h, cudaMemcpyAsync(h->marg_lists.ptr, lists.data(), lists.size() * sizeof(int), cudaMemcpyHostToDevice,
                                h->stream), alloc);
    if (code_prior_weight > 0.0)
      DFK_CUDA(h, cudaMemcpyAsync(h->marg_code.ptr, code_m_host, C * sizeof(double), cudaMemcpyHostToDevice, h->stream),
               alloc);
    const int* li = h->marg_lists.ptr;
    KfMargDev md{};
    md.n = n;
    md.num_refs = num_refs;
    md.refs = reinterpret_cast<const KfMargRef*>(li);
    md.tile_row = li + o_tr; md.tile_col = li + o_tc; md.mem_loc = li + o_ml;
    md.records = records_dev; md.geo = geo_records_dev;
    md.fpriors = frame_priors_dev; md.fdelta = frame_delta_dev;
    md.kpriors = kf_priors_dev; md.kdelta = kf_delta_dev;
    md.w = code_prior_weight; md.code = h->marg_code.ptr;
    md.tiles = h->marg_dev.ptr;
    md.rhs = md.tiles + (size_t)(T + 1) * B * B;
    md.f = md.rhs + (size_t)(n + 1) * B;
    md.info = info_dev;
    const char* launch = "[Window::MarginalizeKeyframe] kernel launch failed";
    DFK_CUDA(h, launch_window_marg_gather(w->dev, w->kp, md, T, h->stream), launch);
    DFK_CUDA(h, launch_window_eliminate_first(C, n, md.tiles, md.rhs, info_dev, li + o_tk, (int)tasks.size() / 4,
                                              h->stream), launch);
    DFK_CUDA(h, launch_window_marg_finalize(C, md, T, prior_dev, h->stream), launch);
    h->launches += 4;
    return DFK_OK;
  });
}

DfkStatus dfk_window_solver_create(DfkHandle h, const DfkWindow* w, int num_fixed, const int32_t* fixed_vars,
                                   DfkWindowSolver** out)
{
  return guarded(h, [&] {
    if (!w || !out || num_fixed < 0 || (num_fixed > 0 && !fixed_vars))
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] null argument");
    *out = nullptr;
    if (w->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] window and handle live on different devices");
    const int K = w->dev.num_keyframes, C = w->dev.code_size, n = K * (6 + C);
    std::vector<int> fixed(fixed_vars, fixed_vars + num_fixed);
    std::vector<char> seen(n, 0);
    for (int q = 0; q < num_fixed; ++q) {
      if (fixed[q] < 0 || fixed[q] >= n)
        return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] fixed variable " + std::to_string(fixed[q]) +
                                                " outside the window's " + std::to_string(n) + " variables");
      if (seen[fixed[q]]++)
        return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] fixed variable " + std::to_string(fixed[q]) + " listed twice");
    }
    DeviceGuard guard(h->device);
    std::unique_ptr<DfkWindowSolver> s(new (std::nothrow) DfkWindowSolver());
    if (!s) return oom(h);
    s->device = h->device;
    s->num_vars = n; s->code_size = C; s->num_keyframes = K;
    DFK_CUDA(h, window_solver_create(K, C, w->dev.num_frames, w->pair_k0, w->pair_k1, w->link_k0, w->link_k1, w->blk_i,
                                     w->blk_j, w->kp.block_off, fixed, &s->dev),
             "[WindowSolver] workspace allocation failed");
    *out = s.release();
    return DFK_OK;
  });
}

DfkStatus dfk_window_solver_destroy(DfkHandle h, DfkWindowSolver* s)
{
  return guarded(h, [&] {
    if (!s) return DFK_OK;
    DeviceGuard guard(s->device);
    delete s;
    return DFK_OK;
  });
}

DfkStatus dfk_window_solver_tiles(DfkHandle h, const DfkWindowSolver* s, size_t* tiles)
{
  return guarded(h, [&] {
    if (!s || !tiles) return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] null argument");
    *tiles = window_solver_tiles(s->dev);
    return DFK_OK;
  });
}

DfkStatus dfk_window_solve(DfkHandle h, const DfkWindowSolver* s, const float* window_dev, const DfkWindowSolveParams* p,
                           const double* codes, double* dx_dev, int32_t* info_dev)
{
  return guarded(h, [&] {
    if (!s || !window_dev || !p || !dx_dev || !info_dev)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] null argument");
    if (s->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] solver and handle live on different devices");
    if (!(std::isfinite(p->lambda) && p->lambda >= 0.0))
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] lambda must be finite and >= 0");
    if (!(std::isfinite(p->code_prior_weight) && p->code_prior_weight >= 0.0))
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] code_prior_weight must be finite and >= 0");
    if (p->code_prior_weight > 0.0 && !codes)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] code_prior_weight > 0 needs the codes");
    DeviceGuard guard(h->device);
    DFK_CUDA(h, launch_window_solve(s->dev, window_dev, p->lambda, p->code_prior_weight, codes, dx_dev, info_dev,
                                    h->stream, &h->launches),
             "[WindowSolver] kernel launch failed");
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

DfkStatus dfk_reprojection_linearize(DfkHandle h, const float pose0[7], const float pose1[7], const float* code0,
                                     int code_size, const DfkCamera* cam, const DfkImage* prx_orig, const DfkImage* prx_jac,
                                     int num_matches, const float* query_xy, const float* train_xy, float cauchy_delta,
                                     float sigma, float* rows, float* total_err)
{
  return guarded(h, [&] {
    if (!pose0 || !pose1 || !cam || !prx_orig || !prx_jac || !rows || !total_err)
      return fail(h, DFK_ERR_INVALID_ARG, "[ReprojectionFactor::linearize] null argument");
    DfkReprojectionItem it{{}, {}, *cam, *prx_orig, *prx_jac, code0, num_matches, query_xy, train_xy, cauchy_delta, sigma};
    std::copy_n(pose0, 7, it.pose0);
    std::copy_n(pose1, 7, it.pose1);
    DeviceGuard guard(h->device);
    // [the one item's staging | rows | err2], in scratch of its own: an earlier asynchronous batch may still be reading
    // the batches' staging
    const size_t M = (size_t)num_matches, RW = 13 + (size_t)code_size, n_out = 2 * M * RW + M;
    Staged st;
    DFK_TRY(stage(h, "[ReprojectionFactor::linearize] ", false, &it, 1, code_size, n_out * sizeof(float), h->sparse_host,
                  h->sparse_dev, &st));
    const float2* d_query = reinterpret_cast<const float2*>(st.payload);
    float* d_rows = reinterpret_cast<float*>(h->sparse_dev.ptr + st.bytes);
    DFK_CUDA(h, launch_reprojection_rows(code_size, *reinterpret_cast<const ReprojItemDev*>(h->sparse_host.ptr), d_query,
                                         d_query + M, h->params.sfmparams.avg_dpt, d_rows, d_rows + 2 * M * RW, h->stream),
             "[ReprojectionFactor::linearize] kernel launch failed");
    h->launches += 1;
    float* out = reinterpret_cast<float*>(h->sparse_host.ptr + st.bytes);
    DFK_TRY(download(h, out, d_rows, n_out * sizeof(float), "[ReprojectionFactor::linearize] result download failed",
                     "[ReprojectionFactor::linearize] kernel launch failed"));
    memcpy(rows, out, 2 * M * RW * sizeof(float));
    float tot = 0.0f;  // Scalar total_err accumulated in match order (:179,242)
    for (size_t i = 0; i < M; ++i) tot += out[2 * M * RW + i];
    *total_err = tot;
    return DFK_OK;
  });
}

DfkStatus dfk_reprojection_linearize_batch(DfkHandle h, const DfkReprojectionItem* items, int n, int code_size,
                                           float* records_dev)
{
  return guarded(h, [&] {
    if (!items || n < 1 || !records_dev)
      return fail(h, DFK_ERR_INVALID_ARG, "[ReprojectionFactor::linearize batch] null argument / empty batch");
    DeviceGuard guard(h->device);
    Staged st;
    DFK_TRY(stage(h, "[ReprojectionFactor::linearize batch] ", true, items, n, code_size, 0, h->rep_host, h->rep_dev, &st));
    const float2* query_dev = reinterpret_cast<const float2*>(st.payload);
    DFK_CUDA(h, launch_reprojection_records(code_size, reinterpret_cast<const ReprojItemDev*>(h->rep_dev.ptr), n,
                                            query_dev, query_dev + st.total, h->params.sfmparams.avg_dpt, records_dev,
                                            h->stream),
             "[ReprojectionFactor::linearize batch] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

namespace {

// Validates and stages the items of a matching batch; max_n0 / total / hyp_total / max_iterations describe the batch.
// ransac: the camera and RANSAC parameters are checked too.
DfkStatus stage_match(DfkHandle h, const char* what, const DfkMatchItem* items, int n, bool ransac, int* max_n0,
                      int* max_iterations, size_t* hyp_total)
{
  const std::string w(what);
  if (!items || n < 1 || n > 65535)  // blockIdx.y of the kernels is the item
    return fail(h, DFK_ERR_INVALID_ARG, w + "null argument / number of items not in [1, 65535]");
  h->match_host.resize((size_t)n);
  long long total = 0;
  *max_n0 = 0;
  *max_iterations = 0;
  *hyp_total = 0;
  for (int i = 0; i < n; ++i) {
    const DfkMatchItem& it = items[i];
    const std::string at = " in item " + std::to_string(i);
    const DfkFeatureSet* sets[2] = {&it.query, &it.train};
    for (const DfkFeatureSet* f : sets) {
      if (f->descriptor_bytes != 32 && f->descriptor_bytes != 64)
        return fail(h, DFK_ERR_UNSUPPORTED, w + "descriptor size " + std::to_string(f->descriptor_bytes) +
                                                " (only 32, ORB, and 64, BRISK)" + at);
      if (f->num < 0 || (f->num > 0 && (!f->keypoints || !f->descriptors)))
        return fail(h, DFK_ERR_INVALID_ARG, w + "negative feature count or null feature arrays" + at);
      if (((uintptr_t)f->descriptors & 15) != 0 || ((uintptr_t)f->keypoints & 3) != 0)
        return fail(h, DFK_ERR_INVALID_ARG, w + "descriptors must be 16-byte aligned, keypoints 4-byte aligned" + at);
    }
    if (it.query.descriptor_bytes != it.train.descriptor_bytes)
      return fail(h, DFK_ERR_INVALID_ARG, w + "query and train descriptors differ in size" + at);
    if (it.query.num > DFK_MATCH_MAX_QUERIES)
      return fail(h, DFK_ERR_INVALID_ARG, w + "more than DFK_MATCH_MAX_QUERIES query features" + at);
    if (ransac) {
      if (!(std::isfinite(it.cam.fx) && std::isfinite(it.cam.fy) && std::isfinite(it.cam.u0) &&
            std::isfinite(it.cam.v0) && it.cam.fx != 0.0f && it.cam.fy != 0.0f))
        return fail(h, DFK_ERR_INVALID_ARG, w + "camera needs finite intrinsics and fx, fy != 0" + at);
      if (it.max_iterations < 1 || it.max_iterations > DFK_MATCH_MAX_ITERATIONS)
        return fail(h, DFK_ERR_INVALID_ARG, w + "max_iterations not in [1, DFK_MATCH_MAX_ITERATIONS]" + at);
      if (!(it.threshold > 0.0 && std::isfinite(it.threshold)) || !(it.probability > 0.0 && it.probability < 1.0) ||
          !(it.max_dist >= 0.0f))
        return fail(h, DFK_ERR_INVALID_ARG, w + "threshold must be finite and > 0, probability in (0, 1), max_dist >= 0" +
                                                at);
    }
    MatchItemDev& d = h->match_host[(size_t)i];
    d = MatchItemDev{};
    d.kp0 = it.query.keypoints;
    d.kp1 = it.train.keypoints;
    d.d0 = it.query.descriptors;
    d.d1 = it.train.descriptors;
    d.n0 = it.query.num;
    d.n1 = it.train.num;
    d.words = it.query.descriptor_bytes / 4;
    d.out_begin = (int)total;
    total += it.query.num;
    if (ransac) {
      d.max_iterations = it.max_iterations;
      d.hyp_begin = (int)*hyp_total;
      *hyp_total += (size_t)(it.max_iterations + kMatchHyp - 1) / kMatchHyp * kMatchHyp;
      d.fx = it.cam.fx; d.fy = it.cam.fy; d.u0 = it.cam.u0; d.v0 = it.cam.v0;
      d.threshold = it.threshold;
      d.probability = it.probability;
      d.max_dist = it.max_dist;
      d.seed = it.seed;
      *max_iterations = std::max(*max_iterations, it.max_iterations);
    }
    *max_n0 = std::max(*max_n0, it.query.num);
  }
  if (total > INT32_MAX || *hyp_total > (size_t)INT32_MAX)
    return fail(h, DFK_ERR_INVALID_ARG, w + "more than 2^31 - 1 queries or hypotheses in one call");
  DFK_CUDA(h, h->match_items.ensure((size_t)n), (w + "scratch allocation failed").c_str());
  DFK_CUDA(h, cudaMemcpyAsync(h->match_items.ptr, h->match_host.data(), sizeof(MatchItemDev) * (size_t)n,
                              cudaMemcpyHostToDevice, h->stream),
           (w + "upload failed").c_str());
  return DFK_OK;
}

}  // namespace

DfkStatus dfk_hamming_match_batch(DfkHandle h, const DfkMatchItem* items, int n, int32_t* matches_dev)
{
  return guarded(h, [&] {
    const char* what = "[BFMatcher::match batch] ";
    if (!matches_dev) return fail(h, DFK_ERR_INVALID_ARG, std::string(what) + "null output");
    DeviceGuard guard(h->device);
    int max_n0 = 0, max_it = 0;
    size_t hyp = 0;
    DFK_TRY(stage_match(h, what, items, n, false, &max_n0, &max_it, &hyp));
    DFK_CUDA(h, launch_hamming_match(h->match_items.ptr, n, max_n0, reinterpret_cast<int2*>(matches_dev), h->stream),
             "[BFMatcher::match batch] kernel launch failed");
    h->launches += max_n0 > 0 ? 1 : 0;
    return DFK_OK;
  });
}

DfkStatus dfk_reprojection_match_batch(DfkHandle h, const DfkMatchItem* items, int n, int32_t* matches_dev,
                                       int32_t* counts_dev, int32_t* ransac_dev)
{
  return guarded(h, [&] {
    const char* what = "[ReprojectionFactor matches batch] ";
    if (!matches_dev || !counts_dev) return fail(h, DFK_ERR_INVALID_ARG, std::string(what) + "null output");
    DeviceGuard guard(h->device);
    int max_n0 = 0, max_it = 0;
    size_t hyp = 0;
    DFK_TRY(stage_match(h, what, items, n, true, &max_n0, &max_it, &hyp));
    size_t total = 0;
    for (const MatchItemDev& d : h->match_host) total += (size_t)d.n0;
    // [matches (int2 per query) | counts (int per hypothesis slot) | selections (int3 per item)], 16-byte aligned parts
    const size_t b_match = (sizeof(int2) * total + 15) & ~(size_t)15;
    const size_t b_count = (sizeof(int) * hyp + 15) & ~(size_t)15;
    const size_t b_sel = sizeof(int3) * (size_t)n;
    DFK_CUDA(h, h->match_scratch.ensure(b_match + b_count + b_sel + 16), "[ReprojectionFactor matches batch] scratch allocation failed");
    unsigned char* base = h->match_scratch.ptr;
    int3* sel = ransac_dev ? reinterpret_cast<int3*>(ransac_dev) : reinterpret_cast<int3*>(base + b_match + b_count);
    DFK_CUDA(h, launch_reprojection_match(h->match_items.ptr, n, max_n0, max_it, reinterpret_cast<int2*>(base),
                                          reinterpret_cast<int*>(base + b_match), sel,
                                          reinterpret_cast<int3*>(matches_dev), counts_dev, h->stream),
             "[ReprojectionFactor matches batch] kernel launch failed");
    h->launches += 4;
    return DFK_OK;
  });
}

DfkStatus dfk_orb_detect_batch(DfkHandle h, const DfkOrbItem* items, int n, float* keypoints_dev,
                               uint8_t* descriptors_dev, float* angles_dev, float* responses_dev, int32_t* counts_dev)
{
  return guarded(h, [&] {
    const std::string w = "[OrbDetector batch] ";
    if (!items || n < 1 || n > 65535)  // gridDim.z of the FAST kernel is the item
      return fail(h, DFK_ERR_INVALID_ARG, w + "null argument / number of items not in [1, 65535]");
    if (!keypoints_dev || !descriptors_dev || !counts_dev)
      return fail(h, DFK_ERR_INVALID_ARG, w + "null keypoint, descriptor or count output");
    if (((uintptr_t)keypoints_dev & 3) || ((uintptr_t)descriptors_dev & 15) || ((uintptr_t)angles_dev & 3) ||
        ((uintptr_t)responses_dev & 3) || ((uintptr_t)counts_dev & 3))
      return fail(h, DFK_ERR_INVALID_ARG, w + "descriptors must be 16-byte aligned, the other outputs 4-byte aligned");
    h->orb_host.resize((size_t)n);
    long long rows = 0, segs = 0, corners = 0, map = 0, blur = 0;
    int max_rw = 0, max_rh = 0, max_cc = 0, max_segs = 0, max_cap = 0, max_nf = 0;
    for (int i = 0; i < n; ++i) {
      const DfkOrbItem& it = items[i];
      const std::string at = " in item " + std::to_string(i);
      if (!it.image.ptr || it.image.width > DFK_ORB_MAX_SIDE || it.image.height > DFK_ORB_MAX_SIDE ||
          it.image.pitch_bytes < it.image.width)
        return fail(h, DFK_ERR_INVALID_ARG, w + "image needs a pointer, width and height <= DFK_ORB_MAX_SIDE and "
                                                "pitch_bytes >= width" + at);
      if (it.nfeatures < 1 || it.nfeatures > DFK_MATCH_MAX_QUERIES)
        return fail(h, DFK_ERR_INVALID_ARG, w + "nfeatures not in [1, DFK_MATCH_MAX_QUERIES]" + at);
      if (it.fast_threshold < 0 || it.fast_threshold > 255)
        return fail(h, DFK_ERR_INVALID_ARG, w + "fast_threshold not in [0, 255]" + at);
      if (it.capacity < it.nfeatures)
        return fail(h, DFK_ERR_INVALID_ARG, w + "capacity < nfeatures" + at);
      const bool big = it.image.width >= DFK_OM_MIN_SIZE && it.image.height >= DFK_OM_MIN_SIZE;
      OrbItemDev& d = h->orb_host[(size_t)i];
      d = OrbItemDev{};
      d.img = static_cast<const uint8_t*>(it.image.ptr);
      d.pitch = it.image.pitch_bytes;
      d.rw = big ? (int)it.image.width - 2 * DFK_OM_EDGE : 0;
      d.rh = big ? (int)it.image.height - 2 * DFK_OM_EDGE : 0;
      d.tiles_x = (d.rw + kOrbTileW - 1) / kOrbTileW;
      d.tiles_y = (d.rh + kOrbTileH - 1) / kOrbTileH;
      d.nfeatures = it.nfeatures;
      d.threshold = it.fast_threshold;
      d.capacity = it.capacity;
      d.out_begin = (int)std::min(rows, (long long)INT32_MAX);
      d.map_begin = (size_t)map;
      d.seg_begin = (int)std::min(segs, (long long)INT32_MAX);
      d.corner_begin = (int)std::min(corners, (long long)INT32_MAX);
      d.corner_cap = ((d.rw + 1) / 2) * ((d.rh + 1) / 2);  // one corner per 2 x 2 pixels at most survives NMS
      d.blur_begin = (size_t)blur;
      rows += it.capacity;
      segs += (long long)d.rh * d.tiles_x;
      corners += d.corner_cap;
      map += (long long)d.rw * d.rh;
      if (big) blur += (long long)(d.rw + 2 * DFK_OM_PATTERN_R) * (d.rh + 2 * DFK_OM_PATTERN_R);
      max_rw = std::max(max_rw, d.rw);
      max_rh = std::max(max_rh, d.rh);
      max_cc = std::max(max_cc, d.corner_cap);
      max_segs = std::max(max_segs, d.rh * d.tiles_x);
      max_cap = std::max(max_cap, it.capacity);
      max_nf = std::max(max_nf, it.nfeatures);
    }
    if (rows > INT32_MAX || corners > INT32_MAX || segs > INT32_MAX)
      return fail(h, DFK_ERR_INVALID_ARG, w + "more than 2^31 - 1 output rows or scratch entries in one call");
    DeviceGuard guard(h->device);
    // one allocation: [hist | stats | segments | corner positions | keys | angles | row map | score maps | blurred
    // images], 16-byte parts
    auto part = [](size_t bytes) { return (bytes + 15) & ~(size_t)15; };
    const size_t b_hist = part(sizeof(int) * 256 * (size_t)n), b_stats = part(sizeof(int) * 4 * (size_t)n);
    const size_t b_seg = part(sizeof(int) * (size_t)segs), b_c = part(sizeof(uint32_t) * (size_t)corners);
    const size_t b_rows = part(sizeof(int) * (size_t)rows), b_map = part((size_t)map), b_blur = part((size_t)blur);
    DFK_CUDA(h, h->orb_items.ensure((size_t)n), "[OrbDetector batch] scratch allocation failed");
    DFK_CUDA(h, h->orb_scratch.ensure(b_hist + b_stats + b_seg + 3 * b_c + b_rows + b_map + b_blur),
             "[OrbDetector batch] scratch allocation failed");
    unsigned char* p = h->orb_scratch.ptr;
    OrbScratchDev s;
    s.hist = reinterpret_cast<int*>(p);
    s.stats = reinterpret_cast<int*>(p += b_hist);
    s.seg = reinterpret_cast<int*>(p += b_stats);
    s.pos = reinterpret_cast<uint32_t*>(p += b_seg);
    s.key = reinterpret_cast<uint32_t*>(p += b_c);
    s.angle = reinterpret_cast<float*>(p += b_c);
    s.rows = reinterpret_cast<int*>(p += b_c);
    s.map = p += b_rows;
    s.blur = p + b_map;
    DFK_CUDA(h, cudaMemcpyAsync(h->orb_items.ptr, h->orb_host.data(), sizeof(OrbItemDev) * (size_t)n,
                                cudaMemcpyHostToDevice, h->stream),
             "[OrbDetector batch] upload failed");
    DFK_CUDA(h, launch_orb_detect(h->orb_items.ptr, n, s, max_rw, max_rh, max_cc, max_segs, max_cap, max_nf,
                                  keypoints_dev, descriptors_dev, angles_dev, responses_dev, counts_dev, h->stream),
             "[OrbDetector batch] kernel launch failed");
    h->launches += max_rw > 0 ? 7 : 5;
    return DFK_OK;
  });
}

DfkStatus dfk_sparse_geometric_linearize(DfkHandle h, const float pose0[7], const float pose1[7], const float* code0,
                                         const float* code1, int code_size, const DfkCamera* cam, const DfkImage* prx0_orig,
                                         const DfkImage* prx0_jac, const DfkImage* prx1_orig, const DfkImage* prx1_jac,
                                         const DfkImage* dpt_grad1, int num_points, const int* points_xy, float huber_delta,
                                         float* rows, int* num_valid)
{
  return guarded(h, [&] {
    if (!pose0 || !pose1 || !cam || !prx0_orig || !prx0_jac || !prx1_orig || !prx1_jac || !dpt_grad1 || !rows)
      return fail(h, DFK_ERR_INVALID_ARG, "[SparseGeometricFactor::linearize] null argument");
    DfkSparseGeometricItem it{{}, {}, *cam, *prx0_orig, *prx0_jac, *prx1_orig, *prx1_jac, *dpt_grad1, code0, code1,
                              num_points, points_xy, huber_delta};
    std::copy_n(pose0, 7, it.pose0);
    std::copy_n(pose1, 7, it.pose1);
    DeviceGuard guard(h->device);
    // [the one item's staging | rows], apart from the batches' staging
    const size_t M = (size_t)num_points, RW = 13 + 2 * (size_t)code_size;
    Staged st;
    DFK_TRY(stage(h, "[SparseGeometricFactor::linearize] ", false, &it, 1, code_size, M * RW * sizeof(float),
                  h->sparse_host, h->sparse_dev, &st));
    float* d_rows = reinterpret_cast<float*>(h->sparse_dev.ptr + st.bytes);
    DFK_CUDA(h, launch_sparse_geometric_rows(code_size, *reinterpret_cast<const GeoItemDev*>(h->sparse_host.ptr),
                                             reinterpret_cast<const int2*>(st.payload), h->params.sfmparams.avg_dpt,
                                             d_rows, h->stream),
             "[SparseGeometricFactor::linearize] kernel launch failed");
    h->launches += 1;
    float* out = reinterpret_cast<float*>(h->sparse_host.ptr + st.bytes);
    DFK_TRY(download(h, out, d_rows, M * RW * sizeof(float), "[SparseGeometricFactor::linearize] result download failed",
                     "[SparseGeometricFactor::linearize] kernel launch failed"));
    memcpy(rows, out, M * RW * sizeof(float));
    int nv = 0;  // rows that are not all zero
    for (size_t i = 0; i < M; ++i) nv += std::any_of(out + i * RW, out + (i + 1) * RW, [](float v) { return v != 0.0f; });
    if (num_valid) *num_valid = nv;
    return DFK_OK;
  });
}

DfkStatus dfk_sparse_geometric_linearize_batch(DfkHandle h, const DfkSparseGeometricItem* items, int n, int code_size,
                                               float* records_dev)
{
  return guarded(h, [&] {
    if (!items || n < 1 || !records_dev)
      return fail(h, DFK_ERR_INVALID_ARG, "[SparseGeometricFactor::linearize batch] null argument / empty batch");
    DeviceGuard guard(h->device);
    Staged st;
    DFK_TRY(stage(h, "[SparseGeometricFactor::linearize batch] ", true, items, n, code_size, 0, h->geo_host, h->geo_dev,
                  &st));
    DFK_CUDA(h, launch_sparse_geometric_records(code_size, reinterpret_cast<const GeoItemDev*>(h->geo_dev.ptr), n,
                                                reinterpret_cast<const int2*>(st.payload), h->params.sfmparams.avg_dpt,
                                                records_dev, h->stream),
             "[SparseGeometricFactor::linearize batch] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_reprojection_error_batch(DfkHandle h, const DfkReprojectionItem* items, int n, int code_size, float* out_dev)
{
  return guarded(h, [&] {
    if (!items || n < 1 || !out_dev)
      return fail(h, DFK_ERR_INVALID_ARG, "[ReprojectionFactor::error batch] null argument / empty batch");
    DeviceGuard guard(h->device);
    Staged st;
    DFK_TRY(stage(h, "[ReprojectionFactor::error batch] ", true, items, n, code_size, 0, h->rep_host, h->rep_dev, &st));
    const float2* query_dev = reinterpret_cast<const float2*>(st.payload);
    DFK_CUDA(h, launch_reprojection_error(code_size, reinterpret_cast<const ReprojItemDev*>(h->rep_dev.ptr), n, query_dev,
                                          query_dev + st.total, h->params.sfmparams.avg_dpt, out_dev, h->stream),
             "[ReprojectionFactor::error batch] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_sparse_geometric_error_batch(DfkHandle h, const DfkSparseGeometricItem* items, int n, int code_size,
                                           float* out_dev)
{
  return guarded(h, [&] {
    if (!items || n < 1 || !out_dev)
      return fail(h, DFK_ERR_INVALID_ARG, "[SparseGeometricFactor::error batch] null argument / empty batch");
    DeviceGuard guard(h->device);
    Staged st;
    DFK_TRY(stage(h, "[SparseGeometricFactor::error batch] ", true, items, n, code_size, 0, h->geo_host, h->geo_dev, &st));
    DFK_CUDA(h, launch_sparse_geometric_error(code_size, reinterpret_cast<const GeoItemDev*>(h->geo_dev.ptr), n,
                                              reinterpret_cast<const int2*>(st.payload), h->params.sfmparams.avg_dpt,
                                              out_dev, h->stream),
             "[SparseGeometricFactor::error batch] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

// ---------------------------------------------------------------------------------------------- window problem
DfkStatus dfk_window_problem_create(DfkHandle h, const DfkWindowProblemDesc* d, DfkWindowProblem** out)
{
  return guarded(h, [&] {
    const std::string what = "[WindowProblem] ";
    if (!d || !out || !d->window) return fail(h, DFK_ERR_INVALID_ARG, what + "null argument");
    *out = nullptr;
    const DfkWindow* w = d->window;
    if (w->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, what + "window and handle live on different devices");
    const int K = w->dev.num_keyframes, F = w->dev.num_frames, C = w->dev.code_size, B = 6 + C, NP = K + F;
    const int nd = d->num_dense, nr = d->num_reproj, ng = d->num_geo, ndep = d->num_depth, ne = d->num_error;
    const int mf = d->num_frame_priors, nkm = (int)w->prior_kf.size();
    if (nd < 0 || nr < 0 || ng < 0 || ndep < 0 || ne < 0 || mf < 0 || ne > 65535 || ndep > 65535)
      return fail(h, DFK_ERR_INVALID_ARG, what + "negative item count / more than 65535 error or depth items");
    if (nd + nr != w->dev.num_items || ng != w->dev.num_links)
      return fail(h, DFK_ERR_INVALID_ARG, what + "the items do not match the window's records (" +
                                              std::to_string(w->dev.num_items) + " records, " +
                                              std::to_string(w->dev.num_links) + " links)");
    if ((nd && (!d->dense || !d->dense_slots)) || (nr && (!d->reproj || !d->reproj_slots)) ||
        (ng && (!d->geo || !d->geo_slots || !d->geo_records_dev)) || (ndep && (!d->depth || !d->depth_slots)) ||
        (ne && (!d->error || !d->error_slots || !d->error_depth)) || !d->records_dev ||
        (mf && (!d->frame_prior_kf || !d->frame_prior_rows || !d->frame_prior_x0)) ||
        (w->kp.num_priors && (!d->kf_prior_rows || !d->kf_prior_x0)))
      return fail(h, DFK_ERR_INVALID_ARG, what + "null argument");
    // slots: pose slots name a keyframe or a frame, code slots a keyframe
    auto bad_slot = [&](const char* kind, int i, const char* which) {
      return fail(h, DFK_ERR_INVALID_ARG, what + kind + " item " + std::to_string(i) + ": " + which +
                                              " slot out of range");
    };
    for (int i = 0; i < nd; ++i) {
      const DfkWindowItemSlots& s = d->dense_slots[i];
      if (!slot_ok(s.pose0, 0, NP)) return bad_slot("dense", i, "pose0");
      if (!slot_ok(s.pose1, 0, NP)) return bad_slot("dense", i, "pose1");
      if (!slot_ok(s.code0, 0, K)) return bad_slot("dense", i, "code0");
    }
    for (int i = 0; i < nr; ++i) {
      const DfkWindowItemSlots& s = d->reproj_slots[i];
      if (!slot_ok(s.pose0, 0, NP)) return bad_slot("reprojection", i, "pose0");
      if (!slot_ok(s.pose1, 0, NP)) return bad_slot("reprojection", i, "pose1");
      if (!slot_ok(s.code0, 0, K)) return bad_slot("reprojection", i, "code0");
    }
    for (int i = 0; i < ng; ++i) {
      const DfkWindowItemSlots& s = d->geo_slots[i];
      if (!slot_ok(s.pose0, 0, NP)) return bad_slot("geometric", i, "pose0");
      if (!slot_ok(s.pose1, 0, NP)) return bad_slot("geometric", i, "pose1");
      if (!slot_ok(s.code0, 0, K)) return bad_slot("geometric", i, "code0");
      if (!slot_ok(s.code1, 0, K)) return bad_slot("geometric", i, "code1");
    }
    for (int i = 0; i < ndep; ++i)
      if (!slot_ok(d->depth_slots[i].code0, 0, K)) return bad_slot("depth", i, "code0");
    for (int i = 0; i < ne; ++i) {
      const DfkWindowItemSlots& s = d->error_slots[i];
      if (!slot_ok(s.pose0, 0, NP)) return bad_slot("error", i, "pose0");
      if (!slot_ok(s.pose1, 0, NP)) return bad_slot("error", i, "pose1");
      if (!slot_ok(d->error_depth[i], 0, ndep)) return bad_slot("error", i, "depth");
    }
    for (int i = 0; i < mf; ++i)
      if (!slot_ok(d->frame_prior_kf[i], 0, K))
        return fail(h, DFK_ERR_INVALID_ARG, what + "frame prior " + std::to_string(i) + " names a keyframe outside the window");
    DeviceGuard guard(h->device);
    std::unique_ptr<DfkWindowProblem> p(new (std::nothrow) DfkWindowProblem());
    if (!p) return oom(h);
    p->device = h->device; p->w = w;
    p->K = K; p->F = F; p->C = C; p->B = B;
    p->nd = nd; p->nr = nr; p->ng = ng; p->ndep = ndep; p->ne = ne; p->mf = mf; p->nkm = nkm;
    p->S = (size_t)NP * 7 + (size_t)K * C;
    p->avg_dpt = h->params.sfmparams.avg_dpt;
    p->huber_delta = h->params.sfmparams.huber_delta;
    p->records = d->records_dev; p->geo_records = d->geo_records_dev;
    const char* amsg = "[WindowProblem] allocation failed";
    const std::vector<float> zero_code(std::max(C, 1), 0.0f);
    // ---- dense items: the batch's checks, kernel choice and tile plan, with a code slot of the problem's own each
    if (nd > 0) {
      std::vector<DfkSfmWorkItem> t(d->dense, d->dense + nd);
      for (auto& it : t) it.code = zero_code.data();
      DFK_TRY(choose_step_kernel(h, t.data(), nd, C, &p->step));
      DFK_CUDA(h, p->dense_codes.ensure((size_t)nd * C), amsg);
      h->codes_host.assign((size_t)nd * C, 0.0f);
      // build_items files every camera level in the handle's ray cache; the problem builds tables of its own (below),
      // so the entries this call adds are dropped again: they would never be built and would count toward a flush
      if (h->ray_flush) {  // the flush build_items would start with, done here so that the count below holds
        h->ray_cache.clear();
        h->ray_flush = false;
      }
      const size_t rays_before = h->ray_cache.size();
      const DfkStatus bs = build_items(h, t.data(), nd, C, p->step.tile_px, p->step.max_ctas, p->dense_codes.ptr, &p->plan);
      h->ray_cache.resize(rays_before);
      h->ray_flush = false;
      h->ray_pending.clear();
      DFK_TRY(bs);
      std::vector<SfmItemDev> items = h->items_host;
      // ray tables of its own: the handle's cache may flush (and free) its tables
      std::vector<const SfmItemDev*> owner;
      for (auto& it : items) {
        size_t r = 0;
        for (; r < owner.size(); ++r) {
          const SfmItemDev& o = *owner[r];
          if (o.fx == it.fx && o.fy == it.fy && o.u0 == it.u0 && o.v0 == it.v0 && o.width == it.width &&
              o.height == it.height)
            break;
        }
        if (r == owner.size()) {
          owner.push_back(&it);
          p->rays.emplace_back();
          DFK_CUDA(h, p->rays.back().ensure((size_t)it.width + it.height), amsg);
        }
        it.ray_tab = p->rays[r].ptr;
      }
      p->dense_tmpl = items;
      DFK_CUDA(h, p->dense.ensure(nd), amsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->dense.ptr, items.data(), sizeof(SfmItemDev) * nd, cudaMemcpyHostToDevice, h->stream),
               "[WindowProblem] upload failed");
      DFK_CUDA(h, launch_sfm_ray_tables(p->dense.ptr, nd, h->stream), "[WindowProblem] kernel launch failed");
      h->launches += 1;
    }
    // ---- sparse links: the batches' checks and staging, into blocks of the problem's own
    if (nr > 0) {
      std::vector<DfkReprojectionItem> t(d->reproj, d->reproj + nr);
      for (auto& it : t) it.code = zero_code.data();
      Staged st;
      DFK_TRY(stage(h, what + "reprojection ", true, t.data(), nr, C, 0, p->rep_host, p->rep, &st));
      p->rep_payload = st.payload;
      p->rep_total = st.total;
    }
    if (ng > 0) {
      std::vector<DfkSparseGeometricItem> t(d->geo, d->geo + ng);
      for (auto& it : t) it.code0 = it.code1 = zero_code.data();
      Staged st;
      DFK_TRY(stage(h, what + "geometric ", true, t.data(), ng, C, 0, p->geo_host, p->geo, &st));
      p->geo_payload = st.payload;
    }
    // ---- the error path: depth decodes into scratch of the problem's own, and the error items reading it
    std::vector<size_t> dep_off(ndep + 1, 0);
    for (int i = 0; i < ndep; ++i) {
      const DfkDepthDecodeItem& it = d->depth[i];
      const uint32_t W = it.dpt.width, H = it.dpt.height;
      if (W == 0 || H == 0 || !img_ok(&it.prx_orig, W, H, 1) || !img_ok(&it.prx_jac, W, H, C))
        return fail(h, DFK_ERR_INVALID_ARG, what + "inconsistent image views in depth item " + std::to_string(i));
      dep_off[i + 1] = dep_off[i] + (((size_t)W * H + 3) & ~(size_t)3);
    }
    if (ndep > 0) {
      DFK_CUDA(h, p->depth_scratch.ensure(dep_off[ndep]), amsg);
      const size_t desc_bytes = (sizeof(DepthDecodeDesc) * (size_t)ndep + 15) & ~(size_t)15;
      const size_t total = desc_bytes + sizeof(float) * (size_t)ndep * C;
      DFK_CUDA(h, p->depth.ensure(total), amsg);
      std::vector<unsigned char> hb(total, 0);
      DepthDecodeDesc* descs = reinterpret_cast<DepthDecodeDesc*>(hb.data());
      const float* codes_dev = reinterpret_cast<const float*>(p->depth.ptr + desc_bytes);
      for (int i = 0; i < ndep; ++i) {
        const DfkDepthDecodeItem& it = d->depth[i];
        DepthDecodeDesc& dd = descs[i];
        dd.prx = view_of(&it.prx_orig);
        dd.jac = view_of(&it.prx_jac);
        dd.dpt = p->depth_scratch.ptr + dep_off[i];
        dd.dpt_pitch = it.dpt.width;
        dd.code = codes_dev + (size_t)i * C;
        dd.width = (int)it.dpt.width;
        dd.height = (int)it.dpt.height;
        dd.nblocks = update_depth_blocks(dd.width, dd.height);
        dd.vector = update_depth_vector(C, dd.code, dd.jac) ? 1 : 0;
        p->depth_max_blocks = std::max(p->depth_max_blocks, dd.nblocks);
      }
      DFK_CUDA(h, cudaMemcpyAsync(p->depth.ptr, hb.data(), total, cudaMemcpyHostToDevice, h->stream),
               "[WindowProblem] upload failed");
    }
    if (ne > 0) {
      std::vector<EvalErrorDesc> descs(ne);
      std::vector<double> areas(ne);
      for (int i = 0; i < ne; ++i) {
        const DfkSfmWorkItem& it = d->error[i];
        const DfkDepthDecodeItem& dep = d->depth[d->error_depth[i]];
        const DfkImage dpt{p->depth_scratch.ptr + dep_off[d->error_depth[i]], (size_t)dep.dpt.width * 4, dep.dpt.width,
                           dep.dpt.height};
        const uint32_t W = it.img0.width, H = it.img0.height;
        if (it.code)
          return fail(h, DFK_ERR_INVALID_ARG, what + "error item " + std::to_string(i) +
                                                  ": no fused depth decode (the depth comes from its depth item)");
        if (W == 0 || H == 0 || !img_ok(&it.img0, W, H, 1) || !img_ok(&it.img1, W, H, 1) || !img_ok(&dpt, W, H, 1))
          return fail(h, DFK_ERR_INVALID_ARG, what + "inconsistent image views in error item " + std::to_string(i));
        if (!cam_ok(&it.cam, W, H))
          return fail(h, DFK_ERR_INVALID_ARG, what + "camera viewport larger than the image views in error item " +
                                                  std::to_string(i));
        EvalErrorDesc& e = descs[i];
        const float ident[7] = {0, 0, 0, 1, 0, 0, 0};
        e.pc = make_pixel_cam(ident, &it.cam, 1, 0.0f);  // as dfk_sfm_evaluate_error: border 1, min_dpt 0
        e.img0 = view_of(&it.img0); e.img1 = view_of(&it.img1); e.dpt0 = view_of(&dpt);
        e.width = (int)W;
        e.height = (int)H;
        e.nblocks = eval_error_blocks(e.width, e.height);
        e.scratch_row = p->err_rows;
        p->err_rows += e.nblocks;
        p->err_max_blocks = std::max(p->err_max_blocks, e.nblocks);
        areas[i] = (double)W * (double)H;
      }
      DFK_CUDA(h, p->err.ensure(ne), amsg);
      DFK_CUDA(h, p->areas.ensure(ne), amsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->err.ptr, descs.data(), sizeof(EvalErrorDesc) * ne, cudaMemcpyHostToDevice, h->stream),
               "[WindowProblem] upload failed");
      DFK_CUDA(h, cudaMemcpyAsync(p->areas.ptr, areas.data(), sizeof(double) * ne, cudaMemcpyHostToDevice, h->stream),
               "[WindowProblem] upload failed");
      p->err_tmpl = descs;
      p->areas_tmpl = areas;
    }
    DFK_CUDA(h, p->err_out.ensure(std::max<size_t>(1, 2 * (size_t)(ne + nr + ng))), amsg);
    // ---- slots, in the repose kernel's order
    std::vector<int4> slots;
    auto push = [&](const DfkWindowItemSlots* s, int n) {
      for (int i = 0; i < n; ++i) slots.push_back(make_int4(s[i].pose0, s[i].pose1, s[i].code0, s[i].code1));
    };
    push(d->dense_slots, nd); push(d->error_slots, ne); push(d->reproj_slots, nr); push(d->geo_slots, ng);
    push(d->depth_slots, ndep);
    p->slots_tmpl.assign(slots.begin(), slots.begin() + nd + ne);
    if (!slots.empty()) {
      DFK_CUDA(h, p->slots.ensure(slots.size()), amsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->slots.ptr, slots.data(), sizeof(int4) * slots.size(), cudaMemcpyHostToDevice,
                                  h->stream),
               "[WindowProblem] upload failed");
    }
    // ---- priors: rows, frozen points, the keyframe of every delta row, add_priors' lists
    const size_t PD = DFK_PRIOR_DOUBLES(C), X = 7 + (size_t)C;
    std::vector<int> dkf;
    std::vector<double> x0;
    if (mf > 0) {
      DFK_CUDA(h, p->frows.ensure(mf * PD), amsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->frows.ptr, d->frame_prior_rows, sizeof(double) * mf * PD, cudaMemcpyHostToDevice,
                                  h->stream),
               "[WindowProblem] upload failed");
      dkf.assign(d->frame_prior_kf, d->frame_prior_kf + mf);
      x0.assign(d->frame_prior_x0, d->frame_prior_x0 + mf * X);
      std::vector<int> lists(K + 1 + mf, 0);
      for (int i = 0; i < mf; ++i) lists[d->frame_prior_kf[i] + 1] += 1;
      for (int k = 0; k < K; ++k) lists[k + 1] += lists[k];
      std::vector<int> next(lists.begin(), lists.begin() + K);
      for (int i = 0; i < mf; ++i) lists[K + 1 + next[d->frame_prior_kf[i]]++] = i;
      DFK_CUDA(h, p->fp_lists.ensure(lists.size()), amsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->fp_lists.ptr, lists.data(), sizeof(int) * lists.size(), cudaMemcpyHostToDevice,
                                  h->stream),
               "[WindowProblem] upload failed");
    }
    if (w->kp.num_priors > 0) {
      const size_t kd = (size_t)w->prior_off.back();
      DFK_CUDA(h, p->kfrows.ensure(kd), amsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->kfrows.ptr, d->kf_prior_rows, sizeof(double) * kd, cudaMemcpyHostToDevice, h->stream),
               "[WindowProblem] upload failed");
      dkf.insert(dkf.end(), w->prior_kf.begin(), w->prior_kf.end());
      x0.insert(x0.end(), d->kf_prior_x0, d->kf_prior_x0 + nkm * X);
    }
    if (!dkf.empty()) {
      DFK_CUDA(h, p->delta_kf.ensure(dkf.size()), amsg);
      DFK_CUDA(h, p->x0.ensure(x0.size()), amsg);
      DFK_CUDA(h, p->delta.ensure(dkf.size() * B), amsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->delta_kf.ptr, dkf.data(), sizeof(int) * dkf.size(), cudaMemcpyHostToDevice, h->stream),
               "[WindowProblem] upload failed");
      DFK_CUDA(h, cudaMemcpyAsync(p->x0.ptr, x0.data(), sizeof(double) * x0.size(), cudaMemcpyHostToDevice, h->stream),
               "[WindowProblem] upload failed");
    }
    // ---- state (zero codes, identity poses until set_state), the gauge solver, the LM's small read-back block
    DFK_CUDA(h, p->state.ensure(2 * p->S), amsg);
    std::vector<double> init(2 * p->S, 0.0);
    for (int s = 0; s < 2 * NP; ++s) init[(size_t)(s / NP) * p->S + (size_t)(s % NP) * 7 + 3] = 1.0;
    DFK_CUDA(h, cudaMemcpyAsync(p->state.ptr, init.data(), sizeof(double) * init.size(), cudaMemcpyHostToDevice, h->stream),
             "[WindowProblem] upload failed");
    const std::vector<int> gauge{0, 1, 2, 3, 4, 5};
    DFK_CUDA(h, window_solver_create(K, C, F, w->pair_k0, w->pair_k1, w->link_k0, w->link_k1, w->blk_i, w->blk_j,
                                     w->kp.block_off, gauge, &p->solver[1]),
             "[WindowProblem] solver workspace allocation failed");
    DFK_CUDA(h, p->small.ensure(8 * sizeof(double) + 16), amsg);
    DFK_CUDA(h, p->small_host.ensure(8 * sizeof(double) + 16), amsg);
    DFK_CUDA(h, cudaStreamSynchronize(h->stream), "[WindowProblem] upload failed");  // the host staging is freed next
    *out = p.release();
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_destroy(DfkHandle h, DfkWindowProblem* p)
{
  return guarded(h, [&] {
    if (!p) return DFK_OK;
    DeviceGuard guard(p->device);
    delete p;
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_set_state(DfkHandle h, DfkWindowProblem* p, const double* poses, const double* codes)
{
  return guarded(h, [&] {
    if (!p || !poses || (!codes && p->K * p->C > 0)) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] null argument");
    if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    const size_t np = (size_t)(p->K + p->F) * 7;
    DFK_CUDA(h, cudaMemcpyAsync(p->st(p->cur), poses, sizeof(double) * np, cudaMemcpyDefault, h->stream),
             "[WindowProblem] state copy failed");
    if (p->K * p->C > 0)
      DFK_CUDA(h, cudaMemcpyAsync(p->st(p->cur) + np, codes, sizeof(double) * (p->S - np), cudaMemcpyDefault, h->stream),
               "[WindowProblem] state copy failed");
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_get_state(DfkHandle h, const DfkWindowProblem* p, double* poses, double* codes)
{
  return guarded(h, [&] {
    if (!p || !poses || (!codes && p->K * p->C > 0)) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] null argument");
    if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    const size_t np = (size_t)(p->K + p->F) * 7;
    DFK_CUDA(h, cudaMemcpyAsync(poses, p->st(p->cur), sizeof(double) * np, cudaMemcpyDefault, h->stream),
             "[WindowProblem] state copy failed");
    if (p->K * p->C > 0)
      DFK_CUDA(h, cudaMemcpyAsync(codes, p->st(p->cur) + np, sizeof(double) * (p->S - np), cudaMemcpyDefault, h->stream),
               "[WindowProblem] state copy failed");
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_linearize(DfkHandle h, DfkWindowProblem* p, float* window_dev)
{
  return guarded(h, [&] {
    if (!p || !window_dev) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem::linearize] null argument");
    if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    return problem_linearize(h, p, p->st(p->cur), window_dev);
  });
}

DfkStatus dfk_window_problem_error(DfkHandle h, DfkWindowProblem* p, double* out_dev)
{
  return guarded(h, [&] {
    if (!p || !out_dev) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem::error] null argument");
    if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    DFK_TRY(problem_error(h, p, p->st(p->cur), 0.0));
    DFK_CUDA(h, cudaMemcpyAsync(out_dev, p->energy(), sizeof(double) * DFK_WINDOW_ERROR_DOUBLES, cudaMemcpyDeviceToDevice,
                                h->stream),
             "[WindowProblem::error] copy failed");
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_retract(DfkHandle h, DfkWindowProblem* p, const double* dx_dev)
{
  return guarded(h, [&] {
    if (!p || !dx_dev) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem::retract] null argument");
    if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    // into the other state, which then becomes the problem's
    DFK_CUDA(h, launch_window_retract(p->st(p->cur), p->st(1 - p->cur), dx_dev, p->K, p->F, p->C, h->stream),
             "[WindowProblem::retract] kernel launch failed");
    h->launches += 1;
    p->cur = 1 - p->cur;
    return DFK_OK;
  });
}

DfkStatus dfk_window_lm(DfkHandle h, DfkWindowProblem* p, const DfkLMParams* prm, DfkLMTrace* tr)
{
  return guarded(h, [&] {
    DeviceGuard guard(h->device);
    ProblemLMOps ops;
    DFK_TRY(lm_setup(h, p, prm, tr, "WindowLM", &ops));
    return lm_run(*prm, ops, tr);
  });
}

DfkStatus dfk_window_problem_set_active(DfkHandle h, DfkWindowProblem* p, const uint8_t* dense_active,
                                        const uint8_t* error_active)
{
  return guarded(h, [&] {
    const char* what = "[WindowProblem::set_active] ";
    if (!p || (p->nd > 0 && !dense_active) || (!error_active && p->ne != p->nd))
      return fail(h, DFK_ERR_INVALID_ARG, std::string(what) +
                                              "null argument (error_active may be NULL only when num_error == num_dense)");
    if (p->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    return problem_set_active(h, p, dense_active, error_active ? error_active : dense_active);
  });
}

DfkStatus dfk_window_lm_levels(DfkHandle h, DfkWindowProblem* p, const DfkLMParams* prm, const DfkLevelSchedule* sc,
                               DfkLMTrace* tr, DfkLevelTrace* lt)
{
  return guarded(h, [&] {
    const std::string what = "[WindowLMLevels] ";
    if (!p || !sc) return fail(h, DFK_ERR_INVALID_ARG, what + "null argument");
    const int nd = p->nd, ne = p->ne, L = sc->num_levels;
    if (L < 1 || !sc->iters || (nd > 0 && !sc->dense_level) || sc->num_pairs < 0 ||
        (sc->num_pairs > 0 && !sc->pair_steps_done))
      return fail(h, DFK_ERR_INVALID_ARG, what + "num_levels < 1, or null iters / dense_level / pair_steps_done");
    if (ne > 0 && ne != nd && (!sc->error_pair || !sc->error_level))
      return fail(h, DFK_ERR_INVALID_ARG, what + "error_pair and error_level are required when num_error != num_dense");
    for (int l = 0; l < L; ++l)
      if (sc->iters[l] < 0) return fail(h, DFK_ERR_INVALID_ARG, what + "iters[" + std::to_string(l) + "] < 0");
    // the schedule's pairs: the distinct window pairs of the dense items, in window order
    std::vector<int> dpair(nd), ids;
    for (int i = 0; i < nd; ++i) ids.push_back(p->w->item_pair[i]);
    std::sort(ids.begin(), ids.end());
    ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
    if ((int)ids.size() != sc->num_pairs)
      return fail(h, DFK_ERR_INVALID_ARG, what + "num_pairs " + std::to_string(sc->num_pairs) + ", but the dense items" +
                                              " cover " + std::to_string(ids.size()) + " pairs");
    for (int i = 0; i < nd; ++i)
      dpair[i] = (int)(std::lower_bound(ids.begin(), ids.end(), p->w->item_pair[i]) - ids.begin());
    for (int i = 0; i < nd; ++i)
      if (sc->dense_level[i] < 0 || sc->dense_level[i] >= L)
        return fail(h, DFK_ERR_INVALID_ARG, what + "dense item " + std::to_string(i) + ": level outside [0, num_levels)");
    std::vector<int> epair(ne), elevel(ne);
    for (int i = 0; i < ne; ++i) {
      epair[i] = sc->error_pair ? sc->error_pair[i] : dpair[i];
      elevel[i] = sc->error_level ? sc->error_level[i] : sc->dense_level[i];
      if (epair[i] < 0 || epair[i] >= sc->num_pairs || elevel[i] < 0 || elevel[i] >= L)
        return fail(h, DFK_ERR_INVALID_ARG, what + "error item " + std::to_string(i) +
                                                ": pair or level out of range");
    }
    for (int q = 0; q < sc->num_pairs; ++q)
      if (sc->pair_steps_done[q] < 0)
        return fail(h, DFK_ERR_INVALID_ARG, what + "pair_steps_done[" + std::to_string(q) + "] < 0");
    DeviceGuard guard(h->device);
    struct LevelOps : ProblemLMOps {
      const DfkLevelSchedule* sc;
      const std::vector<int>* dpair;
      const std::vector<int>* epair;
      const std::vector<int>* elevel;
      std::vector<uint8_t> dm, em;
      DfkStatus set_levels(const int* lvl)
      {
        for (size_t i = 0; i < dm.size(); ++i) dm[i] = lvl[(*dpair)[i]] == sc->dense_level[i];
        for (size_t i = 0; i < em.size(); ++i) em[i] = lvl[(*epair)[i]] == (*elevel)[i];
        return problem_set_active(h, p, dm.data(), em.data());
      }
    } ops;
    DFK_TRY(lm_setup(h, p, prm, tr, "WindowLMLevels", &ops));
    ops.sc = sc;
    ops.dpair = &dpair;
    ops.epair = &epair;
    ops.elevel = &elevel;
    ops.dm.assign(nd, 1);
    ops.em.assign(ne, 1);
    return lm_levels_run(*prm, *sc, ops, tr, lt);
  });
}

}  // extern "C"
