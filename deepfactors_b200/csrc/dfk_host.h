// dfk_host.h -- host-side pieces that the C ABI's units (dfk_api.cu, dfk_api_sparse.cu, dfk_api_window.cu) share:
// scratch buffers, the handle, error reporting, argument checks, the dense RunStep planning and the sparse staging.
// Internal to libdfk.so.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "dfk.h"
#include "dfk_internal.h"
#include "dfk_se3.cuh"

using namespace dfk;

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
  // dfk_orb_detect_pyramid_batch: [one-level items | gather items | resize items] (bytes, one H2D per call from
  // orb_pyr_host); its level images and staged rows follow the detector's scratch in orb_scratch
  DeviceBuf<unsigned char> orb_pyr_dev;
  std::vector<unsigned char> orb_pyr_host;
  // dfk_preprocess_batch: [item descriptors | pyramid level descriptors L x n] (bytes, one H2D per call from pp_host)
  // and the normalising items' tile partials
  DeviceBuf<unsigned char> pp_dev;
  std::vector<unsigned char> pp_host;
  DeviceBuf<double> pp_partials;
  // dfk_keyframe_mesh_batch: [item descriptors | decode descriptors | codes] (bytes, one H2D per call from mesh_host)
  // and [segment masks | segment bases | decoded depths] (bytes)
  DeviceBuf<unsigned char> mesh_dev;
  std::vector<unsigned char> mesh_host;
  DeviceBuf<unsigned char> mesh_scratch;
  // the dfk_bow_* calls: the call's descriptors (one H2D per call from bow_host), the transform's per-descriptor words
  // when the caller passes none, and a query's [sums n x size | hits n x size] (bytes)
  DeviceBuf<unsigned char> bow_dev;
  std::vector<unsigned char> bow_host;
  DeviceBuf<int32_t> bow_words;
  DeviceBuf<unsigned char> bow_scratch;
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

inline DfkStatus fail(DfkHandle h, DfkStatus s, const std::string& msg)
{
  if (h) h->err = msg;
  return s;
}

// out-of-memory exit of an extern "C" entry point (never throws itself)
inline DfkStatus oom(DfkHandle h) noexcept
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

inline DfkStatus cuda_fail(DfkHandle h, cudaError_t e, const char* what)
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
inline DfkStatus download(DfkHandle h, void* host, const void* dev, size_t bytes, const char* copy_what,
                          const char* sync_what)
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

// ---------------------------------------------------------------------------- validation helpers
inline bool img_ok(const DfkImage* im, uint32_t w, uint32_t h, uint32_t floats_per_px)
{
  return im && im->ptr && im->width == w && im->height == h && (im->pitch_bytes % 4 == 0) &&
         im->pitch_bytes >= (size_t)w * floats_per_px * 4;
}

// The validity window comes from the camera (PixelValid: u < cam.width - border, pinhole_camera_impl.h:102-108) while the
// bilinear taps index the images: a camera larger than the level it is used with (e.g. a level-0 camera with level-1
// buffers) would read outside them.  The reference has no such check (it would read out of bounds); here it is an
// argument error.
inline bool cam_ok(const DfkCamera* cam, uint32_t w, uint32_t h)
{
  return cam && cam->width <= (float)w && cam->height <= (float)h && cam->width >= 0.0f && cam->height >= 0.0f;
}

inline View view_of(const DfkImage* im)
{
  return View{static_cast<const float*>(im->ptr), (uint32_t)(im->pitch_bytes / 4)};
}

inline PixelCam make_pixel_cam(const float pose[7], const DfkCamera* cam, int border, float min_dpt)
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

// ---------------------------------------------------------------------------- descriptors and tickets
// One EvalErrorDesc from the relative pose p10 = pose1^-1 * pose0, with the border 1 and min_dpt 0 of
// dfk_sfm_evaluate_error (dense_sfm.h:91).  Its partial rows start at *rows, which grows by them, as *max_blocks does
// to its grid.
inline void set_eval_error_desc(EvalErrorDesc& d, const DfkCamera& cam, const float p10[7], const DfkImage& img0,
                                const DfkImage& img1, const DfkImage& dpt0, int* rows, int* max_blocks)
{
  d.pc = make_pixel_cam(p10, &cam, 1, 0.0f);
  d.img0 = view_of(&img0); d.img1 = view_of(&img1); d.dpt0 = view_of(&dpt0);
  d.width = (int)img0.width;
  d.height = (int)img0.height;
  d.nblocks = eval_error_blocks(d.width, d.height);
  d.scratch_row = *rows;
  *rows += d.nblocks;
  *max_blocks = std::max(*max_blocks, d.nblocks);
}

// One DepthDecodeDesc: the item's code is at code_dev, its depth goes to dpt (pitch in floats)
inline void set_depth_decode_desc(DepthDecodeDesc& d, const DfkDepthDecodeItem& it, int code_size,
                                  const float* code_dev, float* dpt, uint32_t dpt_pitch, int* max_blocks)
{
  d.prx = view_of(&it.prx_orig);
  d.jac = view_of(&it.prx_jac);
  d.dpt = dpt;
  d.dpt_pitch = dpt_pitch;
  d.code = code_dev;
  d.width = (int)it.dpt.width;
  d.height = (int)it.dpt.height;
  d.nblocks = update_depth_blocks(d.width, d.height);
  d.vector = update_depth_vector(code_size, d.code, d.jac) ? 1 : 0;
  *max_blocks = std::max(*max_blocks, d.nblocks);
}

// n self-resetting tickets of a batched kernel: they must be zero when first used, so a buffer that grows is zeroed
// whole
inline DfkStatus ensure_tickets(DfkHandle h, DeviceBuf<unsigned int>& t, size_t n, const char* alloc_what,
                                const char* memset_what)
{
  if (t.cap >= n) return DFK_OK;
  DFK_CUDA(h, t.ensure(n), alloc_what);
  DFK_CUDA(h, cudaMemsetAsync(t.ptr, 0, sizeof(unsigned int) * t.cap, h->stream), memset_what);
  return DFK_OK;
}

// ---------------------------------------------------------------------------- dense RunStep (dfk_api.cu)
// The RunStep kernel a batch runs on (the Gram mode, the code size and the grad1 layout decide) and its launch shape
struct StepKernel {
  bool tc = false, wide = false;
  int tile_px = 0, max_ctas = 0;
  size_t pfloats = 0;  // floats per partial
};

DfkStatus choose_step_kernel(DfkHandle h, const DfkSfmWorkItem* items, int n, int code_size, StepKernel* k);
DfkStatus build_items(DfkHandle h, const DfkSfmWorkItem* items, int n, int code_size, int tile_px, int max_ctas,
                      const float* codes_dev, SfmItemDev* out, SfmLaunchPlan* plan);
void plan_tiles(SfmItemDev* items, int n, int max_ctas, SfmLaunchPlan* plan);
DfkStatus launch_step(DfkHandle h, const StepKernel& k, int code_size, const SfmItemDev* items_dev, int n,
                      const SfmLaunchPlan& plan, float* partials_dev, float* records_dev);

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
inline cudaError_t host_block(std::vector<unsigned char>& v, size_t bytes, unsigned char** p)
{
  v.assign(bytes, 0);
  *p = v.data();
  return cudaSuccess;
}
inline cudaError_t host_block(PinnedBuf<unsigned char>& b, size_t bytes, unsigned char** p)
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
