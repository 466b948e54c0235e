// dfk_api_sparse.cu -- C ABI of libdfk.so (see include/dfk.h), sparse factors: the reprojection and sparse geometric
// factors (single and batched linearisation, batched error), keypoint matching and ORB detection.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "dfk.h"
#include "dfk_host.h"
#include "dfk_internal.h"
#include "dfk_orb_model.h"
#include "dfk_orb_pyramid_model.h"

using namespace dfk;

extern "C" {

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
    Staged<DfkReprojectionItem> st;
    DFK_TRY(stage(h, "[ReprojectionFactor::linearize] ", false, &it, 1, code_size, n_out * sizeof(float), h->sparse_host,
                  h->sparse_dev, &st));
    const float2* d_query = st.payload.at(h->sparse_dev.ptr);
    float* d_rows = reinterpret_cast<float*>(h->sparse_dev.ptr + st.bytes);
    DFK_CUDA(h, launch_reprojection_rows(code_size, st.descs.at(h->sparse_host.ptr)[0], d_query,
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
    Staged<DfkReprojectionItem> st;
    DFK_TRY(stage(h, "[ReprojectionFactor::linearize batch] ", true, items, n, code_size, 0, h->staging, h->rep_dev, &st));
    const float2* query_dev = st.payload.at(h->rep_dev.ptr);
    DFK_CUDA(h, launch_reprojection_records(code_size, st.descs.at(h->rep_dev.ptr), n,
                                            query_dev, query_dev + st.total, h->params.sfmparams.avg_dpt, records_dev,
                                            h->stream),
             "[ReprojectionFactor::linearize batch] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

namespace {

// Validates and stages the items of a matching batch (*items_dev); max_n0 / queries / hyp_total / max_iterations
// describe the batch.  ransac: the camera and RANSAC parameters are checked too.
DfkStatus stage_match(DfkHandle h, const char* what, const DfkMatchItem* items, int n, bool ransac,
                      const MatchItemDev** items_dev, int* max_n0, int* max_iterations, size_t* queries,
                      size_t* hyp_total)
{
  const std::string w(what);
  if (!items || n < 1 || n > 65535)  // blockIdx.y of the kernels is the item
    return fail(h, DFK_ERR_INVALID_ARG, w + "null argument / number of items not in [1, 65535]");
  Staging s(h->staging);
  const Part<MatchItemDev> descs = s.add<MatchItemDev>(n);
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
    MatchItemDev& d = descs.at(s.host())[i];
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
  *queries = (size_t)total;
  DFK_TRY(s.upload(h, h->match_items, w));
  *items_dev = descs.at(s.dev);
  return DFK_OK;
}

}  // namespace

DfkStatus dfk_hamming_match_batch(DfkHandle h, const DfkMatchItem* items, int n, int32_t* matches_dev)
{
  return guarded(h, [&] {
    const char* what = "[BFMatcher::match batch] ";
    if (!matches_dev) return fail(h, DFK_ERR_INVALID_ARG, std::string(what) + "null output");
    DeviceGuard guard(h->device);
    const MatchItemDev* items_dev = nullptr;
    int max_n0 = 0, max_it = 0;
    size_t total = 0, hyp = 0;
    DFK_TRY(stage_match(h, what, items, n, false, &items_dev, &max_n0, &max_it, &total, &hyp));
    DFK_CUDA(h, launch_hamming_match(items_dev, n, max_n0, reinterpret_cast<int2*>(matches_dev), h->stream),
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
    const MatchItemDev* items_dev = nullptr;
    int max_n0 = 0, max_it = 0;
    size_t total = 0, hyp = 0;
    DFK_TRY(stage_match(h, what, items, n, true, &items_dev, &max_n0, &max_it, &total, &hyp));
    // [matches (int2 per query) | counts (int per hypothesis slot) | selections (int3 per item)]
    Layout L;
    const Part<int2> match_at = L.add<int2>(total);
    const Part<int> count_at = L.add<int>(hyp);
    const Part<int3> sel_at = L.add<int3>(n);
    DFK_CUDA(h, h->match_scratch.ensure(L.bytes), "[ReprojectionFactor matches batch] scratch allocation failed");
    unsigned char* base = h->match_scratch.ptr;
    int3* sel = ransac_dev ? reinterpret_cast<int3*>(ransac_dev) : sel_at.at(base);
    DFK_CUDA(h, launch_reprojection_match(items_dev, n, max_n0, max_it, match_at.at(base), count_at.at(base), sel,
                                          reinterpret_cast<int3*>(matches_dev), counts_dev, h->stream),
             "[ReprojectionFactor matches batch] kernel launch failed");
    h->launches += 4;
    return DFK_OK;
  });
}

}  // extern "C"

namespace {

// The one-level detector's plan over its items (images, or (image, level) pairs of a pyramid): each item's
// OrbItemDev and the scratch sizes and launch shape of the batch.
struct OrbPlan {
  long long rows = 0, segs = 0, corners = 0, map = 0, blur = 0;
  int max_rw = 0, max_rh = 0, max_cc = 0, max_segs = 0, max_cap = 0, max_nf = 0;

  // An item of w x h pixels (its image pointer is set by the caller); its rows follow the rows before it
  void add(OrbItemDev& d, int w, int h, int nfeatures, int threshold, int capacity)
  {
    const bool big = w >= DFK_OM_MIN_SIZE && h >= DFK_OM_MIN_SIZE;
    d = OrbItemDev{};
    d.rw = big ? w - 2 * DFK_OM_EDGE : 0;
    d.rh = big ? h - 2 * DFK_OM_EDGE : 0;
    d.tiles_x = (d.rw + kOrbTileW - 1) / kOrbTileW;
    d.tiles_y = (d.rh + kOrbTileH - 1) / kOrbTileH;
    d.nfeatures = nfeatures;
    d.threshold = threshold;
    d.capacity = capacity;
    d.out_begin = (int)std::min(rows, (long long)INT32_MAX);
    d.map_begin = (size_t)map;
    d.seg_begin = (int)std::min(segs, (long long)INT32_MAX);
    d.corner_begin = (int)std::min(corners, (long long)INT32_MAX);
    d.corner_cap = ((d.rw + 1) / 2) * ((d.rh + 1) / 2);  // one corner per 2 x 2 pixels at most survives NMS
    d.blur_begin = (size_t)blur;
    rows += capacity;
    segs += (long long)d.rh * d.tiles_x;
    corners += d.corner_cap;
    map += (long long)d.rw * d.rh;
    if (big) blur += (long long)(d.rw + 2 * DFK_OM_PATTERN_R) * (d.rh + 2 * DFK_OM_PATTERN_R);
    max_rw = std::max(max_rw, d.rw);
    max_rh = std::max(max_rh, d.rh);
    max_cc = std::max(max_cc, d.corner_cap);
    max_segs = std::max(max_segs, d.rh * d.tiles_x);
    max_cap = std::max(max_cap, capacity);
    max_nf = std::max(max_nf, nfeatures);
  }
  bool too_big() const { return rows > INT32_MAX || corners > INT32_MAX || segs > INT32_MAX; }

  // The detector's scratch for n items, as parts of L: [hist | stats | segments | corner positions | keys | angles |
  // row map | score maps | blurred images]
  struct Parts {
    Part<int> hist, stats, seg;
    Part<uint32_t> pos, key;
    Part<float> angle;
    Part<int> rows;
    Part<uint8_t> map, blur;
    OrbScratchDev at(unsigned char* base) const
    {
      return OrbScratchDev{map.at(base), seg.at(base), hist.at(base), stats.at(base), pos.at(base), key.at(base),
                           angle.at(base), rows.at(base), blur.at(base)};
    }
  };
  Parts scratch(Layout& L, int n) const
  {
    return Parts{L.add<int>(256 * (size_t)n), L.add<int>(4 * (size_t)n), L.add<int>((size_t)segs),
                   L.add<uint32_t>((size_t)corners), L.add<uint32_t>((size_t)corners), L.add<float>((size_t)corners),
                   L.add<int>((size_t)rows), L.add<uint8_t>((size_t)map), L.add<uint8_t>((size_t)blur)};
  }
  cudaError_t launch(const OrbItemDev* items_dev, int n, const OrbScratchDev& s, float* keypoints,
                     uint8_t* descriptors, float* angles, float* responses, int* counts, cudaStream_t stream) const
  {
    return launch_orb_detect(items_dev, n, s, max_rw, max_rh, max_cc, max_segs, max_cap, max_nf, keypoints,
                             descriptors, angles, responses, counts, stream);
  }
  int launches() const { return max_rw > 0 ? 7 : 5; }
};

// The checks an ORB item of either call shares; the failure text, or null
const char* orb_item_error(const DfkImage& im, int nfeatures, int fast_threshold, int capacity)
{
  if (!im.ptr || im.width > DFK_ORB_MAX_SIDE || im.height > DFK_ORB_MAX_SIDE || im.pitch_bytes < im.width)
    return "image needs a pointer, width and height <= DFK_ORB_MAX_SIDE and pitch_bytes >= width";
  if (nfeatures < 1 || nfeatures > DFK_MATCH_MAX_QUERIES) return "nfeatures not in [1, DFK_MATCH_MAX_QUERIES]";
  if (fast_threshold < 0 || fast_threshold > 255) return "fast_threshold not in [0, 255]";
  if (capacity < nfeatures) return "capacity < nfeatures";
  return nullptr;
}

// The size of level k of a pyramid item, and whether the level is built: at least DFK_OM_MIN_SIZE both ways.  The
// built levels k >= 1 are the resize items; the call counts them with this before it stages them.
bool orb_level(const DfkOrbPyramidItem& it, int k, int* lw, int* lh)
{
  const float scale = dfk_opm_level_scale(it.scale_factor, k);
  *lw = k ? dfk_opm_level_size((int)it.image.width, scale) : (int)it.image.width;
  *lh = k ? dfk_opm_level_size((int)it.image.height, scale) : (int)it.image.height;
  return *lw >= DFK_OM_MIN_SIZE && *lh >= DFK_OM_MIN_SIZE;
}

}  // namespace

extern "C" {

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
    Staging st(h->staging);
    const Part<OrbItemDev> items_at = st.add<OrbItemDev>(n);
    OrbPlan plan;
    for (int i = 0; i < n; ++i) {
      const DfkOrbItem& it = items[i];
      if (const char* e = orb_item_error(it.image, it.nfeatures, it.fast_threshold, it.capacity))
        return fail(h, DFK_ERR_INVALID_ARG, w + e + " in item " + std::to_string(i));
      OrbItemDev& d = items_at.at(st.host())[i];
      plan.add(d, (int)it.image.width, (int)it.image.height, it.nfeatures, it.fast_threshold, it.capacity);
      d.img = static_cast<const uint8_t*>(it.image.ptr);
      d.pitch = it.image.pitch_bytes;
    }
    if (plan.too_big())
      return fail(h, DFK_ERR_INVALID_ARG, w + "more than 2^31 - 1 output rows or scratch entries in one call");
    DeviceGuard guard(h->device);
    Layout S;
    const OrbPlan::Parts scratch = plan.scratch(S, n);
    DFK_CUDA(h, h->orb_scratch.ensure(S.bytes), "[OrbDetector batch] scratch allocation failed");
    DFK_TRY(st.upload(h, h->orb_items, w));
    DFK_CUDA(h, plan.launch(items_at.at(st.dev), n, scratch.at(h->orb_scratch.ptr), keypoints_dev, descriptors_dev,
                            angles_dev, responses_dev, counts_dev, h->stream),
             "[OrbDetector batch] kernel launch failed");
    h->launches += plan.launches();
    return DFK_OK;
  });
}

DfkStatus dfk_orb_detect_pyramid_batch(DfkHandle h, const DfkOrbPyramidItem* items, int n, float* keypoints_dev,
                                       uint8_t* descriptors_dev, float* angles_dev, float* responses_dev,
                                       int32_t* octaves_dev, int32_t* counts_dev)
{
  static_assert(kOrbMaxLevels == DFK_ORB_MAX_LEVELS && DFK_OPM_MAX_LEVELS == DFK_ORB_MAX_LEVELS, "level bound");
  return guarded(h, [&] {
    const std::string w = "[OrbDetector pyramid batch] ";
    if (!items || n < 1 || n > 65535)  // gridDim.y of the gather kernel is the item
      return fail(h, DFK_ERR_INVALID_ARG, w + "null argument / number of items not in [1, 65535]");
    if (!keypoints_dev || !descriptors_dev || !counts_dev)
      return fail(h, DFK_ERR_INVALID_ARG, w + "null keypoint, descriptor or count output");
    if (((uintptr_t)keypoints_dev & 3) || ((uintptr_t)descriptors_dev & 15) || ((uintptr_t)angles_dev & 3) ||
        ((uintptr_t)responses_dev & 3) || ((uintptr_t)octaves_dev & 3) || ((uintptr_t)counts_dev & 3))
      return fail(h, DFK_ERR_INVALID_ARG, w + "descriptors must be 16-byte aligned, the other outputs 4-byte aligned");
    // validation, and each item's levels: one one-level item per (image, level), level images for k >= 1 while they
    // are at least 63 x 63 (a smaller level and every level after it has no features)
    long long subs = 0, out_rows = 0;
    size_t nres = 0;  // levels k >= 1 that are built: the resize items
    for (int i = 0; i < n; ++i) {
      const DfkOrbPyramidItem& it = items[i];
      const std::string at = " in item " + std::to_string(i);
      if (const char* e = orb_item_error(it.image, it.nfeatures, it.fast_threshold, it.capacity))
        return fail(h, DFK_ERR_INVALID_ARG, w + e + at);
      if (!(std::isfinite(it.scale_factor) && it.scale_factor > 1.0f))
        return fail(h, DFK_ERR_INVALID_ARG, w + "scale_factor must be finite and > 1" + at);
      if (it.nlevels < 1 || it.nlevels > DFK_ORB_MAX_LEVELS)
        return fail(h, DFK_ERR_INVALID_ARG, w + "nlevels not in [1, DFK_ORB_MAX_LEVELS]" + at);
      subs += it.nlevels;
      out_rows += it.capacity;
      for (int k = 1, lw, lh; k < it.nlevels; ++k) nres += orb_level(it, k, &lw, &lh);
    }
    if (subs > 65535)  // gridDim.z of the FAST kernel is the (image, level) item
      return fail(h, DFK_ERR_INVALID_ARG, w + "more than 65535 levels over the items of one call");
    if (out_rows > INT32_MAX) return fail(h, DFK_ERR_INVALID_ARG, w + "more than 2^31 - 1 output rows in one call");
    // one upload: [one-level items | gather items | resize items by level]
    Staging up(h->staging);
    const Part<OrbItemDev> sub_at = up.add<OrbItemDev>((size_t)subs);
    const Part<OrbGatherDev> gat_at = up.add<OrbGatherDev>(n);
    const Part<OrbResizeDev> res_at = up.add<OrbResizeDev>(nres);
    OrbItemDev* sub = sub_at.at(up.host());
    OrbGatherDev* gather = gat_at.at(up.host());
    // the resize items by level, their source and destination as offsets into the level images until those are
    // allocated (SIZE_MAX: the caller's image)
    struct LevelJob {
      OrbResizeDev r;
      size_t src, dst;
      const void* image;
    };
    std::vector<std::vector<LevelJob>> resize(DFK_ORB_MAX_LEVELS);
    std::vector<size_t> sub_level((size_t)subs, SIZE_MAX);  // each (image, level)'s image, as above
    OrbPlan plan;
    size_t level_bytes = 0;
    for (int i = 0, sb = 0; i < n; sb += items[i].nlevels, ++i) {
      const DfkOrbPyramidItem& it = items[i];
      int budget[DFK_ORB_MAX_LEVELS];
      dfk_opm_budgets(it.nfeatures, it.scale_factor, it.nlevels, budget);
      OrbGatherDev& g = gather[i];
      g.sub_begin = sb;
      g.nlevels = it.nlevels;
      g.out_begin = i ? gather[(size_t)i - 1].out_begin + items[i - 1].capacity : 0;
      g.capacity = it.capacity;
      int pw = (int)it.image.width, ph = (int)it.image.height;
      for (int k = 0; k < it.nlevels; ++k) {
        g.scale[k] = dfk_opm_level_scale(it.scale_factor, k);
        int lw, lh;
        const bool built = orb_level(it, k, &lw, &lh);
        if (built && k) {
          const size_t src = sub_level[(size_t)sb + k - 1];
          const size_t src_pitch = src == SIZE_MAX ? it.image.pitch_bytes : (size_t)pw;
          resize[(size_t)k].push_back(LevelJob{OrbResizeDev{nullptr, src_pitch, nullptr, pw, ph, lw, lh}, src,
                                               level_bytes, it.image.ptr});
          sub_level[(size_t)sb + k] = level_bytes;
          level_bytes += (size_t)lw * lh;
        }
        // a level with no budget, or too small, is an empty item
        const bool live = built && budget[k] > 0;
        plan.add(sub[(size_t)sb + k], live ? lw : 0, live ? lh : 0, budget[k], it.fast_threshold, it.capacity);
        sub[(size_t)sb + k].pitch = k && built ? (size_t)lw : it.image.pitch_bytes;
        pw = lw;
        ph = lh;
      }
    }
    if (plan.too_big())
      return fail(h, DFK_ERR_INVALID_ARG, w + "more than 2^31 - 1 staged rows or scratch entries in one call");
    DeviceGuard guard(h->device);
    // the detector's scratch, then [level images | staged keypoints | descriptors | angles | responses | counts]
    const size_t srows = (size_t)plan.rows;
    Layout S;
    const OrbPlan::Parts det = plan.scratch(S, (int)subs);
    const Part<uint8_t> lev_at = S.add<uint8_t>(level_bytes);
    const Part<float> kp_at = S.add<float>(2 * srows);
    const Part<uint8_t> desc_at = S.add<uint8_t>(32 * srows);
    const Part<float> ang_at = S.add<float>(srows), resp_at = S.add<float>(srows);
    const Part<int> cnt_at = S.add<int>((size_t)subs);
    DFK_CUDA(h, h->orb_scratch.ensure(S.bytes), "[OrbDetector pyramid batch] scratch allocation failed");
    unsigned char* base = h->orb_scratch.ptr;
    unsigned char* levels = lev_at.at(base);
    auto level_ptr = [&](size_t off, const void* image) {
      return off == SIZE_MAX ? static_cast<const uint8_t*>(image) : static_cast<const uint8_t*>(levels + off);
    };
    for (int i = 0, sb = 0; i < n; sb += items[i].nlevels, ++i)
      for (int k = 0; k < items[i].nlevels; ++k)
        sub[(size_t)sb + k].img = level_ptr(sub_level[(size_t)sb + k], items[i].image.ptr);
    OrbResizeDev* rh = res_at.at(up.host());
    for (const std::vector<LevelJob>& v : resize)
      for (const LevelJob& job : v) {
        *rh = job.r;
        rh->src = level_ptr(job.src, job.image);
        rh->dst = levels + job.dst;
        ++rh;
      }
    DFK_TRY(up.upload(h, h->orb_pyr_dev, w));
    // the chain of levels: level k of every image from its level k - 1
    for (int k = 1, j = 0; k < DFK_ORB_MAX_LEVELS; ++k) {
      const std::vector<LevelJob>& v = resize[(size_t)k];
      if (v.empty()) continue;
      int mw = 0, mh = 0;
      for (const LevelJob& job : v) {
        mw = std::max(mw, job.r.dw);
        mh = std::max(mh, job.r.dh);
      }
      DFK_CUDA(h, launch_orb_resize_level(res_at.at(up.dev) + j, (int)v.size(), mw, mh, h->stream),
               "[OrbDetector pyramid batch] kernel launch failed");
      j += (int)v.size();
      h->launches += 1;
    }
    DFK_CUDA(h, plan.launch(sub_at.at(up.dev), (int)subs, det.at(base), kp_at.at(base), desc_at.at(base),
                            ang_at.at(base), resp_at.at(base), cnt_at.at(base), h->stream),
             "[OrbDetector pyramid batch] kernel launch failed");
    h->launches += plan.launches();
    const OrbStagingDev st{kp_at.at(base), desc_at.at(base), ang_at.at(base), resp_at.at(base), cnt_at.at(base)};
    DFK_CUDA(h, launch_orb_gather(gat_at.at(up.dev), n, sub_at.at(up.dev), st, plan.max_cap, keypoints_dev,
                                  descriptors_dev, angles_dev, responses_dev, octaves_dev, counts_dev, h->stream),
             "[OrbDetector pyramid batch] kernel launch failed");
    h->launches += 1;
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
    Staged<DfkSparseGeometricItem> st;
    DFK_TRY(stage(h, "[SparseGeometricFactor::linearize] ", false, &it, 1, code_size, M * RW * sizeof(float),
                  h->sparse_host, h->sparse_dev, &st));
    float* d_rows = reinterpret_cast<float*>(h->sparse_dev.ptr + st.bytes);
    DFK_CUDA(h, launch_sparse_geometric_rows(code_size, st.descs.at(h->sparse_host.ptr)[0],
                                             st.payload.at(h->sparse_dev.ptr), h->params.sfmparams.avg_dpt,
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
    Staged<DfkSparseGeometricItem> st;
    DFK_TRY(stage(h, "[SparseGeometricFactor::linearize batch] ", true, items, n, code_size, 0, h->staging, h->geo_dev,
                  &st));
    DFK_CUDA(h, launch_sparse_geometric_records(code_size, st.descs.at(h->geo_dev.ptr), n,
                                                st.payload.at(h->geo_dev.ptr), h->params.sfmparams.avg_dpt,
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
    Staged<DfkReprojectionItem> st;
    DFK_TRY(stage(h, "[ReprojectionFactor::error batch] ", true, items, n, code_size, 0, h->staging, h->rep_dev, &st));
    const float2* query_dev = st.payload.at(h->rep_dev.ptr);
    DFK_CUDA(h, launch_reprojection_error(code_size, st.descs.at(h->rep_dev.ptr), n, query_dev,
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
    Staged<DfkSparseGeometricItem> st;
    DFK_TRY(stage(h, "[SparseGeometricFactor::error batch] ", true, items, n, code_size, 0, h->staging, h->geo_dev, &st));
    DFK_CUDA(h, launch_sparse_geometric_error(code_size, st.descs.at(h->geo_dev.ptr), n,
                                              st.payload.at(h->geo_dev.ptr), h->params.sfmparams.avg_dpt,
                                              out_dev, h->stream),
             "[SparseGeometricFactor::error batch] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

}  // extern "C"
