// dfk_api_sparse.cu -- C ABI of libdfk.so (see include/dfk.h), sparse factors: the reprojection and sparse geometric
// factors (single and batched linearisation, batched error), keypoint matching and ORB detection.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>

#include "dfk.h"
#include "dfk_host.h"
#include "dfk_internal.h"
#include "dfk_orb_model.h"

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

}  // extern "C"
