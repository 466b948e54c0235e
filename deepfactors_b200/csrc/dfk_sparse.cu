// dfk_sparse.cu -- the sparse factors on the device: ReprojectionFactor::linearize
// (sources/core/gtsam/reprojection_factor.cpp:157-269), the same factors batched straight into normal-equation records
// (reprojection_records_kernel), and SparseGeometricFactor::linearize (second half of the file), rows and records
// (sparse_geometric_records_kernel).  Both records kernels share one Gram scaffold (gram_records).
//
// The reference evaluates this sparse keypoint factor on the CPU and, to read the code Jacobian at <= a few thousand
// keypoints, forces a device -> host mirror of the keyframe's WHOLE level-0 code-Jacobian pyramid
// (kf_->pyr_jac.GetCpuLevel(0), :193; 39 MB at 640x480, C = 32).  Here the rows are gathered where the data lives: one
// thread per match reads its C-float Jacobian row and proximity, decodes the depth, warps the keypoint, and writes the
// two rows of the JacobianFactor [ dErr/dPose0 (6) | dErr/dPose1 (6) | dErr/dCode0 (C) | b (1) ]; ~1 MB goes back.
//
// Per match i (query keypoint in the keyframe, train keypoint in the frame):
//   (xi, yi)  = integer pixel of the query (the reference indexes with (int)query.x / implicit size_t conversions, :194-195,
//               and FindCorrespondence takes std::size_t x, y, warping.h:206)
//   dpt0      = DepthFromCode(c0, prx_J_cde, prx_0code, avg_dpt = 2)                       :198, warping.h:52-69
//   corr      = FindCorrespondence(xi, yi, dpt0, cam, pose10, 1, 0, check_bounds = false)  :199-200  (valid <=> Z > 0)
//   invalid   -> zero rows                                                                   :204-212
//   J_cde     = FindCorrespondenceJacobianCode (2 x C)                                       :217-218, warping.h:294-313
//   J_pose10  = FindCorrespondenceJacobianPose (2 x 6);  J_pose0/1 = J_pose10 * pose10_J_pose0/1   :221-229
//   diff      = pix1(train) - corr.pix1 ; err = |diff| ; w = CauchyWeight(err, huber_delta)  :232-239, m_estimators.h:43-48
//   rows *= w ; total_err += err^2 ; rows /= sigma                                           :242-253
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "dfk_geom.cuh"
#include "dfk_internal.h"

namespace dfk {

namespace {

// The per-match body of ReprojectionFactor::linearize: writes the two rows r0, r1 of factor `it`'s match (q, tr) (zero
// when the correspondence is invalid) and its squared unweighted error; returns whether the correspondence is valid.
// Shared by the single-factor kernel and the batched one, so the batched rows are those of dfk_reprojection_linearize by
// construction.
// kJac = false writes b (r0[12 + C], r1[12 + C]) and err2 only, so the Jacobian work is dead code.
template <int C, bool kJac = true>
__device__ __forceinline__ bool reprojection_match_rows(const ReprojItemDev& it, float2 q, float2 tr, float avg_dpt,
                                                        float* r0, float* r1, float* err2)
{
  constexpr int RW = 13 + C;
  const SparsePose& sp = it.sp;
  const float* __restrict__ code = it.code;
  const View prx_orig = it.prx_orig, jac = it.jac;
  const int width = it.width, height = it.height;
  const float cauchy_delta = it.cauchy_delta, sigma = it.sigma;
  const int xi = (int)q.x, yi = (int)q.y;
  bool valid = xi >= 0 && yi >= 0 && xi < width && yi < height;  // the reference would read out of bounds
  float dpt0 = 0.f, X = 0.f, Y = 0.f, Z = 0.f, px = 0.f, py = 0.f, pz = 0.f, xn = 0.f, yn = 0.f;
  const float* jr = nullptr;
  if (valid) {
    jr = jac.ptr + (size_t)yi * jac.pitch + (size_t)xi * C;
    float dot = 0.0f;
    for (int k = 0; k < C; ++k) dot += __ldg(jr + k) * code[k];  // (prx_J_cde * code)(0), left to right
    const float prx = __ldg(prx_orig.ptr + (size_t)yi * prx_orig.pitch + xi) + dot;
    dpt0 = avg_dpt / prx - avg_dpt;
    // Reproject + se3 * pt (quaternion rotate as Sophus does)
    xn = ((float)xi - sp.u0) / sp.fx;
    yn = ((float)yi - sp.v0) / sp.fy;
    const float P0 = xn * dpt0, P1 = yn * dpt0, P2 = dpt0;
    float uv0 = sp.q[1] * P2 - sp.q[2] * P1, uv1 = sp.q[2] * P0 - sp.q[0] * P2, uv2 = sp.q[0] * P1 - sp.q[1] * P0;
    uv0 += uv0; uv1 += uv1; uv2 += uv2;
    px = (P0 + sp.q[3] * uv0) + (sp.q[1] * uv2 - sp.q[2] * uv1);
    py = (P1 + sp.q[3] * uv1) + (sp.q[2] * uv0 - sp.q[0] * uv2);
    pz = (P2 + sp.q[3] * uv2) + (sp.q[0] * uv1 - sp.q[1] * uv0);
    X = px + sp.t[0]; Y = py + sp.t[1]; Z = pz + sp.t[2];
    valid = Z > 0.0f;  // depth > min_dpt (0); bounds are not checked (check_bounds = false)
  }
  if (!valid) {
    if constexpr (kJac) {
      for (int k = 0; k < RW; ++k) { r0[k] = 0.0f; r1[k] = 0.0f; }
    } else {
      r0[RW - 1] = 0.0f;
      r1[RW - 1] = 0.0f;
    }
    *err2 = 0.0f;
    return false;
  }
  const float u = sp.fx * X / Z + sp.u0, v = sp.fy * Y / Z + sp.v0;  // Project
  // ProjectPointJacobian
  const float c00 = sp.fx / Z, c02 = -(sp.fx * X) / Z / Z, c11 = sp.fy / Z, c12 = -(sp.fy * Y) / Z / Z;
  // corr_J_pose10 = dCam * [I | -hat(R pt)]
  const float A0[6] = {c00, 0.f, c02, c02 * py, c00 * pz - c02 * px, -(c00 * py)};
  const float A1[6] = {0.f, c11, c12, c12 * py - c11 * pz, -(c12 * px), c11 * px};
  // pix1_J_dpt = dCam * R * (xn, yn, 1);  dpt_J_prx = -avg / prx^2
  const float q0 = sp.R[0] * xn + sp.R[1] * yn + sp.R[2];
  const float q1 = sp.R[3] * xn + sp.R[4] * yn + sp.R[5];
  const float q2 = sp.R[6] * xn + sp.R[7] * yn + sp.R[8];
  const float pr = avg_dpt / (avg_dpt + dpt0);
  const float dJ = -avg_dpt / (pr * pr);
  const float jd0 = (c00 * q0 + c02 * q2) * dJ, jd1 = (c11 * q1 + c12 * q2) * dJ;
  const float d0 = tr.x - u, d1 = tr.y - v;
  const float err = sqrtf(d0 * d0 + d1 * d1);
  // CauchyWeight(x, delta): a = delta / x; abs(a) / sqrt(2) * sqrt(log(1 + 1 / a / a)).  NaN at err == 0 (a = inf), as in
  // the reference (m_estimators.h:44-48): a match that lands exactly on its keypoint makes the whole factor NaN.
  // log1pf, not logf(1 + s): the reference's float 1 + 1 / a^2 rounds away the weight's digits once a >> 1 and gives
  // w = 0 below err = delta / 4096 (the true weight tends to 1 / sqrt(2)); log1pf keeps it to fp32 accuracy.
  const float a = cauchy_delta / err;
  const float w = fabsf(a) / sqrtf(2.0f) * sqrtf(log1pf(1.0f / a / a));
  if constexpr (kJac) {
    for (int j = 0; j < 6; ++j) {
      float s00 = 0.f, s01 = 0.f, s10 = 0.f, s11 = 0.f;
      for (int k = 0; k < 6; ++k) {
        s00 += A0[k] * sp.P0[k * 6 + j];
        s01 += A0[k] * sp.P1[k * 6 + j];
        s10 += A1[k] * sp.P0[k * 6 + j];
        s11 += A1[k] * sp.P1[k * 6 + j];
      }
      r0[j] = s00 * w / sigma; r0[6 + j] = s01 * w / sigma;
      r1[j] = s10 * w / sigma; r1[6 + j] = s11 * w / sigma;
    }
    for (int k = 0; k < C; ++k) {
      const float jc = __ldg(jr + k);
      r0[12 + k] = jd0 * jc * w / sigma;
      r1[12 + k] = jd1 * jc * w / sigma;
    }
  }
  r0[12 + C] = d0 * w / sigma;
  r1[12 + C] = d1 * w / sigma;
  *err2 = err * err;
  return true;
}

// One thread per match of the single factor `it`: rows 2m and 2m + 1, err2[m].
template <int C>
__global__ void __launch_bounds__(128)
reprojection_rows_kernel(const __grid_constant__ ReprojItemDev it, const float2* __restrict__ query,
                         const float2* __restrict__ train, float avg_dpt, float* __restrict__ rows, float* __restrict__ err2)
{
  constexpr int RW = 13 + C;
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= it.num_matches) return;
  const int i = it.match_begin + m;
  float* r0 = rows + (size_t)(2 * m) * RW;
  float e2;
  reprojection_match_rows<C>(it, query[i], train[i], avg_dpt, r0, r0 + RW, &e2);
  err2[m] = e2;
}

// Geometry of a batched records kernel: rows of RW floats, RPI rows per item (2 per reprojection match, 1 per geometric
// point), NT threads, CH items per chunk (their RPI CH rows are the dynamic shared memory), NS CTAs per factor.  CTA s of
// a factor owns the slice [s NT EPT, (s + 1) NT EPT) of the packed upper triangle of the augmented RW^2 Gram, EPT entries
// per thread; every CTA of the factor recomputes the chunk rows itself.
template <int RW_, int RPI_, int NT_, int CH_, int NS_>
struct GramCfg {
  static constexpr int RW = RW_, RPI = RPI_, NT = NT_, CH = CH_, NS = NS_;
  static constexpr int NE = RW * (RW + 1) / 2;
  static constexpr int EPT = (NE + NT * NS - 1) / (NT * NS);
  static constexpr size_t SMEM = sizeof(float) * RPI * CH * RW;
};
template <int C>
using RepCfg = GramCfg<13 + C, 2, C >= 64 ? 256 : 128, C >= 64 ? 64 : 128, 1>;
// C = 128: 36315 entries, four CTAs of 256 x 36 per factor
template <int C>
using GeoCfg = GramCfg<13 + 2 * C, 1, C >= 32 ? 256 : 128, C >= 128 ? 64 : 128, C >= 128 ? 4 : 1>;

// a factor's descriptor into shared memory, word by word; ends with the barrier that publishes it
template <int NT, class Item>
__device__ __forceinline__ void load_item(const Item* __restrict__ src_item, Item& it)
{
  static_assert(sizeof(Item) % 4 == 0, "descriptor copied as words");
  const uint32_t* src = reinterpret_cast<const uint32_t*>(src_item);
  uint32_t* dst = reinterpret_cast<uint32_t*>(&it);
  for (int k = threadIdx.x; k < (int)(sizeof(Item) / 4); k += NT) dst[k] = src[k];
  __syncthreads();
}

// The Gram scaffold of the batched kernels.  Factor blockIdx.x has M items; item_rows(i, rows) writes item i's RPI rows
// and returns whether it is valid.  The items are walked in chunks of CH; every thread of the chunk writes one item's
// rows into shared memory, then every thread sums the chunk's rows, in row order, for the Gram entries it owns and adds
// that chunk sum to its running totals.  No atomics: a factor's record depends on that factor only, and each entry has
// one owner whatever the grid.  The epilogue writes the RunStep record layout: JtJ = the (RW-1) upper block of the Gram
// of [A | b], Jtr = -A^T b, residual = b^T b, inliers = valid items.
template <class Cfg, class RowFn>
__device__ __forceinline__ void gram_records(int M, float* __restrict__ records, RowFn item_rows)
{
  constexpr int RW = Cfg::RW, NP = RW - 1, NH = NP * (NP + 1) / 2, REC = NH + NP + 2;
  constexpr int NT = Cfg::NT, CH = Cfg::CH, EPT = Cfg::EPT, RPI = Cfg::RPI;
  extern __shared__ float rows[];  // [RPI CH][RW]
  const int e0 = blockIdx.y * NT * EPT;  // first entry of this CTA's slice
  // the entries this thread owns: e = e0 + threadIdx.x + k NT of the packed upper triangle, (ea[k], eb[k]) in [0, RW)^2
  int ea[EPT], eb[EPT];
  {
    int a = 0, first = 0;  // first = packed index of (a, a)
#pragma unroll
    for (int k = 0; k < EPT; ++k) {
      const int e = e0 + threadIdx.x + k * NT;
      while (a < RW - 1 && e >= first + (RW - a)) { first += RW - a; ++a; }
      ea[k] = e < Cfg::NE ? a : 0;
      eb[k] = e < Cfg::NE ? a + (e - first) : 0;
    }
  }
  float acc[EPT];
#pragma unroll
  for (int k = 0; k < EPT; ++k) acc[k] = 0.0f;
  int inliers = 0;
  for (int base = 0; base < M; base += CH) {
    const int cnt = min(CH, M - base);
    bool valid = false;
    if ((int)threadIdx.x < cnt) valid = item_rows(base + threadIdx.x, rows + RPI * threadIdx.x * RW);
    inliers += __syncthreads_count(valid);  // also the barrier between the row writes and the Gram
    // the chunk's rows are summed on their own and then added to the running total: an entry is a chain of RPI CH
    // products plus one add per chunk, not one serial chain over all rows (whose fp32 error grows with M)
    float part[EPT];
#pragma unroll
    for (int k = 0; k < EPT; ++k) part[k] = 0.0f;
    for (int r = 0; r < RPI * cnt; ++r) {
      const float* row = rows + r * RW;
#pragma unroll
      for (int k = 0; k < EPT; ++k) part[k] = fmaf(row[ea[k]], row[eb[k]], part[k]);
    }
#pragma unroll
    for (int k = 0; k < EPT; ++k) acc[k] += part[k];
    __syncthreads();
  }
  float* rec = records + (size_t)blockIdx.x * REC;
#pragma unroll
  for (int k = 0; k < EPT; ++k) {
    if (e0 + (int)threadIdx.x + k * NT >= Cfg::NE) break;
    const int a = ea[k], b = eb[k];
    if (b < NP) rec[a * NP - (a * (a - 1)) / 2 + (b - a)] = acc[k];  // JtJ
    else if (a < NP) rec[NH + a] = -acc[k];                          // Jtr = -A^T b
    else rec[NH + NP] = acc[k];                                      // residual = b^T b
  }
  if (threadIdx.x == 0 && blockIdx.y == 0) rec[NH + NP + 1] = __uint_as_float((uint32_t)inliers);
}

// One CTA per factor, two rows per match (row 2i, then 2i + 1).
template <int C>
__global__ void __launch_bounds__(RepCfg<C>::NT)
reprojection_records_kernel(const ReprojItemDev* __restrict__ items, const float2* __restrict__ query,
                            const float2* __restrict__ train, float avg_dpt, float* __restrict__ records)
{
  __shared__ ReprojItemDev it;
  load_item<RepCfg<C>::NT>(items + blockIdx.x, it);
  gram_records<RepCfg<C>>(it.num_matches, records, [&](int m, float* r0) {
    const int i = it.match_begin + m;
    float e2;
    return reprojection_match_rows<C>(it, query[i], train[i], avg_dpt, r0, r0 + 13 + C, &e2);
  });
}

// ---------------------------------------------------------------------------------------------------------------------
// SparseGeometricFactor::linearize (sources/core/gtsam/sparse_geometric_factor.cpp:157-271): one row per sampled pixel of
// keyframe 0 -- the depth keyframe 1 decodes at the (nearest-neighbour) correspondence against the depth of the warped
// point.  The reference runs it on the CPU over host mirrors of BOTH keyframes' level-0 proximity / code-Jacobian
// pyramids and of kf1's depth gradient (:181-183, :207-209, :220).  One thread per point:
//   dpt0   = DepthFromCode(c0, prx0_J_cde, prx0_0code, avg_dpt)                                   :186
//   corr   = FindCorrespondence(pt, dpt0, cam, pose10)  (border 1, min_dpt 0, bounds checked)     :187-198
//   dpt1_p = corr.tpt.z ; pix1_nn = (int) corr.pix1 ; dpt1 = DepthFromCode(c1, kf1 @ pix1_nn)      :201-210
//   err    = dpt1 - dpt1_p                                                                         :213
//   J_pose0/1 = ( TransformJacobianPose.row(2) - dpt_grad * corr_J_pose10 ) * pose10_J_pose0/1     :223-238
//   J_cde0 = (R ray).z * DepthJacobianPrx(dpt0) * prx0_J_cde - dpt_grad * corr_J_cde0              :241-246
//   J_cde1 = -DepthJacobianPrx(dpt1) * prx1_J_cde                                                  :249
//   everything * HuberWeight(err, huber_delta)                                                     :252-258
// The decode and the validity chain use round-to-nearest intrinsics in the reference's operation order (as the dense
// kernels do), so the set of valid rows and the nearest-neighbour pixels are those of the CPU evaluation.
//
// The per-point body: writes the row r of factor `it`'s point pt (zero when the correspondence is invalid) and returns
// whether it is valid.  Shared by the single-factor kernel and the batched one, so the batched rows are those of
// dfk_sparse_geometric_linearize by construction.
// kJac = false writes b (r[12 + 2 C]) only, so the Jacobian work is dead code.
template <int C, bool kJac = true>
__device__ __forceinline__ bool sparse_geometric_point_row(const GeoItemDev& it, int2 pt, float avg_dpt, float* r)
{
  constexpr int RW = 13 + 2 * C;
  const SparsePose& sp = it.sp;
  const float cam_w = it.cam_w, cam_h = it.cam_h;
  const float* __restrict__ code0 = it.code0;
  const float* __restrict__ code1 = it.code1;
  const View prx0 = it.prx0, jac0 = it.jac0, prx1 = it.prx1, jac1 = it.jac1, grad1 = it.grad1;
  const int width = it.width, height = it.height;
  const float huber_delta = it.huber_delta;
  bool valid = pt.x >= 0 && pt.y >= 0 && pt.x < width && pt.y < height;  // the reference would read out of bounds
  Warped w;
  w.valid = false;
  float dpt0 = 0.0f;
  const float* jr0 = nullptr;
  if (valid) {
    jr0 = jac0.ptr + (size_t)pt.y * jac0.pitch + (size_t)pt.x * C;
    float dot = 0.0f;
    for (int k = 0; k < C; ++k) dot = __fadd_rn(dot, __fmul_rn(__ldg(jr0 + k), code0[k]));  // (prx_J_cde * code)(0), left to right
    dpt0 = prx_to_depth(__fadd_rn(__ldg(prx0.ptr + (size_t)pt.y * prx0.pitch + pt.x), dot), avg_dpt);
    w = warp_pixel((float)pt.x, (float)pt.y, dpt0, sp.q, sp.t, sp.fx, sp.fy, sp.u0, sp.v0, 1.0f, __fsub_rn(cam_w, 1.0f),
                   __fsub_rn(cam_h, 1.0f), 0.0f);
    valid = w.valid;
  }
  if (!valid) {
    if constexpr (kJac) {
      for (int k = 0; k < RW; ++k) r[k] = 0.0f;
    } else {
      r[RW - 1] = 0.0f;
    }
    return false;
  }
  const int nx = (int)w.u, ny = (int)w.v;  // pix1.cast<int>()
  const float* jr1 = jac1.ptr + (size_t)ny * jac1.pitch + (size_t)nx * C;
  float dot1 = 0.0f;
  for (int k = 0; k < C; ++k) dot1 = __fadd_rn(dot1, __fmul_rn(__ldg(jr1 + k), code1[k]));
  const float dpt1 = prx_to_depth(__fadd_rn(__ldg(prx1.ptr + (size_t)ny * prx1.pitch + nx), dot1), avg_dpt);
  const float err = __fsub_rn(dpt1, w.tz);
  const float g0 = __ldg(grad1.ptr + (size_t)ny * grad1.pitch + 2 * nx), g1 = __ldg(grad1.ptr + (size_t)ny * grad1.pitch + 2 * nx + 1);
  const float X = w.tx, Y = w.ty, Z = w.tz;
  const float c00 = sp.fx / Z, c02 = -(sp.fx * X) / Z / Z, c11 = sp.fy / Z, c12 = -(sp.fy * Y) / Z / Z;  // ProjectPointJacobian
  const float A0[6] = {c00, 0.f, c02, c02 * w.py, c00 * w.pz - c02 * w.px, -(c00 * w.py)};  // corr_J_pose10 = dCam [I | -hat(R pt)]
  const float A1[6] = {0.f, c11, c12, c12 * w.py - c11 * w.pz, -(c12 * w.px), c11 * w.px};
  const float T2[6] = {0.f, 0.f, 1.f, w.py, -w.px, 0.f};  // row 2 of TransformJacobianPose
  float B[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) B[k] = T2[k] - (g0 * A0[k] + g1 * A1[k]);
  const float hw = huber_weight(err, huber_delta);
  if constexpr (kJac) {
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        s0 += B[k] * sp.P0[k * 6 + j];
        s1 += B[k] * sp.P1[k * 6 + j];
      }
      r[j] = s0 * hw;
      r[6 + j] = s1 * hw;
    }
    // pix1_J_dpt = dCam * R * ray ; (R ray).z ; dpt_J_prx = -avg / prx^2
    const float q0 = sp.R[0] * w.xn + sp.R[1] * w.yn + sp.R[2];
    const float q1 = sp.R[3] * w.xn + sp.R[4] * w.yn + sp.R[5];
    const float q2 = sp.R[6] * w.xn + sp.R[7] * w.yn + sp.R[8];
    const float pr0 = avg_dpt / (avg_dpt + dpt0), dJ0 = -avg_dpt / (pr0 * pr0);
    const float jd0 = (c00 * q0 + c02 * q2) * dJ0, jd1 = (c11 * q1 + c12 * q2) * dJ0;
    const float e0 = (q2 * dJ0 - (g0 * jd0 + g1 * jd1)) * hw;
    const float pr1 = avg_dpt / (avg_dpt + dpt1), dJ1 = -avg_dpt / (pr1 * pr1);
    const float e1 = -dJ1 * hw;
    for (int k = 0; k < C; ++k) {
      r[12 + k] = e0 * __ldg(jr0 + k);
      r[12 + C + k] = e1 * __ldg(jr1 + k);
    }
  }
  r[12 + 2 * C] = err * hw;
  return true;
}

// One thread per point of the single factor `it`: row m.
template <int C>
__global__ void __launch_bounds__(128)
sparse_geometric_rows_kernel(const __grid_constant__ GeoItemDev it, const int2* __restrict__ points, float avg_dpt,
                             float* __restrict__ rows)
{
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= it.num_points) return;
  sparse_geometric_point_row<C>(it, points[it.point_begin + m], avg_dpt, rows + (size_t)m * (13 + 2 * C));
}

// Factor blockIdx.x, entry slice blockIdx.y (GeoCfg<C>::NS CTAs per factor), one row per point.
template <int C>
__global__ void __launch_bounds__(GeoCfg<C>::NT)
sparse_geometric_records_kernel(const GeoItemDev* __restrict__ items, const int2* __restrict__ points, float avg_dpt,
                                float* __restrict__ records)
{
  __shared__ GeoItemDev it;
  load_item<GeoCfg<C>::NT>(items + blockIdx.x, it);
  gram_records<GeoCfg<C>>(it.num_points, records, [&](int m, float* r) {
    return sparse_geometric_point_row<C>(it, points[it.point_begin + m], avg_dpt, r);
  });
}

// ---------------------------------------------------------------------------------------------------------------------
// The error() half of both factors: b^T b and the valid items of factor blockIdx.x, nothing else.  One CTA of Cfg::CH
// threads per factor walks the items in the records kernel's chunks; thread t computes item base + t's b entries
// (item_b(i, b), RPI of them, zero when invalid) into shared memory, then thread 0 sums the chunk's RPI cnt squares in
// row order with the records kernel's fmaf chain and adds that chunk sum to the total.  That is exactly how gram_records
// forms the (RW-1, RW-1) entry of the augmented Gram, so out[2 f] is bit for bit the residual of factor f's record.
// out[2 f + 1] = valid items (u32 bits).
template <class Cfg, class BFn>
__device__ __forceinline__ void sparse_error(int M, float* __restrict__ out, BFn item_b)
{
  constexpr int RPI = Cfg::RPI, CH = Cfg::CH;
  __shared__ float bs[RPI * CH];
  float acc = 0.0f;
  int inliers = 0;
  for (int base = 0; base < M; base += CH) {
    const int cnt = min(CH, M - base);
    bool valid = false;
    if ((int)threadIdx.x < cnt) {
      float b[RPI];
      valid = item_b(base + threadIdx.x, b);
#pragma unroll
      for (int r = 0; r < RPI; ++r) bs[RPI * threadIdx.x + r] = b[r];
    }
    inliers += __syncthreads_count(valid);
    if (threadIdx.x == 0) {
      float part = 0.0f;
      for (int r = 0; r < RPI * cnt; ++r) part = fmaf(bs[r], bs[r], part);
      acc += part;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out[2 * (size_t)blockIdx.x] = acc;
    out[2 * (size_t)blockIdx.x + 1] = __uint_as_float((uint32_t)inliers);
  }
}

template <int C>
__global__ void __launch_bounds__(RepCfg<C>::CH)
reprojection_error_kernel(const ReprojItemDev* __restrict__ items, const float2* __restrict__ query,
                          const float2* __restrict__ train, float avg_dpt, float* __restrict__ out)
{
  __shared__ ReprojItemDev it;
  load_item<RepCfg<C>::CH>(items + blockIdx.x, it);
  sparse_error<RepCfg<C>>(it.num_matches, out, [&](int m, float (&b)[2]) {
    const int i = it.match_begin + m;
    float r[2][13 + C], e2;
    const bool valid = reprojection_match_rows<C, false>(it, query[i], train[i], avg_dpt, r[0], r[1], &e2);
    b[0] = r[0][12 + C];
    b[1] = r[1][12 + C];
    return valid;
  });
}

template <int C>
__global__ void __launch_bounds__(GeoCfg<C>::CH)
sparse_geometric_error_kernel(const GeoItemDev* __restrict__ items, const int2* __restrict__ points, float avg_dpt,
                              float* __restrict__ out)
{
  __shared__ GeoItemDev it;
  load_item<GeoCfg<C>::CH>(items + blockIdx.x, it);
  sparse_error<GeoCfg<C>>(it.num_points, out, [&](int m, float (&b)[1]) {
    float r[13 + 2 * C];
    const bool valid = sparse_geometric_point_row<C, false>(it, points[it.point_begin + m], avg_dpt, r);
    b[0] = r[12 + 2 * C];
    return valid;
  });
}

// Calls f(std::integral_constant<int, C>{}) for the code sizes the sparse kernels are instantiated for.
template <class F>
cudaError_t with_sparse_code_size(int code_size, F&& f)
{
  switch (code_size) {
    case 8: return f(std::integral_constant<int, 8>{});
    case 16: return f(std::integral_constant<int, 16>{});
    case 32: return f(std::integral_constant<int, 32>{});
    case 64: return f(std::integral_constant<int, 64>{});
    case 128: return f(std::integral_constant<int, 128>{});
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

bool sparse_supported(int code_size)
{
  return with_sparse_code_size(code_size, [](auto) { return cudaSuccess; }) == cudaSuccess;
}

cudaError_t launch_reprojection_rows(int code_size, const ReprojItemDev& item, const float2* query_dev,
                                     const float2* train_dev, float avg_dpt, float* rows_dev, float* err2_dev, cudaStream_t s)
{
  return with_sparse_code_size(code_size, [&](auto cs) {
    reprojection_rows_kernel<cs.value><<<(item.num_matches + 127) / 128, 128, 0, s>>>(item, query_dev, train_dev, avg_dpt,
                                                                                      rows_dev, err2_dev);
    return cudaGetLastError();
  });
}

cudaError_t launch_reprojection_records(int code_size, const ReprojItemDev* items_dev, int num_items, const float2* query_dev,
                                        const float2* train_dev, float avg_dpt, float* records_dev, cudaStream_t s)
{
  return with_sparse_code_size(code_size, [&](auto cs) {
    using Cfg = RepCfg<cs.value>;
    const cudaError_t e = cudaFuncSetAttribute(reprojection_records_kernel<cs.value>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
    if (e != cudaSuccess) return e;
    reprojection_records_kernel<cs.value><<<num_items, Cfg::NT, Cfg::SMEM, s>>>(items_dev, query_dev, train_dev, avg_dpt,
                                                                               records_dev);
    return cudaGetLastError();
  });
}

cudaError_t launch_sparse_geometric_rows(int code_size, const GeoItemDev& item, const int2* points_dev, float avg_dpt,
                                         float* rows_dev, cudaStream_t s)
{
  return with_sparse_code_size(code_size, [&](auto cs) {
    sparse_geometric_rows_kernel<cs.value><<<(item.num_points + 127) / 128, 128, 0, s>>>(item, points_dev, avg_dpt,
                                                                                         rows_dev);
    return cudaGetLastError();
  });
}

cudaError_t launch_sparse_geometric_records(int code_size, const GeoItemDev* items_dev, int num_items, const int2* points_dev,
                                            float avg_dpt, float* records_dev, cudaStream_t s)
{
  return with_sparse_code_size(code_size, [&](auto cs) {
    using Cfg = GeoCfg<cs.value>;
    const cudaError_t e = cudaFuncSetAttribute(sparse_geometric_records_kernel<cs.value>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
    if (e != cudaSuccess) return e;
    sparse_geometric_records_kernel<cs.value><<<dim3(num_items, Cfg::NS), Cfg::NT, Cfg::SMEM, s>>>(items_dev, points_dev,
                                                                                                   avg_dpt, records_dev);
    return cudaGetLastError();
  });
}

cudaError_t launch_reprojection_error(int code_size, const ReprojItemDev* items_dev, int num_items, const float2* query_dev,
                                      const float2* train_dev, float avg_dpt, float* out_dev, cudaStream_t s)
{
  return with_sparse_code_size(code_size, [&](auto cs) {
    reprojection_error_kernel<cs.value><<<num_items, RepCfg<cs.value>::CH, 0, s>>>(items_dev, query_dev, train_dev,
                                                                                 avg_dpt, out_dev);
    return cudaGetLastError();
  });
}

cudaError_t launch_sparse_geometric_error(int code_size, const GeoItemDev* items_dev, int num_items, const int2* points_dev,
                                          float avg_dpt, float* out_dev, cudaStream_t s)
{
  return with_sparse_code_size(code_size, [&](auto cs) {
    sparse_geometric_error_kernel<cs.value><<<num_items, GeoCfg<cs.value>::CH, 0, s>>>(items_dev, points_dev, avg_dpt,
                                                                                     out_dev);
    return cudaGetLastError();
  });
}

}  // namespace dfk
