// dfk_window.cu -- device-side assembly of a keyframe window's block-sparse normal equations from the per-(pair, level)
// result records of SfmAligner::RunStep, i.e. what the factor graph does with them
// (sources/core/gtsam/photometric_factor.cpp:105-161: JtJ blocks G11 G12 G13 G22 G23 G33, g = -Jtr;  :275-282 residual
// rescale res / inliers * W * H) summed over the factors of a window (one factor per pair and level,
// sources/core/mapping/df_work.cpp:211-225), in the variable order [pose_k (6) | code_k (C)] per keyframe.
//
// Block-sparse layout (fp32, the buffer ONE all-reduce sums across GPUs; SURVEY 8e), B = 6 + C:
//   [ K diagonal blocks, B x B row-major, full symmetric ]   keyframe k's pose/code Hessian
//   [ K gradient blocks, B ]                                 g = -sum Jtr
//   [ P coupling blocks, B x 6 row-major ]                   pair p = (k0 -> k1): rows = k0's [pose0 | code0], cols = k1's pose1
//   [ f, inliers ]                                           sum of rescaled residuals (items with overlap), of the
//                                                            residuals of unscaled records (area 0) and of the links,
//                                                            photometric inliers
//   [ L link blocks, B x B row-major ]                       geometric link l = (k0 -> k1): rows = k0's [pose0 | code0],
//                                                            cols = k1's [pose1 | code1]
// A pair (k0 -> k1) adds its pose0/code0 blocks to keyframe k0's diagonal block, pose1 x pose1 to k1's, and the
// [pose0; code0] x pose1 coupling to its own block.  A geometric link (sparse_geometric_factor.cpp: keys pose0, pose1,
// code0, code1) adds its (pose0, code0) block to k0's diagonal block, its whole (pose1, code1) block to k1's, and the
// cross block to its own link block.
//
// Deterministic by construction: a GATHER, not a scatter -- every output element is owned by one thread, which sums the
// contributions of its items in list order, then those of the links (no float atomics).  One launch: grid = K + P + L + 1
// jobs.  Without links every element is the same chain of adds as in a photometric / reprojection-only window.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_internal.h"

namespace dfk {

namespace {

__device__ __forceinline__ int packed_index(int i, int j, int NP) { return i * NP - (i * (i - 1)) / 2 + (j - i); }
// entry (a, b) of the symmetric (12+C)^2 Hessian of a record
__device__ __forceinline__ float rec_h(const float* rec, int a, int b, int NP)
{
  return a <= b ? rec[packed_index(a, b, NP)] : rec[packed_index(b, a, NP)];
}

// window row r of a link's keyframe k0 / k1 -> record row: pose0 0..5, pose1 6..11, code0 12..12+C-1, code1 12+C..
__device__ __forceinline__ int link_row0(int r) { return r < 6 ? r : 6 + r; }
__device__ __forceinline__ int link_row1(int r, int C) { return r < 6 ? 6 + r : 6 + C + r; }

__global__ void __launch_bounds__(256)
window_assemble_kernel(WindowDev w, const float* __restrict__ records, const float* __restrict__ geo,
                       float* __restrict__ out)
{
  const int C = w.code_size, B = 6 + C, NP = 12 + C;
  const int NH = NP * (NP + 1) / 2, REC = NH + NP + 2;
  const int NG = 12 + 2 * C, NHG = NG * (NG + 1) / 2, RECG = NHG + NG + 2;
  float* tail = out + (size_t)w.num_keyframes * (B * B + B) + (size_t)w.num_pairs * B * 6;
  const int job = blockIdx.x;
  if (job < w.num_keyframes) {
    // ---- diagonal block + gradient of keyframe k: items where k is the keyframe (k0) contribute the whole block, items
    // where k is the frame (k1) contribute pose1 x pose1 / g(pose1)
    const int k = job;
    float* D = out + (size_t)k * B * B;
    float* g = out + (size_t)w.num_keyframes * B * B + (size_t)k * B;
    const int a0 = w.kf0_ptr[k], a1 = w.kf0_ptr[k + 1];
    const int b0 = w.kf1_ptr[k], b1 = w.kf1_ptr[k + 1];
    const int l00 = w.lk0_ptr[k], l01 = w.lk0_ptr[k + 1];
    const int l10 = w.lk1_ptr[k], l11 = w.lk1_ptr[k + 1];
    for (int e = threadIdx.x; e < B * B + B; e += blockDim.x) {
      float s = 0.0f;
      if (e < B * B) {
        const int r = e / B, c = e - r * B;
        // window row r of keyframe k0 -> record row: pose0 0..5, code0 12..12+C-1
        const int lr = r < 6 ? r : 6 + r, lc = c < 6 ? c : 6 + c;
        for (int q = a0; q < a1; ++q) s += rec_h(records + (size_t)w.kf0_items[q] * REC, lr, lc, NP);
        if (r < 6 && c < 6)
          for (int q = b0; q < b1; ++q) s += rec_h(records + (size_t)w.kf1_items[q] * REC, 6 + r, 6 + c, NP);
        for (int q = l00; q < l01; ++q) s += rec_h(geo + (size_t)w.lk0_links[q] * RECG, link_row0(r), link_row0(c), NG);
        for (int q = l10; q < l11; ++q)
          s += rec_h(geo + (size_t)w.lk1_links[q] * RECG, link_row1(r, C), link_row1(c, C), NG);
        D[e] = s;
      } else {
        const int r = e - B * B;
        const int lr = r < 6 ? r : 6 + r;
        for (int q = a0; q < a1; ++q) s -= records[(size_t)w.kf0_items[q] * REC + NH + lr];
        if (r < 6)
          for (int q = b0; q < b1; ++q) s -= records[(size_t)w.kf1_items[q] * REC + NH + 6 + r];
        for (int q = l00; q < l01; ++q) s -= geo[(size_t)w.lk0_links[q] * RECG + NHG + link_row0(r)];
        for (int q = l10; q < l11; ++q) s -= geo[(size_t)w.lk1_links[q] * RECG + NHG + link_row1(r, C)];
        g[r] = s;
      }
    }
  } else if (job < w.num_keyframes + w.num_pairs) {
    // ---- coupling block of pair p: [pose0; code0] x pose1, summed over the pair's items (its pyramid levels)
    const int p = job - w.num_keyframes;
    float* O = out + (size_t)w.num_keyframes * (B * B + B) + (size_t)p * B * 6;
    const int i0 = w.pair_ptr[p], i1 = w.pair_ptr[p + 1];
    for (int e = threadIdx.x; e < B * 6; e += blockDim.x) {
      const int r = e / 6, c = e - r * 6;
      const int lr = r < 6 ? r : 6 + r;
      float s = 0.0f;
      for (int q = i0; q < i1; ++q) s += rec_h(records + (size_t)w.pair_items[q] * REC, lr, 6 + c, NP);
      O[e] = s;
    }
  } else if (job < w.num_keyframes + w.num_pairs + w.num_links) {
    // ---- link block of geometric link l: k0's [pose0; code0] x k1's [pose1 | code1], from its one record
    const int l = job - w.num_keyframes - w.num_pairs;
    float* O = tail + 2 + (size_t)l * B * B;
    const float* rec = geo + (size_t)l * RECG;
    for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
      const int r = e / B, c = e - r * B;
      O[e] = rec_h(rec, link_row0(r), link_row1(c, C), NG);
    }
  } else {
    // ---- energy: f = sum res / inliers * W * H over items with overlap (photometric_factor.cpp:275-282) + res of the
    // unscaled records (reprojection factors, error() = 1/2 |b|^2, reprojection_factor.cpp:148), photometric inliers
    __shared__ float red_f[8], red_i[8];
    float f = 0.0f, ni = 0.0f;
    for (int i = threadIdx.x; i < w.num_items; i += blockDim.x) {
      const float* rec = records + (size_t)i * REC;
      const uint32_t inl = __float_as_uint(rec[NH + NP + 1]);
      if (w.item_area[i] == 0.0f) {  // unscaled record (reprojection factor): b^T b as it is, no photometric inliers
        f += rec[NH + NP];
      } else {
        if (inl > 0) f += rec[NH + NP] / (float)inl * w.item_area[i];
        ni += (float)inl;
      }
    }
    // geometric links: b^T b as it is (error() = 1/2 |b|^2 of the JacobianFactor), after the items
    for (int l = threadIdx.x; l < w.num_links; l += blockDim.x) f += geo[(size_t)l * RECG + NHG + NG];
    // fixed-order block reduction: lanes by xor butterfly, warps in index order
    for (int o = 16; o > 0; o >>= 1) {
      f += __shfl_xor_sync(0xffffffffu, f, o);
      ni += __shfl_xor_sync(0xffffffffu, ni, o);
    }
    if ((threadIdx.x & 31) == 0) {
      red_f[threadIdx.x >> 5] = f;
      red_i[threadIdx.x >> 5] = ni;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float sf = 0.0f, si = 0.0f;
      for (int k = 0; k < (int)(blockDim.x >> 5); ++k) {
        sf += red_f[k];
        si += red_i[k];
      }
      tail[0] = sf;
      tail[1] = si;
    }
  }
}

}  // namespace

cudaError_t launch_window_assemble(const WindowDev& w, const float* records_dev, const float* geo_records_dev,
                                   float* out_dev, cudaStream_t stream)
{
  window_assemble_kernel<<<w.num_keyframes + w.num_pairs + w.num_links + 1, 256, 0, stream>>>(w, records_dev,
                                                                                             geo_records_dev, out_dev);
  return cudaGetLastError();
}

}  // namespace dfk
