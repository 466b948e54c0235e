// dfk_sfm_wide.cu -- SfmAligner::RunStep hot path for the wide code sizes (C = 64, 128), fp32 CUDA-core Gram.
//
// Same contract as dfk_sfm_fp32.cu (kernel_step_calculate + DenseSfm + the two-stage reduction of the
// reference: sources/cuda/cu_sfmaligner.cpp:40-70, sources/common/algorithm/dense_sfm.h:133-201,
// sources/cuda/kernel_utils.h:51-69) for the code sizes the reference declares but cannot launch (its
// per-thread 1 x (12+C) item does not fit at C >= 64: cu_sfmaligner.cpp:170-173, instantiations commented
// out at :210-211).
//
// What differs from the C <= 32 kernel: the reduced system G = sum m^T m has (7+C)^2 entries -- 45 / 153
// upper 8x8 blocks at C = 64 / 128 -- so a block is owned by a THREAD (64 register accumulators), not by a
// warp.  KS threads share one block and split the tile's compacted pixels round-robin; their partial sums
// meet in a fixed shuffle order when the CTA leaves an item, so results are bitwise reproducible.
//   * front-end: the CUDA-core pipeline of dfk_sfm_frontend.cuh (persistent CTAs, static tile ranges, TMA
//     staging of jac / img0 / dpt0 rows, one thread per pixel), with a tile of 128 (C = 64) or 64 (C = 128)
//     pixels so two stages fit.  This file writes the reduced row m = w * [ e*jc (C) | a (6) | diff ]
//     pixel-major and compacted into M[pixel][NFP].
//   * Gram threads: for every valid pixel of their split, 2+2 LDS.128 and 64 FMA.
// CUDA-core bound (9.8 kFMA per pixel at C = 128).  DFK_GRAM_AUTO runs these sizes on the tensor-core kernel
// (dfk_sfm_tc.cu); this one is the DFK_GRAM_FP32 engine and AUTO's engine for grad1 rows the tensor-core
// kernel cannot gather (not 8-byte aligned).
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_async.cuh"
#include "dfk_internal.h"
#include "dfk_sfm_frontend.cuh"

namespace dfk {

namespace {

constexpr int kStages = 2;

template <int C>
struct WideCfg {
  using Cfg = SfmCfg<C>;
  static constexpr int TILE = sfm_wide_tile_pixels(C);
  static constexpr int KS = (C >= 128) ? 2 : 8;  // threads per 8x8 block (power of two, <= 32)
  static constexpr int FE_THREADS = TILE;
  static constexpr int GRAM_THREADS = ((Cfg::NBLK * KS + 31) / 32) * 32;
  static constexpr int GRAM_WARPS = GRAM_THREADS / 32;
  static constexpr int THREADS = FE_THREADS + GRAM_THREADS;
};

template <int C>
using Smem = CoreSmem<C, WideCfg<C>::TILE, kStages>;

template <int C>
__global__ void __launch_bounds__(WideCfg<C>::THREADS, 1)
sfm_step_wide_kernel(const SfmItemDev* __restrict__ items, int num_items, int num_tiles, float* __restrict__ partials)
{
  using Cfg = SfmCfg<C>;
  using W = WideCfg<C>;
  constexpr int NFP = Cfg::NFP;
  constexpr int NB = Cfg::NB;
  constexpr int NBLK = Cfg::NBLK;
  constexpr int KS = W::KS;
  constexpr int FE = W::FE_THREADS;
  constexpr int NV = C / 4;  // float4 chunks per code-Jacobian row
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem<C>& sm = *reinterpret_cast<Smem<C>*>(smem_raw);

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  int g_lo, g_hi;
  cta_tiles(num_tiles, g_lo, g_hi);

  if (tid == 0) sm.init_barriers(W::GRAM_WARPS);
  __syncthreads();
  if (g_lo >= g_hi) return;

  if (tid < FE) {
    // ========================================================================= front-end
    frontend_role(sm, items, num_items, g_lo, g_hi,
                  [&](float* Mb, const float* jc_row, const float (&feat)[8], bool ok, int idx, int) {
                    if (!ok) return;
                    const float sc = feat[0];
                    // rotated float4 order: lane l touches chunk (k4 + l) % NV => reads (row stride 4C bytes) and
                    // writes (row stride 4*NFP bytes, NFP % 32 == 8) are both free of bank conflicts
                    const float4* src = reinterpret_cast<const float4*>(jc_row);
                    float4* dst = reinterpret_cast<float4*>(&Mb[idx * NFP]);
#pragma unroll 8
                    for (int k4 = 0; k4 < NV; ++k4) {
                      const int kk4 = (k4 + lane) % NV;
                      const float4 v = src[kk4];
                      dst[kk4] = make_float4(sc * v.x, sc * v.y, sc * v.z, sc * v.w);
                    }
                    dst[NV] = make_float4(feat[1], feat[2], feat[3], feat[4]);
                    dst[NV + 1] = make_float4(feat[5], feat[6], feat[7], 0.0f);
                  });
    return;
  }

  // =========================================================================== Gram threads
  const int gt = tid - FE;
  const int braw = gt / KS;
  const int ks = gt % KS;
  const bool active = braw < NBLK;
  const int b = active ? braw : 0;
  int bi = 0, rem = b;
  while (rem >= NB - bi) {
    rem -= NB - bi;
    ++bi;
  }
  const int bj = bi + rem;
  float acc[64];
#pragma unroll
  for (int e = 0; e < 64; ++e) acc[e] = 0.0f;

  gram_role(
      sm, g_lo, g_hi,
      [&](const float* Mb, int nvalid) {
        const float4* Mr = reinterpret_cast<const float4*>(&Mb[8 * bi]);
        const float4* Mc = reinterpret_cast<const float4*>(&Mb[8 * bj]);
#pragma unroll 1
        for (int p = ks; p < nvalid; p += KS) {
          const float4 r0 = Mr[p * (NFP / 4)], r1 = Mr[p * (NFP / 4) + 1];
          const float4 c0 = Mc[p * (NFP / 4)], c1 = Mc[p * (NFP / 4) + 1];
          const float r[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
          const float c[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
#pragma unroll
          for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[8 * j + k] = fmaf(r[j], c[k], acc[8 * j + k]);
        }
      },
      [&](int slot, unsigned int inliers) {
        // the KS threads of a block sit in adjacent lanes: butterfly in fixed order, split 0 stores
#pragma unroll
        for (int e = 0; e < 64; ++e) {
          float v = acc[e];
#pragma unroll
          for (int m = 1; m < KS; m <<= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
          acc[e] = v;
        }
        float* P = partials + (size_t)slot * Cfg::PARTIAL_FLOATS;
        if (active && ks == 0) {
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            float4* row = reinterpret_cast<float4*>(&P[(8 * bi + r) * NFP + 8 * bj]);
            row[0] = make_float4(acc[8 * r + 0], acc[8 * r + 1], acc[8 * r + 2], acc[8 * r + 3]);
            row[1] = make_float4(acc[8 * r + 4], acc[8 * r + 5], acc[8 * r + 6], acc[8 * r + 7]);
          }
          if (braw == 0) reinterpret_cast<unsigned int*>(P)[NFP * NFP] = inliers;
        }
#pragma unroll
        for (int e = 0; e < 64; ++e) acc[e] = 0.0f;
      });
}

template <int C>
cudaError_t launch_impl(const SfmItemDev* items_dev, const SfmLaunchPlan& plan, float* partials_dev,
                        cudaStream_t stream, cudaEvent_t ev_start, cudaEvent_t ev_stop)
{
  const size_t smem = sizeof(Smem<C>);
  cudaError_t err = cudaFuncSetAttribute(sfm_step_wide_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
  if (err != cudaSuccess) return err;
  if (ev_start) cudaEventRecord(ev_start, stream);
  sfm_step_wide_kernel<C><<<plan.num_ctas, WideCfg<C>::THREADS, smem, stream>>>(items_dev, plan.num_items,
                                                                               plan.num_tiles, partials_dev);
  if (ev_stop) cudaEventRecord(ev_stop, stream);
  return cudaGetLastError();
}

}  // namespace

bool sfm_wide_supported(int code_size) { return code_size == 64 || code_size == 128; }

cudaError_t launch_sfm_wide(int code_size, const SfmItemDev* items_dev, const SfmLaunchPlan& plan,
                            float* partials_dev, cudaStream_t stream, cudaEvent_t ev_start, cudaEvent_t ev_stop)
{
  switch (code_size) {
    case 64: return launch_impl<64>(items_dev, plan, partials_dev, stream, ev_start, ev_stop);
    case 128: return launch_impl<128>(items_dev, plan, partials_dev, stream, ev_start, ev_stop);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace dfk
