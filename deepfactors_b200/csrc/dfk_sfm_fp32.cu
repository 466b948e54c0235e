// dfk_sfm_fp32.cu -- SfmAligner::RunStep hot path, fp32 CUDA-core Gram variant (sm_90a).
//
// Replaces kernel_step_calculate + DenseSfm + runReductions/finalizeReduction +
// kernel_finalize_reduction of the reference (sources/cuda/cu_sfmaligner.cpp:40-70,
// sources/common/algorithm/dense_sfm.h:133-201, sources/cuda/kernel_utils.h:51-69).
//
// Design (see DESIGN.md "fp32 Gram kernel"):
//   * ONE persistent launch evaluates a whole list of (pair, level) items.  The pixel stream
//     of every item is cut into tiles of 256 linear pixels; CTA c owns a contiguous range of
//     the global tile sequence (static => bitwise reproducible results), tiles inside an item
//     are visited in a strided order so that spatially clustered invalid regions balance out.
//   * The front-end is the CUDA-core pipeline of dfk_sfm_frontend.cuh: per tile the TMA engine
//     (cp.async.bulk, 1-D row segments) stages the code-Jacobian rows (C contiguous floats per
//     pixel), img0 and dpt0 into a 3-deep shared-memory ring; 8 front-end warps (one thread per
//     pixel) run the per-pixel row (exact-order validity chain, gathers of img1/grad1, reduced row
//     m = w*[ e*jc (C) | a (6) | diff (1) ]).  This file writes the row, compacted to valid pixels
//     and zero-padded to a multiple of 32, K-major into a double-buffered tile M[feature][pixel].
//   * NBLK "Gram" warps each own one 8x8 block of the upper triangle of G = sum m^T m
//     ((7+C)^2, the (6+C) reduced system + gradient + energy of SURVEY Appendix A) with lanes
//     striding over pixels; 64 register accumulators per thread, operands via conflict-free
//     LDS.  Accumulators are reduce-scattered across lanes only when the CTA leaves an item.
//   * A second, wide kernel sums the per-CTA partials in fixed order and expands the reduced
//     system to the reference's (12+C) layout with the host-computed relative-pose Jacobians:
//     JtJ = E^T G E,  E = [[P0,P1,0],[0,0,I]].
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_async.cuh"
#include "dfk_geom.cuh"
#include "dfk_internal.h"
#include "dfk_sfm_frontend.cuh"

namespace dfk {

namespace {

constexpr int kStages = 3;
constexpr int kFeWarps = kTilePixels / 32;  // one front-end thread per tile pixel

template <int C>
using Smem = CoreSmem<C, kTilePixels, kStages>;

// reduce-scatter of 64 per-lane accumulators: afterwards lane l holds the warp-wide sums of
// entries 2l and 2l+1 in acc[0], acc[1].  62 shuffles; fixed order => deterministic.
__device__ __forceinline__ void reduce_scatter64(float (&acc)[64], int lane)
{
#pragma unroll
  for (int m = 16, n = 64; m >= 1; m >>= 1, n >>= 1) {
    const bool up = (lane & m) != 0;
#pragma unroll
    for (int i = 0; i < n / 2; ++i) {
      const float send = up ? acc[i] : acc[i + n / 2];
      const float keep = up ? acc[i + n / 2] : acc[i];
      acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, m);
    }
  }
}

template <int C>
__global__ void __launch_bounds__((kFeWarps + SfmCfg<C>::NBLK) * 32, sfm_fp32_ctas_per_sm(C))
sfm_step_fp32_kernel(const SfmItemDev* __restrict__ items, int num_items, int num_tiles, float* __restrict__ partials)
{
  using Cfg = SfmCfg<C>;
  constexpr int NFP = Cfg::NFP;
  constexpr int NB = Cfg::NB;
  constexpr int NBLK = Cfg::NBLK;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem<C>& sm = *reinterpret_cast<Smem<C>*>(smem_raw);

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  int g_lo, g_hi;
  cta_tiles(num_tiles, g_lo, g_hi);

  if (tid == 0) sm.init_barriers(NBLK);
  __syncthreads();
  if (g_lo >= g_hi) return;

  if (warp < kFeWarps) {
    // ========================================================================= front-end
    // M is feature-major; rows nvalid .. nvalid rounded up to 32 are zero, so the Gram warps read whole warps of pixels
    frontend_role(sm, items, num_items, g_lo, g_hi,
                  [&](float* Mb, const float* jc_row, const float (&feat)[8], bool ok, int idx, int nvalid) {
                    if (ok) {
                      const float sc = feat[0];
                      constexpr int NV = C / 4;
                      const int rot = (NV >= 8) ? lane : (lane / (8 / (NV < 8 ? NV : 8)));
                      const float4* src = reinterpret_cast<const float4*>(jc_row);
#pragma unroll
                      for (int k4 = 0; k4 < NV; ++k4) {
                        const int kk4 = (k4 + rot) % NV;
                        const float4 v = src[kk4];
                        Mb[(kk4 * 4 + 0) * kTilePixels + idx] = sc * v.x;
                        Mb[(kk4 * 4 + 1) * kTilePixels + idx] = sc * v.y;
                        Mb[(kk4 * 4 + 2) * kTilePixels + idx] = sc * v.z;
                        Mb[(kk4 * 4 + 3) * kTilePixels + idx] = sc * v.w;
                      }
#pragma unroll
                      for (int j = 0; j < 7; ++j) Mb[(C + j) * kTilePixels + idx] = feat[1 + j];
#pragma unroll
                      for (int j = C + 7; j < NFP; ++j) Mb[j * kTilePixels + idx] = 0.0f;
                    } else if (idx < ((nvalid + 31) & ~31)) {
#pragma unroll
                      for (int j = 0; j < NFP; ++j) Mb[j * kTilePixels + idx] = 0.0f;
                    }
                  });
    return;
  }

  // =========================================================================== Gram warps
  const int b = warp - kFeWarps;
  // block index -> (bi, bj), bi <= bj, row-major over the upper triangle
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
        // 32-bit shared-window addresses + explicit ld.shared keep the loop at 64 accumulators + 12 operands
        const uint32_t mr = smem_u32(Mb) + 4u * ((8 * bi) * kTilePixels + lane);
        const uint32_t mc = smem_u32(Mb) + 4u * ((8 * bj) * kTilePixels + lane);
        const int steps = (nvalid + 31) >> 5;
        for (int s = 0; s < steps; ++s) {
          float r[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) r[j] = lds_f32(mr + 4u * (j * kTilePixels + s * 32));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float c[4];
#pragma unroll
            for (int k = 0; k < 4; ++k)
              c[k] = (bi == bj) ? r[4 * h + k] : lds_f32(mc + 4u * ((4 * h + k) * kTilePixels + s * 32));
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
              for (int k = 0; k < 4; ++k) acc[j * 8 + 4 * h + k] = fmaf(r[j], c[k], acc[j * 8 + 4 * h + k]);
          }
        }
      },
      [&](int slot, unsigned int inliers) {
        reduce_scatter64(acc, lane);
        float* P = partials + (size_t)slot * Cfg::PARTIAL_FLOATS;
        const int e0 = 2 * lane;  // entries e0, e0+1 of the 8x8 block: row e0/8, cols e0%8, e0%8+1
        float2 v = make_float2(acc[0], acc[1]);
        *reinterpret_cast<float2*>(&P[(8 * bi + (e0 >> 3)) * NFP + 8 * bj + (e0 & 7)]) = v;
        if (b == 0 && lane == 0) reinterpret_cast<unsigned int*>(P)[NFP * NFP] = inliers;
#pragma unroll
        for (int e = 0; e < 64; ++e) acc[e] = 0.0f;
      });
}

template <int C>
cudaError_t launch_impl(const SfmItemDev* items_dev, const SfmLaunchPlan& plan, float* partials_dev,
                        cudaStream_t stream, cudaEvent_t ev_start, cudaEvent_t ev_stop)
{
  using Cfg = SfmCfg<C>;
  const size_t smem = sizeof(Smem<C>);
  cudaError_t err = cudaFuncSetAttribute(sfm_step_fp32_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
  if (err != cudaSuccess) return err;
  const int threads = (kFeWarps + Cfg::NBLK) * 32;
  if (ev_start) cudaEventRecord(ev_start, stream);
  sfm_step_fp32_kernel<C><<<plan.num_ctas, threads, smem, stream>>>(items_dev, plan.num_items, plan.num_tiles,
                                                                    partials_dev);
  if (ev_stop) cudaEventRecord(ev_stop, stream);
  return cudaGetLastError();
}

}  // namespace

bool sfm_fp32_supported(int code_size) { return code_size == 8 || code_size == 16 || code_size == 32; }

size_t sfm_partial_floats(int code_size)
{
  switch (code_size) {
    case 8: return SfmCfg<8>::PARTIAL_FLOATS;
    case 16: return SfmCfg<16>::PARTIAL_FLOATS;
    case 32: return SfmCfg<32>::PARTIAL_FLOATS;
    case 64: return SfmCfg<64>::PARTIAL_FLOATS;
    case 128: return SfmCfg<128>::PARTIAL_FLOATS;
    default: return 0;
  }
}

int sfm_max_ctas()
{
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms > 0 ? sms : 1;
}

cudaError_t launch_sfm_fp32(int code_size, const SfmItemDev* items_dev, const SfmLaunchPlan& plan,
                            float* partials_dev, cudaStream_t stream, cudaEvent_t ev_start, cudaEvent_t ev_stop)
{
  switch (code_size) {
    case 8: return launch_impl<8>(items_dev, plan, partials_dev, stream, ev_start, ev_stop);
    case 16: return launch_impl<16>(items_dev, plan, partials_dev, stream, ev_start, ev_stop);
    case 32: return launch_impl<32>(items_dev, plan, partials_dev, stream, ev_start, ev_stop);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace dfk
