// dfk_sfm_tc.cu -- SfmAligner::RunStep hot path, Hopper warpgroup tensor-core Gram variant (sm_90a, C = 32).
//
// Same contract as dfk_sfm_fp32.cu (replaces kernel_step_calculate + DenseSfm + the two-kernel
// reduction of sources/cuda/cu_sfmaligner.cpp:40-70,149-185, dense_sfm.h:133-201), different engine
// for the reduced Gram  G = sum_p m_p^T m_p,  m = w*[ e*jc (32) | a (6) | diff (1) ]  (39 features):
//
//   Split precision ("3xTF32" folded into one product): every feature value v is split exactly into h = v with the
//   low 13 mantissa bits cleared (exactly representable in tf32) and l = v - h.  With A = [h rows ; l rows] and B = h,
//   the tf32 MMAs yield HH = sum h h^T and LH = sum l h^T;  G = HH + LH + LH^T  drops only the l*l terms (~2^-22).
//
//   One CTA is one warpgroup (128 threads, one pixel each, kTcCtasPerSm CTAs per SM).  Per 128-pixel tile every thread
//   runs the per-pixel front-end ((optional depth decode,) exact-order validity chain, bilinear gathers, Jacobian row,
//   Huber -> s = w*e, w*a[6], w*diff); the warp then reads its 32 pixels' code-Jacobian rows straight from global
//   memory, COALESCED (lane = 16-byte chunk lane&7 of pixel 4i + lane/8), scales them by the pixel's s (one shuffle),
//   splits them into h / l and stores them K-major (pixels along K) into the CTA's operand buffer; each thread adds
//   its own pixel's 7 pose / residual values.  Invalid pixels contribute exact zeros.  After one CTA barrier the
//   warpgroup issues 16 x wgmma.m64n56k8 (K = 8 pixels each) and, without waiting, goes on with the next tile's
//   gathers; it waits for the MMAs only before it overwrites the operand buffer.
//
//   Operand buffer: 10 groups of 8 feature rows --
//     0-2 code-l 0-23 | 3-6 code-h 0-31 | 7 pose-h (features 0-6, row 7 zero) | 8 code-l 24-31 | 9 pose-l.
//   Inside a group, the core matrix of pixels 4q..4q+3 sits at q * kLbo, feature row r of it at r * 16.  kLbo and kSbo
//   carry 16 bytes of padding each, so the code-h and pose stores of a warp hit 32 different banks (the code-l stores
//   of groups 0 and 8 share banks: 2-way).
//     D = A x B^T, A = groups 0-7 (M = 64: code-l 0-23, then all 40 h rows), B = groups 3-9 (N = 56: all 40 h rows, then
//     code-l 24-31 and pose-l).  Both are contiguous, so one descriptor stride serves each.  With the 40 features
//     f = code 0-31 | pose/residual 32-39:  HH[i][j] = D[24 + i][j];  LH[i][j] = D[i][j] for i < 24 and
//     D[24 + j][16 + i] for i >= 24.  Only D[0-23][40-55] (l*l terms) is unused.
//   The accumulator lives in registers (28 floats per thread).  A chain is cut every kFlushTiles tiles and at item
//   boundaries: its fragments are staged in the (then idle) operand buffer, combined into G = (HH + LH) + LH^T and added
//   in round-to-nearest fp32 to the CTA's partial in global memory (single writer per address, program order), in the
//   fp32 kernel's format (SfmCfg<32>: G row-major, upper triangle).
//
//   Input stream: the code-Jacobian rows, img0 and dpt0 are read once, through loads that do not allocate in L1 (L1 is
//   left to the bilinear gathers of img1 / grad1, the only loads that reuse lines; the fused depth decode reads the code
//   rows a first time through L1, so that the Gram's second read hits there).  Nothing is prefetched: on H100
//   both a per-thread L2 prefetch of the pixel's code row and bulk L2 prefetches of a later tile made the kernel slower.
//
// The per-item block, the static tile->CTA assignment, the in-item tile permutation and the per-pixel row (ray table,
// validity chain, gathers, Jacobian row, Huber) come from dfk_sfm_frontend.cuh, as in the fp32 and wide kernels; this
// kernel keeps its own tile walk (every warp owns a copy of the item block) and its cross-lane depth decode.  The
// per-CTA partials and the wide deterministic finalize are those of the fp32 kernel.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "dfk_async.cuh"
#include "dfk_geom.cuh"
#include "dfk_internal.h"
#include "dfk_sfm_frontend.cuh"
#include "dfk_sfm_tc_common.cuh"
#include "dfk_wgmma.cuh"

namespace dfk {

namespace {

constexpr int C = 32;
constexpr int TILE = kTcTilePixels;  // 128
constexpr int THREADS = 128;         // one warpgroup, one pixel per thread
constexpr int NWARP = THREADS / 32;
constexpr uint32_t kLbo = 128 + 16;           // core matrices adjacent in K (4 pixels)
constexpr uint32_t kSbo = 32 * kLbo + 16;     // 8-row groups (a group spans the tile's 32 core matrices)
constexpr uint32_t OP_BYTES = 10 * kSbo;
#ifndef DFK_FLUSH_TILES
#define DFK_FLUSH_TILES 8
#endif
constexpr int kFlushTiles = DFK_FLUSH_TILES;  // accumulation chain length (tiles)
using Cfg = SfmCfg<C>;                         // the partial: G row-major NFP x NFP, then the inlier count
// D (64 x 56) staged row-major at a flush; the odd row stride keeps the column reads of LH conflict-free
constexpr int kDStride = 57;
static_assert(64 * kDStride * 4 <= 7 * kSbo, "the staged D must leave row 7 of the pose groups alone");
// LH[i][j] in the staged D
__device__ __forceinline__ int lh(int i, int j) { return i < 24 ? i * kDStride + j : (24 + j) * kDStride + 16 + i; }

struct Smem {
  alignas(128) unsigned char op[OP_BYTES];
  SfmItem<C> item[NWARP];
};

#ifdef DFK_EXP_CTA_CLOCKS
// experiment (tools/cta_tail.py): per CTA of the last launch, %globaltimer at entry and exit, (tiles << 32 | tiles with
// a valid pixel) and the SM it ran on
constexpr int kClockCtas = 8192;
__device__ unsigned long long g_cta_clocks[kClockCtas][4];
__device__ __forceinline__ unsigned long long global_ns()
{
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#endif

__global__ void __launch_bounds__(THREADS, kTcCtasPerSm)
sfm_step_tc_kernel(const SfmItemDev* __restrict__ items, int num_tiles, float* __restrict__ partials)
{
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
#ifdef DFK_EXP_CTA_CLOCKS
  const unsigned long long t_entry = global_ns();
  int valid_tiles = 0;
#endif
  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  int g_lo, g_hi;
  cta_tiles(num_tiles, g_lo, g_hi);
  const int ntiles = g_hi - g_lo;
  if (ntiles <= 0) return;

  // row 7 of the pose groups (7 and 9) is never written: zeros
  if (tid < 64)
    *reinterpret_cast<float4*>(sm.op + (tid < 32 ? 7 : 9) * kSbo + (tid & 31) * kLbo + 7 * 16) =
        make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();

  const uint32_t op = smem_u32(sm.op);
  // code-Jacobian stores: this lane holds features 4c..4c+3 of pixel 4 i8 + r of the warp's 32 pixels
  const int c = lane & 7, r = lane >> 3;
  const uint32_t in_group = (uint32_t)(8 * warp) * kLbo + (uint32_t)(c & 1) * 64u + (uint32_t)r * 4u;
  const uint32_t code_l = op + (uint32_t)((c >> 1) < 3 ? (c >> 1) : 8) * kSbo + in_group;
  const uint32_t code_h = op + (uint32_t)(3 + (c >> 1)) * kSbo + in_group;
  // pose stores: this thread's own pixel
  const uint32_t pose_h = op + 7u * kSbo + (uint32_t)(8 * warp + (lane >> 2)) * kLbo + (uint32_t)(lane & 3) * 4u;
  const uint32_t pose_l = pose_h + 2u * kSbo;

  float acc[28];
#pragma unroll
  for (int q = 0; q < 28; ++q) acc[q] = 0.0f;  // never read before a chain's first MMA overwrites them
  SfmItem<C>& I = sm.item[warp];
  int it = 0;
  int cur_item = -1;
  uint32_t item_hi = 0;  // end of the global tile range of the item in shared memory
  int tiles_in_chain = 0, chain_valid = 0, pslot = 0;
  bool fresh = true;
  unsigned int inliers = 0;

  // close the chain: combine G = (HH + LH) + LH^T of the chain's accumulators and add it to the partial (the first
  // chain of an item in this CTA stores).  D goes through the operand buffer, free once the chain's MMAs have completed;
  // the next tile's operand stores rewrite every byte the MMAs read.  The accumulators are only ever written by the MMAs
  // (a chain's first MMA overwrites them), so ptxas can keep them in flight across the next tile's front-end
  auto flush = [&](bool item_end) {
    wgmma_wait_all();
    float* P = partials + (size_t)pslot * Cfg::PARTIAL_FLOATS;
    if (fresh || chain_valid > 0) {  // uniform across the CTA, like all chain bookkeeping
      const bool have = chain_valid > 0;
      float* Ds = reinterpret_cast<float*>(sm.op);
      if (have) {
        __syncthreads();  // every warp's share of the chain's MMAs has completed
        const int m0 = 16 * warp + (lane >> 2);
#pragma unroll
        for (int q = 0; q < 28; ++q)
          Ds[(m0 + 8 * ((q >> 1) & 1)) * kDStride + 8 * (q >> 2) + 2 * (lane & 3) + (q & 1)] = acc[q];
        __syncthreads();
      }
      // entries (i, j), i <= j < NF, of the row-major NFP x NFP partial: the ones the finalize reads
      for (int e = tid; e < Cfg::NFP * Cfg::NFP; e += THREADS) {
        const int i = e / Cfg::NFP, j = e - Cfg::NFP * i;
        if (i > j || j >= Cfg::NF) continue;
        float g = 0.0f;
        if (have) g = (Ds[(24 + i) * kDStride + j] + Ds[lh(i, j)]) + Ds[lh(j, i)];
        put_partial(P + e, g, fresh);
      }
      if (have) __syncthreads();  // the staged D is read before the next tile's operand stores overwrite it
    }
    if (item_end && tid == 0) reinterpret_cast<unsigned int*>(P)[Cfg::NFP * Cfg::NFP] = inliers;
    fresh = false;
    chain_valid = 0;
    tiles_in_chain = 0;
  };

  for (int i = 0; i < ntiles; ++i) {
    const int g = g_lo + i;
    // chain bookkeeping is uniform across the CTA: every warp walks the same tiles
    if (cur_item < 0 || (uint32_t)g >= item_hi) {
      if (cur_item >= 0) flush(true);
      while ((uint32_t)g >= items[it].tile_begin + items[it].num_tiles) ++it;
      __syncwarp();
      load_item(I, items[it], lane, (int)blockIdx.x);
      load_code(I, items[it], C, lane, 32);
      __syncwarp();
      cur_item = it;
      item_hi = I.tile_begin + I.num_tiles;
      pslot = (int)I.slot;
      fresh = true;
      inliers = 0;
    } else if (tiles_in_chain == kFlushTiles) {
      flush(false);
    }
    uint32_t n;
    const uint32_t p0 = tile_origin<TILE>(I, g, n);
    const uint32_t s = 32u * (uint32_t)warp + (uint32_t)lane;  // pixel slot in the tile
    const bool inb = s < n;
    const bool blk_live = 32u * (uint32_t)warp < n;  // else: a block past the end of the item's last tile
    const uint32_t W = I.width;
    const bool a16 = (I.flags & ITEM_FLAG_BULK) != 0;
    const bool fused = (I.flags & ITEM_FLAG_FUSED_DEPTH) != 0;
    // block origin (uniform) by one division, then this thread's pixel by wrap-around; lanes past the end of the
    // tile shadow the block's first pixel (their loads stay in bounds, their contribution is zero)
    uint32_t x0;
    const uint32_t y0 = div_magic(blk_live ? p0 + 32u * (uint32_t)warp : p0, W, I.mag_width, x0);
    uint32_t pxx = x0 + (inb ? (uint32_t)lane : 0u), py = y0;
    while (pxx >= W) {
      pxx -= W;
      ++py;
    }
    const float* __restrict__ jac = I.jac;
    const uint32_t joff = py * I.jac_pitch + pxx * C;  // this pixel's code-Jacobian row (floats)
    float feat[8];
    bool ok = false;
    if (blk_live) {
      const float2 ray = table_ray(I, pxx, py);  // issued before the decode: its latency hides behind it
      float d = ld_stream(I.dpt0 + (size_t)py * I.dpt0_pitch + pxx);
      const float i0 = ld_stream(I.img0 + (size_t)py * I.img0_pitch + pxx);
      if (fused) {
        // dpt0 is prx_orig: decode the depth from the pixel's code-Jacobian row -- same arithmetic as
        // update_depth_kernel (chunk fma chains, then the xor-butterfly over the 8 chunk sums, here ACROSS the 8
        // lanes that hold the chunks of one pixel), publish it, and carry on with it
        const float4 cc = *reinterpret_cast<const float4*>(&I.code[4 * (lane & 7)]);
        float mine = 0.0f;
#pragma unroll
        for (int i8 = 0; i8 < 8; ++i8) {
          const uint32_t offk = __shfl_sync(0xffffffffu, joff, 4 * i8 + (lane >> 3));
          float p = chunk_dot(load_chunk_l1(jac + offk + 4 * (lane & 7), a16), cc);
          p = __fadd_rn(p, __shfl_xor_sync(0xffffffffu, p, 4));
          p = __fadd_rn(p, __shfl_xor_sync(0xffffffffu, p, 2));
          p = __fadd_rn(p, __shfl_xor_sync(0xffffffffu, p, 1));
          const float got = __shfl_sync(0xffffffffu, p, 8 * (lane & 3));  // pixel 4 i8 + (lane & 3)
          if ((lane >> 2) == i8) mine = got;
        }
        d = prx_to_depth(__fadd_rn(d, mine), I.avg_dpt);
        if (inb) I.dpt_out[(size_t)py * I.dpt_out_pitch + pxx] = d;
      }
      if (inb) ok = pixel_row(I, pxx, py, ray, d, i0, true, feat);  // the API guarantees 8-byte grad1 rows here
    }
    if (!ok) {
#pragma unroll
      for (int f = 0; f < 8; ++f) feat[f] = 0.0f;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    float4 v[8];
#pragma unroll
    for (int i8 = 0; i8 < 8; ++i8) {
      const uint32_t offk = __shfl_sync(0xffffffffu, joff, 4 * i8 + r);
      v[i8] = make_float4(0.f, 0.f, 0.f, 0.f);
      if ((bal >> (4 * i8 + r)) & 1u) v[i8] = load_chunk(jac + offk + 4 * c, a16);
    }
    // ---- the operand buffer is free once the previous tile's MMAs have completed ---------------------------------------
    wgmma_wait_all();
#pragma unroll
    for (int i8 = 0; i8 < 8; ++i8) {
      const float sk = __shfl_sync(0xffffffffu, feat[0], 4 * i8 + r);
      const float x[4] = {sk * v[i8].x, sk * v[i8].y, sk * v[i8].z, sk * v[i8].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float h = tf32_trunc(x[e]);
        const uint32_t off = (uint32_t)i8 * kLbo + (uint32_t)e * 16u;
        sts32(code_h + off, h);
        sts32(code_l + off, x[e] - h);
      }
    }
#pragma unroll
    for (int f = 0; f < 7; ++f) {
      const float h = tf32_trunc(feat[1 + f]);
      sts32(pose_h + (uint32_t)f * 16u, h);
      sts32(pose_l + (uint32_t)f * 16u, feat[1 + f] - h);
    }
    fence_proxy_async_smem();  // generic-proxy writes -> visible to the MMA's operand fetch
    const int nv = __syncthreads_count(ok);
    if (nv > 0) {
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < TILE / 8; ++kk) {
        const uint32_t k_off = (uint32_t)kk * 2u * kLbo;
        const bool accumulate = kk > 0 || chain_valid > 0;
#ifndef DFK_EXP_NOMMA  // experiment (wrong results): no MMA at all
        wgmma_m64n56k8_tf32(acc, make_wgmma_desc_kmajor(op + k_off, kLbo, kSbo),
                            make_wgmma_desc_kmajor(op + 3u * kSbo + k_off, kLbo, kSbo), accumulate);
#endif
      }
      wgmma_commit();
    }
    chain_valid += nv;
    inliers += (unsigned)nv;
    ++tiles_in_chain;
#ifdef DFK_EXP_CTA_CLOCKS
    valid_tiles += nv > 0;
#endif
  }
  flush(true);
#ifdef DFK_EXP_CTA_CLOCKS
  __syncthreads();
  if (tid == 0 && blockIdx.x < kClockCtas) {
    unsigned int smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    unsigned long long* o = g_cta_clocks[blockIdx.x];
    o[0] = t_entry;
    o[1] = global_ns();
    o[2] = ((unsigned long long)ntiles << 32) | (unsigned)valid_tiles;
    o[3] = smid;
  }
#endif
}

}  // namespace

bool sfm_tc_supported(int code_size) { return code_size == 32; }

cudaError_t launch_sfm_tc(const SfmItemDev* items_dev, const SfmLaunchPlan& plan, float* partials_dev,
                          cudaStream_t stream, cudaEvent_t ev_start, cudaEvent_t ev_stop)
{
  const size_t smem = sizeof(Smem);
  static const cudaError_t attr_err =  // once per process, not once per launch
      cudaFuncSetAttribute(sfm_step_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem));
  cudaError_t err = attr_err;
  if (err != cudaSuccess) return err;
  if (ev_start) cudaEventRecord(ev_start, stream);
  sfm_step_tc_kernel<<<plan.num_ctas, THREADS, smem, stream>>>(items_dev, plan.num_tiles, partials_dev);
  if (ev_stop) cudaEventRecord(ev_stop, stream);
  return cudaGetLastError();
}

}  // namespace dfk

#ifdef DFK_EXP_CTA_CLOCKS
// the per-CTA records of the last step kernel launch (n <= 8192 CTAs, 4 u64 each); synchronises the device
extern "C" int dfk_exp_cta_clocks(unsigned long long* out, int n)
{
  if (n < 0 || n > dfk::kClockCtas) return -1;
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  return cudaMemcpyFromSymbol(out, dfk::g_cta_clocks, sizeof(unsigned long long) * 4 * (size_t)n) == cudaSuccess ? 0 : -1;
}
#endif
