// dfk_sfm_tc_wide.cu -- SfmAligner::RunStep hot path, Hopper warpgroup tensor-core Gram for the wide code sizes
// (sm_90a, C = 64, 128).
//
// Same contract and the same split-precision product as dfk_sfm_tc.cu (C = 32), for the reduced Gram
// G = sum_p m_p^T m_p,  m = w*[ e*jc (C) | a (6) | diff (1) | 0 ]  (F = C + 8 features): every value v splits exactly into
// h = v with the low 13 mantissa bits cleared and l = v - h, and G = HH + LH + LH^T drops only the l*l terms.
//
//   Packing (dfk_internal.h, TcCfg): A = [ code-l 0..S-1 ; h 0..F-1 ], B = [ h 0..F-1 ; code-l S..C-1 ; pose-l ],
//   S = C - 8, so D = A x B^T (2C x (C + 24)) holds every h*h and l*h product G needs.  The operand buffer holds the
//   F/4 groups of 8 feature rows once, in the order  code-l 0..S-1 | h 0..F-1 | code-l S..C-1 | pose-l:  A is its
//   first 2C rows, B its last C + 24 rows, one descriptor stride each.  Inside a group the core matrix of pixels
//   4q..4q+3 sits at q * kLbo, feature row r of it at r * 16; kLbo / kSbo carry 16 bytes of padding each, so the
//   code-row stores of a warp (8 lanes along 32 features x 4 pixels) hit 32 different banks.
//
//   CTA: NWG warpgroups over one operand buffer of 128 pixels (K = 128 per tile), each warpgroup owning two 64-row
//   M-tiles of D in registers (C = 64: one warpgroup, 88 floats per thread, two CTAs per SM; C = 128: two warpgroups,
//   152 floats per thread, one CTA per SM).  Warp w runs the per-pixel front-end for the PW = 32 / NWG pixels
//   PW w .. PW w + PW - 1 (lane < PW: its own pixel), then the warp reads those pixels' code-Jacobian rows straight
//   from global memory, coalesced (lane = 16-byte chunk lane & 7 of a 32-feature block of pixel 4i + lane / 8),
//   scales them by the pixel's s (one shuffle), splits them into h / l and stores them K-major.  Invalid pixels
//   contribute exact zeros, and a tile with no valid pixel issues no MMA.  After one CTA barrier every warpgroup issues
//   16 k-steps x 2 M-tiles of wgmma.m64nNk8 and, without waiting, goes on with the next tile's gathers; it waits for
//   its MMAs only before the operand buffer is overwritten (with two warpgroups, a CTA barrier after the wait keeps
//   one warpgroup from overwriting what the other still reads).
//   A chain is cut every kFlushTiles tiles and at item boundaries: its fragments are added in round-to-nearest fp32 to
//   the CTA's partial (single writer per address, program order).  Only what the finalize reads is written: neither
//   the l*l block nor the lower triangle of HH.
//
//   Input stream: as in dfk_sfm_tc.cu, the code rows, img0 and dpt0 are read once through loads that do not allocate
//   in L1; the fused depth decode reads the code rows a first time through L1 (chunk_dot per float4, then the
//   butterfly of dfk_geom.cuh over the C/4 chunk sums: the offsets >= 8 inside a lane's registers, 4, 2, 1 across
//   the 8 lanes), bit for bit what dfk_update_depth computes.
//
// The per-item block, the tile -> CTA assignment, the in-item tile permutation and the per-pixel row come from
// dfk_sfm_frontend.cuh; the finalize is the tensor-core one of dfk_sfm_finalize.cu.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_async.cuh"
#include "dfk_geom.cuh"
#include "dfk_internal.h"
#include "dfk_sfm_frontend.cuh"
#include "dfk_sfm_tc_common.cuh"
#include "dfk_wgmma.cuh"

namespace dfk {

namespace {

constexpr int TILE = 128;
static_assert(TILE == sfm_tc_tile_pixels(64) && TILE == sfm_tc_tile_pixels(128), "tile size");
constexpr uint32_t kLbo = 128 + 16;        // core matrices adjacent in K (4 pixels)
constexpr uint32_t kSbo = 32 * kLbo + 16;  // 8-row groups (a group spans the tile's 32 core matrices)
constexpr int kFlushTiles = 8;             // accumulation chain length (tiles)

template <int C>
struct WgCfg {
  using T = TcCfg<C>;
  static constexpr int NWG = C >= 128 ? 2 : 1;  // warpgroups
  static constexpr int THREADS = 128 * NWG;
  static constexpr int NWARP = THREADS / 32;
  static constexpr int PW = 32 / NWG;          // pixels per warp
  static constexpr int N = T::COLS;            // C + 24
  static constexpr int NACC = N / 2;           // accumulator floats per thread and M-tile
  static constexpr int NCB = C / 32;           // 32-feature blocks of a code row
  static constexpr int GROUPS = T::F / 4;      // 8-row groups of the operand buffer
  static constexpr int G_H = T::S / 8;         // first h group (= B's first group)
  static constexpr int G_LT = G_H + T::F / 8;  // code-l S..C-1, then pose-l
  static constexpr uint32_t OP_BYTES = GROUPS * kSbo;
  static_assert(T::ROWS == 128 * NWG, "two 64-row M-tiles per warpgroup");
};

template <int C>
struct Smem {
  alignas(128) unsigned char op[WgCfg<C>::OP_BYTES];
  SfmItem<C> item[WgCfg<C>::NWARP];
};

template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, bool accumulate)
{
  if constexpr (N == 88) wgmma_m64n88k8_tf32(d, a_desc, b_desc, accumulate);
  else wgmma_m64n152k8_tf32(d, a_desc, b_desc, accumulate);
}

template <int C>
__global__ void __launch_bounds__(WgCfg<C>::THREADS, sfm_tc_ctas_per_sm(C))
sfm_step_tc_wide_kernel(const SfmItemDev* __restrict__ items, int num_tiles, float* __restrict__ partials)
{
  using W = WgCfg<C>;
  using T = TcCfg<C>;
  constexpr int PW = W::PW;
  constexpr int N = W::N;
  constexpr int NACC = W::NACC;
  constexpr int NCB = W::NCB;
  constexpr int NQ = PW / 4;  // pixel quads per warp
  // quads whose code rows are loaded before the wait for the MMAs: all of them at C = 64; none at C = 128, where the
  // 152 accumulators leave registers for one quad at a time (each quad is loaded, then stored, after the wait)
  constexpr int PRE = C >= 128 ? 0 : NQ;
  constexpr int S = T::S;
  constexpr int F = T::F;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem<C>& sm = *reinterpret_cast<Smem<C>*>(smem_raw);
  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int wg = tid >> 7;
  int g_lo, g_hi;
  cta_tiles(num_tiles, g_lo, g_hi);
  const int ntiles = g_hi - g_lo;
  if (ntiles <= 0) return;

  // row 7 of the pose groups (the zero feature) is never written: zeros
  for (int e = tid; e < (int)(W::OP_BYTES / 16); e += W::THREADS)
    reinterpret_cast<float4*>(sm.op)[e] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();

  const uint32_t op = smem_u32(sm.op);
  // code-Jacobian stores: this lane holds features 32 cb + 4 c .. + 3 of pixel 4 i + r of the warp's PW pixels
  const int c = lane & 7, r = lane >> 3;
  const uint32_t in_group = (uint32_t)(PW / 4 * warp) * kLbo + (uint32_t)(c & 1) * 64u + (uint32_t)r * 4u;
  const uint32_t code_l = op + (uint32_t)(c >> 1) * kSbo + in_group;  // code-l of features 4 c .. + 3 (block 0)
  const uint32_t code_lt = op + (uint32_t)W::G_LT * kSbo + in_group;  // code-l of features S .. C - 1
  // pose stores: the lane's own pixel (lane < PW)
  const int own = lane % PW;
  const uint32_t own_off = (uint32_t)((PW * warp + own) >> 2) * kLbo + (uint32_t)(own & 3) * 4u;
  const uint32_t pose_h = op + (uint32_t)(W::G_H + C / 8) * kSbo + own_off;
  constexpr uint32_t kPoseL = (uint32_t)(W::G_LT + 1 - W::G_H - C / 8) * kSbo;  // pose-l group - pose-h group

  float acc[2][NACC];
#pragma unroll
  for (int t = 0; t < 2; ++t)
#pragma unroll
    for (int q = 0; q < NACC; ++q) acc[t][q] = 0.0f;  // never read before a chain's first MMA overwrites them
  SfmItem<C>& I = sm.item[warp];
  int it = 0;
  int cur_item = -1;
  uint32_t item_hi = 0;  // end of the global tile range of the item in shared memory
  int tiles_in_chain = 0, chain_valid = 0, pslot = 0;
  bool fresh = true;
  unsigned int inliers = 0;

  // close the chain: add the accumulators to the partial (the first chain of an item in this CTA stores)
  auto flush = [&](bool item_end) {
    wgmma_wait_all();
    float* P = partials + (size_t)pslot * T::PARTIAL_FLOATS;
    if (fresh || chain_valid > 0) {
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        const int m0 = 64 * (2 * wg + t) + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
        for (int q = 0; q < NACC; ++q) {
          const int m = m0 + 8 * ((q >> 1) & 1);
          const int n = 8 * (q >> 2) + 2 * (lane & 3) + (q & 1);
          // rows < S of columns >= F: l*l terms; rows >= S of columns < F: HH, read for j >= i only
          const bool used = m < S ? n < F : (n >= F || n >= m - S);
          if (used) put_partial(P + n * T::ROWS + m, chain_valid > 0 ? acc[t][q] : 0.0f, fresh);
        }
      }
    }
    if (item_end && tid == 0) reinterpret_cast<unsigned int*>(P)[T::INLIERS] = inliers;
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
    const uint32_t s = (uint32_t)(PW * warp + own);  // pixel slot in the tile
    const bool inb = lane < PW && s < n;
    const bool blk_live = (uint32_t)(PW * warp) < n;  // else: a block past the end of the item's last tile
    const uint32_t Wd = I.width;
    const bool a16 = (I.flags & ITEM_FLAG_BULK) != 0;
    const bool fused = (I.flags & ITEM_FLAG_FUSED_DEPTH) != 0;
    // block origin (uniform) by one division, then this lane's pixel by wrap-around; lanes that own no pixel of the
    // tile shadow the block's first pixel (their loads stay in bounds, their contribution is zero)
    uint32_t x0;
    const uint32_t y0 = div_magic(blk_live ? p0 + (uint32_t)(PW * warp) : p0, Wd, I.mag_width, x0);
    uint32_t pxx = x0 + (inb ? (uint32_t)own : 0u), py = y0;
    while (pxx >= Wd) {
      pxx -= Wd;
      ++py;
    }
    const float* __restrict__ jac = I.jac;
    const uint32_t joff = py * I.jac_pitch + pxx * C;  // this lane's pixel's code-Jacobian row (floats)
    float feat[8];
    bool ok = false;
    if (blk_live) {
      const float2 ray = table_ray(I, pxx, py);
      float d = ld_stream(I.dpt0 + (size_t)py * I.dpt0_pitch + pxx);
      const float i0 = ld_stream(I.img0 + (size_t)py * I.img0_pitch + pxx);
      if (fused) {
        // dpt0 is prx_orig: decode the depth from the pixel's code-Jacobian row with the arithmetic of
        // update_depth_kernel, here across the 8 lanes (and the NCB registers) that hold the chunks of one pixel
        float mine = 0.0f;
#pragma unroll
        for (int i4 = 0; i4 < PW / 4; ++i4) {
          const uint32_t offk = __shfl_sync(0xffffffffu, joff, 4 * i4 + r);
          float p[NCB];
#pragma unroll
          for (int cb = 0; cb < NCB; ++cb) {
            const float4 cc = *reinterpret_cast<const float4*>(&I.code[32 * cb + 4 * c]);
            p[cb] = chunk_dot(load_chunk_l1(jac + offk + 32 * cb + 4 * c, a16), cc);
          }
#pragma unroll
          for (int o = NCB / 2; o > 0; o >>= 1)  // chunk offsets C/8 .. 8: inside the lane
#pragma unroll
            for (int j = 0; j < o; ++j) p[j] = __fadd_rn(p[j], p[j + o]);
          float q = p[0];
          q = __fadd_rn(q, __shfl_xor_sync(0xffffffffu, q, 4));
          q = __fadd_rn(q, __shfl_xor_sync(0xffffffffu, q, 2));
          q = __fadd_rn(q, __shfl_xor_sync(0xffffffffu, q, 1));
          const float got = __shfl_sync(0xffffffffu, q, 8 * (lane & 3));  // pixel 4 i4 + (lane & 3)
          if ((own >> 2) == i4) mine = got;
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
    float4 v[NQ][NCB];
    auto load_quad = [&](int i4) {
      const uint32_t offk = __shfl_sync(0xffffffffu, joff, 4 * i4 + r);
      const bool live = (bal >> (4 * i4 + r)) & 1u;
#pragma unroll
      for (int cb = 0; cb < NCB; ++cb) {
        v[i4][cb] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live) v[i4][cb] = load_chunk(jac + offk + 32 * cb + 4 * c, a16);
      }
    };
#pragma unroll
    for (int i4 = 0; i4 < PRE; ++i4) load_quad(i4);
    // ---- the operand buffer is free once every warpgroup's MMAs of the previous tile have completed -------------------
    wgmma_wait_all();
    if constexpr (W::NWG > 1) __syncthreads();
#pragma unroll
    for (int i4 = 0; i4 < NQ; ++i4) {
      if (i4 >= PRE) load_quad(i4);
      const float sk = __shfl_sync(0xffffffffu, feat[0], 4 * i4 + r);
#pragma unroll
      for (int cb = 0; cb < NCB; ++cb) {
        const float x[4] = {sk * v[i4][cb].x, sk * v[i4][cb].y, sk * v[i4][cb].z, sk * v[i4][cb].w};
        // feature group 4 cb + c / 2: its h rows, and its l rows (only the last 8 code features have theirs in B)
        const uint32_t gh = code_l + (uint32_t)(W::G_H + 4 * cb) * kSbo;
        const uint32_t gl = (cb < NCB - 1 || c < 6) ? code_l + (uint32_t)(4 * cb) * kSbo : code_lt;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float h = tf32_trunc(x[e]);
          const uint32_t off = (uint32_t)i4 * kLbo + (uint32_t)e * 16u;
          sts32(gh + off, h);
          sts32(gl + off, x[e] - h);
        }
      }
    }
    if (lane < PW) {
#pragma unroll
      for (int f = 0; f < 7; ++f) {
        const float h = tf32_trunc(feat[1 + f]);
        sts32(pose_h + (uint32_t)f * 16u, h);
        sts32(pose_h + kPoseL + (uint32_t)f * 16u, feat[1 + f] - h);
      }
    }
    fence_proxy_async_smem();  // generic-proxy writes -> visible to the MMA's operand fetch
    const int nv = __syncthreads_count(ok);
    if (nv > 0) {
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < TILE / 8; ++kk) {
        const uint32_t k_off = (uint32_t)kk * 2u * kLbo;
        const bool accumulate = kk > 0 || chain_valid > 0;
        const uint64_t b_desc = make_wgmma_desc_kmajor(op + (uint32_t)W::G_H * kSbo + k_off, kLbo, kSbo);
#pragma unroll
        for (int t = 0; t < 2; ++t)
          wgmma_tf32<N>(acc[t], make_wgmma_desc_kmajor(op + (uint32_t)(8 * (2 * wg + t)) * kSbo + k_off, kLbo, kSbo),
                        b_desc, accumulate);
      }
      wgmma_commit();
    }
    chain_valid += nv;
    inliers += (unsigned)nv;
    ++tiles_in_chain;
  }
  flush(true);
}

template <int C>
cudaError_t launch_impl(const SfmItemDev* items_dev, const SfmLaunchPlan& plan, float* partials_dev,
                        cudaStream_t stream, cudaEvent_t ev_start, cudaEvent_t ev_stop)
{
  const size_t smem = sizeof(Smem<C>);
  // above the 48 KB default: the limit belongs to the current device, and a process may run handles on several
  cudaError_t err =
      cudaFuncSetAttribute(sfm_step_tc_wide_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (err != cudaSuccess) return err;
  if (ev_start) cudaEventRecord(ev_start, stream);
  sfm_step_tc_wide_kernel<C><<<plan.num_ctas, WgCfg<C>::THREADS, smem, stream>>>(items_dev, plan.num_tiles,
                                                                                  partials_dev);
  if (ev_stop) cudaEventRecord(ev_stop, stream);
  return cudaGetLastError();
}

}  // namespace

bool sfm_tc_wide_supported(int code_size) { return code_size == 64 || code_size == 128; }

cudaError_t launch_sfm_tc_wide(int code_size, const SfmItemDev* items_dev, const SfmLaunchPlan& plan,
                               float* partials_dev, cudaStream_t stream, cudaEvent_t ev_start, cudaEvent_t ev_stop)
{
  switch (code_size) {
    case 64: return launch_impl<64>(items_dev, plan, partials_dev, stream, ev_start, ev_stop);
    case 128: return launch_impl<128>(items_dev, plan, partials_dev, stream, ev_start, ev_stop);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace dfk
