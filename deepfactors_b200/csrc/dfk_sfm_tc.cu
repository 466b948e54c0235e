// dfk_sfm_tc.cu -- SfmAligner::RunStep hot path, Hopper warpgroup tensor-core Gram (sm_90a, C = 32, 64, 128).
//
// Same contract as dfk_sfm_fp32.cu (replaces kernel_step_calculate + DenseSfm + the two-kernel reduction of
// sources/cuda/cu_sfmaligner.cpp:40-70,149-185, dense_sfm.h:133-201), different engine for the reduced Gram
// G = sum_p m_p^T m_p,  m = w*[ e*jc (C) | a (6) | diff (1) | 0 ]  (F = C + 8 features):
//
//   Split precision ("3xTF32" folded into one product): every feature value v is split exactly into h = v with the
//   low 13 mantissa bits cleared (exactly representable in tf32) and l = v - h.  The tf32 MMAs yield HH = sum h h^T and
//   LH = sum l h^T;  G = HH + LH + LH^T  drops only the l*l terms (~2^-22).
//
//   Packing (dfk_internal.h, TcCfg): A = [ code-l 0..S-1 ; h 0..F-1 ], B = [ h 0..F-1 ; code-l S..C-1 ; pose-l ],
//   S = C - 8, so D = A x B^T (2C x (C + 24)) holds every h*h and l*h product G needs.  The operand buffer holds the
//   F/4 groups of 8 feature rows once, in the order  code-l 0..S-1 | h 0..F-1 | code-l S..C-1 | pose-l:  A is its
//   first 2C rows, B its last C + 24 rows, one descriptor stride each (C = 32: 10 groups, A = groups 0-7, M = 64,
//   B = groups 3-9, N = 56).  Inside a group the core matrix of pixels 4q..4q+3 sits at q * kLbo, feature row r of it
//   at r * 16; kLbo / kSbo carry 16 bytes of padding each, so the code-h and pose stores of a warp hit 32 different
//   banks.  Every tile writes every byte the descriptors read except row 7 (the zero feature) of the pose-h and pose-l
//   groups, which the prologue zeroes.
//
//   CTA: NWG warpgroups over one operand buffer of 128 pixels (K = 128 per tile), each warpgroup owning MT 64-row
//   M-tiles of D in registers (C = 32: one warpgroup, one M-tile, 28 floats per thread, four CTAs per SM; C = 64: one
//   warpgroup, two M-tiles, 88 floats per thread, two CTAs per SM; C = 128: two warpgroups, two M-tiles each, 152
//   floats per thread, one CTA per SM).  Warp w runs the per-pixel front-end ((optional depth decode,) exact-order
//   validity chain, bilinear gathers, Jacobian row, Huber -> s = w*e, w*a[6], w*diff) for the PW = 32 / NWG pixels
//   PW w .. PW w + PW - 1 (lane < PW: its own pixel), and the warp reads the valid pixels' code-Jacobian rows straight
//   from global memory, coalesced (lane = 16-byte chunk lane & 7 of a 32-feature block of pixel 4i + lane / 8): at
//   C = 32 right after the validity chain and the ballot, so that they load while the gathers run; at C = 64 and 128
//   after the Huber weight.  Then it scales them by the pixel's s (one shuffle), splits them into h / l and stores them
//   K-major; each lane < PW adds its own pixel's 7 pose / residual values.  Invalid pixels contribute exact zeros, and
//   a tile with no valid pixel issues no MMA; at C = 32 it stops right after the validity chain (one CTA barrier that
//   counts the tile's valid pixels), before the code rows, the gathers and the operand stores.
//   After one CTA barrier every warpgroup issues 16 k-steps x MT M-tiles of wgmma.m64nNk8 and, without waiting, goes on
//   with the next tile's gathers; it waits for its MMAs only before the operand buffer is overwritten (with two
//   warpgroups, a CTA barrier after the wait keeps one warpgroup from overwriting what the other still reads).
//
//   A chain is cut every kFlushTiles tiles and at item boundaries and added in round-to-nearest fp32 to the CTA's
//   partial (single writer per address, program order).  What the partial holds is sfm_tc_writes_d(C):
//     C = 32: the fragments are staged in the (then idle) operand buffer, combined into G = (HH + LH) + LH^T and
//             written in the fp32 kernel's format (SfmCfg<32>: G row-major, upper triangle);
//     C = 64, 128: D itself (TcCfg<C>, column-major), only what the finalize reads: neither the l*l block nor the
//             lower triangle of HH.
//
//   Input stream: the code-Jacobian rows, img0 and dpt0 are read once, through loads that do not allocate in L1 (L1 is
//   left to the bilinear gathers of img1 / grad1, the only loads that reuse lines; the fused depth decode reads the code
//   rows a first time through L1, so that the Gram's second read hits there: chunk_dot per float4, then the butterfly
//   of dfk_geom.cuh over the C/4 chunk sums, the offsets >= 8 inside a lane's registers, 4, 2, 1 across the 8 lanes,
//   bit for bit what dfk_update_depth computes).  Nothing is prefetched: on H100 both a per-thread L2 prefetch of the
//   pixel's code row and bulk L2 prefetches of a later tile made the kernel slower.
//
// The per-item block, the static tile->CTA assignment, the in-item tile permutation and the per-pixel row (ray table,
// validity chain, gathers, Jacobian row, Huber) come from dfk_sfm_frontend.cuh, as in the fp32 and wide kernels; this
// kernel keeps its own tile walk (every warp owns a copy of the item block) and its cross-lane depth decode.  The
// deterministic finalize is dfk_sfm_finalize.cu's, for the partial format above.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_async.cuh"
#include "dfk_geom.cuh"
#include "dfk_internal.h"
#include "dfk_sfm_frontend.cuh"
#include "dfk_wgmma.cuh"

namespace dfk {

namespace {

constexpr int TILE = kSfmTcTilePixels;     // 128
constexpr uint32_t kLbo = 128 + 16;        // core matrices adjacent in K (4 pixels)
constexpr uint32_t kSbo = 32 * kLbo + 16;  // 8-row groups (a group spans the tile's 32 core matrices)
#ifndef DFK_FLUSH_TILES
#define DFK_FLUSH_TILES 8
#endif
constexpr int kFlushTiles = DFK_FLUSH_TILES;  // accumulation chain length (tiles)

template <int C>
struct WgCfg {
  using T = TcCfg<C>;
  static constexpr int NWG = C >= 128 ? 2 : 1;     // warpgroups
  static constexpr int THREADS = 128 * NWG;
  static constexpr int NWARP = THREADS / 32;
  static constexpr int MT = T::ROWS / (64 * NWG);  // 64-row M-tiles of D per warpgroup
  static constexpr int PW = 32 / NWG;              // pixels per warp
  static constexpr int N = T::COLS;                // C + 24
  static constexpr int NACC = N / 2;               // accumulator floats per thread and M-tile
  static constexpr int NCB = C / 32;               // 32-feature blocks of a code row
  static constexpr int GROUPS = T::F / 4;          // 8-row groups of the operand buffer
  static constexpr int G_H = T::S / 8;             // first h group (= B's first group)
  static constexpr int G_LT = G_H + T::F / 8;      // code-l S..C-1, then pose-l
  static constexpr uint32_t OP_BYTES = GROUPS * kSbo;
};

template <int C>
struct Smem {
  alignas(128) unsigned char op[WgCfg<C>::OP_BYTES];
  SfmItem<C> item[WgCfg<C>::NWARP];
};

// the C = 32 flush stages D (64 x 56) row-major in the operand buffer; the odd row stride keeps the column reads of LH
// conflict-free
constexpr int kDStride = 57;
static_assert(64 * kDStride * 4 <= 7 * kSbo, "the staged D must leave row 7 of the pose groups alone");
// LH[i][j] in the staged D
__device__ __forceinline__ int lh(int i, int j) { return i < 24 ? i * kDStride + j : (24 + j) * kDStride + 16 + i; }

__device__ __forceinline__ float tf32_trunc(float v) { return __uint_as_float(__float_as_uint(v) & 0xffffe000u); }

__device__ __forceinline__ void sts32(uint32_t addr, float v)
{
  // no "memory" clobber: the only plain shared-memory accesses of the front-end are reads of its item copy; volatile
  // keeps the stores ordered with the proxy fence (which carries the clobber)
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v));
}

// read-once input stream (code-Jacobian rows, img0, dpt0): read-only path, no L1 allocation
__device__ __forceinline__ float ld_stream(const float* p)
{
  float v;
  asm("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}

// 16 bytes of a code-Jacobian row; rows of items without the BULK flag are only 4-byte aligned
__device__ __forceinline__ float4 load_chunk(const float* __restrict__ p, bool aligned16)
{
  if (aligned16) {
    float4 v;
    asm("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
        : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
        : "l"(p));
    return v;
  }
  return make_float4(ld_stream(p), ld_stream(p + 1), ld_stream(p + 2), ld_stream(p + 3));
}

// the same 16 bytes through L1: the fused depth decode reads every chunk the Gram reads again a little later (the
// no-allocate loads of load_chunk still hit lines that are in L1)
__device__ __forceinline__ float4 load_chunk_l1(const float* __restrict__ p, bool aligned16)
{
  if (aligned16) return __ldg(reinterpret_cast<const float4*>(p));
  return make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3));
}

// the first chain of an item in this CTA stores, later chains add (single writer per address, program order)
__device__ __forceinline__ void put_partial(float* p, float v, bool fresh)
{
  if (fresh)
    __stcg(p, v);
  else
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, bool accumulate)
{
  if constexpr (N == 56) wgmma_m64n56k8_tf32(d, a_desc, b_desc, accumulate);
  else if constexpr (N == 88) wgmma_m64n88k8_tf32(d, a_desc, b_desc, accumulate);
  else wgmma_m64n152k8_tf32(d, a_desc, b_desc, accumulate);
}

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

template <int C>
__global__ void __launch_bounds__(WgCfg<C>::THREADS, sfm_tc_ctas_per_sm(C))
sfm_step_tc_kernel(const SfmItemDev* __restrict__ items, int num_tiles, float* __restrict__ partials)
{
  using W = WgCfg<C>;
  using T = TcCfg<C>;
  using Cfg = SfmCfg<C>;
  constexpr int MT = W::MT;
  constexpr int PW = W::PW;
  constexpr int N = W::N;
  constexpr int NACC = W::NACC;
  constexpr int NCB = W::NCB;
  constexpr int NQ = PW / 4;  // pixel quads per warp
  // quads whose code rows are loaded before the wait for the MMAs: all of them at C = 32 and 64; none at C = 128, where
  // the 152 accumulators leave registers for one quad at a time (each quad is loaded, then stored, after the wait)
  constexpr int PRE = C >= 128 ? 0 : NQ;
  // C = 32 issues the code rows between the validity chain and the gathers (DESIGN §4.1); C = 64 and 128, whose 88 / 152
  // accumulators already take them to 255 registers, issue them after the Huber weight
  constexpr bool EARLY_ROWS = C == 32;
  constexpr int S = T::S;
  constexpr int F = T::F;
  constexpr bool kRawD = sfm_tc_writes_d(C);
  constexpr int PARTIAL_FLOATS = kRawD ? T::PARTIAL_FLOATS : Cfg::PARTIAL_FLOATS;
  constexpr int INLIERS = kRawD ? T::INLIERS : Cfg::NFP * Cfg::NFP;  // offset of the inlier count (u32)
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Smem<C>& sm = *reinterpret_cast<Smem<C>*>(smem_raw);
#ifdef DFK_EXP_CTA_CLOCKS
  const unsigned long long t_entry = global_ns();
  int valid_tiles = 0;
#endif
  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int wg = W::NWG > 1 ? tid >> 7 : 0;
  int g_lo, g_hi;
  cta_tiles(num_tiles, g_lo, g_hi);
  const int ntiles = g_hi - g_lo;
  if (ntiles <= 0) return;

  // row 7 of the pose-h and pose-l groups (the zero feature) is never written: zeros.  C = 32 zeroes just these rows;
  // C = 64 and 128 zero the whole buffer, since the C = 128 kernel compiled with the row-7 form ran slower (DESIGN §4.2c)
  if constexpr (C == 32) {
    if (tid < 64)
      *reinterpret_cast<float4*>(sm.op + (tid < 32 ? W::G_H + C / 8 : W::G_LT + 1) * kSbo + (tid & 31) * kLbo + 7 * 16) =
          make_float4(0.f, 0.f, 0.f, 0.f);
  } else {
    for (int e = tid; e < (int)(W::OP_BYTES / 16); e += W::THREADS)
      reinterpret_cast<float4*>(sm.op)[e] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();

  const uint32_t op = smem_u32(sm.op);
  // code-Jacobian stores: this lane holds features 32 cb + 4 c .. + 3 of pixel 4 i + r of the warp's PW pixels
  const int c = lane & 7, r = lane >> 3;
  const uint32_t in_group = (uint32_t)(PW / 4 * warp) * kLbo + (uint32_t)(c & 1) * 64u + (uint32_t)r * 4u;
  // h and l rows of features 32 cb + 4 c .. + 3: h at code_h + 4 cb groups, l at code_l + 4 cb groups, except in the
  // last block, whose last 8 features have their l rows in B (group G_LT)
  const uint32_t code_l_last = op + (uint32_t)((c >> 1) < 3 ? (c >> 1) + 4 * (NCB - 1) : W::G_LT) * kSbo + in_group;
  const uint32_t code_h = op + (uint32_t)(W::G_H + (c >> 1)) * kSbo + in_group;
  const uint32_t code_l = op + (uint32_t)(c >> 1) * kSbo + in_group;
  // pose stores: the lane's own pixel (lane < PW)
  const int own = lane % PW;
  const uint32_t pose_h =
      op + (uint32_t)(W::G_H + C / 8) * kSbo + (uint32_t)(PW / 4 * warp + (own >> 2)) * kLbo + (uint32_t)(own & 3) * 4u;
  const uint32_t pose_l = pose_h + (uint32_t)(W::G_LT + 1 - W::G_H - C / 8) * kSbo;

  float acc[MT][NACC];
#pragma unroll
  for (int t = 0; t < MT; ++t)
#pragma unroll
    for (int q = 0; q < NACC; ++q) acc[t][q] = 0.0f;  // never read before a chain's first MMA overwrites them
  SfmItem<C>& I = sm.item[warp];
  uint32_t item_hi = 0;  // end of the global tile range of the item in shared memory
  int it = 0;
  int cur_item = -1;
  int tiles_in_chain = 0, chain_valid = 0, pslot = 0;
  bool fresh = true;
  unsigned int inliers = 0;

  // close the chain: add it to the partial (the first chain of an item in this CTA stores).  The accumulators are only
  // ever written by the MMAs (a chain's first MMA overwrites them), so ptxas can keep them in flight across the next
  // tile's front-end
  auto flush = [&](bool item_end) {
    wgmma_wait_all();
    float* P = partials + (size_t)pslot * PARTIAL_FLOATS;
    if (fresh || chain_valid > 0) {  // uniform across the CTA, like all chain bookkeeping
      if constexpr (kRawD) {
#pragma unroll
        for (int t = 0; t < MT; ++t) {
          const int m0 = 64 * (MT * wg + t) + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
          for (int q = 0; q < NACC; ++q) {
            const int m = m0 + 8 * ((q >> 1) & 1);
            const int n = 8 * (q >> 2) + 2 * (lane & 3) + (q & 1);
            // rows < S of columns >= F: l*l terms; rows >= S of columns < F: HH, read for j >= i only
            const bool used = m < S ? n < F : (n >= F || n >= m - S);
            if (used) put_partial(P + n * T::ROWS + m, chain_valid > 0 ? acc[t][q] : 0.0f, fresh);
          }
        }
      } else {
        // G = (HH + LH) + LH^T.  D goes through the operand buffer, free once the chain's MMAs have completed; the next
        // tile's operand stores rewrite every byte the MMAs read
        static_assert(C == 32 && MT == 1, "the staged D is the one M-tile of one warpgroup at C = 32");
        const bool have = chain_valid > 0;
        float* Ds = reinterpret_cast<float*>(sm.op);
        if (have) {
          __syncthreads();  // every warp's share of the chain's MMAs has completed
          const int m0 = 16 * warp + (lane >> 2);
#pragma unroll
          for (int q = 0; q < NACC; ++q)
            Ds[(m0 + 8 * ((q >> 1) & 1)) * kDStride + 8 * (q >> 2) + 2 * (lane & 3) + (q & 1)] = acc[0][q];
          __syncthreads();
        }
        // entries (i, j), i <= j < NF, of the row-major NFP x NFP partial: the ones the finalize reads
        for (int e = tid; e < Cfg::NFP * Cfg::NFP; e += W::THREADS) {
          const int i = e / Cfg::NFP, j = e - Cfg::NFP * i;
          if (i > j || j >= Cfg::NF) continue;
          float g = 0.0f;
          if (have) g = (Ds[(S + i) * kDStride + j] + Ds[lh(i, j)]) + Ds[lh(j, i)];
          put_partial(P + e, g, fresh);
        }
        if (have) __syncthreads();  // the staged D is read before the next tile's operand stores overwrite it
      }
    }
    if (item_end && tid == 0) reinterpret_cast<unsigned int*>(P)[INLIERS] = inliers;
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
    // the per-pixel row in its two halves (dfk_sfm_frontend.cuh): the validity first, then the gathers, Jacobian and
    // Huber of the valid pixels
    Warped w;
    float d = 0.0f, i0 = 0.0f;
    bool ok = false;
    if (blk_live) {
      const float2 ray = table_ray(I, pxx, py);  // issued before the decode: its latency hides behind it
      d = ld_stream(I.dpt0 + (size_t)py * I.dpt0_pitch + pxx);
      i0 = ld_stream(I.img0 + (size_t)py * I.img0_pitch + pxx);
      if (fused) {
        // dpt0 is prx_orig: decode the depth from the pixel's code-Jacobian row with the arithmetic of
        // update_depth_kernel's vector body, here across the 8 lanes (and the NCB registers) that hold the chunks of
        // one pixel
        float4 cc[NCB];
#pragma unroll
        for (int cb = 0; cb < NCB; ++cb) cc[cb] = *reinterpret_cast<const float4*>(&I.code[32 * cb + 4 * (lane & 7)]);
        float mine = 0.0f;
#pragma unroll
        for (int i4 = 0; i4 < NQ; ++i4) {
          const uint32_t offk = __shfl_sync(0xffffffffu, joff, 4 * i4 + r);
          float p[NCB];
#pragma unroll
          for (int cb = 0; cb < NCB; ++cb) p[cb] = chunk_dot(load_chunk_l1(jac + offk + 32 * cb + 4 * (lane & 7), a16), cc[cb]);
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
      if (inb) {
        w = pixel_warp(I, ray, d);
        ok = w.valid;
      }
    }
    // C = 32: a tile without a valid pixel (about a third of them at the reference poses) ends here, once every warp knows
    // its validity: no code rows, gathers, operand stores or MMAs, and no wait for the previous tile's MMAs.  Its chain
    // bookkeeping is the same as if it had run (it counts towards the flush), so the sums are bitwise the same
    if constexpr (C == 32) {
      if (__syncthreads_count(ok) == 0) {
        ++tiles_in_chain;
        continue;
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    float4 v[NQ][NCB];
    const float* jc = jac + 4 * c;  // this lane's 16-byte chunk of a 32-feature block of a code row
    auto load_quad = [&](int i4) {
      const uint32_t offk = __shfl_sync(0xffffffffu, joff, 4 * i4 + r);
      const bool live = (bal >> (4 * i4 + r)) & 1u;
#pragma unroll
      for (int cb = 0; cb < NCB; ++cb) {
        v[i4][cb] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live) v[i4][cb] = load_chunk(jc + offk + 32 * cb, a16);
      }
    };
    // EARLY_ROWS: the valid pixels' code rows are issued as soon as the ballot is known, and load while the gathers run
    if constexpr (EARLY_ROWS) {
#pragma unroll
      for (int i4 = 0; i4 < PRE; ++i4) load_quad(i4);
    }
    float feat[8];
    if (ok) {
      valid_pixel_row(I, pxx, py, w, d, i0, true, feat);  // the API guarantees 8-byte grad1 rows here
    } else {
#pragma unroll
      for (int f = 0; f < 8; ++f) feat[f] = 0.0f;
    }
    if constexpr (!EARLY_ROWS) {
#pragma unroll
      for (int i4 = 0; i4 < PRE; ++i4) load_quad(i4);
    }
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
        const uint32_t gh = code_h + (uint32_t)(4 * cb) * kSbo;
        const uint32_t gl = cb < NCB - 1 ? code_l + (uint32_t)(4 * cb) * kSbo : code_l_last;
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
        sts32(pose_l + (uint32_t)f * 16u, feat[1 + f] - h);
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
#ifndef DFK_EXP_NOMMA  // experiment (wrong results): no MMA at all
        const uint64_t b_desc = make_wgmma_desc_kmajor(op + (uint32_t)W::G_H * kSbo + k_off, kLbo, kSbo);
#pragma unroll
        for (int t = 0; t < MT; ++t)
          wgmma_tf32<N>(acc[t], make_wgmma_desc_kmajor(op + (uint32_t)(8 * (MT * wg + t)) * kSbo + k_off, kLbo, kSbo),
                        b_desc, accumulate);
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

template <int C>
cudaError_t launch_impl(const SfmItemDev* items_dev, const SfmLaunchPlan& plan, float* partials_dev,
                        cudaStream_t stream, cudaEvent_t ev_start, cudaEvent_t ev_stop)
{
  constexpr size_t smem = sizeof(Smem<C>);
  // above the 48 KB default the kernel needs the opt-in, which belongs to the current device (a process may run handles
  // on several), so it is set on every launch; below it, a launch makes no driver call besides the launch itself
  if constexpr (smem > 48 * 1024) {
    const cudaError_t err =
        cudaFuncSetAttribute(sfm_step_tc_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err != cudaSuccess) return err;
  }
  if (ev_start) cudaEventRecord(ev_start, stream);
  sfm_step_tc_kernel<C><<<plan.num_ctas, WgCfg<C>::THREADS, smem, stream>>>(items_dev, plan.num_tiles, partials_dev);
  if (ev_stop) cudaEventRecord(ev_stop, stream);
  return cudaGetLastError();
}

}  // namespace

bool sfm_tc_supported(int code_size) { return code_size == 32 || code_size == 64 || code_size == 128; }

cudaError_t launch_sfm_tc(int code_size, const SfmItemDev* items_dev, const SfmLaunchPlan& plan, float* partials_dev,
                          cudaStream_t stream, cudaEvent_t ev_start, cudaEvent_t ev_stop)
{
  switch (code_size) {
    case 32: return launch_impl<32>(items_dev, plan, partials_dev, stream, ev_start, ev_stop);
    case 64: return launch_impl<64>(items_dev, plan, partials_dev, stream, ev_start, ev_stop);
    case 128: return launch_impl<128>(items_dev, plan, partials_dev, stream, ev_start, ev_stop);
    default: return cudaErrorInvalidValue;
  }
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
