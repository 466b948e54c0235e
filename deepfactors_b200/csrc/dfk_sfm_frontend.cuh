// dfk_sfm_frontend.cuh -- what the three SfmAligner::RunStep kernels (dfk_sfm_tc.cu: tensor cores, C = 32, 64, 128;
// dfk_sfm_fp32.cu; dfk_sfm_wide.cu)
// share in front of their Gram engines:
//   * the per-item parameter block kept in shared memory (one per CTA, one per warp in the tensor-core kernel);
//   * the static tile -> CTA assignment and the in-item tile permutation: tile k of an item is processed as
//     (k * perm_mul) % num_tiles (dfk_internal.h);
//   * the per-pixel row of the reduced system -- the one place where the exact-order validity chain, valid0, the
//     bilinear gathers, the Jacobian row and the Huber weight meet (DESIGN §2: inlier sets bit-identical to the CPU);
//   * the CUDA-core pipeline of the fp32 and wide kernels: a ring of tile stages filled by the bulk-copy engine (row
//     segments, one issuing thread) or by a cooperative copy for items whose buffers are not 16-byte friendly; a
//     front-end role, one thread per tile pixel, that writes the tile's rows compacted (valid pixels first) into a
//     double-buffered M; and the Gram-role scaffold that drains M.  A kernel supplies its M layout and its block
//     accumulation / flush.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_async.cuh"
#include "dfk_geom.cuh"
#include "dfk_internal.h"

namespace dfk {

// per-item parameters the front-end needs, copied to shared memory when a CTA (warp) enters an item
template <int MAXCODE>
struct SfmItem {
  float q[4];
  float t[3];
  float R[9];
  float fx, fy, u0, v0, border, ulim, vlim, min_dpt, avg_dpt, huber_delta;
  const float* img0;
  const float* img1;
  const float* dpt0;
  float* valid0;
  const float* jac;
  const float* grad1;
  const float* ray_tab;
  float* dpt_out;  // fused depth decode (ITEM_FLAG_FUSED_DEPTH): decoded depth goes here, dpt0 then is prx_orig
  uint32_t img0_pitch, img1_pitch, dpt0_pitch, valid0_pitch, jac_pitch, grad1_pitch, dpt_out_pitch;
  uint32_t width, height, num_pixels, tile_begin, num_tiles, perm_mul, flags, slot, mag_tiles, mag_width;
  alignas(16) float code[MAXCODE];  // fused depth decode: the latent code of the item
};

// lanes 0-20 of one warp copy the fields; a caller with more threads passes its thread index (the others skip).
// Callers sync afterwards.
template <int MAXCODE>
__device__ __forceinline__ void load_item(SfmItem<MAXCODE>& dst, const SfmItemDev& src, int lane, int cta)
{
  if (lane < 4) dst.q[lane] = src.q[lane];
  if (lane >= 4 && lane < 7) dst.t[lane - 4] = src.t[lane - 4];
  if (lane >= 8 && lane < 17) dst.R[lane - 8] = src.R[lane - 8];
  if (lane == 17) {
    dst.fx = src.fx; dst.fy = src.fy; dst.u0 = src.u0; dst.v0 = src.v0;
    dst.border = src.border; dst.ulim = src.ulim; dst.vlim = src.vlim;
    dst.min_dpt = src.min_dpt; dst.avg_dpt = src.avg_dpt; dst.huber_delta = src.huber_delta;
  }
  if (lane == 18) {
    dst.img0 = src.img0; dst.img1 = src.img1; dst.dpt0 = src.dpt0; dst.valid0 = src.valid0;
    dst.jac = src.jac; dst.grad1 = src.grad1; dst.ray_tab = src.ray_tab;
    dst.dpt_out = src.dpt_out; dst.dpt_out_pitch = src.dpt_out_pitch;
  }
  if (lane == 19) {
    dst.img0_pitch = src.img0_pitch; dst.img1_pitch = src.img1_pitch; dst.dpt0_pitch = src.dpt0_pitch;
    dst.valid0_pitch = src.valid0_pitch; dst.jac_pitch = src.jac_pitch; dst.grad1_pitch = src.grad1_pitch;
  }
  if (lane == 20) {
    dst.width = src.width; dst.height = src.height; dst.num_pixels = src.num_pixels;
    dst.tile_begin = src.tile_begin; dst.num_tiles = src.num_tiles; dst.perm_mul = src.perm_mul;
    dst.flags = src.flags;
    dst.mag_tiles = src.mag_tiles;
    dst.mag_width = src.mag_width;
    dst.slot = src.partial_begin + (uint32_t)cta - src.first_cta;
  }
}

// fused depth decode: the item's latent code -> shared memory (callers sync afterwards)
template <int MAXCODE>
__device__ __forceinline__ void load_code(SfmItem<MAXCODE>& dst, const SfmItemDev& src, int code_size, int tid, int nthreads)
{
  if (src.flags & ITEM_FLAG_FUSED_DEPTH)
    for (int k = tid; k < code_size; k += nthreads) dst.code[k] = __ldg(src.code + k);
}

// a / b and a % b through the precomputed mag = floor(2^32 / b): multiply-high, one correction step
__device__ __forceinline__ uint32_t div_magic(uint32_t a, uint32_t b, uint32_t mag, uint32_t& rem)
{
  uint32_t q = __umulhi(a, mag);
  uint32_t r = a - q * b;
  if (r >= b) {
    ++q;
    r -= b;
  }
  rem = r;
  return q;
}

// CTA c owns the global tiles [c*T/G, (c+1)*T/G): static, so results are bitwise reproducible
__device__ __forceinline__ void cta_tiles(int num_tiles, int& g_lo, int& g_hi)
{
  g_lo = (int)(((long long)blockIdx.x * num_tiles) / gridDim.x);
  g_hi = (int)(((long long)(blockIdx.x + 1) * num_tiles) / gridDim.x);
}

// first pixel p0 and pixel count n of global tile g of item I (an SfmItemDev or its shared-memory copy)
template <int TILE, class ItemT>
__device__ __forceinline__ uint32_t tile_origin(const ItemT& I, int g, uint32_t& n)
{
  uint32_t tau;
  div_magic(((uint32_t)g - I.tile_begin) * I.perm_mul, I.num_tiles, I.mag_tiles, tau);  // host: k * perm_mul < 2^32
  const uint32_t p0 = tau * TILE;
  n = min((uint32_t)TILE, I.num_pixels - p0);
  return p0;
}

// normalised ray (xn, yn) of pixel (x, y) from the item's table (a kernel may issue these loads early to hide them)
template <int MAXCODE>
__device__ __forceinline__ float2 table_ray(const SfmItem<MAXCODE>& I, uint32_t x, uint32_t y)
{
  return make_float2(__ldg(I.ray_tab + x), __ldg(I.ray_tab + I.width + y));
}

// The per-pixel row of the reduced system for pixel (x, y) with ray = table_ray(I, x, y), depth d and img0 value i0:
// exact-order validity chain; for a valid pixel valid0 = 1 and feat = w * [e | a0..a5 | diff].  Returns the validity;
// feat is left alone for an invalid pixel.  It is the two halves below: pixel_warp, which needs no gather, and
// valid_pixel_row; a kernel may run them apart, to issue loads that depend on the validity before the gathers.
template <int MAXCODE>
__device__ __forceinline__ Warped pixel_warp(const SfmItem<MAXCODE>& I, float2 ray, float d)
{
  return warp_ray(ray.x, ray.y, d, I.q, I.t, I.fx, I.fy, I.u0, I.v0, I.border, I.ulim, I.vlim, I.min_dpt);
}

// the row of a pixel whose warp w = pixel_warp(I, ray, d) is valid
template <int MAXCODE>
__device__ __forceinline__ void valid_pixel_row(const SfmItem<MAXCODE>& I, uint32_t x, uint32_t y, const Warped& w,
                                                float d, float i0, bool grad_aligned8, float (&feat)[8])
{
  I.valid0[(size_t)y * I.valid0_pitch + x] = 1.0f;  // dense_sfm.h:161
  int ix, iy;
  float fu, fv, gx, gy;
  bilin_setup(w.u, w.v, ix, iy, fu, fv);
#ifdef DFK_EXP_NOGATHER  // experiment (wrong results): sample at the pixel itself -> coalesced taps
  ix = (int)x < (int)I.width - 1 ? (int)x : (int)I.width - 2;
  iy = (int)y < (int)I.height - 1 ? (int)y : (int)I.height - 2;
#endif
  sample_grad(I.grad1, I.grad1_pitch, grad_aligned8, ix, iy, fu, fv, gx, gy);
  const float i1 = sample_scalar(I.img1, I.img1_pitch, ix, iy, fu, fv);
  float a[6], c00, c02, c11, c12;
  pose_jacobian_row(w, I.fx, I.fy, gx, gy, a, c00, c02, c11, c12);
  const float e = prx_jacobian(w, I.R, d, I.avg_dpt, gx, gy, c00, c02, c11, c12);
  const float diff = i0 - i1;
  const float hw = huber_weight(diff, I.huber_delta);
  feat[0] = hw * e;
#pragma unroll
  for (int f = 0; f < 6; ++f) feat[1 + f] = hw * a[f];
  feat[7] = hw * diff;
}

template <int MAXCODE>
__device__ __forceinline__ bool pixel_row(const SfmItem<MAXCODE>& I, uint32_t x, uint32_t y, float2 ray, float d,
                                          float i0, bool grad_aligned8, float (&feat)[8])
{
  const Warped w = pixel_warp(I, ray, d);
  if (!w.valid) return false;
  valid_pixel_row(I, x, y, w, d, i0, grad_aligned8, feat);
  return true;
}

// fused depth decode from a staged code-Jacobian row: the arithmetic of update_depth_kernel's vector body (dfk_geom.cuh)
template <int C>
__device__ __forceinline__ float staged_depth(const float* row, const float* code, float prx, float avg_dpt)
{
  const float4* r4 = reinterpret_cast<const float4*>(row);
  const float4* c4 = reinterpret_cast<const float4*>(code);
  float part[C / 4];
#pragma unroll
  for (int k4 = 0; k4 < C / 4; ++k4) part[k4] = chunk_dot(r4[k4], c4[k4]);
  return prx_to_depth(__fadd_rn(prx, butterfly_sum<C / 4>(part)), avg_dpt);
}

// ====================================================================== CUDA-core pipeline (fp32 and wide kernels)

struct TileMeta {
  int nvalid;
  int item_changed;  // 1 if this tile starts a new item for this CTA
  int slot;          // partial slot of the tile's item
  int pad;
};

// TILE pixels per tile, one front-end thread each; a ring of STAGES tile stages; M double-buffered
template <int C, int TILE, int STAGES>
struct CoreSmem {
  alignas(128) float jc[STAGES][TILE * C];
  alignas(16) float M[2][TILE * SfmCfg<C>::NFP];  // layout: the kernel's
  alignas(16) float img0[STAGES][TILE];
  alignas(16) float dpt0[STAGES][TILE];
  alignas(8) uint64_t full_tma[STAGES];
  uint64_t m_full[2];
  uint64_t m_empty[2];
  TileMeta meta[2];
  SfmItem<C> item;
  int cnt[TILE / 32];  // valid counts per front-end warp

  // one thread, before the CTA's first barrier
  __device__ void init_barriers(uint32_t gram_warps)
  {
    for (int s = 0; s < STAGES; ++s) mbar_init(&full_tma[s], 1);
    for (int b = 0; b < 2; ++b) {
      mbar_init(&m_full[b], TILE / 32);  // one arrival per front-end warp (every arrival wakes the waiters)
      mbar_init(&m_empty[b], gram_warps);
    }
    mbar_fence_init();
  }
};

// Issue the bulk copies of global tile g (item `it`) into ring stage `st`.  One thread.
template <int C, int TILE, int STAGES>
__device__ __forceinline__ void issue_tile_loads(CoreSmem<C, TILE, STAGES>& sm, const SfmItemDev* __restrict__ items,
                                                 int it, int g, int st)
{
  const SfmItemDev& I = items[it];
  uint32_t n;
  const uint32_t p0 = tile_origin<TILE>(I, g, n);
  const uint32_t W = I.width;
  uint32_t y = p0 / W;
  uint32_t x = p0 - y * W;
  mbar_arrive_expect_tx(&sm.full_tma[st], n * (C + 2) * 4u);
  uint32_t slot = 0;
  while (slot < n) {
    const uint32_t seg = min(W - x, n - slot);
    bulk_g2s(&sm.jc[st][slot * C], I.jac + (size_t)y * I.jac_pitch + (size_t)x * C, seg * C * 4u, &sm.full_tma[st]);
    bulk_g2s(&sm.img0[st][slot], I.img0 + (size_t)y * I.img0_pitch + x, seg * 4u, &sm.full_tma[st]);
    bulk_g2s(&sm.dpt0[st][slot], I.dpt0 + (size_t)y * I.dpt0_pitch + x, seg * 4u, &sm.full_tma[st]);
    slot += seg;
    x = 0;
    ++y;
  }
}

// cooperative (non-TMA) staging by the TILE front-end threads for items whose buffers are not 16-byte friendly
template <int C, int TILE, int STAGES>
__device__ __forceinline__ void coop_tile_loads(CoreSmem<C, TILE, STAGES>& sm, uint32_t p0, uint32_t n, int st, int tid)
{
  const SfmItem<C>& I = sm.item;
  const uint32_t W = I.width;
  for (uint32_t s = tid; s < n; s += TILE) {
    const uint32_t p = p0 + s;
    const uint32_t y = p / W, x = p - y * W;
    sm.img0[st][s] = __ldg(I.img0 + (size_t)y * I.img0_pitch + x);
    sm.dpt0[st][s] = __ldg(I.dpt0 + (size_t)y * I.dpt0_pitch + x);
  }
  for (uint32_t e = tid; e < n * C; e += TILE) {
    const uint32_t s = e / C, kk = e - s * C;
    const uint32_t p = p0 + s;
    const uint32_t y = p / W, x = p - y * W;
    sm.jc[st][e] = __ldg(I.jac + (size_t)y * I.jac_pitch + (size_t)x * C + kk);
  }
}

// Front-end role (threads 0 .. TILE-1) over the CTA's tiles [g_lo, g_hi).  Per tile: stage it, run the per-pixel row,
// then write_row(M, jc_row, feat, ok, row, nvalid) puts the pixel into M[buf] -- the tile's valid pixels take rows
// 0 .. nvalid-1 in pixel order, the invalid ones the rows after them -- and the tile is published to the Gram role.
template <int C, int TILE, int STAGES, class WriteRow>
__device__ __forceinline__ void frontend_role(CoreSmem<C, TILE, STAGES>& sm, const SfmItemDev* __restrict__ items,
                                              int num_items, int g_lo, int g_hi, WriteRow write_row)
{
  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  // item cursors: `it` for the tile being processed, `it_pf` for the prefetcher
  int it = 0;
  while (it + 1 < num_items && (uint32_t)g_lo >= items[it].tile_begin + items[it].num_tiles) ++it;
  int it_pf = it;
  uint32_t tma_phase_bits = 0;  // bit s = parity to wait for on stage s
  int cur_item = -1;

  // prologue: prefetch the first STAGES tiles
  if (tid == 0) {
    for (int j = 0; j < STAGES && g_lo + j < g_hi; ++j) {
      const int g = g_lo + j;
      while ((uint32_t)g >= items[it_pf].tile_begin + items[it_pf].num_tiles) ++it_pf;
      if (items[it_pf].flags & ITEM_FLAG_BULK) issue_tile_loads(sm, items, it_pf, g, j);
    }
  }

  for (int g = g_lo, i = 0; g < g_hi; ++g, ++i) {
    const int st = i % STAGES;
    const int buf = i & 1;
    while ((uint32_t)g >= items[it].tile_begin + items[it].num_tiles) ++it;
    const bool changed = (it != cur_item);
    if (changed) {
      named_bar_sync(1, TILE);  // everyone finished reading the previous item's params
      load_item(sm.item, items[it], tid, (int)blockIdx.x);
      load_code(sm.item, items[it], C, tid, TILE);
      cur_item = it;
      named_bar_sync(1, TILE);
    }
    const SfmItem<C>& I = sm.item;
    uint32_t n;
    const uint32_t p0 = tile_origin<TILE>(I, g, n);
    if (I.flags & ITEM_FLAG_BULK) {
      mbar_wait(&sm.full_tma[st], (tma_phase_bits >> st) & 1u);
      tma_phase_bits ^= (1u << st);
    } else {
      coop_tile_loads(sm, p0, n, st, tid);
      named_bar_sync(1, TILE);
    }

    float feat[8];  // s = w*e, w*a[0..5], w*diff
    bool ok = false;
    const uint32_t s = tid;
    if (s < n) {
      const uint32_t p = p0 + s;
      const uint32_t y = p / I.width, x = p - y * I.width;
      float d = sm.dpt0[st][s];
      if (I.flags & ITEM_FLAG_FUSED_DEPTH) {
        // the stage holds prx_orig: decode the depth and publish it
        d = staged_depth<C>(&sm.jc[st][s * C], I.code, d, I.avg_dpt);
        I.dpt_out[(size_t)y * I.dpt_out_pitch + x] = d;
      }
      ok = pixel_row(I, x, y, table_ray(I, x, y), d, sm.img0[st][s], (I.flags & ITEM_FLAG_GRAD_ALIGNED) != 0, feat);
    }

    // ---- compaction: valid pixels first ------------------------------------------------------------------------
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    const int before = __popc(bal & ((1u << lane) - 1u));  // valid lanes below this one
    if (lane == 0) sm.cnt[warp] = __popc(bal);
    // the M buffer we are about to overwrite must have been drained by the Gram role (tile i-2)
    mbar_wait(&sm.m_empty[buf], ((i >> 1) & 1u) ^ 1u);
    named_bar_sync(1, TILE);
    int nvalid = 0, base_valid = 0;
#pragma unroll
    for (int w2 = 0; w2 < TILE / 32; ++w2) {
      if (w2 == warp) base_valid = nvalid;
      nvalid += sm.cnt[w2];
    }
    const int row = ok ? base_valid + before : nvalid + (32 * warp - base_valid) + (lane - before);
    write_row(sm.M[buf], &sm.jc[st][s * C], feat, ok, row, nvalid);
    if (tid == 0) {
      sm.meta[buf].nvalid = nvalid;
      sm.meta[buf].item_changed = changed ? 1 : 0;
      sm.meta[buf].slot = (int)I.slot;
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.m_full[buf]);  // release: M tile + meta visible to the Gram role
    named_bar_sync(1, TILE);                      // all front-end threads are done with ring stage `st`
    if (tid == 0) {
      const int gn = g + STAGES;
      if (gn < g_hi) {
        while ((uint32_t)gn >= items[it_pf].tile_begin + items[it_pf].num_tiles) ++it_pf;
        if (items[it_pf].flags & ITEM_FLAG_BULK) issue_tile_loads(sm, items, it_pf, gn, st);
      }
    }
  }
}

// Gram-role scaffold over the CTA's tiles [g_lo, g_hi), run by every Gram warp: wait for M[buf], flush(slot, inliers)
// the item the CTA leaves, accumulate(M, nvalid) the tile, hand M[buf] back to the front-end.
template <class SmemT, class Accumulate, class Flush>
__device__ __forceinline__ void gram_role(SmemT& sm, int g_lo, int g_hi, Accumulate accumulate, Flush flush)
{
  const int lane = threadIdx.x & 31;
  unsigned int inliers = 0;
  int cur_slot = -1;
  for (int g = g_lo, i = 0; g < g_hi; ++g, ++i) {
    const int buf = i & 1;
    mbar_wait(&sm.m_full[buf], (i >> 1) & 1u);
    const TileMeta meta = sm.meta[buf];
    if (meta.item_changed) {
      if (cur_slot >= 0) {
        flush(cur_slot, inliers);
        inliers = 0;
      }
      cur_slot = meta.slot;
    }
    inliers += (unsigned)meta.nvalid;
    accumulate(sm.M[buf], meta.nvalid);
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.m_empty[buf]);
  }
  if (cur_slot >= 0) flush(cur_slot, inliers);
}

}  // namespace dfk
