// dfk_match.cu -- the matching step of a ReprojectionFactor (reprojection_factor.cpp:56-65) for a batch of factors:
// brute-force Hamming matching, eight-point RANSAC (dfk_match_model.h) and distance pruning.  Every kernel takes the
// whole batch in one launch; nothing uses atomics, so every result is deterministic.  This file is compiled without
// FMA contraction so that the fp64 model rounds as the host build of dfk_match_model.h does.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_internal.h"
#include "dfk_match_model.h"

namespace dfk {
namespace {

constexpr int kMatchThreads = 128;  // queries per CTA of the matcher
constexpr int kMatchTile = 128;     // train descriptors per shared-memory tile
constexpr int kHypWarps = 4;        // the hypothesis kernel: 4 warps score kMatchHyp hypotheses
constexpr int kCompactThreads = 512;

template <int W>  // 32-bit words per descriptor: 8 (ORB, 32 bytes) or 16 (BRISK, 64 bytes)
__device__ __forceinline__ void match_body(const MatchItemDev& it, uint32_t* tile, int2* out)
{
  const int q = blockIdx.x * kMatchThreads + threadIdx.x;
  const bool active = q < it.n0;
  uint32_t qd[W];
  if (active) {
    const uint4* src = reinterpret_cast<const uint4*>(it.d0 + (size_t)q * (4 * W));
#pragma unroll
    for (int k = 0; k < W / 4; ++k) {
      const uint4 v = __ldg(src + k);
      qd[4 * k] = v.x; qd[4 * k + 1] = v.y; qd[4 * k + 2] = v.z; qd[4 * k + 3] = v.w;
    }
  }
  int best = 0x7fffffff, best_j = -1;
  for (int j0 = 0; j0 < it.n1; j0 += kMatchTile) {
    const int m = min(kMatchTile, it.n1 - j0);
    const uint4* src = reinterpret_cast<const uint4*>(it.d1 + (size_t)j0 * (4 * W));
    for (int k = threadIdx.x; k < m * (W / 4); k += kMatchThreads) reinterpret_cast<uint4*>(tile)[k] = __ldg(src + k);
    __syncthreads();
    if (active) {
      for (int jj = 0; jj < m; ++jj) {
        const uint4* td = reinterpret_cast<const uint4*>(tile + jj * W);
        int d = 0;
#pragma unroll
        for (int k = 0; k < W / 4; ++k) {
          const uint4 v = td[k];
          d += __popc(qd[4 * k] ^ v.x) + __popc(qd[4 * k + 1] ^ v.y) + __popc(qd[4 * k + 2] ^ v.z) +
               __popc(qd[4 * k + 3] ^ v.w);
        }
        if (d < best) {  // strict: ties keep the lowest train index
          best = d;
          best_j = j0 + jj;
        }
      }
    }
    __syncthreads();
  }
  if (active) out[it.out_begin + q] = best_j < 0 ? make_int2(-1, -1) : make_int2(best_j, best);
}

// one CTA per (128 queries, item): out[out_begin + q] = (argmin_j popcount(d0[q] ^ d1[j]), distance)
__global__ void __launch_bounds__(kMatchThreads) hamming_match_kernel(const MatchItemDev* __restrict__ items,
                                                                      int2* __restrict__ out)
{
  __shared__ __align__(16) uint32_t tile[kMatchTile * 16];
  const MatchItemDev it = items[blockIdx.y];
  if ((int)blockIdx.x * kMatchThreads >= it.n0) return;
  if (it.words == 8) match_body<8>(it, tile, out);
  else match_body<16>(it, tile, out);
}

// hypothesis h's model from the item's match list (int2 rows: train index, distance)
__device__ __forceinline__ int hypothesis_model(const MatchItemDev& it, const int2* m, int h, double R[9], double t[3])
{
  return dfk_mm_hypothesis(it.seed, h, it.n0, it.kp0, it.kp1, reinterpret_cast<const int32_t*>(m), 2, it.fx, it.fy,
                           it.u0, it.v0, R, t);
}

// One CTA per (kMatchHyp hypotheses, item): lane h of warp 0 builds hypothesis h's model, then the four warps score every
// match under every model; lane h of each warp counts hypothesis h's inliers among that warp's matches, and the four
// warp counts are added in warp order.  counts[hyp_begin + h] = inliers of hypothesis h (0 for an invalid one).
__global__ void __launch_bounds__(kHypWarps * 32) ransac_hypotheses_kernel(const MatchItemDev* __restrict__ items,
                                                                          const int2* __restrict__ matches,
                                                                          int* __restrict__ counts)
{
  __shared__ double sm_model[kMatchHyp][12];
  __shared__ int sm_valid[kMatchHyp];
  __shared__ int sm_count[kHypWarps][kMatchHyp];
  const MatchItemDev it = items[blockIdx.y];
  const int h0 = blockIdx.x * kMatchHyp;
  if (it.n0 < DFK_MM_SAMPLE || it.n1 == 0 || h0 >= it.max_iterations) return;
  const int2* m = matches + it.out_begin;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp == 0) {
    const int h = h0 + lane;
    double R[9], t[3];
    const int valid = h < it.max_iterations ? hypothesis_model(it, m, h, R, t) : 0;
    sm_valid[lane] = valid;
    if (valid) {
      for (int k = 0; k < 9; ++k) sm_model[lane][k] = R[k];
      for (int k = 0; k < 3; ++k) sm_model[lane][9 + k] = t[k];
    }
  }
  __syncthreads();
  int mine = 0;  // lane h: inliers of hypothesis h0 + h among this warp's matches
  for (int base = warp * 32; base < it.n0; base += kHypWarps * 32) {
    const int q = base + lane;
    double f0[3], f1[3];
    if (q < it.n0) {
      const int j = m[q].x;
      dfk_mm_bearing(it.kp0[2 * q], it.kp0[2 * q + 1], it.fx, it.fy, it.u0, it.v0, f0);
      dfk_mm_bearing(it.kp1[2 * j], it.kp1[2 * j + 1], it.fx, it.fy, it.u0, it.v0, f1);
    }
    for (int hh = 0; hh < kMatchHyp; ++hh) {
      bool inl = false;
      if (sm_valid[hh] && q < it.n0) inl = dfk_mm_score(sm_model[hh], sm_model[hh] + 9, f0, f1) < it.threshold;
      const unsigned b = __ballot_sync(0xffffffffu, inl);
      if (lane == hh) mine += __popc(b);
    }
  }
  sm_count[warp][lane] = mine;
  __syncthreads();
  if (warp == 0 && h0 + lane < it.max_iterations) {
    int c = 0;
    for (int w = 0; w < kHypWarps; ++w) c += sm_count[w][lane];
    counts[it.hyp_begin + h0 + lane] = c;
  }
}

// One warp per item: the sequential loop of the adaptive RANSAC over the per-hypothesis counts, 32 hypotheses at a
// time.  A hypothesis replaces the best only with strictly more inliers; after it, the loop stops at the first h with
// h + 1 >= dfk_mm_needed(best); the bound is evaluated at every h from the running best, which only changes at a
// replacement, so it is the sequential loop's value.  select[i] = (best hypothesis or -1, its inliers, evaluated).
__global__ void __launch_bounds__(128) ransac_select_kernel(const MatchItemDev* __restrict__ items, int n,
                                                            const int* __restrict__ counts, int3* __restrict__ select)
{
  const int i = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= n) return;
  const MatchItemDev it = items[i];
  int best = 0, best_h = -1, evaluated = 0;
  if (it.n0 >= DFK_MM_SAMPLE && it.n1 > 0) {
    for (int h0 = 0; h0 < it.max_iterations; h0 += 32) {
      const int h = h0 + lane;
      const bool in = h < it.max_iterations;
      const int c = in ? counts[it.hyp_begin + h] : 0;
      int run = c;  // inclusive prefix maximum over the chunk
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, run, o);
        if (lane >= o) run = max(run, v);
      }
      int prev = __shfl_up_sync(0xffffffffu, run, 1);
      prev = lane == 0 ? best : max(prev, best);  // the best before h
      const int cur = max(prev, c);               // the best after h
      const bool replace = in && c > prev;
      const bool stop = in && cur > 0 && (double)(h + 1) >= dfk_mm_needed(cur, it.n0, it.probability);
      const unsigned sb = __ballot_sync(0xffffffffu, stop || (in && h + 1 == it.max_iterations));
      const int last = sb ? __ffs(sb) - 1 : 31;  // the last hypothesis of this chunk the loop evaluates
      const unsigned rb = __ballot_sync(0xffffffffu, replace) & ((2u << last) - 1u);  // lanes <= last (2u << 31 wraps to 0)
      if (rb) {
        const int r = 31 - __clz(rb);
        best_h = h0 + r;
        best = __shfl_sync(0xffffffffu, cur, r);
      }
      evaluated = h0 + last + 1;
      if (sb) break;
    }
  }
  if (lane == 0) select[i] = make_int3(best_h, best, evaluated);
}

// One CTA per item: the inliers of the selected hypothesis with distance <= max_dist, sorted by (distance, query):
// key = distance << 16 | query is unique, and an entry's place is the number of smaller keys.
__global__ void __launch_bounds__(kCompactThreads) compact_matches_kernel(const MatchItemDev* __restrict__ items,
                                                                         const int2* __restrict__ matches,
                                                                         const int3* __restrict__ select,
                                                                         int3* __restrict__ out, int* __restrict__ num_out)
{
  __shared__ uint32_t keys[kMatchMaxQueries];
  __shared__ double sm_model[12];
  __shared__ int sm_valid;
  const MatchItemDev it = items[blockIdx.x];
  const int3 sel = select[blockIdx.x];
  const int2* m = matches + it.out_begin;
  if (threadIdx.x == 0) {
    double R[9], t[3];
    const int valid = sel.x >= 0 ? hypothesis_model(it, m, sel.x, R, t) : 0;
    sm_valid = valid;
    for (int k = 0; k < 9; ++k) sm_model[k] = valid ? R[k] : 0.0;
    for (int k = 0; k < 3; ++k) sm_model[9 + k] = valid ? t[k] : 0.0;
  }
  __syncthreads();
  if (!sm_valid) {
    if (threadIdx.x == 0) num_out[blockIdx.x] = 0;
    return;
  }
  for (int q = threadIdx.x; q < it.n0; q += kCompactThreads) {
    const int2 mq = m[q];
    double f0[3], f1[3];
    dfk_mm_bearing(it.kp0[2 * q], it.kp0[2 * q + 1], it.fx, it.fy, it.u0, it.v0, f0);
    dfk_mm_bearing(it.kp1[2 * mq.x], it.kp1[2 * mq.x + 1], it.fx, it.fy, it.u0, it.v0, f1);
    const bool keep = dfk_mm_score(sm_model, sm_model + 9, f0, f1) < it.threshold && (float)mq.y <= it.max_dist;
    keys[q] = keep ? ((uint32_t)mq.y << 16 | (uint32_t)q) : 0xffffffffu;
  }
  __syncthreads();
  for (int q = threadIdx.x; q < it.n0; q += kCompactThreads) {
    const uint32_t k = keys[q];
    if (k == 0xffffffffu) continue;
    int rank = 0;
    for (int j = 0; j < it.n0; ++j) rank += keys[j] < k;
    out[it.out_begin + rank] = make_int3(q, m[q].x, (int)(k >> 16));
  }
  // the number kept, summed in a fixed order
  __shared__ int sm_kept[kCompactThreads / 32];
  int c = 0;
  for (int q = threadIdx.x; q < it.n0; q += kCompactThreads) c += keys[q] != 0xffffffffu;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) sm_kept[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < kCompactThreads / 32; ++w) s += sm_kept[w];
    num_out[blockIdx.x] = s;
  }
}

}  // namespace

cudaError_t launch_hamming_match(const MatchItemDev* items_dev, int n, int max_n0, int2* matches_dev, cudaStream_t s)
{
  if (max_n0 > 0) {
    dim3 grid((unsigned)((max_n0 + kMatchThreads - 1) / kMatchThreads), (unsigned)n);
    hamming_match_kernel<<<grid, kMatchThreads, 0, s>>>(items_dev, matches_dev);
  }
  return cudaGetLastError();
}

cudaError_t launch_reprojection_match(const MatchItemDev* items_dev, int n, int max_n0, int max_iterations,
                                      int2* matches_dev, int* counts_dev, int3* select_dev, int3* out_dev,
                                      int* num_out_dev, cudaStream_t s)
{
  cudaError_t e = launch_hamming_match(items_dev, n, max_n0, matches_dev, s);
  if (e != cudaSuccess) return e;
  dim3 grid((unsigned)((max_iterations + kMatchHyp - 1) / kMatchHyp), (unsigned)n);
  ransac_hypotheses_kernel<<<grid, kHypWarps * 32, 0, s>>>(items_dev, matches_dev, counts_dev);
  ransac_select_kernel<<<(unsigned)((n + 3) / 4), 128, 0, s>>>(items_dev, n, counts_dev, select_dev);
  compact_matches_kernel<<<(unsigned)n, kCompactThreads, 0, s>>>(items_dev, matches_dev, select_dev, out_dev,
                                                                 num_out_dev);
  return cudaGetLastError();
}

}  // namespace dfk
