// dfk_bow_train.cu -- DBoW2 vocabulary training on the device (include/dfk.h dfk_bow_vocabulary_train, DESIGN.md
// section 4.15): hierarchical k-means++ with Hamming distance and bitwise majority means, one tree level at a time.
// Everything is integer: distances, min_dist and its sums (int64), and the majority counts (int32; shared-memory
// counters, integer atomics only where the order does not matter).  The random draws are dfk_bow_model.h's, built with
// -fmad=false like dfk_bow.cu.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk.h"
#include "dfk_bow_model.h"
#include "dfk_internal.h"

namespace dfk {
namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kThreads = 256;  // every CTA of the training kernels
constexpr int kWarps = kThreads / 32;

__device__ __forceinline__ int popc4(uint4 a, uint4 b)
{
  return __popc(a.x ^ b.x) + __popc(a.y ^ b.y) + __popc(a.z ^ b.z) + __popc(a.w ^ b.w);
}

template <int Q>
__device__ __forceinline__ int dist(const uint4 (&x)[Q], const uint4* c)
{
  int d = 0;
#pragma unroll
  for (int j = 0; j < Q; ++j) d += popc4(x[j], c[j]);
  return d;
}

template <int Q>
__device__ __forceinline__ void load(uint4 (&x)[Q], const uint4* p)
{
#pragma unroll
  for (int j = 0; j < Q; ++j) x[j] = p[j];
}

// the nearest of nc centres, strict < in cluster order
template <int Q>
__device__ __forceinline__ int nearest(const uint4 (&x)[Q], const uint4* centres, int nc)
{
  int best = 0, bd = dist<Q>(x, centres);
  for (int c = 1; c < nc; ++c) {
    const int d = dist<Q>(x, centres + (size_t)c * Q);
    if (d < bd) {
      bd = d;
      best = c;
    }
  }
  return best;
}

// sum over the CTA (every thread gets it); red [kWarps]
__device__ __forceinline__ long long block_sum(long long v, long long* red)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  long long t = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) t += red[w];
  return t;
}

// exclusive prefix over the CTA's threads in thread order; red [kWarps]
__device__ __forceinline__ long long block_excl(long long v, long long* red)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long y = __shfl_up_sync(kFull, incl, o);
    if (lane >= o) incl += y;
  }
  __syncthreads();
  if (lane == 31) red[warp] = incl;
  __syncthreads();
  long long before = incl - v;
  for (int w = 0; w < warp; ++w) before += red[w];
  return before;
}

// The first index in [0, n) whose inclusive prefix sum of md reaches t (1 <= t <= the sum of md); thread i scans the
// contiguous range [i per, (i + 1) per).  *pick is written by the one thread whose range holds it.
__device__ __forceinline__ void find_cut(const int* md, int n, long long t, long long* red, int* pick)
{
  const int per = (n + kThreads - 1) / kThreads, lo = min((int)threadIdx.x * per, n), hi = min(lo + per, n);
  long long local = 0;
  for (int i = lo; i < hi; ++i) local += md[i];
  const long long excl = block_excl(local, red);
  if (excl < t && t <= excl + local) {
    long long acc = excl;
    for (int i = lo; i < hi; ++i) {
      acc += md[i];
      if (acc >= t) {
        *pick = i;
        break;
      }
    }
  }
  __syncthreads();
}

// Stable destinations of one tile of kThreads elements (c < 0: no element): an element's destination is running[c]
// plus the tile's earlier elements of cluster c; running[c] then advances by the tile's count.  wcnt [kWarps][32] is
// zero on entry and on exit.
__device__ __forceinline__ int tile_dest(int c, int* running, int (*wcnt)[32])
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned peers = __match_any_sync(kFull, c);
  const int before = __popc(peers & ((1u << lane) - 1u));
  if (c >= 0 && before == 0) wcnt[warp][c] = __popc(peers);
  __syncthreads();
  int dst = -1;
  if (c >= 0) {
    dst = running[c] + before;
    for (int w = 0; w < warp; ++w) dst += wcnt[w][c];
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    int add = 0;
    for (int w = 0; w < kWarps; ++w) {
      add += wcnt[w][threadIdx.x];
      wcnt[w][threadIdx.x] = 0;
    }
    running[threadIdx.x] += add;
  }
  __syncthreads();
  return dst;
}

// The majority means of nc clusters from per-(cluster, bit) counts: thread b owns bit b (and b + kThreads, ...), so a
// warp owns whole 32-bit words and a ballot assembles each.  count(c, b) and members(c) are read through functors.
template <int Q, class Count, class Members>
__device__ __forceinline__ void majority(uint4* centres, int nc, Count count, Members members)
{
  uint32_t* cw = reinterpret_cast<uint32_t*>(centres);
  for (int b = threadIdx.x; b < Q * 128; b += kThreads)
    for (int c = 0; c < nc; ++c) {
      const unsigned word = __ballot_sync(kFull, count(c, b) > members(c) / 2);
      if ((b & 31) == 0) cw[(size_t)c * Q * 4 + (b >> 5)] = word;
    }
}

// ------------------------------------------------------------------------------------------ small nodes: one CTA each
// Dynamic shared memory: X [max_m, Q] uint4 | C [k, Q] uint4 | counts [k, 128 Q] int | min_dist [max_m] int |
// assignment [max_m] uint8.
template <int Q>
__global__ void __launch_bounds__(kThreads) bow_train_small_kernel(BowTrainLevel lv, const int* small_idx, int max_m)
{
  extern __shared__ uint4 tsm[];
  __shared__ long long red[kWarps], target;
  __shared__ int members[32], running[32], wcnt[kWarps][32];
  __shared__ int pick, changed;
  constexpr int BITS = Q * 128;
  const int g = small_idx[blockIdx.x], k = lv.k, tid = threadIdx.x;
  const BowTrainNode nd = lv.nodes[g];
  const int m = nd.m;
  uint4* X = tsm;
  uint4* C = X + (size_t)max_m * Q;
  int* cnt = reinterpret_cast<int*>(C + (size_t)k * Q);
  int* md = cnt + (size_t)k * BITS;
  unsigned char* asg = reinterpret_cast<unsigned char*>(md + max_m);
  const uint4* src = lv.in + (size_t)nd.begin * Q;
  for (int j = tid; j < m * Q; j += kThreads) X[j] = src[j];
  if (tid < 32) members[tid] = 0;
  for (int j = tid; j < kWarps * 32; j += kThreads) wcnt[j >> 5][j & 31] = 0;
  __syncthreads();
  int nc, rounds = 0, capped = 0;
  if (m <= k) {
    nc = m;
    for (int j = tid; j < m * Q; j += kThreads) C[j] = X[j];
    for (int i = tid; i < m; i += kThreads) asg[i] = (unsigned char)i;
    if (tid < m) members[tid] = 1;
  } else {
    // seeding (initiateClustersKMpp)
    uint64_t s = nd.key;
    if (tid == 0) pick = (int)dfk_bow_draw_index(&s, m);
    __syncthreads();
    nc = 1;
    for (int j = tid; j < Q; j += kThreads) C[j] = X[(size_t)pick * Q + j];
    __syncthreads();
    for (int i = tid; i < m; i += kThreads) {
      uint4 x[Q];
      load<Q>(x, X + (size_t)i * Q);
      md[i] = dist<Q>(x, C);
    }
    while (nc < k) {
      long long local = 0;
      const uint4* last = C + (size_t)(nc - 1) * Q;
      for (int i = tid; i < m; i += kThreads) {
        int d = md[i];
        if (d > 0) {
          uint4 x[Q];
          load<Q>(x, X + (size_t)i * Q);
          d = min(d, dist<Q>(x, last));
          md[i] = d;
        }
        local += d;
      }
      const long long sum = block_sum(local, red);
      if (sum == 0) break;
      if (tid == 0) target = dfk_bow_cut_target(dfk_bow_draw_cut(&s, sum));
      __syncthreads();
      find_cut(md, m, target, red, &pick);
      for (int j = tid; j < Q; j += kThreads) C[(size_t)nc * Q + j] = X[(size_t)pick * Q + j];
      ++nc;
      __syncthreads();
    }
    // rounds: assign, then stop or take the means
    for (int i = tid; i < m; i += kThreads) asg[i] = 0xff;
    for (;;) {
      ++rounds;
      if (tid < 32) members[tid] = 0;
      if (tid == 0) changed = 0;
      __syncthreads();
      bool ch = false;
      for (int i = tid; i < m; i += kThreads) {
        uint4 x[Q];
        load<Q>(x, X + (size_t)i * Q);
        const int c = nearest<Q>(x, C, nc);
        ch |= asg[i] != c;
        asg[i] = (unsigned char)c;
        atomicAdd(&members[c], 1);
      }
      if (ch) changed = 1;
      __syncthreads();
      if (rounds > 1 && !changed) break;
      if (rounds == DFK_BOW_TRAIN_MAX_ROUNDS) {
        capped = 1;
        break;
      }
      const uint32_t* Xw = reinterpret_cast<const uint32_t*>(X);
      for (int b = tid; b < BITS; b += kThreads) {
        for (int c = 0; c < nc; ++c) cnt[c * BITS + b] = 0;
        const int w = b >> 5, sh = b & 31;
        for (int i = 0; i < m; ++i) cnt[asg[i] * BITS + b] += (Xw[(size_t)i * Q * 4 + w] >> sh) & 1u;
      }
      __syncthreads();
      majority<Q>(C, nc, [&](int c, int b) { return cnt[c * BITS + b]; }, [&](int c) { return members[c]; });
      __syncthreads();
    }
  }
  // outputs, then the stable partition into the children
  if (tid == 0) {
    lv.nc[g] = nc;
    lv.rounds[g] = rounds;
    lv.capped[g] = capped;
  }
  for (int j = tid; j < nc * Q; j += kThreads) lv.centres[(size_t)g * k * Q + j] = C[j];
  if (tid < 32) {
    const int c = tid;
    const int mc = c < nc ? members[c] : 0;
    if (c < k) lv.sizes[(size_t)g * k + c] = c < nc ? mc : 0;
    int incl = mc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(kFull, incl, o);
      if (c >= o) incl += y;
    }
    running[c] = nd.begin + incl - mc;
  }
  __syncthreads();
  for (int base = 0; base < m; base += kThreads) {
    const int i = base + tid;
    const int dst = tile_dest(i < m ? (int)asg[i] : -1, running, wcnt);
    if (i < m)
#pragma unroll
      for (int j = 0; j < Q; ++j) lv.out[(size_t)dst * Q + j] = X[(size_t)i * Q + j];
  }
}

// ----------------------------------------------------------------------------- large nodes: kBowTrainChunk per CTA
__global__ void bow_train_seed_first_kernel(BowTrainLevel lv, BowTrainLarge lg)
{
  __shared__ int pick;
  const int j = blockIdx.x, g = lg.node[j];
  const BowTrainNode nd = lv.nodes[g];
  if (threadIdx.x == 0) {
    uint64_t s = nd.key;
    pick = (int)dfk_bow_draw_index(&s, nd.m);
    lg.rng[j] = s;
    lg.seeding[j] = 1;
    lg.active[j] = 1;
    lg.changed[j] = 0;
    lv.nc[g] = 1;
    lv.rounds[g] = 0;
    lv.capped[g] = 0;
  }
  __syncthreads();
  for (int q = threadIdx.x; q < lv.q; q += blockDim.x)
    lv.centres[(size_t)g * lv.k * lv.q + q] = lv.in[(size_t)(nd.begin + pick) * lv.q + q];
}

// min_dist against the latest centre (first: against the first centre, for every member), and its chunk sums
template <int Q>
__global__ void __launch_bounds__(kThreads) bow_train_min_dist_kernel(BowTrainLevel lv, BowTrainLarge lg, int first)
{
  __shared__ long long red[kWarps];
  const int2 ch = lg.chunk[blockIdx.x];
  if (!lg.seeding[ch.x]) return;
  const int g = lg.node[ch.x];
  const BowTrainNode nd = lv.nodes[g];
  const uint4* last = lv.centres + ((size_t)g * lv.k + lv.nc[g] - 1) * Q;
  const int end = min(ch.y + kBowTrainChunk, nd.m);
  long long local = 0;
  for (int i = ch.y + threadIdx.x; i < end; i += kThreads) {
    const int r = nd.begin + i;
    int d = first ? 1 : lg.min_dist[r];
    if (d > 0) {
      uint4 x[Q];
      load<Q>(x, lv.in + (size_t)r * Q);
      const int e = dist<Q>(x, last);
      d = first ? e : min(d, e);
      lg.min_dist[r] = d;
    }
    local += d;
  }
  const long long s = block_sum(local, red);
  if (threadIdx.x == 0) lg.chunk_sum[blockIdx.x] = s;
}

// one warp per large node: dist_sum over its chunks; stop seeding at 0, else draw the cut and find its chunk
__global__ void bow_train_draw_kernel(BowTrainLarge lg)
{
  const int j = blockIdx.x, lane = threadIdx.x;
  if (!lg.seeding[j]) return;
  const int c0 = lg.chunk_first[j], c1 = lg.chunk_first[j + 1];
  long long s = 0;
  for (int c = c0 + lane; c < c1; c += 32) s += lg.chunk_sum[c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(kFull, s, o);
  if (lane != 0) return;
  if (s == 0) {
    lg.seeding[j] = 0;
    return;
  }
  uint64_t st = lg.rng[j];
  const long long t = dfk_bow_cut_target(dfk_bow_draw_cut(&st, s));
  lg.rng[j] = st;
  long long acc = 0;
  for (int c = c0; c < c1; ++c) {
    const long long v = lg.chunk_sum[c];
    if (acc + v >= t) {
      lg.cut_chunk[j] = c;
      lg.cut_rem[j] = t - acc;
      return;
    }
    acc += v;
  }
}

// the chunk holding the cut finds its member and appends it as the next centre
__global__ void __launch_bounds__(kThreads) bow_train_pick_kernel(BowTrainLevel lv, BowTrainLarge lg)
{
  __shared__ long long red[kWarps];
  __shared__ int pick;
  const int2 ch = lg.chunk[blockIdx.x];
  if (!lg.seeding[ch.x] || lg.cut_chunk[ch.x] != (int)blockIdx.x) return;
  const int g = lg.node[ch.x];
  const BowTrainNode nd = lv.nodes[g];
  const int nc = lv.nc[g];
  find_cut(lg.min_dist + nd.begin + ch.y, min(kBowTrainChunk, nd.m - ch.y), lg.cut_rem[ch.x], red, &pick);
  const int r = nd.begin + ch.y + pick;
  for (int q = threadIdx.x; q < lv.q; q += kThreads)
    lv.centres[((size_t)g * lv.k + nc) * lv.q + q] = lv.in[(size_t)r * lv.q + q];
  __syncthreads();
  if (threadIdx.x == 0) lv.nc[g] = nc + 1;
}

// One round's assignment of a chunk, its members per cluster and its per-(cluster, bit) counts, added to the node's.
// Dynamic shared memory: C [k, Q] uint4 | X [chunk, Q] uint4 | counts [k, 128 Q] int | assignment [chunk] uint8.
template <int Q>
__global__ void __launch_bounds__(kThreads) bow_train_assign_kernel(BowTrainLevel lv, BowTrainLarge lg)
{
  extern __shared__ uint4 tsm[];
  __shared__ int members[32], changed;
  constexpr int BITS = Q * 128;
  const int2 ch = lg.chunk[blockIdx.x];
  if (!lg.active[ch.x]) return;
  const int g = lg.node[ch.x], k = lv.k, tid = threadIdx.x;
  const BowTrainNode nd = lv.nodes[g];
  const int nc = lv.nc[g], n = min(kBowTrainChunk, nd.m - ch.y), r0 = nd.begin + ch.y;
  uint4* C = tsm;
  uint4* X = C + (size_t)k * Q;
  int* cnt = reinterpret_cast<int*>(X + (size_t)kBowTrainChunk * Q);
  unsigned char* asg = reinterpret_cast<unsigned char*>(cnt + (size_t)k * BITS);
  for (int j = tid; j < nc * Q; j += kThreads) C[j] = lv.centres[(size_t)g * k * Q + j];
  for (int j = tid; j < n * Q; j += kThreads) X[j] = lv.in[(size_t)r0 * Q + j];
  if (tid < 32) members[tid] = 0;
  if (tid == 0) changed = 0;
  __syncthreads();
  bool chg = false;
  for (int i = tid; i < n; i += kThreads) {
    uint4 x[Q];
    load<Q>(x, X + (size_t)i * Q);
    const int c = nearest<Q>(x, C, nc);
    chg |= lg.assign[r0 + i] != c;
    lg.assign[r0 + i] = (unsigned char)c;
    asg[i] = (unsigned char)c;
    atomicAdd(&members[c], 1);
  }
  if (chg) changed = 1;
  __syncthreads();
  const uint32_t* Xw = reinterpret_cast<const uint32_t*>(X);
  int* bits = lg.bits + (size_t)ch.x * k * BITS;
  for (int b = tid; b < BITS; b += kThreads) {
    for (int c = 0; c < nc; ++c) cnt[c * BITS + b] = 0;
    const int w = b >> 5, sh = b & 31;
    for (int i = 0; i < n; ++i) cnt[asg[i] * BITS + b] += (Xw[(size_t)i * Q * 4 + w] >> sh) & 1u;
    for (int c = 0; c < nc; ++c)
      if (cnt[c * BITS + b]) atomicAdd(&bits[c * BITS + b], cnt[c * BITS + b]);
  }
  if (tid < nc) {
    if (members[tid]) atomicAdd(&lg.members[(size_t)ch.x * k + tid], members[tid]);
    lg.chunk_counts[(size_t)blockIdx.x * k + tid] = members[tid];
  }
  if (tid == 0 && changed) lg.changed[ch.x] = 1;
}

// One CTA per large node after its round: stop (converged, or the round cap), or take the means; clear the counts.
template <int Q>
__global__ void __launch_bounds__(kThreads) bow_train_update_kernel(BowTrainLevel lv, BowTrainLarge lg)
{
  __shared__ int stop;
  constexpr int BITS = Q * 128;
  const int j = blockIdx.x;
  if (!lg.active[j]) return;
  const int g = lg.node[j], k = lv.k, nc = lv.nc[g];
  int* bits = lg.bits + (size_t)j * k * BITS;
  int* members = lg.members + (size_t)j * k;
  if (threadIdx.x == 0) {
    const int rounds = ++lv.rounds[g];
    stop = 0;
    if (rounds > 1 && !lg.changed[j]) stop = 1;
    else if (rounds == DFK_BOW_TRAIN_MAX_ROUNDS) stop = 2;
    if (stop) lg.active[j] = 0;
    if (stop == 2) lv.capped[g] = 1;
    lg.changed[j] = 0;
  }
  __syncthreads();
  if (!stop)
    majority<Q>(lv.centres + (size_t)g * k * Q, nc, [&](int c, int b) { return bits[c * BITS + b]; },
                [&](int c) { return members[c]; });
  __syncthreads();
  for (int b = threadIdx.x; b < BITS; b += kThreads)
    for (int c = 0; c < nc; ++c) bits[c * BITS + b] = 0;
  if (threadIdx.x < nc) members[threadIdx.x] = 0;
}

// one warp per large node: group sizes, and each chunk's first output row per cluster
__global__ void bow_train_bases_kernel(BowTrainLevel lv, BowTrainLarge lg)
{
  const int j = blockIdx.x, c = threadIdx.x, g = lg.node[j], k = lv.k;
  const int nc = lv.nc[g], c0 = lg.chunk_first[j], c1 = lg.chunk_first[j + 1];
  int tot = 0;
  if (c < nc)
    for (int ch = c0; ch < c1; ++ch) tot += lg.chunk_counts[(size_t)ch * k + c];
  if (c < k) lv.sizes[(size_t)g * k + c] = tot;
  int incl = tot;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(kFull, incl, o);
    if (c >= o) incl += y;
  }
  if (c >= nc) return;
  int base = lv.nodes[g].begin + incl - tot;
  for (int ch = c0; ch < c1; ++ch) {
    lg.chunk_base[(size_t)ch * k + c] = base;
    base += lg.chunk_counts[(size_t)ch * k + c];
  }
}

// the stable partition of each chunk's members into their clusters' output rows
template <int Q>
__global__ void __launch_bounds__(kThreads) bow_train_scatter_kernel(BowTrainLevel lv, BowTrainLarge lg)
{
  __shared__ int running[32], wcnt[kWarps][32];
  const int2 ch = lg.chunk[blockIdx.x];
  const int g = lg.node[ch.x], k = lv.k, tid = threadIdx.x;
  const BowTrainNode nd = lv.nodes[g];
  const int nc = lv.nc[g], n = min(kBowTrainChunk, nd.m - ch.y), r0 = nd.begin + ch.y;
  if (tid < 32) running[tid] = tid < nc ? lg.chunk_base[(size_t)blockIdx.x * k + tid] : 0;
  for (int j = tid; j < kWarps * 32; j += kThreads) wcnt[j >> 5][j & 31] = 0;
  __syncthreads();
  for (int base = 0; base < n; base += kThreads) {
    const int i = base + tid;
    const int dst = tile_dest(i < n ? (int)lg.assign[r0 + i] : -1, running, wcnt);
    if (i < n)
#pragma unroll
      for (int j = 0; j < Q; ++j) lv.out[(size_t)dst * Q + j] = lv.in[(size_t)(r0 + i) * Q + j];
  }
}

__global__ void bow_train_place_kernel(BowTrainLevel lv, const int* row_first, uint4* tree_desc)
{
  const int g = blockIdx.x, n = lv.nc[g] * lv.q;
  const uint4* src = lv.centres + (size_t)g * lv.k * lv.q;
  uint4* dst = tree_desc + (size_t)row_first[g] * lv.q;
  for (int j = threadIdx.x; j < n; j += blockDim.x) dst[j] = src[j];
}

__global__ void bow_train_count_kernel(const BowItemDev* items, const int32_t* words_out, const int32_t* counts,
                                       int32_t* word_images)
{
  const BowItemDev it = items[blockIdx.x];
  const int c = counts[blockIdx.x];
  for (int j = threadIdx.x; j < c; j += blockDim.x) atomicAdd(&word_images[words_out[it.out_begin + j]], 1);
}

template <int Q>
size_t small_smem(int k, int max_m)
{
  return (size_t)max_m * Q * 16 + (size_t)k * Q * 16 + (size_t)k * Q * 128 * 4 + (size_t)max_m * 4 +
         (((size_t)max_m + 15) & ~(size_t)15);
}

template <int Q>
size_t assign_smem(int k)
{
  return (size_t)k * Q * 16 + (size_t)kBowTrainChunk * Q * 16 + (size_t)k * Q * 128 * 4 + kBowTrainChunk;
}

template <int Q>
cudaError_t small_q(const BowTrainLevel& lv, const int* idx, int n, int max_m, cudaStream_t s)
{
  const size_t smem = small_smem<Q>(lv.k, max_m);
  cudaError_t e = cudaFuncSetAttribute(bow_train_small_kernel<Q>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  if (e != cudaSuccess) return e;
  bow_train_small_kernel<Q><<<n, kThreads, smem, s>>>(lv, idx, max_m);
  return cudaGetLastError();
}

template <int Q>
cudaError_t seed_q(const BowTrainLevel& lv, const BowTrainLarge& lg, int nl, int chunks, cudaStream_t s)
{
  bow_train_seed_first_kernel<<<nl, 32, 0, s>>>(lv, lg);
  for (int c = 1; c < lv.k; ++c) {
    bow_train_min_dist_kernel<Q><<<chunks, kThreads, 0, s>>>(lv, lg, c == 1);
    bow_train_draw_kernel<<<nl, 32, 0, s>>>(lg);
    bow_train_pick_kernel<<<chunks, kThreads, 0, s>>>(lv, lg);
  }
  return cudaGetLastError();
}

template <int Q>
cudaError_t rounds_q(const BowTrainLevel& lv, const BowTrainLarge& lg, int nl, int chunks, int rounds,
                     cudaStream_t s)
{
  const size_t smem = assign_smem<Q>(lv.k);
  cudaError_t e = cudaFuncSetAttribute(bow_train_assign_kernel<Q>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  if (e != cudaSuccess) return e;
  for (int r = 0; r < rounds; ++r) {
    bow_train_assign_kernel<Q><<<chunks, kThreads, smem, s>>>(lv, lg);
    bow_train_update_kernel<Q><<<nl, kThreads, 0, s>>>(lv, lg);
  }
  return cudaGetLastError();
}

template <int Q>
cudaError_t partition_q(const BowTrainLevel& lv, const BowTrainLarge& lg, int nl, int chunks, cudaStream_t s)
{
  bow_train_bases_kernel<<<nl, 32, 0, s>>>(lv, lg);
  bow_train_scatter_kernel<Q><<<chunks, kThreads, 0, s>>>(lv, lg);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_bow_train_small(const BowTrainLevel& lv, const int* small_idx, int n_small, int max_m,
                                   cudaStream_t s)
{
  switch (lv.q) {
    case 2: return small_q<2>(lv, small_idx, n_small, max_m, s);
    case 3: return small_q<3>(lv, small_idx, n_small, max_m, s);
    case 4: return small_q<4>(lv, small_idx, n_small, max_m, s);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_bow_train_seed(const BowTrainLevel& lv, const BowTrainLarge& lg, int n_large, int chunks,
                                  cudaStream_t s)
{
  switch (lv.q) {
    case 2: return seed_q<2>(lv, lg, n_large, chunks, s);
    case 3: return seed_q<3>(lv, lg, n_large, chunks, s);
    case 4: return seed_q<4>(lv, lg, n_large, chunks, s);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_bow_train_rounds(const BowTrainLevel& lv, const BowTrainLarge& lg, int n_large, int chunks,
                                    int rounds, cudaStream_t s)
{
  switch (lv.q) {
    case 2: return rounds_q<2>(lv, lg, n_large, chunks, rounds, s);
    case 3: return rounds_q<3>(lv, lg, n_large, chunks, rounds, s);
    case 4: return rounds_q<4>(lv, lg, n_large, chunks, rounds, s);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_bow_train_partition(const BowTrainLevel& lv, const BowTrainLarge& lg, int n_large, int chunks,
                                       cudaStream_t s)
{
  switch (lv.q) {
    case 2: return partition_q<2>(lv, lg, n_large, chunks, s);
    case 3: return partition_q<3>(lv, lg, n_large, chunks, s);
    case 4: return partition_q<4>(lv, lg, n_large, chunks, s);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_bow_train_place(const BowTrainLevel& lv, int G, const int* row_first, uint4* tree_desc,
                                   cudaStream_t s)
{
  bow_train_place_kernel<<<G, 128, 0, s>>>(lv, row_first, tree_desc);
  return cudaGetLastError();
}

cudaError_t launch_bow_train_count(const BowItemDev* items_dev, int n, const int32_t* words_out,
                                   const int32_t* counts, int32_t* word_images, cudaStream_t s)
{
  bow_train_count_kernel<<<n, 128, 0, s>>>(items_dev, words_out, counts, word_images);
  return cudaGetLastError();
}

}  // namespace dfk
