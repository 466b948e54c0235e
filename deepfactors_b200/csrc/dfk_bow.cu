// dfk_bow.cu -- DBoW2 retrieval on the device (include/dfk.h dfk_bow_*, DESIGN.md section 4.11): the vocabulary
// descent, the bag-of-words vector, the database query and the score.  The arithmetic is dfk_bow_model.h, built with
// -fmad=false as the sequential CPU build of the specification is; every sum runs in the order the specification gives.
#include <cuda_runtime.h>
#include <stdint.h>

#include <climits>

#include "dfk_bow_model.h"
#include "dfk_internal.h"

namespace dfk {
namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kDescendWarps = 8;   // descriptors per CTA of the descent
constexpr int kAssembleThreads = 256;
constexpr int kQueryWarps = 8;     // entries per CTA of the sums
constexpr int kRankThreads = 256;  // entries per CTA of the ranks
constexpr int kScoreWarps = 8;

__device__ __forceinline__ int vec_count(const int32_t* count, int capacity)
{
  const int c = *count;
  return c < 0 ? 0 : (c > capacity ? capacity : c);
}

// the first position of words[0, n) that is >= w (the words ascending)
__device__ __forceinline__ int lower_bound(const int32_t* words, int n, int32_t w)
{
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (words[mid] < w) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// One warp per descriptor: lane c holds the distance to child c, a shuffle argmin over (distance, child) picks the
// next node (strict < in children order: the smallest child index wins a tie).  Q = descriptor_bytes / 16.
template <int Q>
__global__ void __launch_bounds__(kDescendWarps * 32) bow_descend_kernel(BowVocDev v, const BowItemDev* items,
                                                                          int32_t* feature_words)
{
  const BowItemDev it = items[blockIdx.y];
  const int f = blockIdx.x * kDescendWarps + (threadIdx.x >> 5);
  if (f >= it.num) return;
  const int lane = threadIdx.x & 31;
  uint4 q[Q];
  const uint4* src = reinterpret_cast<const uint4*>(it.descriptors) + (size_t)f * Q;
#pragma unroll
  for (int j = 0; j < Q; ++j) q[j] = src[j];
  int node = 0;
  int2 ch = v.child[0];
  for (int depth = 0; depth < DFK_BOW_MODEL_MAX_DEPTH && ch.y > 0; ++depth) {
    unsigned key = UINT_MAX;
    if (lane < ch.y) {
      const uint4* r = v.desc + (size_t)(ch.x + lane) * Q;
      int d = 0;
#pragma unroll
      for (int j = 0; j < Q; ++j) {
        const uint4 a = r[j];
        d += dfk_bow_popc(a.x ^ q[j].x) + dfk_bow_popc(a.y ^ q[j].y) + dfk_bow_popc(a.z ^ q[j].z) +
             dfk_bow_popc(a.w ^ q[j].w);
      }
      key = ((unsigned)d << 5) | (unsigned)lane;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) key = min(key, __shfl_xor_sync(kFull, key, o));
    node = ch.x + (int)(key & 31u);
    ch = v.child[node];
  }
  if (lane == 0) {
    const int w = v.word[node];
    feature_words[it.out_begin + f] = v.word_weight[w] > 0.0 ? w : -1;
  }
}

// One CTA per item: sort the kept words (bitonic, in shared memory), run-length them, then the values (w added count
// times) and the L1 norm as one serial chain in word order.  Shared memory: keys [P] | run starts [P + 1], P the power
// of two >= the item's descriptor count.
__global__ void __launch_bounds__(kAssembleThreads) bow_assemble_kernel(const BowItemDev* items,
                                                                         const int32_t* feature_words,
                                                                         const double* word_weight, int32_t* words_out,
                                                                         double* values_out, int32_t* counts)
{
  extern __shared__ int bow_sm[];
  __shared__ int warp_runs[kAssembleThreads / 32];
  __shared__ double norm_sm;
  const BowItemDev it = items[blockIdx.x];
  const int m = it.num, tid = threadIdx.x;
  int P = 1;
  while (P < m) P <<= 1;
  int* keys = bow_sm;
  int* st = bow_sm + P;
  const int32_t* fw = feature_words + it.out_begin;
  for (int j = tid; j < P; j += kAssembleThreads) keys[j] = (j < m && fw[j] >= 0) ? fw[j] : INT_MAX;
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int i = tid; i < P; i += kAssembleThreads) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const int a = keys[i], b = keys[ixj];
          if ((a > b) == ((i & k) == 0)) {
            keys[i] = b;
            keys[ixj] = a;
          }
        }
      }
    }
  __syncthreads();
  // run starts: thread t owns the contiguous chunk [t c, (t + 1) c)
  const int c = (P + kAssembleThreads - 1) / kAssembleThreads, lo = min(tid * c, P), hi = min(lo + c, P);
  auto is_start = [&](int j) { return keys[j] != INT_MAX && (j == 0 || keys[j] != keys[j - 1]); };
  int mine = 0;
  for (int j = lo; j < hi; ++j) mine += is_start(j);
  const int lane = tid & 31, warp = tid >> 5;
  int incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(kFull, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) warp_runs[warp] = incl;
  __syncthreads();
  int before = incl - mine, runs = 0;
  for (int w = 0; w < kAssembleThreads / 32; ++w) {
    if (w < warp) before += warp_runs[w];
    runs += warp_runs[w];
  }
  for (int j = lo; j < hi; ++j) {
    if (is_start(j)) st[before++] = j;
    // the end of the kept words: st[runs]
    if (keys[j] != INT_MAX && (j + 1 == P || keys[j + 1] == INT_MAX)) st[runs] = j + 1;
  }
  if (tid == 0 && keys[0] == INT_MAX) st[0] = 0;
  __syncthreads();
  int32_t* wo = words_out + it.out_begin;
  double* vo = values_out + it.out_begin;
  for (int r = tid; r < runs; r += kAssembleThreads) {
    const int w = keys[st[r]];
    wo[r] = w;
    vo[r] = dfk_bow_repeat(word_weight[w], st[r + 1] - st[r]);
  }
  __syncthreads();
  if (tid == 0) {
    double norm = 0.0;
    for (int r = 0; r < runs; ++r) norm += fabs(vo[r]);
    norm_sm = norm;
  }
  __syncthreads();
  const double norm = norm_sm;
  if (norm > 0.0)
    for (int r = tid; r < runs; r += kAssembleThreads) vo[r] = vo[r] / norm;
  if (tid == 0) counts[blockIdx.x] = runs;
}

__global__ void bow_add_kernel(const BowAddDev* adds, int32_t* st_words, double* st_values, long long* entry_offsets,
                               int32_t* entry_counts)
{
  const BowAddDev a = adds[blockIdx.x];
  const int c = vec_count(a.count, a.capacity);
  for (int j = threadIdx.x; j < c; j += blockDim.x) {
    st_words[a.offset + j] = a.words[j];
    st_values[a.offset + j] = a.values[j];
  }
  if (threadIdx.x == 0) {
    entry_offsets[a.entry] = a.offset;
    entry_counts[a.entry] = c;
  }
}

// One warp per (query, entry): lanes binary-search the entry's words in the query's (shared memory), and the hit
// terms are added in word order through shuffles, the first one initialising the sum.  Shared memory: the query's
// values [cap] | words [cap].
__global__ void __launch_bounds__(kQueryWarps * 32) bow_query_sums_kernel(BowDbDev db, const BowQueryDev* queries,
                                                                           int cap, double* sums, uint8_t* hits)
{
  extern __shared__ double bow_qsm[];
  const BowQueryDev q = queries[blockIdx.y];
  double* qv = bow_qsm;
  int32_t* qw = reinterpret_cast<int32_t*>(bow_qsm + cap);
  const int qc = vec_count(q.count, q.capacity);
  for (int j = threadIdx.x; j < qc; j += blockDim.x) {
    qv[j] = q.values[j];
    qw[j] = q.words[j];
  }
  __syncthreads();
  const int e = blockIdx.x * kQueryWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (e >= db.size) return;
  bool any = false;
  double sum = 0.0;
  if (q.max_id == -1 || e < q.max_id) {
    const int ec = db.counts[e];
    const int32_t* ew = db.words + db.offsets[e];
    const double* ev = db.values + db.offsets[e];
    for (int base = 0; base < ec; base += 32) {
      const int j = base + lane;
      bool hit = false;
      double t = 0.0;
      if (j < ec) {
        const int32_t w = ew[j];
        const int p = lower_bound(qw, qc, w);
        if (p < qc && qw[p] == w) {
          hit = true;
          t = dfk_bow_l1_term(qv[p], ev[j]);
        }
      }
      unsigned mask = __ballot_sync(kFull, hit);
      while (mask) {
        const int b = __ffs(mask) - 1;
        mask &= mask - 1;
        const double tb = __shfl_sync(kFull, t, b);
        if (any) sum += tb;
        else sum = tb;
        any = true;
      }
    }
  }
  if (lane == 0) {
    const size_t k = (size_t)blockIdx.y * db.size + e;
    sums[k] = sum;
    hits[k] = any ? 1 : 0;
  }
}

// One thread per (query, entry): the entry's rank among the hits by (sum, entry id) places its row.  Every CTA counts
// the hits while it ranks; the first CTA of the query writes the count.
__global__ void __launch_bounds__(kRankThreads) bow_query_rank_kernel(int size, const BowQueryDev* queries,
                                                                      const double* sums, const uint8_t* hits,
                                                                      int32_t* ids, double* scores, int32_t* counts)
{
  __shared__ double ts[kRankThreads];
  __shared__ uint8_t th[kRankThreads];
  const BowQueryDev q = queries[blockIdx.y];
  const double* s = sums + (size_t)blockIdx.y * size;
  const uint8_t* hh = hits + (size_t)blockIdx.y * size;
  const int e = blockIdx.x * kRankThreads + threadIdx.x;
  const bool mine = e < size && hh[e];
  const double my = mine ? s[e] : 0.0;
  int rank = 0, total = 0;
  for (int t0 = 0; t0 < size; t0 += kRankThreads) {
    __syncthreads();
    const int j = t0 + threadIdx.x;
    ts[threadIdx.x] = j < size ? s[j] : 0.0;
    th[threadIdx.x] = j < size ? hh[j] : 0;
    __syncthreads();
    const int lim = min(kRankThreads, size - t0);
    for (int k = 0; k < lim; ++k)
      if (th[k]) {
        ++total;
        const double o = ts[k];
        rank += (o < my || (o == my && t0 + k < e)) ? 1 : 0;
      }
  }
  if (mine && rank < q.max_results) {
    ids[q.row_begin + rank] = e;
    scores[q.row_begin + rank] = dfk_bow_final_score(my);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) counts[blockIdx.y] = total;
}

// One warp per item: score(a = the entry's vector, b = the item's), the merge over a's words with b binary-searched.
__global__ void __launch_bounds__(kScoreWarps * 32) bow_score_kernel(BowDbDev db, const BowScoreDev* items, int n,
                                                                      double* out)
{
  const int i = blockIdx.x * kScoreWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= n) return;
  const BowScoreDev it = items[i];
  const int bc = vec_count(it.count, it.capacity);
  const int ec = db.counts[it.entry];
  const int32_t* ew = db.words + db.offsets[it.entry];
  const double* ev = db.values + db.offsets[it.entry];
  double sum = 0.0;
  for (int base = 0; base < ec; base += 32) {
    const int j = base + lane;
    bool hit = false;
    double t = 0.0;
    if (j < ec) {
      const int32_t w = ew[j];
      const int p = lower_bound(it.words, bc, w);
      if (p < bc && it.words[p] == w) {
        hit = true;
        t = dfk_bow_l1_term(ev[j], it.values[p]);
      }
    }
    unsigned mask = __ballot_sync(kFull, hit);
    while (mask) {
      const int b = __ffs(mask) - 1;
      mask &= mask - 1;
      sum += __shfl_sync(kFull, t, b);
    }
  }
  if (lane == 0) out[i] = dfk_bow_final_score(sum);
}

}  // namespace

cudaError_t launch_bow_transform(const BowVocDev& v, const BowItemDev* items_dev, int n, int max_num,
                                 int32_t* feature_words, int32_t* words_out, double* values_out, int32_t* counts,
                                 cudaStream_t s)
{
  if (max_num > 0) {
    const dim3 grid((max_num + kDescendWarps - 1) / kDescendWarps, n);
    switch (v.q) {
      case 2: bow_descend_kernel<2><<<grid, kDescendWarps * 32, 0, s>>>(v, items_dev, feature_words); break;
      case 3: bow_descend_kernel<3><<<grid, kDescendWarps * 32, 0, s>>>(v, items_dev, feature_words); break;
      case 4: bow_descend_kernel<4><<<grid, kDescendWarps * 32, 0, s>>>(v, items_dev, feature_words); break;
      default: return cudaErrorInvalidValue;
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  int P = 1;
  while (P < max_num) P <<= 1;
  const size_t smem = sizeof(int) * (2 * (size_t)P + 1);
  cudaError_t e = cudaFuncSetAttribute(bow_assemble_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  bow_assemble_kernel<<<n, kAssembleThreads, smem, s>>>(items_dev, feature_words, v.word_weight, words_out, values_out,
                                                        counts);
  return cudaGetLastError();
}

cudaError_t launch_bow_add(const BowAddDev* adds_dev, int n, int32_t* st_words, double* st_values,
                           long long* entry_offsets, int32_t* entry_counts, cudaStream_t s)
{
  bow_add_kernel<<<n, 128, 0, s>>>(adds_dev, st_words, st_values, entry_offsets, entry_counts);
  return cudaGetLastError();
}

cudaError_t launch_bow_query(const BowDbDev& db, const BowQueryDev* queries_dev, int n, int max_cap, double* sums,
                             uint8_t* hits, int32_t* ids, double* scores, int32_t* counts, cudaStream_t s)
{
  const size_t smem = (sizeof(double) + sizeof(int32_t)) * (size_t)max_cap;
  cudaError_t e = cudaFuncSetAttribute(bow_query_sums_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  bow_query_sums_kernel<<<dim3((db.size + kQueryWarps - 1) / kQueryWarps, n), kQueryWarps * 32, smem, s>>>(
      db, queries_dev, max_cap, sums, hits);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  bow_query_rank_kernel<<<dim3((db.size + kRankThreads - 1) / kRankThreads, n), kRankThreads, 0, s>>>(
      db.size, queries_dev, sums, hits, ids, scores, counts);
  return cudaGetLastError();
}

cudaError_t launch_bow_score(const BowDbDev& db, const BowScoreDev* items_dev, int n, double* out, cudaStream_t s)
{
  bow_score_kernel<<<(n + kScoreWarps - 1) / kScoreWarps, kScoreWarps * 32, 0, s>>>(db, items_dev, n, out);
  return cudaGetLastError();
}

}  // namespace dfk
