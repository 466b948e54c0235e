// dfk_orb.cu -- cv::ORB with one pyramid level (the reference's OrbDetector, features/feature_detection.h) for a batch
// of images: FAST-9 with non-maximum suppression, the first cut by FAST score, Harris responses and orientations, the
// second cut by response and the rBRIEF descriptors.  Seven kernels take the whole batch (see launch_orb_detect).  The
// integer atomics only count (histograms); every position comes from a scan or a sort, so the output is deterministic.
// This file is compiled without FMA contraction so that the fp32 / fp64 model (dfk_orb_model.h) rounds as its host
// build does.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_internal.h"
#include "dfk_orb_model.h"
#include "dfk_orb_pattern.h"

namespace dfk {
namespace {

constexpr int kWarps = 8;             // warps per CTA of the per-segment / per-corner / per-keypoint kernels
constexpr int kScanThreads = 1024;    // the per-image kernels
constexpr int kMaxBlocksPerItem = 128;
constexpr int kReach = DFK_OM_PATTERN_R;  // the blurred image covers R widened by this

__constant__ int8_t c_pattern[DFK_ORB_PATTERN_PAIRS * 4] = {DFK_ORB_PATTERN_DATA};

__device__ __forceinline__ int warp_sum(int v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Exclusive scan of one int per thread over a CTA of kScanThreads; *total gets the sum.  smem: 33 ints.
__device__ int block_exclusive_scan(int v, int* smem, int* total)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) smem[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = smem[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    smem[lane] = w;  // inclusive over warps
  }
  __syncthreads();
  const int before = (warp ? smem[warp - 1] : 0) + x - v;
  *total = smem[31];
  __syncthreads();
  return before;
}

// 1. FAST scores of a 32 x 8 tile of R and its 1-pixel ring, non-maximum suppression, the score map, the tile rows'
// corner counts and the score histogram.  Block (32, 8), grid (tiles x, tiles y, item).
__global__ void __launch_bounds__(kOrbTileW * kOrbTileH) orb_fast_kernel(const OrbItemDev* __restrict__ items,
                                                                        OrbScratchDev s)
{
  const OrbItemDev it = items[blockIdx.z];
  if ((int)blockIdx.x >= it.tiles_x || (int)blockIdx.y >= it.tiles_y) return;
  constexpr int PW = kOrbTileW + 8, PH = kOrbTileH + 8, SW = kOrbTileW + 2, SH = kOrbTileH + 2;
  __shared__ uint8_t pix[PH][PW];
  __shared__ int score[SH][SW];
  const int tid = threadIdx.y * kOrbTileW + threadIdx.x;
  // pixels from (x0 - 4, y0 - 4): always inside the image for the ring of R, clamped past it (those scores are unused)
  const int x0 = DFK_OM_EDGE + blockIdx.x * kOrbTileW, y0 = DFK_OM_EDGE + blockIdx.y * kOrbTileH;
  const int W = it.rw + 2 * DFK_OM_EDGE, H = it.rh + 2 * DFK_OM_EDGE;
  for (int i = tid; i < PW * PH; i += kOrbTileW * kOrbTileH) {
    const int px = min(x0 - 4 + i % PW, W - 1), py = min(y0 - 4 + i / PW, H - 1);
    pix[i / PW][i % PW] = __ldg(it.img + (size_t)py * it.pitch + px);
  }
  __syncthreads();
  for (int i = tid; i < SW * SH; i += kOrbTileW * kOrbTileH) {
    const int sx = i % SW, sy = i / SW;  // pixel (x0 - 1 + sx, y0 - 1 + sy), at pix[sy + 3][sx + 3]
    int v[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) v[k] = pix[sy + 3 + dfk_om_circle_y(k)][sx + 3 + dfk_om_circle_x(k)];
    score[sy][sx] = dfk_om_fast_score(pix[sy + 3][sx + 3], v, it.threshold);
  }
  __syncthreads();
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int rx = blockIdx.x * kOrbTileW + tx, ry = blockIdx.y * kOrbTileH + ty;  // position in R
  const bool inside = rx < it.rw && ry < it.rh;
  const int sc = score[ty + 1][tx + 1];
  bool keep = inside && sc >= 0;
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx)
      if (dx || dy) keep = keep && sc > max(score[ty + 1 + dy][tx + 1 + dx], 0);  // a non-corner counts as 0
  if (inside) s.map[it.map_begin + (size_t)ry * it.rw + rx] = keep ? (uint8_t)(sc + 1) : (uint8_t)0;
  const unsigned ballot = __ballot_sync(0xffffffffu, keep);
  if (tx == 0 && ry < it.rh) s.seg[it.seg_begin + ry * it.tiles_x + blockIdx.x] = __popc(ballot);
  if (keep) atomicAdd(&s.hist[blockIdx.z * 256 + sc], 1);
}

// 1b. The blurred image over R widened by kReach, which is every pixel a descriptor samples.  A tile of 32 x 8 outputs
// stages its pixels and their 7-tap row sums in shared memory; each output is then the 7-tap column sum of row sums.
// A row sum is the same fp64 expression whichever output uses it, so this is dfk_om_blur bit for bit.  Block (32, 8),
// grid (tiles x, tiles y, item).
__global__ void __launch_bounds__(kOrbTileW * kOrbTileH) orb_blur_kernel(const OrbItemDev* __restrict__ items,
                                                                        OrbScratchDev s)
{
  const OrbItemDev it = items[blockIdx.z];
  if (it.rw == 0) return;
  const int bw = it.rw + 2 * kReach, bh = it.rh + 2 * kReach;
  if ((int)blockIdx.x * kOrbTileW >= bw || (int)blockIdx.y * kOrbTileH >= bh) return;
  constexpr int PW = kOrbTileW + 6, PH = kOrbTileH + 6;
  __shared__ uint8_t pix[PH][PW];
  __shared__ double rows[PH][kOrbTileW];
  const int tid = threadIdx.y * kOrbTileW + threadIdx.x;
  // output (bx, by) is pixel (bx + 13, by + 13); the tile reads pixels from 3 before its first output, clamped past the
  // image (those outputs are not written)
  const int W = it.rw + 2 * DFK_OM_EDGE, H = it.rh + 2 * DFK_OM_EDGE;
  const int x0 = blockIdx.x * kOrbTileW + DFK_OM_EDGE - kReach - 3, y0 = blockIdx.y * kOrbTileH + DFK_OM_EDGE - kReach - 3;
  for (int i = tid; i < PW * PH; i += kOrbTileW * kOrbTileH)
    pix[i / PW][i % PW] = __ldg(it.img + (size_t)min(y0 + i / PW, H - 1) * it.pitch + min(x0 + i % PW, W - 1));
  __syncthreads();
  for (int i = tid; i < PH * kOrbTileW; i += kOrbTileW * kOrbTileH) {
    const int r = i / kOrbTileW, c = i % kOrbTileW;
    double acc = 0.0;
#pragma unroll
    for (int k = 0; k < 7; ++k) acc += dfk_om_gauss_tap(k) * (double)pix[r][c + k];
    rows[r][c] = acc;
  }
  __syncthreads();
  const int bx = blockIdx.x * kOrbTileW + threadIdx.x, by = blockIdx.y * kOrbTileH + threadIdx.y;
  if (bx >= bw || by >= bh) return;
  double acc = 0.0;
#pragma unroll
  for (int k = 0; k < 7; ++k) acc += dfk_om_gauss_tap(k) * rows[threadIdx.y + k][threadIdx.x];
  s.blur[it.blur_begin + (size_t)by * bw + bx] = (uint8_t)(int)rint(acc);
}

// 2. Per image: the segment counts become offsets (raster order), and the first cut's score threshold.
__global__ void __launch_bounds__(kScanThreads) orb_scan_kernel(const OrbItemDev* __restrict__ items, OrbScratchDev s)
{
  const OrbItemDev it = items[blockIdx.x];
  __shared__ int smem[33];
  __shared__ int hist[256];
  for (int i = threadIdx.x; i < 256; i += kScanThreads) hist[i] = s.hist[blockIdx.x * 256 + i];
  __syncthreads();
  const int nseg = it.rh * it.tiles_x;
  int running = 0;
  for (int base = 0; base < nseg; base += kScanThreads) {
    const int i = base + threadIdx.x;
    const int v = i < nseg ? s.seg[it.seg_begin + i] : 0;
    int total;
    const int ex = block_exclusive_scan(v, smem, &total);
    if (i < nseg) s.seg[it.seg_begin + i] = running + ex;
    running += total;
  }
  if (threadIdx.x == 0) {
    // every corner whose score is at least the (2 nfeatures)-th largest
    int thr = 0, cand = running;
    if (running > 2 * it.nfeatures) {
      int above = 0;
      thr = 255;
      while (above + hist[thr] < 2 * it.nfeatures) above += hist[thr--];
      cand = above + hist[thr];
    }
    int* st = s.stats + 4 * blockIdx.x;
    st[0] = running;
    st[1] = thr;
    st[2] = cand;
    st[3] = 0;
  }
}

// 3. Raster-order compaction: one warp per segment writes its corners at the segment's offset.
__global__ void __launch_bounds__(kWarps * 32) orb_compact_kernel(const OrbItemDev* __restrict__ items,
                                                                 OrbScratchDev s)
{
  const OrbItemDev it = items[blockIdx.y];
  const int lane = threadIdx.x & 31;
  const int nseg = it.rh * it.tiles_x;
  for (int g = blockIdx.x * kWarps + (threadIdx.x >> 5); g < nseg; g += gridDim.x * kWarps) {
    const int ry = g / it.tiles_x, rx = (g % it.tiles_x) * kOrbTileW + lane;
    const int v = rx < it.rw ? s.map[it.map_begin + (size_t)ry * it.rw + rx] : 0;
    const unsigned ballot = __ballot_sync(0xffffffffu, v != 0);
    if (v) {
      const int c = it.corner_begin + s.seg[it.seg_begin + g] + __popc(ballot & ((1u << lane) - 1u));
      s.pos[c] = (uint32_t)(ry + DFK_OM_EDGE) << 16 | (uint32_t)(rx + DFK_OM_EDGE);
      s.key[c] = (uint32_t)(v - 1);
    }
  }
}

// 4. One warp per corner: a corner that passed the first cut gets its Harris response (as a sort key) and its angle;
// every other corner gets key 0.
__global__ void __launch_bounds__(kWarps * 32) orb_harris_kernel(const OrbItemDev* __restrict__ items,
                                                                OrbScratchDev s)
{
  const OrbItemDev it = items[blockIdx.y];
  const int lane = threadIdx.x & 31;
  const int ncorner = s.stats[4 * blockIdx.y], thr = s.stats[4 * blockIdx.y + 1];
  for (int i = blockIdx.x * kWarps + (threadIdx.x >> 5); i < ncorner; i += gridDim.x * kWarps) {
    const int c = it.corner_begin + i;
    if ((int)s.key[c] < thr) {  // warp-uniform
      if (lane == 0) s.key[c] = 0u;
      continue;
    }
    const uint32_t p = s.pos[c];
    const int x = (int)(p & 0xffffu), y = (int)(p >> 16);
    // Harris over the 7 x 7 block: lane handles block positions lane and lane + 32
    int a = 0, b = 0, cc = 0;
    for (int q = lane; q < DFK_OM_HARRIS_BLOCK * DFK_OM_HARRIS_BLOCK; q += 32) {
      const int bx = x + q % 7 - 3, by = y + q / 7 - 3;
      int nb[9];
#pragma unroll
      for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int k = 0; k < 3; ++k) nb[3 * j + k] = __ldg(it.img + (size_t)(by + j - 1) * it.pitch + (bx + k - 1));
      const int ix = dfk_om_harris_ix(nb), iy = dfk_om_harris_iy(nb);
      a += ix * ix;
      b += iy * iy;
      cc += ix * iy;
    }
    // moments over the radius-15 disc: lane handles column u = lane - 15
    int m01 = 0, m10 = 0;
    if (lane <= 2 * DFK_OM_HALF_PATCH) {
      const int u = lane - DFK_OM_HALF_PATCH, au = u < 0 ? -u : u;
      for (int v = -DFK_OM_HALF_PATCH; v <= DFK_OM_HALF_PATCH; ++v) {
        if (au > dfk_om_umax(v < 0 ? -v : v)) continue;
        const int val = __ldg(it.img + (size_t)(y + v) * it.pitch + (x + u));
        m10 += u * val;
        m01 += v * val;
      }
    }
    a = warp_sum(a);
    b = warp_sum(b);
    cc = warp_sum(cc);
    m01 = warp_sum(m01);
    m10 = warp_sum(m10);
    if (lane == 0) {
      s.key[c] = dfk_om_response_key(dfk_om_harris_response(a, b, cc));
      s.angle[c] = dfk_om_angle(m01, m10);
    }
  }
}

__device__ __forceinline__ float key_response(uint32_t k)
{
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// 5. Per image: the second cut and the output order.  A radix select finds K, the key of the min(nfeatures,
// candidates)-th largest response; the keys above K (fewer than nfeatures) are sorted in shared memory by (key
// descending, corner index), and the corners whose key equals K follow in corner (raster) order.  Writes the row ->
// corner map of the first `capacity` rows and the count.  Dynamic shared memory: a power of two >= nfeatures of
// 64-bit entries.
__global__ void __launch_bounds__(kScanThreads) orb_select_kernel(const OrbItemDev* __restrict__ items,
                                                                 OrbScratchDev s, int* counts)
{
  extern __shared__ unsigned long long sorted[];
  __shared__ int hist[256];
  __shared__ int smem[33];
  __shared__ uint32_t sel[2];  // prefix, remaining rank
  const OrbItemDev it = items[blockIdx.x];
  const int ncorner = s.stats[4 * blockIdx.x], ncand = s.stats[4 * blockIdx.x + 2];
  const uint32_t* key = s.key + it.corner_begin;
  const int k = min(it.nfeatures, ncand);
  if (k == 0) {
    if (threadIdx.x == 0) counts[blockIdx.x] = 0;
    return;
  }
  if (threadIdx.x == 0) { sel[0] = 0u; sel[1] = (uint32_t)k; }
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += kScanThreads) hist[i] = 0;
    __syncthreads();
    const uint32_t prefix = sel[0], hi = shift == 24 ? 0u : ~0u << (shift + 8);
    for (int i = threadIdx.x; i < ncorner; i += kScanThreads) {
      const uint32_t v = key[i];
      if ((v & hi) == prefix) atomicAdd(&hist[(v >> shift) & 255u], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int rank = (int)sel[1], bin = 255;
      while (hist[bin] < rank) rank -= hist[bin--];
      sel[0] = prefix | (uint32_t)bin << shift;
      sel[1] = (uint32_t)rank;
    }
    __syncthreads();
  }
  const uint32_t K = sel[0];
  // the keys above K, compacted in corner order, then sorted
  int ng = 0;
  for (int base = 0; base < ncorner; base += kScanThreads) {
    const int i = base + threadIdx.x;
    const bool g = i < ncorner && key[i] > K;
    int total;
    const int at = ng + block_exclusive_scan(g ? 1 : 0, smem, &total);
    if (g) sorted[at] = (unsigned long long)(~key[i]) << 32 | (uint32_t)i;
    ng += total;
  }
  int np = 1;
  while (np < ng) np <<= 1;
  for (int i = ng + threadIdx.x; i < np; i += kScanThreads) sorted[i] = ~0ull;
  __syncthreads();
  for (int size = 2; size <= np; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < np; i += kScanThreads) {
        const int j = i ^ stride;
        if (j > i) {
          const unsigned long long a = sorted[i], b = sorted[j];
          if ((a > b) == ((i & size) == 0)) { sorted[i] = b; sorted[j] = a; }
        }
      }
      __syncthreads();
    }
  int* rows = s.rows + it.out_begin;
  for (int i = threadIdx.x; i < min(ng, it.capacity); i += kScanThreads) rows[i] = (int)(uint32_t)sorted[i];
  // the keys equal to K, in corner order
  int ne = 0;
  for (int base = 0; base < ncorner; base += kScanThreads) {
    const int i = base + threadIdx.x;
    const bool e = i < ncorner && key[i] == K;
    int total;
    const int at = ng + ne + block_exclusive_scan(e ? 1 : 0, smem, &total);
    if (e && at < it.capacity) rows[at] = i;
    ne += total;
  }
  if (threadIdx.x == 0) {
    counts[blockIdx.x] = ng + ne;
    s.stats[4 * blockIdx.x + 3] = ng + ne;
  }
}

// 6. One warp per output row: the keypoint, angle, response and descriptor.  Lane j computes descriptor byte j (bits
// 8j .. 8j + 7, 16 pattern points) from the blurred image.
__global__ void __launch_bounds__(kWarps * 32) orb_describe_kernel(const OrbItemDev* __restrict__ items,
                                                                  OrbScratchDev s, float* keypoints,
                                                                  uint8_t* descriptors, float* angles,
                                                                  float* responses)
{
  __shared__ int8_t pattern[DFK_ORB_PATTERN_PAIRS * 4];
  for (int i = threadIdx.x; i < DFK_ORB_PATTERN_PAIRS * 4; i += kWarps * 32) pattern[i] = c_pattern[i];
  __syncthreads();
  const OrbItemDev it = items[blockIdx.y];
  const int lane = threadIdx.x & 31;
  const int nrows = min(s.stats[4 * blockIdx.y + 3], it.capacity);
  const int bw = it.rw + 2 * kReach;
  for (int r = blockIdx.x * kWarps + (threadIdx.x >> 5); r < nrows; r += gridDim.x * kWarps) {
    const int c = it.corner_begin + s.rows[it.out_begin + r];
    const uint32_t p = s.pos[c];
    const int x = (int)(p & 0xffffu), y = (int)(p >> 16);
    const float angle = s.angle[c];
    // the keypoint in the blurred image
    const uint8_t* B = s.blur + it.blur_begin + (size_t)(y - DFK_OM_EDGE + kReach) * bw + (x - DFK_OM_EDGE + kReach);
    float ca, sa;
    dfk_om_rotation(angle, &ca, &sa);
    uint32_t byte = 0;
#pragma unroll
    for (int bit = 0; bit < 8; ++bit) {
      const int j = 8 * lane + bit;
      int x0, y0, x1, y1;
      dfk_om_rotate(pattern[4 * j], pattern[4 * j + 1], ca, sa, &x0, &y0);
      dfk_om_rotate(pattern[4 * j + 2], pattern[4 * j + 3], ca, sa, &x1, &y1);
      byte |= (uint32_t)(B[y0 * bw + x0] < B[y1 * bw + x1]) << bit;
    }
    const size_t row = (size_t)it.out_begin + r;
    descriptors[32 * row + lane] = (uint8_t)byte;
    if (lane == 0) {
      keypoints[2 * row] = (float)x;
      keypoints[2 * row + 1] = (float)y;
      if (angles) angles[row] = angle;
      if (responses) responses[row] = key_response(s.key[c]);
    }
  }
}

int blocks_for(int work, int per_block) { return max(1, min(kMaxBlocksPerItem, (work + per_block - 1) / per_block)); }

}  // namespace

cudaError_t launch_orb_detect(const OrbItemDev* items_dev, int n, const OrbScratchDev& s, int max_rw, int max_rh,
                              int max_corner_cap, int max_segs, int max_capacity, int max_nfeatures,
                              float* keypoints, uint8_t* descriptors, float* angles, float* responses, int* counts,
                              cudaStream_t stream)
{
  cudaError_t e = cudaMemsetAsync(s.hist, 0, sizeof(int) * 256 * (size_t)n, stream);
  if (e != cudaSuccess) return e;
  if (max_rw > 0 && max_rh > 0) {
    const dim3 block(kOrbTileW, kOrbTileH);
    orb_fast_kernel<<<dim3((max_rw + kOrbTileW - 1) / kOrbTileW, (max_rh + kOrbTileH - 1) / kOrbTileH, n), block, 0,
                      stream>>>(items_dev, s);
    orb_blur_kernel<<<dim3((max_rw + 2 * kReach + kOrbTileW - 1) / kOrbTileW,
                           (max_rh + 2 * kReach + kOrbTileH - 1) / kOrbTileH, n), block, 0, stream>>>(items_dev, s);
  }
  orb_scan_kernel<<<n, kScanThreads, 0, stream>>>(items_dev, s);
  orb_compact_kernel<<<dim3(blocks_for(max_segs, kWarps), n), kWarps * 32, 0, stream>>>(items_dev, s);
  orb_harris_kernel<<<dim3(blocks_for(max_corner_cap, kWarps), n), kWarps * 32, 0, stream>>>(items_dev, s);
  int sort_n = 1;
  while (sort_n < max_nfeatures) sort_n <<= 1;  // fewer than nfeatures keys lie above the cut
  const size_t smem = sizeof(unsigned long long) * (size_t)sort_n;
  e = cudaFuncSetAttribute(orb_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  orb_select_kernel<<<n, kScanThreads, smem, stream>>>(items_dev, s, counts);
  orb_describe_kernel<<<dim3(blocks_for(max_capacity, kWarps), n), kWarps * 32, 0, stream>>>(
      items_dev, s, keypoints, descriptors, angles, responses);
  return cudaGetLastError();
}

}  // namespace dfk
