// dfk_preprocess.cu -- DeepFactors::PreprocessImage (core/deepfactors.cpp:634-680) of many camera frames on the device
// (sm_90a): the remap to the network camera, the gray and float conversion and the optional normalisation.  The
// per-pixel model is dfk_preprocess_model.h, shared with the sequential CPU build of the specification that checks the
// kernels; this unit is built with -fmad=false so that it rounds as that build does.  The pyramid that follows runs on
// the batched blur-down and Sobel kernels of dfk_simple.cu.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_internal.h"

namespace dfk {

namespace {

constexpr int kThreads = DFK_PM_TILE_W * DFK_PM_TILE_H;
static_assert(kThreads == DFK_PM_TREE, "one tile is one tree of the fixed summation order");

// The pairwise tree of the fixed order (dfk_preprocess_model.h) over a[0..256), b[0..256) in shared memory; the sums
// end in a[0], b[0]
__device__ __forceinline__ void tree_sum(double* a, double* b)
{
  __syncthreads();
#pragma unroll
  for (int stride = DFK_PM_TREE / 2; stride > 0; stride >>= 1) {
    if ((int)threadIdx.x < stride) {
      a[threadIdx.x] = a[threadIdx.x] + a[threadIdx.x + stride];
      b[threadIdx.x] = b[threadIdx.x] + b[threadIdx.x + stride];
    }
    __syncthreads();
  }
}

// Row blockIdx.y is item n, block blockIdx.x its tile (row-major over the output); blocks past the item's tiles return.
// One thread per output pixel: the map, the four taps, the colour, gray and float pixel.  A normalising item also
// writes the tile's fp64 sums of f and f^2 (partials[2 (partial_begin + tile) + {0, 1}]).
__global__ void __launch_bounds__(kThreads) preprocess_kernel(const PpItemDev* __restrict__ items,
                                                             double* __restrict__ partials)
{
  const PpItemDev& it = items[blockIdx.y];
  const int tile = blockIdx.x;
  if (tile >= it.tiles) return;
  const int ty = tile / it.tiles_x, tx = tile - ty * it.tiles_x;
  const int j = tx * DFK_PM_TILE_W + (int)(threadIdx.x % DFK_PM_TILE_W);
  const int r = ty * DFK_PM_TILE_H + (int)(threadIdx.x / DFK_PM_TILE_W);
  float f = 0.0f;
  if (j < it.w && r < it.h) {
    const DfkPmMap map = it.map;
    uint8_t c[3];
    dfk_pm_remap_pixel(&map, it.src, it.src_pitch, it.sw, it.sh, j, r, c);
    if (it.color) {
      uint8_t* o = it.color + (size_t)r * it.color_pitch + 3 * (size_t)j;
      o[0] = c[0];
      o[1] = c[1];
      o[2] = c[2];
    }
    const uint8_t g = dfk_pm_gray(c);
    if (it.gray) it.gray[(size_t)r * it.gray_pitch + j] = g;
    f = dfk_pm_float(g);
    if (it.level0) it.level0[(size_t)r * it.level0_pitch + j] = f;
  }
  if (!it.normalize) return;
  __shared__ double s1[kThreads], s2[kThreads];
  s1[threadIdx.x] = (double)f;
  s2[threadIdx.x] = (double)f * (double)f;  // exact: a product of two fp32 values fits in fp64
  tree_sum(s1, s2);
  if (threadIdx.x == 0) {
    partials[2 * ((size_t)it.partial_begin + tile)] = s1[0];
    partials[2 * ((size_t)it.partial_begin + tile) + 1] = s2[0];
  }
}

// The statistics of the items that normalise, one CTA per item: the item's tile partials summed in the fixed order
// (thread t sums tiles t, t + 256, ..., then the tree), once per item.  (mu, sigma) go to the item's moments scratch and,
// when asked, to its stats row.
__global__ void __launch_bounds__(kThreads) preprocess_stats_kernel(const PpItemDev* __restrict__ items,
                                                                   const double* __restrict__ partials)
{
  const PpItemDev& it = items[blockIdx.x];
  if (!it.normalize) return;
  __shared__ double s1[kThreads], s2[kThreads];
  double a = 0.0, b = 0.0;
  const double* p = partials + 2 * (size_t)it.partial_begin;
  for (int k = threadIdx.x; k < it.tiles; k += kThreads) {
    a = a + __ldg(p + 2 * (size_t)k);
    b = b + __ldg(p + 2 * (size_t)k + 1);
  }
  s1[threadIdx.x] = a;
  s2[threadIdx.x] = b;
  tree_sum(s1, s2);
  if (threadIdx.x != 0) return;
  double mu, sigma;
  dfk_pm_stats(s1[0], s2[0], (double)it.w * (double)it.h, &mu, &sigma);
  it.moments[0] = mu;
  it.moments[1] = sigma;
  if (it.stats) {
    it.stats[0] = mu;
    it.stats[1] = sigma;
  }
}

// Level 0 of the items that normalise and have levels, rewritten as f' = (f - mu) / sigma; same grid as
// preprocess_kernel.
__global__ void __launch_bounds__(kThreads) preprocess_normalize_kernel(const PpItemDev* __restrict__ items)
{
  const PpItemDev& it = items[blockIdx.y];
  const int tile = blockIdx.x;
  if (!it.normalize || !it.level0 || tile >= it.tiles) return;
  const int ty = tile / it.tiles_x, tx = tile - ty * it.tiles_x;
  const int j = tx * DFK_PM_TILE_W + (int)(threadIdx.x % DFK_PM_TILE_W);
  const int r = ty * DFK_PM_TILE_H + (int)(threadIdx.x / DFK_PM_TILE_W);
  if (j >= it.w || r >= it.h) return;
  const double mu = __ldg(it.moments), sigma = __ldg(it.moments + 1);
  float* px = it.level0 + (size_t)r * it.level0_pitch + j;
  *px = dfk_pm_normalize(*px, mu, sigma);
}

}  // namespace

cudaError_t launch_preprocess(const PpItemDev* items_dev, int n, int max_tiles, bool normalize, double* partials,
                              cudaStream_t s)
{
  const dim3 grid((unsigned)max_tiles, (unsigned)n);
  preprocess_kernel<<<grid, kThreads, 0, s>>>(items_dev, partials);
  if (!normalize) return cudaGetLastError();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  preprocess_stats_kernel<<<(unsigned)n, kThreads, 0, s>>>(items_dev, partials);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  preprocess_normalize_kernel<<<grid, kThreads, 0, s>>>(items_dev);
  return cudaGetLastError();
}

}  // namespace dfk
