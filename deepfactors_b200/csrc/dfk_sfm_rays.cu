// dfk_sfm_rays.cu -- normalised ray tables of the SfmAligner::RunStep kernels (all three engines read them).
//
// Reproject's IEEE divisions (x - u0) / fx and (y - v0) / fy (dfk_geom.cuh ray_coord) depend only on the column / row
// and the camera level, so the handle keeps one table per camera level and builds it once, on the call that first
// names that level.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_geom.cuh"
#include "dfk_internal.h"

namespace dfk {

namespace {

// one CTA per item: xn[x] = (x - u0)/fx for x < W, then yn[y] = (y - v0)/fy for y < H
__global__ void sfm_ray_tables_kernel(const SfmItemDev* __restrict__ items)
{
  const SfmItemDev& I = items[blockIdx.x];
  float* dst = const_cast<float*>(I.ray_tab);
  for (uint32_t x = threadIdx.x; x < I.width; x += blockDim.x) dst[x] = ray_coord((float)x, I.u0, I.fx);
  for (uint32_t y = threadIdx.x; y < I.height; y += blockDim.x) dst[I.width + y] = ray_coord((float)y, I.v0, I.fy);
}

}  // namespace

cudaError_t launch_sfm_ray_tables(const SfmItemDev* items_dev, int num_items, cudaStream_t stream)
{
  sfm_ray_tables_kernel<<<num_items, 256, 0, stream>>>(items_dev);
  return cudaGetLastError();
}

}  // namespace dfk
