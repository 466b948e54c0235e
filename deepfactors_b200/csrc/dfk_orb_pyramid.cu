// dfk_orb_pyramid.cu -- the scale pyramid of cv::ORB with nlevels > 1 (dfk_orb_detect_pyramid_batch): the batched
// level resize, one launch per level, and the gather that puts the one-level detector's staged rows of every level in
// level order.  The detection itself is dfk_orb.cu's, run over (image, level) items.  Compiled without FMA contraction
// so that the resize taps (dfk_orb_pyramid_model.h) round as their host build does.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_internal.h"
#include "dfk_orb_pyramid_model.h"

namespace dfk {
namespace {

constexpr int kResizeW = 32, kResizeH = 8;
constexpr int kGatherThreads = 256;
constexpr int kMaxGatherBlocks = 64;

// One output pixel per thread.  Block (32, 8), grid (tiles x, tiles y, item of the level).
__global__ void __launch_bounds__(kResizeW * kResizeH) orb_resize_kernel(const OrbResizeDev* __restrict__ items)
{
  const OrbResizeDev it = items[blockIdx.z];
  const int x = blockIdx.x * kResizeW + threadIdx.x, y = blockIdx.y * kResizeH + threadIdx.y;
  if (x >= it.dw || y >= it.dh) return;
  int ox, cx, oy, cy;
  dfk_opm_tap(x, it.sw, it.dw, &ox, &cx);
  dfk_opm_tap(y, it.sh, it.dh, &oy, &cy);
  const int ox1 = min(ox + 1, it.sw - 1), oy1 = min(oy + 1, it.sh - 1);
  const uint8_t* r0 = it.src + (size_t)oy * it.src_pitch;
  const uint8_t* r1 = it.src + (size_t)oy1 * it.src_pitch;
  it.dst[(size_t)y * it.dw + x] =
      (uint8_t)dfk_opm_resize_px(__ldg(r0 + ox), __ldg(r0 + ox1), __ldg(r1 + ox), __ldg(r1 + ox1), cx, cy);
}

// Per image: the levels' counts become first rows (a serial prefix over at most 16 levels), then one thread per output
// row copies the staged row of its level, scales the keypoint by s_k and writes the octave.  Grid (blocks, image).
__global__ void __launch_bounds__(kGatherThreads) orb_gather_kernel(const OrbGatherDev* __restrict__ items,
                                                                   const OrbItemDev* __restrict__ subs,
                                                                   OrbStagingDev st, float* keypoints,
                                                                   uint8_t* descriptors, float* angles,
                                                                   float* responses, int32_t* octaves, int32_t* counts)
{
  __shared__ int first[kOrbMaxLevels + 1];
  __shared__ int begin[kOrbMaxLevels];
  const OrbGatherDev it = items[blockIdx.y];
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int k = 0; k < it.nlevels; ++k) {
      first[k] = acc;
      acc += st.counts[it.sub_begin + k];
      begin[k] = subs[it.sub_begin + k].out_begin;
    }
    first[it.nlevels] = acc;
    if (blockIdx.x == 0) counts[blockIdx.y] = acc;
  }
  __syncthreads();
  const int nrows = min(first[it.nlevels], it.capacity);
  for (int r = blockIdx.x * kGatherThreads + threadIdx.x; r < nrows; r += gridDim.x * kGatherThreads) {
    int k = 0;
    while (r >= first[k + 1]) ++k;
    const size_t src = (size_t)begin[k] + (r - first[k]), dst = (size_t)it.out_begin + r;
    const float s = it.scale[k];
    keypoints[2 * dst] = st.keypoints[2 * src] * s;
    keypoints[2 * dst + 1] = st.keypoints[2 * src + 1] * s;
    const uint4* d = reinterpret_cast<const uint4*>(st.descriptors) + 2 * src;
    reinterpret_cast<uint4*>(descriptors)[2 * dst] = d[0];
    reinterpret_cast<uint4*>(descriptors)[2 * dst + 1] = d[1];
    if (angles) angles[dst] = st.angles[src];
    if (responses) responses[dst] = st.responses[src];
    if (octaves) octaves[dst] = k;
  }
}

}  // namespace

cudaError_t launch_orb_resize_level(const OrbResizeDev* items_dev, int count, int max_w, int max_h, cudaStream_t stream)
{
  if (count < 1 || max_w < 1 || max_h < 1) return cudaSuccess;
  orb_resize_kernel<<<dim3((max_w + kResizeW - 1) / kResizeW, (max_h + kResizeH - 1) / kResizeH, count),
                      dim3(kResizeW, kResizeH), 0, stream>>>(items_dev);
  return cudaGetLastError();
}

cudaError_t launch_orb_gather(const OrbGatherDev* items_dev, int n, const OrbItemDev* subs_dev, const OrbStagingDev& st,
                              int max_capacity, float* keypoints, uint8_t* descriptors, float* angles,
                              float* responses, int32_t* octaves, int32_t* counts, cudaStream_t stream)
{
  const int blocks = max(1, min(kMaxGatherBlocks, (max_capacity + kGatherThreads - 1) / kGatherThreads));
  orb_gather_kernel<<<dim3(blocks, n), kGatherThreads, 0, stream>>>(items_dev, subs_dev, st, keypoints, descriptors,
                                                                   angles, responses, octaves, counts);
  return cudaGetLastError();
}

}  // namespace dfk
