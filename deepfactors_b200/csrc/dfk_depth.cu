// dfk_depth.cu -- DepthAligner<float,CS>::RunStep (sources/cuda/cu_depthaligner.cpp:32-113): code-only alignment of
// the decoded depth to a target depth map.  Per pixel (every pixel counts, there is no validity test):
//     dpt  = DepthFromCode(code, prx_J_cde, prx_orig(x,y), avg_dpt)              warping.h:52-69
//     diff = tgt_dpt(x,y) - dpt                                                  cu_depthaligner.cpp:56
//     J    = -2 * abs(diff) * DepthJacobianPrx(dpt, avg_dpt) * prx_J_cde         :59, warping.h:44-50
//     inliers += 1; residual += diff^2; Jtr += J^T diff; JtJ += upper(J^T J)     :61-64
// i.e. the Gram of the augmented row m = [ s * jc (C) | diff ],  s = -2 |diff| dDpt/dPrx : G[:C,:C] = JtJ,
// G[:C,C] = Jtr, G[C,C] = residual -- the code block of the SfM Gram without the warp.  The reference hard-codes
// avg_dpt = 2 in this kernel (:44); here it is the handle's DenseSfmParams::avg_dpt (SURVEY App. B quirk 11).
//
// Used by DepthPriorFactor only, which the reference never constructs (SURVEY 2 #4): a correct, deterministic,
// single-launch kernel, not a tuned one.  Blocks stream 64-pixel chunks: the scaled rows go to shared memory, every
// thread owns a fixed set of entries of the packed upper triangle of G and accumulates them in registers; per-block
// partials go to scratch and the last block to arrive (atomic ticket) sums them in block order.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_geom.cuh"
#include "dfk_internal.h"

namespace dfk {

namespace {

constexpr int kThreads = 256;
constexpr int kChunk = 64;  // pixels per chunk

template <int C>
__global__ void __launch_bounds__(kThreads)
depth_step_kernel(const float* __restrict__ code, int width, int height, View tgt, View prx_orig, View jac, float avg_dpt,
                  float* __restrict__ scratch, unsigned int* __restrict__ counter, float* __restrict__ out)
{
  constexpr int NA = C + 1;                 // augmented row: s*jc | diff
  constexpr int NE = NA * (NA + 1) / 2;     // packed upper triangle of the augmented Gram
  constexpr int EPT = (NE + kThreads - 1) / kThreads;
  __shared__ float M[kChunk][NA + 1];       // +1: rows start in different banks
  __shared__ float cs[C];
  __shared__ bool is_last;
  const int tid = threadIdx.x;
  for (int k = tid; k < C; k += kThreads) cs[k] = code[k];
  // entry e of this thread -> (i, j), i <= j, row-major packed
  int ei[EPT], ej[EPT];
#pragma unroll
  for (int q = 0; q < EPT; ++q) {
    int e = q * kThreads + tid;
    if (e >= NE) e = 0;
    int i = 0, rem = e;
    while (rem >= NA - i) {
      rem -= NA - i;
      ++i;
    }
    ei[q] = i;
    ej[q] = i + rem;
  }
  float acc[EPT];
#pragma unroll
  for (int q = 0; q < EPT; ++q) acc[q] = 0.0f;
  __syncthreads();
  const int area = width * height;
  const int nchunks = (area + kChunk - 1) / kChunk;
  for (int ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
    // ---- stage the chunk: 4 threads per pixel, each a quarter of the code dimension --------------------------------
    {
      const int p = tid >> 2, part = tid & 3;
      const int i = ch * kChunk + p;
      const bool in = i < area;
      const int y = in ? i / width : 0, x = in ? i - y * width : 0;
      const float* jr = jac.ptr + (size_t)y * jac.pitch + (size_t)x * C;
      float dot = 0.0f;
      // DepthFromCode: prx = prx_0code + prx_J_cde . code, summed left to right like the 1xC * Cx1 product (warping.h:58)
      // -- the four partial ranges are combined in order below
      float part_dot = 0.0f;
      for (int k = part * (C / 4); k < (part + 1) * (C / 4); ++k) part_dot = fmaf(__ldg(jr + k), cs[k], part_dot);
      dot = part_dot;
      dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      dot += __shfl_xor_sync(0xffffffffu, dot, 2);
      const float prx = (in ? __ldg(prx_orig.ptr + (size_t)y * prx_orig.pitch + x) : 1.0f) + dot;
      const float dpt = avg_dpt / prx - avg_dpt;                                  // ProxToDepth, warping.h:30-35
      const float diff = in ? __ldg(tgt.ptr + (size_t)y * tgt.pitch + x) - dpt : 0.0f;
      const float pr2 = avg_dpt / (avg_dpt + dpt);                                // DepthJacobianPrx, warping.h:44-50
      const float s = in ? -2.0f * fabsf(diff) * (-avg_dpt / (pr2 * pr2)) : 0.0f;
      for (int k = part * (C / 4); k < (part + 1) * (C / 4); ++k) M[p][k] = in ? s * __ldg(jr + k) : 0.0f;
      if (part == 0) M[p][C] = diff;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < EPT; ++q) {
      float a = acc[q];
      const int i = ei[q], j = ej[q];
#pragma unroll 8
      for (int p = 0; p < kChunk; ++p) a = fmaf(M[p][i], M[p][j], a);
      acc[q] = a;
    }
    __syncthreads();
  }
  // ---- per-block partial -> scratch; the last block sums the partials in block order ---------------------------------
  float* mine = scratch + (size_t)blockIdx.x * NE;
#pragma unroll
  for (int q = 0; q < EPT; ++q) {
    const int e = q * kThreads + tid;
    if (e < NE) mine[e] = acc[q];
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned int ticket = atomicAdd(counter, 1u);
    is_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // record layout of JTJJrReductionItem<float, C>: [JtJ packed upper C(C+1)/2 | Jtr C | residual | inliers (u32 bits)]
  constexpr int NH = C * (C + 1) / 2;
  for (int e = tid; e < NE; e += kThreads) {
    float s = 0.0f;
    for (int b = 0; b < (int)gridDim.x; ++b) s += __ldcg(scratch + (size_t)b * NE + e);
    int i = 0, rem = e;
    while (rem >= NA - i) {
      rem -= NA - i;
      ++i;
    }
    const int j = i + rem;
    if (j < C) out[i * C - (i * (i - 1)) / 2 + (j - i)] = s;   // JtJ(i, j)
    else if (i < C) out[NH + i] = s;                           // Jtr(i) = sum s*jc_i * diff
    else out[NH + C] = s;                                      // residual
  }
  if (tid == 0) {
    out[NH + C + 1] = __uint_as_float((unsigned int)area);     // inliers: every pixel (:61)
    *counter = 0;                                              // self-resetting for the next launch on this stream
  }
}

template <int C>
cudaError_t launch(const float* code_dev, int width, int height, View tgt, View prx_orig, View jac, float avg_dpt,
                   float* scratch, unsigned int* counter, float* out_dev, int blocks, cudaStream_t s)
{
  depth_step_kernel<C><<<blocks, kThreads, 0, s>>>(code_dev, width, height, tgt, prx_orig, jac, avg_dpt, scratch, counter,
                                                  out_dev);
  return cudaGetLastError();
}

}  // namespace

size_t depth_partial_floats(int code_size) { return (size_t)(code_size + 1) * (code_size + 2) / 2; }

bool depth_supported(int code_size)
{
  return code_size == 8 || code_size == 16 || code_size == 32 || code_size == 64 || code_size == 128;
}

cudaError_t launch_depth_step(const float* code_dev, int code_size, int width, int height, View tgt, View prx_orig,
                              View jac, float avg_dpt, float* scratch, unsigned int* counter, float* out_dev, int blocks,
                              cudaStream_t s)
{
  switch (code_size) {
    case 8: return launch<8>(code_dev, width, height, tgt, prx_orig, jac, avg_dpt, scratch, counter, out_dev, blocks, s);
    case 16: return launch<16>(code_dev, width, height, tgt, prx_orig, jac, avg_dpt, scratch, counter, out_dev, blocks, s);
    case 32: return launch<32>(code_dev, width, height, tgt, prx_orig, jac, avg_dpt, scratch, counter, out_dev, blocks, s);
    case 64: return launch<64>(code_dev, width, height, tgt, prx_orig, jac, avg_dpt, scratch, counter, out_dev, blocks, s);
    case 128: return launch<128>(code_dev, width, height, tgt, prx_orig, jac, avg_dpt, scratch, counter, out_dev, blocks, s);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace dfk
