// dfk_simple.cu -- the thin kernels around the SfM hot path (sm_90a):
//   SE3Aligner::RunStep     cu_se3aligner.cpp:37-59,153-176  + lucas_kanade_se3.h:41-77
//   SE3Aligner::Warp        cu_se3aligner.cpp:61-113,125-151
//   SfmAligner::EvaluateError  cu_sfmaligner.cpp:72-97,120-147 + dense_sfm.h:79-119
//   UpdateDepth             cu_image_proc.cpp:248-277 + warping.h:30-69
//   SobelGradients          cu_image_proc.cpp:57-113
//   GaussianBlurDown        cu_image_proc.cpp:134-184
//   SquaredError            cu_image_proc.cpp:190-242
// (file:line into jczarnowski/DeepFactors @ bffc78a).
//
// All reductions are single-launch: per-thread register accumulation over a grid-stride loop,
// warp-shuffle + shared-memory block reduction, per-block partials to scratch, and the LAST block
// to arrive (atomic ticket) sums the partials in block order -- deterministic, no host sync, no
// second launch (the reference needs kernel_finalize_reduction + cudaDeviceSynchronize,
// kernel_utils.h:51-69, launch_utils.h:28).
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_geom.cuh"
#include "dfk_gn.cuh"
#include "dfk_internal.h"

namespace dfk {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// Block-level reduction of NV floats + one counter, then last-block finalize.
// out[0..NV) = sums, out[NV] = counter bits.  scratch: nblocks * 32 floats.  NV <= 31.
// `block` / `nblocks` are this block's index and the number of blocks that take part (blockIdx.x / gridDim.x for a
// one-reduction grid; one row of a batched grid otherwise), so every reduction of the same size sums in the same order.
template <int NV>
__device__ __forceinline__ bool reduce_finalize(float (&v)[NV], unsigned int cnt, int block, int nblocks,
                                                float* __restrict__ scratch, unsigned int* __restrict__ counter,
                                                float* __restrict__ out)
{
  static_assert(NV <= 31, "one scratch row is 32 floats");
  __shared__ float red[kWarps][32];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = warp_sum(v[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) red[warp][i] = v[i];
    red[warp][NV] = __uint_as_float(cnt);
  }
  __syncthreads();
  if (warp == 0 && lane <= NV) {
    if (lane < NV) {
      float s = 0.0f;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) s += red[w][lane];
      scratch[block * 32 + lane] = s;
    } else {
      unsigned int c = 0;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) c += __float_as_uint(red[w][NV]);
      scratch[block * 32 + NV] = __uint_as_float(c);
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int ticket = atomicAdd(counter, 1u);
    is_last = (ticket == (unsigned int)nblocks - 1u);
  }
  __syncthreads();
  if (!is_last) return false;
  __threadfence();
  // last block: warp w sums blocks w, w+kWarps, ... ; then warp order
  float s = 0.0f;
  unsigned int c = 0;
  if (lane <= NV) {
    for (int b = warp; b < nblocks; b += kWarps) {
      const float x = __ldcg(&scratch[b * 32 + lane]);
      if (lane < NV) s += x;
      else c += __float_as_uint(x);
    }
  }
  __syncthreads();
  red[warp][lane] = (lane < NV) ? s : __uint_as_float(c);
  __syncthreads();
  if (warp == 0 && lane <= NV) {
    if (lane < NV) {
      float t = 0.0f;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) t += red[w][lane];
      out[lane] = t;
    } else {
      unsigned int t = 0;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) t += __float_as_uint(red[w][NV]);
      out[NV] = __uint_as_float(t);
    }
  }
  if (threadIdx.x == 0) *counter = 0;  // self-resetting for the next launch on this stream
  return true;
}

// ------------------------------------------------------------------------------ SE3 RunStep
// The per-pixel body of SE3Aligner::RunStep (lucas_kanade_se3.h:41-77): this thread's pixels first, first + stride, ...
// of one problem, accumulated into acc (21 JtJ packed upper, 6 Jtr, 1 residual) and the inlier count.  Shared by the
// single-problem and the batched kernel, so a problem gives the same sums whichever of the two evaluates it.
__device__ __forceinline__ void se3_accumulate(const PixelCam& pc, float huber_delta, int width, int height, View img0,
                                               View img1, View dpt0, View grad1, bool grad_aligned, int first,
                                               int stride, float (&acc)[28], unsigned int& inl)
{
#pragma unroll
  for (int i = 0; i < 28; ++i) acc[i] = 0.0f;
  inl = 0;
  const int area = width * height;
  for (int i = first; i < area; i += stride) {
    const int y = i / width, x = i - y * width;
    const float d = __ldg(dpt0.ptr + (size_t)y * dpt0.pitch + x);
    const Warped w = warp_pixel((float)x, (float)y, d, pc.q, pc.t, pc.fx, pc.fy, pc.u0, pc.v0, pc.border, pc.ulim,
                                pc.vlim, pc.min_dpt);
    if (!w.valid) continue;
    int ix, iy;
    float fu, fv, gx, gy;
    bilin_setup(w.u, w.v, ix, iy, fu, fv);
    sample_grad(grad1.ptr, grad1.pitch, grad_aligned, ix, iy, fu, fv, gx, gy);
    const float i1 = sample_scalar(img1.ptr, img1.pitch, ix, iy, fu, fv);
    float a[6], c00, c02, c11, c12;
    pose_jacobian_row(w, pc.fx, pc.fy, gx, gy, a, c00, c02, c11, c12);
    float diff = __ldg(img0.ptr + (size_t)y * img0.pitch + x) - i1;
    const float hw = huber_weight(diff, huber_delta);
    diff *= hw;
#pragma unroll
    for (int k = 0; k < 6; ++k) a[k] *= hw;
    inl += 1;
    acc[27] = fmaf(diff, diff, acc[27]);
    int h = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
      acc[21 + r] = fmaf(a[r], diff, acc[21 + r]);
#pragma unroll
      for (int c = r; c < 6; ++c) {
        acc[h] = fmaf(a[r], a[c], acc[h]);
        ++h;
      }
    }
  }
}

// Tracking mode: the pose lives in device memory; the last block of the previous launch updated it, this launch
// reads it, ...
__device__ __forceinline__ void se3_load_pose(PixelCam& pc, const float* pose_dev)
{
#pragma unroll
  for (int k = 0; k < 4; ++k) pc.q[k] = pose_dev[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) pc.t[k] = pose_dev[4 + k];
}

// ... and its own last block applies the next Gauss-Newton update.  A system without inliers leaves the pose alone, bit
// for bit, as the reference's tracker does (it skips the update when no pixel is valid): gn_update_pose would apply a
// zero step and then renormalise the quaternion in fp32, which moves most unit quaternions by an ulp or so.  Called by
// the last block of a problem only.
__device__ __forceinline__ void se3_track_update(const float* out, float* pose_dev, float* __restrict__ history)
{
  __syncthreads();  // out[0..28] was written by warp 0 of this block
  if (threadIdx.x == 0) {
    float pose[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) pose[k] = pose_dev[k];
    if (history) {  // [29 system | 7 pose the system was evaluated at]
#pragma unroll 1
      for (int k = 0; k < 29; ++k) history[k] = out[k];
#pragma unroll
      for (int k = 0; k < 7; ++k) history[29 + k] = pose[k];
    }
    if (__float_as_uint(out[28]) == 0u) return;  // no inliers
    float sys[27];
#pragma unroll 1
    for (int k = 0; k < 27; ++k) sys[k] = out[k];
    if (gn_update_pose(sys, pose)) {
#pragma unroll
      for (int k = 0; k < 7; ++k) pose_dev[k] = pose[k];
    }
  }
}

__global__ void __launch_bounds__(kThreads)
se3_step_kernel(PixelCam pc, float huber_delta, int width, int height, View img0, View img1, View dpt0, View grad1,
                bool grad_aligned, float* __restrict__ scratch, unsigned int* __restrict__ counter,
                float* __restrict__ out, float* pose_dev, float* __restrict__ history)
{
  if (pose_dev) se3_load_pose(pc, pose_dev);  // tracking mode (pose_dev != nullptr)
  float acc[28];
  unsigned int inl;
  se3_accumulate(pc, huber_delta, width, height, img0, img1, dpt0, grad1, grad_aligned,
                 blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x, acc, inl);
  const bool last = reduce_finalize<28>(acc, inl, blockIdx.x, gridDim.x, scratch, counter, out);
  if (pose_dev && last) se3_track_update(out, pose_dev, history);
}

// N tracking problems advanced in lockstep, one Gauss-Newton iteration of every problem per launch.  Row blockIdx.y is
// problem n; it uses the first d.nblocks blocks of the row (what se3_step_kernel's grid would be for that level), the
// rest of the row returns at once and takes no ticket.  Problem n owns scratch rows [n * scratch_stride, +nblocks),
// counters[n], out[32 n .. +29) and the pose poses[8 n .. +7); its last block updates that pose.
__global__ void __launch_bounds__(kThreads)
se3_track_batch_kernel(const Se3TrackDesc* __restrict__ descs, float huber_delta, float* __restrict__ scratch,
                       int scratch_stride, unsigned int* __restrict__ counters, float* __restrict__ outs, float* poses)
{
  const int n = blockIdx.y;
  const Se3TrackDesc& d = descs[n];
  const int nblocks = d.nblocks;
  if ((int)blockIdx.x >= nblocks) return;
  float* pose_dev = poses + 8 * (size_t)n;
  float* out = outs + 32 * (size_t)n;
  PixelCam pc = d.pc;
  se3_load_pose(pc, pose_dev);
  float acc[28];
  unsigned int inl;
  se3_accumulate(pc, huber_delta, d.width, d.height, d.img0, d.img1, d.dpt0, d.grad1, d.grad_aligned != 0,
                 blockIdx.x * blockDim.x + threadIdx.x, nblocks * blockDim.x, acc, inl);
  const bool last = reduce_finalize<28>(acc, inl, blockIdx.x, nblocks, scratch + (size_t)n * scratch_stride * 32,
                                        counters + n, out);
  if (last) se3_track_update(out, pose_dev, nullptr);
}

// ------------------------------------------------------------------------------ EvaluateError
__global__ void __launch_bounds__(kThreads)
eval_error_kernel(PixelCam pc, float huber_delta, int width, int height, View img0, View img1, View dpt0,
                  float* __restrict__ scratch, unsigned int* __restrict__ counter, float* __restrict__ out)
{
  float acc[1] = {0.0f};
  unsigned int inl = 0;
  const int area = width * height;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < area; i += gridDim.x * blockDim.x) {
    const int y = i / width, x = i - y * width;
    const float d = __ldg(dpt0.ptr + (size_t)y * dpt0.pitch + x);
    const Warped w = warp_pixel((float)x, (float)y, d, pc.q, pc.t, pc.fx, pc.fy, pc.u0, pc.v0, pc.border, pc.ulim,
                                pc.vlim, pc.min_dpt);
    if (!w.valid) continue;
    int ix, iy;
    float fu, fv;
    bilin_setup(w.u, w.v, ix, iy, fu, fv);
    float diff = __ldg(img0.ptr + (size_t)y * img0.pitch + x) - sample_scalar(img1.ptr, img1.pitch, ix, iy, fu, fv);
    diff *= huber_weight(diff, huber_delta);
    inl += 1;
    acc[0] = fmaf(diff, diff, acc[0]);
  }
  reduce_finalize<1>(acc, inl, blockIdx.x, gridDim.x, scratch, counter, out);
}

// ------------------------------------------------------------------------------ Warp
__global__ void __launch_bounds__(kThreads)
warp_kernel(PixelCam pc, int width, int height, View img0, View img1, View dpt0, float* __restrict__ img2,
            uint32_t img2_pitch, float* __restrict__ scratch, unsigned int* __restrict__ counter,
            float* __restrict__ out)
{
  float acc[1] = {0.0f};
  unsigned int inl = 0;
  const int area = width * height;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < area; i += gridDim.x * blockDim.x) {
    const int y = i / width, x = i - y * width;
    const float d = __ldg(dpt0.ptr + (size_t)y * dpt0.pitch + x);
    const Warped w = warp_pixel((float)x, (float)y, d, pc.q, pc.t, pc.fx, pc.fy, pc.u0, pc.v0, pc.border, pc.ulim,
                                pc.vlim, pc.min_dpt);
    float sampled = 0.0f;
    if (w.valid) {
      int ix, iy;
      float fu, fv;
      bilin_setup(w.u, w.v, ix, iy, fu, fv);
      sampled = sample_scalar(img1.ptr, img1.pitch, ix, iy, fu, fv);
      inl += 1;
      acc[0] += __ldg(img0.ptr + (size_t)y * img0.pitch + x) - sampled;  // signed (cu_se3aligner.cpp:106)
    }
    img2[(size_t)y * img2_pitch + x] = sampled;
  }
  reduce_finalize<1>(acc, inl, blockIdx.x, gridDim.x, scratch, counter, out);
}

// ------------------------------------------------------------------------------ SquaredError
__global__ void __launch_bounds__(kThreads)
squared_error_kernel(int width, int height, View a, View b, float* __restrict__ scratch,
                     unsigned int* __restrict__ counter, float* __restrict__ out)
{
  float acc[1] = {0.0f};
  const int area = width * height;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < area; i += gridDim.x * blockDim.x) {
    const int y = i / width, x = i - y * width;
    const float d = __ldg(a.ptr + (size_t)y * a.pitch + x) - __ldg(b.ptr + (size_t)y * b.pitch + x);
    acc[0] = fmaf(d, d, acc[0]);
  }
  reduce_finalize<1>(acc, 0u, blockIdx.x, gridDim.x, scratch, counter, out);
}

// ------------------------------------------------------------------------------ UpdateDepth
// LPP lanes cooperate on one pixel: lane `sub` owns float4 chunks sub, sub+LPP, ... of the C code
// Jacobians, so a warp reads 32 consecutive float4 (512 contiguous bytes) per instruction.
template <int C>
__global__ void __launch_bounds__(kThreads)
update_depth_kernel(const float* __restrict__ code, int width, int height, View prx, View jac, float avg_dpt,
                    float* __restrict__ dpt, uint32_t dpt_pitch)
{
  constexpr int NV = C / 4;                  // float4 chunks per pixel
  constexpr int LPP = NV < 32 ? NV : 32;     // lanes per pixel
  constexpr int PPW = 32 / LPP;              // pixels per warp instruction
  constexpr int CPL = NV / LPP;              // chunks per lane
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPP, pw = lane / LPP;
  float4 cd[CPL];
#pragma unroll
  for (int j = 0; j < CPL; ++j) cd[j] = __ldg(reinterpret_cast<const float4*>(code) + sub + j * LPP);
  const int area = width * height;
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int base = warp_global * PPW; base < area; base += nwarps * PPW) {
    const int p = base + pw;
    float dot = 0.0f;
    int x = 0, y = 0;
    if (p < area) {
      y = p / width;
      x = p - y * width;
      const float4* row = reinterpret_cast<const float4*>(jac.ptr + (size_t)y * jac.pitch + (size_t)x * C);
#pragma unroll
      for (int j = 0; j < CPL; ++j) {
        const float4 v = __ldg(row + sub + j * LPP);
        dot = fmaf(v.x, cd[j].x, dot);
        dot = fmaf(v.y, cd[j].y, dot);
        dot = fmaf(v.z, cd[j].z, dot);
        dot = fmaf(v.w, cd[j].w, dot);
      }
    }
#pragma unroll
    for (int o = LPP / 2; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    if (p < area && sub == 0) {
      const float prxv = __fadd_rn(__ldg(prx.ptr + (size_t)y * prx.pitch + x), dot);  // ProxFromCode warping.h:52-59
      dpt[(size_t)y * dpt_pitch + x] = prx_to_depth(prxv, avg_dpt);  // same order as the fused RunStep front-ends
    }
  }
}

// generic (any C, any alignment) fallback: one thread per pixel
__global__ void __launch_bounds__(kThreads)
update_depth_generic_kernel(const float* __restrict__ code, int C, int width, int height, View prx, View jac,
                            float avg_dpt, float* __restrict__ dpt, uint32_t dpt_pitch)
{
  const int area = width * height;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < area; i += gridDim.x * blockDim.x) {
    const int y = i / width, x = i - y * width;
    const float* row = jac.ptr + (size_t)y * jac.pitch + (size_t)x * C;
    float dot = 0.0f;
    for (int k = 0; k < C; ++k) dot = fmaf(__ldg(row + k), __ldg(code + k), dot);
    const float prxv = __ldg(prx.ptr + (size_t)y * prx.pitch + x) + dot;
    dpt[(size_t)y * dpt_pitch + x] = avg_dpt / prxv - avg_dpt;
  }
}

// ------------------------------------------------------------------------------ Sobel
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__global__ void __launch_bounds__(kThreads)
sobel_kernel(int width, int height, View img, float* __restrict__ grad, uint32_t grad_pitch)
{
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= width || y >= height) return;
  float p[3][3];
#pragma unroll
  for (int py = -1; py <= 1; ++py)
#pragma unroll
    for (int px = -1; px <= 1; ++px)
      p[py + 1][px + 1] = __ldg(img.ptr + (size_t)clampi(y + py, 0, height - 1) * img.pitch +
                                clampi(x + px, 0, width - 1));
  // same accumulation order as the reference loop (py outer, px inner; zero coefficients are exact no-ops)
  float sdx = 0.0f, sdy = 0.0f;
  sdx = __fadd_rn(sdx, -p[0][0]);  sdy = __fadd_rn(sdy, -p[0][0]);
  sdy = __fadd_rn(sdy, -2.0f * p[0][1]);
  sdx = __fadd_rn(sdx, p[0][2]);   sdy = __fadd_rn(sdy, -p[0][2]);
  sdx = __fadd_rn(sdx, -2.0f * p[1][0]);
  sdx = __fadd_rn(sdx, 2.0f * p[1][2]);
  sdx = __fadd_rn(sdx, -p[2][0]);  sdy = __fadd_rn(sdy, p[2][0]);
  sdy = __fadd_rn(sdy, 2.0f * p[2][1]);
  sdx = __fadd_rn(sdx, p[2][2]);   sdy = __fadd_rn(sdy, p[2][2]);
  grad[(size_t)y * grad_pitch + 2 * x + 0] = sdx * 0.125f;
  grad[(size_t)y * grad_pitch + 2 * x + 1] = sdy * 0.125f;
}

// ------------------------------------------------------------------------------ blur-down
__global__ void __launch_bounds__(kThreads)
blur_down_kernel(int in_w, int in_h, View in, int out_w, int out_h, float* __restrict__ out, uint32_t out_pitch)
{
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= out_w || y >= out_h) return;
  const float k1[5] = {1.f, 4.f, 6.f, 4.f, 1.f};
  float sum = 0.0f;
#pragma unroll
  for (int py = 0; py < 5; ++py) {
    const int ny = clampi(2 * y + py - 2, 0, in_h - 1);
#pragma unroll
    for (int px = 0; px < 5; ++px) {
      const int nx = clampi(2 * x + px - 2, 0, in_w - 1);
      sum = __fadd_rn(sum, __fmul_rn(__ldg(in.ptr + (size_t)ny * in.pitch + nx), k1[px] * k1[py]));
    }
  }
  out[(size_t)y * out_pitch + x] = sum * (1.0f / 256.0f);  // wall == 256 exactly
}

inline int grid_for(int area)
{
  int blocks = (area + kThreads - 1) / kThreads;
  const int cap = kSimpleMaxBlocks;
  return blocks < 1 ? 1 : (blocks > cap ? cap : blocks);
}

}  // namespace

int se3_step_blocks(int width, int height) { return grid_for(width * height); }

cudaError_t launch_se3_track_batch(const Se3TrackDesc* descs_dev, int num_problems, int max_blocks, float huber_delta,
                                   float* scratch, int scratch_stride, unsigned int* counters, float* outs, float* poses,
                                   cudaStream_t s)
{
  const dim3 grid((unsigned)max_blocks, (unsigned)num_problems);
  se3_track_batch_kernel<<<grid, kThreads, 0, s>>>(descs_dev, huber_delta, scratch, scratch_stride, counters, outs,
                                                   poses);
  return cudaGetLastError();
}

cudaError_t launch_se3_step(const PixelCam& pc, float huber_delta, int width, int height, View img0, View img1,
                            View dpt0, View grad1, bool grad_aligned, float* scratch, unsigned int* counter,
                            float* out_dev, cudaStream_t s, float* pose_dev, float* history_dev)
{
  se3_step_kernel<<<grid_for(width * height), kThreads, 0, s>>>(pc, huber_delta, width, height, img0, img1, dpt0,
                                                                grad1, grad_aligned, scratch, counter, out_dev,
                                                                pose_dev, history_dev);
  return cudaGetLastError();
}

cudaError_t launch_eval_error(const PixelCam& pc, float huber_delta, int width, int height, View img0, View img1,
                              View dpt0, float* scratch, unsigned int* counter, float* out_dev, cudaStream_t s)
{
  eval_error_kernel<<<grid_for(width * height), kThreads, 0, s>>>(pc, huber_delta, width, height, img0, img1, dpt0,
                                                                  scratch, counter, out_dev);
  return cudaGetLastError();
}

cudaError_t launch_warp(const PixelCam& pc, int width, int height, View img0, View img1, View dpt0, float* img2,
                        uint32_t img2_pitch, float* scratch, unsigned int* counter, float* out_dev, cudaStream_t s)
{
  warp_kernel<<<grid_for(width * height), kThreads, 0, s>>>(pc, width, height, img0, img1, dpt0, img2, img2_pitch,
                                                            scratch, counter, out_dev);
  return cudaGetLastError();
}

cudaError_t launch_squared_error(int width, int height, View a, View b, float* scratch, unsigned int* counter,
                                 float* out_dev, cudaStream_t s)
{
  squared_error_kernel<<<grid_for(width * height), kThreads, 0, s>>>(width, height, a, b, scratch, counter, out_dev);
  return cudaGetLastError();
}

cudaError_t launch_update_depth(const float* code_dev, int code_size, int width, int height, View prx_orig, View jac,
                                float avg_dpt, float* dpt, uint32_t dpt_pitch, cudaStream_t s)
{
  const int area = width * height;
  const bool aligned = (reinterpret_cast<uintptr_t>(jac.ptr) % 16 == 0) && (jac.pitch % 4 == 0) &&
                       (reinterpret_cast<uintptr_t>(code_dev) % 16 == 0);
  int blocks = (area + kThreads - 1) / kThreads;
  const int cap = 8 * sfm_max_ctas();  // grid-stride loop: one full SM's worth (8 x 256 threads) of blocks per SM
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
#define DFK_UD_CASE(CC)                                                                                       \
  case CC:                                                                                                    \
    if (aligned) {                                                                                            \
      update_depth_kernel<CC><<<blocks, kThreads, 0, s>>>(code_dev, width, height, prx_orig, jac, avg_dpt, dpt, \
                                                          dpt_pitch);                                         \
      return cudaGetLastError();                                                                              \
    }                                                                                                         \
    break;
  switch (code_size) {
    DFK_UD_CASE(4)
    DFK_UD_CASE(8)
    DFK_UD_CASE(16)
    DFK_UD_CASE(32)
    DFK_UD_CASE(64)
    DFK_UD_CASE(128)
    default: break;
  }
#undef DFK_UD_CASE
  update_depth_generic_kernel<<<blocks, kThreads, 0, s>>>(code_dev, code_size, width, height, prx_orig, jac, avg_dpt,
                                                          dpt, dpt_pitch);
  return cudaGetLastError();
}

cudaError_t launch_sobel(int width, int height, View img, float* grad, uint32_t grad_pitch, cudaStream_t s)
{
  dim3 grid((width + 31) / 32, (height + 7) / 8);
  sobel_kernel<<<grid, kThreads, 0, s>>>(width, height, img, grad, grad_pitch);
  return cudaGetLastError();
}

cudaError_t launch_blur_down(int in_w, int in_h, View in, int out_w, int out_h, float* out, uint32_t out_pitch,
                             cudaStream_t s)
{
  dim3 grid((out_w + 31) / 32, (out_h + 7) / 8);
  blur_down_kernel<<<grid, kThreads, 0, s>>>(in_w, in_h, in, out_w, out_h, out, out_pitch);
  return cudaGetLastError();
}

}  // namespace dfk
