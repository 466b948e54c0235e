// dfk_depth_prior.cu -- DepthPriorFactor (sources/core/gtsam/depth_prior_factor.cpp:29-137) for many (keyframe, level)
// items at once: the DepthAligner::RunStep Gram of dfk_depth.cu (same per-pixel arithmetic, same quirks: every pixel
// counts, J = -2 |diff| dDpt/dPrx jc, the handle's avg_dpt) spread over a grid of (item, partial), and the window's
// in-place addition of the depth priors built from those records.
//
// Determinism: item i owns depth_prior_parts(W_i, H_i) partial rows, a number that depends on its own size only.  Partial
// x of item i accumulates the chunks x, x + parts, x + 2 parts, ... in order, in fp32 registers (the chunked Gram of
// dfk_depth.cu, each chunk summed on its own and then added to the row's sum); the finalize sums an item's partials in
// partial order in fp64 and rounds once.  No atomics, so two calls agree bit for bit and an item's record does not
// depend on the other items of the batch.  The error kernel stages the
// same diff per pixel and accumulates diff^2 in the same order as the Gram's residual entry, so its residual is the
// record's bit for bit.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_geom.cuh"
#include "dfk_internal.h"

namespace dfk {

namespace {

constexpr int kThreads = 256;
constexpr int kChunk = 64;          // pixels per chunk
constexpr int kMaxParts = 64;       // partial rows of the largest items
constexpr int kChunksPerPart = 16;  // fewest chunks a partial row covers (small items get fewer rows)

// Stages chunk ch of item d: M[p][0..C) = s * jc (Gram only), M[p][C] = diff; 4 threads per pixel, each a quarter of the
// code dimension (the decode's dot product combined in the order of dfk_depth.cu)
template <int C, bool kGram>
__device__ __forceinline__ void stage_chunk(const DepthPriorDesc& d, const float* cs, float (*M)[C + 2], int ch,
                                            float avg_dpt)
{
  const int tid = threadIdx.x;
  const int p = tid >> 2, part = tid & 3;
  const int area = d.width * d.height;
  const int i = ch * kChunk + p;
  const bool in = i < area;
  const int y = in ? i / d.width : 0, x = in ? i - y * d.width : 0;
  const float* jr = d.jac.ptr + (size_t)y * d.jac.pitch + (size_t)x * C;
  float dot = 0.0f;
  for (int k = part * (C / 4); k < (part + 1) * (C / 4); ++k) dot = fmaf(__ldg(jr + k), cs[k], dot);
  dot += __shfl_xor_sync(0xffffffffu, dot, 1);
  dot += __shfl_xor_sync(0xffffffffu, dot, 2);
  const float prx = (in ? __ldg(d.prx.ptr + (size_t)y * d.prx.pitch + x) : 1.0f) + dot;
  const float dpt = avg_dpt / prx - avg_dpt;                                    // ProxToDepth, warping.h:30-35
  const float diff = in ? __ldg(d.tgt.ptr + (size_t)y * d.tgt.pitch + x) - dpt : 0.0f;
  if (kGram) {
    const float pr2 = avg_dpt / (avg_dpt + dpt);                                // DepthJacobianPrx, warping.h:44-50
    const float s = in ? -2.0f * fabsf(diff) * (-avg_dpt / (pr2 * pr2)) : 0.0f;
    for (int k = part * (C / 4); k < (part + 1) * (C / 4); ++k) M[p][k] = in ? s * __ldg(jr + k) : 0.0f;
  }
  if (part == 0) M[p][C] = diff;
}

// Block (x, i): partial row x of item i.  kGram: the packed upper augmented Gram (NE floats), else diff^2 (1 float).
template <int C, bool kGram>
__global__ void __launch_bounds__(kThreads)
depth_prior_partial_kernel(const DepthPriorDesc* __restrict__ descs, float avg_dpt, float* __restrict__ partials,
                           const uint8_t* __restrict__ stale)
{
  if (stale && !stale[blockIdx.y]) return;  // an item that is not stale keeps its record
  constexpr int NA = C + 1;                 // augmented row: s*jc | diff
  constexpr int NE = NA * (NA + 1) / 2;     // packed upper triangle of the augmented Gram
  constexpr int EPT = (NE + kThreads - 1) / kThreads;
  __shared__ float M[kChunk][C + 2];        // +1 past the augmented row: rows start in different banks
  __shared__ float cs[C];
  const DepthPriorDesc d = descs[blockIdx.y];
  if ((int)blockIdx.x >= d.parts) return;
  const int tid = threadIdx.x;
  for (int k = tid; k < C; k += kThreads) cs[k] = d.code[k];
  const int nchunks = (d.width * d.height + kChunk - 1) / kChunk;
  if (kGram) {
    int ei[EPT], ej[EPT];  // entry e of this thread -> (i, j), i <= j, row-major packed
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
    for (int ch = blockIdx.x; ch < nchunks; ch += d.parts) {
      stage_chunk<C, true>(d, cs, M, ch, avg_dpt);
      __syncthreads();
#pragma unroll
      for (int q = 0; q < EPT; ++q) {
        float a = 0.0f;  // the chunk's sum, then one add onto the row's: fp32 chains of 64 pixels, not 64 x chunks
        const int i = ei[q], j = ej[q];
#pragma unroll 8
        for (int p = 0; p < kChunk; ++p) a = fmaf(M[p][i], M[p][j], a);
        acc[q] += a;
      }
      __syncthreads();
    }
    float* mine = partials + (size_t)(d.part0 + blockIdx.x) * NE;
#pragma unroll
    for (int q = 0; q < EPT; ++q) {
      const int e = q * kThreads + tid;
      if (e < NE) mine[e] = acc[q];
    }
  } else {
    float a = 0.0f;
    __syncthreads();
    for (int ch = blockIdx.x; ch < nchunks; ch += d.parts) {
      stage_chunk<C, false>(d, cs, M, ch, avg_dpt);
      __syncthreads();
      if (tid == 0) {  // the Gram's (C, C) entry, same order
        float c = 0.0f;
        for (int p = 0; p < kChunk; ++p) c = fmaf(M[p][C], M[p][C], c);
        a += c;
      }
      __syncthreads();
    }
    if (tid == 0) partials[d.part0 + blockIdx.x] = a;
  }
}

// Block i: item i's partials summed in partial order in fp64, rounded once, into the record layout of
// JTJJrReductionItem<float, C>: [JtJ packed upper C(C+1)/2 | Jtr C | residual | inliers (u32 bits)], or (error) into
// [residual | inliers (u32 bits)]
template <int C, bool kGram>
__global__ void __launch_bounds__(kThreads)
depth_prior_finalize_kernel(const DepthPriorDesc* __restrict__ descs, const float* __restrict__ partials,
                            float* __restrict__ out, const uint8_t* __restrict__ stale)
{
  if (stale && !stale[blockIdx.x]) return;
  constexpr int NA = C + 1;
  constexpr int NE = NA * (NA + 1) / 2;
  constexpr int NH = C * (C + 1) / 2;
  const DepthPriorDesc d = descs[blockIdx.x];
  const unsigned int area = (unsigned int)(d.width * d.height);
  if (kGram) {
    float* rec = out + (size_t)blockIdx.x * DFK_DEPTH_RECORD_FLOATS(C);
    for (int e = threadIdx.x; e < NE; e += kThreads) {
      double s = 0.0;
      for (int b = 0; b < d.parts; ++b) s += (double)partials[(size_t)(d.part0 + b) * NE + e];
      int i = 0, rem = e;
      while (rem >= NA - i) {
        rem -= NA - i;
        ++i;
      }
      const int j = i + rem;
      if (j < C) rec[i * C - (i * (i - 1)) / 2 + (j - i)] = (float)s;  // JtJ(i, j)
      else if (i < C) rec[NH + i] = (float)s;                          // Jtr(i) = sum s*jc_i * diff
      else rec[NH + C] = (float)s;                                     // residual
    }
    if (threadIdx.x == 0) rec[NH + C + 1] = __uint_as_float(area);     // inliers: every pixel
  } else if (threadIdx.x == 0) {
    double s = 0.0;
    for (int b = 0; b < d.parts; ++b) s += (double)partials[d.part0 + b];
    out[2 * (size_t)blockIdx.x] = (float)s;
    out[2 * (size_t)blockIdx.x + 1] = __uint_as_float(area);
  }
}

template <int C>
cudaError_t launch(const DepthPriorDesc* descs_dev, int n, int max_parts, float avg_dpt, float* partials, float* out,
                   bool gram, cudaStream_t s, const uint8_t* stale)
{
  const dim3 grid((unsigned)max_parts, (unsigned)n);
  if (gram) {
    depth_prior_partial_kernel<C, true><<<grid, kThreads, 0, s>>>(descs_dev, avg_dpt, partials, stale);
    depth_prior_finalize_kernel<C, true><<<n, kThreads, 0, s>>>(descs_dev, partials, out, stale);
  } else {
    depth_prior_partial_kernel<C, false><<<grid, kThreads, 0, s>>>(descs_dev, avg_dpt, partials, stale);
    depth_prior_finalize_kernel<C, false><<<n, kThreads, 0, s>>>(descs_dev, partials, out, stale);
  }
  return cudaGetLastError();
}

// ---- depth priors into an assembled window, in place.  Prior q on keyframe k with weight 1 / sigma_q^2 and records
// [lp_q, lp_{q+1}):  D_k(code, code) += JtJ / sigma^2 (both triangles),  g_k(code) -= Jtr / sigma^2,
// f += residual / sigma^2.  CTA k < K: keyframe k's code block and code gradient, its priors in list order and each
// prior's levels in order, summed in fp64 onto the fp32 entry and rounded once.  CTA K: f, every prior in list order.
__global__ void __launch_bounds__(256)
window_add_depth_priors_kernel(WindowDev w, int m, const int* __restrict__ kf_ptr, const int* __restrict__ kf_priors,
                               const int* __restrict__ level_ptr, const float* __restrict__ sigma,
                               const float* __restrict__ records, float* __restrict__ out)
{
  const int C = w.code_size, B = 6 + C, K = w.num_keyframes;
  const int NH = C * (C + 1) / 2, REC = NH + C + 2;
  if ((int)blockIdx.x < K) {
    const int k = blockIdx.x, q0 = kf_ptr[k], q1 = kf_ptr[k + 1];
    if (q0 == q1) return;
    float* D = out + (size_t)k * B * B;
    float* g = out + (size_t)K * B * B + (size_t)k * B;
    for (int e = threadIdx.x; e < C * C + C; e += blockDim.x) {
      if (e < C * C) {
        const int r = e / C, c = e - r * C;
        const int i = min(r, c), j = max(r, c);
        const int off = i * C - (i * (i - 1)) / 2 + (j - i);
        float* dst = D + (size_t)(6 + r) * B + 6 + c;
        double s = (double)*dst;
        for (int t = q0; t < q1; ++t) {
          const int q = kf_priors[t];
          const double s2 = (double)sigma[q] * (double)sigma[q];
          for (int l = level_ptr[q]; l < level_ptr[q + 1]; ++l)
            s = __dadd_rn(s, __ddiv_rn((double)records[(size_t)l * REC + off], s2));
        }
        *dst = (float)s;
      } else {
        const int r = e - C * C;
        float* dst = g + 6 + r;
        double s = (double)*dst;
        for (int t = q0; t < q1; ++t) {
          const int q = kf_priors[t];
          const double s2 = (double)sigma[q] * (double)sigma[q];
          for (int l = level_ptr[q]; l < level_ptr[q + 1]; ++l)
            s = __dsub_rn(s, __ddiv_rn((double)records[(size_t)l * REC + NH + r], s2));
        }
        *dst = (float)s;
      }
    }
    return;
  }
  if (threadIdx.x != 0) return;
  float* f = out + (size_t)K * (B * B + B) + (size_t)w.num_pairs * B * 6;
  double s = (double)*f;
  for (int q = 0; q < m; ++q) {
    const double s2 = (double)sigma[q] * (double)sigma[q];
    for (int l = level_ptr[q]; l < level_ptr[q + 1]; ++l)
      s = __dadd_rn(s, __ddiv_rn((double)records[(size_t)l * REC + NH + C], s2));
  }
  *f = (float)s;
}

// item blockIdx.x's code from the state, rounded to fp32
__global__ void __launch_bounds__(128)
depth_prior_codes_kernel(const double* __restrict__ state_codes, const int* __restrict__ item_kf, int C,
                         float* __restrict__ out)
{
  const double* c = state_codes + (size_t)item_kf[blockIdx.x] * C;
  for (int k = threadIdx.x; k < C; k += blockDim.x) out[(size_t)blockIdx.x * C + k] = (float)c[k];
}

}  // namespace

cudaError_t launch_depth_prior_codes(const double* state_codes, const int* item_kf, int n, int code_size,
                                     float* codes_out, cudaStream_t s)
{
  if (n == 0) return cudaSuccess;
  depth_prior_codes_kernel<<<n, 128, 0, s>>>(state_codes, item_kf, code_size, codes_out);
  return cudaGetLastError();
}

int depth_prior_parts(int width, int height)
{
  const long long chunks = ((long long)width * height + kChunk - 1) / kChunk;
  return (int)std::min<long long>(kMaxParts, std::max<long long>(1, (chunks + kChunksPerPart - 1) / kChunksPerPart));
}

size_t depth_prior_partial_floats(int code_size, bool gram)
{
  return gram ? (size_t)(code_size + 1) * (code_size + 2) / 2 : 1;
}

cudaError_t launch_depth_prior_batch(int code_size, const DepthPriorDesc* descs_dev, int n, int max_parts, float avg_dpt,
                                     float* partials, float* out_dev, bool gram, cudaStream_t s, const uint8_t* stale)
{
  switch (code_size) {
    case 8: return launch<8>(descs_dev, n, max_parts, avg_dpt, partials, out_dev, gram, s, stale);
    case 16: return launch<16>(descs_dev, n, max_parts, avg_dpt, partials, out_dev, gram, s, stale);
    case 32: return launch<32>(descs_dev, n, max_parts, avg_dpt, partials, out_dev, gram, s, stale);
    case 64: return launch<64>(descs_dev, n, max_parts, avg_dpt, partials, out_dev, gram, s, stale);
    case 128: return launch<128>(descs_dev, n, max_parts, avg_dpt, partials, out_dev, gram, s, stale);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_window_add_depth_priors(const WindowDev& w, int m, const int* kf_ptr_dev, const int* kf_priors_dev,
                                           const int* level_ptr_dev, const float* sigma_dev, const float* records_dev,
                                           float* window_dev, cudaStream_t stream)
{
  window_add_depth_priors_kernel<<<w.num_keyframes + 1, 256, 0, stream>>>(w, m, kf_ptr_dev, kf_priors_dev, level_ptr_dev,
                                                                         sigma_dev, records_dev, window_dev);
  return cudaGetLastError();
}

}  // namespace dfk
