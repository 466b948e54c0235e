// dfk_sfm_finalize.cu -- second stage of SfmAligner::RunStep: fixed-order sum of the per-CTA partials
// + expansion of the reduced (7+C) system to the reference's (12+C) layout.
//
// Replaces kernel_finalize_reduction (sources/cuda/kernel_utils.h:51-69) and the host-side work the
// reference does not need because it accumulates the full 1x(12+C) Jacobian per pixel
// (dense_sfm.h:163-199): with the relative-pose Jacobians P0 = d pose10 / d pose0 and P1 = d pose10 /
// d pose1 (warping.h:120-134, computed on the host like cu_sfmaligner.cpp:164-166),
//     J = [ a*P0 | a*P1 | e*jc ]  =>  JtJ = E^T G E,  Jtr = E^T g,   E = [[P0, P1, 0], [0, 0, I_C]].
//
// grid = (num_items, C + 1): unit u < C is code row u (G[u][u..C-1] and G[u][pose/res columns]); unit C
// is the 7x7 pose/residual block.  8 warps split the partial list (k = warp, warp+8, ...), the cross-
// warp sum runs in warp order => bitwise reproducible.
// Record layout: [JtJ packed upper (NP(NP+1)/2) | Jtr (NP) | residual | inliers (u32 bits)].
//
// Two partial formats:
//   fp32 and wide kernels, tensor-core kernel at C = 32 : G itself, row-major NFP x NFP (features: code 0..C-1,
//                                                         a C..C+5, r C+6), upper blocks valid
//   tensor-core kernel at C = 64, 128 (sfm_tc_writes_d)  : D = A x B^T over split-tf32 h / l rows (TcCfg<C>, stored
//                                                         column-major); G = HH + LH + LH^T
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_internal.h"

namespace dfk {

namespace {

constexpr int kFinWarps = 8;
constexpr int kFinUnroll = 4;

__device__ __forceinline__ int packed_index(int i, int j, int NP) { return i * NP - (i * (i - 1)) / 2 + (j - i); }

template <int C, bool TC>
__global__ void __launch_bounds__(kFinWarps * 32)
sfm_finalize_kernel(const SfmItemDev* __restrict__ items, const float* __restrict__ partials,
                    float* __restrict__ records)
{
  using Cfg = SfmCfg<C>;
  constexpr int NFP = Cfg::NFP;
  constexpr int NP = 12 + C;
  constexpr int NH = NP * (NP + 1) / 2;
  constexpr int REC = NH + NP + 2;
  constexpr int NE = (C + 7 > 49) ? (C + 7) : 49;  // entries per unit (code row: <= C+7, pose unit: 49)
  constexpr int EPL = (NE + 31) / 32;              // entries per lane
  using Tc = TcCfg<C>;
  constexpr int PSTRIDE = TC ? Tc::PARTIAL_FLOATS : Cfg::PARTIAL_FLOATS;
  constexpr int INL_OFF = TC ? Tc::INLIERS : NFP * NFP;
  constexpr int NOFF = TC ? 3 : 1;
  __shared__ float red[kFinWarps][EPL * 32];
  __shared__ unsigned int red_inl[kFinWarps];
  __shared__ float sum[EPL * 32];

  // launched with programmatic stream serialization: the launch itself (and everything above that does not read the
  // partials) overlaps the tail of the step kernel; the partials are valid after this grid-dependency wait
  cudaGridDependencySynchronize();
  const SfmItemDev& I = items[blockIdx.x];
  const int unit = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* P = partials + (size_t)I.partial_begin * PSTRIDE;
  const int np = (int)I.num_ctas;

  // entry e of the unit -> feature pair (i, j), i <= j -> offsets into one partial
  int off[EPL][NOFF];
  bool act[EPL];
#pragma unroll
  for (int q = 0; q < EPL; ++q) {
    const int e = q * 32 + lane;
    int fi, fj;
    if (unit < C) {  // code row `unit`: columns unit .. C+6
      act[q] = (unit + e) < (C + 7);
      fi = unit;
      fj = unit + e;
    } else {  // pose block: entry e -> (e / 7, e % 7), upper part only
      const int r = e / 7, c = e - 7 * r;
      act[q] = (e < 49) && (c >= r);
      fi = C + r;
      fj = C + c;
    }
    if (!act[q]) {
      fi = 0;
      fj = 0;
    }
    if constexpr (TC) {
      off[q][0] = Tc::hh(fi, fj);  // HH[i][j]
      off[q][1] = Tc::lh(fi, fj);  // LH[i][j]
      off[q][2] = Tc::lh(fj, fi);  // LH[j][i]
    } else {
      off[q][0] = fi * NFP + fj;
    }
  }
  float part[EPL];
#pragma unroll
  for (int q = 0; q < EPL; ++q) part[q] = 0.0f;
  unsigned int inl = 0;
  // kFinUnroll partials per trip: their loads are independent, so a trip costs one memory round trip instead of
  // kFinUnroll; the per-trip values are combined in index order, which keeps the summation order fixed
  for (int k0 = warp; k0 < np; k0 += kFinWarps * kFinUnroll) {
    float v[kFinUnroll][EPL];
    unsigned int vi[kFinUnroll];
#pragma unroll
    for (int u = 0; u < kFinUnroll; ++u) {
      const int k = k0 + u * kFinWarps;
      const bool on = k < np;
      const float* Pk = P + (size_t)(on ? k : 0) * PSTRIDE;
#pragma unroll
      for (int q = 0; q < EPL; ++q) {
        v[u][q] = 0.0f;
        if (on && act[q]) {
          if constexpr (TC) v[u][q] = (Pk[off[q][0]] + Pk[off[q][1]]) + Pk[off[q][2]];
          else v[u][q] = Pk[off[q][0]];
        }
      }
      vi[u] = (on && unit == C && lane == 0) ? reinterpret_cast<const unsigned int*>(Pk)[INL_OFF] : 0u;
    }
#pragma unroll
    for (int u = 0; u < kFinUnroll; ++u) {
#pragma unroll
      for (int q = 0; q < EPL; ++q) part[q] += v[u][q];
      inl += vi[u];
    }
  }
#pragma unroll
  for (int q = 0; q < EPL; ++q) red[warp][q * 32 + lane] = part[q];
  if (lane == 0) red_inl[warp] = inl;
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int q = 0; q < EPL; ++q) {
      float s = 0.0f;
#pragma unroll
      for (int w = 0; w < kFinWarps; ++w) s += red[w][q * 32 + lane];
      sum[q * 32 + lane] = s;
    }
  }
  __syncthreads();

  float* rec = records + (size_t)blockIdx.x * REC;
  float* JtJ = rec;
  float* Jtr = rec + NH;
  if (unit < C) {
    const int c = unit;
    // code-code: H[12+c][12+c'] = G[c][c'] , c' >= c
    for (int e = threadIdx.x; e < C - c; e += blockDim.x) JtJ[packed_index(12 + c, 12 + c + e, NP)] = sum[e];
    // pose-code: H[j][12+c] = sum_k P0[k][j] * G[a_k][c] ; H[6+j][12+c] with P1.  G[c][C+k] is entry (C - c) + k
    if (threadIdx.x < 12) {
      const int j = threadIdx.x % 6;
      const float* Pm = threadIdx.x < 6 ? I.P0 : I.P1;
      float s = 0.0f;
#pragma unroll
      for (int k = 0; k < 6; ++k) s = fmaf(Pm[k * 6 + j], sum[(C - c) + k], s);
      JtJ[packed_index(threadIdx.x, 12 + c, NP)] = s;
    }
    if (threadIdx.x == 12) Jtr[12 + c] = sum[(C - c) + 6];
  } else {
    // pose block: Gaa (6x6 symmetric, upper stored at sum[r*7+c]), Gar = sum[r*7+6], Grr = sum[48]
    __shared__ float Gaa[6][6];
    __shared__ float T0[6][6];  // Gaa * P0
    __shared__ float T1[6][6];  // Gaa * P1
    if (threadIdx.x < 36) {
      const int r = threadIdx.x / 6, c = threadIdx.x % 6;
      Gaa[r][c] = (c >= r) ? sum[r * 7 + c] : sum[c * 7 + r];
    }
    __syncthreads();
    if (threadIdx.x < 72) {
      const int m = threadIdx.x / 36, r = (threadIdx.x % 36) / 6, c = threadIdx.x % 6;
      const float* Pm = m ? I.P1 : I.P0;
      float s = 0.0f;
#pragma unroll
      for (int k = 0; k < 6; ++k) s = fmaf(Gaa[r][k], Pm[k * 6 + c], s);
      (m ? T1 : T0)[r][c] = s;
    }
    __syncthreads();
    // H[i][j] for the 12x12 pose part, i <= j:  Pa^T * Gaa * Pb
    for (int e = threadIdx.x; e < 144; e += blockDim.x) {
      const int i = e / 12, j = e % 12;
      if (j < i) continue;
      const float* Pa = (i < 6) ? I.P0 : I.P1;
      const float(*Tb)[6] = (j < 6) ? T0 : T1;
      const int ii = i % 6, jj = j % 6;
      float s = 0.0f;
#pragma unroll
      for (int k = 0; k < 6; ++k) s = fmaf(Pa[k * 6 + ii], Tb[k][jj], s);
      JtJ[packed_index(i, j, NP)] = s;
    }
    if (threadIdx.x >= 160 && threadIdx.x < 172) {
      const int i = threadIdx.x - 160;
      const float* Pa = (i < 6) ? I.P0 : I.P1;
      float s = 0.0f;
#pragma unroll
      for (int k = 0; k < 6; ++k) s = fmaf(Pa[k * 6 + (i % 6)], sum[k * 7 + 6], s);
      Jtr[i] = s;
    }
    if (threadIdx.x == 192) {
      unsigned int tot = 0;
      for (int w = 0; w < kFinWarps; ++w) tot += red_inl[w];
      rec[NH + NP] = sum[48];
      reinterpret_cast<unsigned int*>(rec)[NH + NP + 1] = tot;
    }
  }
}

template <int C, bool TC>
cudaError_t launch_fin(const SfmItemDev* items_dev, int num_items, const float* partials_dev, float* records_dev,
                       cudaStream_t stream)
{
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(num_items, C + 1);
  cfg.blockDim = dim3(kFinWarps * 32);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, sfm_finalize_kernel<C, TC>, items_dev, partials_dev, records_dev);
}

}  // namespace

cudaError_t launch_sfm_finalize(int code_size, bool tc, const SfmItemDev* items_dev, int num_items,
                                const float* partials_dev, float* records_dev, cudaStream_t stream)
{
  if (tc && sfm_tc_writes_d(code_size)) {
    switch (code_size) {
      case 64: return launch_fin<64, true>(items_dev, num_items, partials_dev, records_dev, stream);
      case 128: return launch_fin<128, true>(items_dev, num_items, partials_dev, records_dev, stream);
      default: return cudaErrorInvalidValue;
    }
  }
  switch (code_size) {
    case 8: return launch_fin<8, false>(items_dev, num_items, partials_dev, records_dev, stream);
    case 16: return launch_fin<16, false>(items_dev, num_items, partials_dev, records_dev, stream);
    case 32: return launch_fin<32, false>(items_dev, num_items, partials_dev, records_dev, stream);
    case 64: return launch_fin<64, false>(items_dev, num_items, partials_dev, records_dev, stream);
    case 128: return launch_fin<128, false>(items_dev, num_items, partials_dev, records_dev, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace dfk
