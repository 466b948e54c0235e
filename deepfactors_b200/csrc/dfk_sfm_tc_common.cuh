// dfk_sfm_tc_common.cuh -- what the tensor-core RunStep kernels (dfk_sfm_tc.cu, dfk_sfm_tc_wide.cu) share in front of
// and behind their wgmma products: the exact h / l split, the operand stores, the read-once input stream and the
// partial flush.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace dfk {

__device__ __forceinline__ float tf32_trunc(float v) { return __uint_as_float(__float_as_uint(v) & 0xffffe000u); }

__device__ __forceinline__ void sts32(uint32_t addr, float v)
{
  // no "memory" clobber: the only plain shared-memory accesses of the front-end are reads of its item copy; volatile
  // keeps the stores ordered with the proxy fence (which carries the clobber)
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v));
}

// read-once input stream (code-Jacobian rows, img0, dpt0): read-only path, no L1 allocation
__device__ __forceinline__ float ld_stream(const float* p)
{
  float v;
  asm("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}

// 16 bytes of a code-Jacobian row; rows of items without the BULK flag are only 4-byte aligned
__device__ __forceinline__ float4 load_chunk(const float* __restrict__ p, bool aligned16)
{
  if (aligned16) {
    float4 v;
    asm("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
        : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
        : "l"(p));
    return v;
  }
  return make_float4(ld_stream(p), ld_stream(p + 1), ld_stream(p + 2), ld_stream(p + 3));
}

// the same 16 bytes through L1: the fused depth decode reads every chunk the Gram reads again a little later (the
// no-allocate loads of load_chunk still hit lines that are in L1)
__device__ __forceinline__ float4 load_chunk_l1(const float* __restrict__ p, bool aligned16)
{
  if (aligned16) return __ldg(reinterpret_cast<const float4*>(p));
  return make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3));
}

// the first chain of an item in this CTA stores, later chains add (single writer per address, program order)
__device__ __forceinline__ void put_partial(float* p, float v, bool fresh)
{
  if (fresh)
    __stcg(p, v);
  else
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

}  // namespace dfk
