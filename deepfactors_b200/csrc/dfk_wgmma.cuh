// dfk_wgmma.cuh -- inline-PTX wrappers for the Hopper warpgroup tensor-core path (sm_90a): the shared-memory matrix
// descriptor, wgmma.mma_async m64nNk8 kind tf32 (N = 56, 88, 152) with both operands in shared memory, and the wgmma fences.
// Field layouts follow the PTX ISA chapter "Asynchronous Warpgroup Level Matrix Multiply-Accumulate".
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_async.cuh"

namespace dfk {

// generic-proxy shared-memory writes -> visible to the async proxy (wgmma reading its operands through descriptors)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Shared-memory matrix descriptor, K-major operand, no swizzle: the operand is a grid of core matrices of 8 rows x 16
// bytes (4 tf32 along K), each stored as 128 contiguous bytes (row r at r * 16).  `lbo` = byte distance between core
// matrices adjacent in K, `sbo` = between core matrices adjacent in M / N (8-row groups).
//   [0,14) addr >> 4 | [16,30) lbo >> 4 | [32,46) sbo >> 4 | [62,64) layout = 0 (no swizzle)
__device__ __forceinline__ uint64_t make_wgmma_desc_kmajor(uint32_t smem_addr, uint32_t lbo, uint32_t sbo)
{
  return (uint64_t)((smem_addr & 0x3ffffu) >> 4) | ((uint64_t)((lbo >> 4) & 0x3fffu) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3fffu) << 32);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D = A * B^T (+ D iff `accumulate`).  D 64 x 56 fp32 in registers (the warpgroup's accumulator fragment, 28 floats per
// thread), A 64 x 8 and B 56 x 8 tf32 in shared memory (K-major).  Fragment: d[4 j + 2 h + b] holds row
// 16 * warp + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + b.
__device__ __forceinline__ void wgmma_m64n56k8_tf32(float (&d)[28], uint64_t a_desc, uint64_t b_desc, bool accumulate)
{
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %30, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n56k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27}, "
      "%28, %29, p, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27])
      : "l"(a_desc), "l"(b_desc), "r"((uint32_t)accumulate)
      : "memory");
}

// D = A * B^T (+ D iff `accumulate`), N = 88: D 64 x 88 fp32 (44 floats per thread, fragment as above)
__device__ __forceinline__ void wgmma_m64n88k8_tf32(float (&d)[44], uint64_t a_desc, uint64_t b_desc, bool accumulate)
{
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %46, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n88k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43}, "
      "%44, %45, p, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]),
        "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
        "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43])
      : "l"(a_desc), "l"(b_desc), "r"((uint32_t)accumulate)
      : "memory");
}

// D = A * B^T (+ D iff `accumulate`), N = 152: D 64 x 152 fp32 (76 floats per thread, fragment as above)
__device__ __forceinline__ void wgmma_m64n152k8_tf32(float (&d)[76], uint64_t a_desc, uint64_t b_desc, bool accumulate)
{
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %78, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n152k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75}, "
      "%76, %77, p, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]),
        "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
        "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]),
        "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]),
        "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]),
        "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75])
      : "l"(a_desc), "l"(b_desc), "r"((uint32_t)accumulate)
      : "memory");
}

}  // namespace dfk
