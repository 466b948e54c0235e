// dfk_mesh.cu -- dfk_keyframe_mesh_batch (include/dfk.h, DESIGN.md section 4.12): the keyframe renderer's geometry
// (gui/shaders/drawkf.geom) as a world-frame mesh, and SaveKeyframes' uint16 depth, for many keyframes in one call.
//
// Three launches over every (tile, item); a depth the call decodes is already in scratch (update_depth_kernel,
// enqueued by the call before these):
//   classify  a 32 x 8 tile with a one-pixel halo: the pixel flags of 34 x 10 pixels, the triangle flags of the 33 x 9
//             quads that touch the tile, then per pixel its own T1 / T2 flags and whether it is a corner of an emitted
//             triangle (the four quads that share it), as three 32-bit masks per row segment
//   scan      one CTA per item: the exclusive prefix of the segments' vertex and triangle counts in row-major order,
//             and the item's two counts
//   write     per pixel of an item within its capacities: the uint16 depth, its vertex row (position, normal, colour,
//             pixel index) and the triangles of its quad, whose corners' vertex indices come from their segment's base
//             and mask
// Integer scans only: the rows depend on the item alone.  The per-element arithmetic is dfk_mesh_model.h, compiled
// with -fmad=false (Makefile), as its sequential CPU build is with -ffp-contract=off.
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_internal.h"
#include "dfk_mesh_model.h"
#include "dfk_se3.cuh"

namespace dfk {
namespace {

constexpr int kT = kMeshTileW * kMeshTileH;  // threads per CTA, one pixel each
static_assert(kMeshTileW == 32 && kT % 32 == 0, "a warp is one row segment");
constexpr int kHaloW = kMeshTileW + 2, kHaloH = kMeshTileH + 2;  // pixels x0 - 1 .. x0 + 32, y0 - 1 .. y0 + 8
constexpr int kQuadW = kMeshTileW + 1, kQuadH = kMeshTileH + 1;  // quads x0 .. x0 + 32, y0 - 1 .. y0 + 7

__device__ __forceinline__ float mesh_depth(const MeshItemDev& it, int x, int y)
{
  return (x < 0 || y < 0 || x >= it.w || y >= it.h) ? 0.0f : __ldg(it.dpt.ptr + (size_t)y * it.dpt.pitch + x);
}

__device__ __forceinline__ unsigned mesh_pixel(const MeshItemDev& it, const MeshParamsDev& p, int x, int y, float d)
{
  if (x < 0 || y < 0 || x >= it.w || y >= it.h) return 0u;
  const float vld = it.vld.ptr ? __ldg(it.vld.ptr + (size_t)y * it.vld.pitch + x) : 0.0f;
  const float s = it.std.ptr ? __ldg(it.std.ptr + (size_t)y * it.std.pitch + x) : 0.0f;
  return dfk_mm_pixel(x, y, it.w, it.h, d, it.vld.ptr != nullptr, vld, it.std.ptr != nullptr, s, p.tau, p.draw_noisy);
}

__device__ __forceinline__ long long seg_index(const MeshItemDev& it, int x, int y)
{
  return it.seg_begin + (long long)y * it.tiles_x + (x >> 5);
}

// the item-local vertex index of pixel (x, y), which is a vertex
__device__ __forceinline__ int vertex_index(const MeshItemDev& it, const uint3* __restrict__ segs,
                                           const int2* __restrict__ bases, int x, int y)
{
  const long long s = seg_index(it, x, y);
  return bases[s].x + __popc(segs[s].x & ((1u << (x & 31)) - 1u));
}

__global__ void __launch_bounds__(kT)
keyframe_mesh_classify_kernel(const MeshItemDev* __restrict__ items, MeshParamsDev p, uint3* __restrict__ segs)
{
  const MeshItemDev& it = items[blockIdx.y];
  if ((int)blockIdx.x >= it.tiles) return;
  const int x0 = ((int)blockIdx.x % it.tiles_x) * kMeshTileW, y0 = ((int)blockIdx.x / it.tiles_x) * kMeshTileH;
  __shared__ float sd[kHaloH][kHaloW];
  __shared__ unsigned char sf[kHaloH][kHaloW];
  __shared__ unsigned char sq[kQuadH][kQuadW];
  for (int i = threadIdx.x; i < kHaloH * kHaloW; i += kT) {
    const int r = i / kHaloW, c = i - r * kHaloW, x = x0 - 1 + c, y = y0 - 1 + r;
    const float d = mesh_depth(it, x, y);
    sd[r][c] = d;
    sf[r][c] = (unsigned char)mesh_pixel(it, p, x, y, d);
  }
  __syncthreads();
  // quad (x0 + c, y0 - 1 + r): tr is halo pixel (r, c + 1), tl (r, c), br (r + 1, c + 1), bl (r + 1, c)
  for (int i = threadIdx.x; i < kQuadH * kQuadW; i += kT) {
    const int r = i / kQuadW, c = i - r * kQuadW;
    const unsigned f[4] = {sf[r][c + 1], sf[r][c], sf[r + 1][c + 1], sf[r + 1][c]};
    const float d[4] = {sd[r][c + 1], sd[r][c], sd[r + 1][c + 1], sd[r + 1][c]};
    sq[r][c] = (unsigned char)dfk_mm_quad(x0 + c, y0 - 1 + r, it.w, it.h, p.crop, p.slt, f, d, it.fx, it.fy, it.u0,
                                          it.v0);
  }
  __syncthreads();
  const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5, x = x0 + lx, y = y0 + ly;
  const bool in = x < it.w && y < it.h;
  // pixel (x, y) is tr of quad (x, y), tl of (x + 1, y), br of (x, y - 1) and bl of (x + 1, y - 1)
  const unsigned own = in ? sq[ly + 1][lx] : 0u;
  const unsigned right = sq[ly + 1][lx + 1], up = sq[ly][lx], up_right = sq[ly][lx + 1];
  const bool vertex = in && ((own & DFK_MM_T1) || ((right | up) & (DFK_MM_T1 | DFK_MM_T2)) || (up_right & DFK_MM_T2));
  const unsigned vm = __ballot_sync(0xffffffffu, vertex);
  const unsigned t1 = __ballot_sync(0xffffffffu, own & DFK_MM_T1);
  const unsigned t2 = __ballot_sync(0xffffffffu, own & DFK_MM_T2);
  if (lx == 0 && y < it.h) segs[seg_index(it, x, y)] = make_uint3(vm, t1, t2);
}

// exclusive block scan of (vertices, triangles); *total gets the block's sum
__device__ __forceinline__ int2 block_exclusive_scan(int2 v, int2* total)
{
  __shared__ int2 warp_sum[kT / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int2 inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int a = __shfl_up_sync(0xffffffffu, inc.x, o), b = __shfl_up_sync(0xffffffffu, inc.y, o);
    if (lane >= o) {
      inc.x += a;
      inc.y += b;
    }
  }
  if (lane == 31) warp_sum[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int2 w = lane < kT / 32 ? warp_sum[lane] : make_int2(0, 0);
#pragma unroll
    for (int o = 1; o < kT / 32; o <<= 1) {
      const int a = __shfl_up_sync(0xffffffffu, w.x, o), b = __shfl_up_sync(0xffffffffu, w.y, o);
      if (lane >= o) {
        w.x += a;
        w.y += b;
      }
    }
    if (lane < kT / 32) warp_sum[lane] = w;
  }
  __syncthreads();
  const int2 before = wid > 0 ? warp_sum[wid - 1] : make_int2(0, 0);
  *total = warp_sum[kT / 32 - 1];
  __syncthreads();  // warp_sum is reused by the next call
  return make_int2(before.x + inc.x - v.x, before.y + inc.y - v.y);
}

// one CTA per item: segments in row-major order, kT at a time
__global__ void __launch_bounds__(kT)
keyframe_mesh_scan_kernel(const MeshItemDev* __restrict__ items, const uint3* __restrict__ segs,
                          int2* __restrict__ bases, int32_t* __restrict__ counts)
{
  const MeshItemDev& it = items[blockIdx.x];
  const long long S = (long long)it.h * it.tiles_x;
  int2 carry = make_int2(0, 0);
  for (long long k0 = 0; k0 < S; k0 += kT) {
    const long long k = k0 + threadIdx.x;
    int2 c = make_int2(0, 0);
    if (k < S) {
      const uint3 m = segs[it.seg_begin + k];
      c = make_int2(__popc(m.x), __popc(m.y) + __popc(m.z));
    }
    int2 total;
    const int2 ex = block_exclusive_scan(c, &total);
    if (k < S) bases[it.seg_begin + k] = make_int2(carry.x + ex.x, carry.y + ex.y);
    carry.x += total.x;
    carry.y += total.y;
  }
  if (threadIdx.x == 0) {
    counts[2 * blockIdx.x] = carry.x;
    counts[2 * blockIdx.x + 1] = carry.y;
  }
}

__global__ void __launch_bounds__(kT)
keyframe_mesh_write_kernel(const MeshItemDev* __restrict__ items, MeshParamsDev p, MeshOutDev o,
                           const uint3* __restrict__ segs, const int2* __restrict__ bases)
{
  const int i = blockIdx.y;
  const MeshItemDev& it = items[i];
  if ((int)blockIdx.x >= it.tiles) return;
  if (o.counts[2 * i] > it.v_cap || o.counts[2 * i + 1] > it.t_cap) return;  // overflow: the counts only
  const int x = ((int)blockIdx.x % it.tiles_x) * kMeshTileW + (threadIdx.x & 31);
  const int y = ((int)blockIdx.x / it.tiles_x) * kMeshTileH + (threadIdx.x >> 5);
  if (x >= it.w || y >= it.h) return;
  const long long s = seg_index(it, x, y);
  const uint3 m = segs[s];
  const int2 b = bases[s];
  const unsigned bit = 1u << (x & 31), below = bit - 1u;
  const float d = mesh_depth(it, x, y);
  if (it.depth_u16)
    reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(it.depth_u16) + (size_t)y * it.u16_pitch)[x] =
        dfk_mm_depth_u16(d);
  if (m.x & bit) {
    const long long row = it.v_begin + b.x + __popc(m.x & below);
    float pc[3], pw[3];
    dfk_mm_lift(x, y, d, it.fx, it.fy, it.u0, it.v0, pc);
    se3f::quat_rotate(it.q, pc, pw);
    for (int k = 0; k < 3; ++k) o.positions[3 * row + k] = se3f::add(pw[k], it.t[k]);
    if (o.normals) {
      const float d4[4] = {d, mesh_depth(it, x - 1, y), mesh_depth(it, x, y + 1), mesh_depth(it, x - 1, y + 1)};
      float n1[3], n2[3], nc[3], nw[3];
      dfk_mm_quad_normals(x, y, d4, it.fx, it.fy, it.u0, it.v0, n1, n2);
      dfk_mm_vertex_normal(n1, n2, nc);
      se3f::quat_rotate(it.q, nc, nw);
      for (int k = 0; k < 3; ++k) o.normals[3 * row + k] = nw[k];
    }
    if (o.colors) {
      uint8_t* c = o.colors + 3 * row;
      // a noisy vertex exists only with draw_noisy_pixels, which paints it (drawkf.geom:64-65)
      if (mesh_pixel(it, p, x, y, d) & DFK_MM_NOISY) {
        c[0] = 255;
        c[1] = 0;
        c[2] = 0;
      } else {
        const uint8_t* src = it.color + (size_t)y * it.color_pitch + 3 * (size_t)x;
        c[0] = src[0];
        c[1] = src[1];
        c[2] = src[2];
      }
    }
    if (o.pixels) o.pixels[row] = y * it.w + x;
  }
  if (o.triangles && ((m.y | m.z) & bit)) {
    long long row = it.t_begin + b.y + __popc(m.y & below) + __popc(m.z & below);
    const int tl = vertex_index(it, segs, bases, x - 1, y), br = vertex_index(it, segs, bases, x, y + 1);
    if (m.y & bit) {
      int32_t* t = o.triangles + 3 * row++;
      t[0] = vertex_index(it, segs, bases, x, y);
      t[1] = tl;
      t[2] = br;
    }
    if (m.z & bit) {
      int32_t* t = o.triangles + 3 * row;
      t[0] = br;
      t[1] = tl;
      t[2] = vertex_index(it, segs, bases, x - 1, y + 1);
    }
  }
}

}  // namespace

cudaError_t launch_keyframe_mesh(const MeshItemDev* items_dev, int n, int max_tiles, const MeshParamsDev& p,
                                 const MeshOutDev& o, uint3* segs, int2* bases, cudaStream_t s)
{
  const dim3 grid((unsigned)max_tiles, (unsigned)n);
  keyframe_mesh_classify_kernel<<<grid, kT, 0, s>>>(items_dev, p, segs);
  keyframe_mesh_scan_kernel<<<n, kT, 0, s>>>(items_dev, segs, bases, o.counts);
  keyframe_mesh_write_kernel<<<grid, kT, 0, s>>>(items_dev, p, o, segs, bases);
  return cudaGetLastError();
}

}  // namespace dfk
