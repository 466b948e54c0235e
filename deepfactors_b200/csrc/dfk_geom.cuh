// dfk_geom.cuh -- per-pixel warp / sample / Jacobian math shared by every kernel.
//
// Restates, for sm_90a, the per-pixel functions of the reference (file:line into
// jczarnowski/DeepFactors @ bffc78a):
//   FindCorrespondence                 sources/common/algorithm/warping.h:204-241
//   PinholeCamera::Reproject/Project   sources/common/algorithm/pinhole_camera_impl.h:50-56, 39-45
//   PinholeCamera::PixelValid          pinhole_camera_impl.h:102-108
//   FindCorrespondenceJacobianPose     warping.h:247-257 (+ TransformJacobianPose :156-164,
//                                      ProjectPointJacobian pinhole_camera_impl.h:89-97)
//   FindCorrespondenceJacobianPrx      warping.h:275-291 (+ DepthJacobianPrx :44-50)
//   HuberWeight                        sources/common/algorithm/m_estimators.h:50-56
//   Image2DView::getBilinear           VisionCore (not in tree): floor + lerp of lerps
//
// The chain that decides VALIDITY (reproject -> quaternion rotate -> translate -> depth test ->
// project -> border test) is written with round-to-nearest intrinsics in the exact operation
// order of the reference's CPU evaluation (Eigen/Sophus without FMA contraction), so that inlier
// sets are bit-identical to the CPU path -- the reference's own GPU-vs-CPU test demands equal
// inlier counts (tests/ut_sfmaligner.cpp:320).  Everything downstream of the validity decision
// (Jacobians, bilinear weights, Huber) is free to use FMA contraction.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace dfk {

struct Warped {
  bool valid;
  float u, v;          // pix1
  float px, py, pz;    // R * pt        (TransformJacobianPose needs pose.so3() * pt)
  float tx, ty, tz;    // R * pt + t    (Correspondence::tpt)
  float xn, yn;        // normalised ray (ReprojectDepthJacobian)
};

// q = (x,y,z,w) unit quaternion, t translation.  Exact-order restatement, see header comment.
// Reproject's normalised ray coordinate (pinhole_camera_impl.h:54): (p - c) / f, IEEE division.
// It depends only on the column (row), so kernels may tabulate it per item.
__device__ __forceinline__ float ray_coord(float pf, float c, float f) { return __fdiv_rn(__fsub_rn(pf, c), f); }

__device__ __forceinline__ Warped warp_ray(float xn, float yn, float d, const float* __restrict__ q,
                                           const float* __restrict__ t, float fx, float fy, float u0, float v0,
                                           float border, float ulim, float vlim, float min_dpt)
{
  Warped w;
  // Reproject: PointT point((px - u0)/fx, (py - v0)/fy, 1); return point * depth;
  w.xn = xn;
  w.yn = yn;
  const float X0 = __fmul_rn(w.xn, d), X1 = __fmul_rn(w.yn, d), X2 = d;
  // Eigen QuaternionBase::_transformVector: uv = q.vec x v; uv += uv; v + w*uv + q.vec x uv
  float uv0 = __fsub_rn(__fmul_rn(q[1], X2), __fmul_rn(q[2], X1));
  float uv1 = __fsub_rn(__fmul_rn(q[2], X0), __fmul_rn(q[0], X2));
  float uv2 = __fsub_rn(__fmul_rn(q[0], X1), __fmul_rn(q[1], X0));
  uv0 = __fadd_rn(uv0, uv0);
  uv1 = __fadd_rn(uv1, uv1);
  uv2 = __fadd_rn(uv2, uv2);
  const float c0 = __fsub_rn(__fmul_rn(q[1], uv2), __fmul_rn(q[2], uv1));
  const float c1 = __fsub_rn(__fmul_rn(q[2], uv0), __fmul_rn(q[0], uv2));
  const float c2 = __fsub_rn(__fmul_rn(q[0], uv1), __fmul_rn(q[1], uv0));
  w.px = __fadd_rn(__fadd_rn(X0, __fmul_rn(q[3], uv0)), c0);
  w.py = __fadd_rn(__fadd_rn(X1, __fmul_rn(q[3], uv1)), c1);
  w.pz = __fadd_rn(__fadd_rn(X2, __fmul_rn(q[3], uv2)), c2);
  w.tx = __fadd_rn(w.px, t[0]);
  w.ty = __fadd_rn(w.py, t[1]);
  w.tz = __fadd_rn(w.pz, t[2]);
  w.valid = false;
  w.u = 0.f;
  w.v = 0.f;
  if (w.tz > min_dpt) {
    // Project: fx * X / Z + u0
    w.u = __fadd_rn(__fdiv_rn(__fmul_rn(fx, w.tx), w.tz), u0);
    w.v = __fadd_rn(__fdiv_rn(__fmul_rn(fy, w.ty), w.tz), v0);
    w.valid = (w.u >= border) && (w.u < ulim) && (w.v >= border) && (w.v < vlim);
  }
  return w;
}

__device__ __forceinline__ void bilin_setup(float u, float v, int& ix, int& iy, float& fu, float& fv)
{
  const float flu = floorf(u), flv = floorf(v);
  ix = (int)flu;
  iy = (int)flv;
  fu = u - flu;
  fv = v - flv;
}

__device__ __forceinline__ float lerp2(float q00, float q01, float q10, float q11, float fu, float fv)
{
  const float top = fmaf(fu, q01 - q00, q00);
  const float bot = fmaf(fu, q11 - q10, q10);
  return fmaf(fv, bot - top, top);
}

// scalar image sample
__device__ __forceinline__ float sample_scalar(const float* __restrict__ img, uint32_t pitch, int ix, int iy,
                                               float fu, float fv)
{
  const float* r0 = img + (size_t)iy * pitch + ix;
  const float* r1 = r0 + pitch;
  return lerp2(__ldg(r0), __ldg(r0 + 1), __ldg(r1), __ldg(r1 + 1), fu, fv);
}

// (gx,gy)-interleaved image sample
__device__ __forceinline__ void sample_grad(const float* __restrict__ grad, uint32_t pitch, bool aligned8, int ix,
                                            int iy, float fu, float fv, float& gx, float& gy)
{
  const float* r0 = grad + (size_t)iy * pitch + 2 * ix;
  const float* r1 = r0 + pitch;
  float2 g00, g01, g10, g11;
  if (aligned8) {
    g00 = __ldg(reinterpret_cast<const float2*>(r0));
    g01 = __ldg(reinterpret_cast<const float2*>(r0) + 1);
    g10 = __ldg(reinterpret_cast<const float2*>(r1));
    g11 = __ldg(reinterpret_cast<const float2*>(r1) + 1);
  } else {
    g00 = make_float2(__ldg(r0), __ldg(r0 + 1));
    g01 = make_float2(__ldg(r0 + 2), __ldg(r0 + 3));
    g10 = make_float2(__ldg(r1), __ldg(r1 + 1));
    g11 = make_float2(__ldg(r1 + 2), __ldg(r1 + 3));
  }
  gx = lerp2(g00.x, g01.x, g10.x, g11.x, fu, fv);
  gy = lerp2(g00.y, g01.y, g10.y, g11.y, fu, fv);
}

__device__ __forceinline__ Warped warp_pixel(float xf, float yf, float d, const float* __restrict__ q,
                                             const float* __restrict__ t, float fx, float fy, float u0, float v0,
                                             float border, float ulim, float vlim, float min_dpt)
{
  return warp_ray(ray_coord(xf, u0, fx), ray_coord(yf, v0, fy), d, q, t, fx, fy, u0, v0, border, ulim, vlim, min_dpt);
}

// MUFU approximations (1-2 ulp) for everything downstream of the validity decision; the reference's
// own GPU build uses --use_fast_math for all of it (sources/cuda/CMakeLists.txt:6)
__device__ __forceinline__ float fast_rcp(float x)
{
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float fast_sqrt(float x)
{
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// m_estimators.h:50-56
__device__ __forceinline__ float huber_weight(float x, float delta)
{
  const float aa = fabsf(x);
  return aa <= delta ? 1.0f : fast_sqrt(delta * (2.0f * aa - delta)) * fast_rcp(aa);
}

// a[k] = -(gx*A0[k] + gy*A1[k]),  A = dCam * [I | -hat(R pt)]   (warping.h:156-164,247-257)
__device__ __forceinline__ void pose_jacobian_row(const Warped& w, float fx, float fy, float gx, float gy,
                                                  float (&a)[6], float& c00, float& c02, float& c11, float& c12)
{
  const float iz = fast_rcp(w.tz);
  c00 = fx * iz;
  c11 = fy * iz;
  c02 = -(fx * w.tx) * iz * iz;
  c12 = -(fy * w.ty) * iz * iz;
  a[0] = -(gx * c00);
  a[1] = -(gy * c11);
  a[2] = -(gx * c02 + gy * c12);
  a[3] = -(gx * (c02 * w.py) + gy * (c12 * w.py - c11 * w.pz));
  a[4] = -(gx * (c00 * w.pz - c02 * w.px) + gy * (-(c12 * w.px)));
  a[5] = -(gx * (-(c00 * w.py)) + gy * (c11 * w.px));
}

// err_J_prx = -(grad * pix1_J_prx)  (dense_sfm.h:172-174; warping.h:259-291, :44-50)
__device__ __forceinline__ float prx_jacobian(const Warped& w, const float* __restrict__ R, float d, float avg_dpt,
                                              float gx, float gy, float c00, float c02, float c11, float c12)
{
  const float q0 = R[0] * w.xn + R[1] * w.yn + R[2];
  const float q1 = R[3] * w.xn + R[4] * w.yn + R[5];
  const float q2 = R[6] * w.xn + R[7] * w.yn + R[8];
  const float pJx = c00 * q0 + c02 * q2;
  const float pJy = c11 * q1 + c12 * q2;
  // DepthJacobianPrx: prx = avg/(avg+d); -avg/prx^2 == -(avg+d)^2/avg
  const float s = avg_dpt + d;
  const float dJ = -(s * s) * fast_rcp(avg_dpt);
  return -(gx * pJx + gy * pJy) * dJ;
}

// ---------------------------------------------------------------------------------- reductions
__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}


// ---------------------------------------------------------------------------------------------
// Depth decode shared by update_depth_kernel's vector body and the fused RunStep front-ends (DepthFromCode,
// warping.h:30-69).
// The reference leaves the summation order of the 1xC * Cx1 product to Eigen; this library fixes it so that the
// stand-alone UpdateDepth and the fused path agree bit for bit: per float4 chunk a 4-term fma chain starting from 0,
// then an xor-butterfly over the C/4 chunk sums with offsets NV/2, ..., 1 (what a shuffle-xor all-reduce computes; it
// is invariant under xor-relabelling of the chunks, so a front-end may hold chunk (j ^ m) in register j).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float chunk_dot(const float4 v, const float4 c)
{
  float d = fmaf(v.x, c.x, 0.0f);
  d = fmaf(v.y, c.y, d);
  d = fmaf(v.z, c.z, d);
  return fmaf(v.w, c.w, d);
}
template <int NV>
__device__ __forceinline__ float butterfly_sum(float (&p)[NV])
{
#pragma unroll
  for (int o = NV / 2; o > 0; o >>= 1)
#pragma unroll
    for (int j = 0; j < o; ++j) p[j] = __fadd_rn(p[j], p[j + o]);  // pairs (j, j ^ o) of the live prefix
  return p[0];
}
__device__ __forceinline__ float prx_to_depth(float prx, float avg_dpt)
{
  return __fsub_rn(__fdiv_rn(avg_dpt, prx), avg_dpt);  // ProxToDepth warping.h:30-35
}

}  // namespace dfk
