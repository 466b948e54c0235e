// dfk_se3.cuh -- the fp32 relative pose of a work item (warping.h:98-137), one implementation for the host staging of
// every batch (dfk_api.cu, dfk_host.h) and the device re-posing of a window problem (dfk_window_lm.cu).  Both must give the same
// bits: on the device every product and sum is an explicitly rounded __fmul_rn / __fadd_rn / __fsub_rn, so nvcc cannot
// contract a pair into an FMA; the host compiler targets x86-64 without FMA and does not reassociate, so the plain
// operators there round each operation once in the same order.
#pragma once

#include <cuda_runtime.h>

namespace dfk {
namespace se3f {

__host__ __device__ inline float mul(float a, float b)
{
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ inline float add(float a, float b)
{
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ inline float sub(float a, float b)
{
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}

// Eigen QuaternionBase::_transformVector
__host__ __device__ inline void quat_rotate(const float q[4], const float v[3], float out[3])
{
  float uv0 = sub(mul(q[1], v[2]), mul(q[2], v[1]));
  float uv1 = sub(mul(q[2], v[0]), mul(q[0], v[2]));
  float uv2 = sub(mul(q[0], v[1]), mul(q[1], v[0]));
  uv0 = add(uv0, uv0); uv1 = add(uv1, uv1); uv2 = add(uv2, uv2);
  out[0] = add(add(v[0], mul(q[3], uv0)), sub(mul(q[1], uv2), mul(q[2], uv1)));
  out[1] = add(add(v[1], mul(q[3], uv1)), sub(mul(q[2], uv0), mul(q[0], uv2)));
  out[2] = add(add(v[2], mul(q[3], uv2)), sub(mul(q[0], uv1), mul(q[1], uv0)));
}

__host__ __device__ inline void quat_mul(const float a[4], const float b[4], float o[4])
{
  const float w = sub(sub(sub(mul(a[3], b[3]), mul(a[0], b[0])), mul(a[1], b[1])), mul(a[2], b[2]));
  const float x = sub(add(add(mul(a[3], b[0]), mul(a[0], b[3])), mul(a[1], b[2])), mul(a[2], b[1]));
  const float y = sub(add(add(mul(a[3], b[1]), mul(a[1], b[3])), mul(a[2], b[0])), mul(a[0], b[2]));
  const float z = sub(add(add(mul(a[3], b[2]), mul(a[2], b[3])), mul(a[0], b[1])), mul(a[1], b[0]));
  o[0] = x; o[1] = y; o[2] = z; o[3] = w;
}

__host__ __device__ inline void quat_to_matrix(const float q[4], float R[9])
{
  const float tx = mul(2.f, q[0]), ty = mul(2.f, q[1]), tz = mul(2.f, q[2]);
  const float twx = mul(tx, q[3]), twy = mul(ty, q[3]), twz = mul(tz, q[3]);
  const float txx = mul(tx, q[0]), txy = mul(ty, q[0]), txz = mul(tz, q[0]);
  const float tyy = mul(ty, q[1]), tyz = mul(tz, q[1]), tzz = mul(tz, q[2]);
  R[0] = sub(1.f, add(tyy, tzz)); R[1] = sub(txy, twz);         R[2] = add(txz, twy);
  R[3] = add(txy, twz);         R[4] = sub(1.f, add(txx, tzz)); R[5] = sub(tyz, twx);
  R[6] = sub(txz, twy);         R[7] = add(tyz, twx);         R[8] = sub(1.f, add(txx, tyy));
}

// warping.h:98-137 RelativePose(pose_a, pose_b, jac_a, jac_b): pose_ab = a^-1 * b
__host__ __device__ inline void relative_pose(const float a[7], const float b[7], float ab[7], float* jac_a, float* jac_b)
{
  const float qi[4] = {-a[0], -a[1], -a[2], a[3]};
  const float nta[3] = {-a[4], -a[5], -a[6]};
  float ti[3], tmp[3];
  quat_rotate(qi, nta, ti);
  quat_mul(qi, b, ab);
  quat_rotate(qi, b + 4, tmp);
  ab[4] = add(ti[0], tmp[0]); ab[5] = add(ti[1], tmp[1]); ab[6] = add(ti[2], tmp[2]);
  if (!jac_a && !jac_b) return;
  float Ra[9], RaT[9];
  quat_to_matrix(a, Ra);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) RaT[i * 3 + j] = Ra[j * 3 + i];
  if (jac_a) {
    const float d[3] = {sub(a[4], b[4]), sub(a[5], b[5]), sub(a[6], b[6])};
    float v[3];
    for (int i = 0; i < 3; ++i)
      v[i] = add(add(mul(RaT[i * 3 + 0], d[0]), mul(RaT[i * 3 + 1], d[1])), mul(RaT[i * 3 + 2], d[2]));
    const float hat[9] = {0, -v[2], v[1], v[2], 0, -v[0], -v[1], v[0], 0};
    for (int i = 0; i < 36; ++i) jac_a[i] = 0.f;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        float s = 0.f;
        for (int k = 0; k < 3; ++k) s = add(s, mul(hat[i * 3 + k], RaT[k * 3 + j]));
        jac_a[i * 6 + j] = -RaT[i * 3 + j];
        jac_a[i * 6 + 3 + j] = -s;
        jac_a[(3 + i) * 6 + 3 + j] = -RaT[i * 3 + j];
      }
  }
  if (jac_b) {
    for (int i = 0; i < 36; ++i) jac_b[i] = 0.f;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        jac_b[i * 6 + j] = RaT[i * 3 + j];
        jac_b[(3 + i) * 6 + 3 + j] = RaT[i * 3 + j];
      }
  }
}

// RelativePose(pose1, pose0, J_pose1, J_pose0): q, t and R of pose_10 = pose1^-1 * pose0 and both 6x6 Jacobians, into an
// SfmItemDev or a SparsePose
template <class D>
__host__ __device__ inline void set_relative_pose_only(D& d, const float pose1[7], const float pose0[7])
{
  float p10[7];
  relative_pose(pose1, pose0, p10, d.P1, d.P0);
  for (int k = 0; k < 4; ++k) d.q[k] = p10[k];
  for (int k = 0; k < 3; ++k) d.t[k] = p10[4 + k];
  quat_to_matrix(p10, d.R);
}

}  // namespace se3f
}  // namespace dfk
