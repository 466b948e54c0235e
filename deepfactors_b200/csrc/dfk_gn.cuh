// dfk_gn.cuh -- the 6x6 Gauss-Newton update of the device-side tracking loop (dfk_se3_track), host + device so that
// the CPU tests can run the very same code.
#pragma once

#include <cuda_runtime.h>
#include <math.h>

#if defined(__CUDA_ARCH__)
#define DFK_UNROLL _Pragma("unroll")
#else
#define DFK_UNROLL
#endif

namespace dfk {

// ------------------------------------------------------------------------------ on-device Gauss-Newton update
// camera_tracker.cpp:59-63: update = -JtJ.ldlt().solve(Jtr); translation += update.head<3>();
// so3 = SO3::exp(update.tail<3>()) * so3.  Eigen's LDLT is a robust Cholesky with symmetric (diagonal) pivoting that
// still returns a solution for semi-definite / ill-conditioned systems: pivots not larger than the smallest normal
// float contribute nothing (Eigen's LDLT::solve zeroes those components).  Same here, so a rank-deficient level moves
// the pose where the reference moves it, and an all-zero system gives a zero step.  (The quaternion is still
// renormalised; a tracker iteration without inliers skips this update altogether, se3_track_update in dfk_simple.cu.)
__host__ __device__ inline void ldlt6_solve(float A[6][6] /* full symmetric, destroyed */, const float b[6], float x[6])
{
  // Every array index below is a compile-time constant after unrolling (the pivot swap is a chain of predicated static
  // swaps), so the 6x6 system lives in registers.  (A version with run-time row / column indices gave wrong updates
  // inside se3_step_kernel while the same code was right in a stand-alone kernel.)
  int perm[6];
DFK_UNROLL
  for (int i = 0; i < 6; ++i) perm[i] = i;
DFK_UNROLL
  for (int k = 0; k < 6; ++k) {
    int p = k;
    float best = fabsf(A[k][k]);
DFK_UNROLL
    for (int i = k + 1; i < 6; ++i)
      if (fabsf(A[i][i]) > best) {
        best = fabsf(A[i][i]);
        p = i;
      }
    // P A P^T: rows k <-> p (the finished L columns and the trailing block), then columns k <-> p
DFK_UNROLL
    for (int i = k + 1; i < 6; ++i) {
      if (p == i) {
DFK_UNROLL
        for (int c = 0; c < 6; ++c) { const float t = A[k][c]; A[k][c] = A[i][c]; A[i][c] = t; }
DFK_UNROLL
        for (int r = 0; r < 6; ++r) { const float t = A[r][k]; A[r][k] = A[r][i]; A[r][i] = t; }
        const int t = perm[k]; perm[k] = perm[i]; perm[i] = t;
      }
    }
    const float d = A[k][k];
    if (fabsf(d) > 1.17549435e-38f) {
      float col[6];
DFK_UNROLL
      for (int i = k + 1; i < 6; ++i) col[i] = A[i][k] / d;  // L_ik
DFK_UNROLL
      for (int i = k + 1; i < 6; ++i)
DFK_UNROLL
        for (int j = k + 1; j < 6; ++j) A[i][j] -= col[i] * A[j][k];  // A[j][k] still holds L_jk * d
DFK_UNROLL
      for (int i = k + 1; i < 6; ++i) A[i][k] = col[i];
    } else {
DFK_UNROLL
      for (int i = k + 1; i < 6; ++i) A[i][k] = 0.0f;
    }
  }
  float y[6];
DFK_UNROLL
  for (int i = 0; i < 6; ++i) {
    float v = 0.0f;
DFK_UNROLL
    for (int j = 0; j < 6; ++j)
      if (perm[i] == j) v = b[j];
    y[i] = v;
  }
DFK_UNROLL
  for (int i = 0; i < 6; ++i)
DFK_UNROLL
    for (int k = 0; k < i; ++k) y[i] -= A[i][k] * y[k];
DFK_UNROLL
  for (int i = 0; i < 6; ++i) y[i] = fabsf(A[i][i]) > 1.17549435e-38f ? y[i] / A[i][i] : 0.0f;
DFK_UNROLL
  for (int i = 5; i >= 0; --i)
DFK_UNROLL
    for (int k = i + 1; k < 6; ++k) y[i] -= A[k][i] * y[k];
DFK_UNROLL
  for (int j = 0; j < 6; ++j) {
    float v = 0.0f;
DFK_UNROLL
    for (int i = 0; i < 6; ++i)
      if (perm[i] == j) v = y[i];
    x[j] = v;
  }
}

__host__ __device__ inline bool gn_update_pose(const float* __restrict__ sys /*21 JtJ packed upper, 6 Jtr*/, float* pose /*qx qy qz qw tx ty tz*/)
{
  float A[6][6], b[6];
  int h = 0;
  for (int r = 0; r < 6; ++r)
    for (int c = r; c < 6; ++c) {
      A[r][c] = sys[h];
      A[c][r] = sys[h];
      ++h;
    }
  for (int r = 0; r < 6; ++r) b[r] = -sys[21 + r];
  float x[6];
  ldlt6_solve(A, b, x);
  // Sophus SO3::exp (quaternion form) and left multiplication, then renormalisation
  const float th2 = x[3] * x[3] + x[4] * x[4] + x[5] * x[5];
  const float th = sqrtf(th2);
  float im, re;
  if (th < 1e-10f) {
    im = 0.5f - th2 * (1.0f / 48.0f) + th2 * th2 * (1.0f / 3840.0f);
    re = 1.0f - 0.5f * th2 + th2 * th2 * (1.0f / 384.0f);
  } else {
    im = sinf(0.5f * th) / th;
    re = cosf(0.5f * th);
  }
  const float ax = im * x[3], ay = im * x[4], az = im * x[5], aw = re;
  const float bx = pose[0], by = pose[1], bz = pose[2], bw = pose[3];
  float qx = aw * bx + ax * bw + ay * bz - az * by;
  float qy = aw * by - ax * bz + ay * bw + az * bx;
  float qz = aw * bz + ax * by - ay * bx + az * bw;
  float qw = aw * bw - ax * bx - ay * by - az * bz;
  const float n = sqrtf(qx * qx + qy * qy + qz * qz + qw * qw);
  pose[0] = qx / n; pose[1] = qy / n; pose[2] = qz / n; pose[3] = qw / n;
  pose[4] += x[0]; pose[5] += x[1]; pose[6] += x[2];
  return true;
}


}  // namespace dfk
