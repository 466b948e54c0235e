/* dfk_mesh_oracle.c -- CPU oracle of dfk_keyframe_mesh_batch (TEST INFRASTRUCTURE ONLY).
 *
 * One keyframe at a time, sequentially: the per-element model of deepfactors_b200/csrc/dfk_mesh_model.h pixel by pixel
 * and quad by quad, then the vertices and triangles in row-major order by plain counting, where the device uses tiles,
 * masks and scans.  It takes a decoded depth: the tests check the device's fused decode against dfk_update_depth_batch.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "dfk_mesh_model.h"

/* Eigen's QuaternionBase::_transformVector, as dfk_se3.cuh's quat_rotate computes it (q = (x, y, z, w)) */
static void quat_rotate(const float q[4], const float v[3], float out[3])
{
  float uv0 = q[1] * v[2] - q[2] * v[1];
  float uv1 = q[2] * v[0] - q[0] * v[2];
  float uv2 = q[0] * v[1] - q[1] * v[0];
  uv0 = uv0 + uv0;
  uv1 = uv1 + uv1;
  uv2 = uv2 + uv2;
  out[0] = (v[0] + q[3] * uv0) + (q[1] * uv2 - q[2] * uv1);
  out[1] = (v[1] + q[3] * uv1) + (q[2] * uv0 - q[0] * uv2);
  out[2] = (v[2] + q[3] * uv2) + (q[0] * uv1 - q[1] * uv0);
}

/* the noise test's threshold: log(stdev_thresh / sqrt 2) in fp64, -inf for stdev_thresh <= 0 */
double dfkm_tau(float stdev_thresh)
{
  return stdev_thresh > 0.0f ? log((double)stdev_thresh / sqrt(2.0)) : -INFINITY;
}

void dfkm_depth_u16(const float* d, long long n, uint16_t* out)
{
  for (long long i = 0; i < n; ++i) out[i] = dfk_mm_depth_u16(d[i]);
}

/* One keyframe of W x H pixels, row-major arrays: dpt, std (NULL: none), vld (NULL: none), color uint8 x 3 (NULL:
 * none).  cam = (fx, fy, u0, v0), pose = pose_wk.  Writes counts = (vertices, triangles); when both fit vcap and tcap,
 * the rows (each output may be NULL) as dfk_keyframe_mesh_batch writes them; depth_u16 (may be NULL) likewise.
 * Returns 0 when out of memory. */
int dfkm_mesh(int W, int H, const float* dpt, const float* std, const float* vld, const uint8_t* color,
              const float* cam, const float* pose, float stdev_thresh, float slt, int crop, int draw_noisy, int vcap,
              int tcap, float* positions, float* normals, uint8_t* colors, int32_t* pixels, int32_t* triangles,
              uint16_t* depth_u16, int32_t* counts)
{
  const size_t N = (size_t)W * H;
  const double tau = dfkm_tau(stdev_thresh);
  const float fx = cam[0], fy = cam[1], u0 = cam[2], v0 = cam[3];
  unsigned char* pf = (unsigned char*)malloc(N);
  unsigned char* qf = (unsigned char*)malloc(N);
  int32_t* vid = (int32_t*)malloc(sizeof(int32_t) * N);
  if (!pf || !qf || !vid) {
    free(pf);
    free(qf);
    free(vid);
    return 0;
  }
#define DEPTH(x, y) (((x) < 0 || (y) < 0 || (x) >= W || (y) >= H) ? 0.0f : dpt[(size_t)(y) * W + (x)])
#define FLAGS(x, y) (((x) < 0 || (y) < 0 || (x) >= W || (y) >= H) ? 0u : (unsigned)pf[(size_t)(y) * W + (x)])
#define QUAD(x, y) (((x) < 0 || (y) < 0 || (x) >= W || (y) >= H) ? 0u : (unsigned)qf[(size_t)(y) * W + (x)])
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const size_t i = (size_t)y * W + x;
      pf[i] = (unsigned char)dfk_mm_pixel(x, y, W, H, dpt[i], vld != NULL, vld ? vld[i] : 0.0f, std != NULL,
                                          std ? std[i] : 0.0f, tau, draw_noisy);
    }
  /* quads at every pixel (a quad at x = W or y = -1 has a corner outside the image and emits nothing) */
  long long nt = 0;
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const unsigned f[4] = {FLAGS(x, y), FLAGS(x - 1, y), FLAGS(x, y + 1), FLAGS(x - 1, y + 1)};
      const float d[4] = {DEPTH(x, y), DEPTH(x - 1, y), DEPTH(x, y + 1), DEPTH(x - 1, y + 1)};
      const unsigned t = dfk_mm_quad(x, y, W, H, crop, slt, f, d, fx, fy, u0, v0);
      qf[(size_t)y * W + x] = (unsigned char)t;
      nt += (t & DFK_MM_T1 ? 1 : 0) + (t & DFK_MM_T2 ? 1 : 0);
    }
  long long nv = 0;
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const int v = (QUAD(x, y) & DFK_MM_T1) || ((QUAD(x + 1, y) | QUAD(x, y - 1)) & (DFK_MM_T1 | DFK_MM_T2)) ||
                    (QUAD(x + 1, y - 1) & DFK_MM_T2);
      vid[(size_t)y * W + x] = v ? (int32_t)nv++ : -1;
    }
  counts[0] = (int32_t)nv;
  counts[1] = (int32_t)nt;
  if (nv <= vcap && nt <= tcap) {
    if (depth_u16) dfkm_depth_u16(dpt, (long long)N, depth_u16);
    long long row = 0;
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        const size_t i = (size_t)y * W + x;
        const int32_t r = vid[i];
        if (r >= 0) {
          float p[3], pw[3];
          dfk_mm_lift(x, y, dpt[i], fx, fy, u0, v0, p);
          quat_rotate(pose, p, pw);
          for (int k = 0; k < 3; ++k) {
            if (positions) positions[3 * (size_t)r + k] = pw[k] + pose[4 + k];
          }
          if (normals) {
            const float d[4] = {DEPTH(x, y), DEPTH(x - 1, y), DEPTH(x, y + 1), DEPTH(x - 1, y + 1)};
            float n1[3], n2[3], nc[3];
            dfk_mm_quad_normals(x, y, d, fx, fy, u0, v0, n1, n2);
            dfk_mm_vertex_normal(n1, n2, nc);
            quat_rotate(pose, nc, normals + 3 * (size_t)r);
          }
          if (colors) {
            const int noisy = (pf[i] & DFK_MM_NOISY) != 0;
            for (int k = 0; k < 3; ++k) colors[3 * (size_t)r + k] = noisy ? (k == 0 ? 255 : 0) : color[3 * i + k];
          }
          if (pixels) pixels[r] = (int32_t)i;
        }
        const unsigned t = qf[i];
        if (triangles && (t & DFK_MM_T1)) {
          triangles[3 * row + 0] = vid[i];
          triangles[3 * row + 1] = vid[i - 1];
          triangles[3 * row + 2] = vid[i + W];
          row += 1;
        }
        if (triangles && (t & DFK_MM_T2)) {
          triangles[3 * row + 0] = vid[i + W];
          triangles[3 * row + 1] = vid[i - 1];
          triangles[3 * row + 2] = vid[i + W - 1];
          row += 1;
        }
      }
  }
#undef DEPTH
#undef FLAGS
#undef QUAD
  free(pf);
  free(qf);
  free(vid);
  return 1;
}
