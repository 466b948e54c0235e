/* dfk_mesh_model.h -- the per-element model of dfk_keyframe_mesh_batch (include/dfk.h, DESIGN.md section 4.12): the
 * keyframe renderer's geometry shader (gui/shaders/drawkf.geom) and SaveKeyframes' uint16 depth, in plain C so that the
 * device kernels (dfk_mesh.cu) and a sequential CPU build of the specification compile the same
 * arithmetic.  Both builds run without FMA contraction (nvcc -fmad=false, gcc -ffp-contract=off): every fp32 operation
 * below rounds once, in the order written; sqrtf and the divisions are IEEE (no fast-math on either side).
 *
 *   pixel   validate_pixel / fetch_pixel (drawkf.geom:57-89): depth range, validity, noise and border tests
 *   lift    lift (:36-46): the camera-frame point of a pixel
 *   quad    main (:91-125): crop, the two triangle normals, the slant test, then the triangles (:152-183)
 *   u16     cv::Mat::convertTo(CV_16UC1, 5000) of SaveKeyframes (core/deepfactors.cpp:560)
 */
#ifndef DFK_MESH_MODEL_H_
#define DFK_MESH_MODEL_H_

#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define DFK_MM_FN static __host__ __device__ __forceinline__
#else
#define DFK_MM_FN static inline
#endif

#define DFK_MM_MIN_DEPTH 0.5f /* drawkf.geom:59 */
#define DFK_MM_MAX_DEPTH 10.0f
#define DFK_MM_BORDER 4       /* drawkf.geom:70 */

/* pixel flags */
#define DFK_MM_VALID 1u       /* the pixel may be a triangle corner */
#define DFK_MM_NOISY 2u       /* the noise test holds (with draw_noisy_pixels the pixel stays valid, coloured (255, 0, 0)) */
/* quad flags */
#define DFK_MM_T1 1u          /* T1 = (tr, tl, br) */
#define DFK_MM_T2 2u          /* T2 = (br, tl, bl) */

/* The flags of pixel (x, y) of a W x H keyframe with depth d, validity vld (has_vld = 0: no validity view, every pixel
 * passes) and log-stdev s (has_std = 0: no stdev view, no pixel is noisy).  tau = log(stdev_thresh / sqrt 2) in fp64
 * (-inf for stdev_thresh <= 0): sqrt(2) exp(s) > stdev_thresh decided exactly as (double)s > tau; a NaN s is never
 * noisy.  A NaN depth is invalid (the shader would keep it).  A pixel outside the image is invalid. */
DFK_MM_FN unsigned dfk_mm_pixel(int x, int y, int W, int H, float d, int has_vld, float vld, int has_std, float s,
                                double tau, int draw_noisy)
{
  unsigned f;
  int ok;
  if (x < 0 || y < 0 || x >= W || y >= H) return 0u;
  ok = d >= DFK_MM_MIN_DEPTH && d <= DFK_MM_MAX_DEPTH;
  if (has_vld && !(vld > 0.0f)) ok = 0;
  if (x < DFK_MM_BORDER || x > W - DFK_MM_BORDER || y < DFK_MM_BORDER || y > H - DFK_MM_BORDER) ok = 0;
  f = 0u;
  if (has_std && (double)s > tau) {
    f = DFK_MM_NOISY;
    if (!draw_noisy) ok = 0;
  }
  return ok ? (f | DFK_MM_VALID) : f;
}

/* lift (:36-46): ((x - u0) / fx d, (y - v0) / fy d, d) */
DFK_MM_FN void dfk_mm_lift(int x, int y, float d, float fx, float fy, float u0, float v0, float p[3])
{
  p[0] = (((float)x - u0) / fx) * d;
  p[1] = (((float)y - v0) / fy) * d;
  p[2] = d;
}

/* GLSL normalize: each component over sqrt((v.x v.x + v.y v.y) + v.z v.z) */
DFK_MM_FN void dfk_mm_normalize(float v[3])
{
  const float len = sqrtf((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
  v[0] = v[0] / len;
  v[1] = v[1] / len;
  v[2] = v[2] / len;
}

/* triangle_normal (:29-34): normalize(cross(c - a, b - a)) */
DFK_MM_FN void dfk_mm_tri_normal(const float a[3], const float b[3], const float c[3], float n[3])
{
  const float A0 = c[0] - a[0], A1 = c[1] - a[1], A2 = c[2] - a[2];
  const float B0 = b[0] - a[0], B1 = b[1] - a[1], B2 = b[2] - a[2];
  n[0] = A1 * B2 - A2 * B1;
  n[1] = A2 * B0 - A0 * B2;
  n[2] = A0 * B1 - A1 * B0;
  dfk_mm_normalize(n);
}

/* The camera-frame normals of the quad at (x, y) (:113-120): n1 = n(tr, tl, br), n2 = n(tl, bl, br).  d: the depths of
 * tr = (x, y), tl = (x - 1, y), br = (x, y + 1), bl = (x - 1, y + 1), 0 outside the image. */
DFK_MM_FN void dfk_mm_quad_normals(int x, int y, const float d[4], float fx, float fy, float u0, float v0, float n1[3],
                                   float n2[3])
{
  float tr[3], tl[3], br[3], bl[3];
  dfk_mm_lift(x, y, d[0], fx, fy, u0, v0, tr);
  dfk_mm_lift(x - 1, y, d[1], fx, fy, u0, v0, tl);
  dfk_mm_lift(x, y + 1, d[2], fx, fy, u0, v0, br);
  dfk_mm_lift(x - 1, y + 1, d[3], fx, fy, u0, v0, bl);
  dfk_mm_tri_normal(tr, tl, br, n1);
  dfk_mm_tri_normal(tl, bl, br, n2);
}

/* (n1 + n2) / 2 (:136), before the keyframe's rotation; not renormalised */
DFK_MM_FN void dfk_mm_vertex_normal(const float n1[3], const float n2[3], float n[3])
{
  n[0] = (n1[0] + n2[0]) * 0.5f;
  n[1] = (n1[1] + n2[1]) * 0.5f;
  n[2] = (n1[2] + n2[2]) * 0.5f;
}

/* The triangles of the quad at (x, y) (DFK_MM_T1 | DFK_MM_T2): f and d are the flags and depths of tr, tl, br, bl as in
 * dfk_mm_quad_normals.  The quad is skipped outside the crop (:97-99) and dropped when |n1 . r| < slt or |n2 . r| < slt
 * with r = normalize(((x - u0) / fx, (y - v0) / fy, 1)) (:121-125); a NaN product fails the test and keeps the quad.
 * With slt <= 0 no quad is dropped, so the normals are not computed. */
DFK_MM_FN unsigned dfk_mm_quad(int x, int y, int W, int H, int crop, float slt, const unsigned f[4], const float d[4],
                               float fx, float fy, float u0, float v0)
{
  unsigned t = 0u;
  if (x < crop || x > W - crop || y < crop || y > H - crop) return 0u;
  if ((f[0] & f[1] & f[2]) & DFK_MM_VALID) t |= DFK_MM_T1;
  if ((f[1] & f[2] & f[3]) & DFK_MM_VALID) t |= DFK_MM_T2;
  if (t && slt > 0.0f) {
    float n1[3], n2[3], r[3];
    dfk_mm_quad_normals(x, y, d, fx, fy, u0, v0, n1, n2);
    r[0] = ((float)x - u0) / fx;
    r[1] = ((float)y - v0) / fy;
    r[2] = 1.0f;
    dfk_mm_normalize(r);
    if (fabsf((n1[0] * r[0] + n1[1] * r[1]) + n1[2] * r[2]) < slt) return 0u;
    if (fabsf((n2[0] * r[0] + n2[1] * r[1]) + n2[2] * r[2]) < slt) return 0u;
  }
  return t;
}

/* convertTo(CV_16UC1, 5000): p = d * 5000 in fp32, cvRound (half to even), saturated to [0, 65535].  On x86 cvRound of
 * a NaN or of a value beyond int32 is INT_MIN, which saturates to 0. */
DFK_MM_FN uint16_t dfk_mm_depth_u16(float d)
{
  const float p = d * 5000.0f;
  float r;
  if (!(p < 2147483648.0f)) return 0;
  r = rintf(p);
  return r <= 0.0f ? (uint16_t)0 : (r >= 65535.0f ? (uint16_t)65535 : (uint16_t)r);
}

#endif /* DFK_MESH_MODEL_H_ */
