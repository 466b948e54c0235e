/* dfk_orb_model.h -- the per-point model of dfk_orb_detect_batch (see include/dfk.h and DESIGN.md section 4.9 for the
 * specification): FAST-9 score, Harris response, intensity-centroid orientation (OpenCV's fastAtan2), the rotation of
 * a pattern point and the Gaussian blur of one pixel.  Plain C99, so the same arithmetic builds for the host (a
 * sequential CPU build of the specification checks the kernels) and for the device; both sides compile it without FMA
 * contraction. */
#ifndef DFK_ORB_MODEL_H_
#define DFK_ORB_MODEL_H_

#include <float.h>
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define DFK_OM __host__ __device__ static inline
#else
#define DFK_OM static inline
#endif

#define DFK_OM_EDGE 31         /* edgeThreshold = patchSize: keypoints keep 31 <= x < W - 31, 31 <= y < H - 31 */
#define DFK_OM_MIN_SIZE 63     /* a smaller image has no such position */
#define DFK_OM_HALF_PATCH 15   /* the orientation disc's radius */
#define DFK_OM_HARRIS_BLOCK 7
#define DFK_OM_BLUR_R 3        /* the 7-tap blur */
#define DFK_OM_PATTERN_R 18    /* the largest |rint| coordinate of a rotated pattern point */

/* the 16-pixel Bresenham circle of radius 3, (x, y), in order around it */
DFK_OM int dfk_om_circle_x(int k)
{
  const int cx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
  return cx[k];
}
DFK_OM int dfk_om_circle_y(int k)
{
  const int cy[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
  return cy[k];
}

/* FAST-9 on the centre value c and its circle v[16], threshold t: the score (cv::FAST's cornerScore<16>) if the pixel
 * is a corner, else -1.  s = the largest, over the 16 arcs of 9 contiguous circle pixels and both signs, of the arc's
 * smallest signed difference (v - c for brighter arcs, c - v for darker ones); a corner has s > t, its score is s - 1. */
DFK_OM int dfk_om_fast_score(int c, const int v[16], int t)
{
  /* an arc of 9 holds at least 2 of the 4 compass pixels 0, 4, 8, 12: without 2 of them beyond the threshold on one
   * side there is no corner */
  int nb = 0, nd = 0;
  for (int k = 0; k < 16; k += 4) {
    nb += v[k] > c + t;
    nd += v[k] < c - t;
  }
  if (nb < 2 && nd < 2) return -1;
  int s = -256;
  for (int k = 0; k < 16; ++k) {
    int lo = 255, hi = -255;  /* min and max of v - c over the arc starting at k */
    for (int j = 0; j < 9; ++j) {
      const int d = v[(k + j) & 15] - c;
      lo = d < lo ? d : lo;
      hi = d > hi ? d : hi;
    }
    s = lo > s ? lo : s;
    s = -hi > s ? -hi : s;
  }
  return s > t ? s - 1 : -1;
}

/* Sobel-like derivatives of ORB's HarrisResponses at the centre of the 3 x 3 neighbourhood p (row major) */
DFK_OM int dfk_om_harris_ix(const int p[9]) { return (p[5] - p[3]) * 2 + (p[2] - p[0]) + (p[8] - p[6]); }
DFK_OM int dfk_om_harris_iy(const int p[9]) { return (p[7] - p[1]) * 2 + (p[6] - p[0]) + (p[8] - p[2]); }

/* The Harris response from the 7 x 7 block sums a = sum Ix^2, b = sum Iy^2, c = sum Ix Iy, in fp32 in ORB's order,
 * k = 0.04, scale s = 1 / (4 * 7 * 255) */
DFK_OM float dfk_om_harris_response(int a, int b, int c)
{
  const float harris_k = 0.04f;
  const float scale = 1.f / ((1 << 2) * DFK_OM_HARRIS_BLOCK * 255.f);
  const float scale_sq_sq = scale * scale * scale * scale;
  return ((float)a * (float)b - (float)c * (float)c - harris_k * ((float)a + (float)b) * ((float)a + (float)b)) *
         scale_sq_sq;
}

/* umax[v], v = 0..15: the half width of row v of the orientation disc -- cvRound(sqrt(15^2 - v^2)) for
 * v <= floor(15 sqrt(2) / 2 + 1) = 11, then made symmetric about the diagonal for v >= ceil(15 sqrt(2) / 2) = 11 */
DFK_OM int dfk_om_umax(int v)
{
  const int u[16] = {15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3};
  return u[v];
}

/* cv::fastAtan2(y, x) in degrees, [0, 360): OpenCV's degree-7 odd polynomial, in fp32 */
DFK_OM float dfk_om_fast_atan2(float y, float x)
{
  const float deg = (float)(180 / 3.14159265358979323846);
  const float p1 = 0.9997878412794807f * deg, p3 = -0.3258083974640975f * deg, p5 = 0.1555786518463281f * deg,
              p7 = -0.04432655554792128f * deg;
  const float ax = fabsf(x), ay = fabsf(y);
  float a, c, c2;
  if (ax >= ay) {
    c = ay / (ax + (float)DBL_EPSILON);
    c2 = c * c;
    a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  } else {
    c = ax / (ay + (float)DBL_EPSILON);
    c2 = c * c;
    a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  }
  if (x < 0) a = 180.f - a;
  if (y < 0) a = 360.f - a;
  return a;
}

/* The keypoint angle from the disc's integer moments m01 (sum v I) and m10 (sum u I) */
DFK_OM float dfk_om_angle(int m01, int m10) { return dfk_om_fast_atan2((float)m01, (float)m10); }

/* cos and sin of the angle as the descriptor uses them: theta = angle * (float)(pi / 180), fp32 */
DFK_OM void dfk_om_rotation(float angle, float* a, float* b)
{
  const float theta = angle * (float)(3.14159265358979323846 / 180.f);
  *a = (float)cos((double)theta);
  *b = (float)sin((double)theta);
}

/* The pixel offset of pattern point (px, py) rotated by (a, b) = (cos, sin): rint of the fp32 rotation */
DFK_OM void dfk_om_rotate(int px, int py, float a, float b, int* ix, int* iy)
{
  const float x = (float)px * a - (float)py * b;
  const float y = (float)px * b + (float)py * a;
  *ix = (int)rintf(x);
  *iy = (int)rintf(y);
}

/* The taps of cv::getGaussianKernel(7, 2, CV_64F) */
DFK_OM double dfk_om_gauss_tap(int k)
{
  const double g[7] = {0x1.1f5f62ecc6329p-4, 0x1.0c70fc73ef9b2p-3, 0x1.869471e14678fp-3, 0x1.ba95c068cda51p-3,
                       0x1.869471e14678fp-3, 0x1.0c70fc73ef9b2p-3, 0x1.1f5f62ecc6329p-4};
  return g[k];
}

/* The blurred value of the centre of the 7 x 7 neighbourhood p (row major): the 7-tap row sums, then the 7-tap column
 * sum of them, each accumulated in tap order in fp64, rounded half to even */
DFK_OM int dfk_om_blur(const uint8_t p[49])
{
  double s = 0.0;
  for (int j = 0; j < 7; ++j) {
    double r = 0.0;
    for (int i = 0; i < 7; ++i) r += dfk_om_gauss_tap(i) * (double)p[7 * j + i];
    s += dfk_om_gauss_tap(j) * r;
  }
  return (int)rint(s);
}

/* A key whose unsigned order is the float order of the response (radix select and sort); never 0 */
DFK_OM uint32_t dfk_om_response_key(float r)
{
  union {
    float f;
    uint32_t u;
  } v;
  v.f = r;
  return (v.u & 0x80000000u) ? ~v.u : (v.u | 0x80000000u);
}

#endif  /* DFK_ORB_MODEL_H_ */
