/* dfk_preprocess_model.h -- the per-pixel model of dfk_preprocess_batch (include/dfk.h, DESIGN.md section 4.10), in
 * plain C so that the device kernels (dfk_preprocess.cu) and a sequential CPU build of the specification compile the
 * same arithmetic.  Both builds run without FMA contraction (nvcc -fmad=false, gcc -ffp-contract=off): every fp32 and fp64
 * operation below rounds once, in the order written.
 *
 *   map    cv::initUndistortRectifyMap(K_in, no distortion, R = I, K_out, size, CV_32FC1)
 *   table  cv::remap's INTER_LINEAR weight table (INTER_BITS = 5, INTER_REMAP_COEF_SCALE = 32768)
 *   taps   cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of a uint8 3-channel image
 *   gray   cv::cvtColor(COLOR_RGB2GRAY) on 8U
 *   float  convertTo(CV_32FC1, 1 / 255.0)
 */
#ifndef DFK_PREPROCESS_MODEL_H_
#define DFK_PREPROCESS_MODEL_H_

#include <math.h>
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define DFK_PM_FN static __host__ __device__ __forceinline__
#else
#define DFK_PM_FN static inline
#endif

#define DFK_PM_TAB_BITS 5          /* INTER_BITS: 32 sub-pixel positions per axis */
#define DFK_PM_TAB_SIZE 32
#define DFK_PM_COEF_SCALE 32768    /* INTER_REMAP_COEF_SCALE = 1 << 15 */

/* the map of one (source camera, output camera) pair: iR = K_out^-1 and the source intrinsics, fp64 */
typedef struct {
  double ir[9];
  double fx, fy, u0, v0;
} DfkPmMap;

/* cv::Mat::inv(DECOMP_LU) of a 3 x 3 fp64 matrix: the closed form of cv::invert for n = 3 (det3, then the adjugate
 * times 1 / det, each entry rounded in this order).  Returns 0 for a singular matrix (out untouched). */
DFK_PM_FN int dfk_pm_inv3(const double* m, double* out)
{
#define DFK_PM_M(i, j) m[3 * (i) + (j)]
  double d = DFK_PM_M(0, 0) * (DFK_PM_M(1, 1) * DFK_PM_M(2, 2) - DFK_PM_M(1, 2) * DFK_PM_M(2, 1)) -
             DFK_PM_M(0, 1) * (DFK_PM_M(1, 0) * DFK_PM_M(2, 2) - DFK_PM_M(1, 2) * DFK_PM_M(2, 0)) +
             DFK_PM_M(0, 2) * (DFK_PM_M(1, 0) * DFK_PM_M(2, 1) - DFK_PM_M(1, 1) * DFK_PM_M(2, 0));
  if (d == 0.0) return 0;
  d = 1.0 / d;
  out[0] = (DFK_PM_M(1, 1) * DFK_PM_M(2, 2) - DFK_PM_M(1, 2) * DFK_PM_M(2, 1)) * d;
  out[1] = (DFK_PM_M(0, 2) * DFK_PM_M(2, 1) - DFK_PM_M(0, 1) * DFK_PM_M(2, 2)) * d;
  out[2] = (DFK_PM_M(0, 1) * DFK_PM_M(1, 2) - DFK_PM_M(0, 2) * DFK_PM_M(1, 1)) * d;
  out[3] = (DFK_PM_M(1, 2) * DFK_PM_M(2, 0) - DFK_PM_M(1, 0) * DFK_PM_M(2, 2)) * d;
  out[4] = (DFK_PM_M(0, 0) * DFK_PM_M(2, 2) - DFK_PM_M(0, 2) * DFK_PM_M(2, 0)) * d;
  out[5] = (DFK_PM_M(0, 2) * DFK_PM_M(1, 0) - DFK_PM_M(0, 0) * DFK_PM_M(1, 2)) * d;
  out[6] = (DFK_PM_M(1, 0) * DFK_PM_M(2, 1) - DFK_PM_M(1, 1) * DFK_PM_M(2, 0)) * d;
  out[7] = (DFK_PM_M(0, 1) * DFK_PM_M(2, 0) - DFK_PM_M(0, 0) * DFK_PM_M(2, 1)) * d;
  out[8] = (DFK_PM_M(0, 0) * DFK_PM_M(1, 1) - DFK_PM_M(0, 1) * DFK_PM_M(1, 0)) * d;
#undef DFK_PM_M
  return 1;
}

/* The map of a source camera (fx, fy, u0, v0 at the source's size) and an output camera, their fp32 values widened to
 * fp64.  Returns 0 when K_out is singular (fx or fy of the output camera is 0). */
DFK_PM_FN int dfk_pm_map_init(DfkPmMap* m, float in_fx, float in_fy, float in_u0, float in_v0, float out_fx,
                              float out_fy, float out_u0, float out_v0)
{
  const double k[9] = {(double)out_fx, 0.0, (double)out_u0, 0.0, (double)out_fy, (double)out_v0, 0.0, 0.0, 1.0};
  m->fx = (double)in_fx;
  m->fy = (double)in_fy;
  m->u0 = (double)in_u0;
  m->v0 = (double)in_v0;
  return dfk_pm_inv3(k, m->ir);
}

/* map1 / map2 of output pixel (j, r): x = (r iR01 + iR02) + j iR00 (likewise y, w), u = (float)(fx (x (1 / w)) + u0) */
DFK_PM_FN void dfk_pm_map(const DfkPmMap* m, int j, int r, float* u, float* v)
{
  const double* ir = m->ir;
  const double dj = (double)j, dr = (double)r;
  const double x = (dr * ir[1] + ir[2]) + dj * ir[0];
  const double y = (dr * ir[4] + ir[5]) + dj * ir[3];
  const double w = (dr * ir[7] + ir[8]) + dj * ir[6];
  const double iw = 1.0 / w;
  *u = (float)(m->fx * (x * iw) + m->u0);
  *v = (float)(m->fy * (y * iw) + m->v0);
}

/* cvRound of an fp32 value into int, saturated: rint (half to even), INT_MIN / INT_MAX past the range */
DFK_PM_FN int dfk_pm_round_sat(float p)
{
  if (p >= 2147483648.0f) return 2147483647;
  if (!(p >= -2147483648.0f)) return -2147483647 - 1;
  return (int)rintf(p);
}

/* the fixed-point coordinate of a map value: X = rint(u * 32), integer part X >> 5, sub-pixel position X & 31 */
DFK_PM_FN int dfk_pm_fixed(float u) { return dfk_pm_round_sat(u * (float)DFK_PM_TAB_SIZE); }

/* The four weights of sub-pixel position (tx, ty), taps (0,0), (0,1), (1,0), (1,1) as (dy, dx): OpenCV's
 * initInterTab2D for INTER_LINEAR.  Returns 1 when the sum needed the fix-up to 32768 (never, for bilinear: the
 * tests check the whole table). */
DFK_PM_FN int dfk_pm_weights(int tx, int ty, int* w)
{
  /* scalars rather than an array indexed by data (the first largest / smallest tap), so that the device keeps them in
   * registers */
  const float fx = (float)tx * (1.0f / (float)DFK_PM_TAB_SIZE), fy = (float)ty * (1.0f / (float)DFK_PM_TAB_SIZE);
  const float sc = (float)DFK_PM_COEF_SCALE;
  int w0 = dfk_pm_round_sat(((1.0f - fy) * (1.0f - fx)) * sc), w1 = dfk_pm_round_sat(((1.0f - fy) * fx) * sc);
  int w2 = dfk_pm_round_sat((fy * (1.0f - fx)) * sc), w3 = dfk_pm_round_sat((fy * fx) * sc);
  const int d = w0 + w1 + w2 + w3 - DFK_PM_COEF_SCALE;
  int fired = 0;
  if (d != 0) {
    int big = 0, small = 0, wb = w0, ws = w0;
    if (w1 > wb) { big = 1; wb = w1; }
    if (w1 < ws) { small = 1; ws = w1; }
    if (w2 > wb) { big = 2; wb = w2; }
    if (w2 < ws) { small = 2; ws = w2; }
    if (w3 > wb) { big = 3; wb = w3; }
    if (w3 < ws) { small = 3; ws = w3; }
    const int fix = d < 0 ? big : small;
    w0 -= fix == 0 ? d : 0;
    w1 -= fix == 1 ? d : 0;
    w2 -= fix == 2 ? d : 0;
    w3 -= fix == 3 ? d : 0;
    fired = 1;
  }
  w[0] = w0;
  w[1] = w1;
  w[2] = w2;
  w[3] = w3;
  return fired;
}

/* Output pixel (j, r) of cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of a uint8 3-channel interleaved source of
 * sw x sh pixels, row pitch `pitch` bytes: out[c] = clamp((sum_k w_k src(x0 + dx, y0 + dy)[c] + 2^14) >> 15, 0, 255),
 * a tap outside the source reads 0. */
DFK_PM_FN void dfk_pm_remap_pixel(const DfkPmMap* m, const uint8_t* src, size_t pitch, int sw, int sh, int j, int r,
                                  uint8_t* out)
{
  float u, v;
  dfk_pm_map(m, j, r, &u, &v);
  const int X = dfk_pm_fixed(u), Y = dfk_pm_fixed(v);
  const int x0 = X >> DFK_PM_TAB_BITS, y0 = Y >> DFK_PM_TAB_BITS;
  int w[4];
  dfk_pm_weights(X & (DFK_PM_TAB_SIZE - 1), Y & (DFK_PM_TAB_SIZE - 1), w);
  int s[3] = {0, 0, 0};
  for (int k = 0; k < 4; ++k) {
    const int x = x0 + (k & 1), y = y0 + (k >> 1);
    if (x < 0 || y < 0 || x >= sw || y >= sh) continue;
    const uint8_t* p = src + (size_t)y * pitch + 3 * (size_t)x;
    for (int c = 0; c < 3; ++c) s[c] += w[k] * (int)p[c];
  }
  for (int c = 0; c < 3; ++c) {
    const int o = (s[c] + (1 << 14)) >> 15;
    out[c] = (uint8_t)(o < 0 ? 0 : (o > 255 ? 255 : o));
  }
}

/* COLOR_RGB2GRAY on 8U: channel 0 takes the R weight */
DFK_PM_FN uint8_t dfk_pm_gray(const uint8_t* c)
{
  return (uint8_t)((9798 * (int)c[0] + 19235 * (int)c[1] + 3735 * (int)c[2] + (1 << 14)) >> 15);
}

/* convertTo(CV_32FC1, 1 / 255.0): one fp32 product */
DFK_PM_FN float dfk_pm_float(uint8_t g) { return (float)g * (float)(1.0 / 255.0); }

/* the optional normalisation of a frame from its sums s1 = sum f, s2 = sum f^2 (fp64) over n pixels: mu = s1 / n,
 * sigma = sqrt(max(s2 / n - mu^2, 0)) */
DFK_PM_FN void dfk_pm_stats(double s1, double s2, double n, double* mu, double* sigma)
{
  const double m = s1 / n;
  const double var = s2 / n - m * m;
  *mu = m;
  *sigma = sqrt(var > 0.0 ? var : 0.0);
}

/* f' = (float)(((double)f - mu) / sigma) */
DFK_PM_FN float dfk_pm_normalize(float f, double mu, double sigma) { return (float)(((double)f - mu) / sigma); }

/* The fixed summation order of the sums: the output is cut into tiles of DFK_PM_TILE_W x DFK_PM_TILE_H pixels in
 * row-major tile order; the 256 values of a tile (pixel t = ty * 32 + tx, 0 outside the image) are summed by a
 * pairwise tree, t += t + 128, then t + 64, ..., t + 1; the tiles' sums are summed by thread t of 256 sequentially over
 * tiles t, t + 256, ..., and those 256 sums by the same tree. */
#define DFK_PM_TILE_W 32
#define DFK_PM_TILE_H 8
#define DFK_PM_TREE 256

#endif /* DFK_PREPROCESS_MODEL_H_ */
