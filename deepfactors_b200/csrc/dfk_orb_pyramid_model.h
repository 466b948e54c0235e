/* dfk_orb_pyramid_model.h -- the pyramid model of dfk_orb_detect_pyramid_batch (see include/dfk.h and DESIGN.md section
 * 4.9): the per-level budgets, scales and sizes of cv::ORB with nlevels > 1, and the uint8 bilinear resize
 * (cv::resize with INTER_LINEAR_EXACT and an explicit output size) that makes level k from level k - 1.  Plain C99, so
 * the same arithmetic builds for the host (a sequential CPU build of the specification checks the kernels; the C ABI
 * plans the levels with it) and for the device; both sides compile it without FMA contraction. */
#ifndef DFK_ORB_PYRAMID_MODEL_H_
#define DFK_ORB_PYRAMID_MODEL_H_

#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define DFK_OPM __host__ __device__ static inline
#else
#define DFK_OPM static inline
#endif

#define DFK_OPM_MAX_LEVELS 16  /* DFK_ORB_MAX_LEVELS */

/* The scale of level k: (float)pow((double)s, k) */
DFK_OPM float dfk_opm_level_scale(float s, int k) { return (float)pow((double)s, (double)k); }

/* One side of level k from the side of level 0 and the level's scale: cvRound((float)size / scale), half to even */
DFK_OPM int dfk_opm_level_size(int size, float scale) { return (int)rintf((float)size / scale); }

/* The feature budget of each of L levels: f = (float)(1 / s), d = n (1 - f) / (1 - (float)f^L) in fp32; levels
 * 0 .. L - 2 get cvRound(d), d *= f after each, and the last level gets max(n - their sum, 0) */
DFK_OPM void dfk_opm_budgets(int n, float s, int L, int* out)
{
  const float f = (float)(1.0 / (double)s);
  float d = (float)n * (1.f - f) / (1.f - (float)pow((double)f, (double)L));
  int sum = 0;
  for (int k = 0; k < L - 1; ++k) {
    out[k] = (int)rintf(d);
    sum += out[k];
    d *= f;
  }
  out[L - 1] = n - sum > 0 ? n - sum : 0;
}

/* The taps of output coordinate d along a side resized from src to dst pixels: the source pixel *o and the weight *c1
 * of pixel *o + 1 in 1/256 (pixel *o weighs 256 - *c1).  In fp64: ratio = dst / src, t = (1 / ratio) (d + 0.5) - 0.5;
 * i = floor(t).  Inside, 0 <= i < src - 1: o = i, c1 = rint((t - i) 256), half to even.  Before the first pixel o = 0,
 * past the last o = src - 1, with c1 = 0. */
DFK_OPM void dfk_opm_tap(int d, int src, int dst, int* o, int* c1)
{
  const double ratio = (double)dst / (double)src;
  const double scale = 1.0 / ratio;
  const double t = scale * ((double)d + 0.5) - 0.5;
  const double i = floor(t);
  if (i >= 0.0 && src > 1 && i < (double)(src - 1)) {
    *o = (int)i;
    *c1 = (int)rint((t - i) * 256.0);
  } else {
    *o = i < 0.0 ? 0 : src - 1;
    *c1 = 0;
  }
}

/* One output pixel from its four sources (p00, p01 on the upper row, p10, p11 on the lower) and the taps' weights cx,
 * cy: the row sums keep their 8 fractional bits, the column sum of them is rounded once, half up, from 16 */
DFK_OPM int dfk_opm_resize_px(int p00, int p01, int p10, int p11, int cx, int cy)
{
  const int h0 = p00 * (256 - cx) + p01 * cx, h1 = p10 * (256 - cx) + p11 * cx;
  return (h0 * (256 - cy) + h1 * cy + (1 << 15)) >> 16;
}

#endif  /* DFK_ORB_PYRAMID_MODEL_H_ */
