/* dfk_preprocess_oracle.c -- CPU oracle of dfk_preprocess_batch (TEST INFRASTRUCTURE ONLY).
 *
 * Runs the per-pixel model of deepfactors_b200/csrc/dfk_preprocess_model.h pixel by pixel, and the normalisation's
 * sums in the fixed order that header documents, written out sequentially here rather than as the device's tiles of
 * threads.  The pyramid is not here: tests take it from the SfM oracle's blur-down and Sobel.
 */
#include <stdint.h>
#include <stdlib.h>

#include "dfk_preprocess_model.h"

static int map_of(const float* in_cam, const float* out_cam, DfkPmMap* m)
{
  return dfk_pm_map_init(m, in_cam[0], in_cam[1], in_cam[2], in_cam[3], out_cam[0], out_cam[1], out_cam[2],
                         out_cam[3]);
}

/* map1 / map2 (float [h, w] each) of cv::initUndistortRectifyMap(..., CV_32FC1); cams are (fx, fy, u0, v0).  Returns 0
 * for a singular output camera. */
int dfkp_map(const float* in_cam, const float* out_cam, int w, int h, float* map1, float* map2)
{
  DfkPmMap m;
  if (!map_of(in_cam, out_cam, &m)) return 0;
  for (int r = 0; r < h; ++r)
    for (int j = 0; j < w; ++j) dfk_pm_map(&m, j, r, map1 + (size_t)r * w + j, map2 + (size_t)r * w + j);
  return 1;
}

/* iR = K_out^-1 (9 doubles, row-major) */
int dfkp_inverse(const float* out_cam, double* ir)
{
  DfkPmMap m;
  const float zero[4] = {1.0f, 1.0f, 0.0f, 0.0f};
  if (!map_of(zero, out_cam, &m)) return 0;
  for (int k = 0; k < 9; ++k) ir[k] = m.ir[k];
  return 1;
}

/* the weight table: tab[(ty * 32 + tx) * 4 + k]; returns the number of entries whose sum needed the fix-up */
int dfkp_weights(int32_t* tab)
{
  int fired = 0;
  for (int ty = 0; ty < DFK_PM_TAB_SIZE; ++ty)
    for (int tx = 0; tx < DFK_PM_TAB_SIZE; ++tx) fired += dfk_pm_weights(tx, ty, tab + (ty * DFK_PM_TAB_SIZE + tx) * 4);
  return fired;
}

/* Steps 1-6 of one frame: src uint8 [sh, pitch] (3 channels interleaved), outputs (any may be NULL) color uint8
 * [h, w, 3], gray uint8 [h, w], f float [h, w].  Returns 0 for a singular output camera. */
int dfkp_preprocess(const uint8_t* src, size_t pitch, int sw, int sh, const float* in_cam, const float* out_cam, int w,
                    int h, uint8_t* color, uint8_t* gray, float* f)
{
  DfkPmMap m;
  if (!map_of(in_cam, out_cam, &m)) return 0;
  for (int r = 0; r < h; ++r)
    for (int j = 0; j < w; ++j) {
      uint8_t c[3];
      dfk_pm_remap_pixel(&m, src, pitch, sw, sh, j, r, c);
      const size_t i = (size_t)r * w + j;
      if (color) {
        color[3 * i] = c[0];
        color[3 * i + 1] = c[1];
        color[3 * i + 2] = c[2];
      }
      const uint8_t g = dfk_pm_gray(c);
      if (gray) gray[i] = g;
      if (f) f[i] = dfk_pm_float(g);
    }
  return 1;
}

static void tree(double* a)
{
  for (int stride = DFK_PM_TREE / 2; stride > 0; stride >>= 1)
    for (int t = 0; t < stride; ++t) a[t] = a[t] + a[t + stride];
}

/* (mu, sigma) of f [h, w] from its sums in the fixed order, and f' in place when normalize != 0.  Returns 0 when out of
 * memory. */
int dfkp_normalize(float* f, int w, int h, int normalize, double* stats)
{
  const int tiles_x = (w + DFK_PM_TILE_W - 1) / DFK_PM_TILE_W, tiles_y = (h + DFK_PM_TILE_H - 1) / DFK_PM_TILE_H;
  const int tiles = tiles_x * tiles_y;
  double* part = (double*)malloc(sizeof(double) * 2 * (size_t)tiles);
  if (!part) return 0;
  double a[DFK_PM_TREE], b[DFK_PM_TREE];
  for (int k = 0; k < tiles; ++k) {
    const int ty = k / tiles_x, tx = k - ty * tiles_x;
    for (int t = 0; t < DFK_PM_TREE; ++t) {
      const int j = tx * DFK_PM_TILE_W + t % DFK_PM_TILE_W, r = ty * DFK_PM_TILE_H + t / DFK_PM_TILE_W;
      const double v = (j < w && r < h) ? (double)f[(size_t)r * w + j] : 0.0;
      a[t] = v;
      b[t] = v * v;
    }
    tree(a);
    tree(b);
    part[2 * k] = a[0];
    part[2 * k + 1] = b[0];
  }
  for (int t = 0; t < DFK_PM_TREE; ++t) {
    a[t] = 0.0;
    b[t] = 0.0;
    for (int k = t; k < tiles; k += DFK_PM_TREE) {
      a[t] = a[t] + part[2 * k];
      b[t] = b[t] + part[2 * k + 1];
    }
  }
  free(part);
  tree(a);
  tree(b);
  dfk_pm_stats(a[0], b[0], (double)w * (double)h, &stats[0], &stats[1]);
  if (normalize)
    for (size_t i = 0; i < (size_t)w * h; ++i) f[i] = dfk_pm_normalize(f[i], stats[0], stats[1]);
  return 1;
}
