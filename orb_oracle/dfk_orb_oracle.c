/* dfk_orb_oracle.c -- CPU oracle of dfk_orb_detect_batch and dfk_orb_detect_pyramid_batch (include/dfk.h, DESIGN.md
 * section 4.9).
 *
 * TEST INFRASTRUCTURE ONLY.  One image at a time, the eight steps of the specification in order, sequentially:
 *   FAST-9 scores of every pixel, non-maximum suppression, the border, the first cut by FAST score, Harris responses,
 *   the second cut by response, orientation, descriptors, and the output order (response descending, then y, then x).
 * The per-point model is dfk_orb_model.h itself, compiled here by the host compiler without FMA contraction; the device
 * kernels must reproduce this file's output bit for bit, and the CPU tests check it against cv2.ORB. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "dfk_orb_model.h"
#include "dfk_orb_pattern.h"
#include "dfk_orb_pyramid_model.h"

static const int8_t kPattern[DFK_ORB_PATTERN_PAIRS * 4] = {DFK_ORB_PATTERN_DATA};

void dfko_pattern(int32_t* out)
{
  for (int i = 0; i < DFK_ORB_PATTERN_PAIRS * 4; ++i) out[i] = kPattern[i];
}

#define PIX(x, y) ((int)img[(size_t)(y) * (size_t)pitch + (size_t)(x)])

/* FAST score map: score of a corner, -1 elsewhere (and within 3 pixels of the border) */
void dfko_fast_scores(const uint8_t* img, int w, int h, int pitch, int t, int32_t* score)
{
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      int s = -1;
      if (x >= 3 && x < w - 3 && y >= 3 && y < h - 3) {
        int v[16];
        for (int k = 0; k < 16; ++k) v[k] = PIX(x + dfk_om_circle_x(k), y + dfk_om_circle_y(k));
        s = dfk_om_fast_score(PIX(x, y), v, t);
      }
      score[(size_t)y * w + x] = s;
    }
}

float dfko_harris(const uint8_t* img, int pitch, int x, int y)
{
  int a = 0, b = 0, c = 0;
  for (int dy = -3; dy <= 3; ++dy)
    for (int dx = -3; dx <= 3; ++dx) {
      int p[9];
      for (int j = 0; j < 3; ++j)
        for (int i = 0; i < 3; ++i) p[3 * j + i] = PIX(x + dx + i - 1, y + dy + j - 1);
      const int ix = dfk_om_harris_ix(p), iy = dfk_om_harris_iy(p);
      a += ix * ix;
      b += iy * iy;
      c += ix * iy;
    }
  return dfk_om_harris_response(a, b, c);
}

float dfko_angle(const uint8_t* img, int pitch, int x, int y)
{
  int m01 = 0, m10 = 0;
  for (int v = -DFK_OM_HALF_PATCH; v <= DFK_OM_HALF_PATCH; ++v) {
    const int d = dfk_om_umax(v < 0 ? -v : v);
    for (int u = -d; u <= d; ++u) {
      const int val = PIX(x + u, y + v);
      m10 += u * val;
      m01 += v * val;
    }
  }
  return dfk_om_angle(m01, m10);
}

static int blurred(const uint8_t* img, int pitch, int x, int y)
{
  uint8_t p[49];
  for (int j = 0; j < 7; ++j)
    for (int i = 0; i < 7; ++i) p[7 * j + i] = (uint8_t)PIX(x + i - 3, y + j - 3);
  return dfk_om_blur(p);
}

void dfko_descriptor(const uint8_t* img, int pitch, int x, int y, float angle, uint8_t desc[32])
{
  float a, b;
  dfk_om_rotation(angle, &a, &b);
  memset(desc, 0, 32);
  for (int j = 0; j < DFK_ORB_PATTERN_PAIRS; ++j) {
    int x0, y0, x1, y1;
    dfk_om_rotate(kPattern[4 * j], kPattern[4 * j + 1], a, b, &x0, &y0);
    dfk_om_rotate(kPattern[4 * j + 2], kPattern[4 * j + 3], a, b, &x1, &y1);
    const int bit = blurred(img, pitch, x + x0, y + y0) < blurred(img, pitch, x + x1, y + y1);
    desc[j / 8] |= (uint8_t)(bit << (j % 8));
  }
}

typedef struct {
  int x, y, score;
  float r;
} Cand;

/* descending by key, ties in raster order */
static int by_response(const void* pa, const void* pb)
{
  const Cand *a = (const Cand*)pa, *b = (const Cand*)pb;
  if (a->r != b->r) return a->r > b->r ? -1 : 1;
  if (a->y != b->y) return a->y < b->y ? -1 : 1;
  return (a->x > b->x) - (a->x < b->x);
}

/* The detector on one image.  Writes min(count, capacity) rows of keypoints [2], angles, responses and 32-byte
 * descriptors in the output order, and returns the count (-1 if out of memory). */
int dfko_detect(const uint8_t* img, int w, int h, int pitch, int nfeatures, int t, int capacity, float* keypoints,
                float* angles, float* responses, uint8_t* descriptors)
{
  if (w < DFK_OM_MIN_SIZE || h < DFK_OM_MIN_SIZE) return 0;
  int32_t* score = (int32_t*)malloc(sizeof(int32_t) * (size_t)w * h);
  Cand* c = (Cand*)malloc(sizeof(Cand) * (size_t)w * h);
  if (!score || !c) {
    free(score);
    free(c);
    return -1;
  }
  dfko_fast_scores(img, w, h, pitch, t, score);
  /* 1-2: non-maximum suppression (a non-corner neighbour counts as 0) inside the border, in raster order */
  int n = 0;
  for (int y = DFK_OM_EDGE; y < h - DFK_OM_EDGE; ++y)
    for (int x = DFK_OM_EDGE; x < w - DFK_OM_EDGE; ++x) {
      const int s = score[(size_t)y * w + x];
      if (s < 0) continue;
      int keep = 1;
      for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          const int q = score[(size_t)(y + dy) * w + (x + dx)];
          if ((dx || dy) && !(s > (q < 0 ? 0 : q))) keep = 0;
        }
      if (keep) c[n++] = (Cand){x, y, s, 0.0f};
    }
  /* 3: every corner scoring at least the (2 nfeatures)-th largest score */
  if (n > 2 * nfeatures) {
    int hist[256] = {0};
    for (int i = 0; i < n; ++i) ++hist[c[i].score];
    int thr = 255, above = 0;
    while (above + hist[thr] < 2 * nfeatures) above += hist[thr--];
    int m = 0;
    for (int i = 0; i < n; ++i)
      if (c[i].score >= thr) c[m++] = c[i];
    n = m;
  }
  /* 4-5: Harris responses, every candidate responding at least the nfeatures-th largest response */
  for (int i = 0; i < n; ++i) c[i].r = dfko_harris(img, pitch, c[i].x, c[i].y);
  qsort(c, (size_t)n, sizeof(Cand), by_response);
  if (n > nfeatures) {
    const float cut = c[nfeatures - 1].r;
    int m = nfeatures;
    while (m < n && c[m].r >= cut) ++m;
    n = m;
  }
  /* 6-8: orientation and descriptor of each kept keypoint, already in the output order */
  for (int i = 0; i < n && i < capacity; ++i) {
    const float angle = dfko_angle(img, pitch, c[i].x, c[i].y);
    keypoints[2 * i] = (float)c[i].x;
    keypoints[2 * i + 1] = (float)c[i].y;
    if (angles) angles[i] = angle;
    if (responses) responses[i] = c[i].r;
    dfko_descriptor(img, pitch, c[i].x, c[i].y, angle, descriptors + 32 * (size_t)i);
  }
  free(score);
  free(c);
  return n;
}

/* ------------------------------------------------------------------ the scale pyramid (nlevels > 1) */

/* dst (dw x dh, pitch dw) = src (sw x sh) resized as cv::resize(src, (dw, dh), INTER_LINEAR_EXACT) */
void dfko_resize(const uint8_t* src, int sw, int sh, int spitch, uint8_t* dst, int dw, int dh)
{
  for (int y = 0; y < dh; ++y) {
    int oy, cy;
    dfk_opm_tap(y, sh, dh, &oy, &cy);
    const int oy1 = oy + 1 < sh ? oy + 1 : sh - 1;
    for (int x = 0; x < dw; ++x) {
      int ox, cx;
      dfk_opm_tap(x, sw, dw, &ox, &cx);
      const int ox1 = ox + 1 < sw ? ox + 1 : sw - 1;
      const uint8_t* r0 = src + (size_t)oy * spitch;
      const uint8_t* r1 = src + (size_t)oy1 * spitch;
      dst[(size_t)y * dw + x] = (uint8_t)dfk_opm_resize_px(r0[ox], r0[ox1], r1[ox], r1[ox1], cx, cy);
    }
  }
}

void dfko_budgets(int n, float s, int L, int32_t* out)
{
  int b[DFK_OPM_MAX_LEVELS];
  dfk_opm_budgets(n, s, L, b);
  for (int k = 0; k < L; ++k) out[k] = b[k];
}

/* The detector with L levels of scale factor s on one image: level k (made from level k - 1) runs dfko_detect with
 * its budget, its rows follow the levels before it with the keypoints scaled to level 0 and octave k.  Writes
 * min(total, capacity) rows and level_counts[L], and returns the total (-1 if out of memory). */
int dfko_detect_pyramid(const uint8_t* img, int w, int h, int pitch, int nfeatures, float s, int L, int t, int capacity,
                        float* keypoints, float* angles, float* responses, uint8_t* descriptors, int32_t* octaves,
                        int32_t* level_counts)
{
  int budget[DFK_OPM_MAX_LEVELS];
  dfk_opm_budgets(nfeatures, s, L, budget);
  const uint8_t* prev = img;
  int pw = w, ph = h, pp = pitch, total = 0;
  uint8_t* owned = NULL;
  for (int k = 0; k < L; ++k) {
    const float scale = dfk_opm_level_scale(s, k);
    const int lw = k ? dfk_opm_level_size(w, scale) : w, lh = k ? dfk_opm_level_size(h, scale) : h;
    level_counts[k] = 0;
    if (lw < DFK_OM_MIN_SIZE || lh < DFK_OM_MIN_SIZE) continue;  /* and so is every later level */
    if (k) {
      uint8_t* cur = (uint8_t*)malloc((size_t)lw * lh);
      if (!cur) {
        free(owned);
        return -1;
      }
      dfko_resize(prev, pw, ph, pp, cur, lw, lh);
      free(owned);
      owned = cur;
      prev = cur;
      pw = lw;
      ph = lh;
      pp = lw;
    }
    if (budget[k] == 0) continue;
    const int at = total < capacity ? total : capacity;
    const int n = dfko_detect(prev, pw, ph, pp, budget[k], t, capacity - at, keypoints + 2 * (size_t)at,
                              angles ? angles + at : NULL, responses ? responses + at : NULL,
                              descriptors + 32 * (size_t)at);
    if (n < 0) {
      free(owned);
      return -1;
    }
    const int rows = n < capacity - at ? n : capacity - at;
    for (int i = 0; i < rows; ++i) {
      keypoints[2 * (size_t)(at + i)] *= scale;
      keypoints[2 * (size_t)(at + i) + 1] *= scale;
      if (octaves) octaves[at + i] = k;
    }
    level_counts[k] = n;
    total += n;
  }
  free(owned);
  return total;
}
