/* dfk_match_oracle.c -- CPU oracle of dfk_hamming_match_batch / dfk_reprojection_match_batch (include/dfk.h).
 *
 * TEST INFRASTRUCTURE ONLY.  One factor at a time, in the order the specification states it:
 *   matching  brute force over every (query, train) pair, ties to the lowest train index
 *   RANSAC    the sequential adaptive loop, one hypothesis after the other, each scored over every match
 *   pruning   a stable sort by (distance, query index) of the kept inliers
 * The per-hypothesis fp64 model (sample generator, eight-point solve, decomposition, score) is dfk_match_model.h
 * itself, compiled here by the host compiler without FMA contraction: the device kernels must reproduce this file's
 * selection and lists bit for bit, and the CPU tests check the model against synthetic geometry. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "dfk_match_model.h"

static int popcount8(uint8_t x)
{
  int c = 0;
  for (; x; x &= (uint8_t)(x - 1)) ++c;
  return c;
}

/* out[2 q] = train index, out[2 q + 1] = distance; (-1, -1) for an empty train set */
void dfkm_hamming(const uint8_t* d0, int n0, const uint8_t* d1, int n1, int bytes, int32_t* out)
{
  for (int q = 0; q < n0; ++q) {
    int best = -1, best_j = -1;
    for (int j = 0; j < n1; ++j) {
      int d = 0;
      for (int b = 0; b < bytes; ++b) d += popcount8((uint8_t)(d0[(size_t)q * bytes + b] ^ d1[(size_t)j * bytes + b]));
      if (best_j < 0 || d < best) {
        best = d;
        best_j = j;
      }
    }
    out[2 * q] = best_j;
    out[2 * q + 1] = best_j < 0 ? -1 : best;
  }
}

int dfkm_sample(uint64_t seed, int h, int n, int32_t* idx)
{
  int tmp[DFK_MM_SAMPLE];
  const int ok = dfk_mm_sample(seed, h, n, tmp);
  for (int k = 0; k < DFK_MM_SAMPLE; ++k) idx[k] = ok ? tmp[k] : -1;
  return ok;
}

void dfkm_bearing(float u, float v, double fx, double fy, double u0, double v0, double* f)
{
  dfk_mm_bearing(u, v, fx, fy, u0, v0, f);
}

/* f0, f1: 8 x 3 bearings each */
int dfkm_eightpt(const double* f0, const double* f1, double* e)
{
  return dfk_mm_eightpt((const double(*)[3])f0, (const double(*)[3])f1, e);
}

int dfkm_model(const double* f0, const double* f1, double* R, double* t)
{
  return dfk_mm_model((const double(*)[3])f0, (const double(*)[3])f1, R, t);
}

double dfkm_score(const double* R, const double* t, const double* f0, const double* f1)
{
  return dfk_mm_score(R, t, f0, f1);
}

double dfkm_needed(int best, int n, double probability) { return dfk_mm_needed(best, n, probability); }

typedef struct {
  double fx, fy, u0, v0;
  double threshold, probability;
  float max_dist;
  int32_t max_iterations;
  uint64_t seed;
} DfkmParams;

/* inliers of hypothesis h (0 for an invalid one); scores (may be NULL) gets every match's score, NaN when invalid */
static int hypothesis_count(const DfkmParams* p, int h, const float* kp0, int n0, const float* kp1,
                            const int32_t* train, double* scores)
{
  double R[9], t[3];
  const int valid = dfk_mm_hypothesis(p->seed, h, n0, kp0, kp1, train, 1, p->fx, p->fy, p->u0, p->v0, R, t);
  int c = 0;
  for (int q = 0; q < n0; ++q) {
    double f0[3], f1[3], s = NAN;
    if (valid) {
      dfk_mm_bearing(kp0[2 * q], kp0[2 * q + 1], p->fx, p->fy, p->u0, p->v0, f0);
      dfk_mm_bearing(kp1[2 * train[q]], kp1[2 * train[q] + 1], p->fx, p->fy, p->u0, p->v0, f1);
      s = dfk_mm_score(R, t, f0, f1);
      c += s < p->threshold;
    }
    if (scores) scores[q] = s;
  }
  return c;
}

/* counts[h] for h < num: every hypothesis' inlier count, without the adaptive stop */
void dfkm_hypothesis_counts(const DfkmParams* p, const float* kp0, int n0, const float* kp1, const int32_t* train,
                            int num, int32_t* counts)
{
  for (int h = 0; h < num; ++h) counts[h] = n0 < DFK_MM_SAMPLE ? 0 : hypothesis_count(p, h, kp0, n0, kp1, train, NULL);
}

/* The whole factor: matches (n0 x 2, from dfkm_hamming) -> out rows (query, train, distance), returns their number.
 * stats = (selected hypothesis or -1, its inliers, hypotheses evaluated); scores (may be NULL, n0) = every match's
 * score under the selected hypothesis (NaN without one). */
int dfkm_reprojection_match(const DfkmParams* p, const float* kp0, int n0, const float* kp1, int n1,
                            const int32_t* matches, int32_t* out, int32_t* stats, double* scores)
{
  int best = 0, best_h = -1, h = 0;
  int32_t* train = (int32_t*)malloc(sizeof(int32_t) * (size_t)(n0 > 0 ? n0 : 1));
  for (int q = 0; q < n0; ++q) train[q] = matches[2 * q];
  if (n0 >= DFK_MM_SAMPLE && n1 > 0) {
    double k = INFINITY;
    for (h = 0; h < p->max_iterations; ++h) {
      const int c = hypothesis_count(p, h, kp0, n0, kp1, train, NULL);
      if (c > best) {
        best = c;
        best_h = h;
        k = dfk_mm_needed(best, n0, p->probability);
      }
      if ((double)(h + 1) >= k) {
        ++h;
        break;
      }
    }
  }
  stats[0] = best_h;
  stats[1] = best;
  stats[2] = h;
  int num = 0;
  if (best_h >= 0) {
    double* s = (double*)malloc(sizeof(double) * (size_t)n0);
    hypothesis_count(p, best_h, kp0, n0, kp1, train, s);
    for (int q = 0; q < n0; ++q) {
      if (scores) scores[q] = s[q];
      if (s[q] < p->threshold && (float)matches[2 * q + 1] <= p->max_dist) {
        /* insertion into the list sorted by (distance, query): queries arrive in increasing order */
        int pos = num;
        while (pos > 0 && out[3 * (pos - 1) + 2] > matches[2 * q + 1]) {
          memcpy(out + 3 * pos, out + 3 * (pos - 1), 3 * sizeof(int32_t));
          --pos;
        }
        out[3 * pos] = q;
        out[3 * pos + 1] = matches[2 * q];
        out[3 * pos + 2] = matches[2 * q + 1];
        ++num;
      }
    }
    free(s);
  } else if (scores) {
    for (int q = 0; q < n0; ++q) scores[q] = NAN;
  }
  free(train);
  return num;
}
