/* dfk_match_model.h -- the fp64 model of one eight-point RANSAC hypothesis of dfk_reprojection_match_batch (see
 * include/dfk.h for the specification): sample generator, bearing vectors, eight-point essential matrix, its
 * decomposition, cheirality and opengv's score.  Plain C99, so the same arithmetic builds for the host and for the
 * device; both sides compile it without FMA contraction. */
#ifndef DFK_MATCH_MODEL_H_
#define DFK_MATCH_MODEL_H_

#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define DFK_MM __host__ __device__ static inline
#else
#define DFK_MM static inline
#endif

#define DFK_MM_SAMPLE 8
#define DFK_MM_MAX_DRAWS 256 /* draws per hypothesis before it is declared invalid */
#define DFK_MM_GOLDEN 0x9E3779B97F4A7C15ULL

/* splitmix64's finaliser */
DFK_MM uint64_t dfk_mm_mix(uint64_t z)
{
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}

/* The 8 distinct match indices of hypothesis h over n >= 8 matches.  Draw k (k = 0, 1, ...) is
 *   r = mix(mix(seed + G (h + 1)) + G (k + 1)),  index = ((r >> 32) * n) >> 32   (G = 0x9E3779B97F4A7C15, mod 2^64)
 * and an index already drawn is skipped.  Returns 0 (invalid hypothesis) if 8 distinct indices take more than
 * DFK_MM_MAX_DRAWS draws. */
DFK_MM int dfk_mm_sample(uint64_t seed, int h, int n, int idx[DFK_MM_SAMPLE])
{
  const uint64_t key = dfk_mm_mix(seed + DFK_MM_GOLDEN * (uint64_t)(h + 1));
  int got = 0;
  for (int k = 0; k < DFK_MM_MAX_DRAWS && got < DFK_MM_SAMPLE; ++k) {
    const uint64_t r = dfk_mm_mix(key + DFK_MM_GOLDEN * (uint64_t)(k + 1));
    const int i = (int)(((r >> 32) * (uint64_t)n) >> 32);
    int dup = 0;
    for (int j = 0; j < got; ++j) dup |= idx[j] == i;
    if (!dup) idx[got++] = i;
  }
  return got == DFK_MM_SAMPLE;
}

/* normalize([(u - u0) / fx, (v - v0) / fy, 1]): cv::undistortPoints without distortion, then normalized() */
DFK_MM void dfk_mm_bearing(float u, float v, double fx, double fy, double u0, double v0, double f[3])
{
  const double x = ((double)u - u0) / fx, y = ((double)v - v0) / fy;
  const double nrm = sqrt(x * x + y * y + 1.0);
  f[0] = x / nrm;
  f[1] = y / nrm;
  f[2] = 1.0 / nrm;
}

DFK_MM double dfk_mm_dot3(const double a[3], const double b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

DFK_MM void dfk_mm_cross3(const double a[3], const double b[3], double c[3])
{
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

/* Least-squares depths of a correspondence under X1 = R X0 + t: lam0 R f0 + t ~ lam1 f1.  Returns 1 - c^2 with
 * c = (R f0) . f1 (the normal equations' determinant); a = R f0. */
DFK_MM double dfk_mm_depths(const double R[9], const double t[3], const double f0[3], const double f1[3], double a[3],
                            double* lam0, double* lam1)
{
  a[0] = R[0] * f0[0] + R[1] * f0[1] + R[2] * f0[2];
  a[1] = R[3] * f0[0] + R[4] * f0[1] + R[5] * f0[2];
  a[2] = R[6] * f0[0] + R[7] * f0[1] + R[8] * f0[2];
  const double c = dfk_mm_dot3(a, f1), at = dfk_mm_dot3(a, t), bt = dfk_mm_dot3(f1, t);
  const double det = 1.0 - c * c;
  *lam0 = (c * bt - at) / det;
  *lam1 = (bt - c * at) / det;
  return det;
}

/* opengv's measure: the midpoint triangulation P (frame 1) of the correspondence, reprojected into both views as unit
 * vectors, error = (1 - f0 . P0 / |P0|) + (1 - f1 . P1 / |P1|), P0 = R^T (P1 - t).  Near-parallel rays (1 - c^2 < 1e-15)
 * are a point at infinity along ray 0: error = 1 - c.  A NaN error is never an inlier. */
DFK_MM double dfk_mm_score(const double R[9], const double t[3], const double f0[3], const double f1[3])
{
  double a[3], l0, l1;
  const double det = dfk_mm_depths(R, t, f0, f1, a, &l0, &l1);
  if (!(det >= 1e-15)) return 1.0 - dfk_mm_dot3(a, f1);
  double p1[3], d[3], p0[3];
  for (int i = 0; i < 3; ++i) p1[i] = 0.5 * (l0 * a[i] + t[i] + l1 * f1[i]);
  for (int i = 0; i < 3; ++i) d[i] = p1[i] - t[i];
  p0[0] = R[0] * d[0] + R[3] * d[1] + R[6] * d[2];
  p0[1] = R[1] * d[0] + R[4] * d[1] + R[7] * d[2];
  p0[2] = R[2] * d[0] + R[5] * d[1] + R[8] * d[2];
  const double n0 = sqrt(dfk_mm_dot3(p0, p0)), n1 = sqrt(dfk_mm_dot3(p1, p1));
  return (1.0 - dfk_mm_dot3(f0, p0) / n0) + (1.0 - dfk_mm_dot3(f1, p1) / n1);
}

/* Null vector e (|e| = 1) of the 8 x 9 epipolar system, row k = kron(f1_k, f0_k) (f1^T E f0 = 0, E row-major = e), by
 * Householder QR of its transpose: e is the last column of Q.  Returns 0 when the system has rank < 8 (a diagonal
 * entry of R below 1e-10; every row has norm 1). */
DFK_MM int dfk_mm_eightpt(const double f0[DFK_MM_SAMPLE][3], const double f1[DFK_MM_SAMPLE][3], double e[9])
{
  double m[9][DFK_MM_SAMPLE];
  for (int k = 0; k < DFK_MM_SAMPLE; ++k)
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) m[3 * i + j][k] = f1[k][i] * f0[k][j];
  for (int c = 0; c < DFK_MM_SAMPLE; ++c) {
    double s = 0.0;
    for (int r = c; r < 9; ++r) s += m[r][c] * m[r][c];
    const double nx = sqrt(s);
    if (!(nx > 1e-10)) return 0;
    const double alpha = m[c][c] > 0.0 ? -nx : nx;
    /* v = x - alpha e_c, stored over column c; |v|^2 = 2 (|x|^2 - alpha x_c) */
    m[c][c] -= alpha;
    const double vv = 2.0 * (s - alpha * (m[c][c] + alpha));
    for (int k = c + 1; k < DFK_MM_SAMPLE; ++k) {
      double p = 0.0;
      for (int r = c; r < 9; ++r) p += m[r][c] * m[r][k];
      const double f = 2.0 * p / vv;
      for (int r = c; r < 9; ++r) m[r][k] -= f * m[r][c];
    }
    m[c][c] = m[c][c] / sqrt(vv); /* v normalised in place: H_c = I - 2 v v^T */
    for (int r = c + 1; r < 9; ++r) m[r][c] = m[r][c] / sqrt(vv);
  }
  for (int r = 0; r < 9; ++r) e[r] = r == 8 ? 1.0 : 0.0;
  for (int c = DFK_MM_SAMPLE - 1; c >= 0; --c) {
    double p = 0.0;
    for (int r = c; r < 9; ++r) p += m[r][c] * e[r];
    for (int r = c; r < 9; ++r) e[r] -= 2.0 * p * m[r][c];
  }
  return 1;
}

/* Eigen-decomposition of the symmetric 3x3 S (row-major) by cyclic Jacobi, eigenvalues descending into w, eigenvectors
 * into the columns of V (row-major). */
DFK_MM void dfk_mm_eig3(double S[9], double w[3], double V[9])
{
  for (int i = 0; i < 9; ++i) V[i] = (i % 4 == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 32; ++sweep) {
    const double off = S[1] * S[1] + S[2] * S[2] + S[5] * S[5];
    const double diag = S[0] * S[0] + S[4] * S[4] + S[8] * S[8];
    if (!(off > 1e-32 * diag)) break;
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      const double spq = S[3 * p + q];
      if (spq == 0.0) continue;
      const double theta = (S[3 * q + q] - S[3 * p + p]) / (2.0 * spq);
      const double tt = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
      const double c = 1.0 / sqrt(tt * tt + 1.0), s = tt * c;
      for (int k = 0; k < 3; ++k) { /* S <- S J (columns p, q) */
        const double sp = S[3 * k + p], sq = S[3 * k + q];
        S[3 * k + p] = c * sp - s * sq;
        S[3 * k + q] = s * sp + c * sq;
      }
      for (int k = 0; k < 3; ++k) { /* S <- J^T S (rows p, q) */
        const double sp = S[3 * p + k], sq = S[3 * q + k];
        S[3 * p + k] = c * sp - s * sq;
        S[3 * q + k] = s * sp + c * sq;
      }
      for (int k = 0; k < 3; ++k) {
        const double vp = V[3 * k + p], vq = V[3 * k + q];
        V[3 * k + p] = c * vp - s * vq;
        V[3 * k + q] = s * vp + c * vq;
      }
    }
  }
  for (int i = 0; i < 3; ++i) w[i] = S[4 * i];
  for (int i = 0; i < 2; ++i) /* selection sort, descending; ties keep their order */
    for (int j = i + 1; j < 3; ++j)
      if (w[j] > w[i]) {
        double tw = w[i]; w[i] = w[j]; w[j] = tw;
        for (int k = 0; k < 3; ++k) { double tv = V[3 * k + i]; V[3 * k + i] = V[3 * k + j]; V[3 * k + j] = tv; }
      }
}

/* The eight-point model of one sample: E from dfk_mm_eightpt, projected onto the essential manifold
 * (U diag(1, 1, 0) V^T with U, V proper rotations), its four decompositions in the order
 *   (U W V^T, u3), (U W V^T, -u3), (U W^T V^T, u3), (U W^T V^T, -u3),   W = [0 -1 0; 1 0 0; 0 0 1],
 * and the one with the most sample points at positive depth in both views (dfk_mm_depths), ties to the first.
 * X1 = R X0 + t.  Returns 0 (invalid hypothesis) for a rank-deficient system or sigma_2(E)^2 <= 1e-20 sigma_1(E)^2. */
DFK_MM int dfk_mm_model(const double f0[DFK_MM_SAMPLE][3], const double f1[DFK_MM_SAMPLE][3], double R[9], double t[3])
{
  double e[9];
  if (!dfk_mm_eightpt(f0, f1, e)) return 0;
  double S[9], w[3], V[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) S[3 * i + j] = e[i] * e[j] + e[3 + i] * e[3 + j] + e[6 + i] * e[6 + j];
  dfk_mm_eig3(S, w, V);
  if (!(w[1] > 1e-20 * w[0])) return 0;
  double v1[3] = {V[0], V[3], V[6]}, v2[3] = {V[1], V[4], V[7]}, v3[3];
  dfk_mm_cross3(v1, v2, v3);
  double u1[3], u2[3], u3[3];
  for (int i = 0; i < 3; ++i) u1[i] = e[3 * i] * v1[0] + e[3 * i + 1] * v1[1] + e[3 * i + 2] * v1[2];
  for (int i = 0; i < 3; ++i) u2[i] = e[3 * i] * v2[0] + e[3 * i + 1] * v2[1] + e[3 * i + 2] * v2[2];
  const double n1 = sqrt(dfk_mm_dot3(u1, u1));
  for (int i = 0; i < 3; ++i) u1[i] = u1[i] / n1;
  const double p = dfk_mm_dot3(u1, u2);
  for (int i = 0; i < 3; ++i) u2[i] = u2[i] - p * u1[i];
  const double n2 = sqrt(dfk_mm_dot3(u2, u2));
  if (!(n2 > 0.0)) return 0;
  for (int i = 0; i < 3; ++i) u2[i] = u2[i] / n2;
  dfk_mm_cross3(u1, u2, u3);
  /* U W V^T = -u1 v2^T + u2 v1^T + u3 v3^T;  U W^T V^T = u1 v2^T - u2 v1^T + u3 v3^T */
  double Ra[9], Rb[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double s = u3[i] * v3[j];
      Ra[3 * i + j] = (u2[i] * v1[j] - u1[i] * v2[j]) + s;
      Rb[3 * i + j] = (u1[i] * v2[j] - u2[i] * v1[j]) + s;
    }
  int best = -1, best_front = -1;
  for (int cand = 0; cand < 4; ++cand) {
    const double* Rc = cand < 2 ? Ra : Rb;
    const double sg = (cand & 1) ? -1.0 : 1.0;
    const double tc[3] = {sg * u3[0], sg * u3[1], sg * u3[2]};
    int front = 0;
    for (int k = 0; k < DFK_MM_SAMPLE; ++k) {
      double a[3], l0, l1;
      const double det = dfk_mm_depths(Rc, tc, f0[k], f1[k], a, &l0, &l1);
      front += (det >= 1e-15 && l0 > 0.0 && l1 > 0.0) ? 1 : 0;
    }
    if (front > best_front) {
      best_front = front;
      best = cand;
    }
  }
  const double* Rs = best < 2 ? Ra : Rb;
  const double sg = (best & 1) ? -1.0 : 1.0;
  for (int i = 0; i < 9; ++i) R[i] = Rs[i];
  for (int i = 0; i < 3; ++i) t[i] = sg * u3[i];
  return 1;
}

/* The adaptive iteration bound after a new best of `best` inliers out of n: log(1 - p) / log(1 - w^8), w = best / n,
 * with 1 - w^8 clamped to [2^-52, 1 - 2^-52]. */
DFK_MM double dfk_mm_needed(int best, int n, double probability)
{
  const double w = (double)best / (double)n;
  const double w2 = w * w, w4 = w2 * w2;
  double q = 1.0 - w4 * w4;
  const double eps = 2.220446049250313e-16;
  if (q < eps) q = eps;
  if (q > 1.0 - eps) q = 1.0 - eps;
  return log(1.0 - probability) / log(q);
}

/* Model of hypothesis h of a match list: sample, bearings of the sampled matches, eight-point model.  The matches are
 * the queries 0 .. n - 1 of k0 with train index train[q * train_stride]; keypoints are [x, y] pairs. */
DFK_MM int dfk_mm_hypothesis(uint64_t seed, int h, int n, const float* kp0, const float* kp1, const int32_t* train,
                             int train_stride, double fx, double fy, double u0, double v0, double R[9], double t[3])
{
  int idx[DFK_MM_SAMPLE];
  if (!dfk_mm_sample(seed, h, n, idx)) return 0;
  double f0[DFK_MM_SAMPLE][3], f1[DFK_MM_SAMPLE][3];
  for (int k = 0; k < DFK_MM_SAMPLE; ++k) {
    const int q = idx[k], j = train[q * train_stride];
    dfk_mm_bearing(kp0[2 * q], kp0[2 * q + 1], fx, fy, u0, v0, f0[k]);
    dfk_mm_bearing(kp1[2 * j], kp1[2 * j + 1], fx, fy, u0, v0, f1[k]);
  }
  return dfk_mm_model(f0, f1, R, t);
}

#endif /* DFK_MATCH_MODEL_H_ */
