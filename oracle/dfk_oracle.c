/*
 * dfk_oracle.c -- CPU restatement of the DeepFactors dense-alignment hot path.
 * TEST INFRASTRUCTURE ONLY; PARITY UNPINNED (see dfk_oracle.h for both statements).
 * Build: make -C oracle   (gcc -O2 -ffp-contract=off, no -march flags so that no
 * FMA contraction can change the validity chain's rounding).
 * Citations are into /root/reference (jczarnowski/DeepFactors @ bffc78a).
 */
#include "dfk_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include <time.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* ------------------------------------------------------------------ float flavour */
#define REAL float
#define ACC float
#define SUF(name) name##_f
#define SQRT_ sqrtf
#define SIN_ sinf
#define COS_ cosf
#define FLOOR_ floorf
#define FABS_ fabsf
#include "dfk_oracle_impl.inc"
#undef REAL
#undef ACC
#undef SUF
#undef SQRT_
#undef SIN_
#undef COS_
#undef FLOOR_
#undef FABS_

/* ------------------------------------------------------------------ double flavour */
#define REAL double
#define ACC double
#define SUF(name) name##_d
#define SQRT_ sqrt
#define SIN_ sin
#define COS_ cos
#define FLOOR_ floor
#define FABS_ fabs
#include "dfk_oracle_impl.inc"
#undef REAL
#undef ACC
#undef SUF
#undef SQRT_
#undef SIN_
#undef COS_
#undef FLOOR_
#undef FABS_

void dfko_probe_pixel_d(double x, double y, double dpt, const DfkoCamera* cam, const double pose[7],
                        int border, double min_dpt, double avg_dpt, double out[17])
{
  dfko_probe_pixel_impl_d(x, y, dpt, cam, pose, border, min_dpt, avg_dpt, out);
}

/* ------------------------------------------------------------------ OpenMP CPU baseline */
int dfko_omp_max_threads(void)
{
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

/* Row-major, rows split statically over threads, per-thread float accumulators summed in
 * thread order: the "cpu_omp" baseline of BASELINE.md section 2.  Same per-pixel function
 * as dfko_sfm_run_step_f. */
void dfko_sfm_run_step_f_omp(const float pose0[7], const float pose1[7], int code_size,
                             const DfkoCamera* camf, int width, int height,
                             const float* img0, size_t img0_pitch, const float* img1, size_t img1_pitch,
                             const float* dpt0, size_t dpt0_pitch, float* valid0, size_t valid0_pitch,
                             const float* prx0_jac, size_t jac_pitch, const float* grad1, size_t grad1_pitch,
                             const DfkoSfmParams* prm, int nthreads,
                             float* JtJ, float* Jtr, float* residual, uint64_t* inliers)
{
  float p10[7], P0[36], P1[36];
  dfko_relative_pose_f(pose1, pose0, p10, P1, P0);
  const Cam_f cam = cam_cast_f(camf);
  const int NP = 12 + code_size;
  const int NH = NP * (NP + 1) / 2;
  int nt = nthreads > 0 ? nthreads : dfko_omp_max_threads();
  if (nt > height) nt = height;
  float* scratch = (float*)calloc((size_t)nt * (NH + NP + 2), sizeof(float));
  uint64_t* inl = (uint64_t*)calloc((size_t)nt, sizeof(uint64_t));
#ifdef _OPENMP
#pragma omp parallel for num_threads(nt) schedule(static, 1)
#endif
  for (int t = 0; t < nt; ++t) {
    SfmAcc_f acc;
    acc.C = code_size; acc.NP = NP;
    acc.JtJ = scratch + (size_t)t * (NH + NP + 2);
    acc.Jtr = acc.JtJ + NH;
    acc.residual = 0; acc.inliers = 0;
    acc.rows = NULL; acc.width = width; acc.y_begin = 0;
    const int y0 = (int)((long)height * t / nt), y1 = (int)((long)height * (t + 1) / nt);
    sfm_run_rows_f(y0, y1, 1, p10, P0, P1, code_size, &cam, width, img0, img0_pitch, img1, img1_pitch,
                   dpt0, dpt0_pitch, valid0, valid0_pitch, prx0_jac, jac_pitch, grad1, grad1_pitch, prm, &acc);
    acc.Jtr[NP] = acc.residual;
    inl[t] = acc.inliers;
  }
  for (int i = 0; i < NH; ++i) JtJ[i] = 0;
  for (int i = 0; i < NP; ++i) Jtr[i] = 0;
  *residual = 0; *inliers = 0;
  for (int t = 0; t < nt; ++t) {
    const float* s = scratch + (size_t)t * (NH + NP + 2);
    for (int i = 0; i < NH; ++i) JtJ[i] += s[i];
    for (int i = 0; i < NP; ++i) Jtr[i] += s[NH + i];
    *residual += s[NH + NP];
    *inliers += inl[t];
  }
  free(scratch);
  free(inl);
}

/* ------------------------------------------------------------------ throughput-mode CPU baseline (pthreads) */
typedef struct {
  int evals, loop_order, code_size, nlevels;
  const float* pose0;
  const float* pose1;
  const DfkoLevel* levels;
  const DfkoSfmParams* prm;
  float* rec;  /* NH + NP + 2, thread-private */
  double t_end;
} ThroughputJob;

static double now_s(void)
{
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

static void* throughput_worker(void* arg)
{
  ThroughputJob* j = (ThroughputJob*)arg;
  const int NP = 12 + j->code_size, NH = NP * (NP + 1) / 2;
  for (int e = 0; e < j->evals; ++e)
    for (int l = j->nlevels - 1; l >= 0; --l) { /* level 0 last: its record stays in rec */
      const DfkoLevel* L = &j->levels[l];
      uint64_t inl = 0;
      dfko_sfm_run_step_f(j->pose0, j->pose1, j->code_size, &L->cam, L->width, L->height, L->img0, L->img0_pitch,
                          L->img1, L->img1_pitch, L->dpt0, L->dpt0_pitch, NULL, 0, L->prx0_jac, L->jac_pitch,
                          L->grad1, L->grad1_pitch, j->prm, j->loop_order, j->rec, j->rec + NH, j->rec + NH + NP, &inl);
      j->rec[NH + NP + 1] = (float)inl;
    }
  j->t_end = now_s();
  return NULL;
}

double dfko_sfm_throughput_f(int nthreads, int evals_per_thread, int loop_order, const float pose0[7],
                             const float pose1[7], int code_size, int nlevels, const DfkoLevel* levels,
                             const DfkoSfmParams* params, float* rec_out)
{
  if (nthreads < 1) nthreads = 1;
  const int NP = 12 + code_size, NH = NP * (NP + 1) / 2, REC = NH + NP + 2;
  ThroughputJob* jobs = (ThroughputJob*)calloc((size_t)nthreads, sizeof(ThroughputJob));
  pthread_t* th = (pthread_t*)calloc((size_t)nthreads, sizeof(pthread_t));
  float* recs = (float*)calloc((size_t)nthreads * REC, sizeof(float));
  const double t0 = now_s();
  for (int t = 0; t < nthreads; ++t) {
    jobs[t].evals = evals_per_thread; jobs[t].loop_order = loop_order; jobs[t].code_size = code_size;
    jobs[t].nlevels = nlevels; jobs[t].pose0 = pose0; jobs[t].pose1 = pose1; jobs[t].levels = levels;
    jobs[t].prm = params; jobs[t].rec = recs + (size_t)t * REC; jobs[t].t_end = t0;
    if (pthread_create(&th[t], NULL, throughput_worker, &jobs[t]) != 0) { /* run it here instead */
      throughput_worker(&jobs[t]);
      th[t] = 0;
    }
  }
  double t1 = t0;
  for (int t = 0; t < nthreads; ++t) {
    if (th[t]) pthread_join(th[t], NULL);
    if (jobs[t].t_end > t1) t1 = jobs[t].t_end;
  }
  if (rec_out) memcpy(rec_out, recs, sizeof(float) * REC);
  free(recs); free(th); free(jobs);
  return t1 - t0;
}

/* ------------------------------------------------------------------ UpdateDepth
 * cu_image_proc.cpp:248-264 kernel_update_depth -> warping.h:62-69 DepthFromCode ->
 * :52-59 ProxFromCode (prx_0code + prx_J_cde . code) -> :30-35 ProxToDepth (avg/prx - avg) */
void dfko_update_depth_f(const float* code, int code_size, int width, int height,
                         const float* prx_orig, size_t prx_pitch, const float* prx_jac, size_t jac_pitch,
                         float avg_dpt, float* dpt_out, size_t dpt_pitch)
{
  for (int y = 0; y < height; ++y)
    for (int x = 0; x < width; ++x) {
      const float* jc = prx_jac + (size_t)y * jac_pitch + (size_t)x * code_size;
      float dot = 0.0f;
      for (int k = 0; k < code_size; ++k) dot += jc[k] * code[k];
      const float prx = prx_orig[(size_t)y * prx_pitch + x] + dot;
      dpt_out[(size_t)y * dpt_pitch + x] = avg_dpt / prx - avg_dpt;
    }
}

/* ------------------------------------------------------------------ Sobel (cu_image_proc.cpp:57-92)
 * kx = [[-1,0,1],[-2,0,2],[-1,0,1]], ky = kx^T, clamped border, sum over py outer / px inner, /8 */
static inline int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

void dfko_sobel_gradients_f(int width, int height, const float* img, size_t img_pitch,
                            float* grad, size_t grad_pitch)
{
  static const float kx[3][3] = {{-1, 0, 1}, {-2, 0, 2}, {-1, 0, 1}};
  static const float ky[3][3] = {{-1, -2, -1}, {0, 0, 0}, {1, 2, 1}};
  for (int y = 0; y < height; ++y)
    for (int x = 0; x < width; ++x) {
      float sdx = 0.0f, sdy = 0.0f;
      for (int py = -1; py <= 1; ++py)
        for (int px = -1; px <= 1; ++px) {
          const float pix = img[(size_t)clampi(y + py, 0, height - 1) * img_pitch + clampi(x + px, 0, width - 1)];
          sdx += pix * kx[1 + py][1 + px];
          sdy += pix * ky[1 + py][1 + px];
        }
      grad[(size_t)y * grad_pitch + 2 * x + 0] = sdx / 8;
      grad[(size_t)y * grad_pitch + 2 * x + 1] = sdy / 8;
    }
}

/* ------------------------------------------------------------------ blur-down (cu_image_proc.cpp:134-164)
 * 5x5 binomial, sample at clamp(2x+px-2), clamp(2y+py-2), loop py outer / px inner, kernel(px,py),
 * normalised by the running sum `wall` (=256). */
void dfko_gaussian_blur_down_f(int in_width, int in_height, const float* in, size_t in_pitch,
                               int out_width, int out_height, float* out, size_t out_pitch)
{
  static const float k1[5] = {1, 4, 6, 4, 1};
  for (int y = 0; y < out_height; ++y)
    for (int x = 0; x < out_width; ++x) {
      float sum = 0.0f, wall = 0.0f;
      for (int py = 0; py < 5; ++py)
        for (int px = 0; px < 5; ++px) {
          const int nx = clampi(2 * x + px - 2, 0, in_width - 1);
          const int ny = clampi(2 * y + py - 2, 0, in_height - 1);
          const float kv = k1[px] * k1[py];
          sum += in[(size_t)ny * in_pitch + nx] * kv;
          wall += kv;
        }
      out[(size_t)y * out_pitch + x] = sum / wall;
    }
}

/* ------------------------------------------------------------------ SquaredError (cu_image_proc.cpp:190-206) */
float dfko_squared_error_f(int width, int height, const float* a, size_t a_pitch, const float* b, size_t b_pitch)
{
  float sum = 0.0f;
  for (int y = 0; y < height; ++y)
    for (int x = 0; x < width; ++x) {
      const float d = a[(size_t)y * a_pitch + x] - b[(size_t)y * b_pitch + x];
      sum += d * d;
    }
  return sum;
}

double dfko_squared_error_d(int width, int height, const float* a, size_t a_pitch, const float* b, size_t b_pitch)
{
  double sum = 0.0;
  for (int y = 0; y < height; ++y)
    for (int x = 0; x < width; ++x) {
      const double d = (double)a[(size_t)y * a_pitch + x] - (double)b[(size_t)y * b_pitch + x];
      sum += d * d;
    }
  return sum;
}
