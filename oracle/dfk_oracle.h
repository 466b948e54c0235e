/*
 * dfk_oracle.h -- CPU restatement of the DeepFactors dense-alignment hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product:
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * `--impl reference` legs may load this library, and only as the checker (or
 * as the timed CPU baseline), never as the thing shipped.
 *
 * PARITY UNPINNED.  The reference (jczarnowski/DeepFactors @ bffc78a) cannot be
 * compiled here: its per-pixel math is header templates over Eigen, Sophus and
 * VisionCore, none of which are vendored (all thirdparty/ submodule
 * directories are empty) or installed.  The reference ships no golden vectors
 * for this path either (tests are relational: GPU == CPU, analytic == finite
 * difference, optimisation converges).  This file therefore restates the
 * algorithm from the reference sources, and restates the arithmetic that lives
 * in the absent third-party deps from their published behaviour:
 *   - VisionCore (jczarnowski/vision_core @ 924c5333): Image2DView::getBilinear
 *     (floor, lerp of rows iy/iy+1 at ix/ix+1, no clamping), packed upper
 *     triangular matrix, grid-stride reductions.
 *   - Sophus (strasdat/Sophus @ d0b7315a): SE3 * point = unit-quaternion rotate
 *     (Eigen QuaternionBase::_transformVector) + translate; SO3::exp; inverse.
 *   - Eigen (libeigen/eigen @ deb93ed1): fixed-size products.
 * The oracle is pinned against what the reference's own tests pin: the
 * finite-difference identities (ut_warping, ut_sfmaligner), the SE3 alignment
 * convergence KAT on data/testimg/1047|1052 (ut_se3aligner.cpp:173-211), and
 * OpenCV for Sobel / blur-down (ut_cuda_utils.cpp).  See tests/test_oracle_*.py.
 *
 * Every entry point exists in two arithmetic flavours:
 *   *_f : float accumulation, reference loop order (x outer, y inner) -- the
 *         "reference-like" CPU path of tests/ut_sfmaligner.cpp:303-315.
 *   *_d : double arithmetic on the same fp32 inputs -- the truth used to state
 *         the fp32 tolerance of the CUDA kernels.
 *
 * Conventions (all follow the reference):
 *   pose      float[7] = Sophus::SE3f::data() order: quaternion (x,y,z,w), then
 *             translation (x,y,z).
 *   images    row-major, `pitch` counted in ELEMENTS of the scalar type
 *             (floats), pixel (x,y) at ptr[y*pitch + x]; grad1 holds (gx,gy)
 *             interleaved, pixel (x,y) at ptr[y*pitch + 2x]; prx_jac holds C
 *             contiguous floats per pixel at ptr[y*pitch + x*C]
 *             (sources/core/mapping/keyframe.h:52, dense_sfm.h:150).
 *   JtJ       packed upper triangle, row major: (i,j), i<=j, at
 *             i*NP - i*(i-1)/2 + (j-i).  Column order [pose0 t,w | pose1 t,w |
 *             code] (dense_sfm.h:163-177).
 */
#ifndef DFK_ORACLE_H_
#define DFK_ORACLE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* df::PinholeCamera<float>  (sources/common/algorithm/pinhole_camera.h:43) */
typedef struct {
  float fx, fy, u0, v0;
  float width, height; /* Scalars in the reference too */
} DfkoCamera;

/* df::DenseSfmParams (sources/common/algorithm/dense_sfm.h:36-43) */
typedef struct {
  float huber_delta;
  float ocl_th; /* unused by the reference */
  float avg_dpt;
  float min_dpt;
  int valid_border;
} DfkoSfmParams;

/* ---- SE3 helpers (host side of RunStep; warping.h:98-137, testing_utils.h:72-88) */
void dfko_so3_exp_f(const float omega[3], float q[4]);
void dfko_so3_exp_d(const double omega[3], double q[4]);
void dfko_pose_perturb_f(const float pose[7], int idx, float eps, float out[7]);
void dfko_pose_perturb_d(const double pose[7], int idx, double eps, double out[7]);
/* pose_ab = a^-1 * b ; jac_a, jac_b are 6x6 row-major (may be NULL) */
void dfko_relative_pose_f(const float a[7], const float b[7], float ab[7], float jac_a[36], float jac_b[36]);
void dfko_relative_pose_d(const double a[7], const double b[7], double ab[7], double jac_a[36], double jac_b[36]);

/* ---- per-pixel probe: FindCorrespondence + Jacobians for one pixel, used by the
 * finite-difference tests of ut_warping / ut_sfmaligner.  out[0]=valid, out[1..2]=pix1,
 * out[3..14]=corresp_J_pose (2x6 row major), out[15..16]=pix1_J_prx */
void dfko_probe_pixel_d(double x, double y, double dpt, const DfkoCamera* cam, const double pose[7],
                        int border, double min_dpt, double avg_dpt, double out[17]);

/* ---- SfmAligner::RunStep equivalent (cu_sfmaligner.cpp:149-185 + dense_sfm.h:133-201).
 * loop_order: 0 = x outer / y inner (ut_sfmaligner.cpp:303-315), 1 = row major.
 * JtJ: NP(NP+1)/2, Jtr: NP, NP = 12+code_size.  valid0 is in/out (only set to 1). */
void dfko_sfm_run_step_f(const float pose0[7], const float pose1[7], int code_size,
                         const DfkoCamera* cam, int width, int height,
                         const float* img0, size_t img0_pitch, const float* img1, size_t img1_pitch,
                         const float* dpt0, size_t dpt0_pitch, float* valid0, size_t valid0_pitch,
                         const float* prx0_jac, size_t jac_pitch, const float* grad1, size_t grad1_pitch,
                         const DfkoSfmParams* params, int loop_order,
                         float* JtJ, float* Jtr, float* residual, uint64_t* inliers);
void dfko_sfm_run_step_d(const float pose0[7], const float pose1[7], int code_size,
                         const DfkoCamera* cam, int width, int height,
                         const float* img0, size_t img0_pitch, const float* img1, size_t img1_pitch,
                         const float* dpt0, size_t dpt0_pitch, float* valid0, size_t valid0_pitch,
                         const float* prx0_jac, size_t jac_pitch, const float* grad1, size_t grad1_pitch,
                         const DfkoSfmParams* params, int loop_order,
                         double* JtJ, double* Jtr, double* residual, uint64_t* inliers);
/* The per-pixel rows the two entry points above sum, for image rows y_begin .. y_end-1: pixel (x, y) writes its
 * Huber-weighted row [J (NP) | w*diff] at rows[((y - y_begin) * width + x) * (NP + 1)]; rows of invalid pixels are
 * zero.  Same per-pixel function, so the rows summed in one precision give that precision's JtJ / Jtr up to the
 * summation order.  valid0 as above (full image, only rows in the range are touched). */
void dfko_sfm_pixel_rows_f(const float pose0[7], const float pose1[7], int code_size,
                           const DfkoCamera* cam, int width, int height,
                           const float* img0, size_t img0_pitch, const float* img1, size_t img1_pitch,
                           const float* dpt0, size_t dpt0_pitch, float* valid0, size_t valid0_pitch,
                           const float* prx0_jac, size_t jac_pitch, const float* grad1, size_t grad1_pitch,
                           const DfkoSfmParams* params, int y_begin, int y_end,
                           float* rows, float* residual, uint64_t* inliers);
void dfko_sfm_pixel_rows_d(const float pose0[7], const float pose1[7], int code_size,
                           const DfkoCamera* cam, int width, int height,
                           const float* img0, size_t img0_pitch, const float* img1, size_t img1_pitch,
                           const float* dpt0, size_t dpt0_pitch, float* valid0, size_t valid0_pitch,
                           const float* prx0_jac, size_t jac_pitch, const float* grad1, size_t grad1_pitch,
                           const DfkoSfmParams* params, int y_begin, int y_end,
                           double* rows, double* residual, uint64_t* inliers);
/* OpenMP row-major variant of the _f path: the multi-threaded CPU baseline. nthreads<=0 => all. */
void dfko_sfm_run_step_f_omp(const float pose0[7], const float pose1[7], int code_size,
                             const DfkoCamera* cam, int width, int height,
                             const float* img0, size_t img0_pitch, const float* img1, size_t img1_pitch,
                             const float* dpt0, size_t dpt0_pitch, float* valid0, size_t valid0_pitch,
                             const float* prx0_jac, size_t jac_pitch, const float* grad1, size_t grad1_pitch,
                             const DfkoSfmParams* params, int nthreads,
                             float* JtJ, float* Jtr, float* residual, uint64_t* inliers);
int dfko_omp_max_threads(void);

/* ---- CPU baseline in THROUGHPUT mode: `nthreads` POSIX threads, each evaluating the whole pyramid of one pair
 * (`nlevels` RunStep calls, single-threaded, exactly dfko_sfm_run_step_f) `evals_per_thread` times on the same
 * read-only inputs.  No OpenMP, no shared state: what N host cores can do with the reference's (single-threaded) CPU
 * path.  Returns the wall time in seconds of the slowest thread (start of the first -> end of the last);
 * rec_out (may be NULL) receives thread 0's last result for level 0: [JtJ | Jtr | residual | inliers-as-float]. */
typedef struct {
  DfkoCamera cam;
  int width, height;
  const float* img0; size_t img0_pitch;
  const float* img1; size_t img1_pitch;
  const float* dpt0; size_t dpt0_pitch;
  const float* prx0_jac; size_t jac_pitch;
  const float* grad1; size_t grad1_pitch;
} DfkoLevel;
double dfko_sfm_throughput_f(int nthreads, int evals_per_thread, int loop_order, const float pose0[7],
                             const float pose1[7], int code_size, int nlevels, const DfkoLevel* levels,
                             const DfkoSfmParams* params, float* rec_out);

/* ---- SfmAligner::EvaluateError (cu_sfmaligner.cpp:120-147 + dense_sfm.h:79-119):
 * border 1 / min_dpt 0 defaults of FindCorrespondence, Huber-weighted sum of squares. */
void dfko_sfm_evaluate_error_f(const float pose0[7], const float pose1[7], const DfkoCamera* cam,
                               int width, int height, const float* img0, size_t img0_pitch,
                               const float* img1, size_t img1_pitch, const float* dpt0, size_t dpt0_pitch,
                               const DfkoSfmParams* params, float* residual, uint64_t* inliers);
void dfko_sfm_evaluate_error_d(const float pose0[7], const float pose1[7], const DfkoCamera* cam,
                               int width, int height, const float* img0, size_t img0_pitch,
                               const float* img1, size_t img1_pitch, const float* dpt0, size_t dpt0_pitch,
                               const DfkoSfmParams* params, double* residual, uint64_t* inliers);

/* ---- SE3Aligner::RunStep (cu_se3aligner.cpp:153-176 + lucas_kanade_se3.h:41-77). NP = 6. */
void dfko_se3_run_step_f(const float se3[7], const DfkoCamera* cam, int width, int height,
                         const float* img0, size_t img0_pitch, const float* img1, size_t img1_pitch,
                         const float* dpt0, size_t dpt0_pitch, const float* grad1, size_t grad1_pitch,
                         float huber_delta, float* JtJ /*21*/, float* Jtr /*6*/, float* residual, uint64_t* inliers);
void dfko_se3_run_step_d(const float se3[7], const DfkoCamera* cam, int width, int height,
                         const float* img0, size_t img0_pitch, const float* img1, size_t img1_pitch,
                         const float* dpt0, size_t dpt0_pitch, const float* grad1, size_t grad1_pitch,
                         float huber_delta, double* JtJ, double* Jtr, double* residual, uint64_t* inliers);
/* Its fp64 per-pixel rows [J (6) | w*diff] for image rows y_begin .. y_end-1: pixel (x, y) owns
 * rows[((y - y_begin) * width + x) * 7 ...], zero when invalid.  valid_f32 != 0: the pixel set of the fp32 validity
 * chain (dfko_se3_run_step_f, the kernels) instead of the fp64 one. */
void dfko_se3_pixel_rows_d(const float se3[7], const DfkoCamera* cam, int width, int height,
                           const float* img0, size_t img0_pitch, const float* img1, size_t img1_pitch,
                           const float* dpt0, size_t dpt0_pitch, const float* grad1, size_t grad1_pitch,
                           float huber_delta, int valid_f32, int y_begin, int y_end,
                           double* rows, double* residual, uint64_t* inliers);

/* ---- SE3Aligner::Warp (cu_se3aligner.cpp:61-113,125-151): img2 = img1 warped into frame 0
 * (0 where invalid); residual = signed sum (img0 - sampled). */
void dfko_se3_warp_f(const float se3[7], const DfkoCamera* cam, int width, int height,
                     const float* img0, size_t img0_pitch, const float* img1, size_t img1_pitch,
                     const float* dpt0, size_t dpt0_pitch, float* img2, size_t img2_pitch,
                     float* residual, uint64_t* inliers);
void dfko_se3_warp_d(const float se3[7], const DfkoCamera* cam, int width, int height,
                     const float* img0, size_t img0_pitch, const float* img1, size_t img1_pitch,
                     const float* dpt0, size_t dpt0_pitch, float* img2, size_t img2_pitch,
                     double* residual, uint64_t* inliers);

/* ---- UpdateDepth (cu_image_proc.cpp:248-277, warping.h:30-69) */
void dfko_update_depth_f(const float* code, int code_size, int width, int height,
                         const float* prx_orig, size_t prx_pitch, const float* prx_jac, size_t jac_pitch,
                         float avg_dpt, float* dpt_out, size_t dpt_pitch);
void dfko_update_depth_d(const float* code, int code_size, int width, int height,
                         const float* prx_orig, size_t prx_pitch, const float* prx_jac, size_t jac_pitch,
                         float avg_dpt, double* dpt_out, size_t dpt_pitch);

/* ---- DepthAligner::RunStep (cu_depthaligner.cpp:32-113): every pixel counts; JtJ packed upper C(C+1)/2, Jtr C.
 * avg_dpt is hard-coded to 2 in the reference kernel (:44); a parameter here. */
void dfko_depth_run_step_f(const float* code, int code_size, int width, int height, const float* tgt, size_t tgt_pitch,
                           const float* prx_orig, size_t prx_pitch, const float* prx_jac, size_t jac_pitch, float avg_dpt,
                           float* JtJ, float* Jtr, float* residual, uint64_t* inliers);
void dfko_depth_run_step_d(const float* code, int code_size, int width, int height, const float* tgt, size_t tgt_pitch,
                           const float* prx_orig, size_t prx_pitch, const float* prx_jac, size_t jac_pitch, float avg_dpt,
                           double* JtJ, double* Jtr, double* residual, uint64_t* inliers);
/* Its per-pixel rows [J (C) | diff] for image rows y_begin .. y_end-1: pixel (x, y) owns
 * rows[((y - y_begin) * width + x) * (C + 1) ...]. */
void dfko_depth_pixel_rows_f(const float* code, int code_size, int width, int height, const float* tgt, size_t tgt_pitch,
                             const float* prx_orig, size_t prx_pitch, const float* prx_jac, size_t jac_pitch,
                             float avg_dpt, int y_begin, int y_end, float* rows);
void dfko_depth_pixel_rows_d(const float* code, int code_size, int width, int height, const float* tgt, size_t tgt_pitch,
                             const float* prx_orig, size_t prx_pitch, const float* prx_jac, size_t jac_pitch,
                             float avg_dpt, int y_begin, int y_end, double* rows);

/* ---- ReprojectionFactor::linearize rows (core/gtsam/reprojection_factor.cpp:157-269): rows_out is
 * (2 * num_matches) x (13 + C) row-major [J_pose0 | J_pose1 | J_code0 | b]; returns the sum of squared unweighted errors */
float dfko_reprojection_rows_f(const float pose0[7], const float pose1[7], const float* code, int code_size,
                               const DfkoCamera* cam, int width, int height, const float* prx_orig, size_t prx_pitch,
                               const float* prx_jac, size_t jac_pitch, int num_matches, const float* query_xy,
                               const float* train_xy, float cauchy_delta, float sigma, float avg_dpt, float* rows_out);
double dfko_reprojection_rows_d(const float pose0[7], const float pose1[7], const float* code, int code_size,
                                const DfkoCamera* cam, int width, int height, const float* prx_orig, size_t prx_pitch,
                                const float* prx_jac, size_t jac_pitch, int num_matches, const float* query_xy,
                                const float* train_xy, float cauchy_delta, float sigma, float avg_dpt, double* rows_out);

/* ---- SparseGeometricFactor::linearize rows (core/gtsam/sparse_geometric_factor.cpp:157-271): rows_out is
 * num_points x (13 + 2C) row-major [J_pose0 | J_pose1 | J_code0 | J_code1 | b] (Huber-weighted); returns the number of
 * valid rows.  points_xy: 2 ints per point; dpt_grad1: (gx, gy) interleaved Sobel gradient of keyframe 1's depth */
int dfko_sparse_geometric_rows_f(const float pose0[7], const float pose1[7], const float* code0, const float* code1,
                                 int code_size, const DfkoCamera* cam, int width, int height, const float* prx0_orig,
                                 size_t prx0_pitch, const float* jac0, size_t jac0_pitch, const float* prx1_orig,
                                 size_t prx1_pitch, const float* jac1, size_t jac1_pitch, const float* dpt_grad1,
                                 size_t grad_pitch, int num_points, const int* points_xy, float huber_delta, float avg_dpt,
                                 float* rows_out);
int dfko_sparse_geometric_rows_d(const float pose0[7], const float pose1[7], const float* code0, const float* code1,
                                 int code_size, const DfkoCamera* cam, int width, int height, const float* prx0_orig,
                                 size_t prx0_pitch, const float* jac0, size_t jac0_pitch, const float* prx1_orig,
                                 size_t prx1_pitch, const float* jac1, size_t jac1_pitch, const float* dpt_grad1,
                                 size_t grad_pitch, int num_points, const int* points_xy, float huber_delta, float avg_dpt,
                                 double* rows_out);

/* ---- pyramid construction (cu_image_proc.cpp:57-92, 134-164) and SquaredError (:190-242) */
void dfko_sobel_gradients_f(int width, int height, const float* img, size_t img_pitch,
                            float* grad /* (gx,gy) interleaved */, size_t grad_pitch);
void dfko_gaussian_blur_down_f(int in_width, int in_height, const float* in, size_t in_pitch,
                               int out_width, int out_height, float* out, size_t out_pitch);
float dfko_squared_error_f(int width, int height, const float* a, size_t a_pitch,
                           const float* b, size_t b_pitch);
double dfko_squared_error_d(int width, int height, const float* a, size_t a_pitch,
                            const float* b, size_t b_pitch);

#ifdef __cplusplus
}
#endif
#endif /* DFK_ORACLE_H_ */
