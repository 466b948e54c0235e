/*
 * dfk.h -- C ABI of libdfk.so: H100-native (sm_90a) replacement for the dense
 * alignment hot path of DeepFactors' libdf_cuda.so (sources/cuda).
 *
 * The reference exports C++ class templates over Sophus/Eigen/VisionCore types
 * (not a C ABI); this header is the plain-pointer core a maintainer binds from
 * thin wrappers (see INTEGRATION.md and the headers under include/df/ for the C++ facade that
 * reproduces df::SfmAligner / df::SE3Aligner on top of it).  Every entry point
 * cites the reference interface it replaces; citations are file:line into
 * jczarnowski/DeepFactors @ bffc78a.
 *
 * Conventions
 *   pose      float[7] in Sophus::SE3f::data() order: unit quaternion (x,y,z,w),
 *             translation (x,y,z).
 *   DfkImage  pitched 2-D device view, the stand-in for vc::Image2DView /
 *             vc::Buffer2DView: element (x,y) at (char*)ptr + y*pitch_bytes +
 *             x*elem_size.  `width` counts PIXELS for every kind of image:
 *               scalar images (img, dpt, std, valid, prx_orig): 1 float / pixel
 *               grad1: 2 floats / pixel (gx,gy), Eigen::Matrix<float,1,2>
 *               prx_jac: code_size contiguous floats / pixel
 *                        (sources/core/mapping/keyframe.h:52, dense_sfm.h:150;
 *                        the reference views it as a (W*CS) x H float image)
 *   results   JtJ is the packed upper triangle, row major: (i,j), i<=j, at
 *             i*NP - i*(i-1)/2 + (j-i); column order [pose0 t(3) w(3) | pose1
 *             t(3) w(3) | code(C)] (dense_sfm.h:163-177).  Jtr is NOT negated,
 *             residual is the raw sum of squared weighted residuals
 *             (photometric_factor.cpp:105-106,275-282 do the sign flip/rescale).
 *   errors    every call returns a DfkStatus; dfk_last_error(handle) returns the
 *             message the reference would have thrown (launch_utils.h:26-32
 *             vc::CUDAException, cu_sfmaligner.cpp:171-173 std::runtime_error).
 *   threads   a handle is not re-entrant; different handles are independent
 *             (parameters are kernel arguments, not a process-global __constant__
 *             as in cu_sfmaligner.cpp:34,111).
 */
#ifndef DFK_H_
#define DFK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DFK_VERSION 104

typedef enum {
  DFK_OK = 0,
  DFK_ERR_INVALID_ARG = 1, /* glog CHECK failures of the reference (cu_sfmaligner.cpp:190-191) */
  DFK_ERR_CUDA = 2,        /* vc::CUDAException (launch_utils.h:26-32) */
  DFK_ERR_UNSUPPORTED = 3, /* code size / layout this build has no kernel for */
  DFK_ERR_NOMEM = 4
} DfkStatus;

typedef struct DfkContext* DfkHandle;

/* vc::Image2DView<T, TargetDeviceCUDA> stand-in (VisionCore, not in tree; call sites dense_sfm.h:141-147) */
typedef struct {
  void* ptr;
  size_t pitch_bytes;
  uint32_t width;  /* pixels */
  uint32_t height; /* rows   */
} DfkImage;

/* df::PinholeCamera<float> (sources/common/algorithm/pinhole_camera.h:43, _impl.h:30-31) */
typedef struct {
  float fx, fy, u0, v0;
  float width, height;
} DfkCamera;

/* df::DenseSfmParams (sources/common/algorithm/dense_sfm.h:36-43), same defaults */
typedef struct {
  float huber_delta; /* 0.1  */
  float ocl_th;      /* 1000, unused by the reference */
  float avg_dpt;     /* 2.0  */
  float min_dpt;     /* 0.0  */
  int32_t valid_border; /* 2 */
} DfkDenseSfmParams;

/* df::SfmAlignerParams (sources/cuda/cu_sfmaligner.h:41-48).  The launch-shape members are
 * accepted for source compatibility and validated like the reference (threads % 32 == 0,
 * blocks <= 1024; cu_sfmaligner.cpp:187-203) but the kernels size their own grids. */
typedef struct {
  DfkDenseSfmParams sfmparams;
  int32_t step_threads; /* 32  */
  int32_t step_blocks;  /* 11  */
  int32_t eval_threads; /* 224 */
  int32_t eval_blocks;  /* 66  */
} DfkSfmAlignerParams;

/* How the (6+C)x(6+C) Gauss-Newton Gram is accumulated.
 *   DFK_GRAM_FP32     CUDA-core FFMA, fp32 products and sums (any supported code size)
 *   DFK_GRAM_TF32X3   wgmma tensor cores, split-precision tf32 (hi*hi + lo*hi + hi*lo),
 *                     fp32 accumulate in registers; code sizes 32, 64 and 128, grad1 rows
 *                     8-byte aligned (else DFK_ERR_UNSUPPORTED)
 *   DFK_GRAM_AUTO     tensor cores for code sizes 32, 64 and 128, else FP32; FP32 also for a
 *                     batch whose grad1 rows are not 8-byte aligned */
typedef enum { DFK_GRAM_AUTO = 0, DFK_GRAM_FP32 = 1, DFK_GRAM_TF32X3 = 2 } DfkGramMode;

/* ------------------------------------------------------------------ lifetime / config */

/* Replaces SfmAligner::SfmAligner / SE3Aligner::SE3Aligner (cu_sfmaligner.cpp:102-114,
 * cu_se3aligner.cpp:119-120): owns the reduction scratch (bscratch_) and a stream.
 * device < 0 => current device. */
DfkStatus dfk_create(int device, DfkHandle* out);
DfkStatus dfk_destroy(DfkHandle h);
/* cudaStream_t to launch on; NULL is the legacy default stream (the one the reference uses,
 * with cudaDeviceSynchronize after every launch: launch_utils.h:28).  A new handle launches on a
 * private non-blocking stream; dfk_use_own_stream returns to it. */
DfkStatus dfk_set_stream(DfkHandle h, void* cuda_stream);
DfkStatus dfk_use_own_stream(DfkHandle h);
/* The RunStep kernels are persistent: one launch fills every SM for its whole duration, so a kernel that arrives on
 * another stream meanwhile (the collective of the previous step on a multi-GPU window, bench.py) finds no room, starts
 * when the first CTAs retire and then holds SMs the NEXT step's grid was sized for.  num_sms > 0 sizes the grids for
 * that many SMs and leaves the rest to the concurrent kernel; 0 = all SMs (default).  Results do not depend on it
 * beyond the summation order of the per-CTA partials (deterministic for a given limit).  No reference counterpart: the
 * reference synchronises the device after every launch (launch_utils.h:28). */
DfkStatus dfk_set_sm_limit(DfkHandle h, int num_sms);
void* dfk_get_stream(DfkHandle h);
DfkStatus dfk_synchronize(DfkHandle h);
const char* dfk_last_error(DfkHandle h);
const char* dfk_status_string(DfkStatus s);
int dfk_version(void);
/* 1 if this build has a RunStep kernel for the code size (reference: only 32, cu_sfmaligner.cpp:209) */
int dfk_sfm_supports_code_size(int code_size);

/* Measurement hooks (no reference equivalent; the reference times with std::clock around
 * synchronous calls, sources/common/timing.h:28-45).  With profiling on, every launch of the
 * dominant kernel (the per-tile warp+Gram kernel of RunStep) is bracketed by CUDA events on the
 * launching stream.  dfk_get_profile synchronizes the stream, returns the summed device time
 * of those launches and their count plus the number of ALL kernels this handle launched since the
 * last call, and resets the counters. */
DfkStatus dfk_set_profiling(DfkHandle h, int enabled);
DfkStatus dfk_get_profile(DfkHandle h, double* main_kernel_ms, uint64_t* main_kernel_launches,
                          uint64_t* total_kernel_launches);

/* SfmAligner ctor params + SetEvalThreadsBlocks/SetStepThreadsBlocks (cu_sfmaligner.cpp:187-203) */
DfkStatus dfk_sfm_set_params(DfkHandle h, const DfkSfmAlignerParams* p);
DfkStatus dfk_sfm_get_params(DfkHandle h, DfkSfmAlignerParams* p);
DfkStatus dfk_sfm_set_gram_mode(DfkHandle h, DfkGramMode m);
/* SE3Aligner::SetHuberDelta (cu_se3aligner.h:72), default 0.1 (:85) */
DfkStatus dfk_se3_set_huber_delta(DfkHandle h, float v);

/* ------------------------------------------------------------------ SfmAligner */

/* SfmAligner<float,CS>::RunStep (cu_sfmaligner.h:76-86, cu_sfmaligner.cpp:149-185).
 * code0/std0 are accepted and ignored exactly as the reference kernel ignores them
 * (dense_sfm.h:56-67,133-201); both may be NULL.  valid0 is in/out: set to 1 where a
 * correspondence is valid, never cleared (dense_sfm.h:161).  Synchronous; results land in
 * host memory: JtJ[NP(NP+1)/2], Jtr[NP], NP = 12 + code_size. */
DfkStatus dfk_sfm_run_step(DfkHandle h, const float pose0[7], const float pose1[7],
                           const float* code0, int code_size, const DfkCamera* cam,
                           const DfkImage* img0, const DfkImage* img1, const DfkImage* dpt0,
                           const DfkImage* std0, const DfkImage* valid0, const DfkImage* prx0_jac,
                           const DfkImage* grad1,
                           float* JtJ, float* Jtr, float* residual, uint64_t* inliers);

/* SfmAligner<float,CS>::EvaluateError (cu_sfmaligner.h:67-74, cu_sfmaligner.cpp:120-147):
 * border 1 / min_dpt 0 (dense_sfm.h:91), Huber-weighted squared error + inlier count.
 * std0/grad1 feed only the dead uncertainty weight (dense_sfm.h:100-107); may be NULL. */
DfkStatus dfk_sfm_evaluate_error(DfkHandle h, const float pose0[7], const float pose1[7],
                                 const DfkCamera* cam, const DfkImage* img0, const DfkImage* img1,
                                 const DfkImage* dpt0, const DfkImage* std0, const DfkImage* grad1,
                                 float* residual, uint64_t* inliers);

/* One (keyframe, frame, pyramid level) evaluation of a batch: the unit PhotometricFactor
 * creates per pair and level (sources/core/mapping/df_work.cpp:211-225). */
typedef struct {
  float pose0[7];
  float pose1[7];
  DfkCamera cam;
  DfkImage img0, img1, dpt0, valid0, prx0_jac, grad1;
  /* Optional fused depth decode (PhotometricFactor::UpdateDepthMaps + RunAlignmentStep in one pass,
   * photometric_factor.cpp:229,331-341): when `code` is not NULL, every pixel's depth is decoded first,
   *   dpt0(x,y) = avg_dpt / (prx_orig(x,y) + prx0_jac(x,y,:) . code) - avg_dpt      (warping.h:30-69),
   * written to dpt0 (an OUTPUT in this mode, exactly what dfk_update_depth writes, bit for bit) and used for the warp,
   * so the code Jacobian is read from HBM once instead of twice.  `code` is a HOST pointer to code_size floats. */
  DfkImage prx_orig;
  const float* code;
} DfkSfmWorkItem;

/* floats per device result record for code size C: [JtJ packed | Jtr | residual | inliers(u32 bits)] */
#define DFK_SFM_NP(C) (12 + (C))
#define DFK_SFM_RECORD_FLOATS(C) (DFK_SFM_NP(C) * (DFK_SFM_NP(C) + 1) / 2 + DFK_SFM_NP(C) + 2)

/* Batched RunStep: n work items in one persistent launch (the reference evaluates them one
 * call at a time from ISAM2, mapper.cpp:518-519).  `items` is a HOST array; `records_dev`
 * is DEVICE memory, n * DFK_SFM_RECORD_FLOATS(code_size) floats.  Asynchronous on the
 * handle's stream (no host sync, no D2H). */
DfkStatus dfk_sfm_run_step_batch(DfkHandle h, const DfkSfmWorkItem* items, int n, int code_size,
                                 float* records_dev);
/* Same, then copies the records to host memory and synchronizes. */
DfkStatus dfk_sfm_run_step_batch_host(DfkHandle h, const DfkSfmWorkItem* items, int n, int code_size,
                                      float* records_host);

/* Batched SfmAligner::EvaluateError, the error() half of PhotometricFactor (photometric_factor.cpp:61-81, 197-219):
 * n work items, the same DfkSfmWorkItem as dfk_sfm_run_step_batch, evaluated as dfk_sfm_evaluate_error evaluates one
 * (border 1, min_dpt 0, the handle's huber_delta).  valid0, prx0_jac, grad1 and prx_orig are ignored; `code` must be
 * NULL (the depth is read from dpt0; decode it first with dfk_update_depth_batch), else DFK_ERR_INVALID_ARG.
 * out_dev: DEVICE, 2 floats per item, [residual | inliers (u32 bits)], each bit for bit what dfk_sfm_evaluate_error
 * gives for that item alone, whatever else is in the batch.  1 <= n <= 65535.  One launch, asynchronous on the handle's
 * stream (no host sync, no D2H); every item is validated before anything is enqueued. */
DfkStatus dfk_sfm_evaluate_error_batch(DfkHandle h, const DfkSfmWorkItem* items, int n, float* out_dev);

/* ------------------------------------------------------------------ streaming evaluation from HOST memory
 *
 * The reference's inputs live in host/device mirrored pyramids that are uploaded lazily, one synchronous copy at a
 * time, on first GPU use (sources/cuda/synced_pyramid.h:118-126,178-198).  This is the same hand-over as ONE pipelined
 * call: dfk_sfm_stream_submit takes work items whose image views point at HOST memory (pinned for full speed), uploads
 * them on a copy stream into one of `depth` device slots, evaluates them (dfk_sfm_run_step_batch) on the handle's stream
 * as soon as the upload has landed and sends the result records back -- all asynchronous, so the upload of submission
 * k+1 overlaps the evaluation of submission k.  dfk_sfm_stream_wait blocks until the records of a ticket are in host
 * memory.  Tickets must be waited for in order; at most `depth` submissions may be outstanding.
 * valid0 of a streamed item is device scratch (the mask is neither uploaded nor returned); with the fused depth decode
 * (code != NULL) prx_orig is uploaded instead of dpt0 and the decoded depth stays on the device.
 */
typedef struct DfkSfmStream DfkSfmStream;
DfkStatus dfk_sfm_stream_create(DfkHandle h, int code_size, int max_items, size_t max_bytes_per_submit, int depth,
                                DfkSfmStream** out);
DfkStatus dfk_sfm_stream_destroy(DfkHandle h, DfkSfmStream* s);
DfkStatus dfk_sfm_stream_submit(DfkHandle h, DfkSfmStream* s, const DfkSfmWorkItem* host_items, int n,
                                uint64_t* ticket);
DfkStatus dfk_sfm_stream_wait(DfkHandle h, DfkSfmStream* s, uint64_t ticket, float* records_host);

/* ------------------------------------------------------------------ keyframe window (block-sparse normal equations)
 *
 * What the factor graph does with the RunStep results of a window of keyframes: every (pair, level) result is one
 * PhotometricFactor (sources/core/mapping/df_work.cpp:211-225) whose linearize() slices the (12+C)^2 Hessian into the
 * blocks G11 G12 G13 G22 G23 G33 / g1 g2 g3 of a HessianFactor over (pose0, pose1, code0) with g = -Jtr and the
 * residual rescaled to res / inliers * W * H (sources/core/gtsam/photometric_factor.cpp:105-161, 275-282); the solver
 * then adds the factors of the window into one system.  dfk_window_assemble does that sum ON THE DEVICE, straight from
 * the record buffer of dfk_sfm_run_step_batch, into a packed block-sparse buffer -- the one buffer a multi-GPU
 * Gauss-Newton step all-reduces (pairs shard across GPUs, every rank assembles its own pairs into the same layout).
 *
 * Variables: keyframe k owns [pose_k (6) | code_k (C)], B = 6 + C.  Buffer layout (fp32):
 *   K diagonal blocks  B x B, row-major, full symmetric
 *   K gradients        B            (g = -sum Jtr)
 *   P coupling blocks  B x 6, row-major: rows = [pose0 | code0] of the pair's keyframe k0, columns = pose1 of its k1
 *   2 scalars          f = sum of rescaled residuals over items with overlap + residuals of unscaled records,
 *                      total inliers of the scaled (photometric) records (as a float)
 * Deterministic: every output element is summed by one thread in item order (a gather, no float atomics).
 */
typedef struct DfkWindow DfkWindow;
typedef struct {
  int32_t num_keyframes;
  int32_t num_pairs;
  int32_t num_items;       /* records per evaluation: one per (pair, level) */
  int32_t code_size;
  const int32_t* pair_k0;  /* [num_pairs] keyframe (pose0 / code0) of every pair      (HOST arrays, copied) */
  const int32_t* pair_k1;  /* [num_pairs] frame (pose1)                                                      */
  const int32_t* item_pair;   /* [num_items] pair of every record                                            */
  const int32_t* item_width;  /* [num_items] level size, for the residual rescale; width = height = 0 marks an  */
  const int32_t* item_height; /* UNSCALED record (dfk_reprojection_linearize_batch): its residual enters f as it is
                                 and its inliers are left out of the inlier total                                */
} DfkWindowDesc;
DfkStatus dfk_window_create(DfkHandle h, const DfkWindowDesc* desc, DfkWindow** out);
DfkStatus dfk_window_destroy(DfkHandle h, DfkWindow* w);
/* floats of the block-sparse buffer: K*(B*B + B) + P*6*B + 2 */
size_t dfk_window_floats(const DfkWindow* w);
/* records_dev: num_items records as written by dfk_sfm_run_step_batch (DEVICE).  window_dev: dfk_window_floats()
 * floats (DEVICE), fully overwritten.  Asynchronous on the handle's stream, one launch. */
DfkStatus dfk_window_assemble(DfkHandle h, const DfkWindow* w, const float* records_dev, float* window_dev);

/* A window that also holds num_links sparse geometric links l = (link_k0[l] -> link_k1[l]) (HOST arrays, copied), one
 * record of DFK_GEO_RECORD_FLOATS each (dfk_sparse_geometric_linearize_batch).  The buffer is the layout above with L
 * link blocks appended after the two scalars, so no offset of the layout above moves:
 *   L link blocks      B x B, row-major: rows = [pose | code] of the link's k0, columns = [pose | code] of its k1
 * Link l adds its (pose0, code0) block to k0's diagonal block, its whole (pose1, code1) block to k1's, the matching
 * parts of -Jtr to both gradients and its residual (b^T b) to f; it adds nothing to the inlier total.  An element sums
 * the items in item order, then the links where its keyframe is k0, then those where it is k1, in link order.
 * A link naming a keyframe outside the window or with k0 == k1 is rejected.  num_links = 0 is dfk_window_create. */
DfkStatus dfk_window_create_geometric(DfkHandle h, const DfkWindowDesc* desc, int num_links, const int32_t* link_k0,
                                      const int32_t* link_k1, DfkWindow** out);
/* dfk_window_assemble for a window with links (dfk_window_assemble rejects such a window).  geo_records_dev: DEVICE,
 * num_links records; it may be NULL only when the window has no links, and the buffer is then bit for bit the one
 * dfk_window_assemble writes.  Asynchronous on the handle's stream, one launch. */
DfkStatus dfk_window_assemble_geometric(DfkHandle h, const DfkWindow* w, const float* records_dev,
                                        const float* geo_records_dev, float* window_dev);

/* Tracked frames (Mapper::EnqueueFrame): pose-only variables, one photometric factor keyframe -> frame each.
 * A window of num_frames frames: a pair whose pair_k1 is K + f is frame f's pair (its pose1 is the frame's pose), and
 * every frame must be k1 of exactly one pair, never k0, never in a link, and its pair's items must all be scaled
 * (photometric, one per level).  The buffer is the layout above, links included, followed by
 *   F frame blocks     6 x 6, row-major: pose1 x pose1 of the frame pair's items
 *   F frame gradients  6            (-sum Jtr of pose1)
 * so dfk_window_floats grows by 42 F and no offset above moves.  A frame pair's coupling block is its B x 6 block as
 * for any pair (rows = k0's [pose | code], columns = the frame's pose); its items count toward f and the inlier total.
 * Assemble with dfk_window_assemble_geometric (geo_records_dev NULL without links).  num_frames = 0 is
 * dfk_window_create_geometric.  A rejected call writes nothing. */
DfkStatus dfk_window_create_frames(DfkHandle h, const DfkWindowDesc* desc, int num_links, const int32_t* link_k0,
                                   const int32_t* link_k1, int num_frames, DfkWindow** out);

/* A linear prior on one keyframe's [pose | code] (B = 6 + C): [G (B x B row-major, symmetric) | g (B) | f0], doubles */
#define DFK_PRIOR_DOUBLES(C) ((6 + (C)) * (6 + (C)) + (6 + (C)) + 1)
/* Marginalise the frames frames_host[0..n) (HOST, copied) of window w: for each, the fp64 sums of its pair's items in
 * item order give H_aa (k's [pose | code]), H_ab (x frame pose), H_bb (6 x 6), g_a, g_b (= -sum Jtr) and f_p (the
 * items' rescaled residuals), and prior i (priors_dev + i * DFK_PRIOR_DOUBLES(C), DEVICE) is their Schur complement
 *   G = H_aa - H_ab H_bb^-1 H_ab^T,  g = g_a - H_ab H_bb^-1 g_b,  f0 = f_p - g_b^T H_bb^-1 g_b
 * at the point the records were evaluated at (H_bb undamped).  info_dev[i] (DEVICE int32) = 0, or 1 + the row of H_bb
 * whose pivot was not positive and finite (prior i is then all zero).  One launch, one CTA per frame. */
DfkStatus dfk_window_marginalize_frames(DfkHandle h, const DfkWindow* w, const float* records_dev, int n,
                                        const int32_t* frames_host, double* priors_dev, int32_t* info_dev);
/* Add m priors to an assembled window buffer in place.  Prior i (priors_dev, DEVICE, m * DFK_PRIOR_DOUBLES(C)) is on
 * keyframe prior_kf_host[i] (HOST, copied) and delta_dev[i * B ..] (DEVICE, m * B doubles) = Local(x0_i, x) of that
 * keyframe: [t - t0 | log(R R0^T) | c - c0].  It adds G to D_k, g - G delta to g_k and f0 - 2 g^T delta +
 * delta^T G delta to f (buffer units: f is twice the factor-graph error); the inlier total is unchanged.  Every entry
 * sums its keyframe's priors in list order in fp64 and is rounded once.  With sharded pairs, call it after the
 * all-reduce (on every rank), or the priors are counted once per rank.  One launch. */
DfkStatus dfk_window_add_priors(DfkHandle h, const DfkWindow* w, int m, const int32_t* prior_kf_host,
                                const double* priors_dev, const double* delta_dev, float* window_dev);

/* Sliding the window: keyframe priors.  Marginalising a keyframe m out of a window leaves a dense linear prior over its
 * blanket N(m), the ascending list of the keyframes that share a factor with m (a pair in either direction, a reprojection
 * or geometric link, or a keyframe prior that contains m).  A keyframe prior over the keyframes kf[0..n) (ascending) is
 *   [G (nB x nB, symmetric, row-major) | g (nB) | f0]  doubles, rows / columns in the order of its keyframe list,
 * a factor frozen at the point x0 it was made at: its energy at x is f0 - 2 g^T d + d^T G d, d = Local(x0, x) per member
 * (buffer units, as for DFK_PRIOR_DOUBLES).  Like the frame priors it is never re-linearised. */
#define DFK_KF_PRIOR_DOUBLES(C, n) \
  ((size_t)(n) * (6 + (C)) * (size_t)(n) * (6 + (C)) + (size_t)(n) * (6 + (C)) + 1)
/* the largest blanket dfk_window_marginalize_keyframe accepts */
#define DFK_MAX_BLANKET 16
/* A window that also holds num_kf_priors keyframe priors: prior i covers the keyframes prior_kf[prior_ptr[i] ..
 * prior_ptr[i + 1]) (HOST arrays, copied; each list non-empty, ascending, distinct and inside the window).  The buffer is
 * the dfk_window_create_frames layout followed by
 *   Q prior blocks     B x B, row-major: rows = [pose | code] of keyframe i, columns = [pose | code] of keyframe j
 * one per distinct keyframe pair (i < j) that occurs in some prior, in ascending (i, j) order, so no offset above moves.
 * dfk_window_assemble_geometric zeroes the prior blocks; dfk_window_add_keyframe_priors fills them.  num_kf_priors = 0 is
 * dfk_window_create_frames.  A rejected call writes nothing. */
DfkStatus dfk_window_create_priors(DfkHandle h, const DfkWindowDesc* desc, int num_links, const int32_t* link_k0,
                                   const int32_t* link_k1, int num_frames, int num_kf_priors, const int32_t* prior_ptr,
                                   const int32_t* prior_kf, DfkWindow** out);
/* Add the window's keyframe priors to an assembled buffer in place.  priors_dev: DEVICE, the priors in window order, each
 * DFK_KF_PRIOR_DOUBLES(C, n_i) doubles, back to back.  delta_dev: DEVICE, n_i * B doubles per prior, back to back: Local(x0,
 * x) of each member, [t - t0 | log(R R0^T) | c - c0].  G's diagonal blocks go to D_k, its off-diagonal blocks to the prior
 * blocks, g - G delta to the gradients and f0 - 2 g^T delta + delta^T G delta to f; the inlier total is unchanged.  Every
 * entry sums its terms in fp64 in prior order onto its fp32 value and is rounded once (no atomics).  With sharded pairs,
 * call it after the all-reduce, on every rank.  One launch. */
DfkStatus dfk_window_add_keyframe_priors(DfkHandle h, const DfkWindow* w, const double* priors_dev,
                                         const double* delta_dev, float* window_dev);
/* The blanket N(m) of keyframe m (a host query): kf_out (HOST, at least K - 1 entries) gets the ascending list, *n its
 * length. */
DfkStatus dfk_window_blanket(DfkHandle h, const DfkWindow* w, int m, int32_t* kf_out, int32_t* n);
/* Marginalise keyframe m.  Forms in fp64 the joint system over [m | N(m)] of every factor that touches m, each entry
 * summing, in this order: the records of m's pairs in item order (records_dev, as dfk_window_assemble reads them: -Jtr,
 * residuals rescaled), m's geometric links in link order (geo_records_dev; NULL when the window has no links), the
 * num_frame_priors frame priors on m (frame_priors_dev, DFK_PRIOR_DOUBLES(C) each, at frame_delta_dev, B doubles each),
 * the window's keyframe priors that contain m (kf_priors_dev / kf_delta_dev as dfk_window_add_keyframe_priors takes them;
 * NULL when the window has none), and with code_prior_weight w > 0 the zero-code prior on m (w I, -w c_m, w |c_m|^2;
 * code_m_host: HOST, C doubles).  prior_dev (DEVICE, DFK_KF_PRIOR_DOUBLES(C, n)) gets the Schur complement of m's B
 * variables, H_mm undamped, as a keyframe prior over N(m) at the point the records were evaluated at:
 *   G = H_NN - H_Nm H_mm^-1 H_mN,  g = g_N - H_Nm H_mm^-1 g_m,  f0 = f - g_m^T H_mm^-1 g_m.
 * info_dev (DEVICE int32) = 0, or 1 + the row of H_mm whose pivot was not positive and finite (the prior is then zero).
 * A keyframe that still has tracked frames (marginalise them first), a blanket larger than DFK_MAX_BLANKET
 * (DFK_ERR_UNSUPPORTED) and an empty blanket are rejected; a rejected call writes nothing.  Deterministic (two calls are
 * bit for bit equal), asynchronous on the handle's stream, four launches.  The workspace, the lower B x B tiles of the
 * local system plus one, (n + 2 + n (n + 1) / 2) B^2 + (n + 1) B + 1 doubles (38 MB at n = 16, C = 128), is the handle's
 * grow-only scratch. */
DfkStatus dfk_window_marginalize_keyframe(DfkHandle h, const DfkWindow* w, const float* records_dev,
                                          const float* geo_records_dev, int m, int num_frame_priors,
                                          const double* frame_priors_dev, const double* frame_delta_dev,
                                          const double* kf_priors_dev, const double* kf_delta_dev,
                                          double code_prior_weight, const double* code_m_host, double* prior_dev,
                                          int32_t* info_dev);

/* Damped block-sparse fp64 Cholesky solve of a window's normal equations, straight from its packed buffer.
 *
 * The system is the dense one the buffer stands for (fp32 entries promoted to fp64, every off-diagonal block mirrored):
 *   1. with w = code_prior_weight > 0: + w I on every code block, - w code_k on every code gradient;
 *   2. the fixed variables dropped (solved as identity rows with a zero right-hand side: dx = 0 there);
 *   3. d = diag(H) over the kept variables, + lambda d + 1e-12 max|d| on that diagonal;
 *   4. H dx = g.
 * The unit of sparsity is the B x B tile of a pair of keyframes.  create runs the symbolic elimination in keyframe order
 * (a tile (i, j), i >= j, is nonzero when i = j, when a pair or link joins i and j in either direction, or by fill) and
 * allocates the workspace: (tiles + K) * B * B doubles for the factor, plus K * B doubles and K * C doubles.
 * A solve is deterministic (two solves of the same buffer are bit for bit equal, on any handle of the same GPU model),
 * asynchronous on the handle's stream, and allocates nothing: one load launch, a panel and an update launch per
 * keyframe column, a backward launch per keyframe.
 * A window with F tracked frames (dfk_window_create_frames) adds 6 F variables after the keyframes' (frame f at
 * K B + 6 f); the system is the dense one with the frames' blocks, and d / max|d| of step 3 run over the frames too.
 * Frames are leaves: each is eliminated first, into its keyframe's diagonal tile at load (no fill, the symbolic analysis
 * ignores frame pairs), and its dx follows in one launch after the backward pass.
 * A window with keyframe priors (dfk_window_create_priors): every prior block is a nonzero tile of the symbolic analysis,
 * like a link, and one more load launch adds the prior blocks to their tiles after the links, in to_dense's order. */
typedef struct DfkWindowSolver DfkWindowSolver;
/* fixed_vars: HOST, num_fixed distinct window-variable indices k * B + r (e.g. 0..5 = the gauge keyframe's pose), copied.
 * Out-of-range or duplicated indices are rejected. */
DfkStatus dfk_window_solver_create(DfkHandle h, const DfkWindow* w, int num_fixed, const int32_t* fixed_vars,
                                   DfkWindowSolver** out);
/* h must not be NULL (like every entry point that takes a handle); s may be */
DfkStatus dfk_window_solver_destroy(DfkHandle h, DfkWindowSolver* s);
/* *tiles = the structurally nonzero B x B tiles of the lower factor, fill included */
DfkStatus dfk_window_solver_tiles(DfkHandle h, const DfkWindowSolver* s, size_t* tiles);

typedef struct {
  double lambda;            /* LM damping, >= 0, finite */
  double code_prior_weight; /* >= 0, finite; 0 = no prior */
} DfkWindowSolveParams;

/* window_dev: the packed buffer of dfk_window_assemble[_geometric] for this solver's window (DEVICE, fp32, read only).
 * codes: HOST, K * C doubles, required iff code_prior_weight > 0 (read before the call returns).
 * dx_dev: DEVICE, K * B + 6 F doubles, fully written.  info_dev: DEVICE, one int32: 0, or 1 + the first variable (in
 * elimination order: the frames first, then the keyframes) whose pivot was not positive and finite; dx is then all
 * zero.
 * Every argument is checked before anything is enqueued; a rejected call writes nothing. */
DfkStatus dfk_window_solve(DfkHandle h, const DfkWindowSolver* s, const float* window_dev, const DfkWindowSolveParams* p,
                           const double* codes, double* dx_dev, int32_t* info_dev);

/* ------------------------------------------------------------------ SE3Aligner */

/* SE3Aligner<float>::RunStep (cu_se3aligner.h:65-70, cu_se3aligner.cpp:153-176):
 * JtJ[21] packed upper 6x6, Jtr[6]. */
DfkStatus dfk_se3_run_step(DfkHandle h, const float se3[7], const DfkCamera* cam,
                           const DfkImage* img0, const DfkImage* img1, const DfkImage* dpt0,
                           const DfkImage* grad1,
                           float* JtJ, float* Jtr, float* residual, uint64_t* inliers);

/* One pyramid level of a tracking problem: keyframe image/depth (img0, dpt0), live frame image/gradient (img1,
 * grad1), the level's camera and the Gauss-Newton iteration count (TrackerConfig::iterations_per_level,
 * core/system/camera_tracker.h:45-50). */
typedef struct DfkTrackLevel {
  DfkCamera cam;
  DfkImage img0, img1, dpt0, grad1;
  int iterations;
} DfkTrackLevel;

/* CameraTracker::TrackFrame (core/system/camera_tracker.cpp:42-69): coarse-to-fine Gauss-Newton on pose_ck.
 * levels[0] is the finest level; iteration runs from levels[num_levels-1] down to levels[0].  Per iteration the
 * reference does SE3Aligner::RunStep + cudaDeviceSynchronize + a 120-byte D2H + a host 6x6 LDLT + retraction
 * (update = -JtJ.ldlt().solve(Jtr); t += update.head<3>(); so3 = exp(update.tail<3>()) * so3); here every iteration
 * is ONE launch whose last block solves the 6x6 system and retracts the pose in device memory, all iterations are
 * enqueued back to back and there is a single read-back at the end.
 *   pose_ck         in/out, (qx,qy,qz,qw,tx,ty,tz)
 *   inlier_fraction inliers / area and error = residual / inliers of the last evaluated system (the reference
 *   error           records them on the last iteration of level 0, :65-69); error = +inf when inliers == 0
 *   last_system     optional, 29 floats [JtJ packed upper 21 | Jtr 6 | residual | inliers (u32 bits)]
 *   history         optional, history_capacity x 36 floats: per iteration the 29 floats above + the pose (7) they
 *                   were evaluated at
 * An iteration whose system is not positive definite (e.g. zero inliers) leaves the pose untouched. */
DfkStatus dfk_se3_track(DfkHandle h, float pose_ck[7], const DfkTrackLevel* levels, int num_levels,
                        float* inlier_fraction, float* error, float* last_system, float* history,
                        int history_capacity);

/* One live frame tracked against many keyframes, the loop of DeepFactors::Relocalize (core/deepfactors.cpp:713-743:
 * SetKeyframe + Reset + TrackFrame per keyframe of the map, keep the smallest GetError()) and of the geometry check in
 * LoopDetector::DetectLoop (core/system/loop_detector.cpp:149-168: one TrackFrame per candidate keyframe, then
 * GetInliers() / GetPoseEstimate()).  The reference tracks them one after another; here the num_problems problems
 * advance in lockstep: every Gauss-Newton iteration is ONE launch for all of them, and there is one upload and one
 * read-back per call.  Synchronous.
 *   poses_ck         in/out, num_problems x 7 floats
 *   levels           num_problems x num_levels, problem-major: problem n's pyramid is levels[n * num_levels ...],
 *                    level 0 the finest.  Level sizes may differ between problems; the iteration count of a level
 *                    must be the same for every problem (else DFK_ERR_INVALID_ARG).  1 <= num_problems <= 65535.
 *   inlier_fraction  optional, num_problems floats
 *   error            optional, num_problems floats
 *   last_systems     optional, num_problems x 29 floats
 * Problem n gives exactly what dfk_se3_track(h, poses_ck + 7n, levels + n * num_levels, num_levels, ...) gives, bit for
 * bit, including its two rules: inlier_fraction / error are left untouched when level 0 has no iteration, and a system
 * that is not positive definite leaves that problem's pose alone. */
DfkStatus dfk_se3_track_batch(DfkHandle h, int num_problems, int num_levels, float* poses_ck,
                              const DfkTrackLevel* levels, float* inlier_fraction, float* error,
                              float* last_systems);

/* SE3Aligner<float>::Warp (cu_se3aligner.h:58-63, cu_se3aligner.cpp:125-151): renders img1
 * into frame 0 (img2, 0 where invalid); residual = SIGNED sum(img0 - sampled) (:106). */
DfkStatus dfk_se3_warp(DfkHandle h, const float se3[7], const DfkCamera* cam,
                       const DfkImage* img0, const DfkImage* img1, const DfkImage* dpt0,
                       const DfkImage* img2, float* residual, uint64_t* inliers);

/* ------------------------------------------------------------------ DepthAligner */

/* DepthAligner<float,CS>::RunStep (sources/cuda/cu_depthaligner.h:46-49, cu_depthaligner.cpp:32-113): aligns the depth
 * decoded from `code` (HOST, code_size floats) to target_dpt; every pixel counts.  JtJ[CS(CS+1)/2] packed upper,
 * Jtr[CS], residual = sum diff^2, inliers = W*H.  The reference hard-codes avg_dpt = 2 in this kernel (:44); here it
 * is the handle's DenseSfmParams::avg_dpt (same default).  Synchronous. */
DfkStatus dfk_depth_run_step(DfkHandle h, const float* code, int code_size, const DfkImage* target_dpt,
                             const DfkImage* prx_orig, const DfkImage* prx_jac,
                             float* JtJ, float* Jtr, float* residual, uint64_t* inliers);

/* ------------------------------------------------------------------ sparse keypoint factor */

/* ReprojectionFactor::linearize (sources/core/gtsam/reprojection_factor.cpp:157-269): the Jacobian rows of a keypoint
 * reprojection factor, gathered on the device from the keyframe's level-0 proximity / code-Jacobian buffers instead of
 * mirroring the whole pyramid to the host (kf_->pyr_jac.GetCpuLevel(0), :193).
 *   query_xy / train_xy   HOST, 2 floats per match: matched keypoints in the keyframe / in the frame (:183-186)
 *   rows                  HOST out, (2 * num_matches) x (13 + code_size), row-major:
 *                         [dErr/dPose0 (6) | dErr/dPose1 (6) | dErr/dCode0 (C) | b (1)], already multiplied by the
 *                         Cauchy weight (m_estimators.h:43-48, parameter `cauchy_delta` = the factor's huber_delta_) and
 *                         divided by sigma -- the blocks of gtsam::JacobianFactor(keys, Ab) (:255-268); zero rows for a
 *                         match whose point falls behind the camera (:204-212)
 *   total_err             out, sum of squared UNWEIGHTED reprojection errors (total_err_, :242,258)
 * avg_dpt is hard-coded to 2 there (:171); here it is the handle's DenseSfmParams::avg_dpt.
 * The Cauchy weight is |a| / sqrt(2) * sqrt(log1p(1 / a^2)), a = cauchy_delta / err.  The reference's float
 * log(1 + 1 / a^2) loses the weight as a grows and gives 0 below about err = cauchy_delta / 4096, so a near-exact match,
 * or any match under a large cauchy_delta, drops out of H; this build keeps the weight to fp32 accuracy there (it tends
 * to 1 / sqrt(2)).  A match exactly on its keypoint (err = 0) still gives NaN, as in the reference.  The same weight
 * serves dfk_reprojection_linearize_batch and dfk_reprojection_error_batch.  Synchronous. */
DfkStatus dfk_reprojection_linearize(DfkHandle h, const float pose0[7], const float pose1[7], const float* code0,
                                     int code_size, const DfkCamera* cam, const DfkImage* prx_orig,
                                     const DfkImage* prx_jac, int num_matches, const float* query_xy,
                                     const float* train_xy, float cauchy_delta, float sigma, float* rows,
                                     float* total_err);

/* One ReprojectionFactor of a batch: the arguments of dfk_reprojection_linearize for one factor (k0 -> k1).  A global
 * loop closure (DeepFactors::ProcessFrame -> Mapper::EnqueueLink(..., rep = true), core/deepfactors.cpp:274,
 * mapper.cpp:367-376) and the use_reprojection links (mapper.cpp:314-325) are such factors. */
typedef struct {
  float pose0[7], pose1[7];
  DfkCamera cam;                  /* level 0 (cam_pyr_[0], mapper.cpp:317) */
  DfkImage prx_orig, prx_jac;     /* keyframe k0's level-0 DEVICE buffers */
  const float* code;              /* HOST, code_size floats: code0 of k0 */
  int32_t num_matches;
  const float* query_xy;          /* HOST, 2 floats per match (keypoints in k0) */
  const float* train_xy;          /* HOST, 2 floats per match (keypoints in k1) */
  float cauchy_delta, sigma;      /* rep_huber, rep_sigma (or loop_sigma for a loop closure) */
} DfkReprojectionItem;

/* Batched ReprojectionFactor::linearize straight into normal-equation records: factor i's JacobianFactor [A | b] (the
 * rows of dfk_reprojection_linearize, bit for bit) contributes H += A^T A, g += A^T b and 1/2 |b|^2 to the energy
 * (reprojection_factor.cpp:148,254-268), so its record in the RunStep layout (DFK_SFM_RECORD_FLOATS) is
 *   JtJ = A^T A (packed upper), Jtr = -A^T b, residual = b^T b, inliers = matches with a valid correspondence (u32 bits)
 * and it enters dfk_window_assemble as an unscaled record (item_width = item_height = 0).  records_dev: DEVICE,
 * n * DFK_SFM_RECORD_FLOATS(code_size) floats.  One launch, one CTA per factor, a fixed summation order per factor: a
 * factor's record does not depend on the rest of the batch.  total_err (statistics only) is not computed.
 * Asynchronous on the handle's stream (no host sync, no D2H); the host arrays may be freed when the call returns.
 * Every item is validated before anything is enqueued (1 <= n, num_matches >= 1, sigma > 0, consistent views, non-NULL
 * pointers); a rejected call writes nothing and dfk_last_error names the item. */
DfkStatus dfk_reprojection_linearize_batch(DfkHandle h, const DfkReprojectionItem* items, int n, int code_size,
                                           float* records_dev);

/* SparseGeometricFactor::linearize (sources/core/gtsam/sparse_geometric_factor.cpp:157-271): the Jacobian rows of the
 * sparse depth-consistency factor between two keyframes, evaluated on the device from the keyframes' level-0 proximity /
 * code-Jacobian buffers and keyframe 1's depth gradient instead of host mirrors of all five (:181-183, :207-209, :220).
 *   points_xy    HOST, 2 ints per point: the sampled pixels of keyframe 0 (UniformSampler, uniform_sampler.h:28-32)
 *   dpt_grad1    kf1->dpt_grad: SobelGradients of keyframe 1's level-0 depth (mapper.cpp:998-1000), 2 floats per pixel
 *   rows         HOST out, num_points x (13 + 2 * code_size), row-major:
 *                [dErr/dPose0 (6) | dErr/dPose1 (6) | dErr/dCode0 (C) | dErr/dCode1 (C) | b], already multiplied by the
 *                Huber weight (DenseSfm_RobustLoss, dense_sfm.h:47-50) -- the blocks of gtsam::JacobianFactor(keys, Ab)
 *                (:260-270); zero rows for points whose correspondence is invalid (:190-198)
 *   num_valid    out (may be NULL): rows that are not all zero
 * avg_dpt is hard-coded to 2 there (:166); here it is the handle's DenseSfmParams::avg_dpt.  Synchronous. */
DfkStatus dfk_sparse_geometric_linearize(DfkHandle h, const float pose0[7], const float pose1[7], const float* code0,
                                         const float* code1, int code_size, const DfkCamera* cam, const DfkImage* prx0_orig,
                                         const DfkImage* prx0_jac, const DfkImage* prx1_orig, const DfkImage* prx1_jac,
                                         const DfkImage* dpt_grad1, int num_points, const int* points_xy, float huber_delta,
                                         float* rows, int* num_valid);

/* One SparseGeometricFactor of a batch: the arguments of dfk_sparse_geometric_linearize for one factor (k0 -> k1), as
 * Mapper adds them with use_geometric (mapper.cpp:328-337, 379-388). */
typedef struct {
  float pose0[7], pose1[7];
  DfkCamera cam;                            /* level 0 */
  DfkImage prx0_orig, prx0_jac;             /* keyframe k0, level 0, DEVICE */
  DfkImage prx1_orig, prx1_jac, dpt_grad1;  /* keyframe k1, level 0, DEVICE; dpt_grad1 2 floats per pixel */
  const float* code0;                       /* HOST, code_size floats */
  const float* code1;                       /* HOST, code_size floats */
  int32_t num_points;
  const int32_t* points_xy;                 /* HOST, 2 ints per point */
  float huber_delta;
} DfkSparseGeometricItem;
/* variables of a geometric record, in the JacobianFactor's key order [pose0 (6) | pose1 (6) | code0 (C) | code1 (C)] */
#define DFK_GEO_NP(C) (12 + 2 * (C))
#define DFK_GEO_RECORD_FLOATS(C) (DFK_GEO_NP(C) * (DFK_GEO_NP(C) + 1) / 2 + DFK_GEO_NP(C) + 2)

/* Batched SparseGeometricFactor::linearize straight into normal-equation records: factor i's JacobianFactor [A | b] (the
 * rows of dfk_sparse_geometric_linearize, bit for bit) gives the record
 *   JtJ = A^T A (packed upper, DFK_GEO_NP(C) variables), Jtr = -A^T b, residual = b^T b, inliers = valid points (u32 bits)
 * records_dev: DEVICE, n * DFK_GEO_RECORD_FLOATS(code_size) floats.  One launch; a factor's record is summed in a fixed
 * order by CTAs of its own, so it does not depend on the rest of the batch.  avg_dpt is the handle's
 * DenseSfmParams::avg_dpt.  Asynchronous on the handle's stream (no host sync, no D2H); the host arrays may be freed when
 * the call returns.  Every item is validated before anything is enqueued (1 <= n, num_points >= 1, huber_delta > 0,
 * consistent views, a camera no larger than the views, non-NULL pointers); a rejected call writes nothing and
 * dfk_last_error names the item. */
DfkStatus dfk_sparse_geometric_linearize_batch(DfkHandle h, const DfkSparseGeometricItem* items, int n, int code_size,
                                               float* records_dev);

/* The error() half of the two sparse factors (ReprojectionFactor::error, reprojection_factor.cpp:97-154;
 * SparseGeometricFactor::error, sparse_geometric_factor.cpp:85-142): the same items as the linearize batches, and per
 * factor out_dev (DEVICE, 2 floats per factor) = [b^T b | valid matches / points (u32 bits)], where b is the last column of
 * the factor's JacobianFactor [A | b].  b^T b is bit for bit the residual of the factor's record from the matching
 * linearize batch, so it is twice the factor's error in the linearisation's units and follows the linearisation's
 * validity rules (a point outside the views or behind the camera counts as invalid, not as an out-of-bounds read).  No
 * Jacobian is formed.  One launch, one CTA per factor; asynchronous on the handle's stream; argument checks as for the
 * linearize batches. */
DfkStatus dfk_reprojection_error_batch(DfkHandle h, const DfkReprojectionItem* items, int n, int code_size,
                                       float* out_dev);
DfkStatus dfk_sparse_geometric_error_batch(DfkHandle h, const DfkSparseGeometricItem* items, int n, int code_size,
                                           float* out_dev);

/* ------------------------------------------------------------------ keypoint matching of a reprojection factor */

/* The features of one keyframe (df::Features, features/feature_detection.h: keypoints and descriptors of
 * kf->features), on the device, so that every factor of the keyframe reads one upload. */
typedef struct {
  const float* keypoints;       /* DEVICE [num, 2]: keypoints[i].pt at level 0 */
  const uint8_t* descriptors;   /* DEVICE [num, descriptor_bytes], rows back to back, 16-byte aligned */
  int32_t num;                  /* >= 0 */
  int32_t descriptor_bytes;     /* 32 (ORB, OrbDetector) or 64 (BRISK, BriskDetector); else DFK_ERR_UNSUPPORTED */
} DfkFeatureSet;

/* One factor k0 -> k1 of a matching batch: the arguments of ReprojectionFactor's constructor
 * (reprojection_factor.cpp:56-65).  dfk_hamming_match_batch reads query and train only. */
typedef struct {
  DfkFeatureSet query;          /* k0: kf->features (<= DFK_MATCH_MAX_QUERIES features) */
  DfkFeatureSet train;          /* k1: fr->features, same descriptor_bytes */
  DfkCamera cam;                /* level 0: K of cam_.Matrix<double>() (:61-62); fx, fy != 0 */
  float max_dist;               /* rep_max_dist (30) */
  int32_t max_iterations;       /* rep_ransac_maxiters (1000), in [1, DFK_MATCH_MAX_ITERATIONS] */
  double threshold;             /* rep_ransac_threshold (1e-4f), > 0 */
  double probability;           /* 0.99 (matching.h:48-50), in (0, 1) */
  uint64_t seed;                /* the item's sample generator (dfk_reprojection_match_batch) */
} DfkMatchItem;
#define DFK_MATCH_MAX_QUERIES 8192
#define DFK_MATCH_MAX_ITERATIONS 1000000

/* cv::BFMatcher(cv::NORM_HAMMING).match(kf desc, fr desc) (reprojection_factor.cpp:56-58) for every item: for query q
 * of item i, matches_dev[o_i + q] = (argmin_j popcount(d0[q] ^ d1[j]), that distance), ties to the lowest j (as
 * OpenCV), (-1, -1) when the train set is empty.  o_i = query.num of the items before i.  matches_dev: DEVICE, int32
 * pairs, sum of query.num entries.  One launch (none when every query set is empty), one CTA per 128 queries of an item,
 * train descriptors tiled through shared memory.  Asynchronous on the handle's stream.  Every item is validated before
 * anything is enqueued (1 <= n <= 65535, descriptor sizes, non-NULL and aligned pointers); a rejected call writes
 * nothing and dfk_last_error names the item. */
DfkStatus dfk_hamming_match_batch(DfkHandle h, const DfkMatchItem* items, int n, int32_t* matches_dev);

/* The match list of every item's ReprojectionFactor: its three steps (reprojection_factor.cpp:56-65) on the device.
 *   1. matching      dfk_hamming_match_batch; the RANSAC runs over all query.num matches (a match per query)
 *   2. RANSAC        PruneMatchesEightPoint (features/matching.cpp:75-128), opengv's EIGHTPT relative-pose RANSAC
 *                    restated deterministically:
 *      bearings      f = normalize([(u - u0) / fx, (v - v0) / fy, 1]) in fp64 for both views (matching.cpp:39-58)
 *      samples       hypothesis h in [0, max_iterations) takes 8 distinct matches from splitmix64 of (seed, h): draw
 *                    k = 0, 1, ... is r = mix(mix(seed + G (h + 1)) + G (k + 1)), index = ((r >> 32) * N) >> 32,
 *                    G = 0x9E3779B97F4A7C15, mix = splitmix64's finaliser, repeats skipped; a hypothesis whose 8
 *                    indices take more than 256 draws is invalid.  The batch position does not enter: an item's
 *                    output depends on the item alone.
 *      model (fp64)  E = null vector of the 8 x 9 system f1^T E f0 = 0 (Householder QR); invalid if the system has
 *                    rank < 8.  E -> U diag(1, 1, 0) V^T, and of (U W V^T, +-u3), (U W^T V^T, +-u3) the one with the
 *                    most sample points in front of both cameras, ties to the first (X1 = R X0 + t).
 *      score (fp64)  opengv's: the midpoint triangulation reprojected into both views as unit vectors,
 *                    (1 - f0 . p0) + (1 - f1 . p1); an inlier scores < threshold.  An invalid hypothesis has 0 inliers.
 *      selection     the sequential adaptive loop: in order of h, strictly more inliers replace the best, then
 *                    k = log(1 - p) / log(1 - w^8), w = best / N, 1 - w^8 clamped to [2^-52, 1 - 2^-52]; stop after
 *                    h when h + 1 >= k, or at max_iterations.  Every hypothesis is scored on the device in parallel
 *                    and the loop runs as a scan over the counts: its result is the sequential loop's.
 *      fewer than 8 matches (or none with an inlier): the item yields no matches -- OptimizeRep::ConstructFactors
 *                    drops such a factor (df_work.cpp:336).
 *   3. pruning       PruneMatchesByThreshold (matching.cpp:29-37): the best hypothesis' inliers with distance
 *                    <= max_dist, sorted by (distance, query index).  std::sort leaves equal distances unordered
 *                    there; the order changes only the summation order of the factor's rows.
 * Outputs (DEVICE, int32): matches_dev rows (query, train, distance), item i's list at row o_i (as in
 * dfk_hamming_match_batch), its length in counts_dev[i]; ransac_dev (may be NULL) [n x 3] = (selected hypothesis or -1,
 * its inlier count, hypotheses evaluated).  Four launches for the whole batch (matching, hypotheses, selection,
 * compaction), no atomics: deterministic.  Asynchronous on the handle's stream; validation as dfk_hamming_match_batch,
 * plus the camera and RANSAC parameters. */
DfkStatus dfk_reprojection_match_batch(DfkHandle h, const DfkMatchItem* items, int n, int32_t* matches_dev,
                                       int32_t* counts_dev, int32_t* ransac_dev);

/* ------------------------------------------------------------------ ORB features of a keyframe or frame */

/* One image of an ORB batch: the reference's OrbDetector (features/feature_detection.h), i.e.
 * cv::ORB::create(nfeatures, scale_factor, 1): rep_nfeatures = 500, one pyramid level (rep_nlevels = 1, which makes
 * scale_factor irrelevant), edgeThreshold = patchSize = 31, WTA_K = 2, HARRIS_SCORE. */
typedef struct {
  DfkImage image;               /* DEVICE uint8 gray image (outframe_gray of PreprocessImage), width and height <=
                                   DFK_ORB_MAX_SIDE, pitch_bytes >= width; below 63 x 63 it has no features */
  int32_t nfeatures;            /* in [1, DFK_MATCH_MAX_QUERIES] */
  int32_t fast_threshold;       /* FAST threshold t in [0, 255] (cv::ORB's default 20) */
  int32_t capacity;             /* output rows reserved for the image, >= nfeatures */
} DfkOrbItem;
#define DFK_ORB_MAX_SIDE 16384

/* cv::ORB::detectAndCompute of every item with one pyramid level, bit for bit (DESIGN.md section 4.9):
 *   1. FAST-9    a pixel whose 16-pixel circle of radius 3 lies inside the image is a corner when 9 contiguous circle
 *                pixels are all > I + t or all < I - t; score = (the largest, over the 16 arcs of 9 and both signs, of
 *                the arc's smallest difference) - 1.  A corner survives when its score is strictly greater than each
 *                of its 8 neighbours' (a non-corner counts as 0): cv::FastFeatureDetector(t, true).
 *   2. border    31 <= x < W - 31, 31 <= y < H - 31.
 *   3. first cut KeyPointsFilter::retainBest(2 nfeatures) by FAST score: every corner scoring at least the
 *                (2 nfeatures)-th largest score is kept, ties included.
 *   4. Harris    integer a = sum Ix^2, b = sum Iy^2, c = sum Ix Iy over the 7 x 7 block around the corner, Ix, Iy
 *                ORB's 3 x 3 derivatives; r = ((float)a b - (float)c c - 0.04f (a + b) (a + b)) s^4 in fp32 in that
 *                order, s = 1 / (4 * 7 * 255).
 *   5. second cut retainBest(nfeatures) by r, ties included: more than nfeatures keypoints can come out.
 *   6. angle     the intensity centroid over the radius-15 disc (ORB's umax rows): integer moments m10, m01,
 *                angle = cv::fastAtan2(m01, m10) in degrees, fp32.
 *   7. rBRIEF    256 bits; bit j = B[c + rot(p0_j)] < B[c + rot(p1_j)], byte j / 8, bit j % 8.  B is the image
 *                blurred by the 7-tap Gaussian of sigma 2 (fp64 taps of cv::getGaussianKernel(7, 2), separable, rows
 *                first, rounded half to even); rot rounds (x cos - y sin, x sin + y cos) in fp32 with rint, cos and sin
 *                of angle * (float)(pi / 180).  The pairs p are OpenCV's bit_pattern_31_.
 *   8. order     by response descending, then y, then x (cv::ORB's own order is an artefact of std::nth_element).
 * Outputs (DEVICE), item i's rows at o_i = the sum of the capacities of the items before i:
 *   keypoints_dev   float [rows, 2]: the corner's integer (x, y), as KeyPoint::pt
 *   descriptors_dev uint8 [rows, 32], 16-byte aligned: a slice (keypoints_dev + 2 o_i, descriptors_dev + 32 o_i,
 *                   counts_dev[i]) is the DfkFeatureSet of the image
 *   angles_dev      float [rows] degrees, may be NULL;  responses_dev float [rows], may be NULL
 *   counts_dev      int32 [n]: the true count; when ties push it past capacity only the first capacity rows are written
 * Rows past an item's count are not written.  Seven kernels and one memset for the whole batch; integer atomics only
 * count, every position comes from a scan or a sort: deterministic, and an item's output depends on the item alone.
 * Asynchronous on the handle's stream.  Every item is validated before anything is enqueued (1 <= n <= 65535, the
 * image, nfeatures, fast_threshold, capacity, non-NULL and aligned pointers); a rejected call writes nothing and
 * dfk_last_error names the item. */
DfkStatus dfk_orb_detect_batch(DfkHandle h, const DfkOrbItem* items, int n, float* keypoints_dev,
                               uint8_t* descriptors_dev, float* angles_dev, float* responses_dev, int32_t* counts_dev);

/* One image of an ORB pyramid batch: cv::ORB::create(nfeatures, scale_factor, nlevels) (the reference's OrbDetector
 * with rep_nlevels > 1): firstLevel 0, edgeThreshold = patchSize = 31, WTA_K = 2, HARRIS_SCORE. */
typedef struct {
  DfkImage image;               /* as DfkOrbItem.image */
  int32_t nfeatures;            /* in [1, DFK_MATCH_MAX_QUERIES], shared out among the levels */
  float scale_factor;           /* s: finite, > 1 (cv::ORB's requirement) */
  int32_t nlevels;              /* L in [1, DFK_ORB_MAX_LEVELS] */
  int32_t fast_threshold;       /* in [0, 255] */
  int32_t capacity;             /* output rows reserved for the image, >= nfeatures */
} DfkOrbPyramidItem;
#define DFK_ORB_MAX_LEVELS 16

/* cv::ORB::detectAndCompute with L levels of every item, bit for bit (DESIGN.md section 4.9):
 *   budgets  f = (float)(1 / s), d = nfeatures (1 - f) / (1 - (float)f^L) in fp32; levels 0 .. L - 2 get cvRound(d)
 *            (d *= f after each), the last max(nfeatures - their sum, 0).
 *   levels   level k has scale s_k = (float)pow(s, k) and size (cvRound((float)W / s_k), cvRound((float)H / s_k)); level
 *            0 is the image, level k >= 1 is level k - 1 resized as cv::resize(level k - 1, size_k,
 *            INTER_LINEAR_EXACT): per side, ratio = dst / src and t = (1 / ratio) (d + 0.5) - 0.5 in fp64, source
 *            floor(t) with weight rint(256 (t - floor(t))) of the next pixel (clamped to the edge pixel outside), row
 *            sums in 1/256, the column sum rounded once from 1/65536, half up.
 *   detect   steps 1-7 of dfk_orb_detect_batch on each level with the level's budget.  A level below 63 x 63 (and every
 *            level after it) has no features and is not built.
 *   output   levels ascending, each in dfk_orb_detect_batch's order; a row's keypoint is the level's integer (x, y)
 *            times s_k in fp32 (KeyPoint::pt at level 0; KeyPoint::size would be 31 s_k), its octave k.
 * Outputs (DEVICE) as dfk_orb_detect_batch, item i's rows at o_i = the sum of the capacities of the items before i;
 * octaves_dev int32 [rows], may be NULL.  counts_dev[i] is the true count, the sum of the levels' counts; when ties
 * push it past capacity only the first capacity rows (lower levels first) are written.  One memset and seven kernels
 * detect every (image, level) at once, one resize launch per level builds that level of every image, and a gather
 * kernel places the rows; no floating-point atomics: deterministic, and an item's output depends on the item alone.
 * With L = 1 the rows are dfk_orb_detect_batch's.  Asynchronous on the handle's stream.  Every item is validated
 * before anything is enqueued (1 <= n, the sum of the items' levels <= 65535, and the fields above); a rejected call
 * writes nothing and dfk_last_error names the item and the field. */
DfkStatus dfk_orb_detect_pyramid_batch(DfkHandle h, const DfkOrbPyramidItem* items, int n, float* keypoints_dev,
                                       uint8_t* descriptors_dev, float* angles_dev, float* responses_dev,
                                       int32_t* octaves_dev, int32_t* counts_dev);

/* ------------------------------------------------------------------ cu_image_proc free functions */

/* df::UpdateDepth (cu_image_proc.h:41-44, cu_image_proc.cpp:248-277):
 * dpt = avg/(prx_orig + prx_jac . code) - avg.  code is HOST memory. Asynchronous. */
DfkStatus dfk_update_depth(DfkHandle h, const float* code, int code_size, const DfkImage* prx_orig,
                           const DfkImage* prx_jac, float avg_dpt, const DfkImage* dpt_out);
/* One depth decode of dfk_update_depth_batch, e.g. one (keyframe, level): dpt = avg/(prx_orig + prx_jac . code) - avg.
 * code is a HOST pointer to code_size floats. */
typedef struct {
  DfkImage prx_orig, prx_jac;
  DfkImage dpt; /* out */
  const float* code;
} DfkDepthDecodeItem;
/* n dfk_update_depth calls in one launch (the per-level UpdateDepth loop of Mapper::BuildKeyframe, mapper.cpp:984-991, for
 * many keyframes at once), avg_dpt = the handle's DenseSfmParams::avg_dpt.  Item i is bit for bit
 * dfk_update_depth(h, items[i].code, code_size, &prx_orig, &prx_jac, avg_dpt, &dpt).  The codes go up in one copy.
 * 1 <= n <= 65535.  Asynchronous on the handle's stream. */
DfkStatus dfk_update_depth_batch(DfkHandle h, const DfkDepthDecodeItem* items, int n, int code_size);
/* df::SobelGradients (cu_image_proc.h:27-29, cu_image_proc.cpp:57-113). Asynchronous. */
DfkStatus dfk_sobel_gradients(DfkHandle h, const DfkImage* img, const DfkImage* grad);
/* df::GaussianBlurDown (cu_image_proc.h:31-33, cu_image_proc.cpp:134-184). Asynchronous. */
DfkStatus dfk_gaussian_blur_down(DfkHandle h, const DfkImage* in, const DfkImage* out);
/* The image half of Frame::FillPyramids / BuildKeyframe (core/mapping/frame.h:80-94, mapper.cpp:935-949):
 * imgs[0] is the input; imgs[l] = GaussianBlurDown(imgs[l-1]) and, when grads != NULL, grads[l] =
 * SobelGradients(imgs[l]) for every level.  2*levels-1 launches enqueued back to back on the handle's stream, no host
 * synchronization (the reference synchronizes after each and re-uploads the kernel taps with cudaMemcpyToSymbol,
 * cu_image_proc.cpp:103-112,174-183). */
DfkStatus dfk_build_image_pyramid(DfkHandle h, const DfkImage* imgs, const DfkImage* grads, int levels);
/* df::SquaredError (cu_image_proc.h:35-39, cu_image_proc.cpp:190-242). Synchronous. */
DfkStatus dfk_squared_error(DfkHandle h, const DfkImage* a, const DfkImage* b, float* out);

/* ------------------------------------------------------------------ camera frame preprocessing */

/* One camera frame of dfk_preprocess_batch: DeepFactors::PreprocessImage (core/deepfactors.cpp:634-680) and the image
 * pyramid of UploadLiveFrame / Frame::FillPyramids / Mapper::BuildKeyframe (deepfactors.cpp:616-630, mapper.cpp:935-949)
 * for one frame. */
typedef struct {
  DfkImage src;           /* DEVICE uint8 x 3 interleaved camera frame, width x height in pixels, both in
                             [1, DFK_ORB_MAX_SIDE], pitch_bytes >= 3 * width */
  DfkCamera src_cam;      /* the camera at the source's size (orig_cam_ after ResizeViewport(cols, rows)); fx, fy
                             finite and != 0, u0, v0 finite; its width and height are not used */
  DfkCamera out_cam;      /* the network camera (netcfg_.camera); fx, fy finite and != 0, u0, v0 finite; width x height
                             (whole numbers in [1, DFK_ORB_MAX_SIDE]) is the output size W_o x H_o */
  DfkImage color;         /* out: DEVICE uint8 x 3, W_o x H_o, pitch_bytes >= 3 W_o (kf->color_img); ptr NULL: not
                             wanted */
  DfkImage gray;          /* out: DEVICE uint8, W_o x H_o, pitch_bytes >= W_o; ptr NULL: not wanted.  DfkOrbItem.image
                             takes it as it is */
  const DfkImage* levels; /* HOST array of num_levels DEVICE float views: level 0 is W_o x H_o, level l is
                             (W_{l-1} / 2) x (H_{l-1} / 2) (integer halving, at least 1 x 1); NULL when num_levels = 0 */
  const DfkImage* grads;  /* HOST array of num_levels DEVICE 2-float views of the levels' sizes, or NULL: no gradients */
  int32_t normalize;      /* 1: normalise level 0 by the frame's mean and standard deviation (opts_.normalize_image);
                             0: off (the reference's default) */
} DfkPreprocessItem;

/* For every item, each output pixel (j, r) of W_o x H_o (DESIGN.md section 4.10):
 *   1. map       cv::initUndistortRectifyMap(K_in, no distortion, I, K_out, size, CV_32FC1) (deepfactors.cpp:641-645), fp64
 *                without FMA contraction: K_in, K_out the pinhole matrices of src_cam and out_cam (fp32 widened),
 *                iR = K_out^-1 as cv::Mat::inv(DECOMP_LU) gives it for 3 x 3 (1 / det3 times the adjugate);
 *                x = (r iR01 + iR02) + j iR00, y = (r iR11 + iR12) + j iR10, w = (r iR21 + iR22) + j iR20,
 *                u = (float)(fx_in (x (1 / w)) + u0_in), v = (float)(fy_in (y (1 / w)) + v0_in).
 *   2. fixed     X = rint(u * 32) (fp32 product, half to even, saturated to int), x0 = X >> 5, tx = X & 31; same for Y.
 *   3. weights   cv::remap's INTER_LINEAR table: f = t (1 / 32.f), (1 - f, f) per axis in fp32; tap (dy, dx) in the
 *                order (0,0), (0,1), (1,0), (1,1) weighs rint((float)(wy_dy wx_dx) 32768); a sum != 32768 would be
 *                fixed on the first largest (sum < 32768) or first smallest tap (it never is, for bilinear).
 *   4. colour    cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) (deepfactors.cpp:648-650): per channel s = sum_k w_k
 *                src(x0 + dx, y0 + dy), a tap outside the source reads 0, out = clamp((s + 2^14) >> 15, 0, 255).
 *   5. gray      cv::cvtColor(COLOR_RGB2GRAY) on 8U (:653-654): g = (9798 c0 + 19235 c1 + 3735 c2 + 2^14) >> 15.
 *                Channel 0 takes the R weight, as the reference calls it, whatever order the camera delivers.
 *   6. float     convertTo(CV_32FC1, 1 / 255.0) (:657-658): f = (float)g * (float)(1 / 255.0).
 *   7. normalise (normalize = 1; :660-665) mu = S1 / N, sigma = sqrt(max(S2 / N - mu^2, 0)), N = W_o H_o, S1 and S2
 *                the fp64 sums of f and f^2 in a fixed order (32 x 8 pixel tiles in row-major order, a pairwise tree of
 *                256 within a tile, the tile sums strided over 256 and the same tree); level 0 = (float)((f - mu) /
 *                sigma).  cv::meanStdDev's own summation order is not reproducible, so mu and sigma agree with it to
 *                1e-12 relative (the bound the tests check), not bit for bit.  sigma = 0 (a constant frame) is not
 *                guarded, as in the reference: level 0 is then +-inf, or NaN where f = mu.
 *   8. pyramid   levels[0] = f (or f'), levels[l] = GaussianBlurDown(levels[l-1]), grads[l] = SobelGradients(levels[l])
 *                for every level, level 0 included (UploadLiveFrame skips it; dfk_build_image_pyramid does not); each
 *                bit for bit dfk_gaussian_blur_down / dfk_sobel_gradients of that image alone.
 * Steps 1-6 are bit for bit OpenCV 4.13.  stats_dev (DEVICE double [n, 2], may be NULL): row i = (mu, sigma) of a
 * normalising item; rows of the other items are not written.  One kernel for steps 1-6 of every item, two more when an
 * item normalises (the statistics, once per item, then level 0), then for the whole batch one blur-down launch per
 * level past 0 and, when an item has gradients, one Sobel launch per level.  Deterministic; an item's output depends on
 * the item alone.  Asynchronous on the handle's stream.  Every item is validated before anything is enqueued
 * (1 <= n <= 65535, 0 <= num_levels <= DFK_PREPROCESS_MAX_LEVELS, at most 2^31 - 1 tiles of 32 x 8 output pixels over
 * the normalising items, the views, sizes and cameras above, normalize 0 or 1, stats_dev 8-byte aligned); a rejected
 * call writes nothing and dfk_last_error names the item. */
DfkStatus dfk_preprocess_batch(DfkHandle h, const DfkPreprocessItem* items, int n, int num_levels, double* stats_dev);
/* the most levels a frame of sides <= DFK_ORB_MAX_SIDE has: 16384, 8192, ..., 1 */
#define DFK_PREPROCESS_MAX_LEVELS 15

/* ------------------------------------------------------------------ keyframe meshes (the dense map) */

/* The keyframe renderer's parameters (gui/visualizer.cpp:657-661, the defaults in brackets). */
typedef struct {
  float stdev_thresh;          /* [4.2] a pixel with sqrt(2) exp(log-stdev) > stdev_thresh is noisy; finite */
  float slt_thresh;            /* [0] a quad whose triangle normals meet the pixel's ray at |cos| < slt_thresh is
                                  dropped; finite */
  int32_t crop_pix;            /* [20] quads within crop_pix of the image edge are skipped; >= 0 */
  int32_t draw_noisy_pixels;   /* [0] 1: noisy pixels stay valid and are coloured (255, 0, 0); 0 or 1 */
} DfkKeyframeMeshParams;

/* One keyframe of dfk_keyframe_mesh_batch.  W x H = cam.width x cam.height (whole numbers in [1, DFK_ORB_MAX_SIDE]) is
 * the size of every view.  The depth is dpt, or the decode of (prx_orig, prx_jac, code): set exactly one of dpt.ptr
 * and the three decode fields. */
typedef struct {
  DfkImage dpt;                /* DEVICE float depth (kf->pyr_dpt level 0), or ptr NULL: decode */
  DfkImage prx_orig, prx_jac;  /* DEVICE float proximity and its code Jacobian (code_size floats per pixel) */
  const float* code;           /* HOST code_size floats */
  DfkImage std;                /* DEVICE float log-stdev (kf->pyr_stdev level 0); ptr NULL: no pixel is noisy */
  DfkImage valid;              /* DEVICE float validity (kf->pyr_vld level 0); ptr NULL: every pixel passes */
  DfkImage color;              /* DEVICE uint8 x 3 (kf->color_img, dfk_preprocess_batch's color), pitch_bytes >= 3 W;
                                  ptr NULL: none (then colors_dev must be NULL) */
  DfkCamera cam;               /* the keyframe's camera: fx, fy finite and != 0, u0, v0 finite */
  float pose_wk[7];            /* kf->pose_wk: quaternion (x, y, z, w), translation; finite */
  int32_t vertex_capacity;     /* output vertex rows reserved for the item, >= 0 */
  int32_t triangle_capacity;   /* output triangle rows reserved for the item, >= 0 */
  DfkImage depth_u16;          /* out: DEVICE uint16 W x H, pitch_bytes even and >= 2 W (SaveKeyframes' depth image);
                                  ptr NULL: not wanted */
} DfkKeyframeMeshItem;

/* What drawkf.geom (gui/shaders/drawkf.geom) draws for each item, as a world-frame mesh (DESIGN.md section 4.12).
 * Every value is fp32 without FMA contraction, except tau below.
 *   depth      d = dpt, or bit for bit dfk_update_depth_batch's decode of the item (avg_dpt = the handle's
 *              DenseSfmParams::avg_dpt), each pixel decoded once; 1 <= code_size <= 256 when an item decodes.
 *   pixel      (x, y) is invalid when !(vld > 0) (a NaN vld included), d < 0.5 or d > 10 or d is NaN, or x < 4,
 *              x > W - 4, y < 4 or y > H - 4 (:55-88).  It is noisy when (double)s > tau, s its log-stdev and
 *              tau = log((double)stdev_thresh / sqrt(2.0)) in fp64 (-inf for stdev_thresh <= 0); a NaN s is not noisy.
 *              A noisy pixel is invalid, or with draw_noisy_pixels stays valid with colour (255, 0, 0).  A pixel
 *              outside the image has depth 0 and is invalid.
 *   quad       at (x, y) for every pixel: skipped when x < crop, x > W - crop, y < crop or y > H - crop (:97-99).  Its
 *              corners tr = (x, y), tl = (x - 1, y), br = (x, y + 1), bl = (x - 1, y + 1) lift to p = ((x - u0) / fx d,
 *              (y - v0) / fy d, d); n1 = n(tr, tl, br), n2 = n(tl, bl, br) with n(a, b, c) = normalize(cross(c - a,
 *              b - a)), r = normalize(((x - u0) / fx, (y - v0) / fy, 1)); dropped when |n1 . r| < slt_thresh or
 *              |n2 . r| < slt_thresh (:113-125).  normalize divides each component by sqrtf((v.x v.x + v.y v.y) +
 *              v.z v.z); dot products sum in the same order; a NaN fails every comparison.
 *   triangles  T1 = (tr, tl, br) when tr, tl, br are valid; T2 = (br, tl, bl) when tl, br, bl are valid (:152-183); quads
 *              in row-major order, T1 before T2; corners are item-local vertex indices.
 *   vertices   the pixels that are a corner of an emitted triangle, in row-major order: position pose_wk * p;
 *              colour the color bytes (or (255, 0, 0)); normal R_wk ((n1 + n2) 0.5) of the quad at the vertex's own
 *              (x, y), not renormalised; pixel index y W + x.
 *   u16        depth_u16 = cv::Mat::convertTo(CV_16UC1, 5000) of d (core/deepfactors.cpp:560): (float)(d * 5000),
 *              rounded half to even, saturated to [0, 65535]; a NaN or a product beyond int32 gives 0 (cvRound on x86).
 * Deviations from the shader: T2 keeps T1's winding (the strip flips it when tr is invalid); the normal is in the world
 * frame (the shader's is in clip space, after mvp, :134-136); a NaN depth is invalid (the shader emits a NaN vertex).
 * Outputs (DEVICE), item i's vertex rows at the sum of vertex_capacity over the items before it, its triangle rows
 * likewise:
 *   positions_dev  float [vertex rows, 3]            normals_dev  float [vertex rows, 3], may be NULL
 *   colors_dev     uint8 [vertex rows, 3], may be NULL (then every item needs a color view)
 *   pixels_dev     int32 [vertex rows], may be NULL  triangles_dev int32 [triangle rows, 3], may be NULL
 *   counts_dev     int32 [n, 2]: the item's true vertex and triangle counts
 * An item whose vertex or triangle count exceeds its capacity writes its two counts and nothing else (no rows, no
 * depth_u16); the other items are unaffected.  Rows past a count are not written.  Three kernels over every (tile, item), after one depth
 * decode launch when an item decodes; integer scans only: deterministic, and an item's output depends on the item
 * alone.  Asynchronous on the handle's stream.  Every item is validated before anything is enqueued (1 <= n <= 65535,
 * the sizes, views, camera, pose, capacities and their sums <= 2^31 - 1, the parameters, 4-byte aligned float and int
 * outputs); a rejected call writes nothing and dfk_last_error names the item and the field. */
DfkStatus dfk_keyframe_mesh_batch(DfkHandle h, const DfkKeyframeMeshItem* items, int n, int code_size,
                                  const DfkKeyframeMeshParams* params, float* positions_dev, float* normals_dev,
                                  uint8_t* colors_dev, int32_t* pixels_dev, int32_t* triangles_dev, int32_t* counts_dev);

/* ------------------------------------------------------------------ loop-closure candidates (DBoW2 retrieval) */

/* The bag-of-words retrieval of LoopDetector (core/system/loop_detector.cpp:38-44, 96-112): DBoW2 (commit 3924753)
 * TemplatedVocabulary::transform / score and TemplatedDatabase::add / query with TF_IDF weighting and L1_NORM scoring,
 * no direct index (TemplatedDatabase(voc, false, 0)).  DBoW2 is not vendored; this block is its specification
 * (DESIGN.md section 4.11).  Every value is fp64 and every sum runs in the order stated; nothing is reassociated.
 *   1. vocabulary  node 0 is the root and is not listed; the listed nodes have an id, a parent id, a weight (the idf)
 *                  and a descriptor.  A node's children are in the order the nodes are listed.  A leaf is a node with no
 *                  children; each word names one leaf.
 *   2. word        of a descriptor: from the root, step to the child at the smallest Hamming distance (popcount over
 *                  all descriptor_bytes), strict < in children order (a tie goes to the first child), until a leaf; the
 *                  result is the leaf's word id and weight.
 *   3. vector      a map ordered by word id.  Features in input order; one whose weight is > 0 is added, v[id] += w (the
 *                  first occurrence inserts w, so a word seen n times holds w added n times in sequence, not n w); one
 *                  whose weight is not > 0 is skipped.  Then L1 normalisation: norm = the sum of fabs(value) in
 *                  ascending word order, from 0.0; if norm > 0 every value becomes value / norm.  (No division by the
 *                  word count: L1 scoring normalises.)
 *   4. database    add gives entry ids 0, 1, 2, ... in the order vectors are added; clear empties it.
 *   5. query       (queryL1) for each query word in ascending order and each entry e holding it with e < max_id or
 *                  max_id = -1: t = fabs(q - d) - fabs(q) - fabs(d) (q the query's value, d the entry's).  Per entry the
 *                  first t initialises the sum, later ones are added in word order; only entries with a common word
 *                  appear.  Sorted ascending by sum, cut to max_results, Score = -sum / 2.0.
 *                  Deviation: DBoW2's std::sort leaves the order of equal sums unspecified; here equal sums go in
 *                  ascending entry id.
 *   6. score       (L1Scoring::score(a, b)) a and b merged in ascending word order; from 0.0, each common word adds
 *                  fabs(vi - wi) - fabs(vi) - fabs(wi), vi from a and wi from b; the result is -score / 2.0.  This is not
 *                  the query's operand order, and the two round differently.  Vectors with no common word score -0.0, bit
 *                  for bit DBoW2's result.
 * Only weighting TF_IDF (0) and scoring L1_NORM (0) are implemented; any other is DFK_ERR_UNSUPPORTED. */
#define DFK_BOW_MAX_DEPTH 16
#define DFK_BOW_MAX_NODES 4194304
#define DFK_BOW_WEIGHTING_TF_IDF 0
#define DFK_BOW_SCORING_L1 0

/* A vocabulary as DBoW2's text format lists it.  All arrays are HOST memory, read during dfk_bow_vocabulary_create. */
typedef struct {
  int32_t k;                    /* branching factor, in [1, 32] */
  int32_t L;                    /* depth levels, in [1, DFK_BOW_MAX_DEPTH] */
  int32_t weighting;            /* weightingType: DFK_BOW_WEIGHTING_TF_IDF only */
  int32_t scoring;              /* scoringType: DFK_BOW_SCORING_L1 only */
  int32_t descriptor_bytes;     /* 32 (ORB), 48 (BRISK, the reference's small_voc) or 64 */
  int32_t num_nodes;            /* N, the listed nodes (the root excluded), in [1, DFK_BOW_MAX_NODES] */
  const int32_t* node_ids;      /* [N] in file order: a permutation of 1..N */
  const int32_t* parent_ids;    /* [N] 0 (the root) or a listed id */
  const double* weights;        /* [N] finite and >= 0 */
  const uint8_t* descriptors;   /* [N, descriptor_bytes] */
  int32_t num_words;            /* W >= 1 */
  const int32_t* word_ids;      /* [W] a permutation of 0..W-1 */
  const int32_t* word_nodes;    /* [W] the leaf each word names */
} DfkBowVocabularyDesc;

typedef struct DfkBowVocabulary DfkBowVocabulary;
typedef struct DfkBowDatabase DfkBowDatabase;

/* Validates the whole tree (the ids and word ids are permutations; every parent exists, there is no cycle and every
 * node is reachable from the root; each node has <= k children and depth <= L; every leaf has exactly one word and no
 * internal node has one; the weights are finite and >= 0) and uploads it re-indexed so that each node's children are
 * consecutive rows in their original order.  Synchronous.  A rejected call creates nothing, and dfk_last_error names
 * the node, word or field. */
DfkStatus dfk_bow_vocabulary_create(DfkHandle h, const DfkBowVocabularyDesc* desc, DfkBowVocabulary** out);
DfkStatus dfk_bow_vocabulary_destroy(DfkHandle h, DfkBowVocabulary* voc);

/* A bag-of-words vector on the device: count (a DEVICE pointer, e.g. counts_dev + i of a transform) words in
 * ascending order with their values.  Nothing of it is read on the host, so a transform's output feeds the database
 * with no read-back. */
typedef struct {
  const int32_t* words;         /* DEVICE [capacity] */
  const double* values;         /* DEVICE [capacity], 8-byte aligned */
  const int32_t* count;         /* DEVICE: the word count; read as min(max(count, 0), capacity) */
  int32_t capacity;             /* >= 0 */
} DfkBowVector;

/* Steps 2-3 for every item: item i is the descriptor rows of one image (keypoints is not read: a slice of the
 * dfk_orb_detect_batch output passes as it is); descriptor_bytes must equal the vocabulary's, num in
 * [0, DFK_MATCH_MAX_QUERIES], descriptors 16-byte aligned.  Outputs (DEVICE), item i's rows at o_i = the sum of the
 * capacities before it (capacities HOST, capacities[i] >= num):
 *   words_dev          int32, the vector's words ascending;  values_dev  fp64 (8-byte aligned), their values
 *   counts_dev         int32 [n]: the vector's word count, so (words_dev + o_i, values_dev + o_i, counts_dev + i,
 *                      capacities[i]) is the item's DfkBowVector
 *   feature_words_dev  int32 (may be NULL): the word of each descriptor, -1 for one whose weight is not > 0
 * Two launches for the whole batch (descent: one warp per descriptor; assembly: one CTA per item).  Deterministic, no
 * floating-point atomics; an item's output depends on the item alone.  Asynchronous on the handle's stream.  Every item
 * is validated before anything is enqueued (1 <= n <= 65535); a rejected call writes nothing and dfk_last_error names
 * the item and field. */
DfkStatus dfk_bow_transform_batch(DfkHandle h, const DfkBowVocabulary* voc, const DfkFeatureSet* items,
                                  const int32_t* capacities, int n, int32_t* words_dev, double* values_dev,
                                  int32_t* counts_dev, int32_t* feature_words_dev);

/* An empty database (step 4).  Entries keep their words and values in device storage that grows only: an entry
 * reserves the capacity of the vector it was added from, not its count, so a transform capacity of 2 x 500 rows costs
 * 12 kB per entry however few words the image has (the slack is capacity - count rows of 12 bytes).  clear keeps the
 * storage for reuse; destroy frees it. */
DfkStatus dfk_bow_database_create(DfkHandle h, const DfkBowVocabulary* voc, DfkBowDatabase** out);
DfkStatus dfk_bow_database_destroy(DfkHandle h, DfkBowDatabase* db);
DfkStatus dfk_bow_database_clear(DfkHandle h, DfkBowDatabase* db);
/* the number of entries, known on the host (no synchronisation) */
DfkStatus dfk_bow_database_size(DfkHandle h, const DfkBowDatabase* db, int32_t* size);
/* Adds n vectors in order as entries size, size + 1, ...; *first_entry (may be NULL) receives the first id.  One
 * launch copies them on the device, ordered after earlier work on the handle's stream (a transform's output may be
 * added before it has run).  1 <= n <= 65535 and at most 2^31 - 1 entries; a rejected call adds nothing. */
DfkStatus dfk_bow_database_add(DfkHandle h, DfkBowDatabase* db, const DfkBowVector* vectors, int n,
                               int32_t* first_entry);

/* One query of dfk_bow_database_query_batch */
typedef struct {
  DfkBowVector vector;
  int32_t max_results;          /* >= 1: the rows reserved for the query */
  int32_t max_id;               /* -1 (every entry) or >= 0: entries e < max_id only */
} DfkBowQuery;

/* Step 5 for every query against the database.  Outputs (DEVICE), query i's rows at r_i = the sum of the max_results
 * before it: ids_dev int32 entry ids and scores_dev fp64 Scores (8-byte aligned), best first; counts_dev int32 [n] =
 * DBoW2's ret.size() before the cut, the number of entries with a common word.  Only min(count, max_results) rows are
 * written.  Two launches (one warp per (query, entry) for the sums; the ranks of the sums, which place each row), plus a
 * memset of counts_dev when the database is empty.  The query's words and values sit in shared memory, so a vector's
 * capacity is at most DFK_MATCH_MAX_QUERIES.  Neither kernel indexes by word id, so a malformed vector cannot read out
 * of bounds.  The ranks compare each hit with every other, so the work is n x size^2 comparisons: n x size <= 2^26
 * (the sums' scratch) and n x size^2 <= 2^36 (one query against at most 262,144 entries; 10,000 entries take about
 * 0.5 ms on an H100), and 1 <= n <= 65535; a rejected call writes nothing. */
DfkStatus dfk_bow_database_query_batch(DfkHandle h, const DfkBowDatabase* db, const DfkBowQuery* queries, int n,
                                       int32_t* ids_dev, double* scores_dev, int32_t* counts_dev);

/* One score of dfk_bow_score_batch: score(the entry's vector, vector) */
typedef struct {
  int32_t entry;                /* in [0, size) */
  DfkBowVector vector;
} DfkBowScoreItem;

/* Step 6 for every item: scores_dev[i] (DEVICE fp64, 8-byte aligned) = L1Scoring::score(a, b) with a the entry's
 * vector and b the item's, the operand order of voc_.score(curr_kf->bow_vec, live) (loop_detector.cpp:107).  One launch,
 * one warp per item.  1 <= n <= 65535; a rejected call writes nothing. */
DfkStatus dfk_bow_score_batch(DfkHandle h, const DfkBowDatabase* db, const DfkBowScoreItem* items, int n,
                              double* scores_dev);

/* ------------------------------------------------------------------ keyframe window problem (the LM loop on the device) */

/* A window problem: the keyframe window's Levenberg-Marquardt loop in the library, with the window's state (poses and
 * codes, fp64) on the device.  It holds every work item of a window once, validated and planned at create; between
 * iterations only the pose- and code-dependent fields of the items change, and a device launch rewrites them from the
 * state (bit for bit what the host staging of the batch calls computes from the same fp32-rounded poses and codes).
 *
 * State: K keyframe poses then F tracked-frame poses ((K + F) x 7, the pose convention above), then K codes (K x C).
 * Every item names the state slots it reads (DfkWindowItemSlots): a pose slot s < K is keyframe s, s >= K is frame
 * s - K; a code slot is a keyframe.  The pose and code fields of the template items are ignored.
 *
 * The descriptor describes a window in terms the ABI already has:
 *   window          from any dfk_window_create*; the problem refers to it, so it must outlive the problem
 *   dense           the photometric then the frame (pair, level) items in record order (DfkSfmWorkItem, fused depth
 *                   decode: prx_orig required, dpt0 is the output), with slots (pose0, pose1, code0); record i of
 *                   records_dev
 *   reproj          the reprojection links (DfkReprojectionItem), slots (pose0, pose1, code0); record num_dense + j of
 *                   records_dev (unscaled records, as the window expects them)
 *   geo             the sparse geometric links (DfkSparseGeometricItem), slots (pose0, pose1, code0, code1); record j of
 *                   geo_records_dev
 *   depth           the depth decodes of the error path (DfkDepthDecodeItem, e.g. one per (keyframe, level)), slot
 *                   code0; their dpt views give the size only: the problem decodes into depth scratch of its own
 *   error           the error items (DfkSfmWorkItem without code), slots (pose0, pose1); error_depth[i] is the depth
 *                   item whose decode item i reads (its dpt0 view is ignored)
 *   frame priors    num_frame_priors DFK_PRIOR_DOUBLES(C) rows on keyframes frame_prior_kf, frozen at frame_prior_x0
 *                   ([pose 7 | code C] doubles each)
 *   keyframe priors the window's keyframe priors (dfk_window_create_priors) as dfk_window_add_keyframe_priors takes
 *                   them, frozen at kf_prior_x0 ([pose 7 | code C] doubles per member, prior by prior)
 * Every array is HOST memory and copied, except records_dev / geo_records_dev (DEVICE, the caller's record buffers,
 * which linearize writes and which must outlive the problem).  The image views are the caller's and must outlive it.
 * Create validates every item as the batch calls do, plans the RunStep launch and takes the handle's settings: its Gram
 * mode, SM limit and every DenseSfmParams value (valid_border, min_dpt, avg_dpt, huber_delta) at create hold for every
 * later call of the problem, for all its factor kinds (the RunStep kernel chosen at create also serves every active
 * subset of dfk_window_problem_set_active); later dfk_sfm_set_params / dfk_sfm_set_gram_mode /
 * dfk_set_sm_limit calls do not change it.  An error item must not ask for a fused decode (code NULL).  Create uploads the item arrays, which the problem owns with their code
 * slots and ray tables (no pointer into the handle's shared scratch), creates the solver with the first pose fixed and
 * allocates the depth scratch of the error path.  A rejected create writes nothing. */
typedef struct DfkWindowProblem DfkWindowProblem;
typedef struct {
  int32_t pose0, pose1, code0, code1; /* state slots; -1 where an item kind does not read one */
} DfkWindowItemSlots;
typedef struct {
  const DfkWindow* window;
  int32_t num_dense;
  const DfkSfmWorkItem* dense;
  const DfkWindowItemSlots* dense_slots;
  int32_t num_reproj;
  const DfkReprojectionItem* reproj;
  const DfkWindowItemSlots* reproj_slots;
  int32_t num_geo;
  const DfkSparseGeometricItem* geo;
  const DfkWindowItemSlots* geo_slots;
  int32_t num_depth;
  const DfkDepthDecodeItem* depth;
  const DfkWindowItemSlots* depth_slots;
  int32_t num_error;
  const DfkSfmWorkItem* error;
  const DfkWindowItemSlots* error_slots;
  const int32_t* error_depth;
  int32_t num_frame_priors;
  const int32_t* frame_prior_kf;
  const double* frame_prior_rows;
  const double* frame_prior_x0;
  const double* kf_prior_rows;
  const double* kf_prior_x0;
  float* records_dev;
  float* geo_records_dev;
} DfkWindowProblemDesc;
DfkStatus dfk_window_problem_create(DfkHandle h, const DfkWindowProblemDesc* desc, DfkWindowProblem** out);
/* h must not be NULL; p may be */
DfkStatus dfk_window_problem_destroy(DfkHandle h, DfkWindowProblem* p);
/* poses: (K + F) x 7 doubles, codes: K x C doubles, host or device memory.  Asynchronous on the handle's stream. */
DfkStatus dfk_window_problem_set_state(DfkHandle h, DfkWindowProblem* p, const double* poses, const double* codes);
DfkStatus dfk_window_problem_get_state(DfkHandle h, const DfkWindowProblem* p, double* poses, double* codes);
/* The window buffer at the state: every item re-posed from the state on the device, then the batches in the order of
 * SfmWindowProblem.linearise with every factor stale -- the dense items in one RunStep launch (depth decode fused in),
 * the reprojection links, the geometric links -- the assembly, and the frame and keyframe priors with their deltas
 * Local(x0, x) formed on the device in fp64.  window_dev: DEVICE, dfk_window_floats() floats.  Asynchronous. */
DfkStatus dfk_window_problem_linearize(DfkHandle h, DfkWindowProblem* p, float* window_dev);
/* doubles of dfk_window_problem_error's output */
#define DFK_WINDOW_ERROR_DOUBLES 7
/* The window energy at the state without linearising (SfmWindowProblem.error): out_dev (DEVICE) = [E | photometric |
 * reprojection | geometric | priors | items without inliers | total inliers], each part summed in fp64 in factor order.
 * An item with inliers adds res / inliers * W * H, one without adds 0; a link its b^T b; a prior f0 - 2 g^T d + d^T G d.
 * The keyframes' own depth and the records are not touched.  Asynchronous. */
DfkStatus dfk_window_problem_error(DfkHandle h, DfkWindowProblem* p, double* out_dev);
/* state <- retract(state, dx): t += dt, q = normalize(exp(w) q), c += dc, in fp64, for the keyframes and then the frames
 * (dx_dev: DEVICE, K (6 + C) + 6 F doubles, the solve's layout).  Asynchronous. */
DfkStatus dfk_window_problem_retract(DfkHandle h, DfkWindowProblem* p, const double* dx_dev);

/* window_opt.LMParams; lambda_up and lambda_down finite and > 0 */
typedef struct {
  int32_t iterations;
  double lambda_init, lambda_up, lambda_down, lambda_max;
  int32_t fix_first_pose;   /* 1: variables 0..5 (keyframe 0's pose) are held */
  double code_prior_weight; /* >= 0: adds 1/2 w |c|^2 to the energy and w I / -w c to the solve */
  int32_t use_error;        /* 1: evaluate E at every candidate and linearise accepted points only */
} DfkLMParams;
/* window_opt.LMTrace; the caller's HOST arrays: energy iterations + 1 entries, lambda and accepted iterations each */
typedef struct {
  double* energy;           /* accepted energies, energy[0] = the start point's */
  double* lambda;           /* the damping of every step */
  int32_t* accepted;        /* 1 for an accepted step */
  int32_t num_energies, num_steps, linearisations, error_evaluations;  /* out */
} DfkLMTrace;
/* Levenberg-Marquardt from the problem's state (window_opt.WindowOptimizer.run, the policy of its docstring); on return
 * the state is the last accepted point, and the records describe the point last linearised (without use_error, the
 * last candidate, accepted or not).  Every linearisation re-evaluates every factor (an LM step moves every code, so a
 * linearisation cache would re-evaluate everything anyway).  The state and the accepted and candidate window buffers
 * stay on the device; each step reads back the solve's info and the candidate's energy.  Synchronous. */
DfkStatus dfk_window_lm(DfkHandle h, DfkWindowProblem* p, const DfkLMParams* params, DfkLMTrace* trace);

/* Active items (coarse to fine: one pyramid level per pair at a time, as the reference's OptimizePhoto holds one
 * PhotometricFactor per pair).  dense_active: num_dense bytes, error_active: num_error bytes, both HOST memory and
 * copied; error_active may be NULL only when num_error == num_dense, and then the dense mask is used.  Nonzero = active.
 * After create every item is active.  With a mask:
 *   linearize  the RunStep launch (depth decode fused in) covers the active dense items only, planned over them, so an
 *              inactive item costs no tile; an inactive item's record is all zero (it adds nothing to f or the inliers)
 *              and its dpt0 / valid0 are not written.  The links, the assembly and the priors are unchanged.  An
 *              active item's record is bit for bit dfk_sfm_run_step_batch over the active items in record order.
 *   error      only the active error items are evaluated; an inactive one adds 0 and is counted neither as an item
 *              without inliers nor in the inlier total.
 * The masks hold for every later linearize, error, dfk_window_lm and dfk_window_lm_levels call of the problem until the
 * next set_active (dfk_window_lm_levels leaves those of its last step); all ones restores the create-time launches.
 * The re-plan is host work ordered on the handle's stream (no synchronisation).  A rejected call writes nothing. */
DfkStatus dfk_window_problem_set_active(DfkHandle h, DfkWindowProblem* p, const uint8_t* dense_active,
                                        const uint8_t* error_active);

/* The level schedule of dfk_window_lm_levels (window_opt.LevelSchedule), HOST arrays.  The schedule's pairs are the
 * distinct window pairs of the dense items (the photometric, then the frame pairs), in window order; dense item i
 * belongs to the window's item_pair[i].  Error items: with error_pair NULL (allowed when num_error == num_dense) error
 * item i belongs to dense item i's pair; with error_level NULL (same condition) it has dense item i's level. */
typedef struct {
  int32_t num_levels;
  const int32_t* iters;             /* [num_levels] >= 0: level l is active for iters[l] + 1 steps (pho_iters) */
  const int32_t* dense_level;       /* [num_dense] in [0, num_levels) */
  const int32_t* error_pair;        /* [num_error] schedule pair index, or NULL */
  const int32_t* error_level;       /* [num_error] in [0, num_levels), or NULL */
  int32_t num_pairs;                /* must equal the number of distinct pairs of the dense items */
  const int32_t* pair_steps_done;   /* [num_pairs] >= 0: steps the pair has taken (0 for a new pair) */
  const uint8_t* pair_remove_after; /* [num_pairs] nonzero: inactive once its schedule has run out; may be NULL */
} DfkLevelSchedule;
/* What dfk_window_lm_levels returns besides DfkLMTrace; the caller's HOST arrays, any may be NULL */
typedef struct {
  double* switch_energy;         /* [iterations]: the energy each switch re-linearised to */
  int32_t* pair_levels;          /* [iterations x num_pairs]: the active level of every pair at every step, -1 = off */
  int32_t* pair_steps_done;      /* [num_pairs] out: every pair's position, to continue its schedule in a later window */
  int32_t num_switches;          /* out */
} DfkLevelTrace;
/* Levenberg-Marquardt with per-pair coarse-to-fine levels: the policy of dfk_levels.h (its header comment), with
 * dfk_window_lm's accept / lambda rule and use_error.  A pair's position s is the number of steps it has taken: level
 * num_levels - 1 for its first iters[num_levels - 1] + 1 steps, and so on down to level 0; after its schedule it stays
 * at level 0, or becomes inactive with remove_after.  One LM iteration (accepted or rejected) is one step of every
 * active pair.  When lambda would exceed lambda_max, every pair above level 0 jumps to the first step of the next finer
 * level and lambda restarts at lambda_init; the run ends there only when no pair is above level 0.  Whenever the active
 * set changes, the accepted point is re-linearised under the new mask (counted in trace->linearisations) and its energy
 * becomes f.  On return the problem's mask is the one the last step used.  Synchronous. */
DfkStatus dfk_window_lm_levels(DfkHandle h, DfkWindowProblem* p, const DfkLMParams* params,
                               const DfkLevelSchedule* schedule, DfkLMTrace* trace, DfkLevelTrace* level_trace);

#ifdef __cplusplus
}
#endif
#endif /* DFK_H_ */
