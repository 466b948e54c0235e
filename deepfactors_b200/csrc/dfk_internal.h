// dfk_internal.h -- shared between the translation units of libdfk.so (not installed).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "dfk.h"
#include "dfk_preprocess_model.h"

namespace dfk {

// ---------------------------------------------------------------------------- blobs of typed parts
// A call's staged upload, or its scratch, is one blob of typed parts, each rounded up to 16 bytes: the kernels read
// int2 / int3 / uint4 / double parts.  A Part is where one part starts; the same offset addresses it from the host
// image and from the device copy.
template <class T>
struct Part {
  size_t off = 0;
  T* at(void* base) const { return reinterpret_cast<T*>(static_cast<unsigned char*>(base) + off); }
};

// The sizing pass: add() the parts in blob order; `bytes` is the blob's size
struct Layout {
  size_t bytes = 0;
  template <class T>
  Part<T> add(size_t count)
  {
    const Part<T> p{bytes};
    bytes += (sizeof(T) * count + 15) & ~(size_t)15;
    return p;
  }
};

// ----------------------------------------------------------------------------------------------
// Device-side description of one (keyframe, frame, level) evaluation.  Built on the host by
// dfk_api.cu from a DfkSfmWorkItem: the relative pose and its two 6x6 Jacobians are host work in
// the reference too (cu_sfmaligner.cpp:164-166).
// ----------------------------------------------------------------------------------------------
struct SfmItemDev {
  // pose_10 = pose1^-1 * pose0 : quaternion (x,y,z,w), translation, and the same rotation as a
  // row-major 3x3 (used only for derivative terms, never for the validity chain)
  float q[4];
  float t[3];
  float R[9];
  // camera (pinhole_camera.h:43) + validity window (pinhole_camera_impl.h:102-108)
  float fx, fy, u0, v0;
  float border;  // (float)valid_border
  float ulim;    // width  - border  (float arithmetic as in the reference)
  float vlim;    // height - border
  float min_dpt, avg_dpt, huber_delta;
  // buffers; pitches in floats
  const float* img0;
  const float* img1;
  const float* dpt0;
  float* valid0;
  const float* jac;
  const float* grad1;
  uint32_t img0_pitch, img1_pitch, dpt0_pitch, valid0_pitch, jac_pitch, grad1_pitch;
  uint32_t width, height;
  uint32_t num_pixels;
  // tiling
  uint32_t tile_begin;  // first global tile index of this item
  uint32_t num_tiles;
  uint32_t perm_mul;    // tile k of the item is processed as (k * perm_mul) % num_tiles  (k * perm_mul < 2^32)
  uint32_t mag_tiles;   // floor(2^32 / num_tiles): division by multiply-high + one correction step
  uint32_t mag_width;   // floor(2^32 / width)
  // partial-sum bookkeeping: CTA c (first_cta <= c < first_cta+num_ctas) writes slot
  // partial_begin + (c - first_cta)
  uint32_t first_cta, num_ctas, partial_begin;
  uint32_t flags;  // bit0: bulk-copy (TMA) eligible, bit1: grad1 rows are 8-byte aligned
  // fused depth decode (ITEM_FLAG_FUSED_DEPTH): `dpt0` then points at prx_orig (what the tile loader stages), the decoded
  // depth is written to dpt_out; code = code_size floats in device scratch
  float* dpt_out;
  uint32_t dpt_out_pitch;
  const float* code;
  // normalised ray table of the item's camera level (device memory cached by the handle): xn[0..width), then yn[0..height)
  const float* ray_tab;
  // relative-pose Jacobians (warping.h:120-134), row-major 6x6; used by the finalize kernel
  float P0[36];
  float P1[36];
};

enum : uint32_t { ITEM_FLAG_BULK = 1u, ITEM_FLAG_GRAD_ALIGNED = 2u, ITEM_FLAG_FUSED_DEPTH = 4u };

// Geometry of the fp32 Gram kernel, shared by host planning code and the kernel.
template <int C>
struct SfmCfg {
  static constexpr int NF = C + 7;               // features: code(C) | a(6) | r(1)
  static constexpr int NFP = (NF + 7) & ~7;      // padded to 8
  static constexpr int NB = NFP / 8;             // 8x8 blocks per side
  static constexpr int NBLK = NB * (NB + 1) / 2;  // upper-triangular blocks
  static constexpr int PARTIAL_FLOATS = NFP * NFP + 8;  // G (row major NFP x NFP) | inliers(u32) | pad
};

constexpr int kTilePixels = 256;    // fp32 kernel

// Split-tf32 product of the tensor-core kernel (dfk_sfm_tc.cu), and its partial where sfm_tc_writes_d.  Features f =
// code 0..C-1 | pose/residual C..C+6 | zero C+7 (F = C + 8), each split into h (tf32) and l.  The first S = C - 8 code
// features have their l rows in A, the last 8 code features and the pose/zero group in B:
//   A rows    = code-l 0..S-1 | h 0..F-1                        (M = 2C)
//   B columns = h 0..F-1 | code-l S..C-1 | pose-l (7 + zero)    (N = C + 24)
// The accumulator D = A B^T is stored column-major ([column][row]), then the inlier count:
//   HH[i][j] = D[S + i][j];   LH[i][j] = D[i][j] for i < S,  D[S + j][16 + i] for i >= S.
// Rows 0..S-1 of columns F..N-1 hold only l*l terms and are never written or read.
template <int C>
struct TcCfg {
  static constexpr int S = C - 8;
  static constexpr int F = C + 8;
  static constexpr int ROWS = 2 * C;
  static constexpr int COLS = C + 24;
  static constexpr int PARTIAL_FLOATS = ROWS * COLS + 8;
  static constexpr int INLIERS = ROWS * COLS;  // offset of the inlier count (u32)
  __host__ __device__ static constexpr int hh(int i, int j) { return j * ROWS + S + i; }
  __host__ __device__ static constexpr int lh(int i, int j) { return i < S ? j * ROWS + i : (16 + i) * ROWS + S + j; }
};

// tiles of 128 pixels: K of the wgmma chain per tile
constexpr int kSfmTcTilePixels = 128;
// resident CTAs per SM: C = 32 one warpgroup and ~47 KB of shared memory; C = 64 one warpgroup, ~85 KB;
// C = 128 two warpgroups, ~163 KB
constexpr int sfm_tc_ctas_per_sm(int code_size) { return code_size <= 32 ? 4 : (code_size <= 64 ? 2 : 1); }
// The partial a tensor-core launch writes, for its flush, the partial size and the finalize: D itself (TcCfg<C>,
// sfm_tc_partial_floats) at C = 64, 128; at C = 32 the kernel combines G = HH + LH + LH^T in its flush and writes the
// fp32 kernels' partial (SfmCfg<C>, sfm_partial_floats).
__host__ __device__ constexpr bool sfm_tc_writes_d(int code_size) { return code_size > 32; }
constexpr size_t sfm_tc_partial_floats(int code_size) { return (size_t)(2 * code_size) * (code_size + 24) + 8; }

struct SfmLaunchPlan {
  int num_items = 0;
  int num_tiles = 0;
  int num_ctas = 0;
  int num_partials = 0;
};

// dfk_sfm_fp32.cu
cudaError_t launch_sfm_fp32(int code_size, const SfmItemDev* items_dev, const SfmLaunchPlan& plan,
                            float* partials_dev, cudaStream_t stream, cudaEvent_t ev_start = nullptr,
                            cudaEvent_t ev_stop = nullptr);
// dfk_sfm_rays.cu : fills every item's ray_tab (all three RunStep kernels read it)
cudaError_t launch_sfm_ray_tables(const SfmItemDev* items_dev, int num_items, cudaStream_t stream);
// tc: the partials are the tensor-core kernel's (sfm_tc_writes_d decides their format)
cudaError_t launch_sfm_finalize(int code_size, bool tc, const SfmItemDev* items_dev, int num_items,
                                const float* partials_dev, float* records_dev, cudaStream_t stream);
// dfk_sfm_wide.cu : C = 64 / 128 (thread-owned 8x8 blocks); partial format = the fp32 kernel's
constexpr int sfm_wide_tile_pixels(int code_size) { return code_size >= 128 ? 64 : 128; }
bool sfm_wide_supported(int code_size);
cudaError_t launch_sfm_wide(int code_size, const SfmItemDev* items_dev, const SfmLaunchPlan& plan,
                            float* partials_dev, cudaStream_t stream, cudaEvent_t ev_start = nullptr,
                            cudaEvent_t ev_stop = nullptr);
// dfk_sfm_tc.cu : C = 32, 64, 128
bool sfm_tc_supported(int code_size);
cudaError_t launch_sfm_tc(int code_size, const SfmItemDev* items_dev, const SfmLaunchPlan& plan, float* partials_dev,
                          cudaStream_t stream, cudaEvent_t ev_start = nullptr, cudaEvent_t ev_stop = nullptr);
size_t sfm_partial_floats(int code_size);
// resident CTAs per SM of the fp32 kernel: at C = 8 a CTA is 11 warps and ~60 KB of shared memory, two fit (the front-end
// is latency-bound, so the second CTA nearly doubles the throughput); from C = 16 on the register budget allows one
constexpr int sfm_fp32_ctas_per_sm(int code_size) { return code_size <= 8 ? 2 : 1; }
bool sfm_fp32_supported(int code_size);
int sfm_max_ctas();  // grid size of the persistent kernel on the current device

// dfk_simple.cu : single-pass reductions with a last-block finalize
struct PixelCam {
  float q[4], t[3];
  float fx, fy, u0, v0, border, ulim, vlim, min_dpt;
};
struct View {
  const float* ptr;
  uint32_t pitch;  // floats
};
// Blocks of a single-pass reduction over `area` pixels: one per 256 pixels, at least 1, at most kSimpleMaxBlocks (the
// grid-stride loops take the rest).
int grid_for(int area);
// SE3 step, EvaluateError, UpdateDepth, and Sobel / blur-down (PyrLevelDev) have two launchers each: one item, whose
// descriptor travels with the launch, and a batch, whose descriptors are in device memory (grid max_blocks x num_items).
// Both run the same kernel, so an item gives the same bits either way.
// One (problem, level) of SE3Aligner::RunStep / CameraTracker::TrackFrame.
struct Se3TrackDesc {
  PixelCam pc;  // q / t are overridden by the problem's device pose when tracking
  View img0, img1, dpt0, grad1;
  int width, height;
  int nblocks;  // grid_for(width * height)
  int grad_aligned;
};
// Problem n: scratch rows [n * scratch_stride, + nblocks) (32 floats each), counter n (zero, self-resetting), out[32 n ..
// + 29) the system (21 JtJ, 6 Jtr, residual, inlier bits).  The pose is read from and updated in pose[8 n .. + 7)
// (tracking; a batch always tracks), and history, if not null, receives the system and the pose it was evaluated at (36
// floats).  A single problem with pose null is evaluated at d.pc's pose (RunStep).
cudaError_t launch_se3_step(const Se3TrackDesc& d, float huber_delta, float* scratch, unsigned int* counter, float* out,
                            float* pose, float* history, cudaStream_t s);
cudaError_t launch_se3_step(const Se3TrackDesc* descs_dev, int num_problems, int max_blocks, float huber_delta,
                            float* scratch, int scratch_stride, unsigned int* counters, float* outs, float* poses,
                            cudaStream_t s);
// One item of SfmAligner::EvaluateError: its block count and its scratch rows.
struct EvalErrorDesc {
  PixelCam pc;
  View img0, img1, dpt0;
  int width, height;
  int nblocks;      // grid_for(width * height)
  int scratch_row;  // first of its nblocks scratch rows (32 floats each)
};
// Item n: scratch rows [scratch_row, + nblocks), counter n (zero, self-resetting), out[2 n .. + 2) = [residual |
// inliers (u32 bits)].
cudaError_t launch_eval_error(const EvalErrorDesc& d, float huber_delta, float* scratch, unsigned int* counter,
                              float* out, cudaStream_t s);
cudaError_t launch_eval_error(const EvalErrorDesc* descs_dev, int num_items, int max_blocks, float huber_delta,
                              float* scratch, unsigned int* counters, float* outs, cudaStream_t s);
// One depth decode (UpdateDepth): its block count and kernel body.
struct DepthDecodeDesc {
  View prx, jac;
  float* dpt;
  uint32_t dpt_pitch;
  const float* code;  // code_size floats in device memory
  int width, height;
  int nblocks;  // update_depth_blocks(width, height)
  int vector;   // update_depth_vector(code_size, code, jac)
};
// The decode's grid for a level of this size, and whether it runs the vector body (else the generic one)
int update_depth_blocks(int width, int height);
bool update_depth_vector(int code_size, const float* code_dev, View jac);
cudaError_t launch_update_depth(int code_size, const DepthDecodeDesc& d, float avg_dpt, cudaStream_t s);
cudaError_t launch_update_depth(int code_size, const DepthDecodeDesc* descs_dev, int num_items, int max_blocks,
                                float avg_dpt, cudaStream_t s);
cudaError_t launch_warp(const PixelCam& pc, int width, int height, View img0, View img1, View dpt0, float* img2,
                        uint32_t img2_pitch, float* scratch, unsigned int* counter, float* out_dev /*2*/,
                        cudaStream_t s);
cudaError_t launch_squared_error(int width, int height, View a, View b, float* scratch, unsigned int* counter,
                                 float* out_dev, cudaStream_t s);
// dfk_window.cu : block-sparse window assembly (gather over CSR lists built on the host by dfk_window_create)
struct WindowDev {
  int num_keyframes, num_pairs, num_items, code_size;
  const int* kf0_ptr;     // [K+1] items whose keyframe (k0) is k ...
  const int* kf0_items;   // ... in item order
  const int* kf1_ptr;     // [K+1] items whose frame (k1) is k
  const int* kf1_items;
  const int* pair_ptr;    // [P+1] items of pair p (its levels)
  const int* pair_items;
  const float* item_area; // [n] W * H of the item's level
  int num_links;          // geometric links (k0 -> k1), one record of DFK_GEO_RECORD_FLOATS each
  const int* lk0_ptr;     // [K+1] links whose k0 is k ...
  const int* lk0_links;   // ... in link order
  const int* lk1_ptr;     // [K+1] links whose k1 is k
  const int* lk1_links;
  int num_frames;         // tracked frames (pose-only variables), frame f is pair_k1 = K + f of exactly one pair
  const int* frame_pair;  // [F] the pair of frame f
};
// geo_records_dev may be null when num_links == 0
cudaError_t launch_window_assemble(const WindowDev& w, const float* records_dev, const float* geo_records_dev,
                                   float* out_dev, cudaStream_t stream);
// n frames frames_dev[i]: prior i (DFK_PRIOR_DOUBLES) = Schur complement of the frame's pose in its pair's items
cudaError_t launch_window_marginalize_frames(const WindowDev& w, const float* records_dev, int n, const int* frames_dev,
                                             double* priors_dev, int32_t* info_dev, cudaStream_t stream);
// m priors on keyframes prior_kf (the CSR kf_ptr[K+1] / kf_priors of prior indices per keyframe, in list order)
cudaError_t launch_window_add_priors(const WindowDev& w, int m, const int* kf_ptr_dev, const int* kf_priors_dev,
                                     const double* priors_dev, const double* delta_dev, float* window_dev,
                                     cudaStream_t stream);
// keyframe priors of a window (dfk_window_create_priors), a parameter of their own so that WindowDev and the assembly
// kernel stay as they are.  Device lists built on the host at create.
struct KfPriorDev {
  int num_priors, num_blocks;
  size_t block_off;          // floats: start of the prior blocks in the window buffer
  const int* mem_ptr;        // [Q + 1] members of prior q: mem_ptr[q] .. mem_ptr[q + 1] (delta of q at mem_ptr[q] * B)
  const long long* off;      // [Q] doubles: start of prior q in the priors buffer
  const int* kf_ptr;         // [K + 1] (prior, position) entries of keyframe k, in prior order ...
  const int2* kf_ent;        // ... (q, a): keyframe k is member a of prior q
  const int* blk_ptr;        // [num_blocks + 1] entries of prior block b, in prior order ...
  const int3* blk_ent;       // ... (q, a, c): the block is G_q's (a, c) block, a < c
};
cudaError_t launch_window_add_keyframe_priors(const WindowDev& w, const KfPriorDev& kp, const double* priors_dev,
                                              const double* delta_dev, float* window_dev, cudaStream_t stream);
// One factor of the local system of dfk_window_marginalize_keyframe (local keyframe 0 = m, 1..n = its blanket):
//   kind 0: record item idx, its k0 / k1 are local l0 / l1 (-1: not a local keyframe)
//   kind 1: geometric link idx, local l0 / l1
//   kind 2: frame prior idx on m
//   kind 3: keyframe prior idx of the window (its members' local indices: KfMargDev::mem_loc)
struct KfMargRef {
  int kind, idx, l0, l1;
};
struct KfMargDev {
  int n;                      // blanket size; local system (1 + n) B
  int num_refs;
  const KfMargRef* refs;      // in summation order
  const int* tile_row;        // [T] local tile t = (tile_row, tile_col): column 0 first (diagonal first), then 1..n
  const int* tile_col;
  const int* mem_loc;         // [members of all priors] local index of each member (indexed like KfPriorDev::mem_ptr)
  const float* records;
  const float* geo;
  const double* fpriors;      // frame priors on m and their deltas
  const double* fdelta;
  const double* kpriors;      // the window's keyframe priors and their deltas
  const double* kdelta;
  double w;                   // zero-code prior weight, code of m (device)
  const double* code;
  double* tiles;              // [T + 1] local tiles B x B (slot T: L of m's block)
  double* rhs;                // [(1 + n) B] g, local block 0 becomes z = L^-1 g_m
  double* f;                  // [1]
  int32_t* info;
};
// the local system's tiles, gradient and f: one launch, one CTA per tile + one
cudaError_t launch_window_marg_gather(const WindowDev& w, const KfPriorDev& kp, const KfMargDev& md, int num_tiles,
                                      cudaStream_t stream);
// the prior out of the eliminated local system (after launch_window_eliminate_first): G from the tiles (I, J),
// 1 <= J <= I <= n, g from rhs blocks 1..n, f0 = f - z^T z; all zero when md.info reports a failed pivot
cudaError_t launch_window_marg_finalize(int code_size, const KfMargDev& md, int num_tiles, double* prior_dev,
                                       cudaStream_t stream);

// dfk_window_solve.cu : damped block-sparse fp64 Cholesky of a window buffer.  The symbolic analysis and the workspace
// (cudaMalloc, on the current device) belong to the solver; a solve allocates nothing.
struct WindowSolverDev;
// pairs / links: the window's keyframe lists (a pair whose k1 is K + f belongs to frame f); fixed_vars: distinct
// variable indices in [0, K (6 + C))
// prior_i / prior_j: the window's prior blocks (i < j), at prior_off floats into the buffer
cudaError_t window_solver_create(int num_keyframes, int code_size, int num_frames, const std::vector<int>& pair_k0,
                                 const std::vector<int>& pair_k1, const std::vector<int>& link_k0,
                                 const std::vector<int>& link_k1, const std::vector<int>& prior_i,
                                 const std::vector<int>& prior_j, size_t prior_off,
                                 const std::vector<int>& fixed_vars, WindowSolverDev** out);
void window_solver_destroy(WindowSolverDev* s);
size_t window_solver_tiles(const WindowSolverDev* s);
// codes_host: K * C doubles, read only when prior > 0 (device memory when codes_on_device); *launches += the kernels
// enqueued
cudaError_t launch_window_solve(const WindowSolverDev* s, const float* window_dev, double lambda, double prior,
                                const double* codes_host, double* dx_dev, int32_t* info_dev, cudaStream_t stream,
                                uint64_t* launches, bool codes_on_device = false);
// Gauss-Newton solve with an absolute diagonal term (dfk_window_solver_update): load into the new loaded set, compare it
// column by column with the last update's, re-factorise from the first changed column j0 (*first_column; one 4-byte
// read-back and stream synchronisation when the solver has a reusable prefix), replay the kept columns' updates onto
// the rest, then the forward tail, the full backward pass and the frames.  The first call allocates the incremental
// workspace.
cudaError_t launch_window_solver_update(WindowSolverDev* s, const float* window_dev, double prior, double diag_eps,
                                        const double* codes_host, double* dx_dev, int32_t* info_dev,
                                        cudaStream_t stream, uint64_t* launches, int* first_column,
                                        bool codes_on_device = false);
// growth (dfk_window_solver_create_from): whether s's window can extend prev's (same code size, at least as many
// keyframes, the same fixed variables among prev's), and s taking over prev's longest prefix of columns with the same
// tile pattern (bounded by what prev holds from its last update): factor, stored loaded system and forward pass,
// copied on the stream.  *columns = the prefix.
bool window_solver_extends(const WindowSolverDev* prev, const WindowSolverDev* s);
cudaError_t window_solver_adopt(WindowSolverDev* s, const WindowSolverDev* prev, cudaStream_t stream, int* columns);
// Elimination of local keyframe 0 from a local tile system laid out as KfMargDev (tiles 0..n = column 0, diagonal first,
// then the lower tiles (I, J) of 1..n): the solve's panel launch of column 0 (L of block 0, z = L^-1 g_0, Y_I = H_I0
// L^-T) and its update launch (H_IJ -= Y_I Y_J^T, g_I -= Y_I z).  info gets 0 or 1 + the failed row.
cudaError_t launch_window_eliminate_first(int code_size, int n, double* tiles, double* rhs, int32_t* info,
                                          const void* tasks_dev, int num_tasks, cudaStream_t stream);
// update tasks of that elimination (16 bytes each), built on the host: (target, a, b, rhs_row)
void window_eliminate_first_tasks(int n, std::vector<int>& out);
// dfk_depth.cu : DepthAligner::RunStep
bool depth_supported(int code_size);
size_t depth_partial_floats(int code_size);
cudaError_t launch_depth_step(const float* code_dev, int code_size, int width, int height, View tgt, View prx_orig,
                              View jac, float avg_dpt, float* scratch /*blocks * depth_partial_floats*/,
                              unsigned int* counter, float* out_dev /*C(C+1)/2 + C + 2*/, int blocks, cudaStream_t s);

// dfk_depth_prior.cu : DepthPriorFactor, batched.  One item = one (keyframe, level) of a depth prior.
struct DepthPriorDesc {
  View tgt, prx, jac;
  const float* code;  // code_size floats in device scratch
  int width, height;
  int parts;          // depth_prior_parts(width, height): partial rows of this item ...
  int part0;          // ... from this row of the partial buffer
};
// partial rows of an item of this size (its own size alone decides, so a record never depends on the batch)
int depth_prior_parts(int width, int height);
// floats per partial row: the augmented Gram (gram) or diff^2 alone
size_t depth_prior_partial_floats(int code_size, bool gram);
// gram: n records of DFK_DEPTH_RECORD_FLOATS(code_size) into out_dev; else n rows [residual | inliers (u32 bits)].  Two
// launches: the partial rows (grid max_parts x n), then one block per item sums them in partial order.  stale (device,
// n bytes, optional): the CTAs of an item whose byte is 0 return at once, so its output row is left as it was.
cudaError_t launch_depth_prior_batch(int code_size, const DepthPriorDesc* descs_dev, int n, int max_parts, float avg_dpt,
                                     float* partials, float* out_dev, bool gram, cudaStream_t s,
                                     const uint8_t* stale = nullptr);
// m depth priors (kf_ptr[K+1] / kf_priors: the CSR of prior indices per keyframe, in list order; level_ptr[m+1]: the
// records of each prior; sigma[m]) into an assembled window buffer, in place
// the codes of n depth-prior items from the state's codes (K x C doubles): item i reads keyframe item_kf[i], rounded to
// fp32 (what the host staging of the batch does with the same codes), into codes_out (n x C floats)
cudaError_t launch_depth_prior_codes(const double* state_codes, const int* item_kf, int n, int code_size,
                                     float* codes_out, cudaStream_t s);
cudaError_t launch_window_add_depth_priors(const WindowDev& w, int m, const int* kf_ptr_dev, const int* kf_priors_dev,
                                           const int* level_ptr_dev, const float* sigma_dev, const float* records_dev,
                                           float* window_dev, cudaStream_t stream);

// dfk_sparse.cu : ReprojectionFactor::linearize and SparseGeometricFactor::linearize, rows (one factor) and records (a
// batch); the single call runs the batch's descriptor for one item
bool sparse_supported(int code_size);
struct SparsePose {
  float q[4], t[3], R[9];      // pose_10 = pose1^-1 * pose0
  float P0[36], P1[36];        // pose10_J_pose0 / pose10_J_pose1, row-major 6x6
  float fx, fy, u0, v0;
};
// One ReprojectionFactor.  Its matches are query / train[match_begin, + num_matches); code points at its code_size floats
// in device scratch.
struct ReprojItemDev {
  SparsePose sp;
  View prx_orig, jac;
  const float* code;
  int width, height;
  int num_matches, match_begin;
  float cauchy_delta, sigma;
};
// rows_dev: 2 num_matches rows of 13 + code_size floats; err2_dev: num_matches squared errors
cudaError_t launch_reprojection_rows(int code_size, const ReprojItemDev& item, const float2* query_dev,
                                     const float2* train_dev, float avg_dpt, float* rows_dev, float* err2_dev, cudaStream_t s);
// one CTA per item; records_dev: num_items records of DFK_SFM_RECORD_FLOATS(code_size) floats.  stale (device,
// num_items bytes, optional): an item whose byte is 0 keeps its record (its CTAs return before they write), as in
// launch_sparse_geometric_records
cudaError_t launch_reprojection_records(int code_size, const ReprojItemDev* items_dev, int num_items, const float2* query_dev,
                                        const float2* train_dev, float avg_dpt, float* records_dev, cudaStream_t s,
                                        const uint8_t* stale = nullptr);

// One SparseGeometricFactor.  Its points are points[point_begin, + num_points); code0 / code1 point at its code_size
// floats each in device scratch.
struct GeoItemDev {
  SparsePose sp;
  View prx0, jac0, prx1, jac1, grad1;
  const float* code0;
  const float* code1;
  float cam_w, cam_h;
  int width, height;
  int num_points, point_begin;
  float huber_delta;
};
// rows_dev: num_points rows of 13 + 2 code_size floats
cudaError_t launch_sparse_geometric_rows(int code_size, const GeoItemDev& item, const int2* points_dev, float avg_dpt,
                                         float* rows_dev, cudaStream_t s);
// grid (num_items, 1 or 4 entry slices); records_dev: num_items records of DFK_GEO_RECORD_FLOATS(code_size) floats
cudaError_t launch_sparse_geometric_records(int code_size, const GeoItemDev* items_dev, int num_items, const int2* points_dev,
                                            float avg_dpt, float* records_dev, cudaStream_t s,
                                            const uint8_t* stale = nullptr);
// error() of a batch: one CTA per item; out_dev: num_items x [b^T b | valid matches / points (u32 bits)], b^T b bit for
// bit the residual of the item's record from launch_reprojection_records / launch_sparse_geometric_records
cudaError_t launch_reprojection_error(int code_size, const ReprojItemDev* items_dev, int num_items, const float2* query_dev,
                                      const float2* train_dev, float avg_dpt, float* out_dev, cudaStream_t s);
cudaError_t launch_sparse_geometric_error(int code_size, const GeoItemDev* items_dev, int num_items, const int2* points_dev,
                                          float avg_dpt, float* out_dev, cudaStream_t s);

// dfk_window_lm.cu : the window problem's loop kernels.  The state is [poses num_poses x 7 | codes K x C] doubles; a
// slot int4 is (pose0, pose1, code0, code1).
struct WindowReposeDev {
  int code_size, num_poses;
  const double* state;
  SfmItemDev* dense;       const int4* dense_slots; int num_dense;  // q, t, R, P0, P1 and the fused-decode code
  EvalErrorDesc* error;    const int4* error_slots; int num_error;  // pc.q, pc.t
  ReprojItemDev* rep;      const int4* rep_slots;   int num_rep;    // sp and code
  GeoItemDev* geo;         const int4* geo_slots;   int num_geo;    // sp, code0 and code1
  DepthDecodeDesc* depth;  const int4* depth_slots; int num_depth;  // code (slot .z)
};
cudaError_t launch_window_repose(const WindowReposeDev& a, cudaStream_t stream);
// out = retract(in, dx) for K keyframes (pose and code) and F frames (pose)
cudaError_t launch_window_retract(const double* in, double* out, const double* dx, int K, int F, int C,
                                  cudaStream_t stream);
// delta row r = Local(x0 row r, keyframe ks[r]): [t - t0 | log(R R0^T) | c - c0], B doubles; x0 rows are [pose | code]
cudaError_t launch_window_deltas(const double* state, int num_poses, int C, int n, const int* ks, const double* x0,
                                 double* delta, cudaStream_t stream);
struct WindowEnergyDev {
  int B;
  const float2* err_out;  // [num_error dense | num_rep | num_geo] rows [residual or b^T b | count (u32 bits)]
  const double* areas;    // W * H of each dense error item
  int num_error, num_rep, num_geo;
  const float* buf_f;     // non-null: E is the window buffer's f (linearise mode), the error outputs are not read
  int num_frame_priors;
  const double* frame_rows;   // DFK_PRIOR_DOUBLES each
  const double* frame_delta;  // B each
  int num_kf_priors;
  const double* kf_rows;      // back to back, prior q at kf_row_off[q]
  const long long* kf_row_off;
  const int* kf_mem_ptr;      // [Q + 1] members; deltas at kf_delta + mem_ptr[q] * B
  const double* kf_delta;
  const double* codes;        // K * C, for the code prior 1/2 w |c|^2
  int num_codes;
  double code_prior_weight;
  // depth priors (dfk_window_problem_set_depth_priors), error mode only: prior q's items [level_ptr[q], level_ptr[q+1])
  // of depth_err ([residual | W * H (u32 bits)] rows), weight 1 / sigma[q]^2; their sum goes to *out_depth and is added
  // to E after the other parts
  int num_depth_priors;
  const float2* depth_err;
  const int* depth_level_ptr;
  const float* depth_sigma;
  double* out_depth;
  double* out;  // [E | photometric | reprojection | geometric | priors | items without inliers | inliers | E + code prior]
};
cudaError_t launch_window_energy(const WindowEnergyDev& a, cudaStream_t stream);
// records slot i (i < n, rf floats each) <- sub record src[i]; zeros where src[i] == -1 (an inactive item); left as
// it is where src[i] == kKeepRecord (an active item whose record is still valid: ISAM2's partial linearisation)
constexpr int kKeepRecord = -2;
cudaError_t launch_window_scatter_records(const float* sub, const int* src, int n, int rf, float* records,
                                          cudaStream_t stream);
// dst record map[i].x <- src record map[i].y (rf floats each), one CTA per entry (dfk_window_problem_grow_from)
cudaError_t launch_window_gather_records(const float* src, float* dst, const int2* map, int n, int rf,
                                         cudaStream_t stream);
// ISAM2's relinearisation check (dfk_window_problem_isam2_update), one CTA per key -- pose k is key 2 k, code k key
// 2 k + 1, frame f key 2 K + f: lin_out = lin_in, except that with `check` a key whose delta (the solve's layout)
// has max |delta_key| >= threshold (a NaN never does) moves to lin_in (+) delta_key (the retraction of
// launch_window_retract, codes by addition); moved[key] = 1 for those keys, else 0
cudaError_t launch_window_relinearize(const double* lin_in, double* lin_out, const double* delta, int K, int F, int C,
                                      bool check, double threshold, int32_t* moved, cudaStream_t stream);
// max |d| over the kept variables of the diagonal of a window buffer's dense system (WindowBlocks.to_dense: the
// keyframe blocks, each self pair's (k, k) coupling block added twice in pair order, the frame blocks) plus w on every
// code entry, in fp64; variables 0..5 are skipped when fix_first_pose.  self_pairs: num_self (pair, keyframe) int2.
// One CTA, into *out
cudaError_t launch_window_diag_max(const float* buf, int K, int F, int C, size_t coupling_off, size_t frame_off,
                                   const int2* self_pairs, int num_self, double w, bool fix_first_pose, double* out,
                                   cudaStream_t stream);

// one factor of dfk_hamming_match_batch / dfk_reprojection_match_batch (dfk_match.cu)
struct MatchItemDev {
  const float* kp0;
  const float* kp1;       // [n, 2] keypoints
  const uint8_t* d0;
  const uint8_t* d1;      // [n, 4 * words] descriptors, 16-byte aligned
  int n0, n1, words;
  int out_begin;          // the item's segment of the match outputs: the prefix sum of n0
  int hyp_begin;          // the item's segment of the per-hypothesis counts
  int max_iterations;
  double fx, fy, u0, v0;
  double threshold, probability;
  float max_dist;
  uint64_t seed;
};
constexpr int kMatchHyp = 32;            // hypotheses per CTA of the RANSAC kernel
constexpr int kMatchMaxQueries = 8192;   // query features per item (the compaction sorts them in shared memory)
// matches_dev[out_begin + q] = (train, distance), (-1, -1) for an empty train set
cudaError_t launch_hamming_match(const MatchItemDev* items_dev, int n, int max_n0, int2* matches_dev, cudaStream_t s);
// matching, the hypotheses' inlier counts (counts_dev), the selection (select_dev: best, inliers, evaluated) and the
// sorted, pruned lists (out_dev rows: query, train, distance; num_out_dev: their lengths)
cudaError_t launch_reprojection_match(const MatchItemDev* items_dev, int n, int max_n0, int max_iterations,
                                      int2* matches_dev, int* counts_dev, int3* select_dev, int3* out_dev,
                                      int* num_out_dev, cudaStream_t s);

// one image of dfk_orb_detect_batch (dfk_orb.cu).  The detector works on the region R = [31, W - 31) x [31, H - 31)
// where keypoints may lie, rw x rh pixels (0 x 0 for an image below 63 x 63), cut into FAST tiles of 32 x 8 pixels;
// a segment is one 32-pixel row of a tile, and segments in row-major order are R's raster order.
struct OrbItemDev {
  const uint8_t* img;
  size_t pitch;
  int rw, rh;             // the region R
  int tiles_x, tiles_y;   // FAST tiles over R; tiles_x segments per row
  int nfeatures, threshold, capacity;
  int out_begin;          // the item's first output row: the prefix sum of the capacities
  size_t map_begin;       // bytes of the NMS score map (rw * rh)
  int seg_begin;          // segment counts / offsets (rh * tiles_x)
  int corner_begin;       // corner list (corner_cap entries: at most one corner per 2 x 2 pixels survives NMS)
  int corner_cap;
  size_t blur_begin;      // bytes of the blurred image over R widened by 18 (the pattern's reach): (rw + 36) x (rh + 36)
};
// the batch's scratch, all of it in one grow-only allocation; hist is zeroed before the first kernel
struct OrbScratchDev {
  uint8_t* map;           // NMS'd FAST score + 1 per pixel of R, 0 for no keypoint
  int* seg;               // per segment: its corner count, then its first corner's index
  int* hist;              // [n, 256] FAST score histogram of the kept corners
  int* stats;             // [n, 4]: corners, first-cut score threshold, candidates, 0
  uint32_t* pos;          // corner (y << 16 | x), raster order
  uint32_t* key;          // corner FAST score, then the response key of a candidate (0 for a non-candidate)
  float* angle;           // candidate angle
  int* rows;              // output row -> corner index
  uint8_t* blur;          // the blurred images the descriptors sample
};
constexpr int kOrbTileW = 32, kOrbTileH = 8;
constexpr int kOrbMaxSide = 16384;
cudaError_t launch_orb_detect(const OrbItemDev* items_dev, int n, const OrbScratchDev& s, int max_rw, int max_rh,
                              int max_corner_cap, int max_segs, int max_capacity, int max_nfeatures,
                              float* keypoints, uint8_t* descriptors, float* angles, float* responses, int* counts,
                              cudaStream_t stream);

// dfk_orb_detect_pyramid_batch (dfk_orb_pyramid.cu).  One level k >= 1 of one image: dst (dw x dh, pitch dw) is src
// (sw x sh, the image's level k - 1) resized.
struct OrbResizeDev {
  const uint8_t* src;
  size_t src_pitch;
  uint8_t* dst;
  int sw, sh, dw, dh;
};
constexpr int kOrbMaxLevels = 16;  // DFK_ORB_MAX_LEVELS
// One image: its levels are the one-level items sub_begin .. sub_begin + nlevels - 1, whose rows and counts the
// detector wrote to the staging arrays; the gather places them at out_begin in level order.
struct OrbGatherDev {
  int sub_begin, nlevels;
  int out_begin, capacity;
  float scale[kOrbMaxLevels];  // s_k
};
// The staged rows of the one-level items, indexed by their out_begin
struct OrbStagingDev {
  const float* keypoints;
  const uint8_t* descriptors;
  const float* angles;
  const float* responses;
  const int* counts;  // per one-level item
};
// one level of every image that has it: count resize items, max_w x max_h their largest output
cudaError_t launch_orb_resize_level(const OrbResizeDev* items_dev, int count, int max_w, int max_h, cudaStream_t stream);
cudaError_t launch_orb_gather(const OrbGatherDev* items_dev, int n, const OrbItemDev* subs_dev, const OrbStagingDev& st,
                              int max_capacity, float* keypoints, uint8_t* descriptors, float* angles,
                              float* responses, int32_t* octaves, int32_t* counts, cudaStream_t stream);

// one frame of dfk_preprocess_batch (dfk_preprocess.cu): the output (w x h) is cut into tiles of DFK_PM_TILE_W x
// DFK_PM_TILE_H pixels, one CTA each; pitches in bytes for the uint8 images, in floats for level 0
struct PpItemDev {
  DfkPmMap map;
  const uint8_t* src;
  size_t src_pitch;
  int sw, sh;             // source size
  int w, h;               // output size
  int tiles_x, tiles;
  uint8_t* color;         // null: not wanted
  size_t color_pitch;
  uint8_t* gray;          // null: not wanted
  size_t gray_pitch;
  float* level0;          // null: no levels
  uint32_t level0_pitch;
  int normalize;
  int partial_begin;      // a normalising item's first tile partial (2 doubles each)
  double* moments;        // (mu, sigma) of a normalising item in scratch
  double* stats;          // the caller's stats row of a normalising item, or null
};
// grid (max_tiles, n); normalize: some item normalises (two more launches: the statistics, one CTA per item, then
// level 0 rewritten as f')
cudaError_t launch_preprocess(const PpItemDev* items_dev, int n, int max_tiles, bool normalize, double* partials,
                              cudaStream_t s);
// one level of one frame of a pyramid (dfk_simple.cu); pitches in floats, grad null: no gradient
struct PyrLevelDev {
  float* img;
  uint32_t pitch;
  int w, h;
  float* grad;
  uint32_t grad_pitch;
};
// grad of lv = SobelGradients(img of lv), out = GaussianBlurDown(in); the batches take the n frames of one level
cudaError_t launch_sobel(const PyrLevelDev& lv, cudaStream_t s);
cudaError_t launch_sobel(const PyrLevelDev* lv_dev, int n, int max_w, int max_h, cudaStream_t s);
cudaError_t launch_blur_down(const PyrLevelDev& in, const PyrLevelDev& out, cudaStream_t s);
cudaError_t launch_blur_down(const PyrLevelDev* in_dev, const PyrLevelDev* out_dev, int n, int max_out_w,
                             int max_out_h, cudaStream_t s);

// DBoW2 retrieval (dfk_bow.cu).  The vocabulary on the device, rows re-indexed breadth first so that a node's
// children are consecutive rows: row 0 is the root, desc [rows, q] (q = descriptor_bytes / 16), child[row] = (first
// child row, children; 0 for a leaf), word[row] = the leaf's word (-1 inside), word_weight [words].
struct BowVocDev {
  const uint4* desc;
  const int2* child;
  const int32_t* word;
  const double* word_weight;
  int q;
};
// one image of dfk_bow_transform_batch: its descriptor rows and its first output row
struct BowItemDev {
  const uint8_t* descriptors;
  int num;
  int out_begin;
};
// one vector of dfk_bow_database_add: copied to storage rows [offset, offset + count) as entry `entry`
struct BowAddDev {
  const int32_t* words;
  const double* values;
  const int32_t* count;
  int capacity;
  int entry;
  long long offset;
};
// the database's storage: entry e's words and values start at offsets[e], counts[e] of them
struct BowDbDev {
  const int32_t* words;
  const double* values;
  const long long* offsets;
  const int32_t* counts;
  int size;
};
struct BowQueryDev {
  const int32_t* words;
  const double* values;
  const int32_t* count;
  int capacity;
  int max_results;
  int max_id;
  int row_begin;
};
struct BowScoreDev {
  const int32_t* words;
  const double* values;
  const int32_t* count;
  int capacity;
  int entry;
};
// the descent (grid (max_num / 8, n), none when max_num = 0) then the assembly (one CTA per item)
cudaError_t launch_bow_transform(const BowVocDev& v, const BowItemDev* items_dev, int n, int max_num,
                                 int32_t* feature_words, int32_t* words_out, double* values_out, int32_t* counts,
                                 cudaStream_t s);
cudaError_t launch_bow_add(const BowAddDev* adds_dev, int n, int32_t* st_words, double* st_values,
                           long long* entry_offsets, int32_t* entry_counts, cudaStream_t s);
// db.size >= 1; sums and hits [n, db.size]; max_cap the largest query capacity (its words and values in shared memory)
cudaError_t launch_bow_query(const BowDbDev& db, const BowQueryDev* queries_dev, int n, int max_cap, double* sums,
                             uint8_t* hits, int32_t* ids, double* scores, int32_t* counts, cudaStream_t s);
cudaError_t launch_bow_score(const BowDbDev& db, const BowScoreDev* items_dev, int n, double* out, cudaStream_t s);

// DBoW2 vocabulary training (dfk_bow_train.cu), one tree level at a time.  A node of at most kBowTrainSmallMax
// descriptors runs its whole k-means in one CTA; a larger one is cut into chunks of kBowTrainChunk descriptors, one CTA
// each, for every step.  Rows are descriptor rows of the level's input (in) and output (out): a node's rows [begin,
// begin + m) of `in` are its members in order, and the step writes them to the same rows of `out`, grouped by child in
// cluster order and in their order within each group.
constexpr int kBowTrainSmallMax = 2048;
constexpr int kBowTrainSmallSplit = 256;  // the small nodes launch in two size classes, split here
constexpr int kBowTrainChunk = 1024;
struct BowTrainNode {
  int begin, m;
  unsigned long long key;
};
struct BowTrainLevel {
  const BowTrainNode* nodes;  // [G]
  const uint4* in;
  uint4* out;
  int* nc;                    // [G] children
  int* rounds;                // [G] assignments made (0 when m <= k)
  int* capped;                // [G] 1: stopped by DFK_BOW_TRAIN_MAX_ROUNDS
  int* sizes;                 // [G, k] group sizes
  uint4* centres;             // [G, k, q]
  int k, q;
};
// the large nodes' state, j a large node, ch a chunk, r a row
struct BowTrainLarge {
  const int* node;            // [GL] its index in the level
  const int2* chunk;          // [chunks] (j, first member within the node)
  const int* chunk_first;     // [GL + 1]
  unsigned long long* rng;    // [GL] the node's stream
  int* seeding;               // [GL]
  int* active;                // [GL] still assigning
  int* changed;               // [GL] this round's assignment differs from the last
  int* cut_chunk;             // [GL]
  long long* cut_rem;         // [GL] the cut's target within cut_chunk
  long long* chunk_sum;       // [chunks] sum of min_dist
  int* chunk_counts;          // [chunks, k] members per cluster
  int* chunk_base;            // [chunks, k] first output row per cluster
  int* members;               // [GL, k]
  int* bits;                  // [GL, k, 8 D] members with each bit set
  int* min_dist;              // [rows]
  unsigned char* assign;      // [rows]
};
// every small node of the level (small_idx [n_small], max_m their largest size): one launch
cudaError_t launch_bow_train_small(const BowTrainLevel& lv, const int* small_idx, int n_small, int max_m,
                                   cudaStream_t s);
// the large nodes' seeding (1 + 3 (k - 1) launches), then `rounds` rounds of (assign, update), then the partition
cudaError_t launch_bow_train_seed(const BowTrainLevel& lv, const BowTrainLarge& lg, int n_large, int chunks,
                                  cudaStream_t s);
cudaError_t launch_bow_train_rounds(const BowTrainLevel& lv, const BowTrainLarge& lg, int n_large, int chunks,
                                    int rounds, cudaStream_t s);
cudaError_t launch_bow_train_partition(const BowTrainLevel& lv, const BowTrainLarge& lg, int n_large, int chunks,
                                       cudaStream_t s);
// the level's centres to the tree's rows: node g's children to rows row_first[g] ...
cudaError_t launch_bow_train_place(const BowTrainLevel& lv, int G, const int* row_first, uint4* tree_desc,
                                   cudaStream_t s);
// N_i: for each item, every word of its vector (words_out rows [out_begin, out_begin + counts[i])) counts once
cudaError_t launch_bow_train_count(const BowItemDev* items_dev, int n, const int32_t* words_out,
                                   const int32_t* counts, int32_t* word_images, cudaStream_t s);

// One keyframe of dfk_keyframe_mesh_batch (dfk_mesh.cu).  Its W x H pixels are cut into tiles of kMeshTileW x
// kMeshTileH, one CTA each; a segment is the kMeshTileW pixels of one row of a tile, and its three masks (vertex, T1, T2;
// bit = x % 32) and two bases (the item's vertex and triangle rows before it, in row-major order) live at
// seg_begin + y * tiles_x + x / 32.
constexpr int kMeshTileW = 32;
constexpr int kMeshTileH = 8;
struct MeshItemDev {
  View dpt;                   // the caller's depth, or its decode in scratch
  View std, vld;              // ptr null: absent
  const uint8_t* color;       // null: absent
  size_t color_pitch;         // bytes
  uint16_t* depth_u16;        // null: not wanted
  size_t u16_pitch;           // bytes
  float fx, fy, u0, v0;
  float q[4], t[3];           // pose_wk
  int w, h, tiles_x, tiles;
  long long seg_begin;
  long long v_begin, t_begin; // the item's first output rows
  int v_cap, t_cap;
};
struct MeshParamsDev {
  double tau;                 // log(stdev_thresh / sqrt 2), -inf for stdev_thresh <= 0
  float slt;
  int crop, draw_noisy;
};
struct MeshOutDev {
  float* positions;
  float* normals;
  uint8_t* colors;
  int32_t* pixels;
  int32_t* triangles;
  int32_t* counts;            // [2 n]: vertices, triangles
};
// classify (grid (max tiles, n)), scan (one CTA per item), write rows (grid (max tiles, n)); segs uint3 and bases int2
// per segment, totals int2 per item (scratch)
cudaError_t launch_keyframe_mesh(const MeshItemDev* items_dev, int n, int max_tiles, const MeshParamsDev& p,
                                 const MeshOutDev& o, uint3* segs, int2* bases, cudaStream_t s);

constexpr int kSimpleMaxBlocks = 1024;
constexpr int kSimpleScratchFloats = kSimpleMaxBlocks * 32;

}  // namespace dfk
