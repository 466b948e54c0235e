// dfk_window_solve.cu -- damped block-sparse fp64 Cholesky of a keyframe window's normal equations, straight from the
// packed buffer of dfk_window_assemble[_geometric] (layout: include/dfk.h).
//
// The system is the one WindowOptimizer solves on torch (window_opt.py: dense_solve = to_dense, prior, damped_solve):
// fp32 entries promoted to fp64 and summed in to_dense's order, the code prior w I / -w code, the fixed variables as
// identity rows with a zero right-hand side, and lambda d + 1e-12 max|d| on the diagonal of the kept variables.
//
// Unit of sparsity: the B x B tile of a pair of keyframes (B = 6 + C).  The symbolic analysis (host, at create) marks the
// lower tiles a pair or link touches and the fill of eliminating keyframes in index order, and stores them column by
// column (tile 0 of a column is its diagonal tile).  One solve is, on the handle's stream:
//   load           one launch, one CTA per tile: the tile's blocks summed in to_dense's order (+ prior, fixed rows,
//                  damping; the diagonal CTAs also write the right-hand side)
//   per column j   panel:  one CTA per nonzero tile (i, j).  Each refactors the diagonal tile in shared memory (its own
//                          copy: no CTA waits for another), then solves X L_jj^T = A_ij in place; the diagonal CTA writes
//                          L_jj to a slot of its own and y_j = L_jj^-1 g_j over g_j.
//                  update: one CTA per target tile (i, k), j < k <= i, with (i, j) and (k, j) nonzero: A_ik -= L_ij L_kj^T
//                          (DFMA, 16 x 16 threads with an M x M register tile each); a diagonal target also does
//                          g_i -= L_ij y_j.
//   per row j, descending   backward: one CTA per nonzero tile (j, i), i <= j.  Each solves L_jj^T x_j = y_j in shared
//                          memory (again its own copy); the diagonal CTA writes dx_j, the others y_i -= L_ji^T x_j.
//   frames         (windows with tracked frames) one launch, one CTA per frame: dx_f = S_f^-1 (g_f - O_f^T dx_k).
//   prior load     (windows with keyframe priors) right after the load: the prior blocks into their tiles.
// The column-0 panel and update launches also eliminate a keyframe from the local system of
// dfk_window_marginalize_keyframe (launch_window_eliminate_first).
// Every tile and every rhs block receives at most one update per launch and its updates in column order, every sum runs
// in a fixed order and there are no atomics, so two solves of the same buffer are bit for bit equal.  Ordering comes from
// stream order only: no CTA ever waits for another.
//
// Tracked frames are pose-only leaves with one pair to one keyframe k, so they are eliminated first, each into k's
// diagonal tile by k's load CTA (frame order): S_f = D_f + diag(lambda d_f + eps) = L_f L_f^T (6 x 6, fp64), Y = O_f
// L_f^-T with O_f's rows at fixed variables zero, z = L_f^-1 g_f; then T_kk -= Y Y^T and g_k -= Y z.  This creates no
// fill, so the symbolic analysis ignores frame pairs.  L_f stays in the workspace for the frame launch; a frame pivot
// that is not positive and finite is reported (by column 0's panel, as the first in elimination order) as
// 1 + K B + 6 f + r.
#include <cuda_runtime.h>
#include <limits.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <memory>
#include <set>
#include <type_traits>
#include <vector>

#include "dfk_internal.h"

namespace dfk {

namespace {

constexpr int kThreads = 256;
constexpr int kSmemMax = 227 * 1024;  // opt-in dynamic shared memory per CTA on sm_90

// contribution of one buffer block to a tile, in to_dense's order: kind in the low two bits
enum : int { CONTRIB_PAIR = 0, CONTRIB_PAIR_T = 1, CONTRIB_LINK = 2, CONTRIB_LINK_T = 3 };

struct SolveArgs {
  const float* buf;
  const double* codes;  // K * C, or null without prior
  double* tiles;        // (num_tiles + K) tiles of B * B, row-major; slot num_tiles + j holds L_jj
  double* rhs;          // K * B: g, then y, then (consumed) during the backward pass
  double* dx;
  int32_t* info;
  const int* tile_row;
  const int* tile_col;
  const int* contrib_ptr;  // [num_tiles + 1]
  const int* contrib;
  const int* diag_tile;    // [K]
  const unsigned char* fixed;  // [K * B]
  int K, P;
  int num_tiles;
  double lambda, prior;
  double diag_eps;  // the incremental load's absolute diagonal term (window_solve_load_kernel<B, F, true>)
};

// the tracked frames of a window, a parameter of its own: only the kernels that handle frames take it, so those of a
// window without frames keep SolveArgs' size and their register allocation
struct FrameArgs {
  int L, F;                     // links, tracked frames
  const int* frame_ptr;         // [K + 1] frames of keyframe k: frame_list[frame_ptr[k] .. frame_ptr[k + 1])
  const int* frame_list;
  const int* frame_pair;        // [F]
  const int* frame_kf;          // [F] keyframe of frame f (k0 of its pair)
  double* frame_L;              // [F * 36] Cholesky factor of the damped S_f
  int* frame_bad;               // [F] 0, or 1 + the row whose pivot failed
};

__device__ __forceinline__ size_t tile_off(int t, int B) { return (size_t)t * B * B; }

// ------------------------------------------------------------------------------------------------------------- load
// Value of H(row r of keyframe i, column c of keyframe j) before prior / damping: the diagonal block, then every
// contribution in list order (to_dense: pairs in order, each one's block then its transpose, then links in order).
template <int B>
__device__ double tile_entry(const SolveArgs& a, int t, int r, int c)
{
  const size_t o_c = (size_t)a.K * (B * B + B), o_l = o_c + (size_t)a.P * B * 6 + 2;
  const bool diag = a.tile_row[t] == a.tile_col[t];
  double s = diag ? (double)a.buf[(size_t)a.tile_row[t] * B * B + r * B + c] : 0.0;
  for (int q = a.contrib_ptr[t]; q < a.contrib_ptr[t + 1]; ++q) {
    const int e = a.contrib[q], kind = e & 3, idx = e >> 2;
    if (kind == CONTRIB_PAIR) {
      if (c < 6) s += (double)a.buf[o_c + (size_t)idx * B * 6 + r * 6 + c];
    } else if (kind == CONTRIB_PAIR_T) {
      if (r < 6) s += (double)a.buf[o_c + (size_t)idx * B * 6 + c * 6 + r];
    } else if (kind == CONTRIB_LINK) {
      s += (double)a.buf[o_l + (size_t)idx * B * B + r * B + c];
    } else {
      s += (double)a.buf[o_l + (size_t)idx * B * B + c * B + r];
    }
  }
  return s;
}

// buffer offsets of the frame blocks (6 x 6 each) and of the frame gradients
template <int B>
__device__ __forceinline__ size_t frame_block_off(const SolveArgs& a, const FrameArgs& fa)
{
  return (size_t)a.K * (B * B + B) + (size_t)a.P * B * 6 + 2 + (size_t)fa.L * B * B;
}

// diagonal entry (after the prior) of variable r of keyframe k
template <int B>
__device__ double diag_entry(const SolveArgs& a, int k, int r)
{
  double h = tile_entry<B>(a, a.diag_tile[k], r, r);
  if (a.prior > 0.0 && r >= 6) h = __dadd_rn(h, a.prior);
  return h;
}

// keyframe i's frames into its damped diagonal tile T and its rhs, in frame order (see the file comment).  Kept out
// of the load kernel body for readability.
template <int B>
__device__ __forceinline__ void eliminate_frames(const SolveArgs& a, const FrameArgs& fa, int i, double* T, double eps)
{
  const size_t o_f = frame_block_off<B>(a, fa);
  __syncthreads();  // every thread wrote its T / rhs entries
  __shared__ double sL[36], sz[6], sY[B * 6];
  for (int q = fa.frame_ptr[i]; q < fa.frame_ptr[i + 1]; ++q) {
    const int f = fa.frame_list[q];
    const float* O = a.buf + (size_t)a.K * (B * B + B) + (size_t)fa.frame_pair[f] * B * 6;
    const float* Df = a.buf + o_f + (size_t)f * 36;
    const float* gf = a.buf + o_f + (size_t)fa.F * 36 + (size_t)f * 6;
    if (threadIdx.x == 0) {
      int bad = -1;
      for (int c = 0; c < 6; ++c) {
        double d = (double)Df[c * 7];
        d = __dadd_rn(d, __dadd_rn(__dmul_rn(a.lambda, d), eps));
        for (int k = 0; k < c; ++k) d = __fma_rn(-sL[c * 6 + k], sL[c * 6 + k], d);
        if (bad < 0 && !(d > 0.0 && d <= 1.7976931348623157e308)) bad = c;
        d = sqrt(d);
        sL[c * 6 + c] = d;
        for (int r = c + 1; r < 6; ++r) {
          double v = (double)Df[r * 6 + c];
          for (int k = 0; k < c; ++k) v = __fma_rn(-sL[r * 6 + k], sL[c * 6 + k], v);
          sL[r * 6 + c] = __ddiv_rn(v, d);
        }
        for (int r = 0; r < c; ++r) sL[r * 6 + c] = 0.0;
      }
      for (int c = 0; c < 6; ++c) {
        double v = (double)gf[c];
        for (int k = 0; k < c; ++k) v = __fma_rn(-sL[c * 6 + k], sz[k], v);
        sz[c] = __ddiv_rn(v, sL[c * 6 + c]);
      }
      for (int e = 0; e < 36; ++e) fa.frame_L[(size_t)f * 36 + e] = sL[e];
      fa.frame_bad[f] = bad + 1;
    }
    __syncthreads();
    for (int r = threadIdx.x; r < B; r += blockDim.x)  // Y L^T = O, row by row; a fixed row of O counts as zero
      for (int c = 0; c < 6; ++c) {
        double v = a.fixed[i * B + r] ? 0.0 : (double)O[r * 6 + c];
        for (int k = 0; k < c; ++k) v = __fma_rn(-sY[r * 6 + k], sL[c * 6 + k], v);
        sY[r * 6 + c] = a.fixed[i * B + r] ? 0.0 : __ddiv_rn(v, sL[c * 6 + c]);
      }
    __syncthreads();
    for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
      const int r = e / B, c = e - r * B;
      double s = 0.0;
      for (int k = 0; k < 6; ++k) s = __fma_rn(sY[r * 6 + k], sY[c * 6 + k], s);
      T[e] = __dsub_rn(T[e], s);
    }
    for (int r = threadIdx.x; r < B; r += blockDim.x) {
      double s = 0.0;
      for (int k = 0; k < 6; ++k) s = __fma_rn(sY[r * 6 + k], sz[k], s);
      a.rhs[(size_t)i * B + r] = __dsub_rn(a.rhs[(size_t)i * B + r], s);
    }
    __syncthreads();  // sL / sY are consumed
  }
}

// kFrames = false (a window without frames) is the load kernel without any frame code: same registers, no stack.
// kAbsEps (the incremental update): no lambda, and the diagonal term is a.diag_eps instead of 1e-12 max|d|.
template <int B, bool kFrames, bool kAbsEps = false>
__global__ void __launch_bounds__(kThreads) window_solve_load_kernel(SolveArgs a, FrameArgs fa)
{
  const int t = blockIdx.x;
  const int i = a.tile_row[t], j = a.tile_col[t];
  double* T = a.tiles + tile_off(t, B);
  if (i != j) {
    for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
      const int r = e / B, c = e - r * B;
      const bool fx = a.fixed[i * B + r] | a.fixed[j * B + c];
      T[e] = fx ? 0.0 : tile_entry<B>(a, t, r, c);
    }
    return;
  }
  double eps;
  if constexpr (kAbsEps) {
    eps = a.diag_eps;
  } else {
    // diagonal tile: max |d| over the kept variables of the whole window (every diagonal CTA computes it, max is exact)
    __shared__ double red[kThreads / 32];
    double m = 0.0;
    for (int v = threadIdx.x; v < a.K * B; v += blockDim.x)
      if (!a.fixed[v]) m = fmax(m, fabs(diag_entry<B>(a, v / B, v % B)));
    if constexpr (kFrames)
      for (int v = threadIdx.x; v < fa.F * 6; v += blockDim.x)  // and over the frames' (never fixed)
        m = fmax(m, fabs((double)a.buf[frame_block_off<B>(a, fa) + (v / 6) * 36 + (v % 6) * 7]));
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) m = fmax(m, red[w]);
    eps = __dmul_rn(1e-12, m);
  }
  for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
    const int r = e / B, c = e - r * B;
    const bool fx = a.fixed[i * B + r] | a.fixed[i * B + c];
    double h;
    if (fx) {
      h = r == c ? 1.0 : 0.0;
    } else {
      h = tile_entry<B>(a, t, r, c);
      if (r == c) {
        if (a.prior > 0.0 && r >= 6) h = __dadd_rn(h, a.prior);
        if constexpr (kAbsEps)
          h = __dadd_rn(h, eps);
        else
          h = __dadd_rn(h, __dadd_rn(__dmul_rn(a.lambda, h), eps));  // damped_solve: H + diag(lam d + 1e-12 max|d|)
      }
    }
    T[e] = h;
  }
  for (int r = threadIdx.x; r < B; r += blockDim.x) {
    double g = (double)a.buf[(size_t)a.K * B * B + (size_t)i * B + r];
    if (a.prior > 0.0 && r >= 6) g = __dsub_rn(g, __dmul_rn(a.prior, a.codes[(size_t)i * (B - 6) + r - 6]));
    a.rhs[(size_t)i * B + r] = a.fixed[i * B + r] ? 0.0 : g;
  }
  if (t == 0 && threadIdx.x == 0) *a.info = 0;
  if constexpr (kFrames) eliminate_frames<B>(a, fa, i, T, eps);
}

// prior blocks of a window with keyframe priors: a second load launch, one CTA per tile that has prior blocks, so that
// the load kernel of a window without them stays as it is.  Prior block (i, j), i < j, lands in lower tile (j, i)
// transposed; the fp64 sum continues from the load kernel's value, blocks in order (to_dense: after the links), and a
// fixed row or column stays zero.
struct PriorLoadArgs {
  const int* tiles;     // tiles with prior blocks
  const int* blk_ptr;   // [tiles + 1] their prior blocks, ascending
  const int* blk;
  size_t off;           // floats: start of the prior blocks in the buffer
};

template <int B>
__global__ void __launch_bounds__(kThreads) window_solve_prior_load_kernel(SolveArgs a, PriorLoadArgs pa)
{
  const int t = pa.tiles[blockIdx.x];
  const int i = a.tile_row[t], j = a.tile_col[t];
  double* T = a.tiles + tile_off(t, B);
  for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
    const int r = e / B, c = e - r * B;
    if (a.fixed[i * B + r] | a.fixed[j * B + c]) continue;
    double s = T[e];
    for (int q = pa.blk_ptr[blockIdx.x]; q < pa.blk_ptr[blockIdx.x + 1]; ++q)
      s += (double)a.buf[pa.off + (size_t)pa.blk[q] * B * B + c * B + r];
    T[e] = s;
  }
}

// ------------------------------------------------------------------------------------------------------------ panel
// Rows of the TRSM that fit in shared memory next to L_jj (the whole tile for B <= 118, two passes at B = 134)
template <int B>
struct PanelCfg {
  static constexpr int kRows = (kSmemMax - (B * B + B) * 8) / (B * 8) < B ? (kSmemMax - (B * B + B) * 8) / (B * 8) : B;
  static constexpr int kSmem = (B * B + B + kRows * B) * 8;
};

// Cholesky of the lower triangle of L (row-major B x B, shared) in place; dg[c] = L_cc.  Returns the first column whose
// pivot is not positive and finite, or -1.  Right-looking, two barriers per column.
template <int B>
__device__ int chol_shared(double* L, double* dg)
{
  int bad = -1;
  for (int c = 0; c < B; ++c) {
    const double p = L[c * B + c];
    if (bad < 0 && !(p > 0.0 && p <= 1.7976931348623157e308)) bad = c;
    const double d = sqrt(p);
    for (int r = c + 1 + threadIdx.x; r < B; r += blockDim.x) L[r * B + c] = __ddiv_rn(L[r * B + c], d);
    if (threadIdx.x == 0) dg[c] = d;
    __syncthreads();
    const int n = B - 1 - c;  // trailing rows c+1 .. B-1, lower triangle
    for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
      const int r = c + 1 + e / n, m = c + 1 + e % n;
      if (m <= r) L[r * B + m] = __fma_rn(-L[r * B + c], L[m * B + c], L[r * B + m]);
    }
    __syncthreads();
  }
  return bad;
}

// X L^T = X0 for `rows` rows of X (row-major, stride B, shared): forward substitution, two barriers per column
template <int B>
__device__ void trsm_rows(double* X, int rows, const double* L, const double* dg)
{
  for (int c = 0; c < B; ++c) {
    for (int r = threadIdx.x; r < rows; r += blockDim.x) X[r * B + c] = __ddiv_rn(X[r * B + c], dg[c]);
    __syncthreads();
    const int n = B - 1 - c;
    for (int e = threadIdx.x; e < rows * n; e += blockDim.x) {
      const int r = e / n, m = c + 1 + e % n;
      X[r * B + m] = __fma_rn(-X[r * B + c], L[m * B + c], X[r * B + m]);
    }
    __syncthreads();
  }
}

template <int B>
__global__ void __launch_bounds__(kThreads) window_solve_panel_kernel(SolveArgs a, int j, int col_begin,
                                                                       const int* frame_bad, int F)
{
  extern __shared__ double sm[];
  double* L = sm;
  double* dg = L + B * B;
  double* X = dg + B;
  const int t = col_begin + blockIdx.x;
  const double* A = a.tiles + tile_off(col_begin, B);
  for (int e = threadIdx.x; e < B * B; e += blockDim.x) L[e] = A[e];
  __syncthreads();
  const int bad = chol_shared<B>(L, dg);
  if (t == col_begin) {
    // diagonal: L_jj to its slot, y_j = L_jj^-1 g_j over g_j
    double* Lj = a.tiles + tile_off(a.num_tiles + j, B);
    for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
      const int r = e / B, c = e - r * B;
      Lj[e] = c < r ? L[e] : (c == r ? dg[r] : 0.0);
    }
    double* g = a.rhs + (size_t)j * B;
    for (int e = threadIdx.x; e < B; e += blockDim.x) X[e] = g[e];
    __syncthreads();
    trsm_rows<B>(X, 1, L, dg);
    for (int e = threadIdx.x; e < B; e += blockDim.x) g[e] = X[e];
    if (threadIdx.x == 0 && j == 0)  // the frames were eliminated first: the first failed frame pivot comes first
      for (int f = 0; f < F; ++f)
        if (frame_bad[f] != 0) {
          *a.info = 1 + a.K * B + 6 * f + frame_bad[f] - 1;
          break;
        }
    if (threadIdx.x == 0 && bad >= 0 && *a.info == 0) *a.info = 1 + j * B + bad;
    return;
  }
  double* T = a.tiles + tile_off(t, B);
  for (int r0 = 0; r0 < B; r0 += PanelCfg<B>::kRows) {
    const int rows = min(PanelCfg<B>::kRows, B - r0);
    for (int e = threadIdx.x; e < rows * B; e += blockDim.x) X[e] = T[(size_t)r0 * B + e];
    __syncthreads();
    trsm_rows<B>(X, rows, L, dg);
    for (int e = threadIdx.x; e < rows * B; e += blockDim.x) T[(size_t)r0 * B + e] = X[e];
    __syncthreads();
  }
}

// ----------------------------------------------------------------------------------------------------------- update
// Output sub-blocks of S x S (S a multiple of 16, NSUB x NSUB of them cover the tile), 16 x 16 threads with an M x M
// register tile each, k in chunks of 16 staged through shared memory.
template <int B>
struct UpdCfg {
  static constexpr int kSub = (B + 63) / 64;
  static constexpr int S = (((B + kSub - 1) / kSub) + 15) / 16 * 16;
  static constexpr int M = S / 16;
  static constexpr int KC = 16;
};

struct UpdTask {
  int target, a, b, rhs_row;  // rhs_row >= 0: diagonal target, also g_rhs_row -= L_a y_j
};

// T -= La Lb^T and, with g, g -= La y: one task's arithmetic, shared by the update launch of a column and the head
// replay of an incremental update, so that both round alike.  Each thread reads and writes only its own entries of T
// and g, so consecutive calls on one tile need no barrier between them.
template <int B>
__device__ __forceinline__ void update_tile(double* T, const double* La, const double* Lb, double* g, const double* y)
{
  using Cfg = UpdCfg<B>;
  constexpr int S = Cfg::S, M = Cfg::M, KC = Cfg::KC;
  __shared__ double As[KC][S + 1], Bs[KC][S + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  for (int sr = 0; sr < Cfg::kSub; ++sr)
    for (int sc = 0; sc < Cfg::kSub; ++sc) {
      const int r0 = sr * S, c0 = sc * S;
      double acc[M][M];
#pragma unroll
      for (int u = 0; u < M; ++u)
#pragma unroll
        for (int v = 0; v < M; ++v) acc[u][v] = 0.0;
      for (int k0 = 0; k0 < B; k0 += KC) {
        for (int e = threadIdx.x; e < S * KC; e += kThreads) {
          const int rr = e / KC, kk = e % KC, k = k0 + kk;
          As[kk][rr] = (r0 + rr < B && k < B) ? La[(r0 + rr) * B + k] : 0.0;
          Bs[kk][rr] = (c0 + rr < B && k < B) ? Lb[(c0 + rr) * B + k] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < KC; ++kk) {
          double x[M], y[M];
#pragma unroll
          for (int u = 0; u < M; ++u) x[u] = As[kk][ty + 16 * u];
#pragma unroll
          for (int v = 0; v < M; ++v) y[v] = Bs[kk][tx + 16 * v];
#pragma unroll
          for (int u = 0; u < M; ++u)
#pragma unroll
            for (int v = 0; v < M; ++v) acc[u][v] = __fma_rn(x[u], y[v], acc[u][v]);
        }
        __syncthreads();
      }
#pragma unroll
      for (int u = 0; u < M; ++u)
#pragma unroll
        for (int v = 0; v < M; ++v) {
          const int r = r0 + ty + 16 * u, c = c0 + tx + 16 * v;
          if (r < B && c < B) T[r * B + c] = __dsub_rn(T[r * B + c], acc[u][v]);
        }
    }
  if (g) {
    for (int r = threadIdx.x; r < B; r += kThreads) {
      double s = 0.0;
      for (int m = 0; m < B; ++m) s = __fma_rn(La[r * B + m], y[m], s);
      g[r] = __dsub_rn(g[r], s);
    }
  }
}

template <int B>
__global__ void __launch_bounds__(kThreads) window_solve_update_kernel(SolveArgs a, const UpdTask* tasks, int j)
{
  const UpdTask task = tasks[blockIdx.x];
  update_tile<B>(a.tiles + tile_off(task.target, B), a.tiles + tile_off(task.a, B), a.tiles + tile_off(task.b, B),
                 task.rhs_row >= 0 ? a.rhs + (size_t)task.rhs_row * B : nullptr, a.rhs + (size_t)j * B);
}

// --------------------------------------------------------------------------------------------------------- backward
// launch for row j: CTA 0 writes dx_j; CTA q > 0 owns tile row_tiles[q - 1] = (j, i < j) and does y_i -= L_ji^T x_j
template <int B>
__global__ void __launch_bounds__(kThreads) window_solve_backward_kernel(SolveArgs a, const int* row_tiles, int j)
{
  extern __shared__ double sm[];
  double* L = sm;        // L_jj, row-major
  double* x = L + B * B;
  const double* Lj = a.tiles + tile_off(a.num_tiles + j, B);
  for (int e = threadIdx.x; e < B * B; e += blockDim.x) L[e] = Lj[e];
  for (int e = threadIdx.x; e < B; e += blockDim.x) x[e] = a.rhs[(size_t)j * B + e];
  __syncthreads();
  // L^T x = y: for r = B-1 .. 0, x_r /= L_rr, then x_m -= L_rm x_r for m < r
  for (int r = B - 1; r >= 0; --r) {
    if (threadIdx.x == 0) x[r] = __ddiv_rn(x[r], L[r * B + r]);
    __syncthreads();
    for (int m = threadIdx.x; m < r; m += blockDim.x) x[m] = __fma_rn(-L[r * B + m], x[r], x[m]);
    __syncthreads();
  }
  const bool ok = *a.info == 0;
  if (blockIdx.x == 0) {
    for (int r = threadIdx.x; r < B; r += blockDim.x)
      a.dx[(size_t)j * B + r] = (ok && !a.fixed[j * B + r]) ? x[r] : 0.0;
    return;
  }
  const int t = row_tiles[blockIdx.x - 1], i = a.tile_col[t];
  const double* Lji = a.tiles + tile_off(t, B);
  double* y = a.rhs + (size_t)i * B;
  for (int c = threadIdx.x; c < B; c += blockDim.x) {
    double s = 0.0;
    for (int m = 0; m < B; ++m) s = __fma_rn(Lji[m * B + c], x[m], s);
    y[c] = __dsub_rn(y[c], s);
  }
}

// ----------------------------------------------------------------------------------------------------------- frames
// one CTA of 32 threads per frame f of keyframe k: v = g_f - O_f^T dx_k (lane c < 6, rows in order, fixed rows skipped),
// then dx_f = L_f^-T L_f^-1 v
template <int B>
__global__ void __launch_bounds__(32) window_solve_frames_kernel(SolveArgs a, FrameArgs fa)
{
  __shared__ double v[6];
  const int f = blockIdx.x, p = fa.frame_pair[f];
  const int k = fa.frame_kf[f];
  const size_t o_f = frame_block_off<B>(a, fa);
  if (threadIdx.x < 6) {
    const int c = threadIdx.x;
    const float* O = a.buf + (size_t)a.K * (B * B + B) + (size_t)p * B * 6;
    double s = (double)a.buf[o_f + (size_t)fa.F * 36 + (size_t)f * 6 + c];
    for (int r = 0; r < B; ++r)
      if (!a.fixed[k * B + r]) s = __fma_rn(-(double)O[r * 6 + c], a.dx[(size_t)k * B + r], s);
    v[c] = s;
  }
  __syncwarp();
  if (threadIdx.x == 0) {
    const double* L = fa.frame_L + (size_t)f * 36;
    double y[6];
    for (int c = 0; c < 6; ++c) {
      double s = v[c];
      for (int m = 0; m < c; ++m) s = __fma_rn(-L[c * 6 + m], y[m], s);
      y[c] = __ddiv_rn(s, L[c * 6 + c]);
    }
    for (int c = 5; c >= 0; --c) {
      double s = y[c];
      for (int m = c + 1; m < 6; ++m) s = __fma_rn(-L[m * 6 + c], y[m], s);
      y[c] = __ddiv_rn(s, L[c * 6 + c]);
    }
    const bool ok = *a.info == 0;
    for (int c = 0; c < 6; ++c) a.dx[(size_t)a.K * B + 6 * f + c] = ok ? y[c] : 0.0;
  }
}

// ------------------------------------------------------------------------------------------------------ incremental
// The loaded system of an update (tiles 0 .. T-1 after the load launches, and the rhs blocks), one of two ping-pong sets
// of the incremental workspace: the other holds the previous update's.
struct LoadedSet {
  double* tiles;
  double* rhs;
};

// one CTA per keyframe column j: j0 = min(j0, j) when a tile of column j or rhs block j of `now` differs bit for bit
// from `before`.  *j0 holds the reusable prefix before the launch; atomicMin makes the result independent of CTA order.
__global__ void __launch_bounds__(kThreads) window_update_diff_kernel(LoadedSet now, LoadedSet before,
                                                                      const int* diag_tile, int K, int T, int B,
                                                                      int* j0)
{
  const int j = blockIdx.x;
  const size_t t0 = (size_t)diag_tile[j] * B * B, t1 = (size_t)(j + 1 < K ? diag_tile[j + 1] : T) * B * B;
  const unsigned long long* x = reinterpret_cast<const unsigned long long*>(now.tiles);
  const unsigned long long* y = reinterpret_cast<const unsigned long long*>(before.tiles);
  int diff = 0;
  for (size_t e = t0 + threadIdx.x; e < t1; e += blockDim.x) diff |= x[e] != y[e];
  const unsigned long long* gx = reinterpret_cast<const unsigned long long*>(now.rhs) + (size_t)j * B;
  const unsigned long long* gy = reinterpret_cast<const unsigned long long*>(before.rhs) + (size_t)j * B;
  for (int r = threadIdx.x; r < B; r += blockDim.x) diff |= gx[r] != gy[r];
  if (__syncthreads_or(diff) && threadIdx.x == 0) atomicMin(j0, j);
}

// one CTA per tile t of the columns j0 .. K-1: the loaded tile (and, for a diagonal tile, the loaded rhs block) into the
// working set, then the updates of the kept head columns j < j0 that target it, in column order, as their update
// launches would apply them (update_tile, with y_j from the stored forward pass)
template <int B>
__global__ void __launch_bounds__(kThreads) window_update_replay_kernel(SolveArgs a, LoadedSet now, const double* ystore,
                                                                        const int* rep_ptr, const UpdTask* rep_tasks,
                                                                        int t_begin, int j0)
{
  const int t = t_begin + blockIdx.x;
  const int i = a.tile_row[t];
  const bool diag = i == a.tile_col[t];
  double* T = a.tiles + tile_off(t, B);
  const double* src = now.tiles + tile_off(t, B);
  for (int e = threadIdx.x; e < B * B; e += blockDim.x) T[e] = src[e];
  if (diag)
    for (int r = threadIdx.x; r < B; r += blockDim.x) a.rhs[(size_t)i * B + r] = now.rhs[(size_t)i * B + r];
  __syncthreads();
  for (int q = rep_ptr[t]; q < rep_ptr[t + 1]; ++q) {
    const UpdTask task = rep_tasks[q];
    const int j = a.tile_col[task.a];
    if (j >= j0) break;
    update_tile<B>(T, a.tiles + tile_off(task.a, B), a.tiles + tile_off(task.b, B),
                   task.rhs_row >= 0 ? a.rhs + (size_t)i * B : nullptr, ystore + (size_t)j * B);
  }
}

// one CTA after the forward pass: the kept head's y_j (j < j0) back into the rhs for the backward pass, the new y_j
// (j >= j0) into the store, and info as the panel launches of a full factorisation report it -- the first failed frame
// pivot, else the first keyframe variable whose pivot failed.  A pivot p failed (!(p > 0 && p <= DBL_MAX)) exactly when
// its stored diagonal sqrt(p) of L_jj is not positive and finite, so the kept columns need no record of their own.
template <int B>
__global__ void __launch_bounds__(kThreads) window_update_finish_kernel(SolveArgs a, double* ystore, const int* frame_bad,
                                                                        int F, int j0)
{
  __shared__ int red[kThreads / 32];
  const size_t split = (size_t)j0 * B, n = (size_t)a.K * B;
  for (size_t v = threadIdx.x; v < split; v += blockDim.x) a.rhs[v] = ystore[v];
  for (size_t v = split + threadIdx.x; v < n; v += blockDim.x) ystore[v] = a.rhs[v];
  int first = INT_MAX;
  for (int f = threadIdx.x; f < F; f += blockDim.x)
    if (frame_bad[f] != 0) first = min(first, 6 * f + frame_bad[f] - 1);
  for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = first;
  __syncthreads();
  int fr = INT_MAX;
  for (int w = 0; w < kThreads / 32; ++w) fr = min(fr, red[w]);
  __syncthreads();
  first = INT_MAX;
  for (int v = threadIdx.x; v < a.K * B; v += blockDim.x) {
    const int j = v / B, r = v - j * B;
    const double d = a.tiles[tile_off(a.num_tiles + j, B) + (size_t)r * B + r];
    if (!(d > 0.0 && d <= 1.7976931348623157e308)) first = min(first, v);
  }
  for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = first;
  __syncthreads();
  if (threadIdx.x == 0) {
    int kf = INT_MAX;
    for (int w = 0; w < kThreads / 32; ++w) kf = min(kf, red[w]);
    *a.info = fr != INT_MAX ? 1 + a.K * B + fr : (kf != INT_MAX ? 1 + kf : 0);
  }
}

template <class F>
cudaError_t with_code_size(int code_size, F&& f)
{
  switch (code_size) {
    case 8: return f(std::integral_constant<int, 14>{});
    case 16: return f(std::integral_constant<int, 22>{});
    case 32: return f(std::integral_constant<int, 38>{});
    case 64: return f(std::integral_constant<int, 70>{});
    case 128: return f(std::integral_constant<int, 134>{});
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

// --------------------------------------------------------------------------------------------------------- the plan
struct WindowSolverDev {
  int K = 0, C = 0, B = 0, P = 0, L = 0, F = 0, num_tiles = 0;
  int prior_tiles = 0;        // tiles with prior blocks (0: no prior load launch)
  PriorLoadArgs pa{};
  std::vector<int> col_ptr;   // [K + 1] tiles of column j: [col_ptr[j], col_ptr[j+1]), the first one diagonal
  std::vector<int> upd_ptr;   // [K + 1] update tasks of column j
  std::vector<int> row_ptr;   // [K + 1] backward tiles of row j (off-diagonal, column order)
  // device: one allocation, the uploaded lists (tile_row | tile_col | contrib_ptr | contrib | diag_tile | row_tiles |
  // frame_ptr | frame_list | frame_pair | frame_kf | prior-load lists | tasks | fixed mask), then the workspace (codes |
  // tiles | rhs | the frames' factors and pivot flags)
  unsigned char* blob = nullptr;
  unsigned char* fixed = nullptr;
  double* codes = nullptr;
  double* tiles = nullptr;
  double* rhs = nullptr;
  double* frame_L = nullptr;
  int* frame_bad = nullptr;
  const int *tile_row = nullptr, *tile_col = nullptr, *contrib_ptr = nullptr, *contrib = nullptr, *diag_tile = nullptr,
            *row_tiles = nullptr, *frame_ptr = nullptr, *frame_list = nullptr, *frame_pair = nullptr,
            *frame_kf = nullptr;
  const UpdTask* tasks = nullptr;
  // incremental updates (launch_window_solver_update): the update tasks grouped by target tile, in column order
  const int* rep_ptr = nullptr;  // [num_tiles + 1]
  const UpdTask* rep_tasks = nullptr;
  std::vector<int> tile_row_h;   // host copies for window_solver_create_from
  std::vector<unsigned char> fixed_h;
  // the incremental workspace, allocated by the first update (or create_from): two loaded sets (the last update's and
  // this one's, ping-pong), the forward pass's y, and j0
  unsigned char* inc = nullptr;
  LoadedSet loaded[2]{};
  double* ystore = nullptr;
  int* j0_dev = nullptr;
  int cur = 0;               // loaded[cur]: the loaded system of the last update
  mutable int reuse = 0;     // leading columns whose factor, y and stored loaded system are those of loaded[cur]
  int j0_host = 0;
  ~WindowSolverDev()
  {
    cudaFree(blob);
    cudaFree(inc);
  }
};

size_t window_solver_tiles(const WindowSolverDev* s) { return s ? (size_t)s->num_tiles : 0; }

cudaError_t window_solver_create(int K, int C, int F, const std::vector<int>& pair_k0, const std::vector<int>& pair_k1,
                                 const std::vector<int>& link_k0, const std::vector<int>& link_k1,
                                 const std::vector<int>& prior_i, const std::vector<int>& prior_j, size_t prior_off,
                                 const std::vector<int>& fixed_vars, WindowSolverDev** out)
{
  *out = nullptr;
  const int B = 6 + C, P = (int)pair_k0.size(), L = (int)link_k0.size(), Q = (int)prior_i.size();
  // ---- symbolic elimination in keyframe order: below[j] = rows i > j of the nonzero tiles of column j (a frame pair,
  // k1 >= K, is eliminated at load: no tile, no fill)
  std::vector<std::set<int>> below(K);
  for (int p = 0; p < P; ++p)
    if (pair_k0[p] != pair_k1[p] && pair_k1[p] < K)
      below[std::min(pair_k0[p], pair_k1[p])].insert(std::max(pair_k0[p], pair_k1[p]));
  for (int l = 0; l < L; ++l) below[std::min(link_k0[l], link_k1[l])].insert(std::max(link_k0[l], link_k1[l]));
  for (int q = 0; q < Q; ++q) below[prior_i[q]].insert(prior_j[q]);  // prior_i < prior_j
  for (int j = 0; j < K; ++j) {
    for (auto ia = below[j].begin(); ia != below[j].end(); ++ia)
      for (auto ib = below[j].begin(); ib != ia; ++ib) below[*ib].insert(*ia);  // (ia, ib) fills, ib < ia
  }
  auto s = std::make_unique<WindowSolverDev>();
  s->K = K; s->C = C; s->B = B; s->P = P; s->L = L; s->F = F;
  std::vector<int> tile_row, tile_col;
  s->col_ptr.assign(K + 1, 0);
  std::vector<std::vector<std::pair<int, int>>> col_index(K);  // (row, tile) per column, rows ascending
  for (int j = 0; j < K; ++j) {
    s->col_ptr[j] = (int)tile_row.size();
    tile_row.push_back(j); tile_col.push_back(j);
    col_index[j].push_back({j, s->col_ptr[j]});
    for (int i : below[j]) {
      col_index[j].push_back({i, (int)tile_row.size()});
      tile_row.push_back(i); tile_col.push_back(j);
    }
  }
  const int T = (int)tile_row.size();
  s->num_tiles = T;
  s->col_ptr[K] = T;
  auto tile_of = [&](int i, int j) {  // i >= j, structurally nonzero: binary search of column j's rows
    const auto& ci = col_index[j];
    return std::lower_bound(ci.begin(), ci.end(), std::make_pair(i, -1))->second;
  };
  // ---- contributions per tile, in to_dense's order
  std::vector<std::vector<int>> contrib(T);
  std::vector<int> frame_pair(F), frame_kf(F), frame_ptr(K + 1, 0), frame_list(F);
  for (int p = 0; p < P; ++p) {
    const int k0 = pair_k0[p], k1 = pair_k1[p];
    if (k1 >= K) {
      frame_pair[k1 - K] = p;
      frame_kf[k1 - K] = k0;
      frame_ptr[k0 + 1] += 1;
    } else if (k0 == k1) {
      contrib[tile_of(k0, k0)].push_back(p * 4 + CONTRIB_PAIR);
      contrib[tile_of(k0, k0)].push_back(p * 4 + CONTRIB_PAIR_T);
    } else if (k0 > k1) {
      contrib[tile_of(k0, k1)].push_back(p * 4 + CONTRIB_PAIR);
    } else {
      contrib[tile_of(k1, k0)].push_back(p * 4 + CONTRIB_PAIR_T);
    }
  }
  for (int l = 0; l < L; ++l) {
    const int k0 = link_k0[l], k1 = link_k1[l];
    if (k0 > k1) contrib[tile_of(k0, k1)].push_back(l * 4 + CONTRIB_LINK);
    else contrib[tile_of(k1, k0)].push_back(l * 4 + CONTRIB_LINK_T);
  }
  // prior blocks per tile (blocks ascending: in to_dense's order)
  std::vector<std::vector<int>> pblk(T);
  for (int q = 0; q < Q; ++q) pblk[tile_of(prior_j[q], prior_i[q])].push_back(q);
  std::vector<int> ptiles, pptr(1, 0), pflat;
  for (int t = 0; t < T; ++t)
    if (!pblk[t].empty()) {
      ptiles.push_back(t);
      pflat.insert(pflat.end(), pblk[t].begin(), pblk[t].end());
      pptr.push_back((int)pflat.size());
    }
  // ---- update tasks per column, backward tiles per row
  std::vector<UpdTask> tasks;
  s->upd_ptr.assign(K + 1, 0);
  std::vector<std::vector<int>> row_list(K);
  for (int j = 0; j < K; ++j) {
    s->upd_ptr[j] = (int)tasks.size();
    const auto& ci = col_index[j];
    for (size_t qa = 1; qa < ci.size(); ++qa) {
      row_list[ci[qa].first].push_back(ci[qa].second);
      for (size_t qb = 1; qb <= qa; ++qb)
        tasks.push_back({tile_of(ci[qa].first, ci[qb].first), ci[qa].second, ci[qb].second, qa == qb ? ci[qa].first : -1});
    }
  }
  s->upd_ptr[K] = (int)tasks.size();
  s->row_ptr.assign(K + 1, 0);
  std::vector<int> row_tiles;
  for (int j = 0; j < K; ++j) {
    s->row_ptr[j] = (int)row_tiles.size();
    row_tiles.insert(row_tiles.end(), row_list[j].begin(), row_list[j].end());
  }
  s->row_ptr[K] = (int)row_tiles.size();
  // ---- one allocation: the uploaded lists, then the workspace
  std::vector<int> cptr(T + 1, 0), cflat;
  for (int t = 0; t < T; ++t) {
    cptr[t] = (int)cflat.size();
    cflat.insert(cflat.end(), contrib[t].begin(), contrib[t].end());
  }
  cptr[T] = (int)cflat.size();
  for (int k = 0; k < K; ++k) frame_ptr[k + 1] += frame_ptr[k];
  {
    std::vector<int> next(frame_ptr.begin(), frame_ptr.end() - 1);
    for (int f = 0; f < F; ++f) frame_list[next[frame_kf[f]]++] = f;
  }
  Layout lay;
  const Part<int> tr = lay.add<int>(T), tc = lay.add<int>(T), cp = lay.add<int>(T + 1), cf = lay.add<int>(cflat.size());
  const Part<int> dg = lay.add<int>(K), rt = lay.add<int>(row_tiles.size()), fp = lay.add<int>(K + 1), fl = lay.add<int>(F);
  const Part<int> fr = lay.add<int>(F), fk = lay.add<int>(F), pt = lay.add<int>(ptiles.size()), pp = lay.add<int>(pptr.size());
  const Part<int> pf = lay.add<int>(pflat.size());
  const Part<UpdTask> tk = lay.add<UpdTask>(tasks.size());
  // the same tasks grouped by target (column order within a target: tasks are listed column by column)
  std::vector<int> rptr(T + 1, 0);
  for (const UpdTask& u : tasks) ++rptr[u.target + 1];
  for (int t = 0; t < T; ++t) rptr[t + 1] += rptr[t];
  std::vector<UpdTask> rtasks(tasks.size());
  {
    std::vector<int> next(rptr.begin(), rptr.end() - 1);
    for (const UpdTask& u : tasks) rtasks[next[u.target]++] = u;
  }
  const Part<int> rp = lay.add<int>(T + 1);
  const Part<UpdTask> rk = lay.add<UpdTask>(rtasks.size());
  const Part<unsigned char> fx = lay.add<unsigned char>((size_t)K * B);
  const size_t uploaded = lay.bytes;
  const Part<double> codes = lay.add<double>((size_t)K * C), tiles = lay.add<double>((size_t)(T + K) * B * B);
  const Part<double> rhs = lay.add<double>((size_t)K * B), frame_L = lay.add<double>((size_t)F * 36);
  const Part<int> frame_bad = lay.add<int>(F);
  std::vector<unsigned char> host(uploaded, 0);
  unsigned char* hb = host.data();
  std::copy(tile_row.begin(), tile_row.end(), tr.at(hb));
  std::copy(tile_col.begin(), tile_col.end(), tc.at(hb));
  std::copy(cptr.begin(), cptr.end(), cp.at(hb));
  std::copy(cflat.begin(), cflat.end(), cf.at(hb));
  std::copy(s->col_ptr.begin(), s->col_ptr.end() - 1, dg.at(hb));  // the diagonal tile of column j is its first
  std::copy(row_tiles.begin(), row_tiles.end(), rt.at(hb));
  std::copy(frame_ptr.begin(), frame_ptr.end(), fp.at(hb));
  std::copy(frame_list.begin(), frame_list.end(), fl.at(hb));
  std::copy(frame_pair.begin(), frame_pair.end(), fr.at(hb));
  std::copy(frame_kf.begin(), frame_kf.end(), fk.at(hb));
  std::copy(ptiles.begin(), ptiles.end(), pt.at(hb));
  std::copy(pptr.begin(), pptr.end(), pp.at(hb));
  std::copy(pflat.begin(), pflat.end(), pf.at(hb));
  std::copy(tasks.begin(), tasks.end(), tk.at(hb));
  std::copy(rptr.begin(), rptr.end(), rp.at(hb));
  std::copy(rtasks.begin(), rtasks.end(), rk.at(hb));
  for (int v : fixed_vars) fx.at(hb)[v] = 1;
  s->tile_row_h = tile_row;
  s->fixed_h.assign(fx.at(hb), fx.at(hb) + (size_t)K * B);

  cudaError_t e;
  if ((e = cudaMalloc((void**)&s->blob, lay.bytes)) != cudaSuccess) return e;
  if ((e = cudaMemcpy(s->blob, hb, uploaded, cudaMemcpyHostToDevice)) != cudaSuccess) return e;
  unsigned char* b = s->blob;
  s->tile_row = tr.at(b); s->tile_col = tc.at(b); s->contrib_ptr = cp.at(b); s->contrib = cf.at(b);
  s->diag_tile = dg.at(b); s->row_tiles = rt.at(b);
  s->frame_ptr = fp.at(b); s->frame_list = fl.at(b); s->frame_pair = fr.at(b); s->frame_kf = fk.at(b);
  s->tasks = tk.at(b);
  s->rep_ptr = rp.at(b); s->rep_tasks = rk.at(b);
  s->fixed = fx.at(b); s->codes = codes.at(b); s->tiles = tiles.at(b); s->rhs = rhs.at(b);
  s->frame_L = frame_L.at(b); s->frame_bad = frame_bad.at(b);
  s->prior_tiles = (int)ptiles.size();
  s->pa.tiles = pt.at(b); s->pa.blk_ptr = pp.at(b); s->pa.blk = pf.at(b); s->pa.off = prior_off;
  // kernel attributes once, here: no runtime configuration call in a solve
  e = with_code_size(C, [](auto bc) {
    constexpr int Bv = bc.value;
    cudaError_t r = cudaFuncSetAttribute(window_solve_panel_kernel<Bv>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         PanelCfg<Bv>::kSmem);
    if (r != cudaSuccess) return r;
    return cudaFuncSetAttribute(window_solve_backward_kernel<Bv>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (Bv * Bv + Bv) * 8);
  });
  if (e != cudaSuccess) return e;
  *out = s.release();
  return cudaSuccess;
}

void window_solver_destroy(WindowSolverDev* s) { delete s; }

cudaError_t launch_window_solve(const WindowSolverDev* s, const float* window_dev, double lambda, double prior,
                                const double* codes_host, double* dx_dev, int32_t* info_dev, cudaStream_t stream,
                                uint64_t* launches, bool codes_on_device)
{
  s->reuse = 0;  // the factor is overwritten: a later incremental update starts over
  SolveArgs a{};
  a.buf = window_dev;
  a.codes = prior > 0.0 ? s->codes : nullptr;
  a.tiles = s->tiles; a.rhs = s->rhs; a.dx = dx_dev; a.info = info_dev;
  a.tile_row = s->tile_row; a.tile_col = s->tile_col; a.contrib_ptr = s->contrib_ptr; a.contrib = s->contrib;
  a.diag_tile = s->diag_tile; a.fixed = s->fixed;
  a.K = s->K; a.P = s->P; a.num_tiles = s->num_tiles;
  FrameArgs fa{};
  fa.L = s->L; fa.F = s->F;
  fa.frame_ptr = s->frame_ptr; fa.frame_list = s->frame_list; fa.frame_pair = s->frame_pair; fa.frame_kf = s->frame_kf;
  fa.frame_L = s->frame_L; fa.frame_bad = s->frame_bad;
  a.lambda = lambda; a.prior = prior;
  if (prior > 0.0) {
    // pageable source: the copy is staged before the call returns, so the caller may reuse its array at once.  A
    // window problem passes its device state instead (a device-to-device copy on the stream)
    cudaError_t e = cudaMemcpyAsync(s->codes, codes_host, (size_t)s->K * s->C * sizeof(double),
                                    codes_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, stream);
    if (e != cudaSuccess) return e;
  }
  return with_code_size(s->C, [&](auto bc) {
    constexpr int Bv = bc.value;
    uint64_t n = 0;
    if (s->F > 0)
      window_solve_load_kernel<Bv, true><<<s->num_tiles, kThreads, 0, stream>>>(a, fa);
    else
      window_solve_load_kernel<Bv, false><<<s->num_tiles, kThreads, 0, stream>>>(a, fa);
    ++n;
    if (s->prior_tiles > 0) {
      window_solve_prior_load_kernel<Bv><<<s->prior_tiles, kThreads, 0, stream>>>(a, s->pa);
      ++n;
    }
    for (int j = 0; j < s->K; ++j) {
      const int c0 = s->col_ptr[j], nc = s->col_ptr[j + 1] - c0;
      window_solve_panel_kernel<Bv><<<nc, kThreads, PanelCfg<Bv>::kSmem, stream>>>(a, j, c0, s->frame_bad, s->F);
      ++n;
      const int u0 = s->upd_ptr[j], nu = s->upd_ptr[j + 1] - u0;
      if (nu > 0) {
        window_solve_update_kernel<Bv><<<nu, kThreads, 0, stream>>>(a, s->tasks + u0, j);
        ++n;
      }
    }
    for (int j = s->K - 1; j >= 0; --j) {
      const int r0 = s->row_ptr[j], nr = s->row_ptr[j + 1] - r0;
      window_solve_backward_kernel<Bv><<<1 + nr, kThreads, (Bv * Bv + Bv) * 8, stream>>>(a, s->row_tiles + r0, j);
      ++n;
    }
    if (s->F > 0) {
      window_solve_frames_kernel<Bv><<<s->F, 32, 0, stream>>>(a, fa);
      ++n;
    }
    *launches += n;
    return cudaGetLastError();
  });
}

// ------------------------------------------------------------------------------------------- incremental update
namespace {

cudaError_t ensure_incremental(WindowSolverDev* s)
{
  if (s->inc) return cudaSuccess;
  const size_t K = s->K, B = s->B, T = s->num_tiles;
  Layout lay;
  const Part<double> t0 = lay.add<double>(T * B * B), r0 = lay.add<double>(K * B);
  const Part<double> t1 = lay.add<double>(T * B * B), r1 = lay.add<double>(K * B);
  const Part<double> ys = lay.add<double>(K * B);
  const Part<int> j0 = lay.add<int>(1);
  cudaError_t e = cudaMalloc((void**)&s->inc, lay.bytes);
  if (e != cudaSuccess) return e;
  s->loaded[0] = {t0.at(s->inc), r0.at(s->inc)};
  s->loaded[1] = {t1.at(s->inc), r1.at(s->inc)};
  s->ystore = ys.at(s->inc);
  s->j0_dev = j0.at(s->inc);
  return cudaSuccess;
}

}  // namespace

cudaError_t launch_window_solver_update(WindowSolverDev* s, const float* window_dev, double prior, double diag_eps,
                                        const double* codes_host, double* dx_dev, int32_t* info_dev,
                                        cudaStream_t stream, uint64_t* launches, int* first_column,
                                        bool codes_on_device)
{
  const int reuse = s->reuse;
  s->reuse = 0;  // until this update completes
  cudaError_t e = ensure_incremental(s);
  if (e != cudaSuccess) return e;
  SolveArgs a{};
  a.buf = window_dev;
  a.codes = prior > 0.0 ? s->codes : nullptr;
  a.tiles = s->tiles; a.rhs = s->rhs; a.dx = dx_dev; a.info = info_dev;
  a.tile_row = s->tile_row; a.tile_col = s->tile_col; a.contrib_ptr = s->contrib_ptr; a.contrib = s->contrib;
  a.diag_tile = s->diag_tile; a.fixed = s->fixed;
  a.K = s->K; a.P = s->P; a.num_tiles = s->num_tiles;
  a.lambda = 0.0; a.prior = prior; a.diag_eps = diag_eps;
  FrameArgs fa{};
  fa.L = s->L; fa.F = s->F;
  fa.frame_ptr = s->frame_ptr; fa.frame_list = s->frame_list; fa.frame_pair = s->frame_pair; fa.frame_kf = s->frame_kf;
  fa.frame_L = s->frame_L; fa.frame_bad = s->frame_bad;
  if (prior > 0.0) {
    e = cudaMemcpyAsync(s->codes, codes_host, (size_t)s->K * s->C * sizeof(double),
                        codes_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, stream);
    if (e != cudaSuccess) return e;
  }
  const LoadedSet now = s->loaded[1 - s->cur], before = s->loaded[s->cur];
  SolveArgs al = a;  // the load launches write the new loaded set
  al.tiles = now.tiles; al.rhs = now.rhs;
  uint64_t n = 0;
  e = with_code_size(s->C, [&](auto bc) {
    constexpr int Bv = bc.value;
    if (s->F > 0)
      window_solve_load_kernel<Bv, true, true><<<s->num_tiles, kThreads, 0, stream>>>(al, fa);
    else
      window_solve_load_kernel<Bv, false, true><<<s->num_tiles, kThreads, 0, stream>>>(al, fa);
    ++n;
    if (s->prior_tiles > 0) {
      window_solve_prior_load_kernel<Bv><<<s->prior_tiles, kThreads, 0, stream>>>(al, s->pa);
      ++n;
    }
    return cudaGetLastError();
  });
  if (e != cudaSuccess) return e;
  int j0 = 0;
  if (reuse > 0) {
    // the first changed column decides how many column launches follow: the call's one synchronisation
    s->j0_host = reuse;
    if ((e = cudaMemcpyAsync(s->j0_dev, &s->j0_host, sizeof(int), cudaMemcpyHostToDevice, stream)) != cudaSuccess)
      return e;
    window_update_diff_kernel<<<reuse, kThreads, 0, stream>>>(now, before, s->diag_tile, s->K, s->num_tiles, s->B,
                                                               s->j0_dev);
    ++n;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if ((e = cudaMemcpyAsync(&s->j0_host, s->j0_dev, sizeof(int), cudaMemcpyDeviceToHost, stream)) != cudaSuccess)
      return e;
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
    j0 = s->j0_host;
  }
  s->cur = 1 - s->cur;  // this update's loaded system is the stored one from here on
  e = with_code_size(s->C, [&](auto bc) {
    constexpr int Bv = bc.value;
    if (j0 < s->K) {
      const int t0 = s->col_ptr[j0];
      window_update_replay_kernel<Bv><<<s->num_tiles - t0, kThreads, 0, stream>>>(a, now, s->ystore, s->rep_ptr,
                                                                                   s->rep_tasks, t0, j0);
      ++n;
    }
    for (int j = j0; j < s->K; ++j) {
      const int c0 = s->col_ptr[j], nc = s->col_ptr[j + 1] - c0;
      window_solve_panel_kernel<Bv><<<nc, kThreads, PanelCfg<Bv>::kSmem, stream>>>(a, j, c0, s->frame_bad, s->F);
      ++n;
      const int u0 = s->upd_ptr[j], nu = s->upd_ptr[j + 1] - u0;
      if (nu > 0) {
        window_solve_update_kernel<Bv><<<nu, kThreads, 0, stream>>>(a, s->tasks + u0, j);
        ++n;
      }
    }
    window_update_finish_kernel<Bv><<<1, kThreads, 0, stream>>>(a, s->ystore, s->frame_bad, s->F, j0);
    ++n;
    for (int j = s->K - 1; j >= 0; --j) {
      const int r0 = s->row_ptr[j], nr = s->row_ptr[j + 1] - r0;
      window_solve_backward_kernel<Bv><<<1 + nr, kThreads, (Bv * Bv + Bv) * 8, stream>>>(a, s->row_tiles + r0, j);
      ++n;
    }
    if (s->F > 0) {
      window_solve_frames_kernel<Bv><<<s->F, 32, 0, stream>>>(a, fa);
      ++n;
    }
    return cudaGetLastError();
  });
  *launches += n;
  if (e != cudaSuccess) return e;
  s->reuse = s->K;
  *first_column = j0;
  return cudaSuccess;
}

int window_solver_reusable_columns(const WindowSolverDev* prev, const WindowSolverDev* s)
{
  const int K = std::min(prev->K, s->K);
  int j = 0;
  for (; j < K; ++j) {
    const int a0 = prev->col_ptr[j], a1 = prev->col_ptr[j + 1], b0 = s->col_ptr[j], b1 = s->col_ptr[j + 1];
    if (a0 != b0 || a1 - a0 != b1 - b0 ||
        !std::equal(prev->tile_row_h.begin() + a0, prev->tile_row_h.begin() + a1, s->tile_row_h.begin() + b0))
      break;
  }
  return j;
}

bool window_solver_extends(const WindowSolverDev* prev, const WindowSolverDev* s)
{
  if (prev->C != s->C || prev->K > s->K) return false;
  return std::equal(prev->fixed_h.begin(), prev->fixed_h.end(), s->fixed_h.begin());
}

cudaError_t window_solver_adopt(WindowSolverDev* s, const WindowSolverDev* prev, cudaStream_t stream, int* columns)
{
  const int p = std::min(window_solver_reusable_columns(prev, s), prev->reuse);
  *columns = p;
  if (p == 0) return cudaSuccess;
  cudaError_t e = ensure_incremental(s);
  if (e != cudaSuccess) return e;
  const size_t BB = (size_t)s->B * s->B * sizeof(double), rows = (size_t)p * s->B * sizeof(double);
  const size_t head = (size_t)s->col_ptr[p] * BB;  // the same tiles in both: columns < p are numbered alike
  const LoadedSet& src = prev->loaded[prev->cur];
  const LoadedSet& dst = s->loaded[s->cur];
  const struct { void* d; const void* s; size_t n; } copies[] = {
      {s->tiles, prev->tiles, head},
      {s->tiles + (size_t)s->num_tiles * s->B * s->B, prev->tiles + (size_t)prev->num_tiles * prev->B * prev->B,
       (size_t)p * BB},  // L_jj slots
      {dst.tiles, src.tiles, head},
      {dst.rhs, src.rhs, rows},
      {s->ystore, prev->ystore, rows}};
  for (const auto& c : copies)
    if ((e = cudaMemcpyAsync(c.d, c.s, c.n, cudaMemcpyDeviceToDevice, stream)) != cudaSuccess) return e;
  s->reuse = p;
  return cudaSuccess;
}

// ----------------------------------------------------------------------------------- keyframe marginalisation
// Local tile system (dfk_window_marginalize_keyframe): tiles 0..n are column 0 ((I, 0), diagonal first), tile n + 1 +
// (I - 1) I / 2 + J - 1 is (I, J) for 1 <= J <= I <= n, slot T = n + 1 + n (n + 1) / 2 takes L_00.
void window_eliminate_first_tasks(int n, std::vector<int>& out)
{
  out.clear();
  for (int I = 1; I <= n; ++I)
    for (int J = 1; J <= I; ++J) {
      const UpdTask t{n + 1 + (I - 1) * I / 2 + J - 1, I, J, I == J ? I : -1};
      out.insert(out.end(), {t.target, t.a, t.b, t.rhs_row});
    }
}

cudaError_t launch_window_eliminate_first(int code_size, int n, double* tiles, double* rhs, int32_t* info,
                                          const void* tasks_dev, int num_tasks, cudaStream_t stream)
{
  SolveArgs a{};
  a.tiles = tiles; a.rhs = rhs; a.info = info;
  a.K = n + 1;
  a.num_tiles = n + 1 + n * (n + 1) / 2;
  return with_code_size(code_size, [&](auto bc) {
    constexpr int Bv = bc.value;
    cudaError_t e = cudaFuncSetAttribute(window_solve_panel_kernel<Bv>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         PanelCfg<Bv>::kSmem);
    if (e != cudaSuccess) return e;
    window_solve_panel_kernel<Bv><<<n + 1, kThreads, PanelCfg<Bv>::kSmem, stream>>>(a, 0, 0, nullptr, 0);
    if (num_tasks > 0)
      window_solve_update_kernel<Bv><<<num_tasks, kThreads, 0, stream>>>(a, static_cast<const UpdTask*>(tasks_dev), 0);
    return cudaGetLastError();
  });
}

}  // namespace dfk
