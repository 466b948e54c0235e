// dfk_window.cu -- device-side assembly of a keyframe window's block-sparse normal equations from the per-(pair, level)
// result records of SfmAligner::RunStep, i.e. what the factor graph does with them
// (sources/core/gtsam/photometric_factor.cpp:105-161: JtJ blocks G11 G12 G13 G22 G23 G33, g = -Jtr;  :275-282 residual
// rescale res / inliers * W * H) summed over the factors of a window (one factor per pair and level,
// sources/core/mapping/df_work.cpp:211-225), in the variable order [pose_k (6) | code_k (C)] per keyframe.
//
// Block-sparse layout (fp32, the buffer ONE all-reduce sums across GPUs; SURVEY 8e), B = 6 + C:
//   [ K diagonal blocks, B x B row-major, full symmetric ]   keyframe k's pose/code Hessian
//   [ K gradient blocks, B ]                                 g = -sum Jtr
//   [ P coupling blocks, B x 6 row-major ]                   pair p = (k0 -> k1): rows = k0's [pose0 | code0], cols = k1's pose1
//   [ f, inliers ]                                           sum of rescaled residuals (items with overlap), of the
//                                                            residuals of unscaled records (area 0) and of the links,
//                                                            photometric inliers
//   [ L link blocks, B x B row-major ]                       geometric link l = (k0 -> k1): rows = k0's [pose0 | code0],
//                                                            cols = k1's [pose1 | code1]
//   [ F frame blocks, 6 x 6 ] [ F frame gradients, 6 ]       tracked frame f (a pose-only variable): pose1 x pose1 and
//                                                            -Jtr(pose1) of its one pair (k0 -> K + f)
// A pair (k0 -> k1) adds its pose0/code0 blocks to keyframe k0's diagonal block, pose1 x pose1 to k1's, and the
// [pose0; code0] x pose1 coupling to its own block.  A geometric link (sparse_geometric_factor.cpp: keys pose0, pose1,
// code0, code1) adds its (pose0, code0) block to k0's diagonal block, its whole (pose1, code1) block to k1's, and the
// cross block to its own link block.
//
// Deterministic by construction: a GATHER, not a scatter -- every output element is owned by one thread, which sums the
// contributions of its items in list order, then those of the links (no float atomics).  One launch: grid = K + P + L + F
// + 1 jobs.  Without links every element is the same chain of adds as in a photometric / reprojection-only window; a
// frame pair's items are not in any keyframe's k1 list, so without frames nothing changes either.
//
// Also here: the marginalisation of frames into linear priors on their keyframe (the Schur complement of the frame's
// pose, what ISAM2::marginalizeLeaves leaves for a leaf with one factor) and the addition of such priors to a window;
// and for sliding the window, the keyframe priors: their addition to a window, and the gather and the write-out of the
// marginalisation of a keyframe (its elimination runs the solve's column-0 kernels, dfk_window_solve.cu).
#include <cuda_runtime.h>
#include <stdint.h>

#include "dfk_internal.h"

namespace dfk {

namespace {

__device__ __forceinline__ int packed_index(int i, int j, int NP) { return i * NP - (i * (i - 1)) / 2 + (j - i); }
// entry (a, b) of the symmetric (12+C)^2 Hessian of a record
__device__ __forceinline__ float rec_h(const float* rec, int a, int b, int NP)
{
  return a <= b ? rec[packed_index(a, b, NP)] : rec[packed_index(b, a, NP)];
}

// window row r of a link's keyframe k0 / k1 -> record row: pose0 0..5, pose1 6..11, code0 12..12+C-1, code1 12+C..
__device__ __forceinline__ int link_row0(int r) { return r < 6 ? r : 6 + r; }
__device__ __forceinline__ int link_row1(int r, int C) { return r < 6 ? 6 + r : 6 + C + r; }

__global__ void __launch_bounds__(256)
window_assemble_kernel(WindowDev w, const float* __restrict__ records, const float* __restrict__ geo,
                       float* __restrict__ out)
{
  const int C = w.code_size, B = 6 + C, NP = 12 + C;
  const int NH = NP * (NP + 1) / 2, REC = NH + NP + 2;
  const int NG = 12 + 2 * C, NHG = NG * (NG + 1) / 2, RECG = NHG + NG + 2;
  float* tail = out + (size_t)w.num_keyframes * (B * B + B) + (size_t)w.num_pairs * B * 6;
  const int job = blockIdx.x;
  if (job < w.num_keyframes) {
    // ---- diagonal block + gradient of keyframe k: items where k is the keyframe (k0) contribute the whole block, items
    // where k is the frame (k1) contribute pose1 x pose1 / g(pose1)
    const int k = job;
    float* D = out + (size_t)k * B * B;
    float* g = out + (size_t)w.num_keyframes * B * B + (size_t)k * B;
    const int a0 = w.kf0_ptr[k], a1 = w.kf0_ptr[k + 1];
    const int b0 = w.kf1_ptr[k], b1 = w.kf1_ptr[k + 1];
    const int l00 = w.lk0_ptr[k], l01 = w.lk0_ptr[k + 1];
    const int l10 = w.lk1_ptr[k], l11 = w.lk1_ptr[k + 1];
    for (int e = threadIdx.x; e < B * B + B; e += blockDim.x) {
      float s = 0.0f;
      if (e < B * B) {
        const int r = e / B, c = e - r * B;
        // window row r of keyframe k0 -> record row: pose0 0..5, code0 12..12+C-1
        const int lr = r < 6 ? r : 6 + r, lc = c < 6 ? c : 6 + c;
        for (int q = a0; q < a1; ++q) s += rec_h(records + (size_t)w.kf0_items[q] * REC, lr, lc, NP);
        if (r < 6 && c < 6)
          for (int q = b0; q < b1; ++q) s += rec_h(records + (size_t)w.kf1_items[q] * REC, 6 + r, 6 + c, NP);
        for (int q = l00; q < l01; ++q) s += rec_h(geo + (size_t)w.lk0_links[q] * RECG, link_row0(r), link_row0(c), NG);
        for (int q = l10; q < l11; ++q)
          s += rec_h(geo + (size_t)w.lk1_links[q] * RECG, link_row1(r, C), link_row1(c, C), NG);
        D[e] = s;
      } else {
        const int r = e - B * B;
        const int lr = r < 6 ? r : 6 + r;
        for (int q = a0; q < a1; ++q) s -= records[(size_t)w.kf0_items[q] * REC + NH + lr];
        if (r < 6)
          for (int q = b0; q < b1; ++q) s -= records[(size_t)w.kf1_items[q] * REC + NH + 6 + r];
        for (int q = l00; q < l01; ++q) s -= geo[(size_t)w.lk0_links[q] * RECG + NHG + link_row0(r)];
        for (int q = l10; q < l11; ++q) s -= geo[(size_t)w.lk1_links[q] * RECG + NHG + link_row1(r, C)];
        g[r] = s;
      }
    }
  } else if (job < w.num_keyframes + w.num_pairs) {
    // ---- coupling block of pair p: [pose0; code0] x pose1, summed over the pair's items (its pyramid levels)
    const int p = job - w.num_keyframes;
    float* O = out + (size_t)w.num_keyframes * (B * B + B) + (size_t)p * B * 6;
    const int i0 = w.pair_ptr[p], i1 = w.pair_ptr[p + 1];
    for (int e = threadIdx.x; e < B * 6; e += blockDim.x) {
      const int r = e / 6, c = e - r * 6;
      const int lr = r < 6 ? r : 6 + r;
      float s = 0.0f;
      for (int q = i0; q < i1; ++q) s += rec_h(records + (size_t)w.pair_items[q] * REC, lr, 6 + c, NP);
      O[e] = s;
    }
  } else if (job < w.num_keyframes + w.num_pairs + w.num_links) {
    // ---- link block of geometric link l: k0's [pose0; code0] x k1's [pose1 | code1], from its one record
    const int l = job - w.num_keyframes - w.num_pairs;
    float* O = tail + 2 + (size_t)l * B * B;
    const float* rec = geo + (size_t)l * RECG;
    for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
      const int r = e / B, c = e - r * B;
      O[e] = rec_h(rec, link_row0(r), link_row1(c, C), NG);
    }
  } else if (job < w.num_keyframes + w.num_pairs + w.num_links + w.num_frames) {
    // ---- frame f: pose1 x pose1 block and -Jtr(pose1) of its one pair's items, in item order
    const int f = job - w.num_keyframes - w.num_pairs - w.num_links;
    float* Df = tail + 2 + (size_t)w.num_links * B * B + (size_t)f * 36;
    float* gf = tail + 2 + (size_t)w.num_links * B * B + (size_t)w.num_frames * 36 + (size_t)f * 6;
    const int p = w.frame_pair[f];
    const int i0 = w.pair_ptr[p], i1 = w.pair_ptr[p + 1];
    for (int e = threadIdx.x; e < 42; e += blockDim.x) {
      float s = 0.0f;
      if (e < 36) {
        const int r = e / 6, c = e - r * 6;
        for (int q = i0; q < i1; ++q) s += rec_h(records + (size_t)w.pair_items[q] * REC, 6 + r, 6 + c, NP);
        Df[e] = s;
      } else {
        for (int q = i0; q < i1; ++q) s -= records[(size_t)w.pair_items[q] * REC + NH + 6 + (e - 36)];
        gf[e - 36] = s;
      }
    }
  } else {
    // ---- energy: f = sum res / inliers * W * H over items with overlap (photometric_factor.cpp:275-282) + res of the
    // unscaled records (reprojection factors, error() = 1/2 |b|^2, reprojection_factor.cpp:148), photometric inliers
    __shared__ float red_f[8], red_i[8];
    float f = 0.0f, ni = 0.0f;
    for (int i = threadIdx.x; i < w.num_items; i += blockDim.x) {
      const float* rec = records + (size_t)i * REC;
      const uint32_t inl = __float_as_uint(rec[NH + NP + 1]);
      if (w.item_area[i] == 0.0f) {  // unscaled record (reprojection factor): b^T b as it is, no photometric inliers
        f += rec[NH + NP];
      } else {
        if (inl > 0) f += rec[NH + NP] / (float)inl * w.item_area[i];
        ni += (float)inl;
      }
    }
    // geometric links: b^T b as it is (error() = 1/2 |b|^2 of the JacobianFactor), after the items
    for (int l = threadIdx.x; l < w.num_links; l += blockDim.x) f += geo[(size_t)l * RECG + NHG + NG];
    // fixed-order block reduction: lanes by xor butterfly, warps in index order
    for (int o = 16; o > 0; o >>= 1) {
      f += __shfl_xor_sync(0xffffffffu, f, o);
      ni += __shfl_xor_sync(0xffffffffu, ni, o);
    }
    if ((threadIdx.x & 31) == 0) {
      red_f[threadIdx.x >> 5] = f;
      red_i[threadIdx.x >> 5] = ni;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float sf = 0.0f, si = 0.0f;
      for (int k = 0; k < (int)(blockDim.x >> 5); ++k) {
        sf += red_f[k];
        si += red_i[k];
      }
      tail[0] = sf;
      tail[1] = si;
    }
  }
}

// fixed-order block sum of one double per thread (lanes by xor butterfly, warps in index order); every thread gets it
__device__ double block_sum(double v, double* red)
{
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();  // red is free again
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int k = 0; k < (int)(blockDim.x >> 5); ++k) s += red[k];
  return s;
}

constexpr int kMaxB = 6 + 128;

// ---- marginalisation of frame frames[i] (one CTA each): the fp64 sums of its pair's items, in item order, over the
// record rows a = [pose0 | code0] (keyframe k) and b = pose1 (the frame), then the Schur complement of b:
//   G = H_aa - H_ab H_bb^-1 H_ab^T,  g = g_a - H_ab H_bb^-1 g_b,  f0 = f_p - g_b^T H_bb^-1 g_b
// with H_bb = L L^T (6 x 6, undamped), Y = H_ab L^-T, z = L^-1 g_b: G = H_aa - Y Y^T, g = g_a - Y z, f0 = f_p - z^T z.
// Prior i: [G (B x B row-major) | g (B) | f0].  A pivot of H_bb that is not positive and finite: info[i] = 1 + its
// row, prior all zero.
__global__ void __launch_bounds__(256)
window_marginalize_kernel(WindowDev w, const float* __restrict__ records, const int* __restrict__ frames,
                          double* __restrict__ priors, int32_t* __restrict__ info)
{
  const int C = w.code_size, B = 6 + C, NP = 12 + C;
  const int NH = NP * (NP + 1) / 2, REC = NH + NP + 2;
  __shared__ double Hab[kMaxB * 6], Y[kMaxB * 6], ga[kMaxB], Hbb[36], L[36], gb[6], z[6];
  __shared__ int bad;
  const int p = w.frame_pair[frames[blockIdx.x]];
  const int i0 = w.pair_ptr[p], i1 = w.pair_ptr[p + 1];
  double* G = priors + (size_t)blockIdx.x * (B * B + B + 1);
  double* g = G + B * B;
  for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
    const int r = e / B, c = e - r * B;
    const int lr = r < 6 ? r : 6 + r, lc = c < 6 ? c : 6 + c;
    double s = 0.0;
    for (int q = i0; q < i1; ++q) s += (double)rec_h(records + (size_t)w.pair_items[q] * REC, lr, lc, NP);
    G[e] = s;
  }
  for (int e = threadIdx.x; e < B * 6 + 36 + B + 6; e += blockDim.x) {
    double s = 0.0;
    if (e < B * 6) {
      const int r = e / 6, c = e - r * 6, lr = r < 6 ? r : 6 + r;
      for (int q = i0; q < i1; ++q) s += (double)rec_h(records + (size_t)w.pair_items[q] * REC, lr, 6 + c, NP);
      Hab[e] = s;
    } else if (e < B * 6 + 36) {
      const int r = (e - B * 6) / 6, c = (e - B * 6) % 6;
      for (int q = i0; q < i1; ++q) s += (double)rec_h(records + (size_t)w.pair_items[q] * REC, 6 + r, 6 + c, NP);
      Hbb[e - B * 6] = s;
    } else if (e < B * 7 + 36) {
      const int r = e - B * 6 - 36, lr = r < 6 ? r : 6 + r;
      for (int q = i0; q < i1; ++q) s -= (double)records[(size_t)w.pair_items[q] * REC + NH + lr];
      ga[r] = s;
    } else {
      const int r = e - B * 7 - 36;
      for (int q = i0; q < i1; ++q) s -= (double)records[(size_t)w.pair_items[q] * REC + NH + 6 + r];
      gb[r] = s;
    }
  }
  // f_p: the rescaled residuals of the items with overlap (the items of a frame pair are all scaled)
  double fp = 0.0;
  if (threadIdx.x == 0)
    for (int q = i0; q < i1; ++q) {
      const float* rec = records + (size_t)w.pair_items[q] * REC;
      const uint32_t inl = __float_as_uint(rec[NH + NP + 1]);
      if (inl > 0) fp += (double)rec[NH + NP] / (double)inl * (double)w.item_area[w.pair_items[q]];
    }
  __syncthreads();
  if (threadIdx.x == 0) {
    int b = -1;
    for (int c = 0; c < 6; ++c) {
      double d = Hbb[c * 6 + c];
      for (int m = 0; m < c; ++m) d = __fma_rn(-L[c * 6 + m], L[c * 6 + m], d);
      if (b < 0 && !(d > 0.0 && d <= 1.7976931348623157e308)) b = c;
      d = sqrt(d);
      L[c * 6 + c] = d;
      for (int r = c + 1; r < 6; ++r) {
        double v = Hbb[r * 6 + c];
        for (int m = 0; m < c; ++m) v = __fma_rn(-L[r * 6 + m], L[c * 6 + m], v);
        L[r * 6 + c] = __ddiv_rn(v, d);
      }
    }
    for (int c = 0; c < 6; ++c) {
      double v = gb[c];
      for (int m = 0; m < c; ++m) v = __fma_rn(-L[c * 6 + m], z[m], v);
      z[c] = __ddiv_rn(v, L[c * 6 + c]);
    }
    bad = b;
  }
  __syncthreads();
  if (bad >= 0) {
    for (int e = threadIdx.x; e < B * B + B + 1; e += blockDim.x) G[e] = 0.0;
    if (threadIdx.x == 0) info[blockIdx.x] = 1 + bad;
    return;
  }
  for (int r = threadIdx.x; r < B; r += blockDim.x)  // Y L^T = H_ab, row by row
    for (int c = 0; c < 6; ++c) {
      double v = Hab[r * 6 + c];
      for (int m = 0; m < c; ++m) v = __fma_rn(-Y[r * 6 + m], L[c * 6 + m], v);
      Y[r * 6 + c] = __ddiv_rn(v, L[c * 6 + c]);
    }
  __syncthreads();
  for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
    const int r = e / B, c = e - r * B;
    double s = 0.0;
    for (int m = 0; m < 6; ++m) s = __fma_rn(Y[r * 6 + m], Y[c * 6 + m], s);
    G[e] = __dsub_rn(G[e], s);
  }
  for (int r = threadIdx.x; r < B; r += blockDim.x) {
    double s = 0.0;
    for (int m = 0; m < 6; ++m) s = __fma_rn(Y[r * 6 + m], z[m], s);
    g[r] = __dsub_rn(ga[r], s);
  }
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int m = 0; m < 6; ++m) s = __fma_rn(z[m], z[m], s);
    g[B] = __dsub_rn(fp, s);
    info[blockIdx.x] = 0;
  }
}

// ---- priors into an assembled window, in place.  Prior i on keyframe k with delta_i = Local(x0_i, x):
//   D_k += G,  g_k += g - G delta,  f += f0 - 2 g^T delta + delta^T G delta
// CTA k < K: keyframe k's block and gradient, its priors in list order summed in fp64 onto the fp32 entry, rounded
// once.  CTA K: f, every prior in list order (the inlier total is left alone).
__global__ void __launch_bounds__(256)
window_add_priors_kernel(WindowDev w, int m, const int* __restrict__ kf_ptr, const int* __restrict__ kf_priors,
                         const double* __restrict__ priors, const double* __restrict__ delta, float* __restrict__ out)
{
  const int C = w.code_size, B = 6 + C, PD = B * B + B + 1;
  const int K = w.num_keyframes;
  if ((int)blockIdx.x < K) {
    const int k = blockIdx.x, q0 = kf_ptr[k], q1 = kf_ptr[k + 1];
    if (q0 == q1) return;
    float* D = out + (size_t)k * B * B;
    float* g = out + (size_t)K * B * B + (size_t)k * B;
    for (int e = threadIdx.x; e < B * B + B; e += blockDim.x) {
      if (e < B * B) {
        double s = (double)D[e];
        for (int q = q0; q < q1; ++q) s = __dadd_rn(s, priors[(size_t)kf_priors[q] * PD + e]);
        D[e] = (float)s;
      } else {
        const int r = e - B * B;
        double s = (double)g[r];
        for (int q = q0; q < q1; ++q) {
          const double* P = priors + (size_t)kf_priors[q] * PD;
          const double* d = delta + (size_t)kf_priors[q] * B;
          double gd = 0.0;
          for (int c = 0; c < B; ++c) gd = __fma_rn(P[r * B + c], d[c], gd);
          s = __dadd_rn(s, __dsub_rn(P[B * B + r], gd));
        }
        g[r] = (float)s;
      }
    }
    return;
  }
  __shared__ double red[8];
  float* tail = out + (size_t)K * (B * B + B) + (size_t)w.num_pairs * B * 6;
  double s = (double)tail[0];
  for (int i = 0; i < m; ++i) {
    const double* P = priors + (size_t)i * PD;
    const double* d = delta + (size_t)i * B;
    double gd = 0.0, dGd = 0.0;
    for (int r = threadIdx.x; r < B; r += blockDim.x) {
      double Gd = 0.0;
      for (int c = 0; c < B; ++c) Gd = __fma_rn(P[r * B + c], d[c], Gd);
      gd = __fma_rn(P[B * B + r], d[r], gd);
      dGd = __fma_rn(d[r], Gd, dGd);
    }
    gd = block_sum(gd, red);
    dGd = block_sum(dGd, red);
    s = __dadd_rn(s, __dadd_rn(__fma_rn(-2.0, gd, P[B * B + B]), dGd));
  }
  if (threadIdx.x == 0) tail[0] = (float)s;
}

// ---- keyframe priors into an assembled window, in place.  Prior q over keyframes kf_q (n_q of them) at delta_q:
//   D_k += G_q(a, a),  prior block (i, j) += G_q(a, c),  g_k += (g_q - G_q delta_q)(a),
//   f += f0_q - 2 g_q^T delta_q + delta_q^T G_q delta_q
// (k = kf_q[a], i = kf_q[a], j = kf_q[c]).  CTA k < K: keyframe k's block and gradient; CTA K + b: prior block b; CTA
// K + Qb: f.  Every entry sums its priors in prior order in fp64 onto its fp32 value and is rounded once.
__device__ __forceinline__ const double* kf_prior(const KfPriorDev& kp, const double* priors, int q)
{
  return priors + kp.off[q];
}

__global__ void __launch_bounds__(256)
window_add_kf_priors_kernel(WindowDev w, KfPriorDev kp, const double* __restrict__ priors,
                            const double* __restrict__ delta, float* __restrict__ out)
{
  const int C = w.code_size, B = 6 + C, K = w.num_keyframes;
  const int job = blockIdx.x;
  if (job < K) {
    const int k = job, q0 = kp.kf_ptr[k], q1 = kp.kf_ptr[k + 1];
    if (q0 == q1) return;
    float* D = out + (size_t)k * B * B;
    float* g = out + (size_t)K * B * B + (size_t)k * B;
    for (int e = threadIdx.x; e < B * B + B; e += blockDim.x) {
      if (e < B * B) {
        const int r = e / B, c = e - r * B;
        double s = (double)D[e];
        for (int q = q0; q < q1; ++q) {
          const int p = kp.kf_ent[q].x, a = kp.kf_ent[q].y;
          const size_t nB = (size_t)(kp.mem_ptr[p + 1] - kp.mem_ptr[p]) * B;
          s = __dadd_rn(s, kf_prior(kp, priors, p)[(a * B + r) * nB + a * B + c]);
        }
        D[e] = (float)s;
      } else {
        const int r = e - B * B;
        double s = (double)g[r];
        for (int q = q0; q < q1; ++q) {
          const int p = kp.kf_ent[q].x, a = kp.kf_ent[q].y;
          const int nB = (kp.mem_ptr[p + 1] - kp.mem_ptr[p]) * B;
          const double* G = kf_prior(kp, priors, p) + (size_t)(a * B + r) * nB;
          const double* d = delta + (size_t)kp.mem_ptr[p] * B;
          double gd = 0.0;
          for (int c = 0; c < nB; ++c) gd = __fma_rn(G[c], d[c], gd);
          s = __dadd_rn(s, __dsub_rn(kf_prior(kp, priors, p)[(size_t)nB * nB + a * B + r], gd));
        }
        g[r] = (float)s;
      }
    }
    return;
  }
  if (job < K + kp.num_blocks) {
    const int b = job - K;
    float* O = out + kp.block_off + (size_t)b * B * B;
    for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
      const int r = e / B, c = e - r * B;
      double s = (double)O[e];
      for (int q = kp.blk_ptr[b]; q < kp.blk_ptr[b + 1]; ++q) {
        const int p = kp.blk_ent[q].x, a = kp.blk_ent[q].y, cc = kp.blk_ent[q].z;
        const size_t nB = (size_t)(kp.mem_ptr[p + 1] - kp.mem_ptr[p]) * B;
        s = __dadd_rn(s, kf_prior(kp, priors, p)[(a * B + r) * nB + cc * B + c]);
      }
      O[e] = (float)s;
    }
    return;
  }
  __shared__ double red[8];
  float* tail = out + (size_t)K * (B * B + B) + (size_t)w.num_pairs * B * 6;
  double s = (double)tail[0];
  for (int p = 0; p < kp.num_priors; ++p) {
    const int nB = (kp.mem_ptr[p + 1] - kp.mem_ptr[p]) * B;
    const double* P = kf_prior(kp, priors, p);
    const double* d = delta + (size_t)kp.mem_ptr[p] * B;
    double gd = 0.0, dGd = 0.0;
    for (int r = threadIdx.x; r < nB; r += blockDim.x) {
      double Gd = 0.0;
      for (int c = 0; c < nB; ++c) Gd = __fma_rn(P[(size_t)r * nB + c], d[c], Gd);
      gd = __fma_rn(P[(size_t)nB * nB + r], d[r], gd);
      dGd = __fma_rn(d[r], Gd, dGd);
    }
    gd = block_sum(gd, red);
    dGd = block_sum(dGd, red);
    s = __dadd_rn(s, __dadd_rn(__fma_rn(-2.0, gd, P[(size_t)nB * nB + nB]), dGd));
  }
  if (threadIdx.x == 0) tail[0] = (float)s;
}

// ---- marginalisation of a keyframe m: the local fp64 system over [m | N(m)] of the factors that touch m (KfMargDev).
// CTA t < T: local tile t, each entry summing the refs in order; CTA T: the gradient (every thread its rows) and f
// (block sums in ref order).
// record rows of local keyframe X's variable r in a pair record (k0 / k1 local l0 / l1): up to two (a self pair)
__device__ __forceinline__ int pair_rows(const KfMargRef& f, int X, int r, int* rows)
{
  int n = 0;
  if (X == f.l0) rows[n++] = r < 6 ? r : 6 + r;
  if (X == f.l1 && r < 6) rows[n++] = 6 + r;
  return n;
}

__device__ __forceinline__ int member_pos(const KfPriorDev& kp, const KfMargDev& md, int p, int X)
{
  for (int a = kp.mem_ptr[p]; a < kp.mem_ptr[p + 1]; ++a)
    if (md.mem_loc[a] == X) return a - kp.mem_ptr[p];
  return -1;
}

__global__ void __launch_bounds__(256)
window_marg_gather_kernel(WindowDev w, KfPriorDev kp, KfMargDev md, int num_tiles)
{
  const int C = w.code_size, B = 6 + C, NP = 12 + C;
  const int NH = NP * (NP + 1) / 2, REC = NH + NP + 2;
  const int NG = 12 + 2 * C, NHG = NG * (NG + 1) / 2, RECG = NHG + NG + 2;
  const int PD = B * B + B + 1;
  if ((int)blockIdx.x < num_tiles) {
    const int t = blockIdx.x, I = md.tile_row[t], J = md.tile_col[t];
    double* T = md.tiles + (size_t)t * B * B;
    for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
      const int r = e / B, c = e - r * B;
      double s = 0.0;
      for (int q = 0; q < md.num_refs; ++q) {
        const KfMargRef f = md.refs[q];
        if (f.kind == 0) {
          int ra[2], cb[2];
          const int na = pair_rows(f, I, r, ra), nb = pair_rows(f, J, c, cb);
          const float* rec = md.records + (size_t)f.idx * REC;
          for (int u = 0; u < na; ++u)
            for (int v = 0; v < nb; ++v) s += (double)rec_h(rec, ra[u], cb[v], NP);
        } else if (f.kind == 1) {
          const int ra = I == f.l0 ? link_row0(r) : (I == f.l1 ? link_row1(r, C) : -1);
          const int cb = J == f.l0 ? link_row0(c) : (J == f.l1 ? link_row1(c, C) : -1);
          if (ra >= 0 && cb >= 0) s += (double)rec_h(md.geo + (size_t)f.idx * RECG, ra, cb, NG);
        } else if (f.kind == 2) {
          if (I == 0 && J == 0) s += md.fpriors[(size_t)f.idx * PD + e];
        } else {
          const int a = member_pos(kp, md, f.idx, I), b = member_pos(kp, md, f.idx, J);
          if (a >= 0 && b >= 0) {
            const size_t nB = (size_t)(kp.mem_ptr[f.idx + 1] - kp.mem_ptr[f.idx]) * B;
            s += md.kpriors[kp.off[f.idx] + (a * B + r) * nB + b * B + c];
          }
        }
      }
      if (I == 0 && J == 0 && r == c && r >= 6 && md.w > 0.0) s += md.w;
      T[e] = s;
    }
    return;
  }
  // gradient of local variable (X, r), then f
  const int N = (md.n + 1) * B;
  for (int v = threadIdx.x; v < N; v += blockDim.x) {
    const int X = v / B, r = v - X * B;
    double s = 0.0;
    for (int q = 0; q < md.num_refs; ++q) {
      const KfMargRef f = md.refs[q];
      if (f.kind == 0) {
        int ra[2];
        const int na = pair_rows(f, X, r, ra);
        for (int u = 0; u < na; ++u) s -= (double)md.records[(size_t)f.idx * REC + NH + ra[u]];
      } else if (f.kind == 1) {
        const int ra = X == f.l0 ? link_row0(r) : (X == f.l1 ? link_row1(r, C) : -1);
        if (ra >= 0) s -= (double)md.geo[(size_t)f.idx * RECG + NHG + ra];
      } else if (f.kind == 2) {
        if (X == 0) {
          const double* P = md.fpriors + (size_t)f.idx * PD;
          const double* d = md.fdelta + (size_t)f.idx * B;
          double gd = 0.0;
          for (int c = 0; c < B; ++c) gd = __fma_rn(P[r * B + c], d[c], gd);
          s += P[B * B + r] - gd;
        }
      } else {
        const int a = member_pos(kp, md, f.idx, X);
        if (a >= 0) {
          const int nB = (kp.mem_ptr[f.idx + 1] - kp.mem_ptr[f.idx]) * B;
          const double* P = md.kpriors + kp.off[f.idx];
          const double* d = md.kdelta + (size_t)kp.mem_ptr[f.idx] * B;
          double gd = 0.0;
          for (int c = 0; c < nB; ++c) gd = __fma_rn(P[(size_t)(a * B + r) * nB + c], d[c], gd);
          s += P[(size_t)nB * nB + a * B + r] - gd;
        }
      }
    }
    if (X == 0 && r >= 6 && md.w > 0.0) s -= md.w * md.code[r - 6];
    md.rhs[v] = s;
  }
  __shared__ double red[8];
  double f = 0.0;  // thread 0's running sum; the block sums below are the same on every thread
  for (int q = 0; q < md.num_refs; ++q) {
    const KfMargRef fr = md.refs[q];
    if (fr.kind == 0) {
      if (threadIdx.x == 0) {
        const float* rec = md.records + (size_t)fr.idx * REC;
        const float area = w.item_area[fr.idx];
        const uint32_t inl = __float_as_uint(rec[NH + NP + 1]);
        if (area == 0.0f) f += (double)rec[NH + NP];
        else if (inl > 0) f += (double)rec[NH + NP] / (double)inl * (double)area;
      }
    } else if (fr.kind == 1) {
      if (threadIdx.x == 0) f += (double)md.geo[(size_t)fr.idx * RECG + NHG + NG];
    } else {
      const bool fp = fr.kind == 2;
      const int nB = fp ? B : (kp.mem_ptr[fr.idx + 1] - kp.mem_ptr[fr.idx]) * B;
      const double* P = fp ? md.fpriors + (size_t)fr.idx * PD : md.kpriors + kp.off[fr.idx];
      const double* d = fp ? md.fdelta + (size_t)fr.idx * B : md.kdelta + (size_t)kp.mem_ptr[fr.idx] * B;
      double gd = 0.0, dGd = 0.0;
      for (int r = threadIdx.x; r < nB; r += blockDim.x) {
        double Gd = 0.0;
        for (int c = 0; c < nB; ++c) Gd = __fma_rn(P[(size_t)r * nB + c], d[c], Gd);
        gd = __fma_rn(P[(size_t)nB * nB + r], d[r], gd);
        dGd = __fma_rn(d[r], Gd, dGd);
      }
      gd = block_sum(gd, red);
      dGd = block_sum(dGd, red);
      f = __dadd_rn(f, __dadd_rn(__fma_rn(-2.0, gd, P[(size_t)nB * nB + nB]), dGd));
    }
  }
  if (threadIdx.x == 0) {
    if (md.w > 0.0) {
      double cc = 0.0;
      for (int c = 0; c < C; ++c) cc = __fma_rn(md.code[c], md.code[c], cc);
      f = __fma_rn(md.w, cc, f);
    }
    *md.f = f;
    *md.info = 0;  // the elimination's panel launch reports a failed pivot here
  }
}

// ---- the prior out of the eliminated local system: CTA u < n(n+1)/2 writes tile (I, J) = G block (I-1, J-1) and its
// transpose; the last CTA g (local blocks 1..n of the rhs) and f0 = f - z^T z.  A failed pivot: all zero.
__global__ void __launch_bounds__(256)
window_marg_finalize_kernel(int C, KfMargDev md, int num_tiles, double* __restrict__ prior)
{
  const int B = 6 + C, n = md.n, nB = n * B;
  const bool bad = *md.info != 0;
  const int u = blockIdx.x, nt = n * (n + 1) / 2;
  if (u < nt) {
    const int t = n + 1 + u, I = md.tile_row[t], J = md.tile_col[t];
    const double* T = md.tiles + (size_t)t * B * B;
    for (int e = threadIdx.x; e < B * B; e += blockDim.x) {
      const int r = e / B, c = e - r * B;
      if (I == J && r < c) continue;  // a diagonal tile: its lower triangle writes both halves
      const double v = bad ? 0.0 : T[e];
      prior[(size_t)((I - 1) * B + r) * nB + (J - 1) * B + c] = v;
      prior[(size_t)((J - 1) * B + c) * nB + (I - 1) * B + r] = v;
    }
    return;
  }
  for (int v = threadIdx.x; v < nB; v += blockDim.x) prior[(size_t)nB * nB + v] = bad ? 0.0 : md.rhs[B + v];
  if (threadIdx.x == 0) {
    double zz = 0.0;
    for (int r = 0; r < B; ++r) zz = __fma_rn(md.rhs[r], md.rhs[r], zz);
    prior[(size_t)nB * nB + nB] = bad ? 0.0 : __dsub_rn(*md.f, zz);
  }
}

}  // namespace

cudaError_t launch_window_assemble(const WindowDev& w, const float* records_dev, const float* geo_records_dev,
                                   float* out_dev, cudaStream_t stream)
{
  window_assemble_kernel<<<w.num_keyframes + w.num_pairs + w.num_links + w.num_frames + 1, 256, 0, stream>>>(
      w, records_dev, geo_records_dev, out_dev);
  return cudaGetLastError();
}

cudaError_t launch_window_marginalize_frames(const WindowDev& w, const float* records_dev, int n, const int* frames_dev,
                                             double* priors_dev, int32_t* info_dev, cudaStream_t stream)
{
  window_marginalize_kernel<<<n, 256, 0, stream>>>(w, records_dev, frames_dev, priors_dev, info_dev);
  return cudaGetLastError();
}

cudaError_t launch_window_add_priors(const WindowDev& w, int m, const int* kf_ptr_dev, const int* kf_priors_dev,
                                     const double* priors_dev, const double* delta_dev, float* window_dev,
                                     cudaStream_t stream)
{
  window_add_priors_kernel<<<w.num_keyframes + 1, 256, 0, stream>>>(w, m, kf_ptr_dev, kf_priors_dev, priors_dev,
                                                                    delta_dev, window_dev);
  return cudaGetLastError();
}

cudaError_t launch_window_add_keyframe_priors(const WindowDev& w, const KfPriorDev& kp, const double* priors_dev,
                                              const double* delta_dev, float* window_dev, cudaStream_t stream)
{
  window_add_kf_priors_kernel<<<w.num_keyframes + kp.num_blocks + 1, 256, 0, stream>>>(w, kp, priors_dev, delta_dev,
                                                                                       window_dev);
  return cudaGetLastError();
}

cudaError_t launch_window_marg_gather(const WindowDev& w, const KfPriorDev& kp, const KfMargDev& md, int num_tiles,
                                      cudaStream_t stream)
{
  window_marg_gather_kernel<<<num_tiles + 1, 256, 0, stream>>>(w, kp, md, num_tiles);
  return cudaGetLastError();
}

cudaError_t launch_window_marg_finalize(int code_size, const KfMargDev& md, int num_tiles, double* prior_dev,
                                       cudaStream_t stream)
{
  window_marg_finalize_kernel<<<md.n * (md.n + 1) / 2 + 1, 256, 0, stream>>>(code_size, md, num_tiles, prior_dev);
  return cudaGetLastError();
}

}  // namespace dfk
