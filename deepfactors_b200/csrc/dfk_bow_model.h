/* dfk_bow_model.h -- the per-element arithmetic of DBoW2 retrieval (include/dfk.h dfk_bow_*, DESIGN.md section 4.11),
 * in plain C so that the device build (dfk_bow.cu, nvcc -fmad=false) and a sequential CPU build of the specification
 * (gcc -ffp-contract=off), which checks the kernels, round the same way.  There are no products: every value is a sum
 * or a difference of fp64 numbers taken in the order the callers give, and the L1 norm is a division.
 *
 *   distance   popcount of (a ^ b) over the descriptor's 32-bit words (FBrisk / FORB distance)
 *   l1_term    fabs(x - y) - fabs(x) - fabs(y), left to right: L1Scoring::score and queryL1's per-word term, with
 *              (x, y) = (query, entry) in a query and (a, b) in a score; the two operand orders round differently
 *   score      -sum / 2.0 (a sum of 0.0, i.e. no common word, gives -0.0)
 */
#ifndef DFK_BOW_MODEL_H
#define DFK_BOW_MODEL_H

#include <stdint.h>

#ifdef __CUDACC__
#define DFK_BOW_FN static __host__ __device__ __forceinline__
#else
#include <math.h>
#define DFK_BOW_FN static inline
#endif

/* the deepest tree a descent follows and the widest node (one warp lane per child) */
#define DFK_BOW_MODEL_MAX_DEPTH 16
#define DFK_BOW_MODEL_MAX_K 32

DFK_BOW_FN int dfk_bow_popc(uint32_t x)
{
#if defined(__CUDA_ARCH__)
  return __popc(x);
#else
  return __builtin_popcount(x);
#endif
}

/* Hamming distance of two descriptors of `words` 32-bit words */
DFK_BOW_FN int dfk_bow_distance(const uint32_t* a, const uint32_t* b, int words)
{
  int d = 0;
  for (int i = 0; i < words; ++i) d += dfk_bow_popc(a[i] ^ b[i]);
  return d;
}

DFK_BOW_FN double dfk_bow_l1_term(double x, double y)
{
  return fabs(x - y) - fabs(x) - fabs(y);
}

/* a word seen n >= 1 times: w, then n - 1 more additions of w in sequence (BowVector::addWeight), not n * w */
DFK_BOW_FN double dfk_bow_repeat(double w, int n)
{
  double v = w;
  for (int i = 1; i < n; ++i) v += w;
  return v;
}

DFK_BOW_FN double dfk_bow_final_score(double sum)
{
  return -sum / 2.0;
}

/* ---- vocabulary training (include/dfk.h, the DBoW2 training block): each node's SplitMix64 stream */
DFK_BOW_FN uint64_t dfk_bow_mix64(uint64_t z)
{
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

DFK_BOW_FN uint64_t dfk_bow_next(uint64_t* s)
{
  *s += 0x9E3779B97F4A7C15ull;
  return dfk_bow_mix64(*s);
}

DFK_BOW_FN uint64_t dfk_bow_child_key(uint64_t key, int i)
{
  return dfk_bow_mix64(key + (uint64_t)(i + 1) * 0xD1B54A32D192ED03ull);
}

/* the first centre's index in [0, m) */
DFK_BOW_FN int64_t dfk_bow_draw_index(uint64_t* s, int64_t m)
{
  const uint64_t r = dfk_bow_next(s);
#if defined(__CUDA_ARCH__)
  return (int64_t)__umul64hi(r, (uint64_t)m);
#else
  return (int64_t)(((unsigned __int128)r * (uint64_t)m) >> 64);
#endif
}

/* a cut in (0, dist_sum], dist_sum > 0 */
DFK_BOW_FN double dfk_bow_draw_cut(uint64_t* s, int64_t dist_sum)
{
  double cut;
  do {
    cut = ((double)(dfk_bow_next(s) >> 11) * 0x1p-53) * (double)dist_sum;
  } while (cut == 0.0);
  return cut;
}

/* the least integer prefix sum that is >= cut (cut <= 2^53, so the ceiling is exact) */
DFK_BOW_FN int64_t dfk_bow_cut_target(double cut)
{
  return (int64_t)ceil(cut);
}

#endif /* DFK_BOW_MODEL_H */
