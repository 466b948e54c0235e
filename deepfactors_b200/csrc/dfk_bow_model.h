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

#endif /* DFK_BOW_MODEL_H */
