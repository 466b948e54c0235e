/* dfk_bow_oracle.c -- CPU oracle of the dfk_bow_* calls (TEST INFRASTRUCTURE ONLY).
 *
 * Follows steps 1-6 of include/dfk.h's DBoW2 block literally and sequentially, one descriptor, vector or query at a
 * time: the tree as listed (children in file order, no re-indexing), sorted arrays standing in for DBoW2's std::map,
 * and the per-element arithmetic of deepfactors_b200/csrc/dfk_bow_model.h.  No validation: the callers pass trees
 * that dfk_bow_vocabulary_create accepts.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "dfk_bow_model.h"

typedef struct {
  int n, d32;          /* listed nodes, descriptor words */
  int* first;          /* [n + 2]: children of node id p are kids[first[p] .. first[p + 1]) */
  int* kids;           /* node ids in file order */
  int* word;           /* [n + 1] word of a leaf id, -1 inside */
  double* weight;      /* [n + 1] */
  uint32_t* desc;      /* [n + 1, d32] by node id */
} Voc;

void* dfkb_voc_create(int n, const int32_t* ids, const int32_t* parents, const double* weights, const uint8_t* desc,
                      int bytes, int num_words, const int32_t* word_ids, const int32_t* word_nodes)
{
  Voc* v = (Voc*)calloc(1, sizeof(Voc));
  if (!v) return NULL;
  v->n = n;
  v->d32 = bytes / 4;
  v->first = (int*)calloc((size_t)n + 2, sizeof(int));
  v->kids = (int*)calloc((size_t)n + 1, sizeof(int));
  v->word = (int*)malloc(sizeof(int) * ((size_t)n + 1));
  v->weight = (double*)calloc((size_t)n + 1, sizeof(double));
  v->desc = (uint32_t*)calloc(((size_t)n + 1) * v->d32, sizeof(uint32_t));
  int* fill = (int*)calloc((size_t)n + 2, sizeof(int));
  if (!v->first || !v->kids || !v->word || !v->weight || !v->desc || !fill) return NULL;
  for (int i = 0; i < n; ++i) v->first[parents[i] + 1]++;
  for (int p = 0; p <= n; ++p) v->first[p + 1] += v->first[p];
  memcpy(fill, v->first, sizeof(int) * ((size_t)n + 1));
  for (int i = 0; i < n; ++i) {
    v->kids[fill[parents[i]]++] = ids[i];  /* m_nodes[pid].children.push_back(nid), in file order */
    v->weight[ids[i]] = weights[i];
    memcpy(v->desc + (size_t)ids[i] * v->d32, desc + (size_t)i * bytes, (size_t)bytes);
  }
  for (int i = 0; i <= n; ++i) v->word[i] = -1;
  for (int j = 0; j < num_words; ++j) v->word[word_nodes[j]] = word_ids[j];
  free(fill);
  return v;
}

void dfkb_voc_free(void* p)
{
  Voc* v = (Voc*)p;
  if (!v) return;
  free(v->first);
  free(v->kids);
  free(v->word);
  free(v->weight);
  free(v->desc);
  free(v);
}

/* step 2 for one descriptor */
static void word_of(const Voc* v, const uint32_t* f, int* word, double* weight)
{
  int id = 0;
  do {
    const int* c = v->kids + v->first[id];
    const int nc = v->first[id + 1] - v->first[id];
    int best = c[0];
    int best_d = dfk_bow_distance(f, v->desc + (size_t)best * v->d32, v->d32);
    for (int k = 1; k < nc; ++k) {
      const int d = dfk_bow_distance(f, v->desc + (size_t)c[k] * v->d32, v->d32);
      if (d < best_d) {
        best_d = d;
        best = c[k];
      }
    }
    id = best;
  } while (v->first[id + 1] > v->first[id]);
  *word = v->word[id];
  *weight = v->weight[id];
}

/* steps 2-3 for one image of m descriptors (rows of bytes): feature_words [m] (-1: weight not > 0), the vector's
 * words and values (capacity m); returns its word count */
int dfkb_transform(const void* voc, const uint8_t* desc, int m, int32_t* feature_words, int32_t* words,
                   double* values)
{
  const Voc* v = (const Voc*)voc;
  uint32_t f[16];
  int cnt = 0;
  for (int i = 0; i < m; ++i) {
    memcpy(f, desc + (size_t)i * v->d32 * 4, (size_t)v->d32 * 4);
    int w;
    double wt;
    word_of(v, f, &w, &wt);
    if (!(wt > 0)) {
      feature_words[i] = -1;
      continue;
    }
    feature_words[i] = w;
    /* v.addWeight(id, w): find or insert in the ordered map */
    int lo = 0, hi = cnt;
    while (lo < hi) {
      const int mid = (lo + hi) / 2;
      if (words[mid] < w) lo = mid + 1;
      else hi = mid;
    }
    if (lo < cnt && words[lo] == w) {
      values[lo] += wt;
    } else {
      memmove(words + lo + 1, words + lo, sizeof(int32_t) * (size_t)(cnt - lo));
      memmove(values + lo + 1, values + lo, sizeof(double) * (size_t)(cnt - lo));
      words[lo] = w;
      values[lo] = wt;
      ++cnt;
    }
  }
  double norm = 0.0;
  for (int k = 0; k < cnt; ++k) norm += fabs(values[k]);
  if (norm > 0.0)
    for (int k = 0; k < cnt; ++k) values[k] = values[k] / norm;
  return cnt;
}

static int find(const int32_t* words, int n, int32_t w)
{
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) / 2;
    if (words[mid] < w) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

typedef struct {
  double sum;
  int id;
} Pair;

static int by_sum_then_id(const void* a, const void* b)
{
  const Pair* x = (const Pair*)a;
  const Pair* y = (const Pair*)b;
  if (x->sum < y->sum) return -1;
  if (x->sum > y->sum) return 1;
  return (x->id > y->id) - (x->id < y->id);
}

/* step 5 against entries 0..E-1 (entry e's vector: ew / ev rows [offsets[e], offsets[e] + counts[e])): ids / scores
 * [max_results]; returns the count before the cut, or -1 when out of memory */
int dfkb_query(const int32_t* qw, const double* qv, int qn, int E, const int64_t* offsets, const int32_t* counts,
               const int32_t* ew, const double* ev, int max_results, int max_id, int32_t* ids, double* scores)
{
  double* sums = (double*)calloc((size_t)E + 1, sizeof(double));
  char* has = (char*)calloc((size_t)E + 1, 1);
  if (!sums || !has) return -1;
  /* for each query word, the inverted file's row: the entries holding it, in entry order */
  for (int k = 0; k < qn; ++k)
    for (int e = 0; e < E; ++e) {
      if (!(e < max_id || max_id == -1)) continue;
      const int32_t* w = ew + offsets[e];
      const int p = find(w, counts[e], qw[k]);
      if (p == counts[e] || w[p] != qw[k]) continue;
      const double t = dfk_bow_l1_term(qv[k], ev[offsets[e] + p]);
      if (has[e]) sums[e] += t;
      else sums[e] = t;
      has[e] = 1;
    }
  int cnt = 0;
  for (int e = 0; e < E; ++e) cnt += has[e];
  Pair* r = (Pair*)malloc(sizeof(Pair) * ((size_t)cnt + 1));
  if (!r) return -1;
  int j = 0;
  for (int e = 0; e < E; ++e)
    if (has[e]) r[j++] = (Pair){sums[e], e};
  qsort(r, (size_t)cnt, sizeof(Pair), by_sum_then_id);
  const int keep = cnt < max_results ? cnt : max_results;
  for (int k = 0; k < keep; ++k) {
    ids[k] = r[k].id;
    scores[k] = dfk_bow_final_score(r[k].sum);
  }
  free(r);
  free(sums);
  free(has);
  return cnt;
}

/* step 6: L1Scoring::score(a, b), DBoW2's merge with its lower_bound jumps */
double dfkb_score(const int32_t* aw, const double* av, int an, const int32_t* bw, const double* bv, int bn)
{
  int i = 0, j = 0;
  double score = 0;
  while (i < an && j < bn) {
    if (aw[i] == bw[j]) {
      score += dfk_bow_l1_term(av[i], bv[j]);
      ++i;
      ++j;
    } else if (aw[i] < bw[j]) {
      i += find(aw + i, an - i, bw[j]);
    } else {
      j += find(bw + j, bn - j, aw[i]);
    }
  }
  return dfk_bow_final_score(score);
}
