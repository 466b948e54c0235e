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

#define DFK_BOW_TRAIN_MAX_ROUNDS 1000 /* include/dfk.h */

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

/* ---- vocabulary training: include/dfk.h's DBoW2 training block, followed literally -----------------------------
 * TemplatedVocabulary::create as DBoW2 runs it: HKmeansStep one node at a time in its depth-first recursion, min_dist
 * and its sums in double as DBoW2 keeps them, then createWords and setNodeWeights with a descent per descriptor.  The
 * random draws are dfk_bow_model.h's per-node streams (the block's deviation 1). */
typedef struct {
  int n, cap, k, L, bytes, d32;
  int32_t* parent;     /* [id] */
  int32_t* first;      /* [id] first child id (children are consecutive ids) */
  int32_t* nchild;     /* [id] */
  uint64_t* key;       /* [id] */
  double* weight;      /* [id] */
  uint32_t* desc;      /* [id, d32] */
  int32_t stats[5 + 16]; /* num_nodes, num_words, max_rounds, capped_nodes, empty_clusters, level_max_rounds[16] */
  int failed;
} Tree;

static int tree_add(Tree* t, int parent, const uint32_t* d)
{
  if (t->n == t->cap) {
    const int cap = t->cap ? 2 * t->cap : 1024;
    t->parent = (int32_t*)realloc(t->parent, sizeof(int32_t) * (size_t)cap);
    t->first = (int32_t*)realloc(t->first, sizeof(int32_t) * (size_t)cap);
    t->nchild = (int32_t*)realloc(t->nchild, sizeof(int32_t) * (size_t)cap);
    t->key = (uint64_t*)realloc(t->key, sizeof(uint64_t) * (size_t)cap);
    t->weight = (double*)realloc(t->weight, sizeof(double) * (size_t)cap);
    t->desc = (uint32_t*)realloc(t->desc, sizeof(uint32_t) * (size_t)cap * t->d32);
    if (!t->parent || !t->first || !t->nchild || !t->key || !t->weight || !t->desc) {
      t->failed = 1;
      return -1;
    }
    t->cap = cap;
  }
  const int id = t->n++;
  t->parent[id] = parent;
  t->first[id] = 0;
  t->nchild[id] = 0;
  t->key[id] = 0;
  t->weight[id] = 0.0;
  memcpy(t->desc + (size_t)id * t->d32, d, sizeof(uint32_t) * t->d32);
  return id;
}

static void hkmeans_step(Tree* t, const uint32_t* X, int parent, const int* idx, int m, int level)
{
  if (m == 0 || t->failed) return;
  const int k = t->k, W = t->d32;
  uint32_t* clusters = (uint32_t*)calloc((size_t)k * W, sizeof(uint32_t));
  int* assoc = (int*)malloc(sizeof(int) * (size_t)m);
  int* last = (int*)malloc(sizeof(int) * (size_t)m);
  int* gsize = (int*)calloc((size_t)k, sizeof(int));
  if (!clusters || !assoc || !last || !gsize) {
    t->failed = 1;
    return;
  }
  int nc = 0;
  if (m <= k) {
    for (int i = 0; i < m; ++i) {
      memcpy(clusters + (size_t)i * W, X + (size_t)idx[i] * W, sizeof(uint32_t) * W);
      assoc[i] = i;
      gsize[i] = 1;
    }
    nc = m;
  } else {
    uint64_t s = t->key[parent];
    /* initiateClustersKMpp */
    double* min_dists = (double*)malloc(sizeof(double) * (size_t)m);
    if (!min_dists) {
      t->failed = 1;
      return;
    }
    int ifeature = (int)dfk_bow_draw_index(&s, m);
    memcpy(clusters, X + (size_t)idx[ifeature] * W, sizeof(uint32_t) * W);
    nc = 1;
    for (int i = 0; i < m; ++i) min_dists[i] = (double)dfk_bow_distance(X + (size_t)idx[i] * W, clusters, W);
    while (nc < k) {
      for (int i = 0; i < m; ++i)
        if (min_dists[i] > 0) {
          const double d = (double)dfk_bow_distance(X + (size_t)idx[i] * W, clusters + (size_t)(nc - 1) * W, W);
          if (d < min_dists[i]) min_dists[i] = d;
        }
      double dist_sum = 0.0;
      for (int i = 0; i < m; ++i) dist_sum += min_dists[i];
      if (!(dist_sum > 0)) break;
      const double cut = dfk_bow_draw_cut(&s, (int64_t)dist_sum);
      double up = 0;
      int i = 0;
      for (; i < m; ++i) {
        up += min_dists[i];
        if (up >= cut) break;
      }
      ifeature = i == m ? m - 1 : i;
      memcpy(clusters + (size_t)nc * W, X + (size_t)idx[ifeature] * W, sizeof(uint32_t) * W);
      ++nc;
    }
    free(min_dists);
    /* the rounds */
    int* counts = (int*)malloc(sizeof(int) * (size_t)k * W * 32);
    if (!counts) {
      t->failed = 1;
      return;
    }
    int rounds = 0, first_time = 1;
    for (;;) {
      if (!first_time) {
        /* FBrisk::meanValue of each group */
        memset(counts, 0, sizeof(int) * (size_t)k * W * 32);
        for (int j = 0; j < m; ++j) {
          const uint32_t* x = X + (size_t)idx[j] * W;
          int* cc = counts + (size_t)assoc[j] * W * 32;
          for (int b = 0; b < W * 32; ++b) cc[b] += (x[b / 32] >> (b % 32)) & 1u;
        }
        for (int c = 0; c < nc; ++c) {
          uint32_t* mean = clusters + (size_t)c * W;
          for (int b = 0; b < W * 32; ++b) {
            if (b % 32 == 0) mean[b / 32] = 0;
            if (counts[(size_t)c * W * 32 + b] > gsize[c] / 2) mean[b / 32] |= 1u << (b % 32);
          }
        }
        memcpy(last, assoc, sizeof(int) * (size_t)m);
      }
      for (int c = 0; c < nc; ++c) gsize[c] = 0;
      for (int j = 0; j < m; ++j) {
        const uint32_t* x = X + (size_t)idx[j] * W;
        int best = 0, bd = dfk_bow_distance(x, clusters, W);
        for (int c = 1; c < nc; ++c) {
          const int d = dfk_bow_distance(x, clusters + (size_t)c * W, W);
          if (d < bd) {
            bd = d;
            best = c;
          }
        }
        assoc[j] = best;
        gsize[best]++;
      }
      ++rounds;
      if (first_time) {
        first_time = 0;
        continue;
      }
      int same = 1;
      for (int j = 0; j < m && same; ++j) same = assoc[j] == last[j];
      if (same) break;
      if (rounds == DFK_BOW_TRAIN_MAX_ROUNDS) {
        t->stats[3]++;
        break;
      }
    }
    free(counts);
    if (rounds > t->stats[2]) t->stats[2] = rounds;
    if (rounds > t->stats[4 + level]) t->stats[4 + level] = rounds;
    for (int c = 0; c < nc; ++c) t->stats[4] += gsize[c] == 0;
  }
  /* the children, one block of ids in cluster order */
  const int first = t->n;
  for (int c = 0; c < nc; ++c) {
    const int id = tree_add(t, parent, clusters + (size_t)c * W);
    if (id < 0) return;
    t->key[id] = dfk_bow_child_key(t->key[parent], c);
  }
  t->first[parent] = first;
  t->nchild[parent] = nc;
  if (level < t->L) {
    int* group = (int*)malloc(sizeof(int) * (size_t)m);
    if (!group) {
      t->failed = 1;
      return;
    }
    for (int c = 0; c < nc; ++c) {
      int g = 0;
      for (int j = 0; j < m; ++j)
        if (assoc[j] == c) group[g++] = idx[j];
      if (g > 1) hkmeans_step(t, X, first + c, group, g, level + 1);
    }
    free(group);
  }
  free(clusters);
  free(assoc);
  free(last);
  free(gsize);
}

void* dfkb_train(const uint8_t* desc, int64_t n, int bytes, const int64_t* offsets, int n_img, int k, int L,
                 uint64_t seed)
{
  Tree* t = (Tree*)calloc(1, sizeof(Tree));
  if (!t) return NULL;
  t->k = k;
  t->L = L;
  t->bytes = bytes;
  t->d32 = bytes / 4;
  const uint32_t* X = (const uint32_t*)desc;
  uint32_t zero[16] = {0};
  tree_add(t, -1, zero);
  t->key[0] = seed;
  int* idx = (int*)malloc(sizeof(int) * (size_t)n);
  if (!idx) return NULL;
  for (int64_t i = 0; i < n; ++i) idx[i] = (int)i;
  hkmeans_step(t, X, 0, idx, (int)n, 1);
  free(idx);
  if (t->failed) return NULL;
  /* createWords: leaves in ascending id; setNodeWeights: N_i per word, one per image */
  int* word = (int*)malloc(sizeof(int) * (size_t)t->n);
  int nw = 0;
  for (int id = 1; id < t->n; ++id) word[id] = t->nchild[id] == 0 ? nw++ : -1;
  int* ni = (int*)calloc((size_t)nw + 1, sizeof(int));
  int* seen = (int*)malloc(sizeof(int) * ((size_t)nw + 1));
  for (int j = 0; j < nw; ++j) seen[j] = -1;
  for (int img = 0; img < n_img; ++img)
    for (int64_t f = offsets[img]; f < offsets[img + 1]; ++f) {
      const uint32_t* x = X + (size_t)f * t->d32;
      int id = 0;
      do {
        int best = t->first[id], bd = dfk_bow_distance(x, t->desc + (size_t)best * t->d32, t->d32);
        for (int c = 1; c < t->nchild[id]; ++c) {
          const int d = dfk_bow_distance(x, t->desc + (size_t)(t->first[id] + c) * t->d32, t->d32);
          if (d < bd) {
            bd = d;
            best = t->first[id] + c;
          }
        }
        id = best;
      } while (t->nchild[id] > 0);
      if (seen[word[id]] != img) {
        seen[word[id]] = img;
        ni[word[id]]++;
      }
    }
  for (int id = 1; id < t->n; ++id)
    if (word[id] >= 0 && ni[word[id]] > 0) t->weight[id] = log((double)n_img / (double)ni[word[id]]);
  free(word);
  free(ni);
  free(seen);
  t->stats[0] = t->n - 1;
  t->stats[1] = nw;
  return t;
}

/* the trained tree by id 1..n-1: parent, weight, descriptor; stats [5 + 16] */
int dfkb_train_nodes(const void* p) { return ((const Tree*)p)->n - 1; }

void dfkb_train_get(const void* p, int32_t* parent, double* weight, uint8_t* desc, int32_t* stats)
{
  const Tree* t = (const Tree*)p;
  for (int id = 1; id < t->n; ++id) {
    parent[id - 1] = t->parent[id];
    weight[id - 1] = t->weight[id];
    memcpy(desc + (size_t)(id - 1) * t->bytes, t->desc + (size_t)id * t->d32, (size_t)t->bytes);
  }
  memcpy(stats, t->stats, sizeof(t->stats));
}

void dfkb_train_free(void* p)
{
  Tree* t = (Tree*)p;
  if (!t) return;
  free(t->parent);
  free(t->first);
  free(t->nchild);
  free(t->key);
  free(t->weight);
  free(t->desc);
  free(t);
}
