// dfk_api_bow.cu -- C ABI of libdfk.so (see include/dfk.h), DBoW2 retrieval: the vocabulary, the bag-of-words
// transform, the keyframe database, its query and the score.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <memory>
#include <string>
#include <vector>

#include "dfk.h"
#include "dfk_bow_model.h"
#include "dfk_host.h"
#include "dfk_internal.h"

using namespace dfk;

struct DfkBowVocabulary {
  int device = 0;
  int k = 0, L = 0;
  int descriptor_bytes = 0;
  int num_words = 0;
  DeviceBuf<unsigned char> mem;  // [desc rows x D | child int2 x rows | word int32 x rows | word weights fp64 x W]
  BowVocDev dev{};
  // for dfk_bow_vocabulary_export: where mem's parts lie (the tree is read back from the device on export), and per
  // row the id and weight the node was listed with
  Part<uint4> desc_at{};
  Part<int2> child_at{};
  Part<int32_t> word_at{};
  std::vector<int32_t> ids;
  std::vector<double> weights;
};

struct DfkBowDatabase {
  int device = 0;
  int32_t size = 0;
  long long used = 0;             // storage rows reserved by the entries
  DeviceBuf<int32_t> words;       // storage, grow-only, kept across growth
  DeviceBuf<double> values;
  DeviceBuf<long long> offsets;   // per entry
  DeviceBuf<int32_t> counts;
};

namespace {

bool aligned(const void* p, size_t a) { return ((uintptr_t)p % a) == 0; }

// grows b to hold `need` elements keeping its first `used` (copied on the stream; the old memory's cudaFree waits for
// the copy)
template <typename T>
cudaError_t grow_keep(DeviceBuf<T>& b, size_t need, size_t used, cudaStream_t s)
{
  if (b.cap >= need) return cudaSuccess;
  const size_t n = std::max(need, b.cap * 2);
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, n * sizeof(T));
  if (e != cudaSuccess) return e;
  if (used) e = cudaMemcpyAsync(p, b.ptr, used * sizeof(T), cudaMemcpyDeviceToDevice, s);
  if (e != cudaSuccess) {
    cudaFree(p);
    return e;
  }
  b.release();
  b.ptr = static_cast<T*>(p);
  b.cap = n;
  return cudaSuccess;
}

// a vector the kernels read: the pointers it needs for `capacity` rows
bool vector_ok(const DfkBowVector& v)
{
  return v.capacity >= 0 && v.count && aligned(v.count, 4) && aligned(v.values, 8) && aligned(v.words, 4) &&
         (v.capacity == 0 || (v.words && v.values));
}

BowDbDev db_view(const DfkBowDatabase* db)
{
  return BowDbDev{db->words.ptr, db->values.ptr, db->offsets.ptr, db->counts.ptr, db->size};
}

// dfk_bow_vocabulary_create's body: validates the listed tree and uploads it re-indexed (also the last step of
// dfk_bow_vocabulary_train)
DfkStatus create_vocabulary(DfkHandle h, const DfkBowVocabularyDesc* d, DfkBowVocabulary** out)
{
  const std::string w = "[BowVocabulary] ";
  if (!d || !out) return fail(h, DFK_ERR_INVALID_ARG, w + "null argument");
  *out = nullptr;
  if (d->weighting != DFK_BOW_WEIGHTING_TF_IDF)
    return fail(h, DFK_ERR_UNSUPPORTED, w + "weighting (weightingType) " + std::to_string(d->weighting) +
                                            " is not TF_IDF (0)");
  if (d->scoring != DFK_BOW_SCORING_L1)
    return fail(h, DFK_ERR_UNSUPPORTED, w + "scoring (scoringType) " + std::to_string(d->scoring) +
                                            " is not L1_NORM (0)");
  if (d->k < 1 || d->k > 32) return fail(h, DFK_ERR_INVALID_ARG, w + "k not in [1, 32]");
  if (d->L < 1 || d->L > DFK_BOW_MAX_DEPTH) return fail(h, DFK_ERR_INVALID_ARG, w + "L not in [1, DFK_BOW_MAX_DEPTH]");
  const int D = d->descriptor_bytes;
  if (D != 32 && D != 48 && D != 64) return fail(h, DFK_ERR_INVALID_ARG, w + "descriptor_bytes not 32, 48 or 64");
  const int N = d->num_nodes, W = d->num_words;
  if (N < 1 || N > DFK_BOW_MAX_NODES) return fail(h, DFK_ERR_INVALID_ARG, w + "num_nodes not in [1, DFK_BOW_MAX_NODES]");
  if (W < 1 || W > N) return fail(h, DFK_ERR_INVALID_ARG, w + "num_words not in [1, num_nodes]");
  if (!d->node_ids || !d->parent_ids || !d->weights || !d->descriptors || !d->word_ids || !d->word_nodes)
    return fail(h, DFK_ERR_INVALID_ARG, w + "null array");
  // index of each id (1..N) in file order
  std::vector<int> at((size_t)N + 1, -1);
  for (int i = 0; i < N; ++i) {
    const int id = d->node_ids[i];
    const std::string ni = "node " + std::to_string(i);
    if (id < 1 || id > N) return fail(h, DFK_ERR_INVALID_ARG, w + ni + ": nodeId " + std::to_string(id) + " not in [1, N]");
    if (at[(size_t)id] >= 0) return fail(h, DFK_ERR_INVALID_ARG, w + ni + ": nodeId " + std::to_string(id) + " repeated");
    at[(size_t)id] = i;
    if (!std::isfinite(d->weights[i]) || !(d->weights[i] >= 0.0))
      return fail(h, DFK_ERR_INVALID_ARG, w + ni + ": weight not finite and >= 0");
  }
  // children in file order
  std::vector<int> nchild((size_t)N + 1, 0);
  for (int i = 0; i < N; ++i) {
    const int p = d->parent_ids[i];
    if (p < 0 || p > N || (p > 0 && at[(size_t)p] < 0))
      return fail(h, DFK_ERR_INVALID_ARG, w + "node " + std::to_string(i) + ": parentId " + std::to_string(p) +
                                              " does not exist");
    if (p == d->node_ids[i]) return fail(h, DFK_ERR_INVALID_ARG, w + "node " + std::to_string(i) + ": its own parent");
    if (++nchild[(size_t)p] > d->k)
      return fail(h, DFK_ERR_INVALID_ARG, w + "nodeId " + std::to_string(p) + " has more than k children");
  }
  std::vector<int> first((size_t)N + 2, 0);  // CSR of the children by parent id, file order kept
  for (int p = 0; p <= N; ++p) first[(size_t)p + 1] = first[(size_t)p] + nchild[(size_t)p];
  std::vector<int> kids((size_t)N), fill(first.begin(), first.end() - 1);
  for (int i = 0; i < N; ++i) kids[(size_t)fill[(size_t)d->parent_ids[i]]++] = d->node_ids[i];
  // breadth first from the root: row of each id, depth; a node never reached is on a cycle
  std::vector<int> order;  // ids by row (row 0 = the root, id 0)
  order.reserve((size_t)N + 1);
  std::vector<int> depth((size_t)N + 1, -1), row((size_t)N + 1, -1);
  order.push_back(0);
  depth[0] = 0;
  row[0] = 0;
  for (size_t r = 0; r < order.size(); ++r) {
    const int id = order[r];
    for (int c = first[(size_t)id]; c < first[(size_t)id + 1]; ++c) {
      const int k = kids[(size_t)c];
      depth[(size_t)k] = depth[(size_t)id] + 1;
      if (depth[(size_t)k] > d->L)
        return fail(h, DFK_ERR_INVALID_ARG, w + "node " + std::to_string(at[(size_t)k]) + ": depth > L");
      row[(size_t)k] = (int)order.size();
      order.push_back(k);
    }
  }
  if ((int)order.size() != N + 1) {
    for (int i = 0; i < N; ++i)
      if (row[(size_t)d->node_ids[i]] < 0)
        return fail(h, DFK_ERR_INVALID_ARG, w + "node " + std::to_string(i) + ": not reachable from the root (cycle)");
  }
  // words: a permutation of 0..W-1, each on a leaf, every leaf with one
  std::vector<int> word_of((size_t)N + 1, -1);
  std::vector<char> seen((size_t)W, 0);
  for (int j = 0; j < W; ++j) {
    const int wid = d->word_ids[j], nid = d->word_nodes[j];
    const std::string wj = "word " + std::to_string(j);
    if (wid < 0 || wid >= W) return fail(h, DFK_ERR_INVALID_ARG, w + wj + ": wordId not in [0, W)");
    if (seen[(size_t)wid]) return fail(h, DFK_ERR_INVALID_ARG, w + wj + ": wordId repeated");
    seen[(size_t)wid] = 1;
    if (nid < 1 || nid > N) return fail(h, DFK_ERR_INVALID_ARG, w + wj + ": nodeId does not exist");
    if (nchild[(size_t)nid] > 0) return fail(h, DFK_ERR_INVALID_ARG, w + wj + ": nodeId is not a leaf");
    if (word_of[(size_t)nid] >= 0) return fail(h, DFK_ERR_INVALID_ARG, w + wj + ": the leaf already has a word");
    word_of[(size_t)nid] = wid;
  }
  for (int i = 0; i < N; ++i)
    if (nchild[(size_t)d->node_ids[i]] == 0 && word_of[(size_t)d->node_ids[i]] < 0)
      return fail(h, DFK_ERR_INVALID_ARG, w + "node " + std::to_string(i) + ": a leaf without a word");
  if (nchild[0] == 0) return fail(h, DFK_ERR_INVALID_ARG, w + "the root has no children");
  // the re-indexed tree
  const size_t rows = (size_t)N + 1;
  DfkBowVocabulary* v = new DfkBowVocabulary;
  std::unique_ptr<DfkBowVocabulary> own(v);
  std::vector<unsigned char> host;  // of its own: a tree blob is large, and made once per vocabulary
  Staging s(host);
  const Part<uint4> desc_at = s.add<uint4>(rows * D / 16);
  const Part<int2> child_at = s.add<int2>(rows);
  const Part<int32_t> word_at = s.add<int32_t>(rows);
  const Part<double> ww_at = s.add<double>(W);
  for (size_t r = 0; r < rows; ++r) {
    const int id = order[r];
    if (id > 0) memcpy(desc_at.at(s.host()) + r * (D / 16), d->descriptors + (size_t)at[(size_t)id] * D, (size_t)D);
    const int nc = nchild[(size_t)id];
    child_at.at(s.host())[r] = make_int2(nc ? row[(size_t)kids[(size_t)first[(size_t)id]]] : 0, nc);
    word_at.at(s.host())[r] = id > 0 ? word_of[(size_t)id] : -1;
  }
  for (int j = 0; j < W; ++j) ww_at.at(s.host())[d->word_ids[j]] = d->weights[at[(size_t)d->word_nodes[j]]];
  v->device = h->device;
  v->k = d->k;
  v->L = d->L;
  v->desc_at = desc_at;
  v->child_at = child_at;
  v->word_at = word_at;
  v->ids.assign(order.begin(), order.end());
  v->weights.assign(rows, 0.0);
  for (size_t r = 1; r < rows; ++r) v->weights[r] = d->weights[at[(size_t)order[r]]];
  v->descriptor_bytes = D;
  v->num_words = W;
  DeviceGuard guard(h->device);
  cudaError_t e = v->mem.ensure(s.bytes);
  if (e == cudaSuccess) e = cudaMemcpy(v->mem.ptr, s.host(), s.bytes, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) return cuda_fail(h, e, "[BowVocabulary] upload failed");
  unsigned char* p = v->mem.ptr;
  v->dev = BowVocDev{desc_at.at(p), child_at.at(p), word_at.at(p), ww_at.at(p), D / 16};
  *out = own.release();
  return DFK_OK;
}

}  // namespace

extern "C" {

DfkStatus dfk_bow_vocabulary_create(DfkHandle h, const DfkBowVocabularyDesc* d, DfkBowVocabulary** out)
{
  return guarded(h, [&] { return create_vocabulary(h, d, out); });
}

DfkStatus dfk_bow_vocabulary_destroy(DfkHandle h, DfkBowVocabulary* voc)
{
  return guarded(h, [&] {
    if (voc) {
      DeviceGuard guard(voc->device);
      delete voc;
    }
    return DFK_OK;
  });
}

DfkStatus dfk_bow_transform_batch(DfkHandle h, const DfkBowVocabulary* voc, const DfkFeatureSet* items,
                                  const int32_t* capacities, int n, int32_t* words_dev, double* values_dev,
                                  int32_t* counts_dev, int32_t* feature_words_dev)
{
  return guarded(h, [&] {
    const std::string w = "[BowVocabulary::transform batch] ";
    if (!voc || !items || !capacities || n < 1 || n > 65535)
      return fail(h, DFK_ERR_INVALID_ARG, w + "null argument / number of items not in [1, 65535]");
    if (!words_dev || !values_dev || !counts_dev || !aligned(words_dev, 4) || !aligned(values_dev, 8) ||
        !aligned(counts_dev, 4) || !aligned(feature_words_dev, 4))
      return fail(h, DFK_ERR_INVALID_ARG, w + "null or misaligned output");
    Staging s(h->staging);
    const Part<BowItemDev> items_at = s.add<BowItemDev>(n);
    long long rows = 0;
    int max_num = 0;
    for (int i = 0; i < n; ++i) {
      const DfkFeatureSet& f = items[i];
      const std::string at = " in item " + std::to_string(i);
      if (f.descriptor_bytes != voc->descriptor_bytes)
        return fail(h, DFK_ERR_INVALID_ARG, w + "descriptor_bytes differs from the vocabulary's" + at);
      if (f.num < 0 || f.num > DFK_MATCH_MAX_QUERIES)
        return fail(h, DFK_ERR_INVALID_ARG, w + "num not in [0, DFK_MATCH_MAX_QUERIES]" + at);
      if (f.num > 0 && (!f.descriptors || !aligned(f.descriptors, 16)))
        return fail(h, DFK_ERR_INVALID_ARG, w + "descriptors null or not 16-byte aligned" + at);
      if (capacities[i] < f.num) return fail(h, DFK_ERR_INVALID_ARG, w + "capacity < num" + at);
      items_at.at(s.host())[i] = BowItemDev{f.descriptors, f.num, (int)std::min(rows, (long long)INT32_MAX)};
      rows += capacities[i];
      max_num = std::max(max_num, f.num);
    }
    if (rows > INT32_MAX) return fail(h, DFK_ERR_INVALID_ARG, w + "more than 2^31 - 1 output rows in one call");
    DeviceGuard guard(h->device);
    int32_t* fw = feature_words_dev;
    if (!fw) {
      DFK_CUDA(h, h->bow_words.ensure(std::max<size_t>((size_t)rows, 1)), "[BowVocabulary::transform batch] scratch allocation failed");
      fw = h->bow_words.ptr;
    }
    DFK_TRY(s.upload(h, h->bow_dev, w));
    DFK_CUDA(h, launch_bow_transform(voc->dev, items_at.at(s.dev), n, max_num, fw,
                                     words_dev, values_dev, counts_dev, h->stream),
             "[BowVocabulary::transform batch] kernel launch failed");
    h->launches += max_num > 0 ? 2 : 1;
    return DFK_OK;
  });
}

DfkStatus dfk_bow_database_create(DfkHandle h, const DfkBowVocabulary* voc, DfkBowDatabase** out)
{
  return guarded(h, [&] {
    if (!voc || !out) return fail(h, DFK_ERR_INVALID_ARG, "[BowDatabase] null argument");
    DfkBowDatabase* db = new DfkBowDatabase;
    db->device = h->device;
    *out = db;
    return DFK_OK;
  });
}

DfkStatus dfk_bow_database_destroy(DfkHandle h, DfkBowDatabase* db)
{
  return guarded(h, [&] {
    if (db) {
      DeviceGuard guard(db->device);
      delete db;
    }
    return DFK_OK;
  });
}

DfkStatus dfk_bow_database_clear(DfkHandle h, DfkBowDatabase* db)
{
  return guarded(h, [&] {
    if (!db) return fail(h, DFK_ERR_INVALID_ARG, "[BowDatabase::clear] null database");
    db->size = 0;
    db->used = 0;
    return DFK_OK;
  });
}

DfkStatus dfk_bow_database_size(DfkHandle h, const DfkBowDatabase* db, int32_t* size)
{
  return guarded(h, [&] {
    if (!db || !size) return fail(h, DFK_ERR_INVALID_ARG, "[BowDatabase::size] null argument");
    *size = db->size;
    return DFK_OK;
  });
}

DfkStatus dfk_bow_database_add(DfkHandle h, DfkBowDatabase* db, const DfkBowVector* vectors, int n,
                               int32_t* first_entry)
{
  return guarded(h, [&] {
    const std::string w = "[BowDatabase::add] ";
    if (!db || !vectors || n < 1 || n > 65535)
      return fail(h, DFK_ERR_INVALID_ARG, w + "null argument / number of vectors not in [1, 65535]");
    if ((long long)db->size + n > INT32_MAX) return fail(h, DFK_ERR_INVALID_ARG, w + "more than 2^31 - 1 entries");
    Staging s(h->staging);
    const Part<BowAddDev> adds_at = s.add<BowAddDev>(n);
    long long used = db->used;
    for (int i = 0; i < n; ++i) {
      const DfkBowVector& v = vectors[i];
      if (!vector_ok(v))
        return fail(h, DFK_ERR_INVALID_ARG, w + "vector " + std::to_string(i) +
                                                ": null or misaligned words, values or count, or capacity < 0");
      adds_at.at(s.host())[i] = BowAddDev{v.words, v.values, v.count, v.capacity, db->size + i, used};
      used += v.capacity;
    }
    DeviceGuard guard(h->device);
    const size_t E = (size_t)db->size + n;
    DFK_CUDA(h, grow_keep(db->words, std::max<long long>(used, 1), db->used, h->stream), "[BowDatabase::add] storage allocation failed");
    DFK_CUDA(h, grow_keep(db->values, std::max<long long>(used, 1), db->used, h->stream), "[BowDatabase::add] storage allocation failed");
    DFK_CUDA(h, grow_keep(db->offsets, E, db->size, h->stream), "[BowDatabase::add] storage allocation failed");
    DFK_CUDA(h, grow_keep(db->counts, E, db->size, h->stream), "[BowDatabase::add] storage allocation failed");
    DFK_TRY(s.upload(h, h->bow_dev, w));
    DFK_CUDA(h, launch_bow_add(adds_at.at(s.dev), n, db->words.ptr, db->values.ptr, db->offsets.ptr, db->counts.ptr,
                               h->stream),
             "[BowDatabase::add] kernel launch failed");
    h->launches += 1;
    if (first_entry) *first_entry = db->size;
    db->size += n;
    db->used = used;
    return DFK_OK;
  });
}

DfkStatus dfk_bow_database_query_batch(DfkHandle h, const DfkBowDatabase* db, const DfkBowQuery* queries, int n,
                                       int32_t* ids_dev, double* scores_dev, int32_t* counts_dev)
{
  return guarded(h, [&] {
    const std::string w = "[BowDatabase::query batch] ";
    if (!db || !queries || n < 1 || n > 65535)
      return fail(h, DFK_ERR_INVALID_ARG, w + "null argument / number of queries not in [1, 65535]");
    if (!ids_dev || !scores_dev || !counts_dev || !aligned(ids_dev, 4) || !aligned(scores_dev, 8) ||
        !aligned(counts_dev, 4))
      return fail(h, DFK_ERR_INVALID_ARG, w + "null or misaligned output");
    if ((long long)n * db->size > (1LL << 26))
      return fail(h, DFK_ERR_INVALID_ARG, w + "queries x entries > 2^26");
    // the ranks compare every hit with every other: n x size^2 comparisons, about 0.35 s at the bound on an H100
    if ((double)n * db->size * db->size > (double)(1LL << 36))
      return fail(h, DFK_ERR_INVALID_ARG, w + "queries x entries^2 > 2^36 (the ranking's comparisons)");
    Staging s(h->staging);
    const Part<BowQueryDev> queries_at = s.add<BowQueryDev>(n);
    long long rows = 0;
    int max_cap = 1;
    for (int i = 0; i < n; ++i) {
      const DfkBowQuery& x = queries[i];
      const std::string at = " in query " + std::to_string(i);
      if (!vector_ok(x.vector)) return fail(h, DFK_ERR_INVALID_ARG, w + "null or misaligned vector" + at);
      if (x.vector.capacity > DFK_MATCH_MAX_QUERIES)
        return fail(h, DFK_ERR_INVALID_ARG, w + "vector capacity > DFK_MATCH_MAX_QUERIES" + at);
      if (x.max_results < 1) return fail(h, DFK_ERR_INVALID_ARG, w + "max_results < 1" + at);
      if (x.max_id < -1) return fail(h, DFK_ERR_INVALID_ARG, w + "max_id < -1" + at);
      queries_at.at(s.host())[i] = BowQueryDev{x.vector.words, x.vector.values, x.vector.count, x.vector.capacity,
                                               x.max_results, x.max_id, (int)std::min(rows, (long long)INT32_MAX)};
      rows += x.max_results;
      max_cap = std::max(max_cap, x.vector.capacity);
    }
    if (rows > INT32_MAX) return fail(h, DFK_ERR_INVALID_ARG, w + "more than 2^31 - 1 output rows in one call");
    DeviceGuard guard(h->device);
    if (db->size == 0) {
      DFK_CUDA(h, cudaMemsetAsync(counts_dev, 0, sizeof(int32_t) * (size_t)n, h->stream), "[BowDatabase::query batch] memset failed");
      return DFK_OK;
    }
    const size_t cells = (size_t)n * db->size;
    Layout S;
    const Part<double> sums_at = S.add<double>(cells);
    const Part<unsigned char> hits_at = S.add<unsigned char>(cells);
    DFK_CUDA(h, h->bow_scratch.ensure(S.bytes), "[BowDatabase::query batch] scratch allocation failed");
    DFK_TRY(s.upload(h, h->bow_dev, w));
    DFK_CUDA(h, launch_bow_query(db_view(db), queries_at.at(s.dev), n, max_cap, sums_at.at(h->bow_scratch.ptr),
                                 hits_at.at(h->bow_scratch.ptr), ids_dev, scores_dev, counts_dev, h->stream),
             "[BowDatabase::query batch] kernel launch failed");
    h->launches += 2;
    return DFK_OK;
  });
}

DfkStatus dfk_bow_score_batch(DfkHandle h, const DfkBowDatabase* db, const DfkBowScoreItem* items, int n,
                              double* scores_dev)
{
  return guarded(h, [&] {
    const std::string w = "[BowVocabulary::score batch] ";
    if (!db || !items || n < 1 || n > 65535)
      return fail(h, DFK_ERR_INVALID_ARG, w + "null argument / number of items not in [1, 65535]");
    if (!scores_dev || !aligned(scores_dev, 8)) return fail(h, DFK_ERR_INVALID_ARG, w + "null or misaligned output");
    Staging s(h->staging);
    const Part<BowScoreDev> descs = s.add<BowScoreDev>(n);
    for (int i = 0; i < n; ++i) {
      const DfkBowScoreItem& x = items[i];
      const std::string at = " in item " + std::to_string(i);
      if (x.entry < 0 || x.entry >= db->size) return fail(h, DFK_ERR_INVALID_ARG, w + "entry not in [0, size)" + at);
      if (!vector_ok(x.vector)) return fail(h, DFK_ERR_INVALID_ARG, w + "null or misaligned vector" + at);
      descs.at(s.host())[i] = BowScoreDev{x.vector.words, x.vector.values, x.vector.count, x.vector.capacity, x.entry};
    }
    DeviceGuard guard(h->device);
    DFK_TRY(s.upload(h, h->bow_dev, w));
    DFK_CUDA(h, launch_bow_score(db_view(db), descs.at(s.dev), n, scores_dev, h->stream),
             "[BowVocabulary::score batch] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}


DfkStatus dfk_bow_vocabulary_train(DfkHandle h, const DfkBowTrainDesc* d, DfkBowTrainStats* stats,
                                   DfkBowVocabulary** out)
{
  return guarded(h, [&] {
    const std::string w = "[BowVocabulary::train] ";
    if (!d || !out) return fail(h, DFK_ERR_INVALID_ARG, w + "null argument");
    *out = nullptr;
    if (d->k < 2 || d->k > 32) return fail(h, DFK_ERR_INVALID_ARG, w + "k not in [2, 32]");
    if (d->L < 1 || d->L > DFK_BOW_MAX_DEPTH) return fail(h, DFK_ERR_INVALID_ARG, w + "L not in [1, DFK_BOW_MAX_DEPTH]");
    const int D = d->descriptor_bytes;
    if (D != 32 && D != 48 && D != 64) return fail(h, DFK_ERR_INVALID_ARG, w + "descriptor_bytes not 32, 48 or 64");
    if (d->num_descriptors < 1 || d->num_descriptors > DFK_BOW_TRAIN_MAX_DESCRIPTORS)
      return fail(h, DFK_ERR_INVALID_ARG, w + "num_descriptors not in [1, DFK_BOW_TRAIN_MAX_DESCRIPTORS]");
    if (d->num_images < 1) return fail(h, DFK_ERR_INVALID_ARG, w + "num_images < 1");
    if (!d->descriptors_dev || !aligned(d->descriptors_dev, 16))
      return fail(h, DFK_ERR_INVALID_ARG, w + "descriptors_dev null or not 16-byte aligned");
    if (!d->image_offsets) return fail(h, DFK_ERR_INVALID_ARG, w + "image_offsets null");
    const int N = (int)d->num_descriptors, n_img = d->num_images, k = d->k, L = d->L, Q = D / 16;
    const int64_t* off = d->image_offsets;
    if (off[0] != 0) return fail(h, DFK_ERR_INVALID_ARG, w + "image_offsets[0] is not 0");
    for (int j = 0; j < n_img; ++j) {
      if (off[j + 1] < off[j])
        return fail(h, DFK_ERR_INVALID_ARG, w + "image_offsets decrease at image " + std::to_string(j));
      if (off[j + 1] - off[j] > DFK_MATCH_MAX_QUERIES)
        return fail(h, DFK_ERR_INVALID_ARG, w + "image " + std::to_string(j) + ": more than DFK_MATCH_MAX_QUERIES descriptors");
    }
    if (off[n_img] != N) return fail(h, DFK_ERR_INVALID_ARG, w + "image_offsets[num_images] is not num_descriptors");

    DeviceGuard guard(h->device);
    cudaStream_t st = h->stream;
    // the tree's rows, breadth first (each node's children consecutive; row 0 the root): at most 1 + the sum over the
    // levels of min(k^l, N)
    double bound = 1.0, kl = 1.0;
    for (int l = 1; l <= L; ++l) {
      kl *= k;
      bound += std::min(kl, (double)N);
    }
    const size_t row_cap = (size_t)std::min(bound, (double)DFK_BOW_MAX_NODES + 1.0);
    DeviceBuf<uint4> tree, work[2], level_centres;
    DeviceBuf<int> level_ints, row_first_dev;
    DeviceBuf<unsigned char> large_mem;
    DeviceBuf<int> min_dist;
    DeviceBuf<unsigned char> assign;
    DFK_CUDA(h, tree.ensure(row_cap * Q), "[BowVocabulary::train] allocation failed");
    DFK_CUDA(h, cudaMemsetAsync(tree.ptr, 0, sizeof(uint4) * Q, st), "[BowVocabulary::train] memset failed");
    DFK_CUDA(h, work[0].ensure((size_t)N * Q), "[BowVocabulary::train] allocation failed");
    if (L > 1) DFK_CUDA(h, work[1].ensure((size_t)N * Q), "[BowVocabulary::train] allocation failed");
    if (N > kBowTrainSmallMax) {
      DFK_CUDA(h, min_dist.ensure(N), "[BowVocabulary::train] allocation failed");
      DFK_CUDA(h, assign.ensure(N), "[BowVocabulary::train] allocation failed");
    }
    DfkBowTrainStats sts{};
    std::vector<BowTrainNode> nodes{BowTrainNode{0, N, (unsigned long long)d->seed}};
    std::vector<int> node_row{0};
    std::vector<int2> child(1, make_int2(0, 0));  // per row: (first child row, children)
    const uint4* in = reinterpret_cast<const uint4*>(d->descriptors_dev);
    int outb = 0;
    std::vector<int> ints;
    for (int level = 1; level <= L && !nodes.empty(); ++level) {
      const int G = (int)nodes.size();
      // small nodes in two launches by size, each sized for its own largest node, so that a few nodes near
      // kBowTrainSmallMax do not set the shared memory (and the CTAs per SM) of the many small ones
      std::vector<int> small, large, chunk_first{0};
      std::vector<int2> chunk;
      int max_m[2] = {0, 0}, n_tiny = 0;
      for (int pass = 0; pass < 2; ++pass)
        for (int g = 0; g < G; ++g) {
          const int m = nodes[(size_t)g].m;
          if (m <= kBowTrainSmallMax && (m <= kBowTrainSmallSplit) == (pass == 0)) {
            small.push_back(g);
            max_m[pass] = std::max(max_m[pass], m);
            n_tiny += pass == 0;
          }
        }
      for (int g = 0; g < G; ++g) {
        const int m = nodes[(size_t)g].m;
        if (m > kBowTrainSmallMax) {
          for (int c = 0; c < m; c += kBowTrainChunk) chunk.push_back(make_int2((int)large.size(), c));
          large.push_back(g);
          chunk_first.push_back((int)chunk.size());
        }
      }
      const int ns = (int)small.size(), nl = (int)large.size(), nch = (int)chunk.size();
      Staging s(h->staging);
      const Part<BowTrainNode> nodes_at = s.add<BowTrainNode>(G);
      const Part<int> small_at = s.add<int>(ns);
      const Part<int> large_at = s.add<int>(nl);
      const Part<int2> chunk_at = s.add<int2>(nch);
      const Part<int> chunk_first_at = s.add<int>(nl + 1);
      std::copy(nodes.begin(), nodes.end(), nodes_at.at(s.host()));
      std::copy(small.begin(), small.end(), small_at.at(s.host()));
      std::copy(large.begin(), large.end(), large_at.at(s.host()));
      std::copy(chunk.begin(), chunk.end(), chunk_at.at(s.host()));
      std::copy(chunk_first.begin(), chunk_first.end(), chunk_first_at.at(s.host()));
      DFK_TRY(s.upload(h, h->bow_dev, w));
      // per node of the level: nc | rounds | capped | sizes [G, k], and the centres
      const size_t n_ints = (size_t)G * (3 + k);
      DFK_CUDA(h, level_ints.ensure(n_ints), "[BowVocabulary::train] allocation failed");
      DFK_CUDA(h, level_centres.ensure((size_t)G * k * Q), "[BowVocabulary::train] allocation failed");
      int* li = level_ints.ptr;
      const BowTrainLevel lv{nodes_at.at(s.dev), in, work[outb].ptr, li, li + G, li + 2 * G, li + 3 * G,
                             level_centres.ptr, k, Q};
      for (int pass = 0; pass < 2; ++pass) {
        const int first = pass == 0 ? 0 : n_tiny, n = pass == 0 ? n_tiny : ns - n_tiny;
        if (!n) continue;
        DFK_CUDA(h, launch_bow_train_small(lv, small_at.at(s.dev) + first, n, max_m[pass], st),
                 "[BowVocabulary::train] kernel launch failed");
        h->launches += 1;
      }
      if (nl) {
        Layout S;
        const Part<unsigned long long> rng_at = S.add<unsigned long long>(nl);
        const Part<int> seeding_at = S.add<int>(nl), active_at = S.add<int>(nl), changed_at = S.add<int>(nl);
        const Part<int> cut_chunk_at = S.add<int>(nl);
        const Part<long long> cut_rem_at = S.add<long long>(nl), chunk_sum_at = S.add<long long>(nch);
        const Part<int> counts_at = S.add<int>((size_t)nch * k), base_at = S.add<int>((size_t)nch * k);
        const Part<int> members_at = S.add<int>((size_t)nl * k), bits_at = S.add<int>((size_t)nl * k * D * 8);
        DFK_CUDA(h, large_mem.ensure(S.bytes), "[BowVocabulary::train] allocation failed");
        unsigned char* p = large_mem.ptr;
        const BowTrainLarge lg{large_at.at(s.dev), chunk_at.at(s.dev), chunk_first_at.at(s.dev), rng_at.at(p),
                               seeding_at.at(p), active_at.at(p), changed_at.at(p), cut_chunk_at.at(p),
                               cut_rem_at.at(p), chunk_sum_at.at(p), counts_at.at(p), base_at.at(p),
                               members_at.at(p), bits_at.at(p), min_dist.ptr, assign.ptr};
        // the counts start at zero; each update clears them for the next round
        DFK_CUDA(h, cudaMemsetAsync(members_at.at(p), 0, S.bytes - members_at.off, st),
                 "[BowVocabulary::train] memset failed");
        DFK_CUDA(h, launch_bow_train_seed(lv, lg, nl, nch, st), "[BowVocabulary::train] kernel launch failed");
        h->launches += 1 + 3 * (k - 1);
        // rounds in batches; a node that has stopped skips the rest of its batch, so one read-back per batch suffices
        std::vector<int> active((size_t)nl);
        for (int done = 0; done < DFK_BOW_TRAIN_MAX_ROUNDS;) {
          const int batch = std::min(done < 8 ? 4 : 16, DFK_BOW_TRAIN_MAX_ROUNDS - done);
          DFK_CUDA(h, launch_bow_train_rounds(lv, lg, nl, nch, batch, st), "[BowVocabulary::train] kernel launch failed");
          h->launches += 2 * batch;
          done += batch;
          DFK_TRY(download(h, active.data(), active_at.at(p), sizeof(int) * nl, "[BowVocabulary::train] copy failed",
                           "[BowVocabulary::train] kernel failed"));
          if (std::find(active.begin(), active.end(), 1) == active.end()) break;
        }
        DFK_CUDA(h, launch_bow_train_partition(lv, lg, nl, nch, st), "[BowVocabulary::train] kernel launch failed");
        h->launches += 2;
      }
      ints.resize(n_ints);
      DFK_TRY(download(h, ints.data(), li, sizeof(int) * n_ints, "[BowVocabulary::train] copy failed",
                       "[BowVocabulary::train] kernel failed"));
      const int* nc = ints.data();
      const int* rounds = nc + G;
      const int* capped = nc + 2 * G;
      const int* sizes = nc + 3 * G;
      std::vector<BowTrainNode> next;
      std::vector<int> next_row, row_first((size_t)G);
      for (int g = 0; g < G; ++g) {
        const BowTrainNode& nd = nodes[(size_t)g];
        const int rows = (int)child.size();
        row_first[(size_t)g] = rows;
        if ((size_t)rows + nc[g] > (size_t)DFK_BOW_MAX_NODES + 1)
          return fail(h, DFK_ERR_INVALID_ARG, w + "the tree has more than DFK_BOW_MAX_NODES nodes");
        child[(size_t)node_row[(size_t)g]] = make_int2(rows, nc[g]);
        sts.max_rounds = std::max(sts.max_rounds, rounds[g]);
        sts.level_max_rounds[level - 1] = std::max(sts.level_max_rounds[level - 1], rounds[g]);
        sts.capped_nodes += capped[g];
        int begin = nd.begin;
        for (int c = 0; c < nc[g]; ++c) {
          const int sz = sizes[(size_t)g * k + c];
          child.push_back(make_int2(0, 0));
          if (sz == 0) ++sts.empty_clusters;
          if (level < L && sz > 1) {
            next.push_back(BowTrainNode{begin, sz, (unsigned long long)dfk_bow_child_key(nd.key, c)});
            next_row.push_back(rows + c);
          }
          begin += sz;
        }
      }
      DFK_CUDA(h, row_first_dev.ensure(G), "[BowVocabulary::train] allocation failed");
      DFK_CUDA(h, cudaMemcpyAsync(row_first_dev.ptr, row_first.data(), sizeof(int) * G, cudaMemcpyHostToDevice, st),
               "[BowVocabulary::train] upload failed");
      DFK_CUDA(h, launch_bow_train_place(lv, G, row_first_dev.ptr, tree.ptr, st),
               "[BowVocabulary::train] kernel launch failed");
      h->launches += 1;
      nodes.swap(next);
      node_row.swap(next_row);
      in = work[outb].ptr;
      outb ^= 1;
    }
    const int rows = (int)child.size();
    // words: the leaves, numbered in row order for the idf pass
    std::vector<int> word_row((size_t)rows, -1);
    int W = 0;
    for (int r = 1; r < rows; ++r)
      if (child[(size_t)r].y == 0) word_row[(size_t)r] = W++;
    // N_i: the transform of every image with every word weighing 1 lists each image's words once
    {
      Staging s(h->staging);
      const Part<int2> child_at = s.add<int2>(rows);
      const Part<int32_t> word_at = s.add<int32_t>(rows);
      const Part<double> ww_at = s.add<double>(W);
      const Part<BowItemDev> items_at = s.add<BowItemDev>(n_img);
      std::copy(child.begin(), child.end(), child_at.at(s.host()));
      std::copy(word_row.begin(), word_row.end(), word_at.at(s.host()));
      std::fill(ww_at.at(s.host()), ww_at.at(s.host()) + W, 1.0);
      for (int j = 0; j < n_img; ++j)
        items_at.at(s.host())[j] = BowItemDev{d->descriptors_dev + (size_t)off[j] * D, (int)(off[j + 1] - off[j]),
                                              (int)off[j]};
      DFK_TRY(s.upload(h, h->bow_dev, w));
      Layout S;
      const Part<int32_t> fw_at = S.add<int32_t>(N), words_at = S.add<int32_t>(N);
      const Part<double> values_at = S.add<double>(N);
      const Part<int32_t> counts_at = S.add<int32_t>(n_img), images_at = S.add<int32_t>(W);
      DeviceBuf<unsigned char> idf;
      DFK_CUDA(h, idf.ensure(S.bytes), "[BowVocabulary::train] allocation failed");
      unsigned char* p = idf.ptr;
      DFK_CUDA(h, cudaMemsetAsync(images_at.at(p), 0, sizeof(int32_t) * W, st), "[BowVocabulary::train] memset failed");
      const BowVocDev vd{tree.ptr, child_at.at(s.dev), word_at.at(s.dev), ww_at.at(s.dev), Q};
      for (int i0 = 0; i0 < n_img; i0 += 65535) {
        const int n = std::min(65535, n_img - i0);
        int max_num = 0;
        for (int j = i0; j < i0 + n; ++j) max_num = std::max(max_num, (int)(off[j + 1] - off[j]));
        const BowItemDev* items = items_at.at(s.dev) + i0;
        DFK_CUDA(h, launch_bow_transform(vd, items, n, max_num, fw_at.at(p), words_at.at(p), values_at.at(p),
                                         counts_at.at(p) + i0, st),
                 "[BowVocabulary::train] kernel launch failed");
        DFK_CUDA(h, launch_bow_train_count(items, n, words_at.at(p), counts_at.at(p) + i0, images_at.at(p), st),
                 "[BowVocabulary::train] kernel launch failed");
        h->launches += 3;
      }
      ints.resize((size_t)W);
      DFK_TRY(download(h, ints.data(), images_at.at(p), sizeof(int32_t) * W, "[BowVocabulary::train] copy failed",
                       "[BowVocabulary::train] kernel failed"));
    }
    std::vector<uint8_t> desc((size_t)rows * D);
    DFK_TRY(download(h, desc.data(), tree.ptr, desc.size(), "[BowVocabulary::train] copy failed",
                     "[BowVocabulary::train] kernel failed"));
    // DBoW2's ids: visiting a node numbers its children, then visits those that have children, in order
    std::vector<int> id((size_t)rows, 0);
    int next_id = 1;
    std::vector<std::pair<int, int>> stack{{0, 0}};  // (row, next child to visit)
    for (int c = 0; c < child[0].y; ++c) id[(size_t)(child[0].x + c)] = next_id++;
    while (!stack.empty()) {
      auto& top = stack.back();
      const int2 ch = child[(size_t)top.first];
      if (top.second == ch.y) {
        stack.pop_back();
        continue;
      }
      const int r = ch.x + top.second++;
      if (child[(size_t)r].y == 0) continue;
      for (int c = 0; c < child[(size_t)r].y; ++c) id[(size_t)(child[(size_t)r].x + c)] = next_id++;
      stack.push_back({r, 0});
    }
    // the tree in save's order, weights from the counts
    const int n_nodes = rows - 1;
    std::vector<int32_t> node_ids, parent_ids, word_ids((size_t)W), word_nodes;
    std::vector<double> weights;
    std::vector<uint8_t> descriptors;
    node_ids.reserve((size_t)n_nodes);
    parent_ids.reserve((size_t)n_nodes);
    weights.reserve((size_t)n_nodes);
    descriptors.reserve((size_t)n_nodes * D);
    std::vector<int> parents{0};
    while (!parents.empty()) {
      const int pr = parents.back();
      parents.pop_back();
      for (int c = 0; c < child[(size_t)pr].y; ++c) {
        const int r = child[(size_t)pr].x + c;
        node_ids.push_back(id[(size_t)r]);
        parent_ids.push_back(id[(size_t)pr]);
        double wt = 0.0;
        if (child[(size_t)r].y == 0) {
          const int ni = ints[(size_t)word_row[(size_t)r]];
          if (ni > 0) wt = std::log((double)n_img / (double)ni);
        } else {
          parents.push_back(r);
        }
        weights.push_back(wt);
        descriptors.insert(descriptors.end(), desc.begin() + (size_t)r * D, desc.begin() + (size_t)(r + 1) * D);
      }
    }
    std::vector<std::pair<int, int>> leaves;  // (id, row)
    for (int r = 1; r < rows; ++r)
      if (child[(size_t)r].y == 0) leaves.push_back({id[(size_t)r], r});
    std::sort(leaves.begin(), leaves.end());
    for (int j = 0; j < W; ++j) {
      word_ids[(size_t)j] = j;
      word_nodes.push_back(leaves[(size_t)j].first);
    }
    const DfkBowVocabularyDesc vd{k, L, DFK_BOW_WEIGHTING_TF_IDF, DFK_BOW_SCORING_L1, D, n_nodes, node_ids.data(),
                                  parent_ids.data(), weights.data(), descriptors.data(), W, word_ids.data(),
                                  word_nodes.data()};
    DFK_TRY(create_vocabulary(h, &vd, out));
    sts.num_nodes = n_nodes;
    sts.num_words = W;
    if (stats) *stats = sts;
    return DFK_OK;
  });
}

DfkStatus dfk_bow_vocabulary_export(DfkHandle h, const DfkBowVocabulary* voc, DfkBowVocabularyShape* shape,
                                    int32_t* node_ids, int32_t* parent_ids, double* weights, uint8_t* descriptors,
                                    int32_t* word_ids, int32_t* word_nodes)
{
  return guarded(h, [&] {
    const std::string w = "[BowVocabulary::export] ";
    if (!voc || !shape) return fail(h, DFK_ERR_INVALID_ARG, w + "null argument");
    const int given = !!node_ids + !!parent_ids + !!weights + !!descriptors + !!word_ids + !!word_nodes;
    if (given != 0 && given != 6) return fail(h, DFK_ERR_INVALID_ARG, w + "pass every array or none");
    const int rows = (int)voc->ids.size(), D = voc->descriptor_bytes;
    *shape = DfkBowVocabularyShape{voc->k, voc->L, DFK_BOW_WEIGHTING_TF_IDF, DFK_BOW_SCORING_L1, D, rows - 1,
                                   voc->num_words};
    if (!given) return DFK_OK;
    // the tree's rows [descriptors | children | words], the leading parts of the device blob
    std::vector<unsigned char> tree(voc->word_at.off + sizeof(int32_t) * (size_t)rows);
    DeviceGuard guard(voc->device);
    DFK_CUDA(h, cudaMemcpy(tree.data(), voc->mem.ptr, tree.size(), cudaMemcpyDeviceToHost),
             "[BowVocabulary::export] copy failed");
    unsigned char* base = tree.data();
    const int2* child = voc->child_at.at(base);
    const uint8_t* desc = reinterpret_cast<const uint8_t*>(voc->desc_at.at(base));
    const int32_t* word = voc->word_at.at(base);
    std::vector<int> parents{0};
    int i = 0;
    while (!parents.empty()) {
      const int pr = parents.back();
      parents.pop_back();
      for (int c = 0; c < child[pr].y; ++c, ++i) {
        const int r = child[pr].x + c;
        node_ids[i] = voc->ids[(size_t)r];
        parent_ids[i] = voc->ids[(size_t)pr];
        weights[i] = voc->weights[(size_t)r];
        memcpy(descriptors + (size_t)i * D, desc + (size_t)r * D, (size_t)D);
        if (child[r].y > 0) parents.push_back(r);
      }
    }
    for (int r = 1; r < rows; ++r)
      if (word[r] >= 0) {
        word_ids[word[r]] = word[r];
        word_nodes[word[r]] = voc->ids[(size_t)r];
      }
    return DFK_OK;
  });
}

}  // extern "C"
