// dfk_api_bow.cu -- C ABI of libdfk.so (see include/dfk.h), DBoW2 retrieval: the vocabulary, the bag-of-words
// transform, the keyframe database, its query and the score.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "dfk.h"
#include "dfk_host.h"
#include "dfk_internal.h"

using namespace dfk;

struct DfkBowVocabulary {
  int device = 0;
  int descriptor_bytes = 0;
  int num_words = 0;
  DeviceBuf<unsigned char> mem;  // [desc rows x D | child int2 x rows | word int32 x rows | word weights fp64 x W]
  BowVocDev dev{};
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

}  // namespace

extern "C" {

DfkStatus dfk_bow_vocabulary_create(DfkHandle h, const DfkBowVocabularyDesc* d, DfkBowVocabulary** out)
{
  return guarded(h, [&] {
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
    DfkBowVocabulary* v = new DfkBowVocabulary;
    v->device = h->device;
    v->descriptor_bytes = D;
    v->num_words = W;
    DeviceGuard guard(h->device);
    cudaError_t e = v->mem.ensure(s.bytes);
    if (e == cudaSuccess) e = cudaMemcpy(v->mem.ptr, s.host(), s.bytes, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
      delete v;
      return cuda_fail(h, e, "[BowVocabulary] upload failed");
    }
    unsigned char* p = v->mem.ptr;
    v->dev = BowVocDev{desc_at.at(p), child_at.at(p), word_at.at(p), ww_at.at(p), D / 16};
    *out = v;
    return DFK_OK;
  });
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

}  // extern "C"
