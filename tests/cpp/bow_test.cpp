// bow_test.cpp -- the DBoW2 facade (df/dfk_bow.h) against the C calls it wraps.
//   bow_test parse VOC.yml OUT.bin   LoadText only (no GPU): writes the parsed arrays, which the CPU tests compare with
//                                    the Python loader's
//   bow_test VOC.yml                 on the GPU: BowVocabulary::transform of five images (one empty) equals
//                                    dfk_bow_transform_batch bit for bit; BowDatabase add / query / score / size / clear
//                                    equal the dfk_bow_database_* calls on the same vectors
// Build: see tests/cpp/bow.mk.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <random>
#include <vector>

#include "df/dfk_bow.h"

#define EXPECT(c)                                                                       \
  do {                                                                                  \
    if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } \
  } while (0)

template <typename T>
static void put(std::ofstream& f, const std::vector<T>& v)
{
  f.write(reinterpret_cast<const char*>(v.data()), (std::streamsize)(sizeof(T) * v.size()));
}

static int parse(const char* in, const char* out)
{
  std::ifstream f(in);
  const df::BowVocabularyData d = df::BowVocabularyData::LoadText(f);
  std::ofstream o(out, std::ios::binary);
  const std::vector<int32_t> head{d.k, d.L, d.weighting, d.scoring, d.descriptor_bytes, (int32_t)d.node_ids.size(),
                                  (int32_t)d.word_ids.size()};
  put(o, head);
  put(o, d.node_ids);
  put(o, d.parent_ids);
  put(o, d.weights);
  put(o, d.descriptors);
  put(o, d.word_ids);
  put(o, d.word_nodes);
  std::puts("bow_test parse OK");
  return 0;
}

template <typename T>
static std::vector<T> down(const T* p, size_t n)
{
  std::vector<T> v(n);
  if (n) cudaMemcpy(v.data(), p, sizeof(T) * n, cudaMemcpyDeviceToHost);
  return v;
}

static bool same_bits(const std::vector<double>& a, const std::vector<double>& b)
{
  return a.size() == b.size() && (a.empty() || std::memcmp(a.data(), b.data(), sizeof(double) * a.size()) == 0);
}

int main(int argc, char** argv)
{
  if (argc == 4 && std::strcmp(argv[1], "parse") == 0) return parse(argv[2], argv[3]);
  if (argc != 2) {
    std::puts("usage: bow_test VOC.yml | bow_test parse VOC.yml OUT.bin");
    return 2;
  }
  std::ifstream f(argv[1]);
  const df::BowVocabularyData data = df::BowVocabularyData::LoadText(f);
  const int D = data.descriptor_bytes, n = 5;
  const int nums[n] = {300, 0, 1, 500, 77};
  // descriptors near the vocabulary's nodes, so that words repeat
  std::mt19937 rng(7);
  std::vector<DfkFeatureSet> sets;
  std::vector<int32_t> caps;
  std::vector<void*> keep;
  for (int i = 0; i < n; ++i) {
    std::vector<uint8_t> h((size_t)nums[i] * D);
    for (int r = 0; r < nums[i]; ++r) {
      const size_t node = rng() % data.node_ids.size();
      std::memcpy(&h[(size_t)r * D], &data.descriptors[node * D], (size_t)D);
      for (int b = 0; b < 8; ++b) h[(size_t)r * D + rng() % D] ^= (uint8_t)(1u << (rng() % 8));
    }
    void* p = nullptr;
    cudaMalloc(&p, std::max<size_t>(h.size(), 16));
    if (!h.empty()) cudaMemcpy(p, h.data(), h.size(), cudaMemcpyHostToDevice);
    keep.push_back(p);
    sets.push_back(DfkFeatureSet{nullptr, static_cast<uint8_t*>(p), nums[i], D});
    caps.push_back(nums[i]);
  }
  df::BowVocabulary voc(data);
  std::vector<df::BowVector> vecs(n);
  std::vector<df::BowVector*> outs;
  for (auto& v : vecs) outs.push_back(&v);
  voc.transform(sets, outs);
  df::BowVector single;
  voc.transform(sets[3], single);

  // the C calls on a handle and vocabulary of their own
  DfkHandle h = nullptr;
  EXPECT(dfk_create(-1, &h) == DFK_OK);
  const DfkBowVocabularyDesc desc = data.Desc();
  DfkBowVocabulary* cv = nullptr;
  EXPECT(dfk_bow_vocabulary_create(h, &desc, &cv) == DFK_OK);
  int total = 0;
  for (int c : caps) total += c;
  int32_t *words = nullptr, *counts = nullptr;
  double* values = nullptr;
  cudaMalloc(&words, sizeof(int32_t) * total);
  cudaMalloc(&values, sizeof(double) * total);
  cudaMalloc(&counts, sizeof(int32_t) * n);
  EXPECT(dfk_bow_transform_batch(h, cv, sets.data(), caps.data(), n, words, values, counts, nullptr) == DFK_OK);
  EXPECT(dfk_synchronize(h) == DFK_OK);
  const std::vector<int32_t> hc = down(counts, n);
  std::vector<DfkBowVector> cvecs;
  int o = 0;
  for (int i = 0; i < n; ++i) {
    const std::map<int32_t, double> m = vecs[i].Host();
    const std::vector<int32_t> w = down(words + o, (size_t)hc[i]);
    const std::vector<double> v = down(values + o, (size_t)hc[i]);
    EXPECT((int)m.size() == hc[i]);
    std::vector<int32_t> mw;
    std::vector<double> mv;
    for (const auto& kv : m) {
      mw.push_back(kv.first);
      mv.push_back(kv.second);
    }
    EXPECT(mw == w && same_bits(mv, v));
    if (i == 3) {
      const std::map<int32_t, double> s = single.Host();
      EXPECT(s.size() == m.size() && std::equal(s.begin(), s.end(), m.begin(), [](const auto& a, const auto& b) {
               return a.first == b.first && std::memcmp(&a.second, &b.second, sizeof(double)) == 0;
             }));
    }
    cvecs.push_back(DfkBowVector{words + o, values + o, counts + i, caps[i]});
    o += caps[i];
  }
  EXPECT(hc[1] == 0);

  // the database: facade and C calls on the same vectors
  df::BowDatabase db(voc);
  DfkBowDatabase* cdb = nullptr;
  EXPECT(dfk_bow_database_create(h, cv, &cdb) == DFK_OK);
  for (int i = 0; i < n; ++i) EXPECT(db.add(vecs[i]) == (unsigned)i);
  int32_t first = -1;
  EXPECT(dfk_bow_database_add(h, cdb, cvecs.data(), n, &first) == DFK_OK && first == 0);
  EXPECT(db.size() == (unsigned)n);
  int32_t *ids = nullptr, *qc = nullptr;
  double *sc = nullptr, *ss = nullptr;
  cudaMalloc(&ids, sizeof(int32_t) * 8);
  cudaMalloc(&qc, sizeof(int32_t));
  cudaMalloc(&sc, sizeof(double) * 8);
  cudaMalloc(&ss, sizeof(double));
  for (int i = 0; i < n; ++i)
    for (int max_id : {-1, 2}) {
      std::vector<df::BowDatabase::Result> ret;
      db.query(vecs[i], ret, 3, max_id);
      const DfkBowQuery q{cvecs[i], 3, max_id};
      EXPECT(dfk_bow_database_query_batch(h, cdb, &q, 1, ids, sc, qc) == DFK_OK);
      EXPECT(dfk_synchronize(h) == DFK_OK);
      const int c = std::min(down(qc, 1)[0], 3);
      EXPECT((int)ret.size() == c);
      const std::vector<int32_t> hid = down(ids, (size_t)c);
      const std::vector<double> hsc = down(sc, (size_t)c);
      for (int k = 0; k < c; ++k) EXPECT(ret[k].Id == (unsigned)hid[k] && !std::memcmp(&ret[k].Score, &hsc[k], 8));
      if (nums[i] > 0 && max_id == -1) EXPECT(c >= 1 && ret[0].Id == (unsigned)i);  // an entry finds itself first
      for (int e = 0; e < n; ++e) {
        const double a = voc.score(db, e, vecs[i]);
        const DfkBowScoreItem it{e, cvecs[i]};
        EXPECT(dfk_bow_score_batch(h, cdb, &it, 1, ss) == DFK_OK);
        EXPECT(dfk_synchronize(h) == DFK_OK);
        const double b = down(ss, 1)[0];
        EXPECT(!std::memcmp(&a, &b, 8));
      }
    }
  db.clear();
  EXPECT(db.size() == 0);
  std::vector<df::BowDatabase::Result> ret;
  db.query(vecs[0], ret, 3);
  EXPECT(ret.empty());
  // a rejected call throws with the C message
  bool threw = false;
  try {
    db.score(0, vecs[0]);
  } catch (const std::exception& e) {
    threw = std::strstr(e.what(), "entry not in") != nullptr;
  }
  EXPECT(threw);
  dfk_bow_database_destroy(h, cdb);
  dfk_bow_vocabulary_destroy(h, cv);
  for (void* p : {(void*)words, (void*)values, (void*)counts, (void*)ids, (void*)qc, (void*)sc, (void*)ss}) cudaFree(p);
  for (void* p : keep) cudaFree(p);
  dfk_destroy(h);
  std::puts("bow_test OK");
  return 0;
}
