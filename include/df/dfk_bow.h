// dfk_bow.h -- the DBoW2 calls of LoopDetector (core/system/loop_detector.cpp) on top of the dfk_bow_* C calls
// (include/dfk.h, DBoW2 block): TF_IDF weighting, L1_NORM scoring, no direct index.
//   df::BowVocabularyData          the arrays of DBoW2's vocabulary, in file order
//     ::LoadText(std::istream&)    DBoW2's cv::FileStorage text format (uncompressed .yml)
//     .SaveText(std::ostream&)     TemplatedVocabulary::save's text, which LoadText reads back
//   df::BowVocabulary              owns a handle and the device tree
//     (features, D, k, L, seed)    TemplatedVocabulary(k, L, TF_IDF, L1_NORM).create(features), on the device
//     .Export()                    the tree in DBoW2's save order (dfk_bow_vocabulary_export)
//     .transform(features, v)      voc_.transform(features, bow_vec) on DEVICE descriptors
//     .transform(features[], v[])  many images in one call
//   df::BowVector                  a bag-of-words vector on the device (owns its rows); Host() reads it back
//   df::BowDatabase                TemplatedDatabase(voc, false, 0): add, query, clear, size, score
//     .score(entry, v)             voc_.score(the entry's vector, v)
// Results are DBoW2's (Id, Score) pairs, best first.
#ifndef DFK_BOW_H_
#define DFK_BOW_H_

#include <cuda_runtime.h>

#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <istream>
#include <iterator>
#include <map>
#include <ostream>
#include <stdexcept>
#include <string>
#include <vector>

#include "dfk_facade.h"

namespace df
{

struct BowVocabularyData {
  int k = 0, L = 0, weighting = 0, scoring = 0, descriptor_bytes = 0;
  std::vector<int32_t> node_ids, parent_ids;
  std::vector<double> weights;
  std::vector<uint8_t> descriptors;  // [nodes, descriptor_bytes]
  std::vector<int32_t> word_ids, word_nodes;

  // TemplatedVocabulary::save's text.  Weights go through strtod; a line break inside a quoted descriptor, with or
  // without a trailing backslash, reads as the writer meant it.  Throws std::runtime_error on a malformed file.
  static BowVocabularyData LoadText(std::istream& in)
  {
    std::string raw((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
    std::string t;  // escaped line breaks joined
    t.reserve(raw.size());
    for (size_t i = 0; i < raw.size(); ++i) {
      if (raw[i] == '\\' && i + 1 < raw.size() && (raw[i + 1] == '\n' || raw[i + 1] == '\r')) {
        ++i;
        while (i + 1 < raw.size() && std::isspace((unsigned char)raw[i + 1])) ++i;
        continue;
      }
      t += raw[i];
    }
    BowVocabularyData d;
    auto head = [&](const char* key) {
      const std::string k = std::string(key) + ":";
      for (size_t p = t.find(k); p != std::string::npos; p = t.find(k, p + 1)) {
        const bool line_start = p == 0 || t.find_last_not_of(" \t", p - 1) == std::string::npos ||
                                t[t.find_last_not_of(" \t", p - 1)] == '\n';
        if (line_start) return std::atoi(t.c_str() + p + k.size());
      }
      throw std::runtime_error(std::string("[BowVocabulary::LoadText] no ") + key);
    };
    d.k = head("k");
    d.L = head("L");
    d.scoring = head("scoringType");
    d.weighting = head("weightingType");
    // every flow mapping { key: value, ... } is a node or a word
    for (size_t open = t.find('{'); open != std::string::npos; open = t.find('{', open + 1)) {
      size_t close = open + 1;
      bool quoted = false;
      for (; close < t.size() && (quoted || t[close] != '}'); ++close)
        if (t[close] == '"') quoted = !quoted;
      if (close >= t.size()) throw std::runtime_error("[BowVocabulary::LoadText] unterminated mapping");
      std::map<std::string, std::string> kv;
      size_t p = open + 1;
      while (p < close) {
        const size_t colon = t.find(':', p);
        if (colon == std::string::npos || colon > close) break;
        std::string key = t.substr(p, colon - p);
        key.erase(0, key.find_first_not_of(" \t\r\n,"));
        key.erase(key.find_last_not_of(" \t\r\n") + 1);
        size_t v = colon + 1, end;
        while (v < close && std::isspace((unsigned char)t[v])) ++v;
        if (v < close && t[v] == '"') {
          end = t.find('"', v + 1);
          kv[key] = t.substr(v + 1, end - v - 1);
          end = t.find(',', end);
        } else {
          end = t.find(',', v);
          kv[key] = t.substr(v, std::min(end, close) - v);
        }
        if (end == std::string::npos || end > close) break;
        p = end + 1;
      }
      if (kv.count("wordId")) {
        d.word_ids.push_back(std::atoi(kv["wordId"].c_str()));
        d.word_nodes.push_back(std::atoi(kv["nodeId"].c_str()));
      } else if (kv.count("nodeId") && kv.count("descriptor")) {
        d.node_ids.push_back(std::atoi(kv["nodeId"].c_str()));
        d.parent_ids.push_back(std::atoi(kv["parentId"].c_str()));
        d.weights.push_back(std::strtod(kv["weight"].c_str(), nullptr));
        const char* s = kv["descriptor"].c_str();
        char* e = nullptr;
        int n = 0;
        for (long b = std::strtol(s, &e, 10); e != s; b = std::strtol(s, &e, 10), ++n) {
          d.descriptors.push_back(static_cast<uint8_t>(b));
          s = e;
        }
        if (d.descriptor_bytes == 0) d.descriptor_bytes = n;
        if (n != d.descriptor_bytes)
          throw std::runtime_error("[BowVocabulary::LoadText] descriptors of different lengths");
      }
      open = close;
    }
    if (d.node_ids.empty() || d.word_ids.empty())
      throw std::runtime_error("[BowVocabulary::LoadText] no nodes or no words");
    return d;
  }

  // TemplatedVocabulary::save's text in the layout of DBoW2's own files: nodes and words in this object's order, each
  // node on two lines; weights in OpenCV's double format ("%d." when integral, "%.16e" otherwise), so strtod reads
  // back the same double
  void SaveText(std::ostream& out) const
  {
    char buf[64];
    out << "%YAML:1.0\n---\nvocabulary:\n   k: " << k << "\n   L: " << L << "\n   scoringType: " << scoring
        << "\n   weightingType: " << weighting << "\n   nodes:\n";
    for (size_t i = 0; i < node_ids.size(); ++i) {
      const double w = weights[i];
      if (w == (double)(long long)w && w < 9007199254740992.0 && w > -9007199254740992.0)
        std::snprintf(buf, sizeof buf, "%lld.", (long long)w);
      else
        std::snprintf(buf, sizeof buf, "%.16e", w);
      out << "      - { nodeId:" << node_ids[i] << ", parentId:" << parent_ids[i] << ", weight:" << buf
          << ",\n          descriptor:\"";
      for (int b = 0; b < descriptor_bytes; ++b) out << (int)descriptors[i * (size_t)descriptor_bytes + b] << ' ';
      out << "\" }\n";
    }
    out << "   words:\n";
    for (size_t j = 0; j < word_ids.size(); ++j)
      out << "      - { wordId:" << word_ids[j] << ", nodeId:" << word_nodes[j] << " }\n";
  }

  DfkBowVocabularyDesc Desc() const
  {
    return DfkBowVocabularyDesc{k, L, weighting, scoring, descriptor_bytes, (int32_t)node_ids.size(), node_ids.data(),
                                parent_ids.data(), weights.data(), descriptors.data(), (int32_t)word_ids.size(),
                                word_ids.data(), word_nodes.data()};
  }
};

// A bag-of-words vector on the device with rows for `capacity` words (DBoW2::BowVector)
class BowVector
{
public:
  BowVector() = default;
  explicit BowVector(int capacity) { Reserve(capacity); }
  BowVector(const BowVector&) = delete;
  BowVector& operator=(const BowVector&) = delete;
  BowVector(BowVector&& o) noexcept : mem_(o.mem_), cap_(o.cap_) { o.mem_ = nullptr; o.cap_ = 0; }
  BowVector& operator=(BowVector&& o) noexcept
  {
    std::swap(mem_, o.mem_);
    std::swap(cap_, o.cap_);
    return *this;
  }
  ~BowVector() { cudaFree(mem_); }

  // [values fp64 | words int32 | count int32]; keeps nothing
  void Reserve(int capacity)
  {
    if (capacity <= cap_ && mem_) return;
    cudaFree(mem_);
    mem_ = nullptr;
    const size_t bytes = (sizeof(double) + sizeof(int32_t)) * (size_t)capacity + sizeof(int32_t);
    if (cudaMalloc(&mem_, bytes) != cudaSuccess) throw std::runtime_error("[BowVector] cudaMalloc failed");
    cudaMemset(mem_, 0, bytes);
    cap_ = capacity;
  }
  int capacity() const { return cap_; }
  double* values() const { return static_cast<double*>(mem_); }
  int32_t* words() const { return reinterpret_cast<int32_t*>(values() + cap_); }
  int32_t* count() const { return words() + cap_; }
  DfkBowVector view() const { return DfkBowVector{words(), values(), count(), cap_}; }

  // word id -> value, as DBoW2's map (synchronises)
  std::map<int32_t, double> Host() const
  {
    int32_t c = 0;
    cudaMemcpy(&c, count(), sizeof c, cudaMemcpyDeviceToHost);
    std::vector<int32_t> w((size_t)c);
    std::vector<double> v((size_t)c);
    cudaMemcpy(w.data(), words(), sizeof(int32_t) * w.size(), cudaMemcpyDeviceToHost);
    cudaMemcpy(v.data(), values(), sizeof(double) * v.size(), cudaMemcpyDeviceToHost);
    std::map<int32_t, double> m;
    for (size_t i = 0; i < w.size(); ++i) m[w[i]] = v[i];
    return m;
  }

private:
  void* mem_ = nullptr;
  int cap_ = 0;
};

class BowDatabase;

class BowVocabulary
{
public:
  explicit BowVocabulary(const BowVocabularyData& d) : h_(detail::MakeHandle())
  {
    const DfkBowVocabularyDesc desc = d.Desc();
    detail::Check(h_.get(), dfk_bow_vocabulary_create(h_.get(), &desc, &voc_));
  }
  // TemplatedVocabulary(k, L, TF_IDF, L1_NORM).create(features) on the device (dfk_bow_vocabulary_train, with the
  // per-node random streams of include/dfk.h's training block): descriptors_dev DEVICE [N, descriptor_bytes], 16-byte
  // aligned, image j its rows [image_offsets[j], image_offsets[j + 1]).  Ordered after earlier work on the stream;
  // synchronous.
  BowVocabulary(const uint8_t* descriptors_dev, const std::vector<int64_t>& image_offsets, int descriptor_bytes, int k,
                int L, uint64_t seed = 0)
      : h_(detail::MakeHandle())
  {
    Train(descriptors_dev, image_offsets, descriptor_bytes, k, L, seed);
  }
  // the same from host features, one vector of descriptor_bytes-byte rows per image (DBoW2's getFeatures layout)
  BowVocabulary(const std::vector<std::vector<uint8_t>>& features, int descriptor_bytes, int k, int L,
                uint64_t seed = 0)
      : h_(detail::MakeHandle())
  {
    std::vector<int64_t> off{0};
    for (const auto& f : features) {
      if (f.size() % (size_t)descriptor_bytes) throw std::invalid_argument("[BowVocabulary] a partial descriptor");
      off.push_back(off.back() + (int64_t)(f.size() / descriptor_bytes));
    }
    void* dev = nullptr;
    if (cudaMalloc(&dev, std::max<size_t>((size_t)off.back() * descriptor_bytes, 16)) != cudaSuccess)
      throw std::runtime_error("[BowVocabulary] cudaMalloc failed");
    size_t o = 0;
    for (const auto& f : features) {
      cudaMemcpy(static_cast<uint8_t*>(dev) + o, f.data(), f.size(), cudaMemcpyHostToDevice);
      o += f.size();
    }
    try {
      Train(static_cast<const uint8_t*>(dev), off, descriptor_bytes, k, L, seed);
    } catch (...) {
      cudaFree(dev);
      throw;
    }
    cudaFree(dev);
  }
  ~BowVocabulary() { dfk_bow_vocabulary_destroy(h_.get(), voc_); }
  BowVocabulary(const BowVocabulary&) = delete;
  BowVocabulary& operator=(const BowVocabulary&) = delete;

  DfkHandle handle() const { return h_.get(); }
  const DfkBowVocabulary* get() const { return voc_; }
  void SetStream(void* stream) { detail::Check(h_.get(), dfk_set_stream(h_.get(), stream)); }

  // voc_.transform(features, v): the features' DEVICE descriptor rows; v grows to hold one word per feature
  void transform(const DfkFeatureSet& features, BowVector& v) const
  {
    std::vector<BowVector*> out{&v};
    transform(std::vector<DfkFeatureSet>{features}, out);
  }
  // many images in one call; asynchronous on the handle's stream
  void transform(const std::vector<DfkFeatureSet>& features, const std::vector<BowVector*>& out) const
  {
    if (features.size() != out.size()) throw std::invalid_argument("[BowVocabulary::transform] one vector per image");
    std::vector<int32_t> caps;
    int total = 0;
    for (size_t i = 0; i < features.size(); ++i) {
      out[i]->Reserve(std::max(features[i].num, 1));
      caps.push_back(features[i].num);
      total += features[i].num;
    }
    // one call writes back to back rows; each vector then takes its own copy
    BowVector all(std::max(total, 1));
    std::vector<int32_t*> counts(features.size());
    int32_t* cdev = nullptr;
    if (cudaMalloc(&cdev, sizeof(int32_t) * std::max<size_t>(features.size(), 1)) != cudaSuccess)
      throw std::runtime_error("[BowVocabulary::transform] cudaMalloc failed");
    const DfkStatus st = dfk_bow_transform_batch(h_.get(), voc_, features.data(), caps.data(), (int)features.size(),
                                                 all.words(), all.values(), cdev, nullptr);
    if (st != DFK_OK) {
      cudaFree(cdev);
      detail::Check(h_.get(), st);
    }
    cudaStream_t s = static_cast<cudaStream_t>(dfk_get_stream(h_.get()));
    int o = 0;
    for (size_t i = 0; i < features.size(); ++i) {
      cudaMemcpyAsync(out[i]->words(), all.words() + o, sizeof(int32_t) * caps[i], cudaMemcpyDeviceToDevice, s);
      cudaMemcpyAsync(out[i]->values(), all.values() + o, sizeof(double) * caps[i], cudaMemcpyDeviceToDevice, s);
      cudaMemcpyAsync(out[i]->count(), cdev + i, sizeof(int32_t), cudaMemcpyDeviceToDevice, s);
      o += caps[i];
    }
    cudaStreamSynchronize(s);  // `all` and cdev are freed next
    cudaFree(cdev);
  }

  // voc_.score(a, b) with a = the database entry's vector (the reference scores curr_kf->bow_vec, a keyframe's)
  double score(const BowDatabase& db, int entry, const BowVector& b) const;

  // the tree as DBoW2's save lists it, with the ids the vocabulary was created with (dfk_bow_vocabulary_export)
  BowVocabularyData Export() const
  {
    DfkBowVocabularyShape sh{};
    detail::Check(h_.get(), dfk_bow_vocabulary_export(h_.get(), voc_, &sh, nullptr, nullptr, nullptr, nullptr, nullptr,
                                                      nullptr));
    BowVocabularyData d;
    d.k = sh.k;
    d.L = sh.L;
    d.weighting = sh.weighting;
    d.scoring = sh.scoring;
    d.descriptor_bytes = sh.descriptor_bytes;
    d.node_ids.resize((size_t)sh.num_nodes);
    d.parent_ids.resize((size_t)sh.num_nodes);
    d.weights.resize((size_t)sh.num_nodes);
    d.descriptors.resize((size_t)sh.num_nodes * sh.descriptor_bytes);
    d.word_ids.resize((size_t)sh.num_words);
    d.word_nodes.resize((size_t)sh.num_words);
    detail::Check(h_.get(), dfk_bow_vocabulary_export(h_.get(), voc_, &sh, d.node_ids.data(), d.parent_ids.data(),
                                                      d.weights.data(), d.descriptors.data(), d.word_ids.data(),
                                                      d.word_nodes.data()));
    return d;
  }
  // what training found (zeros for a loaded vocabulary)
  const DfkBowTrainStats& stats() const { return stats_; }

private:
  void Train(const uint8_t* descriptors_dev, const std::vector<int64_t>& image_offsets, int descriptor_bytes, int k,
             int L, uint64_t seed)
  {
    if (image_offsets.size() < 2) throw std::invalid_argument("[BowVocabulary] no images");
    const DfkBowTrainDesc d{k, L, descriptor_bytes, (int32_t)(image_offsets.size() - 1), seed, image_offsets.back(),
                            descriptors_dev, image_offsets.data()};
    detail::Check(h_.get(), dfk_bow_vocabulary_train(h_.get(), &d, &stats_, &voc_));
  }

  detail::HandlePtr h_;
  DfkBowVocabulary* voc_ = nullptr;
  DfkBowTrainStats stats_{};
};

class BowDatabase
{
public:
  struct Result {
    unsigned int Id;
    double Score;
  };

  explicit BowDatabase(const BowVocabulary& voc) : voc_(voc)
  {
    detail::Check(voc_.handle(), dfk_bow_database_create(voc_.handle(), voc_.get(), &db_));
  }
  ~BowDatabase() { dfk_bow_database_destroy(voc_.handle(), db_); }
  BowDatabase(const BowDatabase&) = delete;
  BowDatabase& operator=(const BowDatabase&) = delete;

  // db_.add(v): the entry id; copied on the device
  unsigned int add(const BowVector& v)
  {
    const DfkBowVector x = v.view();
    int32_t first = -1;
    detail::Check(voc_.handle(), dfk_bow_database_add(voc_.handle(), db_, &x, 1, &first));
    return (unsigned int)first;
  }
  void clear() { detail::Check(voc_.handle(), dfk_bow_database_clear(voc_.handle(), db_)); }
  unsigned int size() const
  {
    int32_t n = 0;
    detail::Check(voc_.handle(), dfk_bow_database_size(voc_.handle(), db_, &n));
    return (unsigned int)n;
  }

  // db_.query(v, ret, max_results, max_id): best first; equal scores in ascending entry id (synchronises)
  void query(const BowVector& v, std::vector<Result>& ret, int max_results = 1, int max_id = -1) const
  {
    ret.clear();
    if (max_results < 1) max_results = (int)std::max(size(), 1u);  // DBoW2: max_results <= 0 keeps every result
    const DfkBowQuery q{v.view(), max_results, max_id};
    void* mem = nullptr;  // [scores fp64 | ids int32 | count int32]
    if (cudaMalloc(&mem, (sizeof(double) + sizeof(int32_t)) * (size_t)max_results + sizeof(int32_t)) != cudaSuccess)
      throw std::runtime_error("[BowDatabase::query] cudaMalloc failed");
    double* scores = static_cast<double*>(mem);
    int32_t* ids = reinterpret_cast<int32_t*>(scores + max_results);
    int32_t* count = ids + max_results;
    std::vector<int32_t> hid((size_t)max_results);
    std::vector<double> hsc((size_t)max_results);
    int32_t c = 0;
    const DfkStatus st = dfk_bow_database_query_batch(voc_.handle(), db_, &q, 1, ids, scores, count);
    if (st == DFK_OK) {
      dfk_synchronize(voc_.handle());
      cudaMemcpy(&c, count, sizeof c, cudaMemcpyDeviceToHost);
      c = std::min(c, max_results);
      cudaMemcpy(hid.data(), ids, sizeof(int32_t) * c, cudaMemcpyDeviceToHost);
      cudaMemcpy(hsc.data(), scores, sizeof(double) * c, cudaMemcpyDeviceToHost);
    }
    cudaFree(mem);
    detail::Check(voc_.handle(), st);
    for (int i = 0; i < c; ++i) ret.push_back(Result{(unsigned int)hid[i], hsc[i]});
  }

  // score(entry's vector, v) (synchronises)
  double score(int entry, const BowVector& v) const
  {
    const DfkBowScoreItem it{entry, v.view()};
    double* d = nullptr;
    if (cudaMalloc(&d, sizeof(double)) != cudaSuccess) throw std::runtime_error("[BowDatabase::score] cudaMalloc failed");
    const DfkStatus st = dfk_bow_score_batch(voc_.handle(), db_, &it, 1, d);
    double r = 0.0;
    if (st == DFK_OK) {
      dfk_synchronize(voc_.handle());
      cudaMemcpy(&r, d, sizeof r, cudaMemcpyDeviceToHost);
    }
    cudaFree(d);
    detail::Check(voc_.handle(), st);
    return r;
  }

  const DfkBowDatabase* get() const { return db_; }

private:
  const BowVocabulary& voc_;
  DfkBowDatabase* db_ = nullptr;
};

inline double BowVocabulary::score(const BowDatabase& db, int entry, const BowVector& b) const
{
  return db.score(entry, b);
}

}  // namespace df

#endif  // DFK_BOW_H_
