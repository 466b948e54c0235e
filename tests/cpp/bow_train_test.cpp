// bow_train_test -- df::BowVocabulary's training constructor, Export and df::BowVocabularyData::SaveText (df/dfk_bow.h).
//   bow_train_test text IN.yml OUT.yml
//       LoadText then SaveText (no GPU): the CPU tests compare OUT with IN and with the Python writer
//   bow_train_test train DESC.bin OFFSETS.bin D k L seed OUT.yml
//       DESC.bin uint8 [N, D], OFFSETS.bin int64 [images + 1]: trains from host features, writes SaveText of Export to
//       OUT.yml, prints the stats; then LoadText of OUT.yml through dfk_bow_vocabulary_create must export the same
//       arrays, and a descriptor's word must be the same in both vocabularies
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <sstream>
#include <vector>

#include "df/dfk_bow.h"

static std::vector<char> read_all(const char* path)
{
  std::ifstream f(path, std::ios::binary);
  return std::vector<char>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

static bool same(const df::BowVocabularyData& a, const df::BowVocabularyData& b)
{
  return a.k == b.k && a.L == b.L && a.weighting == b.weighting && a.scoring == b.scoring &&
         a.descriptor_bytes == b.descriptor_bytes && a.node_ids == b.node_ids && a.parent_ids == b.parent_ids &&
         a.descriptors == b.descriptors && a.word_ids == b.word_ids && a.word_nodes == b.word_nodes &&
         a.weights.size() == b.weights.size() &&
         std::memcmp(a.weights.data(), b.weights.data(), sizeof(double) * a.weights.size()) == 0;
}

static int text(const char* in, const char* out)
{
  std::ifstream f(in);
  const df::BowVocabularyData d = df::BowVocabularyData::LoadText(f);
  std::ofstream o(out);
  d.SaveText(o);
  std::puts("bow_train_test text OK");
  return 0;
}

static int train(char** a)
{
  const std::vector<char> raw = read_all(a[0]), offs = read_all(a[1]);
  const int D = std::atoi(a[2]), k = std::atoi(a[3]), L = std::atoi(a[4]);
  const uint64_t seed = std::strtoull(a[5], nullptr, 10);
  std::vector<int64_t> off(offs.size() / 8);
  std::memcpy(off.data(), offs.data(), offs.size());
  std::vector<std::vector<uint8_t>> features;
  for (size_t j = 0; j + 1 < off.size(); ++j)
    features.emplace_back(raw.begin() + off[j] * D, raw.begin() + off[j + 1] * D);
  df::BowVocabulary voc(features, D, k, L, seed);
  const df::BowVocabularyData d = voc.Export();
  {
    std::ofstream o(a[6]);
    d.SaveText(o);
  }
  const DfkBowTrainStats& s = voc.stats();
  std::printf("stats %d %d %d %d %d\n", s.num_nodes, s.num_words, s.max_rounds, s.capped_nodes, s.empty_clusters);
  std::ifstream f(a[6]);
  const df::BowVocabularyData loaded = df::BowVocabularyData::LoadText(f);
  if (!same(d, loaded)) {
    std::puts("LoadText of SaveText differs from the exported arrays");
    return 1;
  }
  df::BowVocabulary back(loaded);
  if (!same(back.Export(), d)) {
    std::puts("the loaded vocabulary exports differently");
    return 1;
  }
  // the first image's words in both vocabularies
  const int n = (int)(off[1] - off[0]);
  if (n > 0) {
    void* dev = nullptr;
    cudaMalloc(&dev, (size_t)n * D);
    cudaMemcpy(dev, raw.data(), (size_t)n * D, cudaMemcpyHostToDevice);
    const DfkFeatureSet fs{nullptr, static_cast<const uint8_t*>(dev), n, D};
    df::BowVector v1, v2;
    voc.transform(fs, v1);
    back.transform(fs, v2);
    cudaFree(dev);
    if (v1.Host() != v2.Host()) {
      std::puts("the trained and the loaded vocabulary transform differently");
      return 1;
    }
  }
  std::puts("bow_train_test OK");
  return 0;
}

int main(int argc, char** argv)
{
  try {
    if (argc == 4 && std::strcmp(argv[1], "text") == 0) return text(argv[2], argv[3]);
    if (argc == 9 && std::strcmp(argv[1], "train") == 0) return train(argv + 2);
  } catch (const std::exception& e) {
    std::printf("error: %s\n", e.what());
    return 1;
  }
  std::puts("usage: bow_train_test text IN.yml OUT.yml | bow_train_test train DESC.bin OFFSETS.bin D k L seed OUT.yml");
  return 2;
}
