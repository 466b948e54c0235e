// match_test.cpp -- the matching facade (df/dfk_matching.h) against the C calls it wraps, on a synthetic two-view scene
// (500 points, 30 % outliers, ORB-sized descriptors matching query q to train q):
//   MatchBatch                   equals a host brute-force Hamming matcher
//   ReprojectionMatches          equals dfk_reprojection_match_batch's list for the same item
//   PruneMatchesByThreshold(PruneMatchesEightPoint(...))   equals ReprojectionMatches, as in the reference's constructor
// Build: see tests/cpp/match.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "df/dfk_matching.h"
#include "df/dfk_standins.h"

#define EXPECT(c)                                                                       \
  do {                                                                                  \
    if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } \
  } while (0)

constexpr int N = 500, D = 32;

template <typename T>
static T* upload(const std::vector<T>& h)
{
  T* p = nullptr;
  if (cudaMalloc(&p, h.size() * sizeof(T)) != cudaSuccess) { std::puts("cudaMalloc failed"); std::exit(2); }
  cudaMemcpy(p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
  return p;
}

int main()
{
  std::mt19937 rng(7);
  std::uniform_real_distribution<double> U(0.0, 1.0);
  const double fx = 500, fy = 500, u0 = 320, v0 = 240, a = 0.05, tx = 0.25, ty = 0.05, tz = -0.1;
  std::vector<float> kp0, kp1;
  while ((int)kp0.size() < 2 * N) {
    const double x = U(rng) * 640, y = U(rng) * 480, z = 2 + 4 * U(rng);
    const double X = (x - u0) / fx * z, Y = (y - v0) / fy * z;  // rotation a about y, then translation
    const double X1 = std::cos(a) * X + std::sin(a) * z + tx, Y1 = Y + ty, Z1 = -std::sin(a) * X + std::cos(a) * z + tz;
    const double x1 = fx * X1 / Z1 + u0, y1 = fy * Y1 / Z1 + v0;
    if (x1 < 0 || x1 >= 640 || y1 < 0 || y1 >= 480) continue;
    const bool outlier = U(rng) < 0.3;
    kp0.insert(kp0.end(), {(float)x, (float)y});
    kp1.insert(kp1.end(), {(float)(outlier ? U(rng) * 640 : x1), (float)(outlier ? U(rng) * 480 : y1)});
  }
  std::vector<uint8_t> d0((size_t)N * D), d1((size_t)N * D);
  for (size_t i = 0; i < d0.size(); ++i) d0[i] = (uint8_t)(rng() & 255);
  for (size_t i = 0; i < d1.size(); ++i) d1[i] = d0[i] ^ (uint8_t)((rng() % 16 == 0) ? 1u << (rng() % 8) : 0u);

  df::Features kf{upload(kp0), upload(d0), N, D}, fr{upload(kp1), upload(d1), N, D};
  df::standin::PinholeCamera cam(500.f, 500.f, 320.f, 240.f, 640.f, 480.f);
  df::ReprojectionMatcher matcher;
  df::MatchParams p;
  p.seed = 3;

  // MatchBatch against a host brute-force matcher
  int32_t* m_dev = nullptr;
  cudaMalloc(&m_dev, sizeof(int32_t) * 2 * N);
  matcher.MatchBatch({df::ReprojectionMatcher::Item(kf, fr, cam, p)}, m_dev);
  std::vector<int32_t> m(2 * N);
  cudaDeviceSynchronize();
  cudaMemcpy(m.data(), m_dev, m.size() * sizeof(int32_t), cudaMemcpyDeviceToHost);
  for (int q = 0; q < N; ++q) {
    int best = 1 << 30, bj = -1;
    for (int j = 0; j < N; ++j) {
      int d = 0;
      for (int b = 0; b < D; ++b) d += __builtin_popcount(d0[q * D + b] ^ d1[j * D + b]);
      if (d < best) best = d, bj = j;
    }
    EXPECT(m[2 * q] == bj && m[2 * q + 1] == best);
  }

  // ReprojectionMatches against the C call
  const std::vector<df::DMatch> rep = matcher.ReprojectionMatches(kf, fr, cam, p);
  int32_t *rows_dev = nullptr, *cnt_dev = nullptr, *ran_dev = nullptr;
  cudaMalloc(&rows_dev, sizeof(int32_t) * 3 * N);
  cudaMalloc(&cnt_dev, sizeof(int32_t));
  cudaMalloc(&ran_dev, sizeof(int32_t) * 3);
  const DfkMatchItem item = df::ReprojectionMatcher::Item(kf, fr, cam, p);
  EXPECT(dfk_reprojection_match_batch(matcher.handle(), &item, 1, rows_dev, cnt_dev, ran_dev) == DFK_OK);
  cudaDeviceSynchronize();
  int cnt = 0, ran[3];
  std::vector<int32_t> rows(3 * N);
  cudaMemcpy(&cnt, cnt_dev, sizeof(int), cudaMemcpyDeviceToHost);
  cudaMemcpy(ran, ran_dev, sizeof(ran), cudaMemcpyDeviceToHost);
  cudaMemcpy(rows.data(), rows_dev, rows.size() * sizeof(int32_t), cudaMemcpyDeviceToHost);
  EXPECT(cnt == (int)rep.size() && cnt > N / 2);
  for (int i = 0; i < cnt; ++i)
    EXPECT(rep[i].queryIdx == rows[3 * i] && rep[i].trainIdx == rows[3 * i + 1] && rep[i].distance == rows[3 * i + 2]);

  // the reference's constructor: PruneMatchesByThreshold(PruneMatchesEightPoint(...), max_dist)
  const std::vector<df::DMatch> eight = matcher.PruneMatchesEightPoint(kf, fr, cam, p);
  EXPECT((int)eight.size() == ran[1]);
  for (size_t i = 1; i < eight.size(); ++i) EXPECT(eight[i - 1].queryIdx < eight[i].queryIdx);
  const std::vector<df::DMatch> pruned = df::PruneMatchesByThreshold(eight, p.max_dist);
  EXPECT(pruned.size() == rep.size());
  for (size_t i = 0; i < rep.size(); ++i)
    EXPECT(pruned[i].queryIdx == rep[i].queryIdx && pruned[i].trainIdx == rep[i].trainIdx &&
           pruned[i].distance == rep[i].distance);
  std::printf("match_test OK: %d matches kept of %d (RANSAC: hypothesis %d, %d inliers, %d evaluated)\n", cnt, N, ran[0],
              ran[1], ran[2]);
  return 0;
}
