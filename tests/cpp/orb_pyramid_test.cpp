// orb_pyramid_test.cpp -- the ORB pyramid facade (df::OrbPyramidDetector of df/dfk_matching.h) against the C call it
// wraps, on two synthetic images of different sizes (smooth random blobs):
//   DetectAndCompute(image)          equals dfk_orb_detect_pyramid_batch's rows and count for the same item
//   DetectAndCompute(images)         gives every image the features it gets alone
//   OrbPyramidDetector(500, 1.2f, 1) equals df::OrbDetector
//   scale_factor 1                   is rejected by the call
// Build: see tests/cpp/orb_pyramid.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <stdexcept>
#include <vector>

#include "df/dfk_matching.h"

#define EXPECT(c)                                                                       \
  do {                                                                                  \
    if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } \
  } while (0)

static std::vector<uint8_t> blobs(int w, int h, unsigned seed)
{
  std::mt19937 rng(seed);
  std::uniform_real_distribution<double> U(0.0, 1.0);
  std::vector<double> acc((size_t)w * h, 60.0);
  for (int b = 0; b < 400; ++b) {
    const double cx = U(rng) * w, cy = U(rng) * h, r = 2 + 6 * U(rng), a = 160 * (U(rng) - 0.3);
    for (int y = std::max(0, (int)(cy - 3 * r)); y < std::min(h, (int)(cy + 3 * r) + 1); ++y)
      for (int x = std::max(0, (int)(cx - 3 * r)); x < std::min(w, (int)(cx + 3 * r) + 1); ++x)
        acc[(size_t)y * w + x] += a * std::exp(-((x - cx) * (x - cx) + (y - cy) * (y - cy)) / (2 * r * r));
  }
  std::vector<uint8_t> img(acc.size());
  for (size_t i = 0; i < acc.size(); ++i) img[i] = (uint8_t)std::min(255.0, std::max(0.0, acc[i] + 8 * U(rng)));
  return img;
}

static DfkImage upload(const std::vector<uint8_t>& img, int w, int h)
{
  void* p = nullptr;
  if (cudaMalloc(&p, img.size()) != cudaSuccess) { std::puts("cudaMalloc failed"); std::exit(2); }
  cudaMemcpy(p, img.data(), img.size(), cudaMemcpyHostToDevice);
  return DfkImage{p, (size_t)w, (uint32_t)w, (uint32_t)h};
}

template <typename T>
static std::vector<T> download(const T* dev, size_t n)
{
  std::vector<T> h(n);
  cudaMemcpy(h.data(), dev, n * sizeof(T), cudaMemcpyDeviceToHost);
  return h;
}

int main()
{
  const int w0 = 320, h0 = 240, w1 = 640, h1 = 480;
  const DfkImage im0 = upload(blobs(w0, h0, 1), w0, h0), im1 = upload(blobs(w1, h1, 2), w1, h1);
  df::OrbPyramidDetector det(500, 1.2f, 8);
  const int cap = det.capacity();

  // the C call on each image alone, octaves included
  float* kp = nullptr;
  uint8_t* desc = nullptr;
  int32_t *oct = nullptr, *cnt = nullptr;
  cudaMalloc(&kp, sizeof(float) * 2 * cap);
  cudaMalloc(&desc, 32 * (size_t)cap);
  cudaMalloc(&oct, sizeof(int32_t) * cap);
  cudaMalloc(&cnt, sizeof(int32_t));
  std::vector<std::vector<float>> ref_kp;
  std::vector<std::vector<uint8_t>> ref_desc;
  std::vector<int> ref_n, top;
  for (const DfkImage& im : {im0, im1}) {
    const DfkOrbPyramidItem item = det.Item(im);
    EXPECT(dfk_orb_detect_pyramid_batch(det.handle(), &item, 1, kp, desc, nullptr, nullptr, oct, cnt) == DFK_OK);
    cudaDeviceSynchronize();
    const int n = download(cnt, 1)[0];
    EXPECT(n > 0 && n <= cap);
    const std::vector<int32_t> o = download(oct, (size_t)n);
    for (int i = 1; i < n; ++i) EXPECT(o[i] >= o[i - 1]);  // levels ascending
    top.push_back(o[n - 1]);
    ref_n.push_back(n);
    ref_kp.push_back(download(kp, 2 * (size_t)n));
    ref_desc.push_back(download(desc, 32 * (size_t)n));
  }
  EXPECT(top[1] > 0);  // the 640 x 480 image has features above level 0

  // one image, then both in one batch
  const df::Features one = det.DetectAndCompute(im0);
  EXPECT(one.num == ref_n[0] && one.descriptor_bytes == 32);
  EXPECT(download(one.keypoints, 2 * (size_t)one.num) == ref_kp[0]);
  EXPECT(download(one.descriptors, 32 * (size_t)one.num) == ref_desc[0]);
  const std::vector<df::Features> both = det.DetectAndCompute(std::vector<DfkImage>{im0, im1});
  EXPECT(both.size() == 2);
  for (int i = 0; i < 2; ++i) {
    EXPECT(both[i].num == ref_n[i]);
    EXPECT(download(both[i].keypoints, 2 * (size_t)both[i].num) == ref_kp[i]);
    EXPECT(download(both[i].descriptors, 32 * (size_t)both[i].num) == ref_desc[i]);
  }

  // with one level the pyramid detector is OrbDetector
  df::OrbPyramidDetector flat(500, 1.2f, 1);
  df::OrbDetector single(500, 1.2f, 1);
  const df::Features a = flat.DetectAndCompute(im1), b = single.DetectAndCompute(im1);
  EXPECT(a.num == b.num);
  EXPECT(download(a.keypoints, 2 * (size_t)a.num) == download(b.keypoints, 2 * (size_t)b.num));
  EXPECT(download(a.descriptors, 32 * (size_t)a.num) == download(b.descriptors, 32 * (size_t)b.num));

  // an invalid setting is the C call's argument error
  bool rejected = false;
  try {
    df::OrbPyramidDetector bad(500, 1.0f, 8);
    bad.DetectAndCompute(im0);
  } catch (const std::exception&) {
    rejected = true;
  }
  EXPECT(rejected);
  std::printf("orb_pyramid_test ok: %d and %d keypoints, top levels %d and %d\n", ref_n[0], ref_n[1], top[0], top[1]);
  return 0;
}
