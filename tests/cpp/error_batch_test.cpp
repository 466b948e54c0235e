// error_batch_test.cpp -- SfmAligner::EvaluateErrorBatch through the drop-in facade: the error() of many (pair, level)
// items in one launch must give, for every item, bit for bit what EvaluateError gives for it alone (the PhotometricFactor
// error of photometric_factor.cpp:61-81 over a window), whatever else is in the batch.  Synthetic images and depth on the
// device: two levels, a far frame (no overlap) and an item repeated.
// Build: see tests/cpp/error_batch.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "df/dfk_facade.h"
#include "df/dfk_standins.h"

using namespace df::standin;

template <typename T>
struct DeviceImage {  // vc::Image2DManaged stand-in
  T* ptr = nullptr;
  size_t pitch = 0, w = 0, h = 0;
  DeviceImage(size_t w_, size_t h_) : w(w_), h(h_)
  {
    if (cudaMallocPitch((void**)&ptr, &pitch, w * sizeof(T), h) != cudaSuccess) { std::puts("cudaMallocPitch failed"); std::exit(2); }
    cudaMemset2D(ptr, pitch, 0, w * sizeof(T), h);
  }
  ~DeviceImage() { cudaFree(ptr); }
  DeviceImage(const DeviceImage&) = delete;
  DeviceImage& operator=(const DeviceImage&) = delete;
  void copyFrom(const T* host) { cudaMemcpy2D(ptr, pitch, host, w * sizeof(T), w * sizeof(T), h, cudaMemcpyHostToDevice); }
  Image2DView<T> view() { return Image2DView<T>(ptr, pitch, w, h); }
};

#define EXPECT(c)                                                        \
  do {                                                                   \
    if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } \
  } while (0)

// one level: keyframe image and depth, frame image
struct Level {
  DeviceImage<float> img0, img1, dpt0;
  Level(int W, int H, float s) : img0(W, H), img1(W, H), dpt0(W, H)
  {
    std::vector<float> a(W * H), b(W * H), d(W * H);
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        a[y * W + x] = 0.5f + 0.25f * std::sin(s * x / 9.0f) * std::cos(s * y / 7.0f);
        b[y * W + x] = 0.5f + 0.25f * std::sin(s * x / 9.0f + 0.4f) * std::cos(s * y / 7.0f - 0.2f);
        const float prx = 0.4f + 0.1f * std::sin(s * x / 20.0f) * std::cos(s * y / 25.0f);
        d[y * W + x] = 2.0f / prx - 2.0f;
      }
    img0.copyFrom(a.data());
    img1.copyFrom(b.data());
    dpt0.copyFrom(d.data());
  }
};

int main()
{
  const int W = 320, H = 240;
  Level l0(W, H, 1.0f), l1(W / 2, H / 2, 2.0f);
  const float fx = W / 2 / 0.5773502691896257f, fy = H / 2 / 0.41421356237309503f;  // testing_utils.h:34-40
  const PinholeCamera c0(fx, fy, W / 2, H / 2, W, H), c1(fx / 2, fy / 2, W / 4, H / 4, W / 2, H / 2);
  const float rot[3] = {0.01f, -0.02f, 0.005f}, trs[3] = {0.02f, -0.01f, 0.01f}, far_t[3] = {0.0f, 0.0f, 30.0f};
  const float zero[3] = {0.0f, 0.0f, 0.0f};
  const SE3 pose0, pose1 = SE3::FromRotTrs(rot, trs), far = SE3::FromRotTrs(zero, far_t);

  typedef df::SfmAligner<float, 32> Aligner;
  Aligner al;
  std::vector<DfkSfmWorkItem> items = {
      Aligner::ErrorItem(pose0, pose1, c0, l0.img0.view(), l0.img1.view(), l0.dpt0.view()),
      Aligner::ErrorItem(pose0, pose1, c1, l1.img0.view(), l1.img1.view(), l1.dpt0.view()),
      Aligner::ErrorItem(pose0, far, c0, l0.img0.view(), l0.img1.view(), l0.dpt0.view()),
      Aligner::ErrorItem(pose1, pose0, c1, l1.img0.view(), l1.img1.view(), l1.dpt0.view())};
  items.push_back(items[1]);
  const auto batch = al.EvaluateErrorBatch(items);
  EXPECT(batch.size() == items.size());
  // what each item evaluates: its level, pose0 and pose1
  const int level_of[5] = {0, 1, 0, 1, 1};
  const SE3* pose0_of[5] = {&pose0, &pose0, &pose0, &pose1, &pose0};
  const SE3* pose1_of[5] = {&pose1, &pose1, &far, &pose0, &pose1};
  for (std::size_t i = 0; i < items.size(); ++i) {
    Level& L = level_of[i] == 0 ? l0 : l1;
    const PinholeCamera& cam = level_of[i] == 0 ? c0 : c1;
    DeviceImage<float> std0(L.img0.w, L.img0.h);
    DeviceImage<Grad> grad1(L.img0.w, L.img0.h);
    const auto s = al.EvaluateError(*pose0_of[i], *pose1_of[i], cam, L.img0.view(), L.img1.view(), L.dpt0.view(),
                                    std0.view(), grad1.view());
    std::printf("item %zu: residual %.9g inliers %zu (single: %.9g %zu)\n", i, batch[i].residual, batch[i].inliers,
                s.residual, s.inliers);
    EXPECT(std::memcmp(&batch[i].residual, &s.residual, sizeof(float)) == 0);
    EXPECT(batch[i].inliers == s.inliers);
  }
  EXPECT(batch[0].inliers > 10000 && batch[2].inliers == 0);

  // a fused depth decode is refused: the depth comes from dpt0
  std::vector<float> code(32, 0.0f);
  items[1].code = code.data();
  bool threw = false;
  try {
    al.EvaluateErrorBatch(items);
  } catch (const std::exception&) {
    threw = true;
  }
  EXPECT(threw);
  std::puts("ERROR_BATCH_TEST_OK");
  return 0;
}
