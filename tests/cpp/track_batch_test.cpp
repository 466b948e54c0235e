// track_batch_test.cpp -- SE3Aligner::TrackLevelsBatch through the drop-in facade: one live frame tracked against
// several keyframes in one call must give, for every keyframe, bit for bit what TrackLevels gives for it alone on a
// fresh aligner (the loops of DeepFactors::Relocalize, core/deepfactors.cpp:713-743, and of LoopDetector::DetectLoop's
// geometry check, core/system/loop_detector.cpp:149-168).  Synthetic two-level pyramids built on the device with the
// facade's GaussianBlurDown / SobelGradients.
// Build: see tests/cpp/track_batch.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
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

// a two-level image pyramid and the matching depth pyramid (2x2 subsampling) of one keyframe
struct KeyframePyr {
  DeviceImage<float> img0, img1, dpt0, dpt1;
  KeyframePyr(int W, int H, const std::vector<float>& img, const std::vector<float>& dpt)
      : img0(W, H), img1(W / 2, H / 2), dpt0(W, H), dpt1(W / 2, H / 2)
  {
    img0.copyFrom(img.data());
    dpt0.copyFrom(dpt.data());
    std::vector<float> d1((size_t)(W / 2) * (H / 2));
    for (int y = 0; y < H / 2; ++y)
      for (int x = 0; x < W / 2; ++x) d1[(size_t)y * (W / 2) + x] = dpt[(size_t)(2 * y) * W + 2 * x];
    dpt1.copyFrom(d1.data());
    auto a = img0.view(), b = img1.view();
    df::GaussianBlurDown(a, b);
  }
  std::vector<Image2DView<float>> imgs() { return {img0.view(), img1.view()}; }
  std::vector<Image2DView<float>> dpts() { return {dpt0.view(), dpt1.view()}; }
};

int main()
{
  const int W = 320, H = 240;
  std::vector<float> img0(W * H), img1(W * H), dpt0(W * H), mimg(W * H), mdpt(W * H);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      img0[y * W + x] = 0.5f + 0.25f * std::sin(x / 9.0f) * std::cos(y / 7.0f);
      img1[y * W + x] = 0.5f + 0.25f * std::sin(x / 9.0f + 0.4f) * std::cos(y / 7.0f - 0.2f);
      const float prx = 0.4f + 0.1f * std::sin(x / 20.0f) * std::cos(y / 25.0f);
      dpt0[y * W + x] = 2.0f / prx - 2.0f;
    }
  for (int y = 0; y < H; ++y)  // decoy: the keyframe mirrored left-right, with its mirrored depth
    for (int x = 0; x < W; ++x) {
      mimg[y * W + x] = img0[y * W + (W - 1 - x)];
      mdpt[y * W + x] = dpt0[y * W + (W - 1 - x)];
    }

  KeyframePyr kf(W, H, img0, dpt0), decoy(W, H, mimg, mdpt);
  // live frame: image pyramid and gradients
  DeviceImage<float> live0(W, H), live1(W / 2, H / 2);
  DeviceImage<Grad> grad0(W, H), grad1(W / 2, H / 2);
  live0.copyFrom(img1.data());
  {
    auto a = live0.view(), b = live1.view();
    df::GaussianBlurDown(a, b);
    auto g0 = grad0.view(), g1 = grad1.view();
    df::SobelGradients(a, g0);
    df::SobelGradients(b, g1);
  }
  std::vector<Image2DView<float>> live = {live0.view(), live1.view()};
  std::vector<Image2DView<Grad>> grads = {grad0.view(), grad1.view()};
  const float fx = W / 2 / 0.5773502691896257f, fy = H / 2 / 0.41421356237309503f;  // testing_utils.h:34-40
  std::vector<PinholeCamera> cams = {PinholeCamera(fx, fy, W / 2, H / 2, W, H),
                                     PinholeCamera(fx / 2, fy / 2, W / 4, H / 4, W / 2, H / 2)};
  const std::vector<int> iters = {6, 4};

  // keyframes [decoy, keyframe, keyframe from a perturbed start]
  const float rot[3] = {0.02f, -0.01f, 0.0f}, trs[3] = {0.03f, 0.0f, -0.02f};
  std::vector<SE3> start = {SE3(), SE3(), SE3::FromRotTrs(rot, trs)};
  std::vector<std::vector<Image2DView<float>>> kf_imgs = {decoy.imgs(), kf.imgs(), kf.imgs()};
  std::vector<std::vector<Image2DView<float>>> kf_dpts = {decoy.dpts(), kf.dpts(), kf.dpts()};

  std::vector<SE3> batch = start;
  df::SE3Aligner<float> aligner;
  const auto stats = aligner.TrackLevelsBatch(batch, cams, kf_imgs, live, kf_dpts, grads, iters);
  EXPECT(stats.size() == start.size());
  for (std::size_t k = 0; k < start.size(); ++k) {
    SE3 single = start[k];
    df::SE3Aligner<float> fresh;
    const auto s = fresh.TrackLevels(single, cams, kf_imgs[k], live, kf_dpts[k], grads, iters);
    std::printf("keyframe %zu: inliers %.4f error %.6g (single: %.4f %.6g)\n", k, stats[k].first, stats[k].second,
                s.first, s.second);
    EXPECT(std::memcmp(batch[k].data(), single.data(), 7 * sizeof(float)) == 0);
    EXPECT(std::memcmp(&stats[k].first, &s.first, sizeof(float)) == 0);
    EXPECT(std::memcmp(&stats[k].second, &s.second, sizeof(float)) == 0);
  }
  // the true keyframe tracks better than the decoy
  EXPECT(stats[1].second < stats[0].second);

  // every keyframe needs its own depth pyramid
  bool threw = false;
  try {
    std::vector<SE3> p = start;
    std::vector<std::vector<Image2DView<float>>> one_dpt = {kf.dpts()};
    aligner.TrackLevelsBatch(p, cams, kf_imgs, live, one_dpt, grads, iters);  // 3 poses, 1 depth pyramid
  } catch (const std::exception&) {
    threw = true;
  }
  EXPECT(threw);
  std::puts("TRACK_BATCH_TEST_OK");
  return 0;
}
