// preprocess_test.cpp -- the frame preprocessing facade (df::FramePreprocessor of df/dfk_preprocess.h) against the C call
// it wraps, on two random frames of different sizes into the SceneNet camera at 256 x 192 with 4 levels:
//   Preprocess(frame, cam, out)     equals dfk_preprocess_batch's colour, gray, levels and gradients for the same item
//   Preprocess(frames, cams, outs)  gives every frame the output it gets alone
//   ResizeViewport                  is the reference's fp32 arithmetic, from a DfkCamera or an accessor-style camera
// Both Preprocess calls take the cameras as INTEGRATION.md passes them: straight from ResizeViewport (DfkCamera), and as
// df::PinholeCamera-style objects.
// Build: see tests/cpp/preprocess.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "df/dfk_preprocess.h"

#define EXPECT(c)                                                                       \
  do {                                                                                  \
    if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } \
  } while (0)

static DfkImage alloc(int w, int h, size_t bpp)
{
  void* p = nullptr;
  if (cudaMalloc(&p, (size_t)w * h * bpp) != cudaSuccess) { std::puts("cudaMalloc failed"); std::exit(2); }
  cudaMemset(p, 0xAB, (size_t)w * h * bpp);
  return DfkImage{p, (size_t)w * bpp, (uint32_t)w, (uint32_t)h};
}

static std::vector<uint8_t> bytes(const DfkImage& im, size_t bpp)
{
  std::vector<uint8_t> v((size_t)im.width * im.height * bpp);
  cudaMemcpy(v.data(), im.ptr, v.size(), cudaMemcpyDeviceToHost);
  return v;
}

static df::PreprocessedFrame outputs(int w, int h, int levels)
{
  df::PreprocessedFrame o;
  o.color = alloc(w, h, 3);
  o.gray = alloc(w, h, 1);
  for (int l = 0; l < levels; ++l, w /= 2, h /= 2) {
    o.levels.push_back(alloc(w, h, 4));
    o.grads.push_back(alloc(w, h, 8));
  }
  return o;
}

static std::vector<std::vector<uint8_t>> contents(const df::PreprocessedFrame& o)
{
  std::vector<std::vector<uint8_t>> c{bytes(o.color, 3), bytes(o.gray, 1)};
  for (const DfkImage& im : o.levels) c.push_back(bytes(im, 4));
  for (const DfkImage& im : o.grads) c.push_back(bytes(im, 8));
  return c;
}

struct Cam {  // df::PinholeCamera<float>'s accessors
  DfkCamera c;
  float fx() const { return c.fx; }
  float fy() const { return c.fy; }
  float u0() const { return c.u0; }
  float v0() const { return c.v0; }
  float width() const { return c.width; }
  float height() const { return c.height; }
};

int main()
{
  const int L = 4, W = 256, H = 192;
  const DfkCamera net{(float)(W / 2) / 0.5773502691896257f, (float)(H / 2) / 0.41421356237309503f, W / 2, H / 2, W, H};
  const DfkCamera tum{525.0f, 525.0f, 319.5f, 239.5f, 640.0f, 480.0f};
  const DfkCamera half = df::ResizeViewport(tum, 320, 240);
  EXPECT(half.fx == 262.5f && half.u0 == 159.75f && half.width == 320.0f);
  const DfkCamera half2 = df::ResizeViewport(Cam{tum}, 320, 240);  // df::PinholeCamera-style accessors
  EXPECT(half2.fx == half.fx && half2.fy == half.fy && half2.u0 == half.u0 && half2.v0 == half.v0 &&
         half2.height == half.height);
  std::mt19937 rng(7);
  const int sizes[2][2] = {{320, 240}, {640, 480}};
  std::vector<DfkImage> frames;
  std::vector<DfkCamera> cams;
  for (const auto& s : sizes) {
    std::vector<uint8_t> img((size_t)s[0] * s[1] * 3);
    for (uint8_t& b : img) b = (uint8_t)(rng() & 255);
    DfkImage f = alloc(s[0], s[1], 3);
    cudaMemcpy(f.ptr, img.data(), img.size(), cudaMemcpyHostToDevice);
    frames.push_back(f);
    cams.push_back(df::ResizeViewport(tum, s[0], s[1]));
  }
  df::FramePreprocessor pre(Cam{net}, L, true);

  // the C call on each frame alone
  std::vector<std::vector<std::vector<uint8_t>>> ref;
  for (int i = 0; i < 2; ++i) {
    const df::PreprocessedFrame o = outputs(W, H, L);
    const DfkPreprocessItem it{frames[i], cams[i], net, o.color, o.gray, o.levels.data(), o.grads.data(), 1};
    EXPECT(dfk_preprocess_batch(pre.handle(), &it, 1, L, nullptr) == DFK_OK);
    cudaDeviceSynchronize();
    ref.push_back(contents(o));
  }
  // one frame through the facade, then both in one call
  const df::PreprocessedFrame one = outputs(W, H, L);
  pre.Preprocess(frames[0], df::ResizeViewport(tum, sizes[0][0], sizes[0][1]), one);  // the INTEGRATION.md line
  cudaDeviceSynchronize();
  EXPECT(contents(one) == ref[0]);
  const df::PreprocessedFrame one_acc = outputs(W, H, L);
  pre.Preprocess(frames[1], Cam{cams[1]}, one_acc);  // an accessor-style camera
  cudaDeviceSynchronize();
  EXPECT(contents(one_acc) == ref[1]);
  const std::vector<df::PreprocessedFrame> both{outputs(W, H, L), outputs(W, H, L)};
  double* stats = nullptr;
  cudaMalloc(&stats, 4 * sizeof(double));
  pre.Preprocess(frames, cams, both, stats);  // std::vector<DfkCamera>
  cudaDeviceSynchronize();
  for (int i = 0; i < 2; ++i) EXPECT(contents(both[i]) == ref[i]);
  const std::vector<df::PreprocessedFrame> both_acc{outputs(W, H, L), outputs(W, H, L)};
  pre.Preprocess(frames, std::vector<Cam>{Cam{cams[0]}, Cam{cams[1]}}, both_acc);
  cudaDeviceSynchronize();
  for (int i = 0; i < 2; ++i) EXPECT(contents(both_acc[i]) == ref[i]);
  double st[4];
  cudaMemcpy(st, stats, sizeof(st), cudaMemcpyDeviceToHost);
  EXPECT(st[0] > 0.0 && st[1] > 0.0 && st[2] > 0.0 && st[3] > 0.0);
  std::printf("preprocess_test OK: mu %.6f %.6f sigma %.6f %.6f\n", st[0], st[2], st[1], st[3]);
  return 0;
}
