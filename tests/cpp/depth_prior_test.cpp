// depth_prior_test.cpp -- df::DepthPriorFactor through the factor header: Linearize over a two-level pyramid must give,
// per level, dfk_depth_run_step's system (the same per-pixel arithmetic, different partial sums), ErrorRows must give each
// record's residual bit for bit and Error 0.5 sum residual / sigma^2, and WindowSystem::AddDepthPrior must place JtJ /
// sigma^2 in both triangles of the keyframe's code block, -Jtr / sigma^2 in its code gradient and residual / sigma^2 in f.
// Build: see tests/cpp/depth_prior.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "df/dfk_factor.h"
#include "df/dfk_standins.h"

using namespace df::standin;

constexpr int CS = 8;
constexpr int NH = CS * (CS + 1) / 2;
constexpr int REC = NH + CS + 2;

struct DeviceImage {  // vc::Image2DManaged stand-in, float pixels of `k` floats each
  float* ptr = nullptr;
  size_t pitch = 0, w = 0, h = 0, k = 1;
  DeviceImage(size_t w_, size_t h_, size_t k_) : w(w_), h(h_), k(k_)
  {
    if (cudaMallocPitch((void**)&ptr, &pitch, w * k * sizeof(float), h) != cudaSuccess) { std::puts("cudaMallocPitch failed"); std::exit(2); }
  }
  ~DeviceImage() { cudaFree(ptr); }
  DeviceImage(const DeviceImage&) = delete;
  DeviceImage& operator=(const DeviceImage&) = delete;
  void copyFrom(const float* host)
  {
    cudaMemcpy2D(ptr, pitch, host, w * k * sizeof(float), w * k * sizeof(float), h, cudaMemcpyHostToDevice);
  }
  Image2DView<float> view() { return Image2DView<float>(ptr, pitch, w * k, h); }
};

#define EXPECT(c)                                                        \
  do {                                                                   \
    if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } \
  } while (0)

int main()
{
  unsigned s = 777u;
  auto rnd = [&s]() { s = s * 1664525u + 1013904223u; return (float)((s >> 8) & 0xffff) / 65536.0f - 0.5f; };
  const int sizes[2][2] = {{96, 72}, {48, 36}};
  float code[CS];
  for (float& c : code) c = 0.2f * rnd();
  std::vector<DeviceImage*> imgs;
  std::vector<df::DepthPriorFactor<CS>::Level> levels;
  for (const auto& sz : sizes) {
    const int W = sz[0], H = sz[1];
    std::vector<float> prx(W * H), tgt(W * H), jac((size_t)W * H * CS);
    for (int i = 0; i < W * H; ++i) {
      prx[i] = 0.45f + 0.2f * rnd();
      float dot = 0.0f;
      for (int k = 0; k < CS; ++k) {
        jac[(size_t)i * CS + k] = 0.02f * rnd();
        dot += jac[(size_t)i * CS + k] * code[k];
      }
      tgt[i] = (2.0f / (prx[i] + dot) - 2.0f) * 1.05f + 0.02f * rnd();
    }
    DeviceImage* t = new DeviceImage(W, H, 1);
    DeviceImage* p = new DeviceImage(W, H, 1);
    DeviceImage* j = new DeviceImage(W, H, CS);
    t->copyFrom(tgt.data());
    p->copyFrom(prx.data());
    j->copyFrom(jac.data());
    imgs.insert(imgs.end(), {t, p, j});
    levels.push_back(df::DepthPriorFactor<CS>::MakeLevel(t->view(), p->view(), j->view()));
  }
  DfkHandle h = nullptr;
  EXPECT(dfk_create(0, &h) == DFK_OK);
  const float sigma = 0.3f;
  df::DepthPriorFactor<CS> f(1, sigma, levels);
  EXPECT(f.num_levels() == 2 && f.keyframe() == 1);
  float *rec_dev = nullptr, *err_dev = nullptr;
  EXPECT(cudaMalloc((void**)&rec_dev, sizeof(float) * REC * 2) == cudaSuccess);
  EXPECT(cudaMalloc((void**)&err_dev, sizeof(float) * 4) == cudaSuccess);
  f.Linearize(h, code, rec_dev);
  f.ErrorRows(h, code, err_dev);
  EXPECT(dfk_synchronize(h) == DFK_OK);
  std::vector<float> rec(REC * 2), err(4);
  EXPECT(cudaMemcpy(rec.data(), rec_dev, sizeof(float) * rec.size(), cudaMemcpyDeviceToHost) == cudaSuccess);
  EXPECT(cudaMemcpy(err.data(), err_dev, sizeof(float) * err.size(), cudaMemcpyDeviceToHost) == cudaSuccess);
  double want_err = 0.0;
  for (int l = 0; l < 2; ++l) {
    const float* r = rec.data() + (size_t)l * REC;
    float JtJ[NH], Jtr[CS], res;
    uint64_t inl;
    EXPECT(dfk_depth_run_step(h, code, CS, &levels[l].target_dpt, &levels[l].prx_orig, &levels[l].prx_jac, JtJ, Jtr, &res,
                              &inl) == DFK_OK);
    uint32_t rin;
    std::memcpy(&rin, r + NH + CS + 1, 4);
    EXPECT(rin == (uint32_t)(sizes[l][0] * sizes[l][1]) && inl == rin);
    double mx = 0.0, d = 0.0;
    for (int e = 0; e < NH; ++e) {
      mx = std::fmax(mx, std::fabs(JtJ[e]));
      d = std::fmax(d, std::fabs((double)r[e] - JtJ[e]));
    }
    std::printf("level %d: max |JtJ - single call| %.3e of max |JtJ| %.3e\n", l, d / mx, mx);
    EXPECT(d <= 1e-5 * mx);
    EXPECT(std::fabs((double)r[NH + CS] - res) <= 1e-5 * std::fabs(res));
    EXPECT(std::memcmp(&err[2 * l], r + NH + CS, 4) == 0);  // bit for bit the record's residual
    want_err += (double)r[NH + CS] / ((double)sigma * sigma);
  }
  EXPECT(std::fabs(f.Error(err.data()) - 0.5 * want_err) <= 1e-12 * want_err);
  // WindowSystem::AddDepthPrior on keyframe 1 of 3
  df::WindowSystem<CS> ws(3);
  for (int l = 0; l < 2; ++l) ws.AddDepthPrior(f.keyframe(), rec.data() + (size_t)l * REC, sigma);
  const int B = 6 + CS, o = B + 6;
  const double s2 = (double)sigma * sigma;
  for (int i = 0; i < CS; ++i)
    for (int j = 0; j < CS; ++j) {
      const int a = std::min(i, j), b = std::max(i, j), e = a * CS - a * (a - 1) / 2 + (b - a);
      const double want = (double)rec[e] / s2 + (double)rec[REC + e] / s2;
      EXPECT(std::fabs(ws.H(o + i, o + j) - want) <= 1e-12 * std::fabs(want));
    }
  for (int i = 0; i < CS; ++i) {
    const double want = -((double)rec[NH + i] / s2 + (double)rec[REC + NH + i] / s2);
    EXPECT(std::fabs(ws.g()[o + i] - want) <= 1e-12 * std::fabs(want));
  }
  EXPECT(std::fabs(ws.f() - want_err) <= 1e-12 * want_err);
  double other = 0.0;  // nothing outside keyframe 1's code block
  for (int r = 0; r < ws.dim(); ++r)
    for (int c = 0; c < ws.dim(); ++c)
      if (!(r >= o && r < o + CS && c >= o && c < o + CS)) other += std::fabs(ws.H(r, c));
  EXPECT(other == 0.0);
  cudaFree(rec_dev);
  cudaFree(err_dev);
  for (DeviceImage* d : imgs) delete d;
  dfk_destroy(h);
  std::puts("DEPTH_PRIOR_TEST_OK");
  return 0;
}
