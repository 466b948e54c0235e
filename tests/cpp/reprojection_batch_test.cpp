// reprojection_batch_test.cpp -- df::LinearizeReprojectionBatch through the factor header: every record of a batch
// must be the Gram of the rows df::LinearizeReprojection returns for that factor alone ([A^T A | -A^T b | b^T b | valid
// matches]), and WindowSystem::AddUnscaled must add its residual to f as it is.  Synthetic level-0 keyframe buffers.
// Build: see tests/cpp/reprojection_batch.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
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
constexpr int NP = 12 + CS;

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
  // the reference views the code Jacobian as a (W * CS) x H float image
  Image2DView<float> view() { return Image2DView<float>(ptr, pitch, w * k, h); }
};

#define EXPECT(c)                                                        \
  do {                                                                   \
    if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } \
  } while (0)

struct Factor {
  SE3 pose0, pose1;
  Code<CS> code;
  std::vector<float> query, train;
};

int main()
{
  const int W = 160, H = 120;
  std::vector<float> prx(W * H), jac((size_t)W * H * CS);
  unsigned s = 12345u;
  auto rnd = [&s]() { s = s * 1664525u + 1013904223u; return (float)((s >> 8) & 0xffff) / 65536.0f - 0.5f; };
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      prx[y * W + x] = 0.4f + 0.1f * std::sin(x / 20.0f) * std::cos(y / 25.0f);
      for (int k = 0; k < CS; ++k) jac[((size_t)y * W + x) * CS + k] = 0.02f * rnd();
    }
  DeviceImage prx_orig(W, H, 1), prx_jac(W, H, CS);
  prx_orig.copyFrom(prx.data());
  prx_jac.copyFrom(jac.data());
  PinholeCamera cam(150.0f, 150.0f, W / 2.0f, H / 2.0f, W, H);

  // three factors of different sizes and codes; factor 1 has matches outside the image
  const int sizes[3] = {300, 7, 129};
  std::vector<Factor> fs(3);
  for (int f = 0; f < 3; ++f) {
    const float rot[3] = {0.01f * f, -0.02f, 0.005f}, trs[3] = {0.05f, -0.02f * f, 0.03f};
    fs[f].pose1 = SE3::FromRotTrs(rot, trs);
    for (int k = 0; k < CS; ++k) fs[f].code[k] = 0.3f * rnd();
    for (int i = 0; i < sizes[f]; ++i) {
      const float qx = 4.0f + (W - 9.0f) * (rnd() + 0.5f), qy = 4.0f + (H - 9.0f) * (rnd() + 0.5f);
      fs[f].query.push_back(qx);
      fs[f].query.push_back(qy);
      fs[f].train.push_back(qx + 3.0f + 2.0f * rnd());
      fs[f].train.push_back(qy - 2.0f + 2.0f * rnd());
    }
  }
  fs[1].query[0] = -4.0f;       // outside the image: zero rows, not an inlier
  fs[1].query[3] = H + 10.0f;

  DfkHandle h = nullptr;
  EXPECT(dfk_create(0, &h) == DFK_OK);
  std::vector<DfkReprojectionItem> items;
  for (auto& f : fs)
    items.push_back(df::ReprojectionItem<CS>(f.pose0, f.pose1, f.code, cam, prx_orig.view(), prx_jac.view(),
                                             (int)f.query.size() / 2, f.query.data(), f.train.data(), 1.5f, 2.0f));
  const size_t REC = DFK_SFM_RECORD_FLOATS(CS);
  float* rec_dev = nullptr;
  EXPECT(cudaMalloc((void**)&rec_dev, sizeof(float) * REC * items.size()) == cudaSuccess);
  df::LinearizeReprojectionBatch<CS>(h, items, rec_dev);
  EXPECT(dfk_synchronize(h) == DFK_OK);
  std::vector<float> rec(REC * items.size());
  EXPECT(cudaMemcpy(rec.data(), rec_dev, sizeof(float) * rec.size(), cudaMemcpyDeviceToHost) == cudaSuccess);

  for (int f = 0; f < 3; ++f) {
    const df::SparseRows rows = df::LinearizeReprojection<CS>(h, fs[f].pose0, fs[f].pose1, fs[f].code, cam, prx_orig.view(),
                                                              prx_jac.view(), sizes[f], fs[f].query.data(),
                                                              fs[f].train.data(), 1.5f, 2.0f);
    // fp64 Gram of the single call's rows [A | b]
    std::vector<double> G((size_t)(NP + 1) * (NP + 1), 0.0);
    int valid = 0;
    for (int r = 0; r < rows.num_rows; ++r) {
      const float* a = rows.row(r);
      bool any = false;
      for (int i = 0; i <= NP; ++i) {
        any = any || a[i] != 0.0f;
        for (int j = 0; j <= NP; ++j) G[(size_t)i * (NP + 1) + j] += (double)a[i] * a[j];
      }
      valid += (r % 2 == 0 && any) ? 1 : 0;
    }
    df::JTJJrReductionItem<float, NP> sys;
    const float* r = rec.data() + REC * f;
    for (int i = 0; i < sys.JtJ.Size; ++i) sys.JtJ.coeff()[i] = r[i];
    for (int i = 0; i < NP; ++i) sys.Jtr[i] = r[sys.JtJ.Size + i];
    sys.residual = r[sys.JtJ.Size + NP];
    unsigned bits;
    std::memcpy(&bits, &r[sys.JtJ.Size + NP + 1], 4);
    sys.inliers = bits;
    double hmax = 0.0, herr = 0.0, gmax = 0.0, gerr = 0.0;
    for (int i = 0; i < NP; ++i) {
      for (int j = 0; j < NP; ++j) {
        hmax = std::fmax(hmax, std::fabs(G[(size_t)i * (NP + 1) + j]));
        herr = std::fmax(herr, std::fabs(sys.JtJ.toDenseMatrix(i, j) - G[(size_t)i * (NP + 1) + j]));
      }
      gmax = std::fmax(gmax, std::fabs(G[(size_t)i * (NP + 1) + NP]));
      gerr = std::fmax(gerr, std::fabs(-sys.Jtr[i] - G[(size_t)i * (NP + 1) + NP]));
    }
    const double res = G[(size_t)NP * (NP + 1) + NP];
    std::printf("factor %d: matches %d valid %d inliers %zu |dH|/max %.2e |dJtr|/max %.2e residual %.6g vs %.6g\n", f,
                sizes[f], valid, sys.inliers, herr / hmax, gerr / gmax, sys.residual, res);
    EXPECT(hmax > 0.0 && herr <= 2e-5 * hmax);
    EXPECT(gerr <= 1e-4 * gmax);
    EXPECT(std::fabs(sys.residual - res) <= 1e-5 * res);
    EXPECT((int)sys.inliers == valid);
    EXPECT(f != 1 || valid == sizes[f] - 2);
    // the window's energy takes the record's residual as it is
    df::WindowSystem<CS> win(2);
    win.AddUnscaled(0, 1, sys);
    EXPECT(win.f() == (double)sys.residual);
    EXPECT(win.H(0, 6) == (double)sys.JtJ.toDenseMatrix(0, 12));  // code0 of keyframe 0 is window column 6
    EXPECT(win.g()[6 + CS] == -(double)sys.Jtr[6]);               // pose1 of keyframe 1
  }
  cudaFree(rec_dev);
  dfk_destroy(h);
  std::puts("REPROJECTION_BATCH_TEST_OK");
  return 0;
}
