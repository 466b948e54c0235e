// geometric_batch_test.cpp -- df::LinearizeSparseGeometricBatch through the factor header: every record of a batch must
// be the Gram of the rows df::LinearizeSparseGeometric returns for that factor alone ([A^T A | -A^T b | b^T b | valid
// points] over [pose0 | pose1 | code0 | code1]), and WindowSystem::AddGeometric must place all four variable blocks,
// including the code0 x code1 coupling, and add the residual to f as it is.  Synthetic level-0 keyframe buffers.
// Build: see tests/cpp/geometric_batch.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
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
constexpr int NG = 12 + 2 * CS;

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
  // a gradient image has Eigen::Matrix<float,1,2> pixels in the reference: its width counts pixels
  Image2DView<float> pixel_view() { return Image2DView<float>(ptr, pitch, w, h); }
};

#define EXPECT(c)                                                        \
  do {                                                                   \
    if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } \
  } while (0)

struct Factor {
  SE3 pose0, pose1;
  Code<CS> code0, code1;
  std::vector<int> points;
};

int main()
{
  const int W = 160, H = 120;
  unsigned s = 4321u;
  auto rnd = [&s]() { s = s * 1664525u + 1013904223u; return (float)((s >> 8) & 0xffff) / 65536.0f - 0.5f; };
  // two keyframes of one smooth scene, each with its own code Jacobian; kf1's depth gradient by central differences
  std::vector<float> prx0(W * H), prx1(W * H), jac0((size_t)W * H * CS), jac1((size_t)W * H * CS), dpt1(W * H),
      grad1((size_t)W * H * 2, 0.0f);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      prx0[y * W + x] = 0.4f + 0.1f * std::sin(x / 20.0f) * std::cos(y / 25.0f);
      prx1[y * W + x] = 0.4f + 0.1f * std::sin(x / 21.0f + 0.3f) * std::cos(y / 24.0f);
      dpt1[y * W + x] = 2.0f / prx1[y * W + x] - 2.0f;
      for (int k = 0; k < CS; ++k) {
        jac0[((size_t)y * W + x) * CS + k] = 0.01f * rnd();
        jac1[((size_t)y * W + x) * CS + k] = 0.01f * rnd();
      }
    }
  for (int y = 1; y < H - 1; ++y)
    for (int x = 1; x < W - 1; ++x) {
      grad1[((size_t)y * W + x) * 2] = 0.5f * (dpt1[y * W + x + 1] - dpt1[y * W + x - 1]);
      grad1[((size_t)y * W + x) * 2 + 1] = 0.5f * (dpt1[(y + 1) * W + x] - dpt1[(y - 1) * W + x]);
    }
  DeviceImage p0(W, H, 1), j0(W, H, CS), p1(W, H, 1), j1(W, H, CS), g1(W, H, 2);
  p0.copyFrom(prx0.data());
  j0.copyFrom(jac0.data());
  p1.copyFrom(prx1.data());
  j1.copyFrom(jac1.data());
  g1.copyFrom(grad1.data());
  PinholeCamera cam(150.0f, 150.0f, W / 2.0f, H / 2.0f, W, H);

  // three factors of different sizes, poses and codes; factor 1 has points outside the image
  const int sizes[3] = {300, 7, 129};
  std::vector<Factor> fs(3);
  for (int f = 0; f < 3; ++f) {
    const float rot[3] = {0.01f * f, -0.02f, 0.005f}, trs[3] = {0.03f, -0.02f * f, 0.04f};
    fs[f].pose1 = SE3::FromRotTrs(rot, trs);
    for (int k = 0; k < CS; ++k) {
      fs[f].code0[k] = 0.3f * rnd();
      fs[f].code1[k] = 0.3f * rnd();
    }
    for (int i = 0; i < sizes[f]; ++i) {
      fs[f].points.push_back(4 + (int)((W - 9) * (rnd() + 0.5f)));
      fs[f].points.push_back(4 + (int)((H - 9) * (rnd() + 0.5f)));
    }
  }
  fs[1].points[0] = -4;       // outside the image: zero row, not an inlier
  fs[1].points[3] = H + 10;

  DfkHandle h = nullptr;
  EXPECT(dfk_create(0, &h) == DFK_OK);
  std::vector<DfkSparseGeometricItem> items;
  for (auto& f : fs)
    items.push_back(df::SparseGeometricItem<CS>(f.pose0, f.pose1, f.code0, f.code1, cam, p0.view(), j0.view(), p1.view(),
                                                j1.view(), g1.pixel_view(), (int)f.points.size() / 2, f.points.data(), 0.1f));
  const size_t REC = DFK_GEO_RECORD_FLOATS(CS);
  float* rec_dev = nullptr;
  EXPECT(cudaMalloc((void**)&rec_dev, sizeof(float) * REC * items.size()) == cudaSuccess);
  df::LinearizeSparseGeometricBatch<CS>(h, items, rec_dev);
  EXPECT(dfk_synchronize(h) == DFK_OK);
  std::vector<float> rec(REC * items.size());
  EXPECT(cudaMemcpy(rec.data(), rec_dev, sizeof(float) * rec.size(), cudaMemcpyDeviceToHost) == cudaSuccess);

  for (int f = 0; f < 3; ++f) {
    const df::SparseRows rows = df::LinearizeSparseGeometric<CS>(h, fs[f].pose0, fs[f].pose1, fs[f].code0, fs[f].code1, cam,
                                                                 p0.view(), j0.view(), p1.view(), j1.view(), g1.pixel_view(),
                                                                 sizes[f], fs[f].points.data(), 0.1f);
    // fp64 Gram of the single call's rows [A | b] and its absolute counterpart (the per-entry error scale)
    std::vector<double> G((size_t)(NG + 1) * (NG + 1), 0.0), S(G.size(), 0.0);
    for (int r = 0; r < rows.num_rows; ++r) {
      const float* a = rows.row(r);
      for (int i = 0; i <= NG; ++i)
        for (int j = 0; j <= NG; ++j) {
          G[(size_t)i * (NG + 1) + j] += (double)a[i] * a[j];
          S[(size_t)i * (NG + 1) + j] += std::fabs((double)a[i] * a[j]);
        }
    }
    df::JTJJrReductionItem<float, NG> sys;
    const float* r = rec.data() + REC * f;
    for (int i = 0; i < sys.JtJ.Size; ++i) sys.JtJ.coeff()[i] = r[i];
    for (int i = 0; i < NG; ++i) sys.Jtr[i] = r[sys.JtJ.Size + i];
    sys.residual = r[sys.JtJ.Size + NG];
    unsigned bits;
    std::memcpy(&bits, &r[sys.JtJ.Size + NG + 1], 4);
    sys.inliers = bits;
    double hr = 0.0, gr = 0.0;  // worst |error| / scale per entry
    for (int i = 0; i < NG; ++i) {
      for (int j = 0; j < NG; ++j) {
        const double sc = S[(size_t)i * (NG + 1) + j];
        if (sc > 0) hr = std::fmax(hr, std::fabs(sys.JtJ.toDenseMatrix(i, j) - G[(size_t)i * (NG + 1) + j]) / sc);
      }
      const double sc = S[(size_t)i * (NG + 1) + NG];
      if (sc > 0) gr = std::fmax(gr, std::fabs(-sys.Jtr[i] - G[(size_t)i * (NG + 1) + NG]) / sc);
    }
    const double res = G[(size_t)NG * (NG + 1) + NG];
    std::printf("factor %d: points %d valid %d inliers %zu worst |dH|/S %.2e |dJtr|/B %.2e residual %.6g vs %.6g\n", f,
                sizes[f], rows.num_valid, sys.inliers, hr, gr, sys.residual, res);
    EXPECT(rows.num_valid > 0);
    EXPECT(hr <= 5e-5 && gr <= 1e-6);
    EXPECT(std::fabs(sys.residual - res) <= 1e-5 * res);
    EXPECT((int)sys.inliers == rows.num_valid);
    EXPECT(f != 1 || rows.num_valid <= sizes[f] - 2);
    // the window: four variable blocks of the link (keyframes 2 -> 0), residual as it is
    df::WindowSystem<CS> win(3);
    win.AddGeometric(2, 0, sys);
    constexpr int B = df::WindowSystem<CS>::Block;
    EXPECT(win.f() == (double)sys.residual);
    EXPECT(win.H(2 * B + 6, 0 * B + 6) == (double)sys.JtJ.toDenseMatrix(12, 12 + CS));  // code0 (kf 2) x code1 (kf 0)
    EXPECT(win.H(0 * B + 6, 2 * B + 6) == (double)sys.JtJ.toDenseMatrix(12 + CS, 12));  // and its transpose
    EXPECT(win.H(0, 0) == (double)sys.JtJ.toDenseMatrix(6, 6));                          // pose1 of kf 0
    EXPECT(win.H(2 * B, 2 * B) == (double)sys.JtJ.toDenseMatrix(0, 0));                  // pose0 of kf 2
    EXPECT(win.g()[6 + CS - 1] == -(double)sys.Jtr[12 + 2 * CS - 1]);                     // code1 of kf 0
    EXPECT(win.g()[B + 3] == 0.0);                                                       // kf 1 untouched
  }
  cudaFree(rec_dev);
  dfk_destroy(h);
  std::puts("GEOMETRIC_BATCH_TEST_OK");
  return 0;
}
