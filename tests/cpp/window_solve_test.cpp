// window_solve_test.cpp -- dfk_window_solve through the C ABI: random positive semi-definite records (pairs as unscaled
// records, sparse geometric links) uploaded to the device, assembled with dfk_window_assemble_geometric and solved; the
// same records added into a df::WindowSystem<CS> on the host, then the prior, the fixed gauge pose and the damping
// applied and the dense fp64 system solved by a host Cholesky.  The record entries are small integers, so the fp32
// buffer holds the host system exactly and dx must agree to fp64 rounding.
// Build: see tests/cpp/window_solve.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "df/dfk_factor.h"

constexpr int CS = 16;
constexpr int B = 6 + CS;
constexpr int NP = 12 + CS, NG = 12 + 2 * CS;

#define EXPECT(c)                                                                    \
  do {                                                                               \
    if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } \
  } while (0)

// record of a random integer Gram: [A^T A packed upper | A^T b | b^T b | inliers bits], n variables
template <int N>
df::JTJJrReductionItem<float, N> random_record(unsigned& s)
{
  auto rnd = [&s]() { s = s * 1664525u + 1013904223u; return (int)((s >> 16) % 5) - 2; };
  std::vector<float> A(2 * N * (N + 1));
  for (auto& a : A) a = (float)rnd();
  df::JTJJrReductionItem<float, N> r;
  int q = 0;
  for (int i = 0; i < N; ++i)
    for (int j = i; j < N; ++j) {
      float s2 = 0.0f;
      for (int m = 0; m < 2 * N; ++m) s2 += A[m * (N + 1) + i] * A[m * (N + 1) + j];
      r.JtJ.coeff()[q++] = s2;
    }
  for (int i = 0; i < N; ++i) {
    float s2 = 0.0f;
    for (int m = 0; m < 2 * N; ++m) s2 += A[m * (N + 1) + i] * A[m * (N + 1) + N];
    r.Jtr[i] = s2;
  }
  r.residual = 1.0f;
  r.inliers = 0;
  return r;
}

template <int N>
void put_record(const df::JTJJrReductionItem<float, N>& r, float* out)
{
  const int nh = N * (N + 1) / 2;
  for (int i = 0; i < nh; ++i) out[i] = r.JtJ.coeff()[i];
  for (int i = 0; i < N; ++i) out[nh + i] = r.Jtr[i];
  out[nh + N] = r.residual;
  out[nh + N + 1] = 0.0f;
}

int main()
{
  const int K = 7;
  const std::vector<int> k0 = {0, 1, 2, 3, 4, 5, 6, 2, 4, 4}, k1 = {1, 2, 3, 4, 5, 6, 0, 0, 1, 4};  // ring + chords + self
  const std::vector<int> g0 = {1, 6}, g1 = {5, 3};
  const int P = (int)k0.size(), L = (int)g0.size();
  unsigned seed = 99u;
  df::WindowSystem<CS> host(K);
  const size_t REC = DFK_SFM_RECORD_FLOATS(CS), GREC = DFK_GEO_RECORD_FLOATS(CS);
  std::vector<float> rec(REC * P), geo(GREC * L);
  for (int p = 0; p < P; ++p) {
    const auto r = random_record<NP>(seed);
    put_record(r, rec.data() + REC * p);
    host.AddUnscaled(k0[p], k1[p], r);
  }
  for (int l = 0; l < L; ++l) {
    const auto r = random_record<NG>(seed);
    put_record(r, geo.data() + GREC * l);
    host.AddGeometric(g0[l], g1[l], r);
  }

  DfkHandle h = nullptr;
  EXPECT(dfk_create(0, &h) == DFK_OK);
  std::vector<int32_t> item_pair(P), zeros(P, 0);
  for (int p = 0; p < P; ++p) item_pair[p] = p;
  DfkWindowDesc desc{K, P, P, CS, k0.data(), k1.data(), item_pair.data(), zeros.data(), zeros.data()};
  DfkWindow* w = nullptr;
  EXPECT(dfk_window_create_geometric(h, &desc, L, g0.data(), g1.data(), &w) == DFK_OK);
  const int n = K * B;
  float *rec_dev, *geo_dev, *buf_dev;
  double* dx_dev;
  int32_t* info_dev;
  EXPECT(cudaMalloc((void**)&rec_dev, rec.size() * 4) == cudaSuccess);
  EXPECT(cudaMalloc((void**)&geo_dev, geo.size() * 4) == cudaSuccess);
  EXPECT(cudaMalloc((void**)&buf_dev, dfk_window_floats(w) * 4) == cudaSuccess);
  EXPECT(cudaMalloc((void**)&dx_dev, n * 8) == cudaSuccess);
  EXPECT(cudaMalloc((void**)&info_dev, 4) == cudaSuccess);
  EXPECT(cudaMemcpy(rec_dev, rec.data(), rec.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess);
  EXPECT(cudaMemcpy(geo_dev, geo.data(), geo.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess);
  EXPECT(dfk_window_assemble_geometric(h, w, rec_dev, geo_dev, buf_dev) == DFK_OK);

  const int32_t fixed[6] = {0, 1, 2, 3, 4, 5};
  DfkWindowSolver* s = nullptr;
  EXPECT(dfk_window_solver_create(h, w, 6, fixed, &s) == DFK_OK);
  size_t tiles = 0;
  EXPECT(dfk_window_solver_tiles(h, s, &tiles) == DFK_OK);
  EXPECT(tiles == 24);  // the symbolic elimination of this graph in keyframe order: 7 diagonal, 11 joined, 6 fill
  std::printf("tiles %zu\n", tiles);
  std::vector<double> codes((size_t)K * CS);
  for (size_t i = 0; i < codes.size(); ++i) codes[i] = 0.01 * (double)((int)(i % 7) - 3);

  for (const double lam : {0.0, 1e-4, 1e3}) {
    for (const double wp : {0.0, 0.5}) {
      const DfkWindowSolveParams prm{lam, wp};
      EXPECT(dfk_window_solve(h, s, buf_dev, &prm, wp > 0 ? codes.data() : nullptr, dx_dev, info_dev) == DFK_OK);
      EXPECT(dfk_synchronize(h) == DFK_OK);  // the solve runs on the handle's stream
      std::vector<double> dx(n);
      int32_t info = -1;
      EXPECT(cudaMemcpy(dx.data(), dx_dev, n * 8, cudaMemcpyDeviceToHost) == cudaSuccess);
      EXPECT(cudaMemcpy(&info, info_dev, 4, cudaMemcpyDeviceToHost) == cudaSuccess);
      EXPECT(info == 0);
      // host: the same system, dense, kept variables 6 .. n-1
      std::vector<double> H = host.H(), g = host.g();
      if (wp > 0)
        for (int k = 0; k < K; ++k)
          for (int c = 0; c < CS; ++c) {
            H[(size_t)(k * B + 6 + c) * n + k * B + 6 + c] += wp;
            g[k * B + 6 + c] -= wp * codes[(size_t)k * CS + c];
          }
      const int m = n - 6;
      std::vector<double> A((size_t)m * m), x(m);
      double dmax = 0.0;
      for (int i = 0; i < m; ++i) dmax = std::fmax(dmax, std::fabs(H[(size_t)(i + 6) * n + i + 6]));
      for (int i = 0; i < m; ++i) {
        for (int j = 0; j < m; ++j) A[(size_t)i * m + j] = H[(size_t)(i + 6) * n + j + 6];
        A[(size_t)i * m + i] += lam * A[(size_t)i * m + i] + 1e-12 * dmax;
        x[i] = g[i + 6];
      }
      for (int j = 0; j < m; ++j) {  // Cholesky, lower, in place
        double d = A[(size_t)j * m + j];
        for (int k = 0; k < j; ++k) d -= A[(size_t)j * m + k] * A[(size_t)j * m + k];
        EXPECT(d > 0);
        d = std::sqrt(d);
        A[(size_t)j * m + j] = d;
        for (int i = j + 1; i < m; ++i) {
          double v = A[(size_t)i * m + j];
          for (int k = 0; k < j; ++k) v -= A[(size_t)i * m + k] * A[(size_t)j * m + k];
          A[(size_t)i * m + j] = v / d;
        }
      }
      for (int i = 0; i < m; ++i) {
        for (int k = 0; k < i; ++k) x[i] -= A[(size_t)i * m + k] * x[k];
        x[i] /= A[(size_t)i * m + i];
      }
      for (int i = m - 1; i >= 0; --i) {
        for (int k = i + 1; k < m; ++k) x[i] -= A[(size_t)k * m + i] * x[k];
        x[i] /= A[(size_t)i * m + i];
      }
      double err = 0.0, scale = 0.0;
      for (int i = 0; i < m; ++i) {
        err = std::fmax(err, std::fabs(dx[i + 6] - x[i]));
        scale = std::fmax(scale, std::fabs(x[i]));
      }
      std::printf("lambda %g prior %g: |dx - host| / |dx| = %.2e\n", lam, wp, err / scale);
      EXPECT(err <= 1e-9 * scale);
      for (int i = 0; i < 6; ++i) EXPECT(dx[i] == 0.0);
    }
  }
  // a rejected call writes nothing and names the problem
  const DfkWindowSolveParams bad{-1.0, 0.0};
  EXPECT(dfk_window_solve(h, s, buf_dev, &bad, nullptr, dx_dev, info_dev) == DFK_ERR_INVALID_ARG);
  std::printf("rejected: %s\n", dfk_last_error(h));
  dfk_window_solver_destroy(h, s);
  dfk_window_destroy(h, w);
  cudaFree(rec_dev);
  cudaFree(geo_dev);
  cudaFree(buf_dev);
  cudaFree(dx_dev);
  cudaFree(info_dev);
  dfk_destroy(h);
  std::puts("WINDOW_SOLVE_TEST_OK");
  return 0;
}
