// window_levels_test.cpp -- df::WindowProblem<CS>::SetActive / OptimizeLevels of the drop-in facade against the C calls
// they wrap (dfk_window_problem_set_active, dfk_window_lm_levels): on a two-keyframe window (pairs both ways, two
// levels per pair, C = 8) a facade problem and a problem made with dfk_window_problem_create from the same descriptor
// must give bit for bit the same records and window buffer under a mask, and the same LM trace, level trace and final
// state for a schedule, in both LM modes; malformed masks and schedules are rejected.
// Build: see tests/cpp/window_levels.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "df/dfk_facade.h"

constexpr int CS = 8, W = 96, H = 72, K = 2, L = 2, N = 4;  // N dense items: (pair, level)

#define EXPECT(c)                                                                       \
  do {                                                                                  \
    if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } \
  } while (0)

static float* dev_floats(const std::vector<float>& host)
{
  float* p = nullptr;
  if (cudaMalloc(&p, host.size() * sizeof(float)) != cudaSuccess) { std::puts("cudaMalloc failed"); std::exit(2); }
  cudaMemcpy(p, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice);
  return p;
}
static DfkImage view(float* p, int floats_per_px) { return DfkImage{p, (size_t)W * floats_per_px * 4, W, H}; }

struct Keyframe {
  float *img, *grad, *prx, *jac, *dpt, *valid;
  explicit Keyframe(float shift)
  {
    std::vector<float> a(W * H), pr(W * H), jc((size_t)W * H * CS), z(W * H, 0.f);
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        a[y * W + x] = 0.5f + 0.25f * std::sin((x + shift) / 6.0f) * std::cos(y / 5.0f);
        pr[y * W + x] = 0.4f + 0.05f * std::sin(x / 17.0f) * std::cos(y / 13.0f);
        for (int c = 0; c < CS; ++c) jc[((size_t)y * W + x) * CS + c] = 0.01f * std::sin(0.3f * c + x / 11.0f + y / 7.0f);
      }
    img = dev_floats(a); prx = dev_floats(pr); jac = dev_floats(jc); dpt = dev_floats(z); valid = dev_floats(z);
    grad = dev_floats(std::vector<float>(2 * W * H, 0.f));
  }
};

int main()
{
  df::SfmAligner<float, CS> al;
  DfkHandle h = al.handle();
  std::vector<Keyframe> kf{Keyframe(0.f), Keyframe(1.5f)};
  for (auto& k : kf) {
    const DfkImage i = view(k.img, 1), g = view(k.grad, 2);
    EXPECT(dfk_sobel_gradients(h, &i, &g) == DFK_OK);
  }
  // two "levels" on the same images with different focal lengths: items of one pair that differ
  const DfkCamera cams[L] = {{80.f, 80.f, W / 2.f, H / 2.f, (float)W, (float)H},
                             {60.f, 60.f, W / 2.f, H / 2.f, (float)W, (float)H}};
  const int32_t k0[2] = {0, 1}, k1[2] = {1, 0}, ip[N] = {0, 0, 1, 1}, iw[N] = {W, W, W, W}, ih[N] = {H, H, H, H};
  const DfkWindowDesc wd{K, 2, N, CS, k0, k1, ip, iw, ih};
  DfkWindow* win = nullptr;
  EXPECT(dfk_window_create(h, &wd, &win) == DFK_OK);
  const float code[CS] = {};
  std::vector<DfkSfmWorkItem> dense(N), error(N);
  std::vector<DfkDepthDecodeItem> depth(K);
  std::vector<DfkWindowItemSlots> dslots(N), eslots(N), depslots(K);
  std::vector<int32_t> edepth(N);
  for (int i = 0; i < N; ++i) {
    const int p = i / L, l = i % L;
    const Keyframe &a = kf[k0[p]], &b = kf[k1[p]];
    DfkSfmWorkItem& d = dense[i];
    std::memset(&d, 0, sizeof(d));
    d.cam = cams[l];
    d.img0 = view(a.img, 1); d.img1 = view(b.img, 1); d.dpt0 = view(a.dpt, 1); d.valid0 = view(a.valid, 1);
    d.prx0_jac = view(a.jac, CS); d.grad1 = view(b.grad, 2); d.prx_orig = view(a.prx, 1); d.code = code;
    error[i] = d;
    error[i].code = nullptr;
    dslots[i] = DfkWindowItemSlots{k0[p], k1[p], k0[p], -1};
    eslots[i] = DfkWindowItemSlots{k0[p], k1[p], -1, -1};
    edepth[i] = k0[p];
  }
  for (int k = 0; k < K; ++k) {
    depth[k] = DfkDepthDecodeItem{view(kf[k].prx, 1), view(kf[k].jac, CS), view(kf[k].dpt, 1), code};
    depslots[k] = DfkWindowItemSlots{-1, -1, k, -1};
  }
  const size_t rf = DFK_SFM_RECORD_FLOATS(CS), rec = N * rf, nf = dfk_window_floats(win);
  float *recA = nullptr, *recB = nullptr, *bufA = nullptr, *bufB = nullptr;
  cudaMalloc(&recA, rec * 4); cudaMalloc(&recB, rec * 4); cudaMalloc(&bufA, nf * 4); cudaMalloc(&bufB, nf * 4);
  DfkWindowProblemDesc desc{};
  desc.window = win;
  desc.num_dense = N; desc.dense = dense.data(); desc.dense_slots = dslots.data();
  desc.num_depth = K; desc.depth = depth.data(); desc.depth_slots = depslots.data();
  desc.num_error = N; desc.error = error.data(); desc.error_slots = eslots.data(); desc.error_depth = edepth.data();
  desc.records_dev = recA;
  df::WindowProblem<CS> fp(h, desc, K, 0);
  desc.records_dev = recB;
  DfkWindowProblem* cp = nullptr;
  EXPECT(dfk_window_problem_create(h, &desc, &cp) == DFK_OK);

  std::vector<double> poses = {0, 0, 0, 1, 0, 0, 0, 0.003, -0.002, 0.001, 1, 0.02, 0.004, -0.01}, codes(K * CS);
  poses[10] = std::sqrt(1.0 - 0.003 * 0.003 - 0.002 * 0.002 - 0.001 * 0.001);
  for (int i = 0; i < K * CS; ++i) codes[i] = 0.01 * std::sin(1.0 + i);
  auto host = [](const float* d, size_t n) {
    std::vector<float> x(n);
    cudaMemcpy(x.data(), d, n * 4, cudaMemcpyDeviceToHost);
    return x;
  };
  auto same = [&](const float* a, const float* b, size_t n) {
    const std::vector<float> x = host(a, n), y = host(b, n);
    return std::memcmp(x.data(), y.data(), n * 4) == 0;
  };
  // ---- a mask: facade and C calls bit for bit, inactive records all zero
  const std::vector<uint8_t> mask = {1, 0, 0, 1};
  fp.SetState(poses, codes);
  fp.SetActive(mask);
  EXPECT(dfk_window_problem_set_state(h, cp, poses.data(), codes.data()) == DFK_OK);
  EXPECT(dfk_window_problem_set_active(h, cp, mask.data(), nullptr) == DFK_OK);
  fp.Linearize(bufA);
  EXPECT(dfk_window_problem_linearize(h, cp, bufB) == DFK_OK);
  EXPECT(dfk_synchronize(h) == DFK_OK);
  EXPECT(same(recA, recB, rec));
  EXPECT(same(bufA, bufB, nf));
  const std::vector<float> r = host(recA, rec);
  for (int i = 0; i < N; ++i) {
    bool zero = true;
    for (size_t k = 0; k < rf; ++k) zero = zero && r[i * rf + k] == 0.0f;
    EXPECT(zero == !mask[i]);
  }
  std::printf("SetActive: facade == C calls bit for bit, inactive records zero\n");
  // ---- a schedule, both LM modes
  df::LevelSchedule s;
  s.iters = {1, 2};
  s.dense_level = {0, 1, 0, 1};
  s.pair_steps_done = {0, 2};
  s.pair_remove_after = {0, 1};
  for (int use_error = 0; use_error < 2; ++use_error) {
    df::LMParams prm;
    prm.iterations = 7;
    prm.lambda_init = 1e-3;
    prm.code_prior_weight = 1e-2;
    prm.use_error = use_error != 0;
    fp.SetState(poses, codes);
    df::LevelTrace lt;
    const df::LMTrace t = fp.OptimizeLevels(prm, s, &lt);
    std::vector<double> fpo, fco;
    fp.GetState(fpo, fco);
    EXPECT(dfk_window_problem_set_state(h, cp, poses.data(), codes.data()) == DFK_OK);
    const DfkLMParams c{7, 1e-3, 10.0, 0.1, 1e6, 1, 1e-2, use_error};
    const DfkLevelSchedule cs{2, s.iters.data(), s.dense_level.data(), nullptr, nullptr, 2, s.pair_steps_done.data(),
                              s.pair_remove_after.data()};
    std::vector<double> en(8), lam(7), sw(7);
    std::vector<int32_t> acc(7), lv(14), done(2);
    DfkLMTrace ct{en.data(), lam.data(), acc.data(), 0, 0, 0, 0};
    DfkLevelTrace clt{sw.data(), lv.data(), done.data(), 0};
    EXPECT(dfk_window_lm_levels(h, cp, &c, &cs, &ct, &clt) == DFK_OK);
    std::vector<double> cpo(poses.size()), cco(codes.size());
    EXPECT(dfk_window_problem_get_state(h, cp, cpo.data(), cco.data()) == DFK_OK);
    EXPECT(dfk_synchronize(h) == DFK_OK);
    EXPECT((int)t.energy.size() == ct.num_energies && (int)t.lambda.size() == ct.num_steps);
    for (int i = 0; i < ct.num_energies; ++i) EXPECT(t.energy[i] == en[i]);
    for (int i = 0; i < ct.num_steps; ++i) EXPECT(t.lambda[i] == lam[i] && t.accepted[i] == (acc[i] != 0));
    EXPECT(t.linearisations == ct.linearisations && t.error_evaluations == ct.error_evaluations);
    EXPECT((int)lt.switch_energy.size() == clt.num_switches && clt.num_switches > 0);
    for (int i = 0; i < clt.num_switches; ++i) EXPECT(lt.switch_energy[i] == sw[i]);
    for (int i = 0; i < ct.num_steps; ++i) EXPECT(lt.pair_levels[i][0] == lv[2 * i] && lt.pair_levels[i][1] == lv[2 * i + 1]);
    EXPECT(lt.pair_steps_done[0] == done[0] && lt.pair_steps_done[1] == done[1]);
    EXPECT(fpo == cpo && fco == cco);
    // pair 0 starts at level 1 for 3 steps; pair 1 starts 2 steps in (one step left at level 1), leaves after level 0
    EXPECT(lv[0] == 1 && lv[1] == 1 && lv[2 * 1 + 1] == 0);
    EXPECT(ct.num_steps == 7 && lv[2 * 6 + 1] == -1);
    std::printf("OptimizeLevels use_error=%d: facade == dfk_window_lm_levels bit for bit; %d switches, energy %.9g -> "
                "%.9g\n", use_error, clt.num_switches, t.energy.front(), t.energy.back());
  }
  // ---- rejections: nothing is written
  bool threw = false;
  try {
    fp.SetActive(std::vector<uint8_t>(N - 1, 1));
  } catch (const std::invalid_argument&) {
    threw = true;
  }
  EXPECT(threw);
  df::LevelSchedule bad = s;
  bad.iters = {1, -1};
  std::vector<double> p0, c0, p1, c1;
  fp.GetState(p0, c0);
  threw = false;
  try {
    fp.OptimizeLevels(df::LMParams(), bad);
  } catch (const df::CUDAException& ex) {
    threw = ex.status == DFK_ERR_INVALID_ARG;
  }
  EXPECT(threw);
  bad = s;
  bad.dense_level = {0, 2, 0, 1};  // a level outside [0, num_levels)
  threw = false;
  try {
    fp.OptimizeLevels(df::LMParams(), bad);
  } catch (const df::CUDAException& ex) {
    threw = ex.status == DFK_ERR_INVALID_ARG;
  }
  EXPECT(threw);
  fp.GetState(p1, c1);
  EXPECT(p0 == p1 && c0 == c1);
  dfk_window_problem_destroy(h, cp);
  dfk_window_destroy(h, win);
  cudaFree(recA); cudaFree(recB); cudaFree(bufA); cudaFree(bufB);
  for (auto& k : kf) for (float* p : {k.img, k.grad, k.prx, k.jac, k.dpt, k.valid}) cudaFree(p);
  std::puts("WINDOW_LEVELS_TEST_OK");
  return 0;
}
