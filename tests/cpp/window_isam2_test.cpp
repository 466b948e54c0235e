// window_isam2_test.cpp -- df::WindowProblem<CS>::UpdateIncremental / MappingSteps / GrowFrom of the drop-in facade
// against the C calls they wrap (dfk_window_problem_isam2_update, dfk_window_map_steps, dfk_window_problem_grow_from):
// on a two-keyframe window (pairs both ways, two levels per pair, C = 8) a facade problem and a problem made with
// dfk_window_problem_create from the same descriptor must give the same ISAM2 counts, bit for bit the same records,
// theta_lin, delta and state over several updates, over a mapping run with works, and after a growth onto twin
// problems; a malformed growth map is rejected.
// Build: see tests/cpp/window_isam2.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
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
  auto state_equal = [&]() {
    std::vector<double> pa, ca, pb(K * 7), cb(K * CS), la, lca, da, lb(K * 7), lcb(K * CS), db(K * (6 + CS));
    fp.GetState(pa, ca);
    fp.GetLinearization(la, lca, da);
    if (dfk_window_problem_get_state(h, cp, pb.data(), cb.data()) != DFK_OK) return false;
    if (dfk_window_problem_get_linearization(h, cp, lb.data(), lcb.data(), db.data()) != DFK_OK) return false;
    dfk_synchronize(h);
    return pa == pb && ca == cb && la == lb && lca == lcb && da == db;
  };
  df::Isam2Params prm;
  prm.relinearize_threshold = 0.002;
  prm.code_prior_weight = 1e-2;
  const DfkIsam2Params cprm{prm.relinearize_threshold, prm.relinearize_skip, prm.code_prior_weight, 1};
  // ---- single updates
  fp.SetState(poses, codes);
  EXPECT(dfk_window_problem_set_state(h, cp, poses.data(), codes.data()) == DFK_OK);
  int moved = 0;
  for (int it = 0; it < 6; ++it) {
    const df::Isam2Result a = fp.UpdateIncremental(prm);
    DfkIsam2Result b{};
    EXPECT(dfk_window_problem_isam2_update(h, cp, &cprm, &b) == DFK_OK);
    EXPECT((a == df::Isam2Result{b.variables_relinearized, b.variables_reeliminated, b.factors_relinearised,
                                 b.first_column}));
    EXPECT(same(recA, recB, rec));
    EXPECT(state_equal());
    moved += a.variables_relinearized;
  }
  std::printf("UpdateIncremental: facade == C calls over 6 updates, %d keys relinearised\n", moved);
  // ---- a mapping run with works, in two calls
  df::LevelSchedule s;
  s.iters = {1, 2};
  s.dense_level = {0, 1, 0, 1};
  s.pair_remove_after = {0, 1};
  fp.SetState(poses, codes);
  EXPECT(dfk_window_problem_set_state(h, cp, poses.data(), codes.data()) == DFK_OK);
  std::vector<DfkWorkState> works;
  std::vector<std::vector<int>> lv;
  std::vector<df::Isam2Result> ra = fp.MappingSteps(prm, s, works, 2, &lv);
  const std::vector<df::Isam2Result> ra2 = fp.MappingSteps(prm, s, works, 40);
  ra.insert(ra.end(), ra2.begin(), ra2.end());
  const DfkLevelSchedule cs{2, s.iters.data(), s.dense_level.data(), nullptr, nullptr, 2, nullptr, s.pair_remove_after.data()};
  std::vector<int32_t> a(64), b(64), f(64), j(64), l(128);
  DfkMapTrace t{a.data(), b.data(), f.data(), j.data(), l.data(), 0};
  std::vector<DfkWorkState> cw(2);
  for (auto& w : cw) {
    w = DfkWorkState{};
    w.active_level = 1; w.iters[0] = 1; w.iters[1] = 2; w.first = 1; w.factor = -1;
  }
  EXPECT(dfk_window_map_steps(h, cp, &cprm, &cs, cw.data(), 42, &t) == DFK_OK);
  EXPECT((int)ra.size() == t.num_steps && t.num_steps > 2);
  for (int i = 0; i < t.num_steps; ++i)
    EXPECT((ra[i] == df::Isam2Result{a[i], b[i], f[i], j[i]}));
  for (int i = 0; i < 2; ++i) EXPECT(lv[i][0] == l[2 * i] && lv[i][1] == l[2 * i + 1]);
  EXPECT(std::memcmp(works.data(), cw.data(), sizeof(DfkWorkState) * 2) == 0);
  EXPECT(same(recA, recB, rec));
  EXPECT(state_equal());
  std::printf("MappingSteps: facade (two calls) == dfk_window_map_steps (one call), %d steps\n", t.num_steps);
  // ---- growth onto twin problems (the same window: every item kept)
  float *recC = nullptr, *recD = nullptr;
  cudaMalloc(&recC, rec * 4); cudaMalloc(&recD, rec * 4);
  cudaMemset(recC, 0, rec * 4); cudaMemset(recD, 0, rec * 4);
  desc.records_dev = recC;
  df::WindowProblem<CS> fg(h, desc, K, 0);
  desc.records_dev = recD;
  DfkWindowProblem* cg = nullptr;
  EXPECT(dfk_window_problem_create(h, &desc, &cg) == DFK_OK);
  std::vector<double> gp, gc;
  fp.GetState(gp, gc);
  fg.SetState(gp, gc);
  EXPECT(dfk_window_problem_set_state(h, cg, gp.data(), gc.data()) == DFK_OK);
  const std::vector<int32_t> keep = {0, 1, 2, 3}, none;
  bool threw = false;
  try {
    fg.GrowFrom(fp, {1, 0, 2, 3}, none, none, none);  // item 0 as old item 1: another level
  } catch (const std::exception&) {
    threw = true;
  }
  EXPECT(threw);
  const int32_t bad[4] = {1, 0, 2, 3};
  EXPECT(dfk_window_problem_grow_from(h, cg, cp, bad, nullptr, nullptr, nullptr) == DFK_ERR_INVALID_ARG);
  fg.GrowFrom(fp, keep, none, none, none);
  EXPECT(dfk_window_problem_grow_from(h, cg, cp, keep.data(), nullptr, nullptr, nullptr) == DFK_OK);
  EXPECT(dfk_synchronize(h) == DFK_OK);
  EXPECT(same(recC, recA, rec) && same(recD, recB, rec));  // the kept records, copied bit for bit
  const df::Isam2Result ga = fg.UpdateIncremental(prm);
  DfkIsam2Result gb{};
  EXPECT(dfk_window_problem_isam2_update(h, cg, &cprm, &gb) == DFK_OK);
  EXPECT((ga == df::Isam2Result{gb.variables_relinearized, gb.variables_reeliminated, gb.factors_relinearised,
                                gb.first_column}));
  EXPECT(same(recC, recD, rec));
  std::printf("GrowFrom: records carried bit for bit, next update equal (first column %d)\n", ga.first_column);
  EXPECT(dfk_window_problem_destroy(h, cg) == DFK_OK);
  EXPECT(dfk_window_problem_destroy(h, cp) == DFK_OK);
  std::puts("WINDOW_ISAM2_TEST_OK");
  return 0;
}
