// window_lm_test.cpp -- df::WindowProblem<CS> of the drop-in facade against the C calls it wraps: on a two-keyframe window
// (pairs both ways, one level, C = 8) a facade problem and a problem made with dfk_window_problem_create from the same
// descriptor must give bit for bit the same records, window buffer, error parts, LM trace and final state, in both LM
// modes; malformed input is rejected.
// Build: see tests/cpp/window_lm.mk.  Needs a GPU to run; compiling it is part of the CPU build check.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "df/dfk_facade.h"

constexpr int CS = 8, W = 96, H = 72, K = 2;

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
  df::SfmAligner<float, CS> al;  // the facade's handle (legacy default stream)
  DfkHandle h = al.handle();
  std::vector<Keyframe> kf{Keyframe(0.f), Keyframe(1.5f)};
  for (auto& k : kf) {
    const DfkImage i = view(k.img, 1), g = view(k.grad, 2);
    EXPECT(dfk_sobel_gradients(h, &i, &g) == DFK_OK);
  }
  const DfkCamera cam{80.f, 80.f, W / 2.f, H / 2.f, (float)W, (float)H};
  const int32_t k0[2] = {0, 1}, k1[2] = {1, 0}, ip[2] = {0, 1}, iw[2] = {W, W}, ih[2] = {H, H};
  const DfkWindowDesc wd{K, 2, 2, CS, k0, k1, ip, iw, ih};
  DfkWindow* win = nullptr;
  EXPECT(dfk_window_create(h, &wd, &win) == DFK_OK);
  const float code[CS] = {};
  std::vector<DfkSfmWorkItem> dense(2), error(2);
  std::vector<DfkDepthDecodeItem> depth(2);
  std::vector<DfkWindowItemSlots> dslots(2), eslots(2), depslots(2);
  std::vector<int32_t> edepth(2);
  for (int p = 0; p < 2; ++p) {
    const Keyframe &a = kf[k0[p]], &b = kf[k1[p]];
    DfkSfmWorkItem& d = dense[p];
    std::memset(&d, 0, sizeof(d));
    d.cam = cam;
    d.img0 = view(a.img, 1); d.img1 = view(b.img, 1); d.dpt0 = view(a.dpt, 1); d.valid0 = view(a.valid, 1);
    d.prx0_jac = view(a.jac, CS); d.grad1 = view(b.grad, 2); d.prx_orig = view(a.prx, 1); d.code = code;
    error[p] = d;
    error[p].code = nullptr;
    dslots[p] = DfkWindowItemSlots{k0[p], k1[p], k0[p], -1};
    eslots[p] = DfkWindowItemSlots{k0[p], k1[p], -1, -1};
    edepth[p] = k0[p];
    depth[p] = DfkDepthDecodeItem{view(kf[p].prx, 1), view(kf[p].jac, CS), view(kf[p].dpt, 1), code};
    depslots[p] = DfkWindowItemSlots{-1, -1, p, -1};
  }
  const size_t rec = 2 * (size_t)DFK_SFM_RECORD_FLOATS(CS), nf = dfk_window_floats(win);
  float *recA = nullptr, *recB = nullptr, *bufA = nullptr, *bufB = nullptr;
  double *errA = nullptr;
  cudaMalloc(&recA, rec * 4); cudaMalloc(&recB, rec * 4); cudaMalloc(&bufA, nf * 4); cudaMalloc(&bufB, nf * 4);
  cudaMalloc(&errA, 8 * DFK_WINDOW_ERROR_DOUBLES);
  DfkWindowProblemDesc desc{};
  desc.window = win;
  desc.num_dense = 2; desc.dense = dense.data(); desc.dense_slots = dslots.data();
  desc.num_depth = 2; desc.depth = depth.data(); desc.depth_slots = depslots.data();
  desc.num_error = 2; desc.error = error.data(); desc.error_slots = eslots.data(); desc.error_depth = edepth.data();
  desc.records_dev = recA;
  df::WindowProblem<CS> fp(h, desc, K, 0);
  desc.records_dev = recB;
  DfkWindowProblem* cp = nullptr;
  EXPECT(dfk_window_problem_create(h, &desc, &cp) == DFK_OK);

  std::vector<double> poses = {0, 0, 0, 1, 0, 0, 0, 0.003, -0.002, 0.001, 1, 0.02, 0.004, -0.01}, codes(K * CS);
  poses[10] = std::sqrt(1.0 - 0.003 * 0.003 - 0.002 * 0.002 - 0.001 * 0.001);
  for (int i = 0; i < K * CS; ++i) codes[i] = 0.01 * std::sin(1.0 + i);
  auto same = [](const void* a, const void* b, size_t bytes) {
    std::vector<unsigned char> x(bytes), y(bytes);
    cudaMemcpy(x.data(), a, bytes, cudaMemcpyDeviceToHost);
    cudaMemcpy(y.data(), b, bytes, cudaMemcpyDeviceToHost);
    return std::memcmp(x.data(), y.data(), bytes) == 0;
  };
  // ---- linearize and error
  fp.SetState(poses, codes);
  EXPECT(dfk_window_problem_set_state(h, cp, poses.data(), codes.data()) == DFK_OK);
  fp.Linearize(bufA);
  EXPECT(dfk_window_problem_linearize(h, cp, bufB) == DFK_OK);
  EXPECT(dfk_synchronize(h) == DFK_OK);
  EXPECT(same(recA, recB, rec * 4));
  EXPECT(same(bufA, bufB, nf * 4));
  const df::WindowError e = fp.Error();
  EXPECT(dfk_window_problem_error(h, cp, errA) == DFK_OK);
  double ec[DFK_WINDOW_ERROR_DOUBLES];
  EXPECT(dfk_synchronize(h) == DFK_OK);
  cudaMemcpy(ec, errA, sizeof(ec), cudaMemcpyDeviceToHost);
  EXPECT(e.energy == ec[0] && e.photometric == ec[1] && e.priors == ec[4] && e.inliers == (int64_t)ec[6]);
  EXPECT(e.inliers > 1000 && e.energy > 0.0);
  std::printf("linearize / error: facade == C calls bit for bit; E = %.9g, %lld inliers\n", e.energy,
              (long long)e.inliers);
  // ---- the LM loop, both modes
  for (int use_error = 0; use_error < 2; ++use_error) {
    df::LMParams prm;
    prm.iterations = 6;
    prm.lambda_init = 1e-3;
    prm.code_prior_weight = 1e-2;
    prm.use_error = use_error != 0;
    fp.SetState(poses, codes);
    const df::LMTrace t = fp.Optimize(prm);
    std::vector<double> fpo, fco;
    fp.GetState(fpo, fco);
    EXPECT(dfk_window_problem_set_state(h, cp, poses.data(), codes.data()) == DFK_OK);
    const DfkLMParams c{6, 1e-3, 10.0, 0.1, 1e6, 1, 1e-2, use_error};
    std::vector<double> en(7), lam(6);
    std::vector<int32_t> acc(6);
    DfkLMTrace ct{en.data(), lam.data(), acc.data(), 0, 0, 0, 0};
    EXPECT(dfk_window_lm(h, cp, &c, &ct) == DFK_OK);
    std::vector<double> cpo(poses.size()), cco(codes.size());
    EXPECT(dfk_window_problem_get_state(h, cp, cpo.data(), cco.data()) == DFK_OK);
    EXPECT(dfk_synchronize(h) == DFK_OK);
    EXPECT((int)t.energy.size() == ct.num_energies && (int)t.lambda.size() == ct.num_steps);
    for (int i = 0; i < ct.num_energies; ++i) EXPECT(t.energy[i] == en[i]);
    for (int i = 0; i < ct.num_steps; ++i) EXPECT(t.lambda[i] == lam[i] && t.accepted[i] == (acc[i] != 0));
    EXPECT(t.linearisations == ct.linearisations && t.error_evaluations == ct.error_evaluations);
    EXPECT(fpo == cpo && fco == cco);
    EXPECT(ct.num_energies >= 2 && t.energy.back() < t.energy.front());
    if (use_error) {
      int accepted = 0;
      for (bool a : t.accepted) accepted += a;
      EXPECT(t.linearisations == 1 + accepted);
    }
    std::printf("LM use_error=%d: facade == dfk_window_lm bit for bit; energy %.9g -> %.9g in %d steps, %d linearisations\n",
                use_error, t.energy.front(), t.energy.back(), ct.num_steps, t.linearisations);
  }
  // ---- rejections
  bool threw = false;
  try {
    fp.SetState(std::vector<double>(3), codes);
  } catch (const std::invalid_argument&) {
    threw = true;
  }
  EXPECT(threw);
  dslots[1].code0 = K;  // a code slot outside the keyframes
  desc.records_dev = recA;
  threw = false;
  try {
    df::WindowProblem<CS> bad(h, desc, K, 0);
  } catch (const df::CUDAException& ex) {
    threw = ex.status == DFK_ERR_INVALID_ARG;
  }
  EXPECT(threw);
  dfk_window_problem_destroy(h, cp);
  dfk_window_destroy(h, win);
  cudaFree(recA); cudaFree(recB); cudaFree(bufA); cudaFree(bufB); cudaFree(errA);
  for (auto& k : kf) for (float* p : {k.img, k.grad, k.prx, k.jac, k.dpt, k.valid}) cudaFree(p);
  std::puts("WINDOW_LM_TEST_OK");
  return 0;
}
