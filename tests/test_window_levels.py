"""CPU tests of the coarse-to-fine window LM (dfk_window_lm_levels, WindowOptimizer.run(schedule=...)): the host-only
policy of dfk_levels.h against WindowOptimizer under the same scripted energies and solve results, the per-pair rule
(level_at) against a transliteration of the reference's OptimizeWork, and the masked host energy sum."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from deepfactors_b200.factors import WindowBlocks
from deepfactors_b200.window_opt import (LevelSchedule, LMParams, OptimizeWork, WindowOptimizer, level_at, level_start,
                                         window_error_sum)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# reads: iterations lambda_init lambda_up lambda_down lambda_max use_error, L iters, P steps_done remove_after, then n
# energies and m infos; prints the trace, the switch energies, the levels of every step, the final positions and the
# calls in order (V = set_levels, L = linearize, E = energy, S = solve, R = retract, A = accept)
DRIVER = r"""
#include <cstdio>
#include <string>
#include <vector>
#include "dfk_levels.h"
struct Ops {
  std::vector<double> e; std::vector<int> inf; size_t ie = 0, ii = 0; std::string log;
  DfkStatus set_levels(const int*) { log += 'V'; return DFK_OK; }
  DfkStatus linearize(bool) { log += 'L'; return DFK_OK; }
  DfkStatus energy(bool, double* f) { log += 'E'; *f = e.at(ie++); return DFK_OK; }
  DfkStatus solve(double, int* info) { log += 'S'; *info = inf.at(ii++); return DFK_OK; }
  DfkStatus retract() { log += 'R'; return DFK_OK; }
  void accept() { log += 'A'; }
};
int main() {
  DfkLMParams p{};
  int L, P, n, m;
  if (scanf("%d %lf %lf %lf %lf %d %d", &p.iterations, &p.lambda_init, &p.lambda_up, &p.lambda_down, &p.lambda_max,
            &p.use_error, &L) != 7) return 2;
  std::vector<int32_t> iters(L);
  for (auto& v : iters) if (scanf("%d", &v) != 1) return 2;
  if (scanf("%d", &P) != 1) return 2;
  std::vector<int32_t> done(P);
  std::vector<uint8_t> rem(P);
  for (auto& v : done) if (scanf("%d", &v) != 1) return 2;
  for (auto& v : rem) { int r; if (scanf("%d", &r) != 1) return 2; v = (uint8_t)r; }
  if (scanf("%d %d", &n, &m) != 2) return 2;
  Ops o;
  o.e.resize(n); o.inf.resize(m);
  for (auto& v : o.e) if (scanf("%lf", &v) != 1) return 2;
  for (auto& v : o.inf) if (scanf("%d", &v) != 1) return 2;
  DfkLevelSchedule sc{};
  sc.num_levels = L; sc.iters = iters.data(); sc.num_pairs = P; sc.pair_steps_done = done.data();
  sc.pair_remove_after = rem.data();
  const int it = p.iterations;
  std::vector<double> en(it + 1), lam(it), sw(it);
  std::vector<int32_t> acc(it), lv((size_t)it * P), out(P);
  DfkLMTrace t{en.data(), lam.data(), acc.data(), 0, 0, 0, 0};
  DfkLevelTrace lt{sw.data(), lv.data(), out.data(), 0};
  if (dfk::lm_levels_run(p, sc, o, &t, &lt) != DFK_OK) return 3;
  printf("%d %d %d %d %d\n", t.num_energies, t.num_steps, t.linearisations, t.error_evaluations, lt.num_switches);
  for (int i = 0; i < t.num_energies; ++i) printf("%.17g ", en[i]);
  printf("\n");
  for (int i = 0; i < t.num_steps; ++i) printf("%.17g %d ", lam[i], acc[i]);
  printf("\n");
  for (int i = 0; i < lt.num_switches; ++i) printf("%.17g ", sw[i]);
  printf("\n");
  for (int i = 0; i < t.num_steps * P; ++i) printf("%d ", lv[i]);
  printf("\n");
  for (int q = 0; q < P; ++q) printf("%d ", out[q]);
  printf("\n%s\n", o.log.c_str());
  return 0;
}
"""


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("levels")
    (d / "drv.cpp").write_text(DRIVER)
    exe = d / "drv"
    subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), "-I",
                    os.path.join(ROOT, "deepfactors_b200", "csrc"), str(d / "drv.cpp"), "-o", str(exe)], check=True)
    return str(exe)


def run_driver(exe, prm, use_error, iters, done, rem, energies, infos):
    inp = f"{prm.iterations} {prm.lambda_init!r} {prm.lambda_up!r} {prm.lambda_down!r} {prm.lambda_max!r} " \
          f"{int(use_error)} {len(iters)} {' '.join(map(str, iters))} {len(done)} {' '.join(map(str, done))} " \
          f"{' '.join(str(int(r)) for r in rem)} {len(energies)} {len(infos)}\n" + \
          " ".join(repr(float(e)) for e in energies) + "\n" + " ".join(str(int(i)) for i in infos) + "\n"
    out = subprocess.run([exe], input=inp, capture_output=True, text=True, check=True).stdout.split("\n")
    ne, ns, lins, errs, nsw = map(int, out[0].split())
    st = out[2].split()
    lv = [int(v) for v in out[4].split()]
    P = len(done)
    return dict(energy=[float(v) for v in out[1].split()], lam=[float(v) for v in st[0::2]],
                accepted=[bool(int(v)) for v in st[1::2]], linearisations=lins, error_evaluations=errs,
                switch_energy=[float(v) for v in out[3].split()], pair_levels=[lv[s * P:(s + 1) * P] for s in range(ns)],
                pair_steps_done=[int(v) for v in out[5].split()], log=out[6])


def run_python(prm, use_error, iters, done, rem, energies, infos):
    """WindowOptimizer.run(schedule=...) with injected linearise / solve / error / set_active on the same scripts"""
    layout = WindowBlocks(2, 1, [(0, 1)])
    off = layout.offsets()[2]
    e, inf = list(energies), list(infos)
    masks = []

    def linearise(poses, codes, todo):
        buf = np.zeros(layout.floats)
        if not use_error:
            buf[off] = e.pop(0)
        return buf, None

    def solve(buf, lam, fixed, w, codes):
        return None if inf.pop(0) != 0 else np.zeros(layout.dim)

    def error(poses, codes):
        return e.pop(0), None

    P, L = len(done), len(iters)
    sched = LevelSchedule(iters=iters, item_level=[l for _ in range(P) for l in range(L)],
                          item_pair=[q for q in range(P) for _ in range(L)], steps_done=done, remove_after=rem)
    opt = WindowOptimizer(layout, linearise, prm, solve=solve, error=error if use_error else None,
                          set_active=lambda dm, em: masks.append(dm))
    _, _, t = opt.run(np.tile([0, 0, 0, 1, 0, 0, 0.0], (2, 1)), np.zeros((2, 1)), schedule=sched)
    return t, masks


def scripts():
    rng = np.random.default_rng(7)
    out = {}
    # every step accepted: pairs at different positions, one remove_after, the schedule runs out mid-run
    out["accepted"] = (dict(iterations=14, lambda_max=1e6), [1, 2, 0], [0, 2, 4, 9], [False, True, False, True],
                       list(np.linspace(100, 1, 80)), [0] * 40)
    # rejections until lambda overflows: stall advances, and the run ends by a stall with no pair above level 0
    out["stalls"] = (dict(iterations=40, lambda_max=1e-2), [3, 3, 3], [0, 1, 7], [False, True, False],
                     [10.0] + [11.0] * 120, [0] * 60)
    # random energies and failed solves: rejected steps at switches, iterations reached mid-level
    e = list(np.linspace(100, 0, 200) + rng.normal(0, 1.0, 200))
    out["random"] = (dict(iterations=23, lambda_max=1e2), [6, 8, 5, 9], [0, 3, 6, 1, 30], [False, True, False, True, True],
                     e, list((rng.uniform(size=100) < 0.15).astype(int)))
    return out


SCRIPTS = scripts()


@pytest.mark.parametrize("use_error", [False, True])
@pytest.mark.parametrize("script", sorted(SCRIPTS))
def test_host_level_policy_matches_window_optimizer(driver, script, use_error):
    kw, iters, done, rem, energies, infos = SCRIPTS[script]
    prm = LMParams(lambda_init=1e-4, lambda_up=10.0, lambda_down=0.1, **kw)
    got = run_driver(driver, prm, use_error, iters, done, rem, energies, infos)
    want, masks = run_python(prm, use_error, iters, done, rem, energies, infos)
    print(f"{script}: accepted {got['accepted']} switches {len(got['switch_energy'])}")
    assert got["accepted"] == want.accepted and got["lam"] == want.lam
    assert got["energy"] == want.energy
    assert got["switch_energy"] == want.switch_energy
    assert got["pair_levels"] == want.pair_levels
    assert got["pair_steps_done"] == want.pair_steps_done
    assert got["linearisations"] == want.linearisations and got["error_evaluations"] == want.error_evaluations
    # one mask per level change, plus the start's
    assert got["log"].count("V") == len(masks) == 1 + len(got["switch_energy"])
    assert got["linearisations"] == 1 + len(got["switch_energy"]) + (sum(got["accepted"]) if use_error else
                                                                     got["log"].count("R"))
    lv = got["pair_levels"]
    # every step is one position of every active pair; a stall jumps
    if script == "accepted":
        P = len(done)
        for q in range(P):
            assert [s[q] for s in lv] == [level_at(iters, done[q] + t, rem[q]) for t in range(len(lv))]
        assert len(lv) == prm.iterations and len(got["switch_energy"]) > 0
        assert any(s[1] == -1 for s in lv) and lv[-1][0] == 0  # a remove_after pair left, the others stay at 0
    if script == "stalls":
        assert len(lv) < prm.iterations  # the run ended by a stall with nothing left to move
        assert all(l <= 0 for l in want.pair_levels[-1])
        assert not any(got["accepted"]) and got["switch_energy"]  # switches right after rejected steps
    if script == "random":
        assert len(lv) == prm.iterations  # iterations reached
        assert any(0 < l for l in lv[-1])  # with a pair mid-schedule


def test_call_order_at_a_switch(driver):
    """a switch re-linearises the accepted point (no retract) and reads its energy"""
    prm = LMParams(iterations=3, lambda_init=1e-4, lambda_max=1e6)
    got = run_driver(driver, prm, False, [0, 0], [0], [False], [5.0, 4.0, 3.0, 2.0, 1.0, 0.5], [0, 0, 0])
    # level 1 for step 0, level 0 from step 1: switch after step 0, none after the last step
    assert got["pair_levels"] == [[1], [0], [0]]
    assert got["log"] == "VLE" + "SRLEA" + "VLE" + "SRLEA" + "SRLEA"
    assert got["switch_energy"] == [3.0]
    got = run_driver(driver, prm, True, [0, 0], [0], [False], [5.0, 4.0, 3.0, 2.0, 1.0, 0.5], [0, 0, 0])
    assert got["log"] == "VLE" + "SRELA" + "VLE" + "SRELA" + "SRELA"


@pytest.mark.parametrize("remove_after", [False, True])
@pytest.mark.parametrize("iters", [[15, 15, 15, 30], [4, 8, 15], [0, 0, 0], [2, 0, 3]])
def test_level_at_is_the_reference_optimize_work(iters, remove_after):
    """the level a pair holds at every step (OptimizeWork::Bookkeeping, then Update) over its whole schedule, and a
    stall (SignalNoRelinearize after Update) moving a pair above level 0 to a fresh start of the next finer level"""
    w = OptimizeWork(iters, remove_after)
    total = sum(i + 1 for i in iters)
    for s in range(total + 4):
        f = w.bookkeeping()
        assert (-1 if f is None else f) == level_at(iters, s, remove_after), s
        w.update()
    assert w.finished()
    rng = np.random.default_rng(len(iters) + remove_after)
    for trial in range(20):
        w, s = OptimizeWork(iters, remove_after), 0
        for step in range(total + 4):
            f = w.bookkeeping()
            assert (-1 if f is None else f) == level_at(iters, s, remove_after), (trial, step)
            w.update()
            s += 1 if level_at(iters, s, remove_after) >= 0 else 0
            lvl = level_at(iters, s, remove_after)
            if lvl > 0 and rng.uniform() < 0.3:
                w.signal_no_relinearize()
                s = level_start(iters, lvl - 1)


def test_masked_energy_sum_matches_numpy():
    rng = np.random.default_rng(2)
    n = 40
    res = rng.uniform(0, 5, n).astype(np.float32)
    inl = rng.integers(0, 50, n).astype(np.uint32)
    inl[::7] = 0
    dense = np.stack([res, inl.view(np.float32)], axis=1)
    areas = list(rng.integers(100, 5000, n).astype(float))
    active = rng.uniform(size=n) < 0.6
    ew = window_error_sum(dense, areas, np.zeros((0, 2)), np.zeros((0, 2)), [1.5], active)
    a = active & (inl > 0)
    want = np.sum(res[a].astype(np.float64) / inl[a] * np.asarray(areas)[a])
    assert abs(ew.photometric - want) <= 1e-12 * want
    assert ew.no_inliers == int((active & (inl == 0)).sum())
    assert ew.inliers == int(inl[active].astype(np.int64).sum())
    assert ew.priors == 1.5
    # all active is the unmasked sum, bit for bit
    assert window_error_sum(dense, areas, [], [], [], np.ones(n, bool)) == window_error_sum(dense, areas, [], [], [])


def test_level_symbols_are_bound():
    from deepfactors_b200 import _lib
    for name in ("dfk_window_problem_set_active", "dfk_window_lm_levels"):
        assert name in _lib.SYMBOLS
