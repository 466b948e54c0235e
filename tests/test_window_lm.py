"""CPU tests of the window problem (dfk_window_problem_*, dfk_window_lm): the ABI table, the host-only LM policy of
dfk_lm.h against WindowOptimizer under the same scripted energies and solve results, and the state slots
SfmWindowProblem.device_problem names for every factor kind."""
import os
import shutil
import subprocess
from collections import namedtuple

import numpy as np
import pytest

from deepfactors_b200.factors import WindowBlocks
from deepfactors_b200.window_opt import LMParams, WindowOptimizer, problem_slots

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# reads: iterations lambda_init lambda_up lambda_down lambda_max use_error, then n energies, then m infos; prints the
# trace and the calls in order (L = linearize, E = energy, S = solve, R = retract, A = accept)
DRIVER = r"""
#include <cstdio>
#include <string>
#include <vector>
#include "dfk_lm.h"
struct Ops {
  std::vector<double> e; std::vector<int> inf; size_t ie = 0, ii = 0; std::string log;
  DfkStatus linearize(bool) { log += 'L'; return DFK_OK; }
  DfkStatus energy(bool, double* f) { log += 'E'; *f = e.at(ie++); return DFK_OK; }
  DfkStatus solve(double, int* info) { log += 'S'; *info = inf.at(ii++); return DFK_OK; }
  DfkStatus retract() { log += 'R'; return DFK_OK; }
  void accept() { log += 'A'; }
};
int main() {
  DfkLMParams p{};
  int n, m;
  if (scanf("%d %lf %lf %lf %lf %d %d %d", &p.iterations, &p.lambda_init, &p.lambda_up, &p.lambda_down, &p.lambda_max,
            &p.use_error, &n, &m) != 8) return 2;
  Ops o;
  o.e.resize(n); o.inf.resize(m);
  for (auto& v : o.e) if (scanf("%lf", &v) != 1) return 2;
  for (auto& v : o.inf) if (scanf("%d", &v) != 1) return 2;
  std::vector<double> en(p.iterations + 1), lam(p.iterations);
  std::vector<int32_t> acc(p.iterations);
  DfkLMTrace t{en.data(), lam.data(), acc.data(), 0, 0, 0, 0};
  if (dfk::lm_run(p, o, &t) != DFK_OK) return 3;
  printf("%d %d %d %d\n", t.num_energies, t.num_steps, t.linearisations, t.error_evaluations);
  for (int i = 0; i < t.num_energies; ++i) printf("%.17g ", en[i]);
  printf("\n");
  for (int i = 0; i < t.num_steps; ++i) printf("%.17g %d ", lam[i], acc[i]);
  printf("\n%s\n", o.log.c_str());
  return 0;
}
"""


def test_window_problem_symbols_are_bound():
    from deepfactors_b200 import _lib
    for name in ("dfk_window_problem_create", "dfk_window_problem_destroy", "dfk_window_problem_set_state",
                 "dfk_window_problem_get_state", "dfk_window_problem_linearize", "dfk_window_problem_error",
                 "dfk_window_problem_retract", "dfk_window_lm"):
        assert name in _lib.SYMBOLS


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("lm")
    (d / "drv.cpp").write_text(DRIVER)
    exe = d / "drv"
    subprocess.run([cxx, "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-I",
                    os.path.join(ROOT, "deepfactors_b200", "csrc"), str(d / "drv.cpp"), "-o", str(exe)], check=True)
    return str(exe)


def run_driver(exe, prm: LMParams, use_error, energies, infos):
    inp = f"{prm.iterations} {prm.lambda_init!r} {prm.lambda_up!r} {prm.lambda_down!r} {prm.lambda_max!r} " \
          f"{int(use_error)} {len(energies)} {len(infos)}\n" + " ".join(repr(float(e)) for e in energies) + "\n" + \
          " ".join(str(int(i)) for i in infos) + "\n"
    out = subprocess.run([exe], input=inp, capture_output=True, text=True, check=True).stdout.split("\n")
    ne, ns, lins, errs = map(int, out[0].split())
    en = [float(v) for v in out[1].split()]
    st = out[2].split()
    lam = [float(v) for v in st[0::2]]
    acc = [bool(int(v)) for v in st[1::2]]
    assert len(en) == ne and len(lam) == ns
    return dict(energy=en, lam=lam, accepted=acc, linearisations=lins, error_evaluations=errs, log=out[3])


def run_python(prm: LMParams, use_error, energies, infos):
    """WindowOptimizer with injected linearise / solve / error consuming the same scripts"""
    layout = WindowBlocks(2, 1, [(0, 1)])
    off = layout.offsets()[2]
    e, inf = list(energies), list(infos)

    def take_energy():
        return e.pop(0)

    def linearise(poses, codes, todo):
        buf = np.zeros(layout.floats)
        if not use_error:
            buf[off] = take_energy()
        return buf, None

    def solve(buf, lam, fixed, w, codes):
        return None if inf.pop(0) != 0 else np.zeros(layout.dim)

    def error(poses, codes):
        return take_energy(), None

    opt = WindowOptimizer(layout, linearise, prm, solve=solve, error=error if use_error else None)
    _, _, t = opt.run(np.tile([0, 0, 0, 1, 0, 0, 0.0], (2, 1)), np.zeros((2, 1)))
    return t


SCRIPTS = {
    # (energies consumed in order, solve infos): accepted steps, a rejection, a failed solve
    "mixed": ([10.0, 9.0, 9.5, 8.0, float("nan"), 7.5, 7.6, 7.0], [0, 0, 1, 0, 0, 0, 0, 0]),
    "all_rejected_until_overflow": ([5.0] + [6.0] * 20, [0] * 20),
    "failed_solves_until_overflow": ([5.0], [1] * 20),
    # lambda_init 1e-10: after two accepted steps lambda is at the 1e-12 floor (1e-10 * 0.1 * 0.1 rounds just above it),
    # and it stays there
    "accepted_down_to_the_floor": ([9.0, 8.0, 7.0, 6.0, 5.0, 4.0, 3.5, 3.0], [0] * 7),
}


@pytest.mark.parametrize("use_error", [False, True])
@pytest.mark.parametrize("script", sorted(SCRIPTS))
def test_host_lm_policy_matches_window_optimizer(driver, script, use_error):
    energies, infos = SCRIPTS[script]
    # error mode consumes no energy for the linearisation of an accepted point: the same script describes the same
    # sequence of candidate energies in both modes
    lam0 = 1e-10 if script == "accepted_down_to_the_floor" else 1e-4
    prm = LMParams(iterations=7, lambda_init=lam0, lambda_up=10.0, lambda_down=0.1, lambda_max=1e-1)
    got = run_driver(driver, prm, use_error, energies, infos)
    want = run_python(prm, use_error, energies, infos)
    if script == "accepted_down_to_the_floor":
        assert all(got["accepted"]) and min(got["lam"]) >= 1e-12 and got["lam"][3:] == [1e-12] * (len(got["lam"]) - 3)
    assert got["accepted"] == want.accepted
    assert got["lam"] == want.lam
    assert got["energy"] == want.energy
    assert got["linearisations"] == want.linearisations
    assert got["error_evaluations"] == want.error_evaluations
    if use_error:
        assert got["linearisations"] == 1 + sum(got["accepted"])


def test_host_lm_policy_call_order(driver):
    """a failed solve evaluates nothing; error mode linearises the start point and accepted candidates only"""
    prm = LMParams(iterations=3, lambda_init=1e-4, lambda_max=1e6)
    got = run_driver(driver, prm, False, [3.0, 2.0, 2.5], [0, 1, 0])
    assert got["log"] == "LE" + "SRLEA" + "S" + "SRLE"
    got = run_driver(driver, prm, True, [3.0, 2.0, 2.5], [0, 1, 0])
    assert got["log"] == "LE" + "SRELA" + "S" + "SRE"


def test_problem_slots_on_the_window_scene_layout():
    """the layout of test_gpu_window_error._window: 3 keyframes, pairs (0,1) (1,2) (2,0) (1,0), two reprojection
    links, three geometric links, a tracked frame on keyframe 1, 2 levels"""
    Link = namedtuple("Link", "k0 k1")
    K, L = 3, 2
    photometric = [(0, 1), (1, 2), (2, 0), (1, 0)]
    links = [Link(0, 2), Link(2, 1)]
    geo = [Link(0, 1), Link(1, 2), Link(2, 0)]
    pairs = photometric + [(ln.k0, ln.k1) for ln in links] + [(1, K + 0)]
    sl = problem_slots(K, L, pairs, len(photometric), links, geo)
    ends = photometric + [(1, 3)]
    assert sl["dense"] == [(a, b, a, -1) for a, b in ends for _ in range(L)]
    assert sl["dense"][-1] == (1, 3, 1, -1)  # the frame's pose is slot K + 0, its code the keyframe's
    assert all(s[2] < K for s in sl["dense"])  # never a frame slot as a code
    assert sl["reproj"] == [(0, 2, 0, -1), (2, 1, 2, -1)]
    assert sl["geo"] == [(0, 1, 0, 1), (1, 2, 1, 2), (2, 0, 2, 0)]
    assert sl["depth"] == [(-1, -1, k, -1) for k in range(K) for _ in range(L)]
    assert sl["error"] == [(a, b, -1, -1) for a, b, _, _ in sl["dense"]]
    assert sl["error_depth"] == [a * L + l for a, _ in ends for l in range(L)]
