"""CPU tests of the mapper's ISAM2 steps with coarse-to-fine works: window_opt.mapping_steps (IncrementalOptimizer +
OptimizeWork + set_active) against a transliteration of Mapper::MappingStep and WorkManager written here, on a fake
problem, and dfk_works.h's state machine (the rule of dfk_window_map_steps) against OptimizeWork."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from deepfactors_b200.factors import WindowBlocks
from deepfactors_b200.window_opt import IncrementalOptimizer, LevelSchedule, OptimizeWork, mapping_steps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS, LEVELS = 4, 3
B = 6 + CS


class FakeProblem:
    """P photometric pairs of LEVELS items each; set_active records the masks; linearise records `todo`; solve returns
    a scripted delta per step (a big one relinearises keyframe 1's pose, so its pairs become stale)"""

    def __init__(self, K, pairs, big_steps=()):
        self.layout = WindowBlocks(K, CS, pairs)
        self.pairs = list(pairs)
        self.masks, self.todos = [], []
        self.big_steps = set(big_steps)
        self.step = 0

    def level_schedule(self, iters):
        n = len(self.pairs)
        return LevelSchedule(iters=list(iters), item_level=[l for _ in range(n) for l in range(LEVELS)],
                             item_pair=[q for q in range(n) for _ in range(LEVELS)], steps_done=[0] * n,
                             remove_after=[False] * n)

    def dense_pairs(self):
        return list(range(len(self.pairs)))

    def set_active(self, mask, error_mask=None):
        self.masks.append(np.asarray(mask, bool).copy())

    def linearise(self, poses, codes, todo, frame_poses=None):
        self.todos.append(sorted(todo))
        buf = np.zeros(self.layout.floats, np.float32)
        K = self.layout.num_keyframes
        buf[:K * B * B].reshape(K, B, B)[:] = np.eye(B, dtype=np.float32)
        return buf, None

    def solve(self, buf, eps, codes):
        d = np.zeros(self.layout.dim)
        if self.step in self.big_steps:
            d[B + 2] = 0.1  # keyframe 1's pose: relinearised at the next update
        self.step += 1
        return d, 0


# ------------------------------------------------------------------------- the reference, transliterated here
class RefWork:
    """OptimizeWork<Scalar> of df_work.cpp:100-190 for one pair: Bookkeeping / Update / SignalNoRelinearize /
    Finished, the factor it holds (its level, None: none)"""

    def __init__(self, iters, remove_after):
        self.orig, self.left = list(iters), list(iters)
        self.active, self.first, self.rm, self.ra = len(iters) - 1, True, False, remove_after
        self.factor = None

    def bookkeeping(self):
        if self.rm:
            self.factor, self.active = None, -2
        if self.first or (self.active >= 0 and self.left[self.active] == self.orig[self.active]):
            self.first, self.factor = False, self.active

    def update(self):
        if self.active >= 0:
            self.left[self.active] -= 1
            if self.left[self.active] < 0:
                self.active -= 1
        if self.ra and self.active < 0:
            self.rm = True

    def signal(self):
        if not self.first:
            self.active -= 1

    def finished(self):
        return self.active == (-2 if self.ra else -1)


def reference_run(pairs, iters, remove_after, big_steps, steps, added=()):
    """MappingStep (mapper.cpp:449-552) with WorkManager (work_manager.cpp: Bookkeeping, Update erasing finished works,
    SignalNoRelinearize) over the fake problem's rule: per step the factors present, the re-linearised pairs, whether
    the works were signalled, and whether work is left.  added = (step, pair) works that join before that step."""
    works = {q: RefWork(iters, remove_after[q]) for q in range(len(pairs)) if all(q != a for _, a in added)}
    graph, lin, moved_next, out = {}, {}, False, []
    for s in range(steps):
        for at, q in added:
            if at == s:
                works[q] = RefWork(iters, remove_after[q])
        if not works:
            break
        for w in works.values():
            w.bookkeeping()
        for q in list(works):
            works[q].update()
            if works[q].finished():
                graph[q] = works[q].factor
                del works[q]
        for q, w in works.items():
            graph[q] = w.factor
        present = {q: f for q, f in graph.items() if f is not None}
        # ISAM2::update: a new factor and every factor on a relinearised key (keyframe 1's pose) are linearised; the
        # window holds every pair from the start, so a pair without a work yet is linearised (to nothing) once
        todo = sorted(q for q in range(len(pairs))
                      if q not in lin or graph.get(q) != lin[q] or (moved_next and 1 in pairs[q]))
        for q in range(len(pairs)):
            lin[q] = graph.get(q)
        signalled = not moved_next
        if signalled:
            for w in works.values():
                w.signal()
        moved_next = s in big_steps
        out.append((present, todo, signalled, bool(works)))
    return out


def host_run(pairs, iters, remove_after, big_steps, steps, added=(), calls=(None,)):
    """mapping_steps on the fake problem, in one call or split at the steps in `calls`"""
    prob = FakeProblem(3, pairs, big_steps)
    opt = IncrementalOptimizer(prob.layout, prob.linearise, prob.solve, np.tile([0, 0, 0, 1.0, 0, 0, 0], (3, 1)),
                               np.zeros((3, CS)))
    works = [OptimizeWork(iters, remove_after[q]) for q in range(len(pairs))]
    late = {q for _, q in added}
    for q in late:
        works[q].erased = True  # not in the manager yet
    out, done = [], 0
    bounds = sorted({b for b in calls if b is not None} | {a for a, _ in added} | {steps})
    for b in bounds:
        for at, q in added:
            if at == done:
                works[q] = OptimizeWork(iters, remove_after[q])
        res, lv = mapping_steps(opt, prob, works, b - done)
        for r, levels in zip(res, lv):
            present = {q: f for q, f in enumerate(levels) if f >= 0}
            out.append((present, prob.todos[len(out)], r.variables_relinearized == 0, None, levels))
        if len(res) < b - done:  # the work manager ran empty
            break
        done = b
    return out, prob, works


def compare(pairs, iters, remove_after, big_steps, steps, added=(), calls=(None,)):
    ref = reference_run(pairs, iters, remove_after, big_steps, steps, added)
    got, prob, works = host_run(pairs, iters, remove_after, big_steps, steps, added, calls)
    assert len(got) == len(ref)
    for s, (g, r) in enumerate(zip(got, ref)):
        assert g[0] == r[0], (s, g[0], r[0])
        assert g[1] == r[1], (s, g[1], r[1])
        assert g[2] == r[2], s
        # the masks are the factors' levels
        want = np.array([g[4][q] == l for q in range(len(pairs)) for l in range(LEVELS)])
        assert np.array_equal(prob.masks[s], want), s
    assert all(w.erased for w in works) == (not ref[-1][3])
    return got, ref


PAIRS = [(0, 1), (1, 0), (1, 2), (2, 1)]


def test_a_level_switch_invalidates_exactly_that_pair():
    # keyframe 1's pose is relinearised after every step, so only the first step signals; pairs (0, 2) and (2, 0) do
    # not read keyframe 1: after the first step they are re-linearised exactly at their own level switches
    pairs = [(0, 1), (1, 0), (0, 2), (2, 0)]
    got, _ = compare(pairs, [2, 1, 1], [False, False, True, False], big_steps=set(range(40)), steps=12)
    switched = 0
    for s in range(1, len(got)):
        changed = {q for q in (2, 3) if got[s][4][q] != got[s - 1][4][q]}
        assert set(got[s][1]) & {2, 3} == changed, s
        assert {0, 1} <= set(got[s][1]), s
        switched += len(changed)
    assert switched >= 2


def test_remove_after_pair_signalled_at_level_zero_lags_one_step():
    got, ref = compare(PAIRS, [1, 0, 1], [False, True, False, True], big_steps=(), steps=20)
    # every step signals (nothing relinearised), so the works fall a level per step without a level start: the plain
    # pairs keep their level-1 factor when they finish; the remove_after pairs run out with them, mark themselves
    # removed at that update and drop their factor one step later
    lv = [g[4] for g in got]
    assert lv[-2] == [1, 1, 1, 1] and lv[-1] == [1, -1, 1, -1] and not ref[-1][3]


def test_a_pair_finishing_by_count():
    got, ref = compare(PAIRS, [2, 2, 3], [False] * 4, big_steps=set(range(100)), steps=30)
    # every update after the first relinearises, so only the first step signals: level 2 ends after that one step,
    # then levels 1 and 0 run by count (iters + 1 steps each)
    assert not ref[-1][3] and len(got) == 1 + (2 + 1) + (2 + 1)


def test_works_added_between_runs_and_a_continued_call():
    added = ((3, 2), (5, 3))
    compare(PAIRS, [1, 2, 1], [False, False, True, True], big_steps={1, 4, 6}, steps=16, added=added)
    one, _, _ = host_run(PAIRS, [1, 2, 1], [False] * 4, {2, 5}, 14)
    split, _, _ = host_run(PAIRS, [1, 2, 1], [False] * 4, {2, 5}, 14, calls=(4, 9))
    assert [g[1:3] + (g[4],) for g in one] == [g[1:3] + (g[4],) for g in split]


# ------------------------------------------------------------------------------- dfk_works.h against OptimizeWork
# reads: L iters, remove_after, n, then n ops (0: one mapping step with a signal afterwards, 1: without); prints per
# step the factor level and the state after it
DRIVER = r"""
#include <cstdio>
#include "dfk_works.h"
int main() {
  int L, ra, n;
  if (scanf("%d", &L) != 1) return 2;
  int32_t it[DFK_MAX_WORK_LEVELS];
  for (int l = 0; l < L; ++l) if (scanf("%d", &it[l]) != 1) return 2;
  if (scanf("%d %d", &ra, &n) != 2) return 2;
  DfkWorkState w = dfk::work_fresh(it, L);
  uint8_t rem = (uint8_t)ra;
  for (int s = 0; s < n; ++s) {
    int op, f;
    if (scanf("%d", &op) != 1) return 2;
    if (dfk::works_empty(&w, 1)) { printf("E\n"); continue; }
    dfk::works_step(&w, 1, it, &rem, &f);
    if (op == 0) dfk::works_signal(&w, 1);
    printf("%d %d %d %d %d %d", f, w.active_level, w.first, w.remove, w.factor, w.erased);
    for (int l = 0; l < L; ++l) printf(" %d", w.iters[l]);
    printf("\n");
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def works_driver(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("works")
    (d / "drv.cpp").write_text(DRIVER)
    exe = d / "drv"
    subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), "-I",
                    os.path.join(ROOT, "deepfactors_b200", "csrc"), str(d / "drv.cpp"), "-o", str(exe)], check=True)
    return str(exe)


def python_works(iters, remove_after, ops):
    w = OptimizeWork(iters, remove_after)
    out = []
    for op in ops:
        if w.erased:
            out.append("E")
            continue
        w.bookkeeping()
        w.update()
        w.erased = w.finished()
        f = -1 if w.factor is None else w.factor
        if op == 0 and not w.erased:
            w.signal_no_relinearize()
        out.append(" ".join(str(int(v)) for v in [f, w.active_level, w.first, w.remove, f, w.erased] + w.iters))
    return out


@pytest.mark.parametrize("seed", range(6))
def test_works_header_is_optimize_work(works_driver, seed):
    rng = np.random.default_rng(seed)
    for trial in range(25):
        L = int(rng.integers(1, 5))
        iters = [int(v) for v in rng.integers(0, 5, L)]
        ra = bool(rng.uniform() < 0.5)
        ops = [int(rng.uniform() < 0.6) for _ in range(int(rng.integers(1, 30)))]
        inp = f"{L} {' '.join(map(str, iters))} {int(ra)} {len(ops)} {' '.join(map(str, ops))}\n"
        got = subprocess.run([works_driver], input=inp, capture_output=True, text=True, check=True).stdout.split("\n")
        assert got[:len(ops)] == python_works(iters, ra, ops), (seed, trial, inp)
