// dfk_levels.h -- the coarse-to-fine policy of dfk_window_lm_levels, host-only C++ (no CUDA), the loop of
// window_opt.WindowOptimizer.run(schedule=...).  It moves every pair of the window through the reference's
// OptimizeWork counter (df_work.cpp:100-190, mapper.cpp:440-538) while running dfk_lm.h's accept / lambda rule:
//   - a pair's state is its position s, the number of steps it has taken (pair_steps_done at the start).  Level
//     num_levels - 1 is active for its first iters[num_levels - 1] + 1 steps, then each finer level l for iters[l] + 1
//     steps (the + 1: OptimizeWork::Update decrements before it tests).  After its schedule a pair stays at level 0,
//     or, with remove_after, becomes inactive (level -1);
//   - one step is one LM iteration, accepted or rejected: afterwards every active pair's s moves by one
//     (WorkManager::Update, once per mapping step);
//   - the stall rule, the LM analogue of SignalNoRelinearize: when lambda would exceed lambda_max, every pair above
//     level 0 jumps to the first step of its next finer level (a fresh level start) and lambda restarts at
//     lambda_init.  Only when no pair is above level 0 does the run end there;
//   - when any pair's level changes between two steps, the accepted point is re-linearised under the new levels
//     (counted in linearisations; with use_error also its error()) and that energy becomes f: energies under different
//     levels are not comparable.  lambda carries over.  No switch follows the last step, so the levels in force on
//     return are the ones the last step used.
// `Ops` is dfk_lm.h's plus
//   DfkStatus set_levels(const int* level)       the active level of every pair (-1: none) becomes the item mask
#pragma once

#include <algorithm>
#include <climits>
#include <cmath>
#include <vector>

#include "dfk.h"

namespace dfk {

// the active level of a pair at position s (-1: inactive)
inline int level_at(const int32_t* iters, int num_levels, long long s, bool remove_after)
{
  for (int l = num_levels - 1; l >= 0; --l) {
    const long long span = (long long)iters[l] + 1;
    if (s < span) return l;
    s -= span;
  }
  return remove_after ? -1 : 0;
}

// the position of the first step at level l
inline long long level_start(const int32_t* iters, int num_levels, int l)
{
  long long s = 0;
  for (int m = num_levels - 1; m > l; --m) s += (long long)iters[m] + 1;
  return s;
}

template <class Ops>
DfkStatus lm_levels_run(const DfkLMParams& p, const DfkLevelSchedule& sc, Ops& ops, DfkLMTrace* tr, DfkLevelTrace* lt)
{
  tr->num_energies = tr->num_steps = tr->linearisations = tr->error_evaluations = 0;
  if (lt) lt->num_switches = 0;
  const int P = sc.num_pairs, L = sc.num_levels;
  const bool err = p.use_error != 0;
  std::vector<long long> pos(sc.pair_steps_done, sc.pair_steps_done + P);
  std::vector<int> lvl(P), next(P);
  auto levels = [&](std::vector<int>& out) {
    for (int q = 0; q < P; ++q)
      out[q] = level_at(sc.iters, L, pos[q], sc.pair_remove_after && sc.pair_remove_after[q]);
  };
  // the accepted point under the current levels: linearised, and its energy f
  auto relinearize = [&](double* f) {
    DfkStatus s = ops.linearize(false);
    if (s != DFK_OK) return s;
    tr->linearisations += 1;
    if ((s = ops.energy(false, f)) != DFK_OK) return s;
    if (err) tr->error_evaluations += 1;
    return DFK_OK;
  };
  double lam = p.lambda_init, f = 0.0;
  levels(lvl);
  DfkStatus s = ops.set_levels(lvl.data());
  if (s != DFK_OK) return s;
  if ((s = relinearize(&f)) != DFK_OK) return s;
  tr->energy[tr->num_energies++] = f;
  for (int it = 0; it < p.iterations; ++it) {
    if (lt && lt->pair_levels) std::copy(lvl.begin(), lvl.end(), lt->pair_levels + (size_t)it * P);
    int info = 0;
    if ((s = ops.solve(lam, &info)) != DFK_OK) return s;
    tr->lambda[tr->num_steps] = lam;
    bool ok = false;
    double cf = 0.0;
    if (info == 0) {
      if ((s = ops.retract()) != DFK_OK) return s;
      if (!err) {
        if ((s = ops.linearize(true)) != DFK_OK) return s;
        tr->linearisations += 1;
      }
      if ((s = ops.energy(true, &cf)) != DFK_OK) return s;
      if (err) tr->error_evaluations += 1;
      ok = std::isfinite(cf) && cf < f;
    }
    tr->accepted[tr->num_steps++] = ok ? 1 : 0;
    if (ok) {
      if (err) {
        if ((s = ops.linearize(true)) != DFK_OK) return s;
        tr->linearisations += 1;
      }
      ops.accept();
      f = cf;
      tr->energy[tr->num_energies++] = f;
      lam = std::max(lam * p.lambda_down, 1e-12);
    } else {
      lam = lam * p.lambda_up;
    }
    for (int q = 0; q < P; ++q)
      if (lvl[q] >= 0) pos[q] += 1;
    if (!ok && lam > p.lambda_max) {  // stall: every pair above level 0 moves one level finer
      bool moved = false;
      for (int q = 0; q < P; ++q) {
        const int l = level_at(sc.iters, L, pos[q], sc.pair_remove_after && sc.pair_remove_after[q]);
        if (l > 0) {
          pos[q] = level_start(sc.iters, L, l - 1);
          moved = true;
        }
      }
      if (!moved) break;
      lam = p.lambda_init;
    }
    if (it + 1 == p.iterations) break;
    levels(next);
    if (next != lvl) {
      lvl = next;
      if ((s = ops.set_levels(lvl.data())) != DFK_OK) return s;
      if ((s = relinearize(&f)) != DFK_OK) return s;
      if (lt && lt->switch_energy) lt->switch_energy[lt->num_switches] = f;
      if (lt) lt->num_switches += 1;
    }
  }
  if (lt && lt->pair_steps_done)
    for (int q = 0; q < P; ++q) lt->pair_steps_done[q] = (int32_t)std::min<long long>(pos[q], INT32_MAX);
  return DFK_OK;
}

}  // namespace dfk
