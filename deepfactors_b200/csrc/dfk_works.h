// dfk_works.h -- the per-pair work rule of dfk_window_map_steps, host-only C++ (no CUDA): the reference's
// OptimizeWork (df_work.cpp:100-190) as window_opt.OptimizeWork transliterates it, and the WorkManager around it
// (work_manager.cpp: Bookkeeping, Update, SignalNoRelinearize).  It is not dfk_levels.h's rule for the LM loop:
//   - a signal (SignalNoRelinearize: the mapping step relinearised nothing) lowers the active level by one and leaves
//     the counters alone, so a later level start is seen only when a counter is still at its initial value;
//   - a remove_after pair (the backward direction of a new connection) that runs out at level 0 marks itself removed at
//     that update and drops its factor at the next bookkeeping: one step later than the level schedule's -1;
//   - bookkeeping (the factor the pair holds) runs before the update (the counter), every mapping step.
// A work that has finished after an update is erased from the manager: it takes no more steps, but its factor stays in
// the graph.
#pragma once

#include "dfk.h"

namespace dfk {

// a fresh work of num_levels levels with counters iters
inline DfkWorkState work_fresh(const int32_t* iters, int num_levels)
{
  DfkWorkState w{};
  w.active_level = num_levels - 1;
  for (int l = 0; l < num_levels; ++l) w.iters[l] = iters[l];
  w.first = 1;
  w.factor = -1;
  return w;
}

inline bool work_finished(const DfkWorkState& w, bool remove_after) { return w.active_level == (remove_after ? -2 : -1); }

// OptimizeWork::Bookkeeping: the factor the pair holds afterwards (-1: none)
inline int work_bookkeeping(DfkWorkState& w, const int32_t* orig)
{
  if (w.remove) {
    w.factor = -1;
    w.active_level = -2;
  }
  const bool level_start = w.active_level >= 0 && w.iters[w.active_level] == orig[w.active_level];
  if (w.first || level_start) {
    w.first = 0;
    w.factor = w.active_level;
  }
  return w.factor;
}

// OptimizeWork::Update
inline void work_update(DfkWorkState& w, bool remove_after)
{
  if (w.active_level >= 0) {
    w.iters[w.active_level] -= 1;
    if (w.iters[w.active_level] < 0) w.active_level -= 1;
  }
  if (remove_after && w.active_level < 0) w.remove = 1;
}

// OptimizeWork::SignalNoRelinearize
inline void work_signal_no_relinearize(DfkWorkState& w)
{
  if (!w.first) w.active_level -= 1;
}

// One mapping step's work bookkeeping and update (WorkManager::Bookkeeping, then WorkManager::Update): the factor
// level of every pair into factor[] (erased works keep theirs); returns whether any work is left in the manager
inline bool works_step(DfkWorkState* w, int n, const int32_t* orig, const uint8_t* remove_after, int* factor)
{
  for (int q = 0; q < n; ++q)
    if (!w[q].erased) work_bookkeeping(w[q], orig);
  bool any = false;
  for (int q = 0; q < n; ++q) {
    const bool ra = remove_after && remove_after[q];
    if (!w[q].erased) {
      work_update(w[q], ra);
      if (work_finished(w[q], ra)) w[q].erased = 1;
    }
    factor[q] = w[q].factor;
    any = any || !w[q].erased;
  }
  return any;
}

// WorkManager::SignalNoRelinearize
inline void works_signal(DfkWorkState* w, int n)
{
  for (int q = 0; q < n; ++q)
    if (!w[q].erased) work_signal_no_relinearize(w[q]);
}

inline bool works_empty(const DfkWorkState* w, int n)
{
  for (int q = 0; q < n; ++q)
    if (!w[q].erased) return false;
  return true;
}

}  // namespace dfk
