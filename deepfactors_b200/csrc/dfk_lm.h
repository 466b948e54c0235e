// dfk_lm.h -- the Levenberg-Marquardt policy of dfk_window_lm, host-only C++ (no CUDA), the loop of
// window_opt.WindowOptimizer.run:
//   - lambda starts at lambda_init; an accepted step multiplies it by lambda_down (floor 1e-12), a rejected one by
//     lambda_up, and the loop stops once it exceeds lambda_max;
//   - a step is accepted iff isfinite(cf) && cf < f;
//   - a failed solve (info != 0) is a rejected step with nothing evaluated;
//   - without use_error every candidate is linearised and its f is the linearisation's; with use_error the candidate's f
//     is its error() and only the start point and accepted candidates are linearised.
// `Ops` does the work (the device pipeline in dfk_api_window.cu, scripted values in the CPU test of this policy):
//   DfkStatus linearize(bool candidate)     linearise the accepted point (false) or the candidate (true)
//   DfkStatus energy(bool candidate, double* f)  f of the point just linearised (use_error = 0) or its error() (1)
//   DfkStatus solve(double lambda, int* info)    the damped step at the accepted point
//   DfkStatus retract()                          the candidate from the accepted point and the step
//   void accept()                                the candidate becomes the accepted point (state and buffer)
#pragma once

#include <algorithm>
#include <cmath>

#include "dfk.h"

namespace dfk {

template <class Ops>
DfkStatus lm_run(const DfkLMParams& p, Ops& ops, DfkLMTrace* tr)
{
  tr->num_energies = tr->num_steps = tr->linearisations = tr->error_evaluations = 0;
  const bool err = p.use_error != 0;
  double lam = p.lambda_init, f = 0.0;
  DfkStatus s = ops.linearize(false);
  if (s != DFK_OK) return s;
  tr->linearisations += 1;
  if ((s = ops.energy(false, &f)) != DFK_OK) return s;
  if (err) tr->error_evaluations += 1;
  tr->energy[tr->num_energies++] = f;
  for (int it = 0; it < p.iterations; ++it) {
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
      if (lam > p.lambda_max) break;
    }
  }
  return DFK_OK;
}

}  // namespace dfk
