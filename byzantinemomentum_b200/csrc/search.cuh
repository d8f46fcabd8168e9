// search.cuh — the transition of the attacks' line search, shared by the score pass of the single-GPU
// search (K2' in SEARCH mode, k2_rowdist.cu) and the step of the d-sharded search (K9, k9_search_step.cu).
#pragma once

#include "dist.cuh"

namespace bz {

// One transition of `line_maximize` (tools/misc.py:468-513, start = 0, delta = 1, ratio = 0.8) after the
// evaluation of x = state->next_x scored y: the Python statements in the same order, in fp64 with
// explicit rounding (no contraction).  NaN never compares greater, as in Python.
__device__ inline void search_step(const SearchTail& s, const double y) {
  SearchState* st = s.state;
  const double x = st->next_x;
  s.trace[2 * s.k] = x;
  s.trace[2 * s.k + 1] = y;
  int32_t code = s.k == 0 ? 0 : *s.status;
  if (code == 0 && s.eval_status != nullptr) code = *s.eval_status;
  *s.status = code;
  double best_x, best_y, delta, prop_x = x;
  int phase;
  if (s.k == 0) {                       // best_x = start; best_y = scape(best_x)
    best_x = x; best_y = y; delta = 1.; phase = 1;
  } else {
    best_x = st->best_x; best_y = st->best_y; delta = st->delta; phase = st->phase;
    if (phase == 1) {                   // expansion
      if (y > best_y) { best_y = y; best_x = prop_x; delta = __dmul_rn(delta, 2.); }
      else            { delta = __dmul_rn(delta, 0.8); phase = 2; }
    } else {                            // contraction
      if (y > best_y) { best_y = y; best_x = prop_x; }
      delta = __dmul_rn(delta, 0.8);
    }
  }
  // the x the next evaluation (if any) takes
  if (phase == 1) {
    prop_x = __dadd_rn(best_x, delta);
  } else if (prop_x < best_x) {
    prop_x = __dadd_rn(prop_x, delta);
  } else {
    double t = __dsub_rn(prop_x, delta);
    while (t < 0.) t = __ddiv_rn(__dadd_rn(t, prop_x), 2.);
    prop_x = t;
  }
  st->best_x = best_x; st->best_y = best_y; st->delta = delta; st->prop_x = prop_x; st->phase = phase;
  st->next_x = prop_x;
  if (s.k == s.evals - 1) s.trace[2 * s.evals] = best_x;
}

}  // namespace bz
