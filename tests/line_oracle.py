# coding: utf-8
"""Restatement of the reference's `tools.line_maximize` (tools/misc.py:468-513), the attacks' factor
search, written from scratch.  TEST INFRASTRUCTURE ONLY: the GPU tests of the device search
(`tests/test_cuda_linesearch.py`) cannot read the reference, so they compare against this;
`tests/test_linesearch_oracle.py` pins it against the reference's own function when $BYZ_REFERENCE
is set."""

def line_maximize(scape, evals=16, start=0., delta=1., ratio=0.8):
  """ Best-effort arg-max of `scape` over x >= 0 with exactly `evals` calls: x = start first, then
  steps of `delta` away from the best x, doubled after every improvement, until one fails; from then
  on steps toward the best x or back, shrunk by `ratio` after every call, halved toward the last x
  while they would go below 0.  Python floats throughout; a NaN score never compares greater. """
  best_x = start
  best_y = scape(best_x)
  left = evals - 1
  expanding = True
  prop_x = best_x
  while left > 0:
    if expanding:
      prop_x = best_x + delta
    elif prop_x < best_x:
      prop_x = prop_x + delta
    else:
      x = prop_x - delta
      while x < 0:
        x = (x + prop_x) / 2
      prop_x = x
    prop_y = scape(prop_x)
    left -= 1
    if prop_y > best_y:
      best_x, best_y = prop_x, prop_y
      if expanding:
        delta = delta * 2
        continue
    if expanding:
      expanding = False
    delta = delta * ratio
  return best_x
