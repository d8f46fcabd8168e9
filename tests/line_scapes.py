# coding: utf-8
"""Scripted score landscapes for the attacks' line search: y_k = scape(k, x_k, evals) for the k-th call of
`line_maximize` (x_k the factor it evaluates, `evals` its budget).  Data only: tests/test_linesearch_oracle.py
runs them through tests/line_oracle.py and the reference's `tools.line_maximize`, and
tests/test_cuda_search_transition.py feeds them to the device transition (`bz_search_step`).

They reach the branches smooth scores do not: exact ties (`y == best_y` does not improve), NaN before,
between and after finite scores, +inf and -inf, -0.0 against +0.0, expansion to the end of the budget
(x = 2^(evals - 1) - 1, past 2^53 at 64 evaluations), long runs of the halving `while x < 0`, fp32
subnormals, FLT_MAX and the sums around fp32's overflow, and increments below one fp32 ulp, which only
tie once y is rounded to fp32."""

import math
import random

NAN, INF = math.nan, math.inf
FLT_MAX = float.fromhex("0x1.fffffep+127")
FLT_TRUE_MIN = float.fromhex("0x1p-149")           # smallest fp32 subnormal
FLT_MIN = float.fromhex("0x1p-126")                # smallest fp32 normal
FLT_INF_EDGE = float.fromhex("0x1.ffffffp+127")    # FLT_MAX + ulp / 2: fl32 rounds it (a tie, to even) to inf

EVALS = list(range(1, 41)) + [64, 200]

def _draws(values, seed, count=256):
  gen = random.Random(seed)
  return [gen.choice(values) for _ in range(count)]

def _gauss(seed, count=256):
  gen = random.Random(seed)
  return [gen.gauss(0., 1.) * 2. ** gen.randint(-20, 20) for _ in range(count)]

_FEW = _draws([0., 1., 2., -1.], 1)
_FEW_ZEROS = _draws([0., -0., FLT_TRUE_MIN, -FLT_TRUE_MIN], 2)
_FEW_EDGES = _draws([FLT_MAX, INF, -INF, NAN, 0., -FLT_MAX], 3)
_RANDOM = _gauss(4)

SCAPES = [
  # expansion to the end of the budget: every call improves
  ("increasing", lambda k, x, evals: float(k)),
  # y = x: improves until fl32(x) reaches inf (x > FLT_MAX, 200 evaluations), then inf ties with inf
  ("increasing-x", lambda k, x, evals: x),
  # improvements below one fp32 ulp of 1: the same fl32 score, so a tie from the second call on
  ("increasing-sub-ulp", lambda k, x, evals: 1. + k * 2. ** -40),
  # fp64 subnormals: fl32 rounds them to +0.0, a tie with the start
  ("increasing-fp64-subnormal", lambda k, x, evals: k * 5e-324),
  # the best x stays 0: x shrinks toward it, the halving loop running about twice per call more
  ("decreasing", lambda k, x, evals: -x),
  ("plateau", lambda k, x, evals: 1.),
  ("plateau-zero", lambda k, x, evals: 0.),
  ("alternating", lambda k, x, evals: (3., 5.)[k % 2]),
  ("alternating-nan", lambda k, x, evals: (2., NAN)[k % 2]),
  # a single interior maximum
  ("unimodal", lambda k, x, evals: -(x - 5.3) ** 2),
  ("few-values", lambda k, x, evals: _FEW[k]),
  ("random", lambda k, x, evals: _RANDOM[k]),
  ("nan-first", lambda k, x, evals: NAN if k == 0 else float(k)),
  ("nan-middle", lambda k, x, evals: NAN if k == evals // 2 else float(k)),
  ("nan-last", lambda k, x, evals: NAN if k == evals - 1 else float(k)),
  ("all-nan", lambda k, x, evals: NAN),
  ("inf-second", lambda k, x, evals: INF if k == 1 else float(k)),
  ("inf-first", lambda k, x, evals: INF if k == 0 else float(k)),
  ("all-inf", lambda k, x, evals: INF),
  ("minus-inf-first", lambda k, x, evals: -INF if k == 0 else -float(k)),
  ("all-minus-inf", lambda k, x, evals: -INF),
  # -0.0 and +0.0 compare equal: neither improves on the other
  ("minus-zero-then-zero", lambda k, x, evals: -0. if k == 0 else 0.),
  ("zero-then-minus-zero", lambda k, x, evals: 0. if k == 0 else -0.),
  ("zeros-and-subnormals", lambda k, x, evals: _FEW_ZEROS[k]),
  ("fp32-subnormals", lambda k, x, evals: k * FLT_TRUE_MIN if k < 8 else FLT_MIN - k * FLT_TRUE_MIN),
  # FLT_MAX, then sums that round to FLT_MAX (a tie) and to inf (an improvement)
  ("flt-max", lambda k, x, evals: (FLT_MAX, FLT_INF_EDGE - 2. ** 76, FLT_MAX, FLT_INF_EDGE, 2. ** 128)[k % 5]),
  ("edges", lambda k, x, evals: _FEW_EDGES[k]),
]
