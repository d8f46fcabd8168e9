# coding: utf-8
"""The restatement of `line_maximize` in tests/line_oracle.py against the reference's own
`tools.line_maximize` (tools/misc.py:468-513) on synthetic scapes: the same x sequence, bit for bit, and the same result.  The GPU tests of the
device search compare against it, since they cannot read the reference.  Runs only when
$BYZ_REFERENCE points at a reference checkout."""

import math
import sys

import pytest

import line_oracle
from oracle import reference

pytestmark = pytest.mark.skipif(reference.find_root() is None, reason="$BYZ_REFERENCE not set (live-reference test)")

def _scapes():
  nan = math.nan
  yield "monotone", lambda x: x
  yield "decreasing", lambda x: -x
  yield "unimodal", lambda x: -(x - 5.3) ** 2
  yield "unimodal-far", lambda x: -(x - 1234.5) ** 2
  yield "plateau", lambda x: 1.
  yield "nan", lambda x: nan
  yield "nan-late", lambda x: nan if x > 3 else x
  yield "nan-first", lambda x: nan if x == 0 else -abs(x - 2)
  yield "below-zero", lambda x: 1. if x == 0 else -x            # every step back from 1 would cross 0
  yield "spiky", lambda x: math.sin(7 * x) * x
  yield "fp32", lambda x: float(__import__("numpy").float32(-(x - 0.7) ** 2))

@pytest.mark.parametrize("evals", [1, 2, 3, 5, 16, 40])
def test_oracle_line_maximize_matches_the_reference(evals):
  reference.load()
  tools = sys.modules["tools"]
  for name, scape in _scapes():
    seen = {"ref": [], "orc": []}
    def traced(key):
      def f(x):
        seen[key].append(x)
        return scape(x)
      return f
    want = tools.line_maximize(traced("ref"), evals=evals)
    got = line_oracle.line_maximize(traced("orc"), evals=evals)
    assert len(seen["ref"]) == evals, name
    assert [x.hex() for x in map(float, seen["orc"])] == [x.hex() for x in map(float, seen["ref"])], (name, evals)
    assert float(got).hex() == float(want).hex(), (name, evals)
  # the contraction halves a step that would go below 0
  xs = []
  line_oracle.line_maximize(lambda x: (xs.append(x), 1. if x == 0 else -x)[1], evals=16)
  assert min(xs) >= 0 and all(x >= 0 for x in xs)
