# coding: utf-8
"""Beyond the goldens of `tests/test_oracle_golden.py`: 21 further stacks of other shapes and seeds
(n = 9…40, d = 65…361; i.i.d. / empire / little / all-NaN rows / ±inf entries / heavily tied values),
whose reference outputs `tests/golden/make_golden.py` records under `tests/golden/live/`, checked
against the oracle with the same comparisons."""

import conftest
from test_oracle_golden import test_oracle_matches_reference as check_call

LIVE_DIR = conftest.GOLDEN_DIR / "live"

def test_oracle_matches_fresh_reference_outputs():
  paths = sorted(LIVE_DIR.glob("golden_live_*.npz"))
  assert len(paths) == 21, [p.name for p in paths]
  checked = 0
  for path in paths:
    golden = conftest.Golden(path)
    for call in golden.calls:
      check_call(golden, call)
      checked += 1
  assert checked > 450, checked
