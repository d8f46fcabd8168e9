# coding: utf-8
"""The rules' `check()` accepts and rejects exactly what the reference's own `check()` does, on the
grid of (rule, n, f, extra keyword arguments) recorded in `tests/golden/check_verdicts.json` by
`tests/golden/make_check_golden.py` (the reference's wrapper raises its UserException on a
rejection, so a different verdict changes what attack.py accepts)."""

import json
import sys

import conftest

sys.path.insert(0, str(conftest.GOLDEN_DIR))
import make_check_golden as fixture  # noqa: E402

def test_check_verdicts_match_the_reference():
  import byzantinemomentum_b200 as bz
  recorded = json.loads((conftest.GOLDEN_DIR / "check_verdicts.json").read_text())
  assert sorted(recorded) == sorted(fixture.RULES)
  points = fixture.grid()
  differ = []
  for rule, verdicts in recorded.items():
    assert len(verdicts) == len(points), rule
    for (n, f, extra), want in zip(points, verdicts):
      got = fixture.verdict(bz.gars[rule].check, n, f, extra)
      if got != want:
        differ.append((rule, n, f, extra, want, got))
  assert not differ, differ[:10]
