#!/usr/bin/env python3
# coding: utf-8
"""Generate `tests/golden/check_verdicts.json`: whether the UNMODIFIED reference's `check()` accepts
(None) or rejects (a message) each rule's arguments on a grid of (n, f, extra keyword arguments), or
raises TypeError, for `tests/test_check_verdicts.py`.  Per rule one string, one letter per point of
`grid()` (a = accept, r = reject, t = TypeError).

    BYZ_REFERENCE=<reference checkout> python tests/golden/make_check_golden.py
"""

import json
import os
import pathlib
import sys

import torch

HERE = pathlib.Path(__file__).resolve().parent
OUT = HERE / "check_verdicts.json"
RULES = ("trmean", "phocas", "meamed", "krum", "bulyan", "brute", "aksel", "cge", "median", "average")
NS = (1, 3, 7, 11, 25)
FS = (0, 1, 2, 3, 5, 12, "x")
EXTRAS = ({}, {"m": 1}, {"m": 99}, {"mode": "n-f"}, {"mode": "zzz"})

def grid():
  return [(n, f, extra) for n in NS for f in FS for extra in EXTRAS]

def verdict(check, n, f, extra):
  """ "a" (accept), "r" (reject) or "t" (TypeError) for check(gradients=<n zero rows of 4>, f=f, **extra). """
  try:
    return "a" if check(gradients=[torch.zeros(4) for _ in range(n)], f=f, **extra) is None else "r"
  except TypeError:
    return "t"

def main():
  sys.path.insert(0, os.environ["BYZ_REFERENCE"])
  saved = sys.stdout, sys.stderr, sys.excepthook
  import aggregators  # wraps stdout/stderr at import (tools/__init__.py:215-216,246)
  sys.stdout, sys.stderr, sys.excepthook = saved
  out = {rule: "".join(verdict(aggregators.gars[rule].check, *point) for point in grid()) for rule in RULES}
  OUT.write_text(json.dumps(out, indent=1) + "\n")

if __name__ == "__main__":
  main()
