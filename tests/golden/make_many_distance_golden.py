#!/usr/bin/env python3
# coding: utf-8
"""Generate `tests/golden/many_distance/golden_md_*.npz`: the outputs and selections of the UNMODIFIED reference for
the distance rules `bz_distance_many` takes above 128 rows — Multi-Krum (several m), Bulyan (including a degenerate
NaN case that raises), Aksel (both modes) and CGE — on stacks of 129 to 1024 rows.  The calls, the fixtures' layout,
the MIN_MARGIN rule and the determined ties are those of `make_wide_distance_golden.py` (its `run_case`), and the
inputs come from `make_golden.make_rows`; only the stacks differ.  The fixtures sit in their own directory:

    BYZ_REFERENCE=<reference checkout> python tests/golden/make_many_distance_golden.py [case name ...]

The reference computes its n(n-1)/2 distances one `sub().norm().item()` at a time (5.3 s for Multi-Krum at n = 1024,
d = 130 on one CPU core), so the large stacks record one f each and the whole run takes minutes.
"""

import json
import sys

import numpy as np
import torch

from make_golden import HERE
from make_wide_distance_golden import run_case

OUT_DIR = HERE / "many_distance"

# (name, kind, n, Byzantine rows, d, seed, f list); Bulyan needs n >= 4f + 3, f = (n - 3) // 4 is its smallest theta
MD_CASES = [
  ("md_iid_n129_d256", "iid", 129, 0, 256, 9301, [31]),                # no alias (u = n); theta = 65
  ("md_empire_n200_d200", "empire", 200, 40, 200, 9302, [40]),
  ("md_little_n256_d200", "little", 256, 50, 200, 9303, [50, 63]),     # f = 63: theta = 128
  ("md_nan_n257_d160", "nan", 257, 60, 160, 9304, [30]),               # NaN Byzantine rows; f < 60: Bulyan raises
  ("md_inf_n511_d128", "inf", 511, 100, 128, 9305, [100]),
  ("md_quant_n512_d128", "quant", 512, 100, 128, 9306, [100]),         # exact ties between distances
  ("md_tiny80_n777_d120", "tiny80", 777, 150, 120, 9307, [150]),       # every key exactly 0
  ("md_nearmax_n1024_d100", "nearmax", 1024, 255, 100, 9308, [255]),   # every key +inf; theta = 512
]

def main(names=()):
  """ names: regenerate only the cases with these names (default: all). """
  torch.set_num_threads(1)  # thread-count independent results where ATen's order depends on it
  OUT_DIR.mkdir(exist_ok=True)
  total = 0
  for case in MD_CASES:
    if names and case[0] not in names:
      continue
    data = run_case(*case)
    path = OUT_DIR / f"golden_{case[0]}.npz"
    np.savez_compressed(path, **data)
    total += path.stat().st_size
    man = json.loads(str(data["manifest"]))
    print(f"{path.name}: {len(man['calls'])} calls, {path.stat().st_size / 1024:.0f} KiB", flush=True)
  print(f"total {total / 1024:.0f} KiB")

if __name__ == "__main__":
  main(sys.argv[1:])
