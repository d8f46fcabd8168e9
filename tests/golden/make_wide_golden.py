#!/usr/bin/env python3
# coding: utf-8
"""Generate `tests/golden/wide/golden_wide_*.npz`: the outputs of the UNMODIFIED reference for the
coordinate-wise rules (average, median, trmean, phocas, meamed) on stacks of 65 to 128 rows, which
`bz_coordinate` accepts.  The distance rules are not recorded (they stop at 64 rows here, and the
reference's brute at n = 128 would never finish).  The inputs come from `make_golden.make_rows`,
the fixtures have the layout of `make_golden.py`'s, and they sit outside the top-level
`golden_*.npz` glob, so only the tests of `bz_coordinate` read them:

    BYZ_REFERENCE=<reference checkout> python tests/golden/make_wide_golden.py [case name ...]
"""

import json
import sys

import numpy as np
import torch

from make_golden import aggregators, make_rows, HERE

# (name, kind, n, Byzantine rows, d, seed, f list)
WIDE_CASES = [
  ("wide_iid_n65_d517", "iid", 65, 10, 517, 9101, [1, 16, 32]),          # smallest n; f up to the largest valid
  ("wide_empire_n100_d600", "empire", 100, 20, 600, 9102, [20, 30, 49]),
  ("wide_nan_n97_d300", "nan", 97, 24, 300, 9103, [24, 40]),
  ("wide_inf_n128_d640", "inf", 128, 20, 640, 9104, [1, 20, 63]),       # +-inf entries, n - 2f up to 126
  ("wide_quant_n80_d512", "quant", 80, 16, 512, 9105, [16, 39]),        # ties and -0
  ("wide_little_n111_d257", "little", 111, 25, 257, 9106, [25, 55]),
  ("wide_nearmax_n128_d160", "nearmax", 128, 0, 160, 9107, [10, 60]),   # sums that overflow
  ("wide_iid_n128_d31", "iid", 128, 0, 31, 9108, [1, 63]),              # d < 32: every column in ATen's tail block
]

def run_case(name, kind, n, nb, d, seed, fs):
  honest, byz = make_rows(kind, n, nb, d, seed)
  honests = [honest[i] for i in range(honest.shape[0])]
  attacks = [byz] * nb if nb else []
  rows = honests + attacks          # the Byzantine rows are ONE tensor object, as attacks/identical.py:86 makes them
  assert len(rows) == n
  out = {"rows": torch.stack(rows).numpy().copy()}
  calls = []
  def record(gar, params, tag):
    rule = aggregators.gars[gar]
    if rule.check(gradients=rows, **params) is not None:
      return
    entry = dict(gar=gar, params=params, tag=tag)
    out[tag + "/out"] = rule.unchecked(gradients=rows, **params).numpy().copy()
    if rule.influence is not None and nb > 0:
      entry["influence"] = float(rule.influence(honests, attacks, **params))
    calls.append(entry)
  record("average", {}, "average")
  record("median", {}, "median")
  for f in fs:
    for gar in ("trmean", "phocas", "meamed"):
      record(gar, dict(f=f), f"{gar}_f{f}")
  manifest = dict(name=name, kind=kind, n=n, nb_byz=nb, d=int(out["rows"].shape[1]), seed=seed, calls=calls,
                  torch=torch.__version__, numpy=np.__version__, threads=torch.get_num_threads())
  out["manifest"] = np.array(json.dumps(manifest))
  return out

def main(names=()):
  """ names: regenerate only the cases with these names (default: all). """
  torch.set_num_threads(1)  # thread-count independent results where ATen's order depends on it
  (HERE / "wide").mkdir(exist_ok=True)
  total = 0
  for case in WIDE_CASES:
    if names and case[0] not in names:
      continue
    data = run_case(*case)
    path = HERE / "wide" / f"golden_{case[0]}.npz"
    np.savez_compressed(path, **data)
    total += path.stat().st_size
    man = json.loads(str(data["manifest"]))
    print(f"{path.name}: {len(man['calls'])} calls, {path.stat().st_size / 1024:.0f} KiB")
  print(f"total {total / 1024:.0f} KiB")

if __name__ == "__main__":
  main(sys.argv[1:])
