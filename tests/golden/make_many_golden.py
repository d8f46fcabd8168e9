#!/usr/bin/env python3
# coding: utf-8
"""Generate `tests/golden/many/golden_many_*.npz`: the outputs of the UNMODIFIED reference for the
coordinate-wise rules (average, median, trmean, phocas, meamed) on stacks of 129 to 1024 rows, which
`bz_coordinate_many` accepts.  Modelled on `make_wide_golden.py`: the inputs come from
`make_golden.make_rows`, the fixtures have the layout of `make_golden.py`'s, and they sit outside the
top-level `golden_*.npz` glob, so only the tests of `bz_coordinate_many` read them.  Every stack records
the smallest f the reference accepts (1: its check rejects f = 0), a middle value and the largest f:

    BYZ_REFERENCE=<reference checkout> python tests/golden/make_many_golden.py [case name ...]
"""

import json
import sys

import numpy as np
import torch

from make_golden import aggregators, make_rows, HERE

# (name, kind, n, Byzantine rows, d, seed): n on both sides of the 256 / 512 bucket edges and at the limit
MANY_CASES = [
  ("many_iid_n129_d300", "iid", 129, 25, 300, 9201),            # one row past bz_coordinate
  ("many_nan_n200_d257", "nan", 200, 40, 257, 9202),
  ("many_inf_n256_d320", "inf", 256, 50, 320, 9203),            # +-inf entries; the largest n of the first bucket
  ("many_quant_n257_d200", "quant", 257, 51, 200, 9204),        # key ties and -0
  ("many_nearmax_n511_d170", "nearmax", 511, 0, 170, 9205),     # sums that overflow
  ("many_tiny_n512_d160", "tiny80", 512, 100, 160, 9206),       # magnitudes near 2^-80: products and sums far below 1
  ("many_iid_n777_d150", "iid", 777, 150, 150, 9207),
  ("many_nan_n1024_d130", "nan", 1024, 200, 130, 9208),         # BZ_MAX_N_MANY
]

def fs_of(n):
  return sorted({1, (n - 1) // 4, (n - 1) // 2})

def run_case(name, kind, n, nb, d, seed):
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
  for f in fs_of(n):
    for gar in ("trmean", "phocas", "meamed"):
      record(gar, dict(f=f), f"{gar}_f{f}")
  manifest = dict(name=name, kind=kind, n=n, nb_byz=nb, d=int(out["rows"].shape[1]), seed=seed, calls=calls,
                  torch=torch.__version__, numpy=np.__version__, threads=torch.get_num_threads())
  out["manifest"] = np.array(json.dumps(manifest))
  return out

def main(names=()):
  """ names: regenerate only the cases with these names (default: all). """
  torch.set_num_threads(1)  # thread-count independent results where ATen's order depends on it
  (HERE / "many").mkdir(exist_ok=True)
  total = 0
  for case in MANY_CASES:
    if names and case[0] not in names:
      continue
    data = run_case(*case)
    path = HERE / "many" / f"golden_{case[0]}.npz"
    np.savez_compressed(path, **data)
    total += path.stat().st_size
    man = json.loads(str(data["manifest"]))
    print(f"{path.name}: {len(man['calls'])} calls, {path.stat().st_size / 1024:.0f} KiB")
  print(f"total {total / 1024:.0f} KiB")

if __name__ == "__main__":
  main(sys.argv[1:])
