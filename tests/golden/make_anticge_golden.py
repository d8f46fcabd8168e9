#!/usr/bin/env python3
# coding: utf-8
"""Generate `tests/golden/anticge/anticge_*.npz`: the outputs of the UNMODIFIED reference attack against CGE
(attacks/anticge.py) on seeded stacks of honest rows, CPU torch:

    BYZ_REFERENCE=<reference checkout> python tests/golden/make_anticge_golden.py [case name ...]

Each fixture holds the [nh, d] fp32 honest rows, f_decl and f_real, how many rows the attack returned and
whether they are one tensor object, the row itself (empty when f_real = 0), and, when the attack ranks the rows,
the order it ranked them in (by object identity from `_compute_normed`), their norms in that order and the
unscaled sum `clone(σ0)` + `add_` over normed[:maxpos], restated from the attack's own statements.  A ranked
case is only recorded when the norms stay apart (relative gap >= MIN_GAP) around every position the attack reads:
the device ranks by the fp32 rounding of fp64 sums, ATen by its own fp32 sums.
"""

import json
import os
import pathlib
import sys

import numpy as np
import torch

REF = os.environ["BYZ_REFERENCE"]
sys.path.insert(0, REF)
_stdout, _stderr, _hook = sys.stdout, sys.stderr, sys.excepthook
import attacks  # noqa: E402  (wraps stdout/stderr at import, like the aggregators package)
sys.stdout, sys.stderr, sys.excepthook = _stdout, _stderr, _hook
anticge = sys.modules["attacks.anticge"]

HERE = pathlib.Path(__file__).resolve().parent
OUT_DIR = HERE / "anticge"
MIN_GAP = 1e-5

def rows_of(kind, nh, d, seed):
  gen = torch.Generator().manual_seed(seed)
  if kind == "zero":
    return torch.zeros(nh, d)
  rows = torch.randn(nh, d, generator=gen) * (0.5 + torch.rand(nh, 1, generator=gen))
  if kind == "nan":
    rows[nh // 3, d // 2] = float("nan")
  elif kind == "inf":
    rows[nh // 2, 3] = float("inf")
    rows[1, 0] = -float("inf")
  elif kind == "overflow":
    # every row's norm finite (~1e18), the attack's sum of squares past FLT_MAX: attnorm = inf
    scale = 1e18 * (1. + torch.arange(nh, dtype=torch.float32)[:, None] / nh)
    rows = rows.abs() * (scale / rows.abs().norm(dim=1, keepdim=True))
  return rows.contiguous()

# (name, kind, nh, d, seed, f_decl, f_real)
CASES = [
  ("n1", "iid", 1, 257, 8301, 1, 1),                    # maxpos = 0: σ0 alone
  ("n7", "iid", 7, 257, 8302, 2, 2),
  ("n25", "iid", 25, 513, 8303, 5, 5),
  ("n25_maxpos0", "iid", 25, 300, 8304, 25, 3),
  ("n25_fill", "iid", 25, 129, 8305, 3, 4),               # f_real > f_decl: NaN
  ("n25_freal0", "iid", 25, 129, 8306, 5, 0),             # []
  ("n25_nan", "nan", 25, 257, 8307, 6, 6),                # a NaN row ranks last (+inf)
  ("n25_inf", "inf", 25, 257, 8308, 6, 2),                # two +-inf rows: +inf keys, stable among themselves
  ("n25_zero", "zero", 25, 100, 8309, 5, 5),              # attnorm = 0: no scaling
  ("n25_overflow", "overflow", 25, 64, 8310, 5, 5),       # attnorm = inf: scaled by -0
  ("n64", "iid", 64, 257, 8311, 16, 16),
  ("n65", "iid", 65, 257, 8312, 16, 16),
  ("n100", "iid", 100, 200, 8313, 24, 24),
  ("n128", "iid", 128, 160, 8314, 31, 31),
  ("n128_maxpos127", "iid", 128, 64, 8316, 1, 1),
]

def gaps_ok(keys, maxpos):
  """ The ranked norms apart around the positions the attack reads (the first maxpos + 1), exact ties (zero rows,
  infinities: the stable order decides) aside. """
  for a, b in zip(keys[:maxpos + 1], keys[1:maxpos + 2]):
    if a != b and np.isfinite(b) and (b - a) / max(abs(b), 1e-300) < MIN_GAP:
      return False
  return True

def run_case(name, kind, nh, d, seed, f_decl, f_real):
  stack = rows_of(kind, nh, d, seed)
  honests = [stack[i].clone() for i in range(nh)]
  out = anticge.attack(honests, f_decl, f_real)
  data = dict(rows=stack.numpy(), f_decl=np.int64(f_decl), f_real=np.int64(f_real), count=np.int64(len(out)),
              aliased=np.int64(all(o is out[0] for o in out)), out=(out[0].numpy() if out else np.zeros(0, np.float32)))
  if f_real <= f_decl:
    normed = anticge._compute_normed(honests)
    order = [next(i for i, h in enumerate(honests) if h is grad) for _, grad in normed]
    keys = [norm for norm, _ in normed]
    maxpos = nh - f_decl
    if not gaps_ok(keys, maxpos):
      raise RuntimeError(f"{name}: norms within {MIN_GAP} of each other; pick another seed")
    presum = normed[0][1].clone().detach_()
    for _, grad in normed[:maxpos]:
      presum.add_(grad)
    data.update(order=np.asarray(order, np.int64), norms=np.asarray(keys, np.float64), presum=presum.numpy())
  manifest = dict(name=name, kind=kind, nh=nh, d=d, seed=seed, torch=torch.__version__, numpy=np.__version__,
                  threads=torch.get_num_threads())
  OUT_DIR.mkdir(exist_ok=True)
  np.savez_compressed(OUT_DIR / f"anticge_{name}.npz", manifest=json.dumps(manifest), **data)
  print(name, "ok")

if __name__ == "__main__":
  wanted = set(sys.argv[1:])
  for case in CASES:
    if not wanted or case[0] in wanted:
      run_case(*case)
