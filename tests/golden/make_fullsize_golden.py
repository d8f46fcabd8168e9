#!/usr/bin/env python3
# coding: utf-8
"""Generate `tests/golden/fullsize_reference.npz`: the UNMODIFIED reference's outputs at
BASELINE.json's full sizes, for `tests/test_cuda_vs_reference_fullsize.py`.

    BYZ_REFERENCE=<reference checkout> python tests/golden/make_fullsize_golden.py

The inputs are not stored: `stack()` regenerates them from torch's CPU generator (the test
calls the same function).  A full output is 5-18 MB, so per output the fixture keeps
  <key>/sha256  digest of the whole output, NaN and -0.0 canonicalised (the bit-exact bars),
  <key>/sha256_body  the same for all but the trailing `d mod 32` columns (trmean's bar);
  <key>/sample  the output at `cols/<d>`, a fixed seeded sample of columns, followed by the
                trailing `d mod 32` columns (the tolerance bars and the trmean tail);
  <key>/influence  the rule's `influence()` on the honest / Byzantine split, where the test checks it;
  <case>/inputs_sha256  digest of the regenerated input rows, so that a host whose torch produces other
                rows is reported as such and not as a kernel mismatch.
"""

import hashlib
import json
import os
import pathlib
import sys

import numpy as np
import torch

HERE = pathlib.Path(__file__).resolve().parent
OUT = HERE / "fullsize_reference.npz"
SAMPLE = 1024

def stack(n, nb, d, seed, dist="empire"):
  """ Distribution B of SURVEY §8(d) (shared mean + per-worker noise scale, nb aliased Byzantine
  rows = -1.1 * mean(honest)) or A (i.i.d. N(0, 1), no Byzantine rows), as CPU rows; (rows, nh). """
  gen = torch.Generator().manual_seed(seed)
  nh = n - nb
  if dist == "iid":
    return [torch.randn(d, generator=gen) for _ in range(n)], nh
  mu = torch.randn(d, generator=gen)
  rows = [mu + (0.5 + i / max(nh - 1, 1)) * torch.randn(d, generator=gen) for i in range(nh)]
  if nb:
    rows += [torch.stack(rows).mean(dim=0).mul(-1.1)] * nb
  return rows, nh

def columns(d):
  """ The stored columns of a length-d output: a seeded sample, then the trailing d mod 32. """
  rng = np.random.default_rng(d)
  body = d - d % 32
  sample = np.sort(rng.choice(body, size=min(SAMPLE, body), replace=False))
  return np.concatenate([sample, np.arange(body, d)]).astype(np.int64)

def digest(values):
  """ sha256 of the fp32 values under value equality (every NaN alike, -0.0 == +0.0). """
  v = np.asarray(values, dtype=np.float32)
  v = np.where(np.isnan(v), np.float32("nan"), v) + np.float32(0.)
  return hashlib.sha256(np.ascontiguousarray(v).tobytes()).hexdigest()

# (case, n, nb, f, d, seed, dist, [(rule, kwargs), ...], influence?)
CASES = []
for dist in ("iid", "empire"):
  CASES.append((f"c1/{dist}", 11, 0 if dist == "iid" else 5, 5, 79_510, 11, dist, [("median", {})], False))
for dist, nb in (("iid", 0), ("empire", 10)):
  CASES.append((f"c2/{dist}", 25, nb, 10, 1_310_922, 12, dist,
                [("trmean", {}), ("median", {}), ("phocas", {}), ("meamed", {}), ("average", {})], False))
for dist, nb in (("empire", 5), ("iid", 0)):
  CASES.append((f"c3/{dist}", 25, nb, 5, 1_310_922, 13, dist,
                [("krum", {}), ("krum", dict(m=1)), ("aksel", {}), ("aksel", dict(mode="n-f")), ("cge", {}), ("bulyan", {})], nb > 0))
for dist, nb in (("empire", 3), ("iid", 0)):
  CASES.append((f"c5/{dist}", 11, nb, 3, 1_310_922, 15, dist, [("brute", {})], nb > 0))
CASES.append(("c4/empire", 51, 12, 12, 36_546_980 // 8, 14, "empire", [("trmean", {}), ("median", {})], False))

def key(case, rule, kwargs):
  return "/".join([case, rule] + [f"{k}={v}" for k, v in sorted(kwargs.items())])

def main():
  ref = os.environ.get("BYZ_REFERENCE")
  if not ref:
    raise SystemExit("set BYZ_REFERENCE to a checkout of the reference")
  sys.path.insert(0, ref)
  saved = sys.stdout, sys.stderr, sys.excepthook
  import aggregators  # wraps stdout/stderr at import (tools/__init__.py:215-216,246)
  sys.stdout, sys.stderr, sys.excepthook = saved
  out = {}
  for case, n, nb, f, d, seed, dist, rules, influence in CASES:
    rows, nh = stack(n, nb, d, seed, dist)
    cols = columns(d)
    out[f"cols/{d}"] = cols
    out[f"{case}/inputs_sha256"] = np.array(digest(torch.stack(rows).numpy()))
    for rule, kwargs in rules:
      want = aggregators.gars[rule].unchecked(gradients=rows, f=f, **kwargs).numpy()
      k = key(case, rule, kwargs)
      out[k + "/sha256"] = np.array(digest(want))
      out[k + "/sha256_body"] = np.array(digest(want[:d - d % 32]))
      out[k + "/sample"] = want[cols].astype(np.float32)
      if influence and rule != "bulyan":
        out[k + "/influence"] = np.array(float(aggregators.gars[rule].influence(rows[:nh], rows[nh:], f=f, **kwargs)))
      print(k, out[k + "/sha256"], flush=True)
  out["manifest"] = np.array(json.dumps(dict(torch=torch.__version__, numpy=np.__version__, threads=torch.get_num_threads())))
  np.savez_compressed(OUT, **out)

if __name__ == "__main__":
  main()
