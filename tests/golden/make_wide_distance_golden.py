#!/usr/bin/env python3
# coding: utf-8
"""Generate `tests/golden/wide_distance/golden_wd_*.npz`: the outputs and selections of the UNMODIFIED
reference for the distance rules `bz_distance` takes above 64 rows — Multi-Krum (several f and m), Bulyan,
Aksel (both modes) and CGE — on stacks of 65 to 128 rows.  Brute is not recorded: C(n, n - f) subsets are
out of reach at these n.  The inputs come from `make_golden.make_rows`, the fixtures have the layout of
`make_golden.py`'s, and they sit in their own directory, outside the `golden_*.npz` and
`wide/golden_wide_*.npz` globs:

    BYZ_REFERENCE=<reference checkout> python tests/golden/make_wide_distance_golden.py [case name ...]

A Multi-Krum, Aksel or CGE call is only recorded when the NumPy oracle's relative margin between the last
selected and the first rejected key is at least MIN_MARGIN (far above the noise of fp32 norms, DESIGN §2),
ties between the aliased Byzantine rows aside: a selection the device may legitimately order otherwise is
no fixture.  On a stack whose every entry is finite, an exact tie between two keys that are both 0 (every
square underflows) or both +inf (the sum of squares overflows) is determined: the stable sort keeps index
order, so such a call is recorded when the tie is there in the oracle's keys and in the reference's recorded
ones alike.  Stacks that hold +-inf or NaN entries keep the margin rule alone: their +inf keys come from
non-finite differences (inf - inf is NaN), a path these magnitude ties are not meant to pin.
"""

import json
import pathlib
import sys

import numpy as np
import torch

from make_golden import aggregators, make_rows, module, ident_index, HERE

sys.path.insert(0, str(pathlib.Path(__file__).resolve().parents[2]))
from oracle import byzoracle as orc  # noqa: E402

OUT_DIR = HERE / "wide_distance"
MIN_MARGIN = 1e-5

# (name, kind, n, Byzantine rows, d, seed, f list); Bulyan needs n >= 4f + 3
WD_CASES = [
  ("wd_iid_n65_d517", "iid", 65, 10, 517, 9201, [5, 15]),              # smallest n; f = 15: theta = 33
  ("wd_empire_n100_d600", "empire", 100, 20, 600, 9202, [20, 24]),
  ("wd_little_n111_d257", "little", 111, 25, 257, 9203, [25, 27]),
  ("wd_nan_n97_d300", "nan", 97, 24, 300, 9204, [24]),                  # NaN Byzantine rows: +inf scores
  ("wd_inf_n128_d640", "inf", 128, 20, 640, 9205, [1, 20, 31]),        # +-inf entries; f = 1: theta = 124
  ("wd_quant_n80_d512", "quant", 80, 16, 512, 9206, [16, 19]),         # exact ties between distances
  ("wd_iid_n128_d100", "iid", 128, 0, 100, 9207, [0, 31]),             # no alias; f = 0: theta = 126
  # the ends of the fp32 range (make_golden.make_rows); u unique rows on both sides of 64 and of 96
  ("wd_tiny80_n100_d200", "tiny80", 100, 20, 200, 9208, [10, 24]),     # u = 81; every key exactly 0
  ("wd_tiny110_n72_d211", "tiny110", 72, 10, 211, 9209, [10, 17]),     # u = 63: one pass; every key 0
  ("wd_huge_n128_d160", "huge", 128, 30, 160, 9210, [5, 31]),          # u = 99; every distance and norm +inf
  ("wd_mixed_n97_d900", "mixed", 97, 2, 900, 9211, [2, 23]),           # u = 96; pairs with a large row +inf
  ("wd_hugebyz_n65_d150", "hugebyz", 65, 10, 150, 9212, [10, 15]),     # u = 56; honest-Byzantine pairs +inf
  ("wd_nearmax_n128_d128", "nearmax", 128, 32, 128, 9213, [5, 31]),    # u = 97; every key +inf
]

def determined_tie(a, b):
  """ Two keys both exactly 0 or both +inf: the stable sorts of the reference and the device keep index order. """
  return a == b and (a == 0 or a == np.inf)

def margin_ok(scores, order, count, nh, ref_sorted, finite_rows):
  """ The gap after the `count` selected keys, ties between aliased rows (indices >= nh) aside; on a stack of
  finite entries (`finite_rows`), a determined tie counts when the reference's keys (`ref_sorted`, in its
  order) tie so there too. """
  keys = [scores[i] for i in order]
  if count >= len(keys):
    return True
  a, b = keys[count - 1], keys[count]
  if order[count - 1] >= nh and order[count] >= nh:
    return True
  if finite_rows and determined_tie(a, b):
    return determined_tie(ref_sorted[count - 1], ref_sorted[count])
  if not (np.isfinite(a) and np.isfinite(b)):
    return a != b
  return (b - a) / max(abs(b), 1e-300) >= MIN_MARGIN

def run_case(name, kind, n, nb, d, seed, fs):
  honest, byz = make_rows(kind, n, nb, d, seed)
  honests = [honest[i] for i in range(honest.shape[0])]
  attacks = [byz] * nb if nb else []
  rows = honests + attacks          # the Byzantine rows are ONE tensor object, as attacks/identical.py:86 makes them
  assert len(rows) == n
  out = {"rows": torch.stack(rows).numpy().copy()}
  np_rows = [out["rows"][i] for i in range(n)]
  nh = n - nb
  finite = bool(np.isfinite(out["rows"]).all())
  calls, skipped = [], []
  def record(gar, params, tag):
    rule = aggregators.gars[gar]
    if rule.check(gradients=rows, **params) is not None:
      return
    entry = dict(gar=gar, params=params, tag=tag)
    thin = False
    if gar == "krum":
      m = params.get("m") or (n - params["f"] - 2)
      scores = module("krum")._compute_scores(rows, params["f"], m)
      out[tag + "/order"] = np.array([ident_index(rows, g) for _, g in scores], dtype=np.int64)
      out[tag + "/scores"] = np.array([s for s, _ in scores], dtype=np.float64)
      _, info = orc.krum(np_rows, return_info=True, **params)
      thin = not margin_ok(info["scores"], info["order"], m, nh, out[tag + "/scores"], finite)
    elif gar == "aksel":
      dlist, c = module("aksel")._compute_distances(rows, params["f"], params.get("mode", "mid"))
      out[tag + "/order"] = np.array([i for i, _ in dlist], dtype=np.int64)
      out[tag + "/dists"] = np.array([x for _, x in dlist], dtype=np.float64)
      entry["c"] = c
      _, info = orc.aksel(np_rows, return_info=True, **params)
      thin = not (np.isnan(out[tag + "/dists"]).any() or margin_ok(info["distances"], info["order"], c, nh, out[tag + "/dists"], finite))
    elif gar == "cge":
      normed = module("cge")._compute_normed(rows)
      out[tag + "/order"] = np.array([ident_index(rows, g) for _, g in normed], dtype=np.int64)
      out[tag + "/norms"] = np.array([s for s, _ in normed], dtype=np.float64)
      _, info = orc.cge(np_rows, return_info=True, **params)
      thin = not margin_ok(info["norms"], info["order"], n - params["f"], nh, out[tag + "/norms"], finite)
    if thin:
      for key in [k for k in out if k.startswith(tag + "/")]:
        del out[key]
      skipped.append(tag)
      return
    try:
      res = rule.unchecked(gradients=rows, **params)
    except Exception as err:        # the reference itself fails on this input (a degenerate Bulyan)
      entry["raises"] = type(err).__name__
      calls.append(entry)
      return
    out[tag + "/out"] = res.numpy().copy()
    calls.append(entry)
  for f in fs:
    record("cge", dict(f=f), f"cge_f{f}")
    for mode in ("mid", "n-f"):
      record("aksel", dict(f=f, mode=mode), f"aksel_f{f}_{mode}")
    m_max = n - f - 2
    for m in sorted({None, 1, max(1, m_max // 2)}, key=lambda x: -1 if x is None else x):
      params = dict(f=f) if m is None else dict(f=f, m=m)
      suffix = "" if m is None else f"_m{m}"
      record("krum", params, f"krum_f{f}{suffix}")
      record("bulyan", params, f"bulyan_f{f}{suffix}")
  manifest = dict(name=name, kind=kind, n=n, nb_byz=nb, d=int(out["rows"].shape[1]), seed=seed, calls=calls, thin_margin_skipped=skipped,
                  torch=torch.__version__, numpy=np.__version__, threads=torch.get_num_threads())
  out["manifest"] = np.array(json.dumps(manifest))
  return out

def main(names=()):
  """ names: regenerate only the cases with these names (default: all). """
  torch.set_num_threads(1)  # thread-count independent results where ATen's order depends on it
  OUT_DIR.mkdir(exist_ok=True)
  total = 0
  for case in WD_CASES:
    if names and case[0] not in names:
      continue
    data = run_case(*case)
    path = OUT_DIR / f"golden_{case[0]}.npz"
    np.savez_compressed(path, **data)
    total += path.stat().st_size
    man = json.loads(str(data["manifest"]))
    print(f"{path.name}: {len(man['calls'])} calls, {path.stat().st_size / 1024:.0f} KiB")
  print(f"total {total / 1024:.0f} KiB")

if __name__ == "__main__":
  main(sys.argv[1:])
