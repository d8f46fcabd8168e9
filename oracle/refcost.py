# coding: utf-8
"""CPU cost model of the reference: the same ATen operator sequence, on CPU tensors.

TEST / BENCH INFRASTRUCTURE ONLY (see `oracle/byzoracle.py` for the rules on who may import
`oracle/`).  The reference is not part of this repository, so where $BYZ_REFERENCE does not point at a
checkout `bench.py --impl reference` and `bench.py`'s `cpu_baseline` time THIS module on the
box's host cores: each function issues the ATen calls the reference's rule issues
(`stack`, `sort`, `median`, `topk`, per-pair `sub`/`norm`/`.item()`, Python-level scoring),
so its run time is the reference's run time on that host.  Its results are checked against
the NumPy oracle and the golden fixtures in `tests/test_refcost.py`.

Citations (reference root): average.py:29, median.py:39, trmean.py:33,48-50,79,91-94,106-109,
krum.py:44-62,80, bulyan.py:49-84, brute.py:44-68,80, aksel.py:37-49,64, cge.py:36-38,53-56.
"""

import itertools
import math

import torch

__all__ = ["RULES", "run"]

def _pairs(n):
  return ((a, b) for a in range(n - 1) for b in range(a + 1, n))

def _norm_of_difference(u, v, keep_nonfinite=False):
  value = u.sub(v).norm().item()
  if not keep_nonfinite and not math.isfinite(value):
    value = math.inf
  return value

def _mean_of(rows):
  return sum(rows).div_(len(rows))

def _closest_to(stacked, count, center):
  n, d = stacked.shape
  picks = stacked.clone().sub_(center).abs_().topk(count, dim=0, largest=False, sorted=False).indices
  picks.mul_(d).add_(torch.arange(0, d, dtype=picks.dtype, device=picks.device))
  return stacked.take(picks).mean(dim=0)

def average(rows, **_):
  return sum(rows) / len(rows)

def median(rows, **_):
  return torch.stack(rows).median(dim=0)[0]

def _trimmed(stacked, f):
  return stacked.sort(dim=0).values[f:stacked.shape[0] - f].mean(dim=0)

def trmean(rows, f, **_):
  return _trimmed(torch.stack(rows), f)

def phocas(rows, f, **_):
  stacked = torch.stack(rows)
  return _closest_to(stacked, stacked.shape[0] - f, _trimmed(stacked, f))

def meamed(rows, f, **_):
  stacked = torch.stack(rows)
  return _closest_to(stacked, stacked.shape[0] - f, stacked.median(dim=0).values)

def _distance_table(rows, keep_nonfinite=False):
  n = len(rows)
  table = [[math.inf] * n for _ in range(n)]
  for a, b in _pairs(n):
    table[a][b] = table[b][a] = _norm_of_difference(rows[a], rows[b], keep_nonfinite)
  return table

def krum(rows, f, m=None, **_):
  n = len(rows)
  m = n - f - 2 if m is None else m
  table = _distance_table(rows)
  scored = []
  for i in range(n):
    others = sorted(table[i][j] for j in range(n) if j != i)
    scored.append((sum(others[:n - f - 1]), i))
  scored.sort(key=lambda pair: pair[0])
  return _mean_of([rows[i] for _, i in scored[:m]])

def bulyan(rows, f, m=None, **_):
  n = len(rows)
  m_max = n - f - 2
  m = m_max if m is None else m
  table = _distance_table(rows)
  scored = sorted(((sum(sorted(table[i])[:m]), i) for i in range(n)), key=lambda pair: pair[0])
  order = [i for _, i in scored]
  finite = sum(1 for score, _ in scored if math.isfinite(score))
  theta = n - 2 * f - 2
  kept = torch.empty(theta, rows[0].shape[0], dtype=rows[0].dtype)
  for it in range(theta):
    m = min(m, m_max - it)
    if it >= 1 and finite - it < m:
      # the reference's pruned `(inf, None)` entries sort ahead of +inf scores: gradients[None]
      raise TypeError("too many non-finite scores")
    kept[it] = _mean_of([rows[i] for i in order[it:it + m]])
  return _closest_to(kept, theta - 2 * f, kept.median(dim=0).values)

def brute(rows, f, **_):
  n = len(rows)
  table = _distance_table(rows, keep_nonfinite=True)
  best, best_diameter = None, None
  for subset in itertools.combinations(range(n), n - f):
    diameter = 0.
    for a, b in itertools.combinations(subset, 2):
      value = table[a][b]
      if not math.isfinite(value):
        break
      diameter = max(diameter, value)
    else:
      if best is None or diameter < best_diameter:
        best, best_diameter = subset, diameter
  assert best is not None
  return _mean_of([rows[i] for i in best])

def aksel(rows, f, mode="mid", **_):
  n = len(rows)
  center = torch.stack(rows).median(dim=0)[0]
  keyed = sorted(((x - center).pow_(2).sum().item(), i) for i, x in enumerate(rows))
  keyed.sort(key=lambda pair: pair[0])
  count = (n + 1) // 2 if mode == "mid" else n - f
  return _mean_of([rows[i] for _, i in keyed[:count]])

def cge(rows, f, **_):
  def key(row):
    value = row.norm().item()
    return value if math.isfinite(value) else math.inf
  ranked = sorted(((key(row), i) for i, row in enumerate(rows)), key=lambda pair: pair[0])
  m = len(rows) - f
  total = rows[ranked[0][1]].clone()
  for _, i in ranked[1:m]:
    total.add_(rows[i])
  return total.div_(m)

def study_metrics(rows):
  """ The operator sequence of tools/pytorch.py:108-121 (average, norm, abs-max, n sub+dot with
  one `.item()` each), for timing beside `bz_avg_dev_max`. """
  mean = rows[0].clone()
  for row in rows[1:]:
    mean.add_(row)
  mean.div_(len(rows))
  length = mean.norm().item()
  largest = mean.abs().max().item()
  spread = 0.
  for row in rows:
    delta = row.sub(mean)
    spread += delta.dot(delta).item()
  return mean, length, spread, largest

RULES = dict(average=average, median=median, trmean=trmean, phocas=phocas, meamed=meamed,
             krum=krum, bulyan=bulyan, brute=brute, aksel=aksel, cge=cge)

def run(name, rows, **params):
  """ One aggregation with rule `name` on a list of CPU tensors. """
  return RULES[name](rows, **params)
