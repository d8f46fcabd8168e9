# coding: utf-8
"""NumPy stand-in for `byzantinemomentum_b200.engine`, built from the oracle's primitives.
Injected into `byzantinemomentum_b200.sharded.aggregate(..., backend=...)` by the CPU tests so
that the multi-rank host logic (what is exchanged, in which order it is summed, what every
rank derives from it) runs under `gloo` without a GPU.  Test infrastructure only."""

import math

import numpy as np
import torch

from oracle import byzoracle as orc

def _np(rows):
  return [r.numpy() for r in rows]

def _t(x, dtype=None):
  t = torch.from_numpy(np.ascontiguousarray(x))
  return t if dtype is None else t.to(dtype)

class OracleBackend:
  # coordinate-wise
  def average(self, rows): return _t(orc.average(_np(rows)))
  def median(self, rows): return _t(orc.median(_np(rows)))
  def trmean(self, rows, f): return _t(orc.trmean(_np(rows), f))
  def phocas(self, rows, f): return _t(orc.phocas(_np(rows), f))
  def meamed(self, rows, f): return _t(orc.meamed(_np(rows), f))
  # phase A
  def pairdist_partial(self, rows):
    g = orc.as_matrix(_np(rows))
    n = g.shape[0]
    part = np.zeros((n, n), dtype=np.float64)
    with np.errstate(all="ignore"):
      for x in range(n - 1):
        diff = (g[x + 1:] - g[x][None, :]).astype(np.float32).astype(np.float64)
        part[x, x + 1:] = np.einsum("ij,ij->i", diff, diff)
    return _t(part)
  def rowdist_partial(self, rows, center=None):
    g = orc.as_matrix(_np(rows))
    with np.errstate(all="ignore"):
      if center is None:
        sq = g.astype(np.float64) ** 2
      else:
        diff = (g - center.numpy()[None, :]).astype(np.float32)
        sq = (diff * diff).astype(np.float32).astype(np.float64)
    return _t(sq.sum(axis=1))
  # phase B: blocks are summed in rank order
  @staticmethod
  def _sum_parts(parts):
    return orc.sum_parts(parts.numpy())
  def _distances(self, parts, n, map_nonfinite):
    sq = self._sum_parts(parts)
    D = np.triu(orc.fp32_norm(sq), 1)
    D = D + D.T
    if map_nonfinite:
      D = np.where(np.isfinite(D), D, np.inf)
    return D
  def krum_select(self, parts, n, f):
    order, _ = orc.krum_order(self._distances(parts, n, True), f)
    return _t(np.array(order, dtype=np.int32))
  def bulyan_select(self, parts, n, f, m):
    order, scores = orc.bulyan_order(self._distances(parts, n, True), f, m)
    finite = sum(1 for s in scores if math.isfinite(s))
    status, mi = 0, m
    for i in range(n - 2 * f - 2):
      mi = min(mi, n - f - 2 - i)
      if i >= 1 and finite - i < mi:
        status = 2
    return _t(np.array(order, dtype=np.int32)), _t(np.array([status], dtype=np.int32))
  def brute_select(self, parts, n, f):
    try:
      sel = orc.brute_selection(self._distances(parts, n, False), f)
      status = 0
    except AssertionError:
      sel, status = list(range(n - f)), 1
    return _t(np.array(sel, dtype=np.int32)), _t(np.array([status], dtype=np.int32))
  def rowdist_select(self, parts, n, sqrt_norm):
    sq = self._sum_parts(parts)
    with np.errstate(all="ignore"):
      if sqrt_norm:
        key = orc.fp32_norm(sq)
        key = np.where(np.isfinite(key), key, np.inf)
      else:
        key = sq.astype(np.float32).astype(np.float64)
    order = sorted(range(n), key=lambda i: (math.isnan(key[i]), key[i] if not math.isnan(key[i]) else 0., i))
    return _t(np.array(order, dtype=np.int32))
  # phase C
  def average_selected(self, rows, selection, count, zero_init=True, divisor=None, status=None):
    g = orc.as_matrix(_np(rows))
    if status is not None and int(status[0]) != 0:
      return torch.full((g.shape[1],), float("nan"))
    idx = list(range(count)) if selection is None else [int(i) for i in selection[:count]]
    total = orc._seq_sum_rows(g, idx, zero_init)
    with np.errstate(all="ignore"):
      return _t((total / np.float32(count if divisor is None else divisor)).astype(np.float32))
  def bulyan_reduce(self, rows, f, m, order, status=None):
    g = orc.as_matrix(_np(rows))
    if status is not None and int(status[0]) != 0:
      return torch.full((g.shape[1],), float("nan"))
    sel = orc.bulyan_stage1(g, [int(i) for i in order], f, m)
    theta = sel.shape[0]
    return _t(orc.closest_mean(sel, theta - 2 * f, orc.median(sel)))

  # study metrics
  def avg_dev_max_async(self, rows):
    g = orc.as_matrix(_np(rows))
    avg = orc.compute_avg_dev_max(list(g))[0]
    with np.errstate(all="ignore"):
      a64 = avg.astype(np.float64)
      absa = np.abs(avg)
      stats = [float(np.sum(a64 * a64)), float("nan") if np.isnan(absa).any() else float(absa.max())]
      for i in range(g.shape[0]):
        diff = (g[i] - avg).astype(np.float32).astype(np.float64)
        stats.append(float(np.sum(diff * diff)))
    return _t(avg), _t(np.array(stats, dtype=np.float64))
