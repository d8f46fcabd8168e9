# coding: utf-8
"""`sharded.study_step` (attack.py:846-866 over d-sharded vectors) under `gloo`, world_size 2, on CPU:
both ranks must return the same scalars, those scalars must match a NumPy fp64 evaluation of the
block on the full vectors, and the shards of the averages must concatenate to the full averages.
The per-shard passes run on a NumPy stand-in (K6 and `bz_rowdots` on the GPU: `-m gpu` tests)."""

import math
import os
import socket

import numpy as np
import pytest

torch = pytest.importorskip("torch")

MOMENTUM = 0.9
KEYS = ("sampled_norm_avg", "sampled_norm_dev", "sampled_norm_max", "honest_norm_avg", "honest_norm_dev", "honest_norm_max",
        "attack_norm_avg", "attack_norm_dev", "attack_norm_max", "defense_norm_avg", "defense_norm_max",
        "cosin_splhon", "cosin_splatt", "cosin_spldef", "cosin_honatt", "cosin_hondef", "cosin_attdef",
        "cosin_sampled", "curv_sampled")
AVERAGES = ("sampled_grad_avg", "honest_grad_avg", "attack_grad_avg")

def _case(name):
  """ (sampleds, honests, attacks, defense, pasts as full vectors) of one named case. """
  ns, nh, na, npast, d, shared = dict(ragged=(8, 6, 3, 3, 601, False), no_attack=(8, 6, 0, 2, 601, False),
                                      same_list=(7, 7, 2, 1, 600, True), many_pasts=(5, 5, 1, 70, 301, False),
                                      nan_on_rank_1=(6, 6, 2, 2, 601, False), zero_defense=(5, 5, 2, 0, 601, True),
                                      empty_shard=(4, 3, 2, 2, 1, False))[name]
  gen = torch.Generator().manual_seed(sum(map(ord, name)))
  rows = lambda k: [torch.randn(d, generator=gen) for _ in range(k)]
  sampleds = rows(ns)
  honests = sampleds[:nh] if shared else rows(nh)
  attacks = [a.mul(-2.) for a in rows(na)]
  defense = torch.zeros(d) if name == "zero_defense" else torch.randn(d, generator=gen) * 0.3
  pasts = rows(npast)
  if name == "nan_on_rank_1":
    sampleds[2][d - 3] = float("nan")          # in the second half of the columns only
  return sampleds, honests, attacks, defense, pasts

CASES = ("ragged", "no_attack", "same_list", "many_pasts", "nan_on_rank_1", "zero_defense", "empty_shard")

def _norm(v):
  """ The fp32 `norm()` of a full vector (+inf past FLT_MAX), as `sampled_norm_avg` holds it. """
  from oracle import byzoracle as orc
  return float(orc.fp32_norm(np.sum(np.asarray(v, dtype=np.float64) ** 2)))

def _worker(rank, world, port, queue):
  import sys, pathlib
  root = pathlib.Path(__file__).resolve().parent.parent
  sys.path.insert(0, str(root)); sys.path.insert(0, str(root / "tests"))
  import torch.distributed as dist
  from byzantinemomentum_b200 import sharded
  from fake_backend import OracleBackend

  class StudyBackend(OracleBackend):
    """ The stand-in plus `bz_rowdots` in fp64, and K6's zeros for an empty shard. """
    def avg_dev_max_async(self, rows):
      if rows[0].numel() == 0:
        return torch.zeros(0), torch.zeros(2 + len(rows), dtype=torch.float64)
      return super().avg_dev_max_async(rows)
    def rowdots_async(self, center, rows):
      c = center.numpy().astype(np.float64)
      return torch.tensor([float(np.dot(r.numpy().astype(np.float64), c)) for r in rows], dtype=torch.float64)

  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    out = {}
    for name in CASES:
      sampleds, honests, attacks, defense, pasts = _case(name)
      lo, hi = sharded.shard_bounds(defense.numel(), world, rank)
      cut = lambda rows: [r[lo:hi].contiguous() for r in rows]
      shard_s = cut(sampleds)
      shared = all(h is s for h, s in zip(honests, sampleds))
      shard_h = shard_s[:len(honests)] if shared else cut(honests)     # same_list: the very same tensors, one K6 pass
      got = sharded.study_step(shard_s, shard_h, cut(attacks), defense[lo:hi].contiguous(),
                               [(p[lo:hi].contiguous(), _norm(p.numpy())) for p in pasts], MOMENTUM, backend=StudyBackend())
      out[name] = {k: (None if v is None else v.numpy().copy()) if k in AVERAGES else v for k, v in got.items()}
    queue.put((rank, out))
  finally:
    dist.destroy_process_group()

def _numpy_study(sampleds, honests, attacks, defense, pasts):
  """ attack.py:846-866 on the full vectors in NumPy fp64 (the averages: the oracle's fp32 order). """
  from oracle import byzoracle as orc
  s_avg, s_norm, s_dev, s_max = orc.compute_avg_dev_max([g.numpy() for g in sampleds])
  h_avg, h_norm, h_dev, h_max = orc.compute_avg_dev_max([g.numpy() for g in honests])
  a_avg, a_norm, a_dev, a_max = orc.compute_avg_dev_max([g.numpy() for g in attacks])
  dfn = defense.numpy()
  d_norm = _norm(dfn)
  dot = lambda a, b: float(np.dot(a.astype(np.float64), b.astype(np.float64)))
  def cos(a, b, na, nb):
    if a is None or b is None:
      return math.nan
    with np.errstate(all="ignore"):
      return float(np.float64(dot(a, b)) / na / nb)
  out = dict(sampled_norm_avg=s_norm, sampled_norm_dev=s_dev, sampled_norm_max=s_max, honest_norm_avg=h_norm, honest_norm_dev=h_dev,
             honest_norm_max=h_max, attack_norm_avg=a_norm, attack_norm_dev=a_dev, attack_norm_max=a_max,
             defense_norm_avg=d_norm, defense_norm_max=float(np.max(np.abs(dfn))),
             cosin_splhon=cos(s_avg, h_avg, s_norm, h_norm), cosin_splatt=cos(s_avg, a_avg, s_norm, a_norm),
             cosin_spldef=cos(s_avg, dfn, s_norm, d_norm), cosin_honatt=cos(h_avg, a_avg, h_norm, a_norm),
             cosin_hondef=cos(h_avg, dfn, h_norm, d_norm), cosin_attdef=cos(a_avg, dfn, a_norm, d_norm))
  if pasts:
    out["cosin_sampled"] = cos(s_avg, pasts[0].numpy(), s_norm, _norm(pasts[0].numpy()))
    out["curv_sampled"] = MOMENTUM * sum(MOMENTUM ** i * dot(s_avg, p.numpy()) for i, p in enumerate(pasts))
  else:
    out["cosin_sampled"] = out["curv_sampled"] = math.nan
  return out, dict(sampled_grad_avg=s_avg, honest_grad_avg=h_avg, attack_grad_avg=a_avg)

def _same(a, b):
  return a == b or (math.isnan(a) and math.isnan(b))

def test_finish_merges_the_ranks_before_the_fp32_rules():
  """ `engine.study_finish` on constructed partial vectors (ns = nh = 2, no attack, one past):
  one rank keeps a -0.0 dot product and the sign of its zero cosine (a sum started from 0.0 would
  give +0.0); two ranks' sums of squares that each fit in fp32 overflow together; a NaN maximum on
  one rank reaches the merged maximum. """
  from byzantinemomentum_b200 import engine
  p = engine.StudyPartials()
  p.sampled_avg = p.honest_avg = torch.zeros(3)
  p.attack_avg = None
  p.counts, p.past_norms = (2, 2, 0), [1.]
  #        s: |avg|^2 max dev dev   h: |avg|^2 max dev dev   <s,h> <s,def> <s,past> <h,def> <def,def> max|def|
  vector = [1., 1., 0., 0.,          1., 1., 0., 0.,          -0.,  0.5,    -0.,     0.5,    4.,       2.]
  p.vector = torch.tensor(vector, dtype=torch.float64)
  one = engine.study_finish(p, [vector], MOMENTUM)
  for key in ("cosin_splhon", "cosin_sampled"):
    assert one[key] == 0. and math.copysign(1., one[key]) == -1., key
  assert one["defense_norm_avg"] == 2. and one["cosin_spldef"] == 0.25 and one["defense_norm_max"] == 2.
  big = list(vector)
  big[0] = 2e38                                      # below FLT_MAX on each rank, 4e38 together
  nan_max = list(big)
  nan_max[1] = math.nan
  two = engine.study_finish(p, [big, nan_max], MOMENTUM)
  assert two["sampled_norm_avg"] == math.inf and math.isnan(two["sampled_norm_max"])
  assert two["honest_norm_avg"] == np.float32(math.sqrt(2.)) and two["honest_norm_max"] == 1.
  assert two["defense_norm_avg"] == np.float32(math.sqrt(8.)) and two["defense_norm_max"] == 2.

def test_two_rank_study_step_matches_the_full_vectors_on_every_rank():
  import torch.multiprocessing as mp
  import parity
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
  ctx = mp.get_context("spawn")
  queue = ctx.Queue()
  procs = [ctx.Process(target=_worker, args=(r, 2, port, queue)) for r in range(2)]
  for p in procs:
    p.start()
  got = dict(queue.get(timeout=180) for _ in procs)
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  for name in CASES:
    per_rank = [got[r][name] for r in (0, 1)]
    assert set(per_rank[0]) == set(KEYS) | set(AVERAGES)
    for key in KEYS:
      assert _same(per_rank[0][key], per_rank[1][key]), (name, key, per_rank[0][key], per_rank[1][key])
    want, want_avgs = _numpy_study(*_case(name))
    for key, ref in want.items():
      val = per_rank[0][key]
      if math.isnan(ref) or math.isinf(ref):
        assert _same(val, ref), (name, key, val, ref)
      else:
        assert abs(val - ref) <= 2e-5 * abs(ref) + 3e-6, (name, key, val, ref)
    for key in AVERAGES:
      if want_avgs[key] is None:
        assert per_rank[0][key] is None and per_rank[1][key] is None, (name, key)
      else:
        parity.assert_bit_exact(np.concatenate([per_rank[0][key], per_rank[1][key]]), want_avgs[key], f"{name} {key}")
  # the cases reach what they are named for
  assert math.isnan(got[0]["nan_on_rank_1"]["sampled_norm_max"]) and math.isnan(got[0]["nan_on_rank_1"]["cosin_splhon"])
  assert math.isnan(got[0]["zero_defense"]["cosin_spldef"]) and got[0]["zero_defense"]["defense_norm_avg"] == 0.
  assert got[1]["empty_shard"]["sampled_grad_avg"].size == 0 and math.isfinite(got[1]["empty_shard"]["cosin_splhon"])
  assert math.isnan(got[0]["no_attack"]["cosin_attdef"]) and math.isfinite(got[0]["many_pasts"]["curv_sampled"])
