# coding: utf-8
"""`sharded.ShardedLineSearch` (the attacks' line search on the d-sharded path) under `gloo`, world_size 2,
on CPU: the collectives the host object runs around its stages, in rank order, with every rank taking
the same factor.  The stages run on a NumPy stand-in (the oracle's rules, the score share in fp64 and the
transition restated from `line_maximize`); the CUDA stages are covered by the `-m gpu` tests.
Both ranks must return the same factor and trace, the x sequence must be `line_maximize` fed with the
y values, every y the fp32 score of the full-vector output, and a rank with an empty shard (d = 1) joins."""

import os
import socket

import numpy as np
import pytest

torch = pytest.importorskip("torch")

CASES = (("krum", 601), ("trmean", 601), ("aksel", 601), ("bulyan", 601), ("cge", 1), ("brute", 1), ("median", 1))
EVALS = 7
N, F = 11, 2

def _inputs(d):
  gen = torch.Generator().manual_seed(d + 3)
  honest = [torch.randn(d, generator=gen) * (0.5 + i / 8.) for i in range(N - F)]
  stck = torch.stack(honest)
  return honest, stck.mean(dim=0), stck.var(dim=0).sqrt_()

class _Shard:
  """ The stages of one rank on the NumPy stand-in (CPU tensors). """
  def __init__(self, be, gar, honest, f_real, f, avg, att, evals, negative, kind, world):
    from byzantinemomentum_b200 import engine, sharded
    self.be, self.gar, self.honest, self.f_real, self.f, self.avg, self.att = be, gar, list(honest), f_real, f, avg, att
    self.evals, self.negative, self.empire = evals, negative, kind == "empire-strict"
    self.d = avg.numel()
    self.n = len(self.honest) + f_real
    self.distance = gar in sharded.DISTANCE_BASED
    self.byz = torch.zeros(self.d)
    self.out = torch.zeros(self.d)
    self.record = torch.zeros(2 * evals + 2, dtype=torch.float64)
    # this rank's part of an exchange is row 0 of the gathered buffer on one rank, as on the device
    self.scores = torch.zeros(world, dtype=torch.float64)
    self.score = self.scores[:1] if world == 1 else torch.zeros(1, dtype=torch.float64)
    if self.distance:
      self.rule = engine._rule(gar, self.n, f)
      self.blocks = torch.zeros((world, self.n * self.n if self.rule.pair else self.n), dtype=torch.float64)
      self.part = self.blocks[0] if world == 1 else torch.zeros(self.blocks.shape[1], dtype=torch.float64)
    self.next_x = 0.
    self.state = None
  def _candidate(self, x, final=False):
    s = np.float32(-x if self.empire or (self.negative and not final) else x)
    if self.empire:
      self.byz = self.avg * float(s)
    else:
      self.byz = self.avg + float(s) * self.att
  def _rows(self):
    return self.honest + [self.byz] * self.f_real
  def _share(self):
    diff = (self.out - self.avg).numpy().astype(np.float64)
    return self.score.fill_(float(np.sum(diff * diff)))
  def evaluate(self, k):
    self.x = 0. if k == 0 else self.next_x
    self._candidate(self.x)
    rows = self._rows()
    if not self.distance:
      if self.d > 0:
        self.out = getattr(self.be, self.gar)(rows) if self.gar in ("average", "median") else getattr(self.be, self.gar)(rows, self.f)
      return self._share()
    if self.d == 0:
      return self.part.zero_()
    if self.rule.pair:
      return self.part.copy_(self.be.pairdist_partial(rows).reshape(-1))
    return self.part.copy_(self.be.rowdist_partial(rows, self.be.median(rows) if self.rule.center else None))
  def conclude(self, blocks):
    rule, n, rows = self.rule, self.n, self._rows()
    parts = blocks.reshape(blocks.shape[0], n, n) if rule.pair else blocks
    picked = getattr(self.be, rule.select + "_select")(parts, n, *rule.select_params)
    sel, status = picked if rule.status else (picked, None)
    self.status = 0 if status is None else int(status[0])
    if self.d > 0:
      if rule.gar == "bulyan":
        self.out = self.be.bulyan_reduce(rows, rule.f, rule.m, sel, status)
      else:
        self.out = self.be.average_selected(rows, sel, rule.count, rule.zero_init, status=status)
    return self._share()
  def step(self, k, scores):
    total = float(scores[0])
    for p in scores[1:].tolist():
      total += p
    y = float(np.float32(total))
    x = self.x
    self.record[2 * k], self.record[2 * k + 1] = x, y
    if k == 0:
      best_x, best_y, delta, phase = x, y, 1., 1
    else:
      best_x, best_y, delta, phase = self.state
      if phase == 1:
        if y > best_y:
          best_x, best_y, delta = x, y, delta * 2.
        else:
          delta, phase = delta * 0.8, 2
      else:
        if y > best_y:
          best_x, best_y = x, y
        delta = delta * 0.8
    if phase == 1:
      prop = best_x + delta
    elif x < best_x:
      prop = x + delta
    else:
      prop = x - delta
      while prop < 0:
        prop = (prop + x) / 2
    self.state = (best_x, best_y, delta, phase)
    self.next_x = prop
    if k == self.evals - 1:
      self.record[2 * self.evals] = best_x
  def finish(self):
    self._candidate(self.record[2 * self.evals].item(), final=True)
    return self.byz

def _worker(rank, world, port, queue):
  import sys, pathlib
  root = pathlib.Path(__file__).resolve().parent.parent
  sys.path.insert(0, str(root)); sys.path.insert(0, str(root / "tests"))
  import torch.distributed as dist
  from byzantinemomentum_b200 import sharded
  from fake_backend import OracleBackend

  class SearchBackend(OracleBackend):
    def search_shard(self, *args):
      return _Shard(self, *args)

  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    got = {}
    for gar, d in CASES:
      honest, avg, att = _inputs(d)
      lo, hi = sharded.shard_bounds(d, world, rank)
      cut = lambda v: v[lo:hi].contiguous()
      search = sharded.ShardedLineSearch(gar, [cut(g) for g in honest], F, F, cut(avg), cut(att), EVALS, negative=True,
                                         backend=SearchBackend())
      byz = search()
      factor, trace = search.result()
      got[gar] = (factor, trace, byz.numpy().copy())
    queue.put((rank, got))
  finally:
    dist.destroy_process_group()

def test_two_ranks_take_the_same_factor():
  import torch.multiprocessing as mp
  import line_oracle
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
  ctx = mp.get_context("spawn")
  queue = ctx.Queue()
  procs = [ctx.Process(target=_worker, args=(r, 2, port, queue)) for r in range(2)]
  for p in procs:
    p.start()
  got = dict(queue.get(timeout=300) for _ in procs)
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  for gar, d in CASES:
    (f0, t0, b0), (f1, t1, b1) = got[0][gar], got[1][gar]
    assert f0 == f1 and [(x.hex(), y.hex()) for x, y in t0] == [(x.hex(), y.hex()) for x, y in t1], gar
    ys = [y for _, y in t0]
    xs = []
    want = line_oracle.line_maximize(lambda x: (xs.append(x), ys[len(xs) - 1])[1], EVALS)
    assert [x for x, _ in t0] == xs and f0 == want, gar
    if d == 1:
      assert b1.size == 0                                  # rank 1's shard is empty and it still joined
    # the factor's Byzantine gradient, concatenated, and every y against the same search on the full vectors
    honest, avg, att = _inputs(d)
    np.testing.assert_array_equal(np.concatenate([b0, b1]), (avg + f0 * att).numpy())
    from byzantinemomentum_b200 import sharded
    from fake_backend import OracleBackend
    class One(OracleBackend):
      def search_shard(self, *args):
        return _Shard(self, *args)
    whole = sharded.ShardedLineSearch(gar, honest, F, F, avg, att, EVALS, negative=True, backend=One())
    whole()
    for (x, y), (xw, yw) in zip(t0, whole.result()[1]):
      if x != xw:
        break                                              # the searches part where two scores tie within rounding
      assert abs(y - yw) <= 1e-6 * abs(yw), (gar, x, y, yw)
