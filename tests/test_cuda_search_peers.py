# coding: utf-8
"""GPU tests of the d-sharded line search with its exchanges over peer memory (`ShardedLineSearch(exchange=
"fused")`, include/byzagg_search_peers.h).

  * One rank (a plain device buffer in the `FusedExchange` layout): trace, factor, Byzantine gradient, the
    rule's last output and the status word are those of `engine.LineSearch`, bit for bit, for all ten
    rules at n = 11, 25, 51, for `identical` (negative) and `empire-strict`.
  * R = 2, 3, 8 ranks emulated on ONE GPU, each with its own buffer in the `FusedExchange` layout and its
    own 64-float pitched copy of its columns, next to R collective instances of the same search (the
    all-gathers replaced by `torch.stack`).  No two grids ever run at once: before each rank's call, the
    test writes into every other rank's slot the block (or score share) that rank's collective stage
    produced, and sets every flag the call waits on; the call must raise its flag on every rank and
    publish exactly its collective stage's bits.  Every rank's trace, factor and `byz` shard, and its
    outputs, are then bit-identical to the collective stages'.  After the first evaluation the pair rules
    take the star pass, and their blocks are those of a pass without the cache.  Shards are empty when
    d < R; two searches run back to back across the 2^32 epoch wrap with the honest rows changed in place
    between them, so a wrong slot or a stale epoch reads another exchange's values.
  * Bulyan's and brute's status words on degenerate data reach every rank.
  * Unaligned rows: "auto" keeps the collective path, an explicit "fused" raises for the pair rules."""

import ctypes
import math

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U32 = 1 << 32
FLAG_WORDS = 16

from test_cuda_linesearch import F_OF, _direction, _honest
from test_cuda_sharded_search import GARS, _bits, _shards, _status

def _s32(v):
  v %= U32
  return v - U32 if v >= 1 << 31 else v

@pytest.mark.parametrize("n", [11, 25, 51])
@pytest.mark.parametrize("gar", GARS)
def test_one_rank_fused_is_the_single_gpu_search(gar, n):
  from byzantinemomentum_b200 import engine, sharded
  f = F_OF[(gar, n)]
  pair = gar in ("krum", "bulyan", "brute")
  for d, offset in ((4099, 0), (1, 0)) + (() if pair else ((1031, 1),)):
    honest = _honest(n - f, d, 11 + d + n, offset)
    for kind, negative in (("identical", True), ("empire-strict", False)):
      avg, att = _direction(honest, kind)
      for evals in (1, 16):
        ref = engine.LineSearch(gar, honest, f, f, avg, att, evals, negative=negative, kind=kind)
        ref()
        got = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, evals, negative=negative, kind=kind, exchange="fused")
        assert got.exchange == "fused"
        byz = got()
        torch.cuda.synchronize()
        what = (gar, n, d, offset, kind, evals)
        assert got._fx.epoch == (2 if gar in sharded.DISTANCE_BASED else 1) * evals, what
        assert torch.equal(_bits(got.record[:-1]), _bits(ref.record[:-1])), (what, got.record, ref.record)
        assert _status(got.record) == _status(ref.record), what
        assert torch.equal(_bits(byz), _bits(ref.byz)), what
        assert torch.equal(_bits(got._shard.out), _bits(ref._out)), what

class _Ranks:
  """ R emulated ranks, each with its own buffer in the `FusedExchange` layout. """
  def __init__(self, R, n):
    from byzantinemomentum_b200 import sharded
    self.R, self.n = R, n
    self.buf = [torch.zeros(2 * n * n + FLAG_WORDS, dtype=torch.float64, device=DEV) for _ in range(R)]
    self.fx = []
    for r in range(R):
      fx = sharded.FusedExchange.__new__(sharded.FusedExchange)
      fx.n, fx.device, fx.group, fx.world, fx.rank, fx.epoch = n, torch.device(DEV), None, R, r, 0
      fx.peer_base = [b.data_ptr() for b in self.buf]
      self.fx.append(fx)
  def slot(self, p, s):
    nn = self.n * self.n
    return self.buf[p][s * nn:(s + 1) * nn]
  def flags(self, p, s):
    return self.buf[p][2 * self.n * self.n:].view(torch.int32)[FLAG_WORDS * s:FLAG_WORDS * (s + 1)]
  def exchange(self, epoch, values, call, tag):
    """ One exchange at `epoch`: rank r's call (call(r)) after every other rank p's slot holds values[p] and
    every flag r waits on is set; r must publish values[r] and raise its flag on every rank. """
    s = epoch % 2
    width = values[0].numel()
    for r in range(self.R):
      for p in range(self.R):
        self.flags(p, s).fill_(_s32(epoch - 2))                 # the slot's previous use
      for p in range(self.R):
        if p != r:
          self.slot(p, s)[:width].copy_(values[p])
          self.flags(r, s)[p] = _s32(epoch)
      self.slot(r, s)[:width].fill_(float("nan"))
      call(r)
      torch.cuda.synchronize()
      assert torch.equal(_bits(self.slot(r, s)[:width]), _bits(values[r])), f"{tag}: rank {r} published other bits"
      for p in range(self.R):
        assert int(self.flags(p, s)[r].item()) == _s32(epoch), f"{tag}: rank {r} did not signal rank {p}"

def _full_pass_block(shard):
  """ This rank's phase-A block of the current rows without a cache (bz_pairdist_partial_reuse). """
  from byzantinemomentum_b200 import _lib
  rows = shard._rows
  n = rows.n
  part = torch.empty(n * n, dtype=torch.float64, device=DEV)
  table = torch.empty(64 * 64, dtype=torch.float64, device=DEV)
  mode = ctypes.c_int(-9)
  ws = torch.empty(int(_lib.lib().bz_workspace_bytes(n)), dtype=torch.uint8, device=DEV)
  rc = _lib.lib().bz_pairdist_partial_reuse(rows.ptrs, n, rows.d, part.data_ptr(), None, None, 0, table.data_ptr(),
                                            ctypes.byref(mode), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
  _lib.check(rc, "bz_pairdist_partial_reuse")
  return part

def _emulate(gar, honest, f, avg, att, R, evals=16, searches=2, start=U32 - 7, negative=False, kind="identical"):
  """ R fused and R collective instances of the search on one GPU, driven exchange by exchange; `searches`
  searches back to back from epoch `start`, the honest rows changed in place between them.  Returns the
  (fused, collective) shards after the last search. """
  from byzantinemomentum_b200 import sharded
  n = len(honest) + f
  vectors = honest + [avg] + ([att] if att is not None else [])
  per_rank = _shards(vectors, R, True)
  nh = len(honest)
  def make(rows):
    return sharded._SearchShard(gar, rows[:nh], f, f, rows[nh], rows[nh + 1] if att is not None else None, evals, negative, kind, R)
  fused = [make(rows) for rows in per_rank]
  coll = [make(rows) for rows in per_rank]
  ranks = _Ranks(R, n)
  for r, shard in enumerate(fused):
    shard.fuse(ranks.fx[r])
  distance = gar in sharded.DISTANCE_BASED
  pair = gar in ("krum", "bulyan", "brute")
  epoch = start
  for search in range(searches):
    if search > 0:
      for rows in per_rank:                                       # new honest content, same tensors
        for i in range(0, nh, 3):
          rows[i].mul_(-1.5).add_(0.25)
    for k in range(evals):
      tag = f"{gar} R={R} search {search} k={k}"
      parts = [c.evaluate(k) for c in coll]
      if distance:
        epoch += 1
        ranks.exchange(epoch, parts, lambda r: fused[r].evaluate_fused(k, epoch), f"{tag} rule")
        shares = [c.conclude(torch.stack(parts)) for c in coll]
        for r, (a, b) in enumerate(zip(fused, coll)):
          assert torch.equal(a._meta[:a._rule.length], b._meta[:b._rule.length]), f"{tag}: rank {r} selection"
          if pair and a._rows.d > 0:
            assert a._mode.value == (1 if k > 0 else 0), f"{tag}: rank {r} pass {a._mode.value}"
            slot = ranks.slot(r, epoch % 2)
            assert torch.equal(_bits(slot), _bits(_full_pass_block(a))), f"{tag}: rank {r} block vs a full pass"
      else:
        for a in fused:
          a.evaluate_fused(k, None)
        shares = parts
      for r, (a, b) in enumerate(zip(fused, coll)):
        torch.cuda.synchronize()
        assert torch.equal(_bits(a.out), _bits(b.out)), f"{tag}: rank {r} rule output"
      epoch += 1
      ranks.exchange(epoch, [s.reshape(1) for s in shares], lambda r: fused[r].score_fused(k, epoch), f"{tag} score")
      scores = torch.stack(shares).reshape(R)
      for c in coll:
        c.step(k, scores)
    for a, b in zip(fused, coll):
      a.finish()
      b.finish()
    torch.cuda.synchronize()
    for r, (a, b) in enumerate(zip(fused, coll)):
      what = (gar, R, search, r)
      assert torch.equal(_bits(a.record[:-1]), _bits(b.record[:-1])), (what, a.record, b.record)
      assert _status(a.record) == _status(b.record), what
      assert torch.equal(_bits(a.byz), _bits(b.byz)), what
  return fused, coll

@pytest.mark.parametrize("R", [2, 3, 8])
@pytest.mark.parametrize("gar", GARS)
def test_emulated_ranks_are_the_collective_stages(gar, R):
  n = 25
  f = F_OF[(gar, n)]
  for d in (4099, R - 1):
    honest = _honest(n - f, d, 17 + R + d)
    avg, att = _direction(honest, "identical")
    fused, _ = _emulate(gar, honest, f, avg, att, R)
    record = fused[0].record
    for s in fused[1:]:
      assert torch.equal(_bits(s.record[:-1]), _bits(record[:-1])), (gar, R, d)

@pytest.mark.parametrize("gar", ["bulyan", "brute"])
def test_status_words_reach_every_rank(gar):
  from byzantinemomentum_b200 import _lib
  n, f = 11, 2 if gar == "bulyan" else 3
  honest = _honest(n - f, 515, 21)
  for k in range(6):                               # non-finite rows (all on rank 0): no finite scores / subsets
    honest[k] = honest[k].clone()
    honest[k][k] = math.nan
  avg, att = _direction(honest[6:], "identical")
  fused, coll = _emulate(gar, honest, f, avg, att, 2, evals=6, searches=1)
  want = _lib.STATUS_DEGENERATE if gar == "bulyan" else _lib.STATUS_NO_FINITE_SET
  for s in fused + coll:
    assert _status(s.record) == want, gar

def test_unaligned_rows_keep_the_collective_path():
  from byzantinemomentum_b200 import sharded
  honest = _honest(20, 1031, 5, offset=1)
  avg, att = _direction(honest, "identical")
  for gar in ("krum", "bulyan", "brute"):
    rows, f = (honest[:8], 2) if gar == "brute" else (honest, 5)      # brute: C(n, n - f) <= 2^31
    assert sharded.ShardedLineSearch(gar, rows, f, f, avg, att, 4).exchange == "nccl"
    with pytest.raises(ValueError, match="16-byte aligned"):
      sharded.ShardedLineSearch(gar, rows, f, f, avg, att, 4, exchange="fused")
  assert sharded.ShardedLineSearch("aksel", honest, 5, 5, avg, att, 4, exchange="fused").exchange == "fused"
