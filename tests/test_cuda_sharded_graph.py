# coding: utf-8
"""GPU tests of the exchanges over peer memory that take their epoch from the exchange buffer
(include/byzagg_peers_next.h) and of the CUDA graphs built on them (`ShardedPlan.graph()`,
`ShardedLineSearch.graph()`).

  * The `_next` calls, exchange by exchange: R = 1, 2, 3, 8 ranks emulated on ONE GPU with the harness of
    test_cuda_search_peers.py (each rank its own buffer in the `FusedExchange` layout; before each rank's call
    every other rank's slot holds its block and every flag the call waits on is set; no two grids at once).
    The flags also hold the epoch the call must derive: this rank's own entries are the two previous epochs,
    or zero (a fresh buffer).  Every call must publish its collective stage's bits into the slot of the
    derived epoch, raise that epoch on every rank and leave the other slot alone, and every rank's trace,
    factor, `byz` and outputs are the collective stages'; for all ten rules at n = 11, 25, 51, with empty
    shards, from a fresh buffer and across the 2^32 wrap.
  * One rank: `ShardedLineSearch(exchange="fused").graph()` and single-rank "nccl" replays are
    `engine.LineSearch` and the eager search bit for bit, with the honest rows changed in place between
    replays and eager calls interleaved; `fx.epoch` stays the epoch the flags hold.  `ShardedPlan.graph()`
    (fused, and "nccl") is `engine.Plan` bit for bit.
  * `ShardedPlan` replays at R = 2, 3 emulated, one exchange per replay, against the eager by-value call.
  * "p2p" and multi-rank "nccl" refuse `graph()`.
No test waits for the peer timeout: every wait is satisfied by preset flags."""

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U32 = 1 << 32
FLAG_WORDS = 16

from test_cuda_linesearch import F_OF, _direction, _honest
from test_cuda_search_peers import _Ranks, _s32
from test_cuda_sharded_search import GARS, _bits, _shards, _status

def _later(a, b):
  """ The later of two epochs, wrap-aware. """
  return b if _s32(b - a) > 0 else a

def _own_epoch(fx):
  """ The last epoch this rank raised, from its own flags (the two slots' [rank] entries). """
  flags = fx.buffer[2 * fx.n * fx.n:].view(torch.int32)
  return _later(int(flags[fx.rank].item()) % U32, int(flags[FLAG_WORDS + fx.rank].item()) % U32)

def _exchange_next(ranks, epoch, values, call, tag):
  """ One exchange that every rank's call must find at `epoch` from the flags alone: the other slot's flags hold
  epoch - 1 and this slot's epoch - 2 (zero for a fresh buffer, epoch 1), the peers' entries in this rank's
  array of this slot hold `epoch`.  The call must publish values[r], raise `epoch` on every rank and leave the
  other slot's flags alone. """
  s, width = epoch % 2, values[0].numel()
  fresh = epoch == 1
  for r in range(ranks.R):
    for p in range(ranks.R):
      ranks.flags(p, s).fill_(0 if fresh else _s32(epoch - 2))
      ranks.flags(p, 1 - s).fill_(_s32(epoch - 1))
    for p in range(ranks.R):
      if p != r:
        ranks.slot(p, s)[:width].copy_(values[p])
        ranks.flags(r, s)[p] = _s32(epoch)
    ranks.slot(r, s)[:width].fill_(float("nan"))
    other = [ranks.flags(p, 1 - s).clone() for p in range(ranks.R)]
    call(r)
    torch.cuda.synchronize()
    assert torch.equal(_bits(ranks.slot(r, s)[:width]), _bits(values[r])), f"{tag}: rank {r} published other bits"
    for p in range(ranks.R):
      assert int(ranks.flags(p, s)[r].item()) == _s32(epoch), f"{tag}: rank {r} did not signal rank {p} at {epoch}"
      assert torch.equal(ranks.flags(p, 1 - s), other[p]), f"{tag}: rank {r} touched the other slot of rank {p}"

def _emulate_next(gar, honest, f, avg, att, R, evals, starts):
  """ R fused instances of the search issuing the `_next` calls, next to R collective instances, one search
  per entry of `starts` (the epoch before its first exchange), the honest rows changed in place between them. """
  from byzantinemomentum_b200 import sharded
  n, nh = len(honest) + f, len(honest)
  per_rank = _shards(honest + [avg, att], R, True)
  def make(rows):
    return sharded._SearchShard(gar, rows[:nh], f, f, rows[nh], rows[nh + 1], evals, True, "identical", R)
  fused, coll = [make(rows) for rows in per_rank], [make(rows) for rows in per_rank]
  ranks = _Ranks(R, n)
  for r, shard in enumerate(fused):
    shard.fuse(ranks.fx[r])
  distance = gar in sharded.DISTANCE_BASED
  for search, epoch in enumerate(starts):
    if search > 0:
      for rows in per_rank:
        for i in range(0, nh, 3):
          rows[i].mul_(-1.5).add_(0.25)
    for k in range(evals):
      tag = f"{gar} n={n} R={R} search {search} k={k}"
      parts = [c.evaluate(k) for c in coll]
      if distance:
        epoch += 1
        _exchange_next(ranks, epoch % U32, parts, lambda r: fused[r].evaluate_fused(k, None), f"{tag} rule")
        shares = [c.conclude(torch.stack(parts)) for c in coll]
        for r, (a, b) in enumerate(zip(fused, coll)):
          assert torch.equal(a._meta[:a._rule.length], b._meta[:b._rule.length]), f"{tag}: rank {r} selection"
      else:
        for a in fused:
          a.evaluate_fused(k, None)
        shares = parts
      torch.cuda.synchronize()
      for r, (a, b) in enumerate(zip(fused, coll)):
        assert torch.equal(_bits(a.out), _bits(b.out)), f"{tag}: rank {r} rule output"
      epoch += 1
      _exchange_next(ranks, epoch % U32, [s.reshape(1) for s in shares], lambda r: fused[r].score_fused(k, None), f"{tag} score")
      scores = torch.stack(shares).reshape(R)
      for c in coll:
        c.step(k, scores)
    for a, b in zip(fused, coll):
      a.finish()
      b.finish()
    torch.cuda.synchronize()
    for r, (a, b) in enumerate(zip(fused, coll)):
      what = (gar, n, R, search, r)
      assert torch.equal(_bits(a.record[:-1]), _bits(b.record[:-1])), (what, a.record, b.record)
      assert _status(a.record) == _status(b.record), what
      assert torch.equal(_bits(a.byz), _bits(b.byz)), what
  return fused

@pytest.mark.parametrize("R", [1, 2, 3, 8])
@pytest.mark.parametrize("n", [11, 25, 51])
@pytest.mark.parametrize("gar", GARS)
def test_next_calls_are_the_by_value_exchanges(gar, n, R):
  f = F_OF[(gar, n)]
  for d in ((4099, R - 1) if R > 1 else (4099,)):                 # d = R - 1: the last rank's shard is empty
    honest = _honest(n - f, d, 7 + R + n + d)
    avg, att = _direction(honest, "identical")
    # a fresh zeroed buffer (the first exchange is epoch 1), then a search across the 2^32 wrap
    _emulate_next(gar, honest, f, avg, att, R, evals=3, starts=(0, U32 - 3))

def _flags_hold(fx):
  return _own_epoch(fx) == fx.epoch % U32

@pytest.mark.parametrize("gar", GARS)
def test_one_rank_search_graph_is_the_single_gpu_search(gar):
  from byzantinemomentum_b200 import engine, sharded
  n, d = 25, 4099
  f = F_OF[(gar, n)]
  honest = _honest(n - f, d, 31)
  avg, att = _direction(honest, "identical")
  evals = 16
  exchanges = (2 if gar in sharded.DISTANCE_BASED else 1) * evals
  ref = engine.LineSearch(gar, honest, f, f, avg, att, evals, negative=True)
  eager = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, evals, negative=True, exchange="fused")
  captured = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, evals, negative=True, exchange="fused")
  single = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, evals, negative=True, exchange="nccl")
  assert single.exchange == "nccl"
  replay, replay_single = captured.graph(), single.graph()
  assert captured._fx.epoch == exchanges and _flags_hold(captured._fx)      # the warm-up's eager search
  for step in range(4):
    if step > 0:
      for i in range(0, n - f, 4):                                # new content, same tensors
        honest[i].mul_(-1.25).add_(0.5)
    ref()
    eager()
    byz = replay()
    byz_single = replay_single()
    if step == 2:
      captured()                                                  # an eager search between two replays
      torch.cuda.synchronize()
      assert torch.equal(_bits(captured.record), _bits(eager.record)), gar
      byz = replay()
    torch.cuda.synchronize()
    what = (gar, step)
    searches = 1 + (step + 1) + (2 if step >= 2 else 0)           # warm-up, one replay per step, then step 2's eager + replay
    assert captured._fx.epoch == exchanges * searches and _flags_hold(captured._fx), what
    for got, got_byz, out in ((captured, byz, captured._shard.out), (single, byz_single, single._shard.out),
                              (eager, eager.byz, eager._shard.out)):
      assert torch.equal(_bits(got.record[:-1]), _bits(ref.record[:-1])), (what, got.exchange, got.record, ref.record)
      assert _status(got.record) == _status(ref.record), what
      assert torch.equal(_bits(got_byz), _bits(ref.byz)), what
      assert torch.equal(_bits(out), _bits(ref._out)), what
    assert captured.result() == ref.result(), what

def _local_fx(sharded, n, device, world=1, rank=0, buffers=None):
  fx = sharded.FusedExchange.__new__(sharded.FusedExchange)
  fx.n, fx.device, fx.group, fx.world, fx.rank, fx.epoch = n, device, None, world, rank, 0
  fx.buffer = torch.zeros(2 * n * n + FLAG_WORDS, dtype=torch.float64, device=device) if buffers is None else buffers[rank]
  fx.peer_base = [fx.buffer.data_ptr()] if buffers is None else [b.data_ptr() for b in buffers]
  return fx

def _fused_plan(sharded, fx, gar, rows, **kw):
  """ `ShardedPlan(exchange="fused")` over the emulated exchange `fx` (registered for the construction only). """
  key = (fx.n, fx.device.index, id(None))
  assert key not in sharded._fused
  sharded._fused[key] = fx
  try:
    plan = sharded.ShardedPlan(gar, rows, exchange="fused", **kw)
  finally:
    del sharded._fused[key]
  assert plan.exchange == "fused" and plan._fx is fx
  return plan

@pytest.mark.parametrize("gar,kw", [("krum", dict(f=5)), ("krum", dict(f=5, m=3)), ("bulyan", dict(f=5))])
def test_one_rank_plan_graph_is_the_plan(gar, kw):
  from byzantinemomentum_b200 import engine, sharded
  n, d = 25, 20011
  rows = _honest(n, d, 53)
  device = rows[0].device
  fx = _local_fx(sharded, n, device)
  plan = _fused_plan(sharded, fx, gar, rows, **kw)
  single = sharded.ShardedPlan(gar, rows, exchange="nccl", **kw)
  ref = engine.Plan(gar, rows, **kw)
  replay, replay_single = plan.graph(), single.graph()
  assert fx.epoch == 1 and _flags_hold(fx)
  calls = 1
  for step in range(6):
    rows[step % n].mul_(-1.5).add_(0.25)
    ref()
    if step % 2:
      out = plan()                                                # eager calls interleave with replays
    else:
      out = replay()
    out_single = replay_single()
    calls += 1
    torch.cuda.synchronize()
    what = (gar, kw, step)
    assert fx.epoch == calls and _flags_hold(fx), what
    assert torch.equal(_bits(out), _bits(ref.out)) and torch.equal(_bits(out_single), _bits(ref.out)), what
    assert torch.equal(plan.selection, ref.selection) and torch.equal(single.selection, ref.selection), what
    assert int(plan.status.item()) == 0, what
  # coordinate-wise: the plan of engine.Plan
  median = sharded.ShardedPlan("median", rows)
  replay = median.graph()
  want = engine.Plan("median", rows)()
  torch.cuda.synchronize()
  assert torch.equal(_bits(replay()), _bits(want))

@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("gar", ["krum", "bulyan"])
def test_emulated_plan_replays_are_the_by_value_calls(gar, R):
  """ R ranks' plans on one GPU, twice: one set replaying its graph, one calling by value.  Before each rank's
  replay (and call) every other rank's slot holds that rank's phase-A block and every flag it waits on is set. """
  from byzantinemomentum_b200 import engine, sharded
  n, f, d = 25, 5, 4099
  full = _honest(n, d, 71 + R)
  per_rank = _shards(full, R, True)
  device = full[0].device
  harness = [_Ranks(R, n), _Ranks(R, n)]                          # [graph, by value]
  plans = [[_fused_plan(sharded, _local_fx(sharded, n, device, R, r, h.buf), gar, per_rank[r], f=f) for r in range(R)]
           for h in harness]
  def blocks():
    return [engine.pairdist_partial(rows).reshape(-1).clone() for rows in per_rank]
  # graph(): the warm-up is an eager exchange at epoch 1 on every rank
  values = blocks()
  replays = [None] * R
  def warm(r):
    replays[r] = plans[0][r].graph()
  harness[0].exchange(1, values, warm, "warm-up")
  for step in range(3):
    for rows in per_rank:
      rows[step].mul_(-1.5).add_(0.25)
    values = blocks()
    epoch = step + 2
    _exchange_next(harness[0], epoch, values, lambda r: replays[r](), f"{gar} R={R} replay {step}")
    for p in plans[1]:
      p._fx.epoch = epoch - 1
    harness[1].exchange(epoch, values, lambda r: plans[1][r](), f"{gar} R={R} call {step}")
    torch.cuda.synchronize()
    for r in range(R):
      a, b = plans[0][r], plans[1][r]
      assert a._fx.epoch == epoch and b._fx.epoch == epoch
      assert torch.equal(_bits(a.out), _bits(b.out)), (gar, R, step, r)
      assert torch.equal(a.selection, b.selection) and torch.equal(a.status, b.status), (gar, R, step, r)

def test_graph_refuses_p2p_and_multi_rank_nccl():
  from byzantinemomentum_b200 import sharded
  n, d = 11, 1031
  rows = _honest(n, d, 3)
  plan = sharded.ShardedPlan("krum", rows, f=2, exchange="nccl")
  plan.exchange = "p2p"                                           # as chosen on a node with symmetric memory
  with pytest.raises(ValueError, match="'p2p'"):
    plan.graph()
  plan.exchange, plan.world = "nccl", 2
  with pytest.raises(ValueError, match="'nccl' on 2 ranks"):
    plan.graph()
  avg, att = _direction(rows[:8], "identical")
  search = sharded.ShardedLineSearch("krum", rows[:8], 3, 3, avg, att, 4, exchange="nccl")
  search.world = 2
  with pytest.raises(ValueError, match="'nccl' on 2 ranks"):
    search.graph()
  assert plan._graph is None and search._graph is None            # refused before any warm-up or capture
