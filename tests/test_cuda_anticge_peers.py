# coding: utf-8
"""GPU tests of the d-sharded attack against CGE with its exchanges over peer memory (`bz_anticge_peers`,
`bz_anticge_peers_next`, `sharded.ShardedAntiCGE(exchange="fused")`).

Ranks are emulated on ONE GPU with the harness of test_cuda_search_peers.py: each rank has its own buffer in the
`FusedExchange` layout, and before a rank's call every other rank's slot of exchange 1 holds its norm block, its slot
of exchange 2 its partial sum of squares, and every flag the call waits on is set; those values come from the
collective stages (`norms`, `sum`, `scale`).  No two grids run at once and no test waits for the peer timeout.

  * R = 1, 2, 3, 4 and nh = 1 ... 128 at maxpos = 0, the middle and nh - 1: each rank publishes the collective path's
    block and partial in the slots of its two epochs and signals both, and its shard, its order and its decision are
    the collective path's bit for bit; every rank has the same order.  Shards from `shard_bounds` (views with
    unaligned starts), and d = 9 over 4 ranks (an empty shard).  Both the by-value and the `_next` calls.
  * The recorded cases of `tests/golden/anticge/` within the bar of test_cuda_anticge.py, on one and three ranks; the
    NaN fill exchanges nothing.
  * Four steps across the 2^32 wrap with the rows changed in place between them.
  * `graph()`: one rank against eager calls and the collective path, emulated replays against by-value calls, and
    the epoch of a buffer shared with a `ShardedPlan`."""

import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import byzoracle as orc
from test_anticge_abi import close, goldens
from test_cuda_anticge import _rows
from test_cuda_search_peers import _Ranks, _s32
from test_cuda_sharded_graph import _fused_plan, _local_fx, _own_epoch

U32 = 1 << 32

def _bits(t):
  t = t.detach().contiguous()
  return t.view(torch.int32) if t.element_size() == 4 else t.view(torch.int64)

def _shards(full, R):
  from byzantinemomentum_b200 import sharded
  d = full[0].numel()
  return [[v[lo:hi] for v in full] for lo, hi in (sharded.shard_bounds(d, R, r) for r in range(R))]

def _order(attack):
  return attack._ws[:4 * attack._prep.n].view(torch.int32)

def _decision(attack):
  """ (factor, apply) K10 left in the workspace. """
  word = attack._ws[1024:1032]
  return float(word[:4].view(torch.float32).item()), int(word[4:].view(torch.int32).item())

def _expected_decision(blocks, partials, order, maxpos):
  """ bz_anticge_scale's decision from the gathered blocks [R, nh] and partials [R], in NumPy. """
  key = orc.fp32_norm(orc.sum_parts(blocks.cpu().numpy()))[int(order[maxpos])]
  key = float(key) if math.isfinite(key) else math.inf
  attnorm = float(orc.fp32_norm(orc.sum_parts(partials.cpu().numpy().reshape(-1, 1)))[0])
  if not attnorm > 0:
    return 1.0, 0
  with np.errstate(over="ignore"):
    return float(np.float32(-math.nextafter(key, 0) / attnorm)), 1

class _Emulated:
  """ R ranks of the fused attack over a `_Ranks` harness, next to R collective instances on the same shards. """
  def __init__(self, per_rank, f_decl, f_real, ranks=None):
    from byzantinemomentum_b200 import sharded
    self.R, self.nh = len(per_rank), len(per_rank[0])
    self.ranks = ranks if ranks is not None else _Ranks(self.R, self.nh)
    self.fused = [sharded.ShardedAntiCGE(rows, f_decl, f_real, exchange="fused") for rows in per_rank]
    self.coll = [sharded.ShardedAntiCGE(rows, f_decl, f_real, exchange="nccl") for rows in per_rank]
    for r, a in enumerate(self.fused):
      a._fuse(self.ranks.fx[r])
    self.maxpos = self.nh - f_decl
  def collective(self):
    """ The collective stages on every rank: (blocks [R, nh], partials [R]). """
    blocks = torch.stack([c.norms().clone() for c in self.coll])
    partials = torch.cat([c.sum(blocks).clone() for c in self.coll])
    for c in self.coll:
      c.scale(partials)
    return blocks, partials
  def step(self, epoch, call, tag):
    """ One step whose exchange 1 is at `epoch` (exchange 2 at epoch + 1): rank r's call(r) after the peers' slots
    and flags are set; the flags also hold the epoch a `_next` call must derive (own entries epoch - 2, epoch - 1). """
    blocks, partials = self.collective()
    torch.cuda.synchronize()
    ranks, nh = self.ranks, self.nh
    e1, e2 = epoch % U32, (epoch + 1) % U32
    s = e1 % 2
    for r in range(self.R):
      for p in range(self.R):
        ranks.flags(p, s).fill_(0 if e1 == 1 else _s32(e1 - 2))
        ranks.flags(p, 1 - s).fill_(_s32(e1 - 1))
      for p in range(self.R):
        if p != r:
          ranks.slot(p, s)[:nh].copy_(blocks[p])
          ranks.slot(p, 1 - s)[:1].copy_(partials[p:p + 1])
          ranks.flags(r, s)[p] = _s32(e1)
          ranks.flags(r, 1 - s)[p] = _s32(e2)
      ranks.slot(r, s)[:nh].fill_(float("nan"))
      ranks.slot(r, 1 - s)[:1].fill_(float("nan"))
      self.fused[r].status.fill_(-1)
      call(r)
      torch.cuda.synchronize()
      what = f"{tag}: rank {r}"
      assert torch.equal(_bits(ranks.slot(r, s)[:nh]), _bits(blocks[r])), f"{what} published other norm sums"
      assert torch.equal(_bits(ranks.slot(r, 1 - s)[:1]), _bits(partials[r:r + 1])), f"{what} published another partial"
      for p in range(self.R):
        assert int(ranks.flags(p, s)[r].item()) == _s32(e1), f"{what} did not signal rank {p} at {e1}"
        assert int(ranks.flags(p, 1 - s)[r].item()) == _s32(e2), f"{what} did not signal rank {p} at {e2}"
      assert int(self.fused[r].status.item()) == 0, what
    self.check(blocks, partials, tag)
  def check(self, blocks, partials, tag):
    order = self.coll[0].order
    want = _expected_decision(blocks, partials, order.cpu().tolist(), self.maxpos)
    for r, (a, c) in enumerate(zip(self.fused, self.coll)):
      what = f"{tag}: rank {r}"
      assert torch.equal(_order(a), c.order) and torch.equal(c.order, order), what
      assert torch.equal(_bits(a.byz), _bits(c.byz)), what
      got = _decision(a)
      assert got[1] == want[1] and np.float32(got[0]).view(np.uint32) == np.float32(want[0]).view(np.uint32), (what, got, want)
  def by_value(self, epoch):
    def call(r):
      self.fused[r]._fx.epoch = epoch - 1
      self.fused[r]()
      assert self.fused[r]._fx.epoch == epoch + 1
    return call
  def next_call(self, r):
    from byzantinemomentum_b200 import engine
    with engine._on(self.fused[r].device):
      self.fused[r]._issue(captured=True)

@pytest.mark.parametrize("R", [1, 2, 3, 4])
@pytest.mark.parametrize("nh", [1, 2, 7, 25, 64, 65, 100, 128])
def test_every_rank_has_the_collective_path_bits(nh, R):
  for d in ((4099, 9) if R == 4 else (4099,)):                       # d = 9 over 4 ranks: shards 3, 3, 3 and 0
    full = _rows(nh, d, 17 * nh + R + d)
    for maxpos in sorted({0, nh // 2, nh - 1}):
      em = _Emulated(_shards(full, R), nh - maxpos, 1)
      tag = f"nh={nh} R={R} d={d} maxpos={maxpos}"
      em.step(1, em.by_value(1), f"{tag} by value")                  # a fresh buffer
      em.step(3, em.next_call, f"{tag} next")

@pytest.mark.parametrize("path", goldens())
def test_goldens_on_one_and_three_ranks(path):
  z = np.load(path)
  full = [torch.from_numpy(r.copy()).to("cuda") for r in z["rows"]]
  f_decl, f_real = int(z["f_decl"]), int(z["f_real"])
  for R in (1, 3):
    em = _Emulated(_shards(full, R), f_decl, f_real)
    if f_real > f_decl:                                              # the NaN fill: no exchange, no epoch
      for r, a in enumerate(em.fused):
        out = a()
        assert a._fx.epoch == 0 and len(out) == f_real
      torch.cuda.synchronize()
      assert all(not b.any() for b in em.ranks.buf)
      got = torch.cat([a.byz for a in em.fused]).cpu().numpy()
      assert np.array_equal(got.view(np.uint32), np.full(got.size, 0x7fc00000, np.uint32))
      continue
    em.step(5, em.by_value(5), f"{path.stem} R={R}")
    if f_real == 0:
      continue
    assert _order(em.fused[0]).cpu().tolist() == z["order"].tolist()
    got = torch.cat([a.byz for a in em.fused]).cpu().numpy()
    assert close(got, z["out"]), (R, np.nanmax(np.abs(got - z["out"]) / np.abs(z["out"])))

@pytest.mark.parametrize("mode", ["by value", "next"])
@pytest.mark.parametrize("R,nh", [(2, 25), (3, 100)])
def test_four_steps_across_the_wrap(R, nh, mode):
  d = 20011
  full = _rows(nh, d, 5 + R)
  em = _Emulated(_shards(full, R), nh // 4, nh // 4)
  for step, epoch in enumerate((U32 - 2, U32, U32 + 2, U32 + 4)):   # exchanges 0xFFFFFFFE, 0xFFFFFFFF, 0, 1, ... 5
    if step > 0:
      for i in range(step, nh, 3):                                    # new content in the same tensors
        full[i].mul_(-1.5).add_(0.25)
    em.step(epoch, em.by_value(epoch) if mode == "by value" else em.next_call, f"step {step} at {epoch % U32:#x}")

def _flags_hold(fx):
  return _own_epoch(fx) == fx.epoch % U32

@pytest.mark.parametrize("nh", [25, 100])
def test_one_rank_graph_is_the_eager_call(nh):
  from byzantinemomentum_b200 import sharded
  d = 20011
  rows = _rows(nh, d, 41 + nh)
  f_decl = nh // 5
  captured = sharded.ShardedAntiCGE(rows, f_decl, 3, exchange="fused")
  eager = sharded.ShardedAntiCGE(rows, f_decl, 3, exchange="fused")
  single = sharded.ShardedAntiCGE(rows, f_decl, 3, exchange="nccl")
  plain = sharded.ShardedAntiCGE(rows, f_decl, 3)
  assert plain.exchange == "nccl" and captured._fx.world == 1
  replay, replay_single = captured.graph(), single.graph()
  fx = captured._fx
  assert fx.epoch == 2 and _flags_hold(fx)                           # the warm-up's eager call
  calls = 1
  for step in range(5):
    if step > 0:
      for i in range(step - 1, nh, 4):
        rows[i].mul_(-1.25).add_(0.5)
    want = plain()
    got = eager()
    if step == 2:
      captured()                                                     # an eager call between two replays
      calls += 1
    out, out_single = replay(), replay_single()
    calls += 1
    torch.cuda.synchronize()
    what = (nh, step)
    assert len(out) == 3 and out[0] is captured.byz and out_single[0] is single.byz, what
    assert fx.epoch == 2 * calls and _flags_hold(fx), what
    for o in (out, out_single, got):
      assert torch.equal(_bits(o[0]), _bits(want[0])), what
    assert torch.equal(_order(captured), plain.order) and int(captured.status.item()) == 0, what

@pytest.mark.parametrize("R", [2, 3])
def test_emulated_replays_are_the_by_value_calls(R):
  nh, d = 25, 4099
  full = _rows(nh, d, 71 + R)
  per_rank = _shards(full, R)
  graphs, calls = _Emulated(per_rank, 5, 5), _Emulated(per_rank, 5, 5)
  replays = [None] * R
  def warm(r):
    replays[r] = graphs.fused[r].graph()                             # one eager call at epochs 1, 2, then the capture
  graphs.step(1, warm, f"R={R} warm-up")
  for step in range(3):
    for i in range(step, nh, 5):
      full[i].mul_(-1.5).add_(0.25)
    epoch = 3 + 2 * step
    graphs.step(epoch, lambda r: replays[r](), f"R={R} replay {step}")
    calls.step(epoch, calls.by_value(epoch), f"R={R} call {step}")
    for r in range(R):
      a, b = graphs.fused[r], calls.fused[r]
      assert a._fx.epoch == b._fx.epoch == epoch + 1, (R, step, r)
      assert torch.equal(_bits(a.byz), _bits(b.byz)) and torch.equal(_order(a), _order(b)), (R, step, r)

def test_epochs_interleave_with_a_plan_on_the_same_buffer():
  from byzantinemomentum_b200 import engine, sharded
  n, d = 25, 20011
  rows = _rows(n, d, 97)
  device = rows[0].device
  fx = _local_fx(sharded, n, device)
  plan = _fused_plan(sharded, fx, "krum", rows, f=5)
  attack = sharded.ShardedAntiCGE(rows, 6, 6, exchange="fused")
  attack._fuse(fx)
  collective = sharded.ShardedAntiCGE(rows, 6, 6, exchange="nccl")
  ref = engine.Plan("krum", rows, f=5)
  plan_replay, attack_replay = plan.graph(), attack.graph()
  epoch = 1 + 2
  assert fx.epoch == epoch and _flags_hold(fx)
  for step in range(6):
    rows[(3 * step) % n].mul_(-1.5).add_(0.25)
    ref()
    want = collective()
    out = plan() if step % 2 else plan_replay()
    epoch += 1
    torch.cuda.synchronize()
    assert fx.epoch == epoch and _flags_hold(fx), step
    got = attack() if step % 3 == 1 else attack_replay()
    epoch += 2
    torch.cuda.synchronize()
    assert fx.epoch == epoch and _flags_hold(fx), step
    assert torch.equal(_bits(out), _bits(ref.out)) and torch.equal(plan.selection, ref.selection), step
    assert torch.equal(_bits(got[0]), _bits(want[0])) and int(attack.status.item()) == 0, step
