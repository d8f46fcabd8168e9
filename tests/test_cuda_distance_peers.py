# coding: utf-8
"""GPU tests of `ShardedPlan(exchange="fused")` where its exchange runs in a kernel of its own: Multi-Krum, Bulyan,
Aksel and CGE above 64 rows (`bz_distance_partial` into a staging buffer, `bz_distance_select_peers` of
libbyzagg_peers.so, `bz_distance_reduce`), and Aksel and CGE up to 64 rows (`bz_rowdist_peers`).

R = 1, 2, 3, 4, 8 ranks are emulated on ONE GPU with the harness of test_cuda_search_peers.py: each rank has its own
buffer in the `FusedExchange` layout; before each rank's call every other rank's slot holds its phase-A block and
every flag the call waits on is set; no two grids at once.  Every rank's call must publish exactly
`bz_distance_partial`'s block into its slot and raise its flag on every rank, and its selection, status and output
shard must be the "nccl" phases' (`bz_distance_partial`, `bz_distance_select` over the R stacked blocks,
`bz_distance_reduce`) bit for bit; with R = 1 they are `engine.Plan`'s.  Rows: n = 65 to 128, distinct or with the
Byzantine rows aliased so that the unique rows take one, three or six passes, the golden stacks (NaN, inf, Bulyan's
failing status), shards with unaligned starts and empty shards.  The by-value and the `_next` calls, four steps
across the 2^32 epoch wrap, and `graph()` replays, alone and on a buffer shared with a `ShardedAntiCGE` or a
`ShardedLineSearch`.  No test waits for the peer timeout: every wait is satisfied by preset flags."""

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from conftest import Golden
from test_cuda_distance_shards import phase_a, phase_b, phase_c, rank_rows
from test_cuda_distance_wide import device_rows, stack
from test_distance_wide_abi import WD_DIR
from test_cuda_linesearch import _direction, _honest
from test_cuda_search_peers import _Ranks
from test_cuda_sharded_graph import U32, _exchange_next, _fused_plan, _local_fx, _own_epoch
from test_cuda_sharded_search import _bits

@pytest.fixture(autouse=True)
def _no_buffer_left_registered():
  """ Every plan here takes the emulated buffer registered for its construction only. """
  from byzantinemomentum_b200 import sharded
  before = dict(sharded._fused)
  yield
  assert sharded._fused == before

DEV = "cuda:0"
GARS = ["krum", "bulyan", "aksel", "cge"]

def _rules(gar, n):
  """ (f, plan keywords, m, mode of the C calls) of the rule's variants on n rows. """
  f = max(0, (n - 3) // 4)
  if gar == "krum":
    return [(f, dict(f=f), n - f - 2, 0), (f, dict(f=f, m=3), 3, 0)]
  if gar == "bulyan":
    return [(f, dict(f=f), n - f - 2, 0)] + ([(f, dict(f=f, m=1), 1, 0)] if n % 2 else [])
  if gar == "aksel":
    return [(f, dict(f=f, mode="mid"), 0, 0), (f, dict(f=f, mode="n-f"), 0, 1)]
  return [(f, dict(f=f), 0, 0)]

def _nccl(gar, shards, f, m, mode):
  """ The collective path on R emulated ranks: every rank's phase-A block, the order + status, every rank's output. """
  from byzantinemomentum_b200 import _lib
  n = len(shards[0])
  ws = torch.empty(_lib.lib().bz_distance_workspace_bytes(n), dtype=torch.uint8, device=DEV)
  blocks = [phase_a(gar, s, ws) for s in shards]
  meta = phase_b(gar, torch.stack(blocks), n, f, m, mode)
  outs = [phase_c(gar, s, f, m, mode, meta) for s in shards]
  return blocks, meta, outs

def _check(gar, plans, meta, outs, what):
  n = plans[0].n
  for r, p in enumerate(plans):
    assert torch.equal(p.selection, meta[:n]), (what, r)
    assert int(p.status.item()) == (int(meta[n].item()) if gar == "bulyan" else 0), (what, r)
    assert torch.equal(_bits(p.out), _bits(outs[r])), (what, r)

def _plans(gar, shards, kw, ranks):
  from byzantinemomentum_b200 import sharded
  n = len(shards[0])
  return [_fused_plan(sharded, _local_fx(sharded, n, torch.device(DEV), ranks.R, r, ranks.buf), gar, shards[r], **kw)
          for r in range(ranks.R)]

def _by_value(ranks, plans, epoch, values, what):
  for p in plans:
    p._fx.epoch = (epoch - 1) % U32
  ranks.exchange(epoch % U32, values, lambda r: plans[r](), what)

def _next(ranks, plans, epoch, values, what):
  from byzantinemomentum_b200 import engine
  def issue(r):
    with engine._on(plans[r].device):
      plans[r]._issue(engine._call, captured=True)
  _exchange_next(ranks, epoch % U32, values, issue, what)

def _steps(gar, full, R, call, epochs, change=True):
  """ The fused plans of every rule variant against the collective path, one exchange per epoch of `epochs`, the
  rows changed in place between steps. """
  n = len(full)
  shards = rank_rows(full, R)
  for f, kw, m, mode in _rules(gar, n):
    ranks = _Ranks(R, n)
    plans = _plans(gar, shards, kw, ranks)
    for k, epoch in enumerate(epochs):
      if k > 0 and change:
        full[(5 * k) % max(1, n // 2)].mul_(-1.5).add_(0.25)
      blocks, meta, outs = _nccl(gar, shards, f, m, mode)
      what = (gar, n, R, kw, epoch)
      call(ranks, plans, epoch, [b.reshape(-1) for b in blocks], what)
      torch.cuda.synchronize()
      _check(gar, plans, meta, outs, what)

def _stack_rows(n, unique, d, seed):
  """ n rows of which n - unique + 1 are one aliased Byzantine tensor (unique == n: all distinct). """
  x, nh = stack(n, n - unique + 1 if unique < n else 0, d, seed)
  return device_rows(x, nh)

def _uniques(n):
  return sorted({u for u in (40, 80, 110) if u < n} | {n})      # 1, 3 and 6 passes, and all distinct

@pytest.mark.parametrize("R", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("n", [65, 66, 96, 97, 100, 127, 128])
@pytest.mark.parametrize("gar", GARS)
def test_every_rank_has_the_nccl_bits(gar, n, R):
  if R > 3 and n not in (65, 100, 128):
    pytest.skip("4 and 8 ranks at the ends and the middle of the range")
  for unique in _uniques(n):
    full = _stack_rows(n, unique, 1031, seed=100 * n + unique + R)   # 1031 columns: unaligned shard starts
    _steps(gar, full, R, _by_value, (U32 - 1, U32, U32 + 1) if unique == n else (7,))

@pytest.mark.parametrize("R", [1, 2, 3, 4])
@pytest.mark.parametrize("n", [65, 97, 128])
@pytest.mark.parametrize("gar", GARS)
def test_next_calls_across_the_wrap(gar, n, R):
  """ The `_next` call derives each epoch from the flags alone: from a fresh buffer, and four steps across 2^32. """
  full = _stack_rows(n, n, 1031, seed=7 * n + R)
  _steps(gar, full, R, _next, (1, 2))
  _steps(gar, full, R, _next, (U32 - 2, U32 - 1, U32, U32 + 1))

@pytest.mark.parametrize("n", [65, 128])
@pytest.mark.parametrize("gar", GARS)
def test_empty_shards(gar, n):
  """ d = 9 over 4 ranks and d = 3 over 8: ranks with empty shards publish zeros and still join. """
  for d, R in ((9, 4), (3, 8)):
    full = _stack_rows(n, n, d, seed=n + d)
    _steps(gar, full, R, _by_value, (3,), change=False)
    _steps(gar, full, R, _next, (4,), change=False)

def _goldens():
  return [pytest.param(path, id=path.stem) for path in sorted(WD_DIR.glob("golden_wd_*.npz"))]

@pytest.mark.parametrize("path", _goldens())
def test_golden_stacks(path):
  """ The reference fixtures (NaN and inf rows, values near the fp32 limits, Bulyan's failing status) on 1, 2 and 3
  ranks: the fused plans are the collective path bit for bit. """
  g = Golden(path)
  rows = device_rows(g.rows, g.nh)
  n = len(rows)
  seen = set()
  for c in g.calls:
    gar, params = c["gar"], c["params"]
    if gar not in GARS:
      continue
    f, m_kw, mode = params["f"], params.get("m"), params.get("mode", "mid")
    key = (gar, f, m_kw, mode)
    if key in seen:
      continue
    seen.add(key)
    kw = dict(f=f) | ({} if m_kw is None else dict(m=m_kw)) | (dict(mode=mode) if gar == "aksel" else {})
    m = (n - f - 2 if m_kw is None else m_kw) if gar in ("krum", "bulyan") else 0
    for R in (1, 2, 3):
      shards = rank_rows(rows, R)
      ranks = _Ranks(R, n)
      plans = _plans(gar, shards, kw, ranks)
      blocks, meta, outs = _nccl(gar, shards, f, m, 1 if mode == "n-f" else 0)
      what = (path.stem, c["tag"], R)
      _by_value(ranks, plans, 5, [b.reshape(-1) for b in blocks], what)
      torch.cuda.synchronize()
      _check(gar, plans, meta, outs, what)
      if "raises" in c:
        assert gar == "bulyan" and int(plans[0].status.item()) == 2, what

@pytest.mark.parametrize("R", [1, 2, 3])
@pytest.mark.parametrize("n", [1, 2, 25, 64])
@pytest.mark.parametrize("gar", ["aksel", "cge"])
def test_aksel_and_cge_up_to_64_rows(gar, n, R):
  """ Aksel and CGE fused up to 64 rows run `bz_rowdist_peers`, whose exchange publishes phase A's n sums. """
  for d in (1031, 4096):
    full = _stack_rows(n, n if n < 25 else n - 4, d, seed=n + d + R)
    _steps(gar, full, R, _by_value, (U32, U32 + 1))
    _steps(gar, full, R, _next, (9, 10))

@pytest.mark.parametrize("gar,n", [("krum", 100), ("bulyan", 128), ("aksel", 65), ("cge", 97), ("aksel", 25), ("cge", 1)])
def test_one_rank_is_the_plan_and_its_graph(gar, n):
  """ One rank: eager calls and graph replays, interleaved, are `engine.Plan` bit for bit, with the rows changed in
  place between steps; `fx.epoch` stays the epoch the flags hold. """
  from byzantinemomentum_b200 import engine, sharded
  rows = _stack_rows(n, n if n < 3 else n - 5, 20011, seed=n)
  kw = dict(f=max(0, (n - 3) // 4))
  fx = _local_fx(sharded, n, torch.device(DEV))
  plan = _fused_plan(sharded, fx, gar, rows, **kw)
  assert (n, 0, id(None)) not in sharded._fused
  ref = engine.Plan(gar, rows, **kw)
  replay = plan.graph()
  assert fx.epoch == 1 and _own_epoch(fx) == 1
  calls = 1
  for step in range(6):
    rows[(3 * step) % max(1, n - 5)].mul_(-1.5).add_(0.25)
    ref()
    out = plan() if step % 2 else replay()
    calls += 1
    torch.cuda.synchronize()
    what = (gar, n, step)
    assert fx.epoch == calls and _own_epoch(fx) == calls, what
    assert torch.equal(_bits(out), _bits(ref.out)) and torch.equal(plan.selection, ref.selection), what
    assert int(plan.status.item()) == (0 if ref.status is None else int(ref.status.item())), what

@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("gar,n", [("krum", 100), ("bulyan", 97), ("aksel", 128), ("cge", 65), ("aksel", 25), ("cge", 64)])
def test_emulated_replays_are_the_by_value_calls(gar, n, R):
  """ R ranks' plans twice: one set replaying its graph (the `_next` call captured), one calling by value. """
  full = _stack_rows(n, n, 4099, seed=11 * n + R)
  shards = rank_rows(full, R)
  f, kw, m, mode = _rules(gar, n)[-1]
  harness = [_Ranks(R, n), _Ranks(R, n)]                          # [graph, by value]
  plans = [_plans(gar, shards, kw, h) for h in harness]
  blocks, _, _ = _nccl(gar, shards, f, m, mode)
  replays = [None] * R
  def warm(r):
    replays[r] = plans[0][r].graph()
  harness[0].exchange(1, [b.reshape(-1) for b in blocks], warm, "warm-up")
  for step in range(3):
    full[step].mul_(-1.5).add_(0.25)
    blocks, meta, outs = _nccl(gar, shards, f, m, mode)
    values = [b.reshape(-1) for b in blocks]
    epoch = step + 2
    _exchange_next(harness[0], epoch, values, lambda r: replays[r](), f"{gar} R={R} replay {step}")
    _by_value(harness[1], plans[1], epoch, values, f"{gar} R={R} call {step}")
    torch.cuda.synchronize()
    for r in range(R):
      assert plans[0][r]._fx.epoch == epoch and plans[1][r]._fx.epoch == epoch
    _check(gar, plans[0], meta, outs, (gar, n, R, step, "replay"))
    _check(gar, plans[1], meta, outs, (gar, n, R, step, "call"))

def test_buffer_shared_with_the_attack_against_cge():
  """ A plan of 100 rows and the attack against CGE of 100 honest rows on one buffer, replays and eager calls
  interleaved: each keeps its bits, and the epoch counts every exchange. """
  from byzantinemomentum_b200 import engine, sharded
  n = 100
  rows = _stack_rows(n, n, 20011, seed=97)
  fx = _local_fx(sharded, n, torch.device(DEV))
  plan = _fused_plan(sharded, fx, "krum", rows, f=24)
  attack = sharded.ShardedAntiCGE(rows, 24, 24, exchange="fused")
  attack._fuse(fx)
  collective = sharded.ShardedAntiCGE(rows, 24, 24, exchange="nccl")
  ref = engine.Plan("krum", rows, f=24)
  plan_replay, attack_replay = plan.graph(), attack.graph()
  epoch = 1 + 2
  assert fx.epoch == epoch and _own_epoch(fx) == epoch
  for step in range(6):
    rows[(3 * step) % n].mul_(-1.5).add_(0.25)
    ref()
    want = collective()
    out = plan() if step % 2 else plan_replay()
    epoch += 1
    got = attack() if step % 3 == 1 else attack_replay()
    epoch += 2
    torch.cuda.synchronize()
    assert fx.epoch == epoch and _own_epoch(fx) == epoch, step
    assert torch.equal(_bits(out), _bits(ref.out)) and torch.equal(plan.selection, ref.selection), step
    assert int(plan.status.item()) == 0, step
    assert torch.equal(_bits(got[0]), _bits(want[0])) and int(attack.status.item()) == 0, step

@pytest.mark.parametrize("gar", ["aksel", "cge"])
def test_buffer_shared_with_the_line_search(gar):
  """ Aksel or CGE on 25 rows and a line search against it on one buffer, replays interleaved. """
  from byzantinemomentum_b200 import engine, sharded
  n, f, d, evals = 25, 5, 4099, 8
  honest = _honest(n - f, d, 41)
  avg, att = _direction(honest, "identical")
  rows = honest + [avg] * f
  fx = _local_fx(sharded, n, torch.device(DEV))
  plan = _fused_plan(sharded, fx, gar, rows, f=f)
  search = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, evals, negative=True, exchange="fused")
  search._fx = fx
  search._shard.fuse(fx)
  ref_plan = engine.Plan(gar, rows, f=f)
  ref_search = engine.LineSearch(gar, honest, f, f, avg, att, evals, negative=True)
  plan_replay, search_replay = plan.graph(), search.graph()
  epoch = 1 + 2 * evals
  assert fx.epoch == epoch and _own_epoch(fx) == epoch
  for step in range(4):
    honest[step].mul_(-1.25).add_(0.5)
    ref_plan()
    ref_search()
    out = plan() if step % 2 else plan_replay()
    epoch += 1
    if step % 2:
      search_replay()
    else:
      search()
    epoch += 2 * evals
    torch.cuda.synchronize()
    assert fx.epoch == epoch and _own_epoch(fx) == epoch, step
    assert torch.equal(_bits(out), _bits(ref_plan.out)) and torch.equal(plan.selection, ref_plan.selection), step
    assert torch.equal(_bits(search.record[:-1]), _bits(ref_search.record[:-1])), step
    assert torch.equal(_bits(search.byz), _bits(ref_search.byz)), step
