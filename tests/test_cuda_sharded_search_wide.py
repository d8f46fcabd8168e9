# coding: utf-8
"""GPU tests of the d-sharded line search against Multi-Krum, Bulyan, Aksel and CGE above 64 rows
(`sharded.ShardedLineSearch(..., wide=True)`, include/byzagg_distance_search_shards.h).

  * One rank, "nccl" and "fused": the record, the status word, `byz` and the rule's last output are those of
    `engine.LineSearch` (`bz_distance_line_search`), bit for bit, at n = 65, 66, 96, 97, 100, 127 and 128, with
    unique-row counts that give 1, 3 and 6 passes, small and large f_real, both kinds, `negative`, 1, 2 and 16
    evaluations, d = 1, 1031 (rows off the 16-byte grid) and 4099.
  * `bz_distance_partial_reuse`: after every evaluation `part` is `bz_distance_partial`'s block of the same rows, bit
    for bit, for every pass shape, with `mode_out` saying which passes ran; unaligned rows, rows that are not the
    previous call's with one new row, and a changed unique count run the full passes.
  * R = 2, 3, 4, 8 ranks on "nccl", emulated on one GPU (the all-gathers replaced by `torch.stack`), shards as
    unaligned views, at the 64-float pitch of `GradientShards`, and empty: the same trace on every rank, the x
    sequence of `line_maximize`, the `byz` shards concatenating to the one-GPU `byz`, every y within 1e-6 of the fp64
    score of the concatenated output.
  * R = 2, 3, 4 on "fused" with the `_Ranks` harness of tests/test_cuda_search_peers.py: every rank publishes the
    "nccl" stage's block and share, and holds its trace, status and `byz`; the `_next` calls across the 2^32 wrap.
  * `graph()` replays equal the eager calls, on a buffer of its own and on one shared with `ShardedPlan` and
    `ShardedAntiCGE`.
  * Bulyan's status on the reference's wide stacks (NaN and inf rows) reaches every rank; d = 1,310,922 on one rank.
  * K2'-star (`bz_rowshare_star`, libbyzagg_star.so): part[c0, n) is `k2_rowshare_wide`'s (bz_distance_partial, CGE),
    bit for bit, at every n in 65..128, for c0 = n - 1 and small c0, at d = 0, 1, 31, 1031 and 1,310,922 (the grid at
    its caps), part[0, c0) untouched; the wide CGE search calls it from its second evaluation on."""

import ctypes
import math

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"

from conftest import Golden
from test_cuda_distance_search import _candidate, _direction, _f_decl, _honest, _xs_of
from test_cuda_search_peers import _Ranks
from test_cuda_sharded_graph import U32, _exchange_next, _fused_plan, _local_fx, _own_epoch
from test_cuda_sharded_search import _bits, _shards, _status
from test_distance_wide_abi import WD_DIR

GARS = ["krum", "bulyan", "aksel", "cge"]
KRUM, BULYAN = 5, 6

def _f_reals(n):
  """ Small and large f_real: n - 40 leaves 41 unique rows (one pass); 1 and n // 10 leave more than 64 (3 or 6). """
  return sorted({1, max(1, n // 10), n - 40})

@pytest.mark.parametrize("n", [65, 66, 96, 97, 100, 127, 128])
@pytest.mark.parametrize("gar", GARS)
def test_one_rank_is_the_single_gpu_search(gar, n):
  from byzantinemomentum_b200 import engine, sharded
  for f_real in _f_reals(n):
    nh = n - f_real
    f = _f_decl(gar, n, f_real)
    for d, offset in ((1, 0), (1031, 1), (4099, 0)):
      honest = _honest(nh, d, 7 + d + n + f_real, offset)
      for kind, negative, evals in (("identical", True, 16), ("identical", False, 1), ("identical", False, 2),
                                    ("empire-strict", False, 16)):
        avg, att = _direction(honest, kind)
        ref = engine.LineSearch(gar, honest, f_real, f, avg, att, evals, negative=negative, kind=kind)
        ref()
        for exchange in ("nccl", "fused"):
          got = sharded.ShardedLineSearch(gar, honest, f_real, f, avg, att, evals, negative=negative, kind=kind,
                                          exchange=exchange, wide=True)
          assert got.exchange == exchange and got._shard.wide
          byz = got()
          torch.cuda.synchronize()
          what = (gar, n, f_real, d, offset, kind, negative, evals, exchange)
          assert torch.equal(_bits(got.record[:-1]), _bits(ref.record[:-1])), (what, got.record, ref.record)
          assert _status(got.record) == _status(ref.record), what
          assert torch.equal(_bits(byz), _bits(ref.byz)), what
          assert torch.equal(_bits(got._shard.out), _bits(ref._out)), what
          if exchange == "fused":
            assert got._fx.epoch == 2 * evals, what

def test_auto_is_nccl_and_without_wide_nothing_changes():
  from byzantinemomentum_b200 import sharded
  honest = _honest(90, 1031, 3)
  avg, att = _direction(honest, "identical")
  assert sharded.ShardedLineSearch("krum", honest, 10, 10, avg, att, 4, wide=True).exchange == "nccl"
  with pytest.raises(ValueError, match="at most 64 rows"):
    sharded.ShardedLineSearch("krum", honest, 10, 10, avg, att, 4)
  # up to 64 rows `wide` is the default search
  small = sharded.ShardedLineSearch("krum", honest[:40], 5, 5, avg, att, 4, wide=True)
  assert not small._shard.wide and small._shard._tables.shape == (2, 64 * 64)

# ---- bz_distance_partial_reuse -------------------------------------------------------------------------------------

def _call(fn, *args):
  from byzantinemomentum_b200 import _lib
  _lib.check(fn(*args), fn.__name__)

def _partial(rows, part, ws):
  from byzantinemomentum_b200 import _lib
  n, d = len(rows), rows[0].numel()
  ptrs = (ctypes.c_void_p * n)(*[r.data_ptr() for r in rows])
  _call(_lib.lib().bz_distance_partial, KRUM, ptrs, n, None, d, part.data_ptr(), ws.data_ptr(), ws.numel(),
        torch.cuda.current_stream().cuda_stream)

def _reuse(rule, rows, part, old_index, tables_in, u_old, tables_out, ws):
  from byzantinemomentum_b200 import _lib
  n, d = len(rows), rows[0].numel()
  ptrs = (ctypes.c_void_p * n)(*[r.data_ptr() for r in rows])
  index = None if old_index is None else (ctypes.c_int32 * n)(*old_index)
  mode = ctypes.c_int(-9)
  _call(_lib.lib().bz_distance_partial_reuse, rule, ptrs, n, d, part.data_ptr(), index,
        None if tables_in is None else tables_in.data_ptr(), u_old, tables_out.data_ptr(), ctypes.byref(mode),
        ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
  return mode.value

# (nh, f_real): unique rows u = nh + 1 -> 1 pass (u = 41), 3 passes (u = 66, 81, 96), 6 passes (u = 97, 101, 128)
SHAPES = [(40, 30), (65, 1), (80, 20), (95, 2), (96, 1), (100, 20), (127, 1)]

@pytest.mark.parametrize("size", SHAPES, ids=lambda s: f"nh{s[0]}_freal{s[1]}")
def test_partial_reuse_is_bz_distance_partial_after_every_evaluation(size):
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  nh, f_real = size
  n = nh + f_real
  ws = torch.empty(int(lib.bz_distance_workspace_bytes(n)), dtype=torch.uint8, device=DEV)
  tables = torch.empty((2, int(lib.bz_distance_pass_tables_bytes()) // 8), dtype=torch.float64, device=DEV)
  for d, offset in ((40_009, 0), (1031, 1)):
    honest = _honest(nh, d, 41 + n + d, offset)
    base = torch.empty(d + offset, device=DEV)
    byz = base[offset:]
    rows = honest + [byz] * f_real
    old_index = list(range(nh)) + [-1] * f_real
    u = nh + 1
    avg, att = _direction(honest, "identical")
    aligned = offset == 0
    for k, x in enumerate((0., 0.5, 7., -2.)):
      byz.copy_(avg + x * att)
      rule = KRUM if k % 2 else BULYAN
      got = torch.full((n * n,), math.nan, dtype=torch.float64, device=DEV)
      want = torch.empty(n * n, dtype=torch.float64, device=DEV)
      if k == 0:
        mode = _reuse(rule, rows, got, None, None, 0, tables[0], ws)
      else:
        mode = _reuse(rule, rows, got, old_index, tables[(k - 1) % 2], u, tables[k % 2], ws)
      _partial(rows, want, ws)
      torch.cuda.synchronize()
      assert mode == (1 if k > 0 and aligned else 0), (size, d, k, mode)
      assert torch.equal(_bits(got), _bits(want)), (size, d, k)
    # in place (tables_in == tables_out), then the fallbacks to the full passes
    byz.copy_(avg - att)
    last = tables[1]
    for old, u_old, star in ((old_index, u, aligned),
                             (list(range(nh)) + [-1] * f_real, u - 1, False),             # another unique count
                             ([0] + list(range(nh - 1)) + [-1] * f_real, u, False),       # a kept row moved
                             ([-1] * n, u, False),                                        # no kept row
                             (None, u, False)):
      got = torch.full((n * n,), math.nan, dtype=torch.float64, device=DEV)
      want = torch.empty(n * n, dtype=torch.float64, device=DEV)
      mode = _reuse(KRUM, rows, got, old, last, u_old, last, ws)
      _partial(rows, want, ws)
      torch.cuda.synchronize()
      assert mode == (1 if star else 0), (size, d, u_old, mode)
      assert torch.equal(_bits(got), _bits(want)), (size, d, u_old)

def test_partial_reuse_on_an_empty_shard_and_aliased_honest_rows():
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  n = 100
  ws = torch.empty(int(lib.bz_distance_workspace_bytes(n)), dtype=torch.uint8, device=DEV)
  tables = torch.empty((2, int(lib.bz_distance_pass_tables_bytes()) // 8), dtype=torch.float64, device=DEV)
  empty = [torch.empty(0, device=DEV) for _ in range(n)]
  part = torch.full((n * n,), math.nan, dtype=torch.float64, device=DEV)
  assert _reuse(KRUM, empty, part, [0] * 90 + [-1] * 10, tables[0], 91, tables[1], ws) == -1
  torch.cuda.synchronize()
  assert torch.all(part == 0.)
  # honest rows that alias one another: their self distances come from the kept tables
  honest = _honest(60, 4099, 5)
  honest = honest + honest[:30]
  byz = torch.empty(4099, device=DEV)
  rows = honest + [byz] * 10
  first = {}
  old_index = [first.setdefault(g.data_ptr(), len(first)) for g in honest] + [-1] * 10
  u = len(first) + 1
  for k, x in enumerate((1., 3.)):
    byz.copy_(honest[0] * x)
    got = torch.empty(n * n, dtype=torch.float64, device=DEV)
    want = torch.empty(n * n, dtype=torch.float64, device=DEV)
    mode = _reuse(BULYAN, rows, got, old_index if k else None, tables[0] if k else None, u if k else 0, tables[k], ws)
    _partial(rows, want, ws)
    torch.cuda.synchronize()
    assert mode == k and torch.equal(_bits(got), _bits(want)), k

# ---- R ranks on "nccl" ---------------------------------------------------------------------------------------------

def _emulate(gar, honest, f_real, f, avg, att, R, pitched, evals=16, negative=False, kind="identical"):
  """ R ShardedLineSearch instances on one GPU driven through the stages; returns (instances, the concatenated rule
  output of every evaluation). """
  from byzantinemomentum_b200 import sharded
  vectors = honest + [avg] + ([att] if att is not None else [])
  per_rank = _shards(vectors, R, pitched)
  nh = len(honest)
  inst = [sharded.ShardedLineSearch(gar, rows[:nh], f_real, f, rows[nh], rows[nh + 1] if att is not None else None, evals,
                                    negative=negative, kind=kind, wide=True) for rows in per_rank]
  outs = []
  for k in range(evals):
    parts = [s.evaluate(k) for s in inst]
    blocks = torch.stack(parts)
    parts = [s.conclude(blocks) for s in inst]
    outs.append(torch.cat([s._shard.out for s in inst]).clone())
    scores = torch.stack(parts).reshape(R)
    for s in inst:
      s.step(k, scores)
  for s in inst:
    s.finish()
  torch.cuda.synchronize()
  return inst, outs

@pytest.mark.parametrize("R", [2, 3, 4, 8])
@pytest.mark.parametrize("gar", GARS)
def test_emulated_ranks_agree_and_match_one_gpu(gar, R):
  from byzantinemomentum_b200 import engine
  for nh, f_real in ((90, 10), (120, 8)):
    n = nh + f_real
    f = _f_decl(gar, n, f_real)
    for d, pitched in ((4099, False), (4099, True), (R - 1, False)):
      honest = _honest(nh, d, 5 + R + d + n)
      avg, att = _direction(honest, "identical")
      inst, outs = _emulate(gar, honest, f_real, f, avg, att, R, pitched)
      what = (gar, R, n, d, pitched)
      record = inst[0].record
      for s in inst[1:]:
        assert torch.equal(_bits(s.record[:-1]), _bits(record[:-1])), what
        assert _status(s.record) == _status(record), what
      factor, trace = inst[0].result()
      xs, ys = [x for x, _ in trace], [y for _, y in trace]
      assert [x.hex() for x in _xs_of(ys)] == [x.hex() for x in xs], what
      ref = engine.LineSearch(gar, honest, f_real, f, avg, att, 16)
      ref()
      byz = torch.cat([s.byz for s in inst])
      assert torch.equal(_bits(byz), _bits(avg + factor * att)), what
      for (x, y), out in zip(trace, outs):
        want = float(((out - avg).double() ** 2).sum())
        assert abs(y - want) <= 1e-6 * abs(want) + 1e-30, (what, x, y, want)
      plain = engine.Plan(gar, honest + [_candidate(avg, att, xs[-1], False, "identical")] * f_real, f=f)()
      assert torch.equal(_bits(outs[-1]), _bits(plain)), what
      if d > R:
        factor_one, _ = ref.result()
        assert factor == factor_one and torch.equal(_bits(byz), _bits(ref.byz)), what

@pytest.mark.parametrize("path", sorted(WD_DIR.glob("golden_wd_*.npz")), ids=lambda p: p.stem)
def test_bulyan_status_reaches_every_rank(path):
  """ The reference's wide stacks (NaN and inf rows among them): the honest rows of each stack, the search against
  Bulyan on 3 emulated ranks; every rank's status word is the one-GPU search's. """
  from byzantinemomentum_b200 import engine
  g = Golden(path)
  nh = g.nh
  n = g.rows.shape[0]
  if nh < 1 or nh >= n:
    pytest.skip("no Byzantine row in this stack")
  honest = [torch.from_numpy(g.rows[i]).to(DEV).contiguous() for i in range(nh)]
  f_real = n - nh
  f = (n - 3) // 4
  avg, att = _direction(honest, "identical")
  engine.config.strict_status = False
  try:
    ref = engine.LineSearch("bulyan", honest, f_real, f, avg, att, 6)
    ref()
    inst, _ = _emulate("bulyan", honest, f_real, f, avg, att, 3, False, evals=6)
    want = _status(ref.record)
    for s in inst:
      assert _status(s.record) == want, (path.stem, _status(s.record), want)
  finally:
    engine.config.strict_status = True

# ---- R ranks on "fused" --------------------------------------------------------------------------------------------

def _emulate_fused(gar, honest, f_real, f, avg, att, R, evals=16):
  """ R fused and R collective stages on one GPU, driven exchange by exchange: the first search passes the epochs by
  value, the second takes them from the flags (the `_next` calls, tests/test_cuda_sharded_graph.py's harness) and
  crosses the 2^32 wrap. """
  from byzantinemomentum_b200 import sharded
  n = len(honest) + f_real
  vectors = honest + [avg, att]
  per_rank = _shards(vectors, R, True)
  nh = len(honest)
  def make(rows):
    return sharded._SearchShard(gar, rows[:nh], f_real, f, rows[nh], rows[nh + 1], evals, False, "identical", R, wide=True)
  fused = [make(rows) for rows in per_rank]
  coll = [make(rows) for rows in per_rank]
  ranks = _Ranks(R, n)
  for r, shard in enumerate(fused):
    shard.fuse(ranks.fx[r])
  epoch = U32 - 2 * evals - 7
  for search in range(2):
    by_value = search == 0
    if search > 0:
      for rows in per_rank:                                       # new honest content, same tensors
        for i in range(0, nh, 7):
          rows[i].mul_(-1.5).add_(0.25)
    for k in range(evals):
      tag = f"{gar} R={R} search {search} k={k}"
      parts = [c.evaluate(k).clone() for c in coll]
      epoch += 1
      e = epoch
      if by_value:
        ranks.exchange(e, parts, lambda r: fused[r].evaluate_fused(k, e), f"{tag} rule")
      else:
        _exchange_next(ranks, e % U32, parts, lambda r: fused[r].evaluate_fused(k, None), f"{tag} rule")
      shares = [c.conclude(torch.stack(parts)) for c in coll]
      torch.cuda.synchronize()
      for r, (a, b) in enumerate(zip(fused, coll)):
        assert torch.equal(a._meta[:n], b._meta[:n]), f"{tag}: rank {r} selection"
        assert torch.equal(_bits(a.out), _bits(b.out)), f"{tag}: rank {r} rule output"
      epoch += 1
      e = epoch
      values = [s.reshape(1) for s in shares]
      if by_value:
        ranks.exchange(e, values, lambda r: fused[r].score_fused(k, e), f"{tag} score")
      else:
        _exchange_next(ranks, e % U32, values, lambda r: fused[r].score_fused(k, None), f"{tag} score")
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
      assert _status(a.record) == _status(b.record) == 0, what
      assert torch.equal(_bits(a.byz), _bits(b.byz)), what
  return fused, coll

@pytest.mark.parametrize("R", [2, 3, 4])
@pytest.mark.parametrize("gar", GARS)
def test_emulated_fused_ranks_are_the_collective_stages(gar, R):
  nh, f_real = 90, 10
  n = nh + f_real
  for d in (4099, R - 1):
    honest = _honest(nh, d, 17 + R + d)
    avg, att = _direction(honest, "identical")
    fused, _ = _emulate_fused(gar, honest, f_real, _f_decl(gar, n, f_real), avg, att, R, evals=8)
    for s in fused[1:]:
      assert torch.equal(_bits(s.record[:-1]), _bits(fused[0].record[:-1])), (gar, R, d)

# ---- graphs --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("gar", GARS)
def test_graph_replays_the_eager_search(gar):
  from byzantinemomentum_b200 import engine, sharded
  nh, f_real, d, evals = 90, 10, 30_011, 8
  f = _f_decl(gar, nh + f_real, f_real)
  honest = _honest(nh, d, 31)
  avg, att = _direction(honest, "identical")
  for exchange in ("nccl", "fused"):
    search = sharded.ShardedLineSearch(gar, honest, f_real, f, avg, att, evals, negative=True, exchange=exchange, wide=True)
    ref = engine.LineSearch(gar, honest, f_real, f, avg, att, evals, negative=True)
    replay = search.graph()
    for step in range(3):
      honest[step].mul_(-1.25).add_(0.5)
      ref()
      replay() if step % 2 == 0 else search()
      torch.cuda.synchronize()
      what = (gar, exchange, step)
      assert torch.equal(_bits(search.record[:-1]), _bits(ref.record[:-1])), what
      assert torch.equal(_bits(search.byz), _bits(ref.byz)), what
      if exchange == "fused":
        assert search._fx.epoch == 2 * evals * (step + 2) and _own_epoch(search._fx) == search._fx.epoch, what

@pytest.mark.parametrize("gar", ["krum", "cge"])
def test_buffer_shared_with_a_plan_and_the_attack_against_cge(gar):
  """ A plan of 100 rows, the attack against CGE of 100 honest rows and a search of 100 rows on one buffer, replays
  and eager calls interleaved: each keeps its bits, and the epoch counts every exchange. """
  from byzantinemomentum_b200 import engine, sharded
  n, nh, f_real, d, evals = 100, 90, 10, 4099, 6
  f = _f_decl(gar, n, f_real)
  honest = _honest(nh, d, 43)
  avg, att = _direction(honest, "identical")
  rows = _honest(n, d, 47)
  fx = _local_fx(sharded, n, torch.device(DEV))
  plan = _fused_plan(sharded, fx, gar, rows, f=f)
  attack = sharded.ShardedAntiCGE(rows, 24, 24, exchange="fused")
  attack._fuse(fx)
  search = sharded.ShardedLineSearch(gar, honest, f_real, f, avg, att, evals, negative=True, exchange="fused", wide=True)
  search._fx = fx
  search._shard.fuse(fx)
  ref_plan = engine.Plan(gar, rows, f=f)
  ref_attack = sharded.ShardedAntiCGE(rows, 24, 24, exchange="nccl")
  ref_search = engine.LineSearch(gar, honest, f_real, f, avg, att, evals, negative=True)
  plan_replay, attack_replay, search_replay = plan.graph(), attack.graph(), search.graph()
  epoch = 1 + 2 + 2 * evals
  assert fx.epoch == epoch and _own_epoch(fx) == epoch
  for step in range(4):
    rows[step].mul_(-1.5).add_(0.25)
    honest[step].mul_(-1.25).add_(0.5)
    ref_plan()
    ref_search()
    want = ref_attack()
    out = plan() if step % 2 else plan_replay()
    got = attack_replay() if step % 2 else attack()
    search_replay() if step % 2 == 0 else search()
    epoch += 1 + 2 + 2 * evals
    torch.cuda.synchronize()
    assert fx.epoch == epoch and _own_epoch(fx) == epoch, step
    assert torch.equal(_bits(out), _bits(ref_plan.out)) and torch.equal(plan.selection, ref_plan.selection), step
    assert torch.equal(_bits(got[0]), _bits(want[0])), step
    assert torch.equal(_bits(search.record[:-1]), _bits(ref_search.record[:-1])), step
    assert torch.equal(_bits(search.byz), _bits(ref_search.byz)), step

def test_headline_size_on_one_rank():
  from byzantinemomentum_b200 import engine, sharded
  nh, f_real, d = 90, 10, 1_310_922
  honest = _honest(nh, d, 9)
  avg, att = _direction(honest, "identical")
  for gar in GARS:
    f = _f_decl(gar, nh + f_real, f_real)
    ref = engine.LineSearch(gar, honest, f_real, f, avg, att, 16, negative=True)
    ref()
    got = sharded.ShardedLineSearch(gar, honest, f_real, f, avg, att, 16, negative=True, wide=True)
    got()
    torch.cuda.synchronize()
    assert torch.equal(_bits(got.record[:-1]), _bits(ref.record[:-1])), gar
    assert torch.equal(_bits(got.byz), _bits(ref.byz)), gar

# ---- K2'-star (bz_rowshare_star, libbyzagg_star.so) ----------------------------------------------------------------

def _star(rows, c0, part, ws):
  from byzantinemomentum_b200 import _lib
  n, d = len(rows), rows[0].numel()
  ptrs = (ctypes.c_void_p * n)(*[r.data_ptr() for r in rows])
  _call(_lib.star_lib().bz_rowshare_star, ptrs, n, c0, d, part.data_ptr(), ws.data_ptr(), ws.numel(),
        torch.cuda.current_stream().cuda_stream)

@pytest.mark.parametrize("d", [0, 1, 31, 1031, 1_310_922])
def test_star_pass_is_k2_rowshare_wide_at_every_n(d):
  """ part[c0, n) of bz_rowshare_star is bz_distance_partial(BZ_RULE_CGE)'s, bit for bit, and part[0, c0) is left as it
  was, at every n in 65..128, for c0 = n - 1 and small c0; d = 1,310,922 puts the grid at its caps. """
  from byzantinemomentum_b200 import _lib
  CGE = 9
  gen = torch.Generator(device=DEV).manual_seed(d + 5)
  honest = torch.randn(127, d, device=DEV, generator=gen) * torch.linspace(0.5, 3., 127, device=DEV)[:, None]
  base = torch.empty(d + 1, device=DEV)
  cand = base[1:] if d % 2 else base[:d]                       # off the 16-byte grid for odd d
  cand.copy_(torch.randn(d, device=DEV, generator=gen) * 2.5)
  ws = torch.empty(int(_lib.lib().bz_distance_workspace_bytes(128)), dtype=torch.uint8, device=DEV)
  star_ws = torch.empty(int(_lib.star_lib().bz_rowshare_star_workspace_bytes(128)), dtype=torch.uint8, device=DEV)
  for n in range(65, 129):
    for c0 in sorted({1, 3, n // 2, n - 1}):
      rows = [honest[i] for i in range(c0)] + [cand] * (n - c0)
      ptrs = (ctypes.c_void_p * n)(*[r.data_ptr() for r in rows])
      want = torch.empty(n, dtype=torch.float64, device=DEV)
      _call(_lib.lib().bz_distance_partial, CGE, ptrs, n, None, d, want.data_ptr(), ws.data_ptr(), ws.numel(),
            torch.cuda.current_stream().cuda_stream)
      got = torch.full((n,), math.nan, dtype=torch.float64, device=DEV)
      got[:c0] = -1.5
      _star(rows, c0, got, star_ws)
      torch.cuda.synchronize()
      assert torch.equal(_bits(got[c0:]), _bits(want[c0:])), (n, c0, d)
      assert torch.all(got[:c0] == -1.5), (n, c0, d)

def test_cge_search_reads_the_candidate_alone_after_the_first_evaluation():
  """ The wide CGE search issues bz_distance_partial at its first evaluation and bz_rowshare_star after. """
  from byzantinemomentum_b200 import _lib, sharded
  honest = _honest(90, 4099, 13)
  avg, att = _direction(honest, "identical")
  search = sharded.ShardedLineSearch("cge", honest, 10, 10, avg, att, 4, wide=True)
  shard = search._shard
  assert shard._phase_a_call(0)[0] is _lib.lib().bz_distance_partial
  for k in (1, 2, 3):
    fn, args = shard._phase_a_call(k)
    assert fn is _lib.star_lib().bz_rowshare_star and args[1:3] == (100, 90)
