# coding: utf-8
"""GPU tests of the attacks' line search on the d-sharded path (`sharded.ShardedLineSearch`,
include/byzagg_search_shards.h).

  * One rank: the trace, the factor, the Byzantine gradient and the rule's last output are those of
    `engine.LineSearch`, bit for bit, for every rule at n in {11, 25, 51}, both candidate kinds,
    `negative` on and off, 1, 2 or 16 evaluations and several d (1, odd, rows off the 16-byte grid).
  * Phase A with distance reuse gives the block of the same call without a cache, bit for bit, for every
    shape of the ring (n = 11, 25, 30, 51); unaligned rows fall back to a full pass with the same block.
  * R ranks emulated on one GPU (R instances driven stage by stage, the all-gathers replaced by
    `torch.stack`), shards as unaligned views and at the 64-float pitch of `GradientShards`, with empty
    shards when d < R: every rank holds the same trace, its x sequence is `line_maximize` fed with its y
    values, the Byzantine shards and the last rule output concatenate to the single-GPU results, and
    every y is the fp64 score of the concatenated output within 1e-6.
  * The status words of Bulyan and brute reach every rank.
The seeded rows have distinct spreads, so the selections have margins: Aksel's and CGE's keys and the
distance tables are summed in another order on the sharded path."""

import ctypes
import math

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"

import line_oracle
from test_cuda_linesearch import F_OF, _candidate, _direction, _honest

GARS = ["average", "median", "trmean", "phocas", "meamed", "krum", "bulyan", "brute", "aksel", "cge"]

def _bits(t):
  return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int64)

def _status(record):
  return int(record[-1:].view(torch.int32)[0])

def _xs_of(ys):
  xs = []
  line_oracle.line_maximize(lambda x: (xs.append(x), ys[len(xs) - 1])[1], len(ys))
  return xs

@pytest.mark.parametrize("n", [11, 25, 51])
@pytest.mark.parametrize("gar", GARS)
def test_one_rank_is_the_single_gpu_search(gar, n):
  from byzantinemomentum_b200 import engine, sharded
  f = F_OF[(gar, n)]
  nh = n - f
  for d, offset in ((1, 0), (1031, 1), (4099, 0)):
    honest = _honest(nh, d, 7 + d + n, offset)
    for kind, negative in (("identical", False), ("identical", True), ("empire-strict", False)):
      avg, att = _direction(honest, kind)
      for evals in (1, 2, 16):
        ref = engine.LineSearch(gar, honest, f, f, avg, att, evals, negative=negative, kind=kind)
        ref()
        got = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, evals, negative=negative, kind=kind)
        byz = got()
        torch.cuda.synchronize()
        what = (gar, n, d, offset, kind, negative, evals)
        assert torch.equal(_bits(got.record[:-1]), _bits(ref.record[:-1])), (what, got.record, ref.record)
        assert _status(got.record) == _status(ref.record), what
        assert torch.equal(_bits(byz), _bits(ref.byz)), what
        assert torch.equal(_bits(got._shard.out), _bits(ref._out)), what

def _phase_a(rows, part, old_index, cache_in, u_old, cache_out, ws):
  from byzantinemomentum_b200 import _lib
  n, d = len(rows), rows[0].numel()
  mode = ctypes.c_int(-9)
  ptrs = (ctypes.c_void_p * n)(*[r.data_ptr() for r in rows])
  index = None if old_index is None else (ctypes.c_int32 * n)(*old_index)
  rc = _lib.lib().bz_pairdist_partial_reuse(ptrs, n, d, part.data_ptr(), index, cache_in, u_old, cache_out,
                                            ctypes.byref(mode), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
  _lib.check(rc, "bz_pairdist_partial_reuse")
  return mode.value

@pytest.mark.parametrize("n", [11, 25, 30, 51])
def test_phase_a_with_reuse_gives_the_block_without_it(n):
  from byzantinemomentum_b200 import _lib
  ws = torch.empty(int(_lib.lib().bz_workspace_bytes(n)), dtype=torch.uint8, device=DEV)
  tables = torch.empty((3, 64 * 64), dtype=torch.float64, device=DEV)
  f = 5 if n > 11 else 3
  nh = n - f
  for d, offset in ((200_003, 0), (4099, 0), (1031, 1)):
    honest = _honest(nh, d, 41 + n + d, offset)
    base = torch.empty(d + offset, device=DEV)
    byz = base[offset:]
    rows = honest + [byz] * f
    old_index = list(range(nh)) + [-1] * f
    u = nh + 1
    avg, att = _direction(honest, "identical")
    byz.copy_(avg - 3. * att)
    first = torch.empty((n, n), dtype=torch.float64, device=DEV)
    mode0 = _phase_a(rows, first, None, None, 0, tables[0].data_ptr(), ws)
    for x in (0.5, 7.):
      byz.copy_(avg + x * att)                          # a new candidate at the same address
      reused = torch.empty((n, n), dtype=torch.float64, device=DEV)
      fresh = torch.empty((n, n), dtype=torch.float64, device=DEV)
      mode1 = _phase_a(rows, reused, old_index, tables[0].data_ptr(), u, tables[1].data_ptr(), ws)
      mode2 = _phase_a(rows, fresh, None, None, 0, tables[2].data_ptr(), ws)
      torch.cuda.synchronize()
      aligned = offset == 0
      assert (mode0, mode1, mode2) == ((0, 1, 0) if aligned else (-1, -1, -1)), (n, d, mode0, mode1, mode2)
      assert torch.equal(_bits(reused), _bits(fresh)), (n, d, x)
      # the layout of the original rows, and the distances themselves
      full = torch.stack(rows).double()
      want = ((full[:, None, :] - full[None, :, :]) ** 2).sum(-1) if d < 10_000 else None
      assert torch.equal(torch.tril(reused), torch.zeros_like(reused))
      assert torch.all(reused[nh:, nh:] == 0.)          # aliases of one finite row
      if want is not None:
        upper = torch.triu(want, 1)
        assert torch.allclose(reused, upper, rtol=1e-5, atol=0.), (n, d)
      tables[0].copy_(tables[1])

def _shards(full, R, pitched):
  """ R lists of this rank's columns of the vectors `full`: views of them (unaligned starts), or copies at
  the 64-float pitch of GradientShards. """
  from byzantinemomentum_b200 import sharded
  d = full[0].numel()
  out = []
  for r in range(R):
    lo, hi = sharded.shard_bounds(d, R, r)
    if pitched:
      pitch = ((d + R - 1) // R + 63) // 64 * 64
      buf = torch.zeros((len(full), pitch), device=DEV)
      out.append([buf[i, :hi - lo].copy_(v[lo:hi]) for i, v in enumerate(full)])
    else:
      out.append([v[lo:hi] for v in full])
  return out

def _emulate(gar, honest, f, avg, att, R, pitched, evals=16, negative=False, kind="identical", wide=False):
  """ R ShardedLineSearch instances on one GPU driven through the stages (`wide`: as they take it); returns
  (instances, the concatenated rule output of every evaluation). """
  from byzantinemomentum_b200 import sharded
  vectors = honest + [avg] + ([att] if att is not None else [])
  per_rank = _shards(vectors, R, pitched)
  nh = len(honest)
  inst = [sharded.ShardedLineSearch(gar, rows[:nh], f, f, rows[nh], rows[nh + 1] if att is not None else None, evals,
                                    negative=negative, kind=kind, wide=wide) for rows in per_rank]
  outs = []
  for k in range(evals):
    parts = [s.evaluate(k) for s in inst]
    if inst[0]._shard.distance:
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

@pytest.mark.parametrize("R", [2, 3, 8])
@pytest.mark.parametrize("gar", GARS)
def test_emulated_ranks_agree_and_match_one_gpu(gar, R):
  import byzantinemomentum_b200 as bz
  n = 25
  f = F_OF[(gar, n)]
  nh = n - f
  for d, pitched in ((4099, False), (4099, True), (R - 1, False)):
    honest = _honest(nh, d, 5 + R + d)
    avg, att = _direction(honest, "identical")
    inst, outs = _emulate(gar, honest, f, avg, att, R, pitched)
    what = (gar, R, d, pitched)
    record = inst[0].record
    for s in inst[1:]:
      assert torch.equal(_bits(s.record[:-1]), _bits(record[:-1])), what
      assert _status(s.record) == _status(record), what
    factor, trace = inst[0].result()
    xs, ys = [x for x, _ in trace], [y for _, y in trace]
    assert [x.hex() for x in _xs_of(ys)] == [x.hex() for x in xs], what
    byz = torch.cat([s.byz for s in inst])
    assert torch.equal(_bits(byz), _bits(avg + factor * att)), what
    for (x, y), out in zip(trace, outs):
      ref = float(((out - avg).double() ** 2).sum())
      assert abs(y - ref) <= 1e-6 * abs(ref) + 1e-30, (what, x, y, ref)
    plain = bz.gars[gar](gradients=honest + [_candidate(avg, att, xs[-1], False, "identical")] * f, f=f)
    assert torch.equal(_bits(outs[-1]), _bits(plain)), what

@pytest.mark.parametrize("gar", ["bulyan", "brute"])
def test_status_words_reach_every_rank(gar):
  from byzantinemomentum_b200 import engine, _lib
  n, f = 11, 2 if gar == "bulyan" else 3
  honest = _honest(n - f, 515, 21)
  for k in range(6):                               # non-finite rows (all on rank 0): no finite scores / subsets
    honest[k] = honest[k].clone()
    honest[k][k] = math.nan
  avg, att = _direction(honest[6:], "identical")
  inst, _ = _emulate(gar, honest, f, avg, att, 2, False)
  want = _lib.STATUS_DEGENERATE if gar == "bulyan" else _lib.STATUS_NO_FINITE_SET
  for s in inst:
    assert _status(s.record) == want, gar
    with pytest.raises(TypeError if gar == "bulyan" else AssertionError):
      s.result()
  engine.config.strict_status = False
  try:
    factor, trace = inst[1].result()
  finally:
    engine.config.strict_status = True
  assert math.isnan(trace[0][1]) and factor == 0.
  assert [x for x, _ in trace] == _xs_of([y for _, y in trace])

def test_line_search_on_one_rank():
  from byzantinemomentum_b200 import engine, sharded
  honest = _honest(20, 30_011, 3)
  avg, att = _direction(honest, "identical")
  factor, byz = sharded.line_search("krum", honest, 5, 5, avg, att, 16, negative=True)
  want, want_byz = engine.line_search("krum", honest, 5, 5, avg, att, 16, negative=True)
  assert factor == want and torch.equal(byz, want_byz)
