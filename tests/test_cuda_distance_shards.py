# coding: utf-8
"""The d-sharded phases of Multi-Krum, Bulyan, Aksel and CGE up to 128 rows on the GPU
(include/byzagg_distance_shards.h, `sharded.ShardedPlan` above 64 rows).  R ranks are emulated on one GPU as
column shards (`sharded.shard_bounds`) of the same rows: phase A per shard, the R blocks stacked in rank order,
phase B, phase C per shard, the shards concatenated.

  * One rank: the phases, and `ShardedPlan` with its `graph()` replay, are `bz_distance` / `engine.Plan` bit for
    bit in output, selection and status.
  * R = 2, 3, 8: the selection is the single-GPU one (seeded stacks whose margins are wide) and the oracle's, the
    output is then the single-GPU output bit for bit, and phase B run twice gives the same bits.  The unique rows
    fit one pass, three or six.
  * Shards that start 4 bytes past a 16-byte boundary (the cp.async distance kernel), a rank with an empty shard,
    rows holding NaN or inf, a degenerate Bulyan stack.
  * Up to 64 rows the phases give the bits of the 64-row phase calls."""

import ctypes

import numpy as np
import pytest

from test_cuda_distance_wide import CODES, call, check_against_oracle, device_rows, stack

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

def _lib():
  from byzantinemomentum_b200 import _lib
  return _lib.lib()

def _ptrs(rows):
  return (ctypes.c_void_p * len(rows))(*[r.data_ptr() for r in rows])

def _stream(dev):
  return torch.cuda.current_stream(dev).cuda_stream

def _ok(code):
  assert code == 0, _lib().bz_last_error().decode()

def rank_rows(rows, R):
  """ The R ranks' rows: columns shard_bounds(d, R, r) of every row, as views (aliased rows stay one tensor). """
  from byzantinemomentum_b200 import sharded
  d = rows[0].numel()
  return [[g[lo:hi] for g in rows] for lo, hi in (sharded.shard_bounds(d, R, r) for r in range(R))]

def _median(rows):
  """ This shard's coordinate-wise median (Aksel's centre), or None for an empty shard. """
  d = rows[0].numel()
  if d == 0:
    return None
  out = torch.empty(d, dtype=torch.float32, device=rows[0].device)
  _ok(_lib().bz_coordinate(1, _ptrs(rows), len(rows), 0, d, out.data_ptr(), _stream(out.device)))
  return out

def phase_a(gar, rows, ws):
  """ bz_distance_partial on one shard: its block (n x n or n fp64). """
  lib, n, d, dev = _lib(), len(rows), rows[0].numel(), rows[0].device
  part = torch.full((n * n if gar in ("krum", "bulyan", "brute") else n,), 7., dtype=torch.float64, device=dev)
  center = _median(rows) if gar == "aksel" else None
  _ok(lib.bz_distance_partial(CODES[gar], _ptrs(rows), n, None if center is None else center.data_ptr(), d,
                              part.data_ptr(), ws.data_ptr(), ws.numel(), _stream(dev)))
  return part

def phase_b(gar, blocks, n, f, m, mode):
  """ bz_distance_select on the stacked blocks: (order, status) as device tensors. """
  meta = torch.full((n + 1,), -1, dtype=torch.int32, device=blocks.device)
  _ok(_lib().bz_distance_select(CODES[gar], blocks.data_ptr(), blocks.shape[0], n, f, m, mode, meta.data_ptr(),
                                meta.data_ptr() + 4 * n, _stream(blocks.device)))
  return meta

def phase_c(gar, rows, f, m, mode, meta):
  lib, n, d, dev = _lib(), len(rows), rows[0].numel(), rows[0].device
  out = torch.full((d,), 7., dtype=torch.float32, device=dev)
  status = meta.data_ptr() + 4 * n if gar in ("bulyan", "brute") else None
  _ok(lib.bz_distance_reduce(CODES[gar], _ptrs(rows), n, f, m, mode, meta.data_ptr(), status, d, out.data_ptr(), _stream(dev)))
  return out

def emulate(gar, rows, R, f, m=None, mode=0):
  """ The three phases on R emulated ranks: (concatenated output, order, status) as numpy, the stacked blocks,
  and the order and status of a second phase B. """
  n = len(rows)
  m = (n - f - 2 if m is None else m) if gar in ("krum", "bulyan") else 0
  shards = rank_rows(rows, R)
  ws = torch.empty(_lib().bz_distance_workspace_bytes(n), dtype=torch.uint8, device=rows[0].device)
  blocks = torch.stack([phase_a(gar, s, ws) for s in shards])
  meta = phase_b(gar, blocks, n, f, m, mode)
  again = phase_b(gar, blocks, n, f, m, mode)
  out = torch.cat([phase_c(gar, s, f, m, mode, meta) for s in shards])
  torch.cuda.synchronize()
  assert torch.equal(meta, again), f"{gar}: phase B is not deterministic"
  return out.cpu().numpy(), meta[:n].cpu().numpy(), int(meta[n].item()), blocks

def same_bits(a, b):
  return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))

RULES = (("krum", None, 0), ("krum", 3, 0), ("bulyan", None, 0), ("aksel", None, 0), ("aksel", None, 1), ("cge", None, 0))

@pytest.mark.parametrize("n", [65, 100, 128])
def test_one_rank_is_bz_distance(n):
  x, nh = stack(n, n // 5, 1031, seed=2000 + n)
  rows = device_rows(x, nh)
  f = (n - 3) // 4
  for gar, m, mode in RULES:
    got, order, status, _ = emulate(gar, rows, 1, f, m, mode)
    want = call(gar, rows, f, m, mode)
    assert same_bits(got, want[0]) and np.array_equal(order, want[1]) and status == want[2], (gar, m, mode)

@pytest.mark.parametrize("n,nb,d", [(80, 30, 4099), (65, 13, 4096), (100, 24, 4099), (128, 0, 2053), (128, 30, 4099)])
@pytest.mark.parametrize("R", [2, 3, 8])
def test_ranks_select_the_single_gpu_rows(n, nb, d, R):
  """ 80 rows of which 30 alias: 51 unique rows, one pass; 65 and 77 unique rows: three passes; 128 and 99:
  six.  d = 4099 and 2053 put shards 4 bytes past a 16-byte boundary. """
  x, nh = stack(n, nb, d, seed=3000 + n + R + nb)
  rows = device_rows(x, nh)
  for f in sorted({1, (n - 3) // 4, min(nb, (n - 3) // 4)}):
    for gar, m, mode in RULES + (("bulyan", 1, 0),):
      what = f"{gar} m={m} mode={mode} n={n} f={f} R={R}"
      got, order, status, _ = emulate(gar, rows, R, f, m, mode)
      want = call(gar, rows, f, m, mode)
      assert np.array_equal(order, want[1]) and status == want[2], what
      assert same_bits(got, want[0]), what
      check_against_oracle(gar, x, nh, got, order, status, f, m, "mid" if mode == 0 else "n-f", what)

@pytest.mark.parametrize("n", [65, 128])
def test_a_rank_with_an_empty_shard(n):
  """ d = 7 on 8 ranks: the last rank's shard is empty; it publishes zeros and still joins. """
  x, nh = stack(n, n // 5, 7, seed=4000 + n)
  rows = device_rows(x, nh)
  f = (n - 3) // 4
  for gar, m, mode in RULES:
    got, order, status, blocks = emulate(gar, rows, 8, f, m, mode)
    assert torch.count_nonzero(blocks[7]).item() == 0, gar
    want = call(gar, rows, f, m, mode)
    assert np.array_equal(order, want[1]) and status == want[2] and same_bits(got, want[0]), gar

@pytest.mark.parametrize("n,f", [(100, 20), (97, 23), (128, 31)])
def test_nan_and_inf_rows_and_a_degenerate_bulyan(n, f):
  """ NaN Byzantine rows (with f below their count Bulyan is degenerate: the status word and the NaN output of
  bz_distance), and an honest row with one +inf coordinate on one rank. """
  for kind in ("nan", "inf"):
    x, nh = stack(n, n // 4, 1031, seed=5000 + n, kind="nan" if kind == "nan" else "spread")
    if kind == "inf":
      x[3, 700] = np.inf
    rows = device_rows(x, nh)
    for gar, m, mode in RULES:
      for R in (1, 3):
        got, order, status, _ = emulate(gar, rows, R, f, m, mode)
        want = call(gar, rows, f, m, mode)
        what = f"{gar} {kind} n={n} f={f} R={R}"
        assert np.array_equal(order, want[1]) and status == want[2] and same_bits(got, want[0]), what
        if gar == "bulyan" and kind == "nan" and n // 4 >= f + 2:
          # more NaN rows than f + 1: every score holds an infinite distance
          assert status == 2 and np.isnan(got).all(), what

@pytest.mark.parametrize("n", [11, 25, 64])
def test_up_to_64_rows_the_phases_are_the_64_row_phase_calls(n):
  from byzantinemomentum_b200 import engine
  lib = _lib()
  x, nh = stack(n, n // 5, 4099, seed=6000 + n)
  rows = device_rows(x, nh)
  dev = rows[0].device
  st = _stream(dev)
  f = (n - 3) // 4
  ws = torch.empty(lib.bz_workspace_bytes(n), dtype=torch.uint8, device=dev)
  for gar, m, mode in RULES + (("brute", None, 0),):
    if gar == "brute" and n > 11:
      continue
    rule = engine._rule(gar, n, f, m, "mid" if mode == 0 else "n-f")
    mm = rule.m if gar in ("krum", "bulyan") else 0
    shards = rank_rows(rows, 2)
    new = emulate(gar, rows, 2, f, m, mode)
    # the 64-row phase calls, as the d-sharded path made them before
    blocks = []
    for s in shards:
      part = torch.full_like(new[3][0], 7.)
      if rule.pair:
        _ok(lib.bz_pairdist_partial(_ptrs(s), n, s[0].numel(), part.data_ptr(), ws.data_ptr(), ws.numel(), st))
      else:
        center = _median(s) if gar == "aksel" else None
        _ok(lib.bz_rowdist_partial(_ptrs(s), n, None if center is None else center.data_ptr(), s[0].numel(), part.data_ptr(),
                                   ws.data_ptr(), ws.numel(), st))
      blocks.append(part)
    blocks = torch.stack(blocks)
    assert torch.equal(blocks.view(torch.int64), new[3].view(torch.int64)), gar
    meta = torch.full((n + 1,), -1, dtype=torch.int32, device=dev)
    o, s_ = meta.data_ptr(), meta.data_ptr() + 4 * n
    if gar == "krum":
      _ok(lib.bz_krum_select(blocks.data_ptr(), 2, n, f, o, st))
    elif gar == "bulyan":
      _ok(lib.bz_bulyan_select(blocks.data_ptr(), 2, n, f, mm, o, s_, st))
    elif gar == "brute":
      _ok(lib.bz_brute_select(blocks.data_ptr(), 2, n, f, o, s_, st))
    else:
      _ok(lib.bz_rowdist_select(blocks.data_ptr(), 2, n, int(gar == "cge"), o, st))
    outs = []
    for s in shards:
      d = s[0].numel()
      out = torch.full((d,), 7., dtype=torch.float32, device=dev)
      if gar == "bulyan":
        _ok(lib.bz_bulyan_reduce(_ptrs(s), n, f, mm, o, s_, d, out.data_ptr(), st))
      else:
        _ok(lib.bz_average_selected(_ptrs(s), n, o, rule.count, int(rule.zero_init), float(rule.count),
                                    s_ if rule.status else None, d, out.data_ptr(), st))
      outs.append(out)
    torch.cuda.synchronize()
    length = rule.length
    assert np.array_equal(meta[:length].cpu().numpy(), new[1][:length]), gar
    if rule.status:
      assert int(meta[n].item()) == new[2], gar
    assert same_bits(torch.cat(outs).cpu().numpy(), new[0]), gar

@pytest.mark.parametrize("n", [65, 100, 128])
def test_sharded_plan_on_one_rank_is_plan(n):
  from byzantinemomentum_b200 import engine, sharded
  x, nh = stack(n, n // 5, 4099, seed=7000 + n)
  rows = device_rows(x, nh)
  f = (n - 3) // 4
  for gar, kw in (("krum", {}), ("krum", dict(m=5)), ("bulyan", {}), ("aksel", {}), ("aksel", dict(mode="n-f")), ("cge", {})):
    plan = sharded.ShardedPlan(gar, rows, f=f, **kw)
    assert plan.exchange == "nccl", gar
    ref = engine.Plan(gar, rows, f=f, **kw)
    want = ref().clone()
    for replayed in (False, True):
      plan.out.fill_(7.)
      got = plan.graph()() if replayed else plan()
      torch.cuda.synchronize()
      what = f"{gar} {kw} n={n} replayed={replayed}"
      assert torch.equal(got.view(torch.int32), want.view(torch.int32)), what
      assert torch.equal(plan.selection, ref.selection), what
      assert (plan.status is None) == (ref.status is None), what
      if plan.status is not None:
        assert int(plan.status.item()) == int(ref.status.item()) == 0, what
  # the rows change in place: the plan follows
  plan = sharded.ShardedPlan("krum", rows, f=f)
  rows[0].mul_(-3.)
  want = engine.Plan("krum", rows, f=f)()
  assert torch.equal(plan().view(torch.int32), want.view(torch.int32))

def test_sharded_plan_refusals_above_64_rows():
  from byzantinemomentum_b200 import sharded
  x, nh = stack(100, 20, 64, seed=8000)
  rows = device_rows(x, nh)
  for exchange in ("p2p", "fused"):
    with pytest.raises(ValueError, match="at most MAX_N = 64 rows, not n = 100"):
      sharded.ShardedPlan("krum", rows, f=10, exchange=exchange)
  with pytest.raises(ValueError, match="maximum of 64"):
    sharded.ShardedPlan("brute", rows, f=1)
  with pytest.raises(ValueError, match="maximum of 128"):
    sharded.ShardedPlan("krum", rows + rows[:29], f=1)
