# coding: utf-8
"""GPU tests of the study metrics and of the attacks' line search against the coordinate-wise rules above 128 rows
(up to 1024: `bz_avg_dev_max_many`, `bz_line_search_many`, libbyzagg_many_tools.so).

  * K6-many at n from 129 to 1024 on the special values of tests/test_cuda_k1_edges.py (NaN, +-inf, -0,
    subnormals, ties), with aligned rows and mixed 4-byte offsets: the average bit-exact against the oracle and
    against `bz_coordinate_many`'s average, the scalars at the bar of tests/test_wide_study_abi.py; the reference's
    recorded outputs; d = 1, every tile edge, the ring wrapped at full depth and d = 1,310,922 at n = 1024;
    determinism; and the call of `bz_avg_dev_max` up to 128 rows.
  * The study block (`engine.study_step(..., many=True)`) at 300 rows against attack.py's statements, and
    `sharded.study_step(..., many=True)` over R = 1, 3 and 8 shards emulated on one GPU.
  * `engine.LineSearch(..., many=True)` for every coordinate-wise rule at n = 129, 300 and 1024 (the checks of
    tests/test_cuda_linesearch.py against `many_gars`), its bits at 100 rows, a CUDA graph of it,
    `ShardedLineSearch(..., many=True)` on one rank and on 3 emulated ranks, and the plugin's device search and
    study metrics with 300 rows."""

import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"

import line_oracle
from oracle import byzoracle as orc
from test_cuda_k1_edges import _device_rows, _stack
from test_cuda_linesearch import _candidate, _direction, _honest
from test_cuda_sharded_search import _bits, _shards, _status, _xs_of
from test_cuda_sharded_study import MOMENTUM, _inputs, _same, _scalars, AVERAGES
from test_cuda_study_step import _study_reference
from test_plugin_attacks import _aggregators, _attacks
from test_many_tools_abi import cases, load
from test_wide_study_abi import check

COORDINATE = ["average", "median", "trmean", "phocas", "meamed"]

def _study(rows):
  from byzantinemomentum_b200 import engine
  avg, norm_avg, norm_dev, norm_max = engine.compute_avg_dev_max(rows, many=True)
  return avg.cpu().numpy(), norm_avg, norm_dev, norm_max

@pytest.mark.parametrize("n", [129, 130, 255, 256, 257, 511, 512, 513, 777, 1023, 1024])
def test_study_metrics_every_bucket_edge_above_128(n):
  from byzantinemomentum_b200 import engine
  d = 1031
  for nonfinite in (True, False):
    x = _stack(n, d, 900 + n, nonfinite=nonfinite)
    want = orc.compute_avg_dev_max(list(x))
    for offsets in ((0,), (0, 1, 2, 3)):
      rows = _device_rows(x, offsets)
      check(_study(rows), *want)
      avg, _ = engine.avg_dev_max_many_async(rows)
      assert torch.equal(_bits(avg), _bits(engine.coordinate_many("average", rows))), (n, offsets)

@pytest.mark.parametrize("case", [c for c in cases() if c.values[0]["hi"] - c.values[0]["lo"] > 128])
def test_study_metrics_match_the_reference_above_128_rows(case):
  rows, avg, norm_avg, norm_dev, norm_max = load(case)
  check(_study([torch.from_numpy(np.ascontiguousarray(r)).to(DEV) for r in rows]), avg, norm_avg, norm_dev, norm_max)

@pytest.mark.parametrize("case", [c for c in cases() if 0 < c.values[0]["hi"] - c.values[0]["lo"] <= 128])
def test_the_fixture_splits_of_128_rows_or_fewer_take_bz_avg_dev_max(case):
  """ Those calls are `bz_avg_dev_max`'s: its bits, whatever they are (above 64 rows it keeps avg^2 below 2^-150,
  which the reference's fp32 norm drops: the `tiny` stack's 100 Byzantine rows show it). """
  from byzantinemomentum_b200 import engine
  rows = [torch.from_numpy(np.ascontiguousarray(r)).to(DEV) for r in load(case)[0]]
  a_avg, a = engine.avg_dev_max_async(rows)
  b_avg, b = engine.avg_dev_max_many_async(rows)
  assert torch.equal(_bits(a_avg), _bits(b_avg)) and torch.equal(a.view(torch.int64), b.view(torch.int64))

def _sizes():
  out = []
  for n, tc in ((200, 64), (400, 32), (1000, 16)):      # K6-many's columns per tile in the buckets of 256, 512, 1024
    # tile edges, and 20 tiles per CTA: the three-stage ring wrapped at full depth many times
    out += [(n, 1), (n, tc - 1), (n, tc), (n, tc + 1), (n, 132 * tc * 20 + 5)]
  return out + [(1024, 1_310_922)]

@pytest.mark.parametrize("n,d", _sizes())
def test_study_metrics_sizes(n, d):
  rng = np.random.default_rng(7 * n + d % 991)
  x = (rng.standard_normal((n, d)) * rng.uniform(0.1, 10., (n, 1))).astype(np.float32)
  want = orc.compute_avg_dev_max(list(x))
  base = torch.from_numpy(x).to(DEV)
  check(_study(list(base)), *want)
  if d > 1 and d < 100_000:
    check(_study(_device_rows(x, (1, 3))), *want)

def test_study_metrics_are_deterministic_and_take_1024_rows():
  from byzantinemomentum_b200 import engine
  for n in (129, 700, 1024):
    rows = [torch.randn(100_003, device=DEV) for _ in range(n)]
    a_avg, a = engine.avg_dev_max_many_async(rows)
    b_avg, b = engine.avg_dev_max_many_async(rows)
    assert a.shape == (n + 2,) and torch.equal(a, b) and torch.equal(a_avg, b_avg), n
  with pytest.raises(ValueError, match="maximum of 1024"):
    engine.avg_dev_max_many_async(rows + rows[:1])
  with pytest.raises(ValueError, match="maximum of 128"):
    engine.avg_dev_max_async(rows[:129])

@pytest.mark.parametrize("n", [1, 2, 64, 65, 128])
def test_up_to_128_rows_it_is_bz_avg_dev_max(n):
  from byzantinemomentum_b200 import engine
  rows = [torch.randn(50_021, device=DEV) for _ in range(n)]
  a_avg, a = engine.avg_dev_max_async(rows)
  b_avg, b = engine.avg_dev_max_many_async(rows)
  assert torch.equal(_bits(a_avg), _bits(b_avg)) and torch.equal(a.view(torch.int64), b.view(torch.int64)), n

@pytest.mark.parametrize("shared", [True, False])
def test_study_step_at_300_rows_matches_the_statements_of_attack_py(shared):
  from byzantinemomentum_b200 import engine
  d = 79_510
  sampleds, honests, attacks, defense, pasts = _inputs(300, 300 if shared else 280, 150, 3, d, shared)
  want, want_avg = _study_reference(sampleds, honests, attacks, defense, pasts, MOMENTUM)
  got = engine.study_step(sampleds, honests, attacks, defense, pasts, MOMENTUM, many=True)
  assert torch.allclose(got["sampled_grad_avg"], want_avg, rtol=1e-6, atol=1e-7)
  for key, ref in want.items():
    val = got[key]
    if math.isnan(ref):
      assert math.isnan(val), key
    else:
      assert abs(val - ref) <= 2e-5 * abs(ref) + 3e-6, (key, val, ref)
  with pytest.raises(ValueError, match="maximum of 128"):
    engine.study_step(sampleds, honests, attacks, defense, pasts, MOMENTUM)

@pytest.mark.parametrize("R", [1, 3, 8])
def test_sharded_study_step_at_300_rows(R):
  from byzantinemomentum_b200 import engine, sharded
  sampleds, honests, attacks, defense, pasts = _inputs(300, 300, 140, 2, 10_007, True)
  want = engine.study_step(sampleds, honests, attacks, defense, pasts, MOMENTUM, many=True)
  d = defense.numel()
  partials = []
  for r in range(R):
    lo, hi = sharded.shard_bounds(d, R, r)
    cut = lambda rows: [g[lo:hi] for g in rows]
    shard_s = cut(sampleds)
    partials.append(engine.study_partials(shard_s, shard_s, cut(attacks), defense[lo:hi], [(g[lo:hi], norm) for g, norm in pasts],
                                          many=True))
  vectors = [p.vector.tolist() for p in partials]
  ranks = [engine.study_finish(p, vectors, MOMENTUM) for p in partials]
  for res in ranks[1:]:
    for key, val in _scalars(ranks[0]).items():
      assert _same(res[key], val), (R, key, res[key], val)
  for key in AVERAGES:
    assert torch.equal(_bits(torch.cat([res[key] for res in ranks])), _bits(want[key])), (R, key)
  for key, ref in _scalars(want).items():
    val = _scalars(ranks[0])[key]
    if R == 1 or math.isnan(ref) or math.isinf(ref):
      assert _same(val, ref), (R, key, val, ref)
    else:
      assert abs(val - ref) <= 2e-5 * abs(ref) + 3e-6, (R, key, val, ref)
  got = sharded.compute_avg_dev_max(sampleds, many=True)
  assert got[0].shape == (d,) and torch.equal(_bits(got[0]), _bits(want["sampled_grad_avg"]))

def _plain(bz, gar, honest, byz, f_real, f):
  return bz.many_gars[gar](gradients=honest + [byz] * f_real, f=f)

def _check_search(bz, gar, honest, f_real, f, avg, att, evals, negative, kind):
  """ tests/test_cuda_linesearch.py's four checks of `LineSearch(..., many=True)`, `many_gars` the plain call. """
  from byzantinemomentum_b200 import engine
  search = engine.LineSearch(gar, honest, f_real, f, avg, att, evals, negative=negative, kind=kind, many=True)
  byz = search()
  factor, trace = search.result()
  xs = [x for x, _ in trace]
  ys = [y for _, y in trace]
  fed = []
  def scape(x):
    fed.append(x)
    return ys[len(fed) - 1]
  want_factor = line_oracle.line_maximize(scape, evals)
  assert [x.hex() for x in fed] == [x.hex() for x in xs], (gar, fed, xs)
  assert factor.hex() == float(want_factor).hex()
  plain_outs = []
  for x, y in trace:
    out = _plain(bz, gar, honest, _candidate(avg, att, x, negative, kind), f_real, f)
    plain_outs.append(out)
    ref = float(((out - avg).double() ** 2).sum())
    if math.isnan(ref):
      assert math.isnan(y), (gar, x, y)
    else:
      assert abs(y - ref) <= 1e-6 * abs(ref) + 1e-30, (gar, x, y, ref)
  assert torch.equal(search._out, plain_outs[-1]), (gar, xs[-1])
  final = avg + factor * att if kind == "identical" else avg.mul(-factor)
  assert torch.equal(byz, final), (gar, factor)
  host_xs, host_ys = [], []
  def eval_factor(x):
    aggregated = _plain(bz, gar, honest, _candidate(avg, att, x, negative, kind), f_real, f)
    aggregated.sub_(avg)
    y = aggregated.dot(aggregated).item()
    host_xs.append(x)
    host_ys.append(y)
    return y
  host_factor = line_oracle.line_maximize(eval_factor, evals)
  if host_factor != factor:
    k = next(i for i, (a, b) in enumerate(zip(host_xs, xs)) if a != b) - 1
    assert abs(host_ys[k] - ys[k]) <= 1e-5 * abs(ys[k]), (gar, k, host_ys, ys)
  return search

F_MANY = {129: (1, 60), 300: (1, 140), 1024: (1, 500)}     # n -> (small f_real, large f_real)

@pytest.mark.parametrize("n", [129, 300, 1024])
@pytest.mark.parametrize("gar", COORDINATE)
def test_line_search_above_128_rows(gar, n):
  import byzantinemomentum_b200 as bz
  for f_real in F_MANY[n]:
    f = f_real
    nh = n - f_real
    for d, offset in ((1031, 0), (1031, 1)):
      honest = _honest(nh, d, 19 + d + n + f_real, offset)
      for kind, negative in (("identical", True), ("identical", False), ("empire-strict", False)):
        avg, att = _direction(honest, kind)
        _check_search(bz, gar, honest, f_real, f, avg, att, 16, negative, kind)

@pytest.mark.parametrize("gar", COORDINATE)
def test_line_search_many_is_bz_line_search_at_100_rows(gar):
  from byzantinemomentum_b200 import engine
  honest = _honest(80, 4099, 31)
  for kind in ("identical", "empire-strict"):
    avg, att = _direction(honest, kind)
    plain = engine.LineSearch(gar, honest, 20, 20, avg, att, 16, negative=True, kind=kind)
    many = engine.LineSearch(gar, honest, 20, 20, avg, att, 16, negative=True, kind=kind, many=True)
    plain()
    many()
    torch.cuda.synchronize()
    assert torch.equal(_bits(plain.record[:-1]), _bits(many.record[:-1])) and _status(plain.record) == _status(many.record)
    assert torch.equal(_bits(plain.byz), _bits(many.byz)) and torch.equal(_bits(plain._out), _bits(many._out))

def test_line_search_graph_above_128_rows():
  from byzantinemomentum_b200 import engine
  for gar, kind in (("median", "identical"), ("trmean", "empire-strict"), ("average", "identical")):
    honest = _honest(250, 30_011, 43)
    avg, att = _direction(honest, kind)
    search = engine.LineSearch(gar, honest, 50, 50, avg, att, 16, negative=True, kind=kind, many=True)
    search()
    torch.cuda.synchronize()
    eager_record, eager_byz = search.record.clone(), search.byz.clone()
    replay = search.graph()
    for _ in range(2):
      search.record.fill_(-1.)
      search.byz.fill_(-1.)
      replay()
      torch.cuda.synchronize()
      assert torch.equal(search.record[:-1], eager_record[:-1]), gar
      assert torch.equal(search.record[-1:].view(torch.int32)[:1], eager_record[-1:].view(torch.int32)[:1])
      assert torch.equal(search.byz, eager_byz), gar

def _emulate(gar, honest, f, avg, att, R, evals=16):
  """ R ShardedLineSearch(..., many=True) instances on one GPU driven through the stages; returns (instances, the
  concatenated rule output of every evaluation). """
  from byzantinemomentum_b200 import sharded
  per_rank = _shards(honest + [avg, att], R, False)
  nh = len(honest)
  inst = [sharded.ShardedLineSearch(gar, rows[:nh], f, f, rows[nh], rows[nh + 1], evals, many=True) for rows in per_rank]
  outs = []
  for k in range(evals):
    parts = [s.evaluate(k) for s in inst]
    outs.append(torch.cat([s._shard.out for s in inst]).clone())
    scores = torch.stack(parts).reshape(R)
    for s in inst:
      s.step(k, scores)
  for s in inst:
    s.finish()
  torch.cuda.synchronize()
  return inst, outs

@pytest.mark.parametrize("gar", COORDINATE)
def test_sharded_line_search_at_300_rows(gar):
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine, sharded
  nh, f = 260, 40
  honest = _honest(nh, 4099, 27)
  avg, att = _direction(honest, "identical")
  ref = engine.LineSearch(gar, honest, f, f, avg, att, 16, many=True)
  ref()
  got = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, 16, many=True)
  byz = got()
  torch.cuda.synchronize()
  assert torch.equal(_bits(got.record[:-1]), _bits(ref.record[:-1])) and _status(got.record) == _status(ref.record), gar
  assert torch.equal(_bits(byz), _bits(ref.byz)) and torch.equal(_bits(got._shard.out), _bits(ref._out)), gar
  inst, outs = _emulate(gar, honest, f, avg, att, 3)
  for s in inst[1:]:
    assert torch.equal(_bits(s.record[:-1]), _bits(inst[0].record[:-1])), gar
  factor, trace = inst[0].result()
  xs, ys = [x for x, _ in trace], [y for _, y in trace]
  assert [x.hex() for x in _xs_of(ys)] == [x.hex() for x in xs], gar
  assert torch.equal(_bits(torch.cat([s.byz for s in inst])), _bits(avg + factor * att)), gar
  for (x, y), out in zip(trace, outs):
    want = float(((out - avg).double() ** 2).sum())
    assert abs(y - want) <= 1e-6 * abs(want) + 1e-30, (gar, x, y, want)
  plain = bz.many_gars[gar](gradients=honest + [_candidate(avg, att, xs[-1], False, "identical")] * f, f=f)
  assert torch.equal(_bits(outs[-1]), _bits(plain)), gar
  with pytest.raises(ValueError, match="at most 128 rows"):
    sharded.ShardedLineSearch(gar, honest, f, f, avg, att, 4)

def test_install_attacks_runs_the_device_search_against_median_with_300_rows():
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine
  aggregators, attacks = _aggregators(), _attacks()
  bz.plugin.install(aggregators, many=True)
  bz.plugin.install_attacks(attacks, many=True)
  honest = _honest(280, 4099, 37)
  defense = aggregators.gars["b200-median"]
  out = attacks.attacks["empire"].checked(grad_honests=honest, f_real=20, f_decl=20, defense=defense, model=None, factor=-16)
  assert isinstance(out, list) and len(out) == 20 and all(o is out[0] for o in out)
  avg = torch.stack(honest).mean(dim=0)
  _, want = engine.line_search("median", honest, 20, 20, avg, avg.neg(), 16, many=True)
  assert torch.equal(_bits(out[0]), _bits(want))

def test_install_tools_handles_300_samples_on_the_device():
  import types
  import byzantinemomentum_b200 as bz
  tools = types.SimpleNamespace(compute_avg_dev_max=lambda samples: pytest.fail("the stock function ran"))
  bz.plugin.install_tools(tools, many=True)
  x = np.random.default_rng(3).standard_normal((300, 5003)).astype(np.float32)
  got = tools.compute_avg_dev_max([torch.from_numpy(r).to(DEV) for r in x])
  check((got[0].cpu().numpy(),) + tuple(got[1:]), *orc.compute_avg_dev_max(list(x)))
