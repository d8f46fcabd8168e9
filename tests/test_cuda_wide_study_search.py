# coding: utf-8
"""GPU tests of the study metrics and of the attacks' line search above 64 rows (up to 128, with the
coordinate-wise rules).

  * K6 over the 128-pointer table (`bz_avg_dev_max`) at every n in 65..128 on the special values of
    tests/test_cuda_k1_edges.py (NaN, +-inf, -0, subnormals, ties), with 16-byte aligned rows and mixed
    4-byte offsets: the average bit-exact against the oracle, the scalars at the bar of
    tests/test_study_metrics.py; also d = 1, 31 and 1,310,922, and the reference's recorded outputs.
  * The whole study block (`engine.study_step`) at 100 rows against attack.py's statements, and
    `sharded.study_step`'s halves over R = 1, 3 and 8 shards emulated on one GPU.
  * `engine.LineSearch` for every coordinate-wise rule at n = 65, 100 and 128 (the checks of
    tests/test_cuda_linesearch.py), a CUDA graph of it, `ShardedLineSearch` on one rank and on 3 emulated
    ranks, and `plugin.install_attacks` running the device search against b200-median with 100 rows."""

import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"

from oracle import byzoracle as orc
from test_cuda_k1_edges import _device_rows, _stack
from test_cuda_linesearch import _candidate, _check_search, _direction, _honest
from test_cuda_sharded_search import _bits, _emulate, _status, _xs_of
from test_cuda_sharded_study import MOMENTUM, _check as _check_shards, _inputs
from test_cuda_study_step import _study_reference
from test_plugin_attacks import _aggregators, _attacks
from test_wide_study_abi import cases, check, load

COORDINATE = ["average", "median", "trmean", "phocas", "meamed"]

def _study(rows):
  import byzantinemomentum_b200 as bz
  avg, norm_avg, norm_dev, norm_max = bz.compute_avg_dev_max(rows)
  return avg.cpu().numpy(), norm_avg, norm_dev, norm_max

@pytest.mark.parametrize("n", range(65, 129))
def test_study_metrics_every_n_above_64(n):
  d = 1031
  for nonfinite in (True, False):
    x = _stack(n, d, 500 + n, nonfinite=nonfinite)
    want = orc.compute_avg_dev_max(list(x))
    for offsets in ((0,), (0, 1, 2, 3)):
      check(_study(_device_rows(x, offsets)), *want)

@pytest.mark.parametrize("n", [65, 100, 128])
@pytest.mark.parametrize("d", [1, 31, 1_310_922])
def test_study_metrics_sizes(n, d):
  rng = np.random.default_rng(7 * n + d % 991)
  x = (rng.standard_normal((n, d)) * rng.uniform(0.1, 10., (n, 1))).astype(np.float32)
  want = orc.compute_avg_dev_max(list(x))
  base = torch.from_numpy(x).to(DEV)
  check(_study(list(base)), *want)
  if d > 1:
    check(_study(_device_rows(x, (1, 3))), *want)

@pytest.mark.parametrize("case", [c for c in cases() if c.values[0]["hi"] > c.values[0]["lo"]])
def test_study_metrics_match_the_reference_above_64_rows(case):
  rows, avg, norm_avg, norm_dev, norm_max = load(case)
  check(_study([torch.from_numpy(np.ascontiguousarray(r)).to(DEV) for r in rows]), avg, norm_avg, norm_dev, norm_max)

def test_study_metrics_are_deterministic_and_avg_dev_max_async_takes_128_rows():
  from byzantinemomentum_b200 import engine
  rows = [torch.randn(300_007, device=DEV) for _ in range(128)]
  a_avg, a = engine.avg_dev_max_async(rows)
  b_avg, b = engine.avg_dev_max_async(rows)
  assert a.shape == (130,) and torch.equal(a, b) and torch.equal(a_avg, b_avg)
  with pytest.raises(ValueError, match="maximum of 128"):
    engine.avg_dev_max_async(rows + rows[:1])

@pytest.mark.parametrize("shared", [True, False])
def test_study_step_at_100_rows_matches_the_statements_of_attack_py(shared):
  from byzantinemomentum_b200 import engine
  d = 79_510
  sampleds, honests, attacks, defense, pasts = _inputs(100, 100 if shared else 90, 30, 3, d, shared)
  want, want_avg = _study_reference(sampleds, honests, attacks, defense, pasts, MOMENTUM)
  got = engine.study_step(sampleds, honests, attacks, defense, pasts, MOMENTUM)
  assert torch.allclose(got["sampled_grad_avg"], want_avg, rtol=1e-6, atol=1e-7)
  for key, ref in want.items():
    val = got[key]
    if math.isnan(ref):
      assert math.isnan(val), key
    else:
      assert abs(val - ref) <= 2e-5 * abs(ref) + 3e-6, (key, val, ref)

@pytest.mark.parametrize("R", [1, 3, 8])
def test_sharded_study_step_at_100_rows(R):
  from byzantinemomentum_b200 import sharded
  _check_shards(_inputs(100, 100, 28, 2, 10_007, True), R)
  got = sharded.compute_avg_dev_max(_inputs(100, 100, 0, 0, 4099, True)[0])
  assert got[0].shape == (4099,)

F_WIDE = {65: (1, 32), 100: (1, 45), 128: (1, 60)}       # n -> (small f_real, large f_real)

@pytest.mark.parametrize("n", [65, 100, 128])
@pytest.mark.parametrize("gar", COORDINATE)
def test_line_search_above_64_rows(gar, n):
  import byzantinemomentum_b200 as bz
  for f_real in F_WIDE[n]:
    f = f_real
    nh = n - f_real
    for d, offset in ((1031, 0), (1031, 1)):
      honest = _honest(nh, d, 17 + d + n + f_real, offset)
      for kind, negative in (("identical", True), ("empire-strict", False)):
        avg, att = _direction(honest, kind)
        _check_search(bz, gar, honest, f_real, f, avg, att, 16, negative, kind)

def test_line_search_graph_above_64_rows():
  from byzantinemomentum_b200 import engine
  for gar, kind in (("median", "identical"), ("trmean", "empire-strict")):
    honest = _honest(90, 30_011, 41)
    avg, att = _direction(honest, kind)
    search = engine.LineSearch(gar, honest, 30, 30, avg, att, 16, negative=True, kind=kind)
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

@pytest.mark.parametrize("gar", COORDINATE)
def test_sharded_line_search_at_100_rows(gar):
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine, sharded
  nh, f = 80, 20
  honest = _honest(nh, 4099, 23)
  avg, att = _direction(honest, "identical")
  ref = engine.LineSearch(gar, honest, f, f, avg, att, 16)
  ref()
  got = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, 16)
  byz = got()
  torch.cuda.synchronize()
  assert torch.equal(_bits(got.record[:-1]), _bits(ref.record[:-1])) and _status(got.record) == _status(ref.record), gar
  assert torch.equal(_bits(byz), _bits(ref.byz)) and torch.equal(_bits(got._shard.out), _bits(ref._out)), gar
  # three ranks emulated on one GPU
  inst, outs = _emulate(gar, honest, f, avg, att, 3, False)
  for s in inst[1:]:
    assert torch.equal(_bits(s.record[:-1]), _bits(inst[0].record[:-1])), gar
  factor, trace = inst[0].result()
  xs, ys = [x for x, _ in trace], [y for _, y in trace]
  assert [x.hex() for x in _xs_of(ys)] == [x.hex() for x in xs], gar
  assert torch.equal(_bits(torch.cat([s.byz for s in inst])), _bits(avg + factor * att)), gar
  for (x, y), out in zip(trace, outs):
    want = float(((out - avg).double() ** 2).sum())
    assert abs(y - want) <= 1e-6 * abs(want) + 1e-30, (gar, x, y, want)
  plain = bz.gars[gar](gradients=honest + [_candidate(avg, att, xs[-1], False, "identical")] * f, f=f)
  assert torch.equal(_bits(outs[-1]), _bits(plain)), gar

def test_sharded_line_search_keeps_the_distance_limit():
  from byzantinemomentum_b200 import sharded
  honest = _honest(60, 257, 5)
  avg, att = _direction(honest, "identical")
  with pytest.raises(ValueError, match="at most 64 rows"):
    sharded.ShardedLineSearch("krum", honest, 5, 5, avg, att, 4)
  with pytest.raises(ValueError, match="at most 128 rows"):
    sharded.ShardedLineSearch("median", _honest(120, 257, 6), 9, 9, avg, att, 4)

def test_install_attacks_runs_the_device_search_against_median_with_100_rows():
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine
  aggregators, attacks = _aggregators(), _attacks()
  bz.plugin.install(aggregators)
  bz.plugin.install_attacks(attacks)
  honest = _honest(80, 4099, 29)
  defense = aggregators.gars["b200-median"]
  out = attacks.attacks["empire"].checked(grad_honests=honest, f_real=20, f_decl=20, defense=defense, model=None, factor=-16)
  assert isinstance(out, list) and len(out) == 20 and all(o is out[0] for o in out)
  avg = torch.stack(honest).mean(dim=0)
  _, want = engine.line_search("median", honest, 20, 20, avg, avg.neg(), 16)
  assert torch.equal(_bits(out[0]), _bits(want))
