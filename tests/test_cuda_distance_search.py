# coding: utf-8
"""GPU tests of the attacks' line search against Multi-Krum, Bulyan, Aksel and CGE up to 128 rows
(`bz_distance_line_search` through `engine.LineSearch`), of `gars.wide_gars` and of `plugin.install(..., wide=True)`.

The checks of tests/test_cuda_linesearch.py::_check_search, with `engine.Plan(gar, honest + [cand] * f_real, f=f_decl)`
(`bz_distance` above 64 rows) in place of `bz.gars`:
  * the x sequence is `line_maximize` (tests/line_oracle.py) fed with the device's own y values, bit for bit;
  * every y_k is fp64 sum((out - avg)^2) of `Plan` on the torch candidate of x_k, within 1e-6;
  * the rule's output of the last evaluation and the returned Byzantine gradient are bit-identical to `Plan` and to
    the torch statements.
The unique-row counts reach one pass with more than 64 rows (K = 1), K = 3 and K = 4 blocks, and 128 unique rows (the
candidate not aliased).  Runs of 1 to 6 evaluations check the star pass of every evaluation through the last output."""

import math

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"

import line_oracle

GARS = ["krum", "bulyan", "aksel", "cge"]
# (nh, f_real) -> unique rows u = nh + 1: K = 1 at n = 70, K = 3 at u = 81, K = 4 at u = 101, u = 128
SIZES = [(40, 30), (80, 10), (100, 20), (127, 1)]

def _f_decl(gar, n, f_real):
  """ f_real where the rule takes it, else the largest f Bulyan takes (n >= 4f + 3). """
  return min(f_real, (n - 3) // 4) if gar == "bulyan" else f_real

def _honest(nh, d, seed, offset=0):
  gen = torch.Generator(device=DEV).manual_seed(seed)
  mu = torch.randn(d, device=DEV, generator=gen)
  rows = []
  for i in range(nh):
    base = torch.empty(d + offset, device=DEV)
    base[offset:] = mu + (0.5 + i / max(nh - 1, 1)) * torch.randn(d, device=DEV, generator=gen)
    rows.append(base[offset:])
  return rows

def _direction(honest, kind):
  stck = torch.stack(honest)
  if kind == "identical":
    return stck.mean(dim=0), stck.var(dim=0).sqrt_()
  avg = honest[0].clone()
  for g in honest[1:]:
    avg.add_(g)
  return avg.div_(len(honest)), None

def _candidate(avg, att, x, negative, kind):
  """ The reference's statements (identical.py:70-72, empire.py:54). """
  if kind == "identical":
    return avg + (-x if negative else x) * att
  return avg.mul(-x)

def _plan(gar, honest, byz, f_real, f):
  from byzantinemomentum_b200 import engine
  plan = engine.Plan(gar, honest + [byz] * f_real, f=f)
  out = plan().clone()
  return out, (None if plan.status is None else int(plan.status.item()))

def _xs_of(ys):
  xs = []
  line_oracle.line_maximize(lambda x: (xs.append(x), ys[len(xs) - 1])[1], len(ys))
  return xs

def _check_search(gar, honest, f_real, f, avg, att, evals, negative, kind):
  from byzantinemomentum_b200 import engine
  search = engine.LineSearch(gar, honest, f_real, f, avg, att, evals, negative=negative, kind=kind)
  byz = search()
  factor, trace = search.result()
  xs, ys = [x for x, _ in trace], [y for _, y in trace]
  assert [x.hex() for x in _xs_of(ys)] == [x.hex() for x in xs], (gar, xs, ys)
  assert factor.hex() == float(line_oracle.line_maximize(lambda x, it=iter(ys): next(it), evals)).hex()
  outs = []
  for x, y in trace:
    out, _ = _plan(gar, honest, _candidate(avg, att, x, negative, kind), f_real, f)
    outs.append(out)
    ref = float(((out - avg).double() ** 2).sum())
    if math.isnan(ref):
      assert math.isnan(y), (gar, x, y)
    else:
      assert abs(y - ref) <= 1e-6 * abs(ref) + 1e-30, (gar, x, y, ref)
  assert torch.equal(search._out, outs[-1]), (gar, xs[-1])
  final = avg + factor * att if kind == "identical" else avg.mul(-factor)
  assert torch.equal(byz, final), (gar, factor)
  return search

@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"nh{s[0]}_freal{s[1]}")
@pytest.mark.parametrize("gar", GARS)
def test_search_matches_plan_above_64_rows(gar, size):
  from byzantinemomentum_b200 import engine
  nh, f_real = size
  n = nh + f_real
  for d, offset in ((1, 0), (1031, 0), (1031, 1)):
    honest = _honest(nh, d, 5 + d + n + offset, offset)
    for kind, negative in (("identical", False), ("identical", True), ("empire-strict", False)):
      if d == 1 and kind != "identical":
        continue
      avg, att = _direction(honest, kind)
      for f in sorted({_f_decl(gar, n, f_real), _f_decl(gar, n, max(1, f_real // 3))}):
        search = _check_search(gar, honest, f_real, f, avg, att, 16, negative, kind)
        assert search._fn is engine._lib.lib().bz_distance_line_search

@pytest.mark.parametrize("gar", ["krum", "bulyan"])
@pytest.mark.parametrize("size", [(40, 30), (100, 20), (127, 1)], ids=lambda s: f"nh{s[0]}_freal{s[1]}")
def test_every_evaluation_s_star_pass(gar, size):
  """ The output of the last evaluation of a run of `evals` evaluations is `Plan`'s at its x: the star pass of each
  evaluation 1 .. 5 leaves the pass tables of the plain call. """
  nh, f_real = size
  n = nh + f_real
  honest = _honest(nh, 40_000, 71 + n)
  avg, att = _direction(honest, "identical")
  for evals in range(1, 7):
    _check_search(gar, honest, f_real, _f_decl(gar, n, f_real), avg, att, evals, True, "identical")

def test_bulyan_on_non_finite_rows():
  """ Non-finite honest rows: every Multi-Krum score is NaN, Bulyan's status word says so, its output is NaN, the NaN
  score never wins, and the strict search raises what the plain call raises. """
  from byzantinemomentum_b200 import engine, _lib
  nh, f_real, f = 90, 10, 10
  honest = _honest(nh, 515, 21)
  for k in range(80):
    honest[k] = honest[k].clone()
    honest[k][k] = math.nan
  avg, att = _direction(honest[80:], "identical")
  out, status = _plan("bulyan", honest, avg + att, f_real, f)
  assert status == _lib.STATUS_DEGENERATE and torch.isnan(out).all()
  with pytest.raises(TypeError):
    engine.line_search("bulyan", honest, f_real, f, avg, att, 16)
  engine.config.strict_status = False
  try:
    search = engine.LineSearch("bulyan", honest, f_real, f, avg, att, 16)
    byz = search()
    factor, trace = search.result()
    status = int(search.record.cpu()[-1:].view(torch.int32)[0])
  finally:
    engine.config.strict_status = True
  assert status == _lib.STATUS_DEGENERATE
  assert all(math.isnan(y) for _, y in trace) and factor == 0. and torch.equal(byz, avg + 0. * att)
  assert [x for x, _ in trace] == _xs_of([y for _, y in trace])
  assert torch.isnan(search._out).all()

def test_a_graph_replays_the_eager_search():
  from byzantinemomentum_b200 import engine
  for gar, kind in (("krum", "identical"), ("bulyan", "identical"), ("aksel", "empire-strict"), ("cge", "identical")):
    honest = _honest(90, 30_011, 31)
    avg, att = _direction(honest, kind)
    f = _f_decl(gar, 110, 20)
    search = engine.LineSearch(gar, honest, 20, f, avg, att, 16, negative=True, kind=kind)
    search()
    torch.cuda.synchronize()
    eager_record, eager_byz, eager_out = search.record.clone(), search.byz.clone(), search._out.clone()
    replay = search.graph()
    for _ in range(2):
      search.record.fill_(-1.)
      search.byz.fill_(-1.)
      search._out.fill_(-1.)
      replay()
      torch.cuda.synchronize()
      assert torch.equal(search.record[:-1], eager_record[:-1]), gar
      assert torch.equal(search.record[-1:].view(torch.int32)[:1], eager_record[-1:].view(torch.int32)[:1]), gar
      assert torch.equal(search.byz, eager_byz) and torch.equal(search._out, eager_out), gar

@pytest.mark.parametrize("gar", GARS + ["brute"])
def test_up_to_64_rows_it_is_bz_line_search(gar):
  """ The same record, byz and out as bz_line_search, with the same arguments and a workspace of the same size. """
  from byzantinemomentum_b200 import engine, _lib
  lib = _lib.lib()
  for nh, f_real, d, offset in ((20, 5, 4099, 0), (50, 14, 1031, 1), (60, 4, 40_000, 0)):
    n = nh + f_real
    f = {"bulyan": (n - 3) // 4, "brute": 2 if n <= 25 else 1}.get(gar, f_real)
    honest = _honest(nh, d, 3 + nh + d, offset)
    avg, att = _direction(honest, "identical")
    search = engine.LineSearch(gar, honest, f_real, f, avg, att, 16, negative=True)
    assert search._fn is lib.bz_line_search
    search()
    torch.cuda.synchronize()
    want = (search.record.clone(), search.byz.clone(), search._out.clone())
    for t in (search.record, search.byz, search._out):
      t.fill_(-1)
    code = lib.bz_distance_line_search(*search._args)
    assert code == 0, lib.bz_last_error()
    torch.cuda.synchronize()
    assert torch.equal(search.record[:-1], want[0][:-1]), (gar, nh, f_real)
    assert torch.equal(search.record[-1:].view(torch.int32)[:1], want[0][-1:].view(torch.int32)[:1]), (gar, nh, f_real)
    assert torch.equal(search.byz, want[1]) and torch.equal(search._out, want[2]), (gar, nh, f_real)

def test_headline_size():
  """ Multi-Krum at n = 100 over d = 1,310,922. """
  honest = _honest(80, 1_310_922, 97)
  avg, att = _direction(honest, "identical")
  _check_search("krum", honest, 20, 20, avg, att, 16, False, "identical")

# ---- gars.wide_gars and the plugin ---------------------------------------------------------------------------------

@pytest.mark.parametrize("gar", GARS)
def test_wide_gars(gar):
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine
  selections = bz._gars._last
  for n in (25, 64, 65, 100, 128):
    f = max(1, (n - 3) // 4) if gar == "bulyan" else n // 5
    rows = _honest(n - 10, 2_003, n) + [torch.randn(2_003, device=DEV)] * 10
    plan = engine.Plan(gar, rows, f=f)
    want = plan().clone()
    got = bz.wide_gars[gar](gradients=rows, f=f)
    assert torch.equal(got, want), (gar, n)
    if n <= 64:
      assert torch.equal(got, bz.gars[gar](gradients=rows, f=f)), (gar, n)
    if bz.wide_gars[gar].influence is None:
      continue
    honests, attacks = rows[:n - 10], rows[n - 10:]
    stored = selections.lookup(gar, (f,) if gar == "krum" else (), rows)
    assert stored is not None and torch.equal(stored[:plan.selection.numel()], plan.selection), (gar, n)
    calls = []
    original = engine.wide_distance
    engine.wide_distance = lambda *args, **kwargs: calls.append(args) or original(*args, **kwargs)
    try:
      ratio = bz.wide_gars[gar].influence(honests, attacks, f=f)
    finally:
      engine.wide_distance = original
    assert calls == []                                   # the stored selection
    count = {"krum": n - f - 2, "aksel": (n + 1) // 2, "cge": n - f}[gar]
    assert ratio == sum(1 for i in plan.selection.tolist()[:count] if i >= n - 10) / count, (gar, n)

@pytest.mark.parametrize("gar", ["krum", "cge"])
def test_install_wide_and_install_attacks_run_the_device_search_on_100_rows(gar, monkeypatch):
  from byzantinemomentum_b200 import engine, plugin
  from test_distance_search_abi import _aggregators, _attacks
  monkeypatch.setattr(plugin, "_installed", {})
  aggregators, attacks = _aggregators(), _attacks()
  plugin.install(aggregators, wide=True, names=[gar])
  plugin.install_attacks(attacks)
  honest = _honest(90, 4_099, 13)
  got = attacks.attacks["little"].checked(grad_honests=honest, f_real=10, f_decl=10, defense=aggregators.gars["b200-" + gar],
                                          model=None, factor=-16)
  assert len(got) == 10 and all(g is got[0] for g in got)
  stck = torch.stack(honest)
  _, byz = engine.line_search(gar, honest, 10, 10, stck.mean(dim=0), stck.var(dim=0).sqrt_(), 16)
  assert torch.equal(got[0], byz), gar
  aggregated = aggregators.gars["b200-" + gar](gradients=honest + got, f=10)
  assert torch.equal(aggregated, _plan(gar, honest, byz, 10, 10)[0]), gar
