# coding: utf-8
"""GPU tests of the attacks' line search against Multi-Krum, Bulyan, Aksel and CGE for 129 to 1024 rows
(`bz_distance_line_search_many` through `engine.LineSearch(..., many_distance=True)`), and of
`plugin.install_attacks(..., many_distance=True)`.

The checks of tests/test_cuda_distance_search.py::_check_search, with `engine.Plan(gar, honest + [cand] * f_real,
f=f_decl, many=True)` (`bz_distance_many`) as the reference:
  * the x sequence is `line_maximize` (tests/line_oracle.py) fed with the device's own y values, bit for bit;
  * every y_k is fp64 sum((out - avg)^2) of `Plan` on the torch candidate of x_k, within 1e-6;
  * the rule's output of the last evaluation and the returned Byzantine gradient are bit-identical to `Plan` and to
    the torch statements.
From the second evaluation on, Multi-Krum and Bulyan compute only the candidate's column of the distance table
(K2-star-many): the table itself is compared with the plain call's, entry by entry, which a selection cannot mask."""

import math
import types

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"

import line_oracle

GARS = ["krum", "bulyan", "aksel", "cge"]
TABLE_OFFSET = 12544                                    # BZ_DISTANCE_MANY_TABLE_OFFSET
# (nh, f_real), u = nh + 1 unique rows: u = 128 with the candidate last in a full tile; u - 1 = 64k (the candidate alone
# in its tile) at u = 129 (the slice count drops from 132 to 66), 193, 257 and 769; few unique rows with n > 128;
# u = 1024 with the candidate not aliased; n = 1024 with f_real = 255
SIZES = [(127, 2), (128, 1), (192, 8), (256, 4), (768, 2), (40, 100), (1023, 1), (769, 255)]

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
  plan = engine.Plan(gar, honest + [byz] * f_real, f=f, many=True)
  out = plan().clone()
  return plan, out

def _xs_of(ys):
  xs = []
  line_oracle.line_maximize(lambda x: (xs.append(x), ys[len(xs) - 1])[1], len(ys))
  return xs

def _upper(ws, u):
  """ The upper triangle (diagonal included) of the u x u table in a bz_distance_many workspace, as int64 bits. """
  table = ws[TABLE_OFFSET:TABLE_OFFSET + 8 * u * u].view(torch.float64).view(u, u)
  rows, cols = torch.triu_indices(u, u, device=ws.device)
  return table[rows, cols].view(torch.int64)

def _check_search(gar, honest, f_real, f, avg, att, evals, negative, kind, table=False):
  from byzantinemomentum_b200 import engine
  search = engine.LineSearch(gar, honest, f_real, f, avg, att, evals, negative=negative, kind=kind, many_distance=True)
  assert search._fn is engine._lib.many_search_lib().bz_distance_line_search_many
  byz = search()
  factor, trace = search.result()
  xs, ys = [x for x, _ in trace], [y for _, y in trace]
  assert [x.hex() for x in _xs_of(ys)] == [x.hex() for x in xs], (gar, xs, ys)
  assert factor.hex() == float(line_oracle.line_maximize(lambda x, it=iter(ys): next(it), evals)).hex()
  for k, (x, y) in enumerate(trace):
    plan, out = _plan(gar, honest, _candidate(avg, att, x, negative, kind), f_real, f)
    ref = float(((out - avg).double() ** 2).sum())
    if math.isnan(ref):
      assert math.isnan(y), (gar, x, y)
    else:
      assert abs(y - ref) <= 1e-6 * abs(ref) + 1e-30, (gar, x, y, ref)
  assert torch.equal(search._out, out), (gar, xs[-1])
  if table:                                     # the last evaluation's table: the plain call's, bit for bit
    u = len(set(t.data_ptr() for t in honest)) + 1
    assert torch.equal(_upper(search._ws, u), _upper(plan._ws, u)), (gar, evals)
  final = avg + factor * att if kind == "identical" else avg.mul(-factor)
  assert torch.equal(byz, final), (gar, factor)
  return search

@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"nh{s[0]}_freal{s[1]}")
@pytest.mark.parametrize("gar", GARS)
def test_search_matches_plan_above_128_rows(gar, size):
  nh, f_real = size
  n = nh + f_real
  for d, offset in ((1, 0), (1031, 0), (1031, 1)):
    honest = _honest(nh, d, 5 + d + n + offset, offset)
    for kind, negative in (("identical", False), ("identical", True), ("empire-strict", False)):
      if d == 1 and kind != "identical":
        continue
      avg, att = _direction(honest, kind)
      _check_search(gar, honest, f_real, _f_decl(gar, n, f_real), avg, att, 16, negative, kind, table=gar in ("krum", "bulyan"))

@pytest.mark.parametrize("gar", ["krum", "bulyan"])
@pytest.mark.parametrize("size", [(128, 1), (192, 8), (40, 100), (768, 2)], ids=lambda s: f"nh{s[0]}_freal{s[1]}")
def test_the_star_column_at_the_edges_of_d(gar, size):
  """ d = 1, 31, 33 (a partial chunk), 256 / 257 (u = 129: one slice, then two), 40,000 (several 1024-column stages
  per slice at u = 769), rows at a 1-float offset. """
  nh, f_real = size
  n = nh + f_real
  for d, offset in ((1, 0), (31, 0), (33, 1), (256, 0), (257, 0), (40_000, 1)):
    honest = _honest(nh, d, 7 + d + n, offset)
    avg, att = _direction(honest, "identical")
    _check_search(gar, honest, f_real, _f_decl(gar, n, f_real), avg, att, 6, True, "identical", table=True)

@pytest.mark.parametrize("gar", ["krum", "bulyan"])
def test_every_evaluation_s_star_column(gar):
  """ After a search of k = 1 .. 6 evaluations, the table is the plain call's on the last candidate. """
  nh, f_real = 300, 40
  honest = _honest(nh, 20_011, 71)
  avg, att = _direction(honest, "identical")
  for evals in range(1, 7):
    _check_search(gar, honest, f_real, _f_decl(gar, nh + f_real, f_real), avg, att, evals, True, "identical", table=True)

def test_bulyan_on_non_finite_rows():
  """ Non-finite honest rows: Bulyan's status word is set, its output is NaN, the NaN score never wins, and the
  strict search raises what the plain call raises. """
  from byzantinemomentum_b200 import engine, _lib
  nh, f_real, f = 290, 10, 10
  honest = _honest(nh, 515, 21)
  for k in range(280):
    honest[k] = honest[k].clone()
    honest[k][k % 515] = math.nan
  avg, att = _direction(honest[280:], "identical")
  plan, out = _plan("bulyan", honest, avg + att, f_real, f)
  assert int(plan.status.item()) == _lib.STATUS_DEGENERATE and torch.isnan(out).all()
  with pytest.raises(TypeError):
    engine.line_search("bulyan", honest, f_real, f, avg, att, 16, many_distance=True)
  engine.config.strict_status = False
  try:
    search = engine.LineSearch("bulyan", honest, f_real, f, avg, att, 16, many_distance=True)
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
    honest = _honest(250, 30_011, 31)
    avg, att = _direction(honest, kind)
    f = _f_decl(gar, 270, 20)
    search = engine.LineSearch(gar, honest, 20, f, avg, att, 16, negative=True, kind=kind, many_distance=True)
    search()
    torch.cuda.synchronize()
    eager_record, eager_byz, eager_out = search.record.clone(), search.byz.clone(), search._out.clone()
    search()
    torch.cuda.synchronize()
    assert torch.equal(search.record[:-1], eager_record[:-1]) and torch.equal(search._out, eager_out), gar
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

@pytest.mark.parametrize("gar", GARS)
def test_up_to_128_rows_it_is_bz_distance_line_search(gar):
  """ The same record, byz and out as bz_distance_line_search, with the same arguments. """
  from byzantinemomentum_b200 import engine, _lib
  lib = _lib.lib()
  for nh, f_real, d, offset in ((20, 5, 4099, 0), (100, 20, 1031, 1), (127, 1, 40_000, 0)):
    n = nh + f_real
    honest = _honest(nh, d, 3 + nh + d, offset)
    avg, att = _direction(honest, "identical")
    search = engine.LineSearch(gar, honest, f_real, _f_decl(gar, n, f_real), avg, att, 16, negative=True, many_distance=True)
    assert search._ws.numel() == lib.bz_distance_line_search_workspace_bytes(n)
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
  """ Multi-Krum at n = 300 over d = 1,310,922. """
  honest = _honest(280, 1_310_922, 97)
  avg, att = _direction(honest, "identical")
  _check_search("krum", honest, 20, 20, avg, att, 6, False, "identical", table=True)

def _registry():
  class Entry:                                    # hashable, like the reference's checked functions
    def __init__(self, unchecked, check):
      self.unchecked, self.check = unchecked, check
  aggregators = types.SimpleNamespace(gars={})
  def register(name, unchecked, check, upper_bound=None, influence=None):
    aggregators.gars[name] = Entry(unchecked, check)
  aggregators.register = register
  return aggregators

def _attacks():
  attacks = types.SimpleNamespace(attacks={})
  stock = types.SimpleNamespace(unchecked=lambda **kwargs: "stock", check=None)
  for name in ("little", "empire", "bulyan", "empire-strict"):
    attacks.attacks[name] = stock
  def register(name, unchecked, check):
    attacks.attacks[name] = types.SimpleNamespace(unchecked=unchecked, check=check)
  attacks.register = register
  return attacks

@pytest.mark.parametrize("gar", ["krum", "cge"])
def test_install_many_distance_and_install_attacks_run_the_device_search_on_300_rows(gar):
  from byzantinemomentum_b200 import engine, plugin
  aggregators, attacks = _registry(), _attacks()
  plugin.install(aggregators, prefix="md-", many_distance=True)
  plugin.install_attacks(attacks, many_distance=True)
  honest = _honest(280, 10_007, 13)
  avg, att = _direction(honest, "identical")
  got = attacks.attacks["little"].unchecked(grad_honests=honest, f_real=20, f_decl=20, defense=aggregators.gars["md-" + gar],
                                            model=None, factor=-16)
  assert got != "stock" and len(got) == 20 and all(g is got[0] for g in got)
  _, want = engine.line_search(gar, honest, 20, 20, avg, att, 16, many_distance=True)
  assert torch.equal(got[0], want)
