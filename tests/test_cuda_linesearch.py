# coding: utf-8
"""GPU parity of the attacks' line search on the device (`engine.LineSearch`, `bz_line_search`).

For every rule at n in {11, 25, 51}, several d (1, odd, rows off the 16-byte grid), both candidate
kinds, `negative` on and off and 1, 2 or 16 evaluations:
  * the x sequence of the trace is `line_maximize` (restated in tests/line_oracle.py) fed with the
    device's own y values, bit for bit, and the trace ends with its result;
  * every y_k is fp64 sum((out - avg)^2) within 1e-6, `out` being the plain `bz.gars[gar]` call on the
    honest rows and the torch candidate row of x_k;
  * the rule's output of the last evaluation and the returned Byzantine gradient are bit-identical to
    the torch statements and the plain call;
  * the factor is the one a host loop of the reference's `eval_factor` statements over this library's
    rules picks, unless the two scores (`dot` order vs K2' order) tie within rounding where they part.
Plus the status words of Bulyan and brute, and a CUDA graph of the whole search."""

import math

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"

import line_oracle

F_OF = {   # (rule, n) -> f: valid for the rule (bulyan n >= 4f + 3, brute C(n, n - f) <= 2^31)
  **{(g, n): f for g in ("average", "median", "trmean", "phocas", "meamed", "krum", "aksel", "cge") for n, f in ((11, 3), (25, 5), (51, 12))},
  ("bulyan", 11): 2, ("bulyan", 25): 5, ("bulyan", 51): 12,
  ("brute", 11): 3, ("brute", 25): 2, ("brute", 51): 1,
}

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

def _plain(bz, gar, honest, byz, f_real, f):
  return bz.gars[gar](gradients=honest + [byz] * f_real, f=f)

def _check_search(bz, gar, honest, f_real, f, avg, att, evals, negative, kind):
  from byzantinemomentum_b200 import engine
  search = engine.LineSearch(gar, honest, f_real, f, avg, att, evals, negative=negative, kind=kind)
  byz = search()
  factor, trace = search.result()
  xs = [x for x, _ in trace]
  ys = [y for _, y in trace]
  # 1. the x sequence: line_maximize fed with the device's y values
  fed = []
  def scape(x):
    fed.append(x)
    return ys[len(fed) - 1]
  want_factor = line_oracle.line_maximize(scape, evals)
  assert [x.hex() for x in fed] == [x.hex() for x in xs], (gar, fed, xs)
  assert factor.hex() == float(want_factor).hex()
  # 2. every score against the plain call on the torch candidate
  plain_outs = []
  for x, y in trace:
    out = _plain(bz, gar, honest, _candidate(avg, att, x, negative, kind), f_real, f)
    plain_outs.append(out)
    ref = float(((out - avg).double() ** 2).sum())
    if math.isnan(ref):
      assert math.isnan(y), (gar, x, y)
    else:
      assert abs(y - ref) <= 1e-6 * abs(ref) + 1e-30, (gar, x, y, ref)
  # 3. the rule's output of the last evaluation and the Byzantine gradient, bit for bit
  assert torch.equal(search._out, plain_outs[-1]), (gar, xs[-1])
  final = avg + factor * att if kind == "identical" else avg.mul(-factor)     # identical.py:83-85: no sign on a searched factor
  assert torch.equal(byz, final), (gar, factor)
  # 4. the host loop of the reference's statements (attacks/identical.py:67-77, empire.py:51-59)
  host_xs, host_ys = [], []
  def eval_factor(x):
    grad_attack = _candidate(avg, att, x, negative, kind)
    aggregated = _plain(bz, gar, honest, grad_attack, f_real, f)
    aggregated.sub_(avg)
    y = aggregated.dot(aggregated).item()
    host_xs.append(x)
    host_ys.append(y)
    return y
  host_factor = line_oracle.line_maximize(eval_factor, evals)
  if host_factor != factor:
    # the two searches part where two scores tie within the summation noise of `dot` vs K2'
    k = next(i for i, (a, b) in enumerate(zip(host_xs, xs)) if a != b) - 1
    assert abs(host_ys[k] - ys[k]) <= 1e-5 * abs(ys[k]), (gar, k, host_ys, ys)
  return search

@pytest.mark.parametrize("n", [11, 25, 51])
@pytest.mark.parametrize("gar", ["average", "median", "trmean", "phocas", "meamed", "krum", "bulyan", "brute", "aksel", "cge"])
def test_device_search_matches_the_host_search(gar, n):
  import byzantinemomentum_b200 as bz
  f = F_OF[(gar, n)]
  f_real = f
  nh = n - f_real
  for d, offset in ((1, 0), (1031, 0), (1031, 1), (4099, 0)):
    honest = _honest(nh, d, 11 + d + n, offset)
    for kind, negative in (("identical", False), ("identical", True), ("empire-strict", False)):
      avg, att = _direction(honest, kind)
      for evals in (1, 2, 16):
        _check_search(bz, gar, honest, f_real, f, avg, att, evals, negative, kind)

def test_distance_rules_reuse_the_table_across_evaluations():
  """ Multi-Krum at n = 25 (aligned rows: the ring and its star pass) over a vector large enough for
  several CTAs: the same bits as the plain calls, which the checks above compare. """
  import byzantinemomentum_b200 as bz
  honest = _honest(20, 200_003, 3)
  avg, att = _direction(honest, "identical")
  for gar in ("krum", "bulyan", "brute"):
    f = 5 if gar != "brute" else 2
    _check_search(bz, gar, honest[:25 - f], f, f, avg, att, 16, False, "identical")

@pytest.mark.parametrize("gar", ["bulyan", "brute"])
def test_failed_evaluations_raise_like_the_plain_call(gar):
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine, _lib
  n, f = 11, 2 if gar == "bulyan" else 3
  honest = _honest(n - f, 515, 21)
  for k in range(6):                               # non-finite rows: no finite Multi-Krum scores / subsets
    honest[k] = honest[k].clone()
    honest[k][k] = math.nan
  avg, att = _direction(honest[6:], "identical")
  with pytest.raises(Exception) as plain:
    _plain(bz, gar, honest, avg + att, f, f)
  expected = type(plain.value)
  assert expected in (TypeError, AssertionError)
  with pytest.raises(expected):
    engine.line_search(gar, honest, f, f, avg, att, 16)
  engine.config.strict_status = False
  try:
    search = engine.LineSearch(gar, honest, f, f, avg, att, 16)
    byz = search()
    factor, trace = search.result()
    status = int(search.record.cpu()[-1:].view(torch.int32)[0])
  finally:
    engine.config.strict_status = True
  assert status in (_lib.STATUS_DEGENERATE, _lib.STATUS_NO_FINITE_SET)
  # the documented behaviour: a failed rule's output is NaN, so its score is NaN and never wins
  assert math.isnan(trace[0][1]) and factor == 0. and torch.equal(byz, avg + 0. * att)
  assert [x for x, _ in trace] == _oracle_xs([y for _, y in trace])

def _oracle_xs(ys):
  xs = []
  line_oracle.line_maximize(lambda x: (xs.append(x), ys[len(xs) - 1])[1], len(ys))
  return xs

def test_a_graph_replays_the_eager_search_bit_for_bit():
  from byzantinemomentum_b200 import engine
  for gar, kind in (("krum", "identical"), ("trmean", "empire-strict"), ("bulyan", "identical"), ("aksel", "identical")):
    honest = _honest(20, 30_011, 31)
    avg, att = _direction(honest, kind)
    search = engine.LineSearch(gar, honest, 5, 5, avg, att, 16, negative=True, kind=kind)
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
