# coding: utf-8
"""`plugin.install_attacks` against stand-ins with the interfaces of the reference's registries
(`attacks`: `attacks`, `register`; `aggregators`: `gars`, `register`, `make_gar`): which calls take the
device search and which run the stock attack unchanged, and what the device path hands the search.
The search itself is a stand-in here (a host loop of `line_maximize`, restated in tests/line_oracle.py);
the CUDA path is covered by tests/test_cuda_linesearch.py."""

import math
import types

import pytest

torch = pytest.importorskip("torch")

import byzantinemomentum_b200 as bz
from byzantinemomentum_b200 import plugin

def _aggregators():
  ns = types.SimpleNamespace(gars={})
  def make_gar(unchecked, check, upper_bound=None, influence=None):
    def checked(**kwargs):
      message = check(**kwargs)
      if message is not None:
        raise RuntimeError(message)
      return unchecked(**kwargs)
    checked.check, checked.checked, checked.unchecked = check, checked, unchecked
    checked.upper_bound, checked.influence = upper_bound, influence
    return checked
  def register(name, unchecked, check, upper_bound=None, influence=None):
    if name in ns.gars:
      raise KeyError(name)
    ns.gars[name] = make_gar(unchecked, check, upper_bound=upper_bound, influence=influence)
  ns.make_gar, ns.register = make_gar, register
  ns.gars["krum"] = make_gar(lambda **kw: "stock rule", lambda **kw: None)
  return ns

def _attacks():
  ns = types.SimpleNamespace(attacks={})
  def register(name, unchecked, check):
    if name in ns.attacks:
      raise KeyError(name)                       # attacks/__init__.py refuses duplicates
    def checked(f_real, **kwargs):
      message = check(f_real=f_real, **kwargs)
      if message is not None:
        raise RuntimeError(message)
      return unchecked(f_real=f_real, **kwargs)
    checked.check, checked.checked, checked.unchecked = check, checked, unchecked
    ns.attacks[name] = checked
  ns.register = register
  for name in ("little", "empire", "bulyan", "empire-strict", "nan"):
    register(name, (lambda name: lambda **kw: ("stock", name, kw))(name), lambda **kw: None)
  return ns

class SearchStandIn:
  """ Records the calls; returns (factor, byz) from a host `line_maximize` over a fixed scape. """
  def __init__(self):
    self.calls = []
  def line_search(self, gar, grad_honests, f_real, f_decl, grad_avg, grad_att, evals, negative=False, kind="identical"):
    self.calls.append(dict(gar=gar, honests=grad_honests, f_real=f_real, f_decl=f_decl, avg=grad_avg, att=grad_att,
                           evals=evals, negative=negative, kind=kind))
    import line_oracle
    factor = line_oracle.line_maximize(lambda x: -(x - 3.) ** 2, evals)
    return factor, grad_avg.mul(-factor) if grad_att is None else grad_avg + factor * grad_att

@pytest.fixture
def setup(monkeypatch):
  aggregators, attacks, backend = _aggregators(), _attacks(), SearchStandIn()
  bz.plugin.install(aggregators)
  stock_krum = aggregators.gars["krum"]
  assert bz.plugin.install_attacks(attacks, backend=backend) == ["little", "empire", "bulyan", "empire-strict"]
  monkeypatch.setattr(plugin, "_is_cuda", lambda tensors: all(t.device.type == "cpu" for t in tensors))   # CPU rows stand for CUDA rows
  gen = torch.Generator().manual_seed(3)
  honest = [torch.randn(33, generator=gen) for _ in range(20)]
  return types.SimpleNamespace(aggregators=aggregators, attacks=attacks, backend=backend, honest=honest, stock_krum=stock_krum)

def _run(s, name, defense, f_real=5, f_decl=5, honest=None, **kwargs):
  return s.attacks.attacks[name].checked(grad_honests=s.honest if honest is None else honest, f_real=f_real, f_decl=f_decl,
                                         defense=defense, model=None, **kwargs)

def test_negative_factor_against_an_installed_rule_runs_the_device_search(setup):
  s = setup
  stck = torch.stack(s.honest)
  avg = stck.mean(dim=0)
  directions = {"little": stck.var(dim=0).sqrt_(), "empire": avg.neg(), "bulyan": torch.zeros(33).index_fill_(0, torch.tensor([32]), 1.)}
  for name, att in directions.items():
    for gar in ("b200-krum", "b200-median", "b200-cge"):
      out = _run(s, name, s.aggregators.gars[gar], factor=-16, negative=name == "little")
      call = s.backend.calls.pop()
      assert (call["gar"], call["evals"], call["negative"], call["kind"], call["f_real"], call["f_decl"]) == \
             (gar[5:], 16, name == "little", "identical", 5, 5)
      assert call["honests"] is s.honest
      assert torch.equal(call["avg"], avg) and torch.equal(call["att"], att), name
      assert len(out) == 5 and all(o is out[0] for o in out)               # one tensor, f_real times
  ones = _run(s, "bulyan", s.aggregators.gars["b200-trmean"], factor=-3, target_idx="all")
  assert torch.equal(s.backend.calls.pop()["att"], torch.ones(33)) and len(ones) == 5
  # empire-strict: the average of clone + add_ + div_, no direction
  _run(s, "empire-strict", s.aggregators.gars["b200-bulyan"], f_decl=4, epsilon=-7)
  call = s.backend.calls.pop()
  want = s.honest[0].clone()
  for g in s.honest[1:]:
    want.add_(g)
  want.div_(20)
  assert call["kind"] == "empire-strict" and call["att"] is None and call["evals"] == 7 and torch.equal(call["avg"], want)

def test_every_other_case_runs_the_stock_attack(setup, monkeypatch):
  s = setup
  ours = s.aggregators.gars["b200-krum"]
  def stock(result, name):
    return isinstance(result, tuple) and result[:2] == ("stock", name)
  assert stock(_run(s, "little", ours, factor=1.5), "little")                     # positive factor: the published grid
  assert stock(_run(s, "empire", ours, factor=4), "empire")
  assert stock(_run(s, "empire-strict", ours, epsilon=2), "empire-strict")
  assert stock(_run(s, "little", s.stock_krum, factor=-16), "little")             # a stock rule
  assert stock(_run(s, "little", lambda **kw: None, factor=-16), "little")        # a --gars mixture (a closure)
  assert stock(_run(s, "empire", ours, factor=-16, f_real=0), "empire")          # nothing to generate
  assert stock(_run(s, "empire", ours, factor=-16, f_real=45), "empire")         # 65 rows > BZ_MAX_N
  assert stock(_run(s, "empire", ours, factor=-16, f_decl=12), "empire")         # the rule rejects f: the stock call raises as before
  assert stock(_run(s, "empire", ours, factor=-16, honest=[g.double() for g in s.honest]), "empire")
  assert stock(_run(s, "nan", ours, factor=-16), "nan")                          # not replaced
  assert not s.backend.calls
  monkeypatch.setattr(plugin, "_is_cuda", lambda tensors: False)                # CPU tensors
  assert stock(_run(s, "little", ours, factor=-16), "little")
  assert not s.backend.calls
  # the stock attack receives every argument unchanged
  kind, name, kw = _run(s, "bulyan", ours, factor=2., negative=True, target_idx=3)
  assert kw["factor"] == 2. and kw["negative"] is True and kw["target_idx"] == 3 and kw["defense"] is ours

def test_override_install_is_recognised_and_the_stock_checks_still_apply(setup):
  s = setup
  bz.plugin.install(s.aggregators, override=True, names=["krum"])
  _run(s, "empire", s.aggregators.gars["krum"], factor=-2)
  assert s.backend.calls.pop()["gar"] == "krum"
  check = s.attacks.attacks["little"].check
  assert check is s.attacks.attacks["little"].checked.check
