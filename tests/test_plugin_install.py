# coding: utf-8
"""`plugin.install` against a stand-in with the reference registry's interface (`gars`,
`register`, `make_gar`: aggregators/__init__.py:42-86), so that the registration logic is
covered without the reference's code."""

import types

import pytest

import byzantinemomentum_b200 as bz

def _registry():
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
      raise KeyError(name)                     # the reference refuses duplicates (:82-84)
    ns.gars[name] = make_gar(unchecked, check, upper_bound=upper_bound, influence=influence)
  ns.make_gar, ns.register = make_gar, register
  ns.gars["krum"] = make_gar(lambda **kw: "stock", lambda **kw: None)
  return ns

def test_install_adds_prefixed_rules_and_is_idempotent():
  ns = _registry()
  names = bz.plugin.install(ns)
  assert names == ["b200-" + name for name in bz.gars]
  assert ns.gars["krum"].unchecked() == "stock"            # stock entries untouched
  rule = ns.gars["b200-krum"]
  assert rule.unchecked is bz.gars["krum"].unchecked and rule.check is bz.gars["krum"].check
  assert rule.upper_bound(25, 5, 10) == bz.gars["krum"].upper_bound(25, 5, 10)
  assert bz.plugin.install(ns) == names                    # second call: nothing to add, no KeyError
  assert bz.plugin.install(ns, prefix="x-", names=["median"]) == ["x-median"] and "x-median" in ns.gars

def test_override_replaces_the_stock_entry_in_place():
  ns = _registry()
  assert bz.plugin.install(ns, override=True, names=["krum"]) == ["krum"]
  assert ns.gars["krum"].unchecked is bz.gars["krum"].unchecked
  assert ns.krum is ns.gars["krum"]                        # module attribute too (aggregators.krum)
  with pytest.raises(RuntimeError):                        # the REGISTRY's wrapper, our check
    ns.gars["krum"].checked(gradients=[0] * 5, f=2)
