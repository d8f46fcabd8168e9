# coding: utf-8
"""Registration of the CUDA rules inside the reference's own registry.

The reference resolves `--gar <name>` through `aggregators.gars` (attack.py:468).  Two
routes lead there without touching a reference file:

  1. `install(aggregators)` — calls the reference's `aggregators.register(name, unchecked,
     check, upper_bound, influence)` (aggregators/__init__.py:71-86) for every rule, under
     `<prefix><name>` (default prefix "b200-"), or replaces the stock entries in place with
     `override=True` (`register` refuses duplicates, :82-84, so the entry is rebuilt with the
     reference's `make_gar`).
  2. the top-level `native` package of this repository: the reference already looks for
     `native.{median,krum,bulyan,brute}.aggregate` and registers `native-<name>` when it finds
     them (median.py:80-87, krum.py:159-166, bulyan.py:137-144, brute.py:149-156).

`install_attacks(attacks)` then lets the line-searching attacks run their whole search on the device
(`engine.line_search`) when the rule they attack is one `install` registered.
"""

import math

from .gars import gars

__all__ = ["install", "install_tools", "install_attacks"]

# The reference registry's entries that `install` made, each mapped to the name of its rule here: the
# attacks replaced by `install_attacks` recognise the rule they attack by identity.
_installed = {}

def _record(aggregators, key, name):
  entry = aggregators.gars.get(key)
  if entry is not None and getattr(entry, "unchecked", None) is gars[name].unchecked:
    _installed[entry] = name

def install(aggregators, prefix="b200-", override=False, names=None):
  """ Register the CUDA rules in the reference's `aggregators` module.
  Args:
    aggregators  The imported reference package (duck-typed: needs `gars`, `register`, `make_gar`)
    prefix       Name prefix of the new entries (ignored with override)
    override     Replace the stock rules under their own names instead
    names        Iterable of rule names to install (default: all)
  Returns:
    List of the registered names
  """
  done = []
  for name in (names or gars.keys()):
    rule = gars[name]
    if override:
      wrapped = aggregators.make_gar(rule.unchecked, rule.check, upper_bound=rule.upper_bound, influence=rule.influence)
      aggregators.gars[name] = wrapped
      setattr(aggregators, name, wrapped)
      _record(aggregators, name, name)
      done.append(name)
    else:
      target = prefix + name
      if target not in aggregators.gars:
        aggregators.register(target, rule.unchecked, rule.check, upper_bound=rule.upper_bound, influence=rule.influence)
      _record(aggregators, target, name)
      done.append(target)
  return done

def install_tools(tools):
  """ Replace `tools.compute_avg_dev_max` (tools/pytorch.py:97, used by attack.py:846-848 for the
  study metrics) with the CUDA version when the samples live on a GPU.  CPU samples keep the
  reference's own function: this is a device kernel, not a CPU reimplementation.
  Args:
    tools  The imported reference `tools` package
  Returns:
    The previous function
  """
  from . import engine, _lib
  stock = tools.compute_avg_dev_max
  def compute_avg_dev_max(samples):
    if len(samples) > 0 and samples[0].is_cuda and len(samples) <= _lib.MAX_N:
      return engine.compute_avg_dev_max(samples)
    return stock(samples)
  compute_avg_dev_max.__doc__ = stock.__doc__
  tools.compute_avg_dev_max = compute_avg_dev_max
  return stock

# ---------------------------------------------------------------------------- #
# The attacks' line search on the device

def _is_cuda(tensors):
  return all(t.is_cuda for t in tensors)

def _device_rule(defense, grad_honests, f_real, f_decl, model):
  """ The name of the rule here that `defense` is, when the attack's search can run on the device:
  `defense` is an entry `install` registered, there are Byzantine rows to generate, every honest
  gradient is a float32 CUDA vector, the rule's input fits BZ_MAX_N rows, and the rule accepts its
  parameters.  None otherwise: the stock attack then runs (and fails, if it must, as it always did). """
  import torch
  from . import _lib
  try:
    name = _installed.get(defense)
  except TypeError:                            # unhashable: not one of ours
    return None
  if name is None or not isinstance(f_real, int) or f_real < 1 or not isinstance(grad_honests, list) or not grad_honests:
    return None
  if len(grad_honests) + f_real > _lib.MAX_N or not _is_cuda(grad_honests):
    return None
  if any(g.dtype != torch.float32 or g.dim() != 1 for g in grad_honests):
    return None
  if gars[name].check(gradients=grad_honests + grad_honests[:1] * f_real, f=f_decl, model=model) is not None:
    return None
  return name

def _little(grad_stck, grad_avg, **kwargs):
  return grad_stck.var(dim=0).sqrt_()

def _empire(grad_stck, grad_avg, **kwargs):
  return grad_avg.neg()

def _bulyan(grad_stck, grad_avg, target_idx=-1, **kwargs):
  import torch
  if target_idx == "all":
    return torch.ones_like(grad_avg)
  assert isinstance(target_idx, int), f"Expected an integer or \"all\" for 'target_idx', got {target_idx!r}"
  grad_att = torch.zeros_like(grad_avg)
  grad_att[target_idx] = 1
  return grad_att

def _identical(stock, direction, backend):
  """ attacks/identical.py:46-86 with the factor search on the device. """
  def attack(grad_honests, f_real, f_decl, defense, model, factor=-16, negative=False, **kwargs):
    rule = _device_rule(defense, grad_honests, f_real, f_decl, model) if factor < 0 else None
    if rule is None:
      return stock(grad_honests=grad_honests, f_real=f_real, f_decl=f_decl, defense=defense, model=model,
                   factor=factor, negative=negative, **kwargs)
    import torch
    grad_stck = torch.stack(grad_honests)
    grad_avg = grad_stck.mean(dim=0)
    grad_att = direction(grad_stck, grad_avg, **kwargs)
    _, byz = backend.line_search(rule, grad_honests, f_real, f_decl, grad_avg, grad_att, math.ceil(-factor),
                                 negative=negative, kind="identical")
    return [byz] * f_real
  return attack

def _empire_strict(stock, backend):
  """ attacks/empire.py:29-65 with the epsilon search on the device. """
  def attack(grad_honests, f_real, f_decl, defense, model, epsilon=1, **kwargs):
    rule = _device_rule(defense, grad_honests, f_real, f_decl, model) if epsilon < 0 else None
    if rule is None:
      return stock(grad_honests=grad_honests, f_real=f_real, f_decl=f_decl, defense=defense, model=model,
                   epsilon=epsilon, **kwargs)
    grad_avg = grad_honests[0].clone().detach()
    for grad in grad_honests[1:]:
      grad_avg.add_(grad)
    grad_avg.div_(len(grad_honests))
    _, byz = backend.line_search(rule, grad_honests, f_real, f_decl, grad_avg, None, math.ceil(-epsilon), kind="empire-strict")
    return [byz] * f_real
  return attack

def install_attacks(attacks, backend=None):
  """ Replace `little`, `empire`, `bulyan` and `empire-strict` in the reference's `attacks` registry
  (attacks/__init__.py: `attacks`, `register`) with versions that, when the factor (epsilon) is negative
  and `defense` is a rule `install` registered, run the whole `line_maximize` search on the device and
  read its outcome once (`engine.line_search`).  The attack direction is computed with the reference's
  torch statements.  Every other call — positive factors, a `--gars` mixture, a stock rule, CPU tensors,
  more than BZ_MAX_N rows — runs the stock attack unchanged.  The reference's `register` builds the
  checked wrappers, with the stock checks.
  Args:
    attacks  The imported reference `attacks` package
    backend  Provider of `line_search` (default: `engine`; tests substitute a stand-in)
  Returns:
    List of the replaced names """
  if backend is None:
    from . import engine as backend
  directions = {"little": _little, "empire": _empire, "bulyan": _bulyan}
  done = []
  for name in ("little", "empire", "bulyan", "empire-strict"):
    stock = attacks.attacks.get(name)
    if stock is None:
      continue
    if name == "empire-strict":
      attack = _empire_strict(stock.unchecked, backend)
    else:
      attack = _identical(stock.unchecked, directions[name], backend)
    del attacks.attacks[name]                  # `register` refuses duplicates
    attacks.register(name, attack, stock.check)
    setattr(attacks, name, attacks.attacks[name])
    done.append(name)
  return done
