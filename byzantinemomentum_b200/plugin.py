# coding: utf-8
"""Registration of the CUDA rules inside the reference's own registry.

The reference resolves `--gar <name>` through `aggregators.gars` (attack.py:468).  Two
routes lead there without touching a reference file:

  1. `install(aggregators)` — calls the reference's `aggregators.register(name, unchecked,
     check, upper_bound, influence)` (aggregators/__init__.py:71-86) for every rule, under
     `<prefix><name>` (default prefix "b200-"), or replaces the stock entries in place with
     `override=True` (`register` refuses duplicates, :82-84, so the entry is rebuilt with the
     reference's `make_gar`).  With `wide=True` it registers krum, bulyan, aksel and cge from
     `gars.wide_gars`, which take up to 128 gradients instead of 64; with `many=True`, average, median,
     trmean, phocas and meamed from `gars.many_gars`, which take up to 1024 gradients instead of 128; with
     `many_distance=True`, krum, bulyan, aksel and cge from `gars.many_distance_gars`, which take up to 1024.
  2. the top-level `native` package of this repository: the reference already looks for
     `native.{median,krum,bulyan,brute}.aggregate` and registers `native-<name>` when it finds
     them (median.py:80-87, krum.py:159-166, bulyan.py:137-144, brute.py:149-156).

`install_attacks(attacks)` then lets the line-searching attacks run their whole search on the device
(`engine.line_search`) when the rule they attack is one `install` registered, and, asked for by name, the
attack against CGE run on the device (`engine.anticge`).  The search takes the rows the entry takes: up to
128 against a wide entry, and against a default entry as many as `bz_line_search` takes
(`engine.search_max_rows`); with `install_attacks(..., many=True)`, up to 1024 against an entry of
`install(..., many=True)`, and with `install_attacks(..., many_distance=True)`, up to 1024 against an entry of
`install(..., many_distance=True)`.
"""

import math

from .gars import gars, wide_gars, many_gars, many_distance_gars

__all__ = ["install", "install_tools", "install_attacks"]

# The reference registry's entries that `install` made, each mapped to the name of its rule here and the most
# rows the device search takes against it: the attacks replaced by `install_attacks` recognise the rule they
# attack by identity.
_installed = {}
# The entries of `_installed` that `install` took from `gars.many_gars`: `install_attacks(..., many=True)` searches against
# them up to MAX_N_MANY rows.
_many_installed = set()
# The entries of `_installed` that `install` took from `gars.many_distance_gars`: `install_attacks(..., many_distance=True)`
# searches against them up to MAX_N_MANY rows.
_many_distance_installed = set()

def _record(aggregators, key, name, rule):
  from . import engine, _lib
  entry = aggregators.gars.get(key)
  if entry is not None and getattr(entry, "unchecked", None) is rule.unchecked:
    # a many_distance entry is its wide entry up to 128 rows, where the device search stops against it
    wide = wide_gars.get(name) is rule or many_distance_gars.get(name) is rule
    _installed[entry] = (name, _lib.MAX_N_DISTANCE if wide else engine.search_max_rows(name))
    if many_gars.get(name) is rule:
      _many_installed.add(entry)
    else:
      _many_installed.discard(entry)
    if many_distance_gars.get(name) is rule:
      _many_distance_installed.add(entry)
    else:
      _many_distance_installed.discard(entry)

def install(aggregators, prefix="b200-", override=False, names=None, wide=False, many=False, many_distance=False):
  """ Register the CUDA rules in the reference's `aggregators` module.
  Args:
    aggregators  The imported reference package (duck-typed: needs `gars`, `register`, `make_gar`)
    prefix       Name prefix of the new entries (ignored with override)
    override     Replace the stock rules under their own names instead
    names        Iterable of rule names to install (default: all)
    wide         Register krum, bulyan, aksel and cge from `gars.wide_gars`: up to 128 gradients, and the
                 attacks' device search against them up to 128 rows.  The default, False, keeps `gars`' entries,
                 which stop at 64 gradients, as every earlier release did; the other six rules are the same
                 either way
    many         Register average, median, trmean, phocas and meamed from `gars.many_gars`: up to 1024 gradients.
                 The attacks' device search against them keeps its 128 rows, unless `install_attacks(..., many=True)`
                 takes it to 1024; above, the stock attack runs and calls the entry for each evaluation.  The default,
                 False, keeps `gars`' entries, which stop at 128
    many_distance  Register krum, bulyan, aksel and cge from `gars.many_distance_gars`: up to 1024 gradients.  The
                 attacks' device search against them keeps its 128 rows, as against a wide entry, unless
                 `install_attacks(..., many_distance=True)` takes it to 1024; above, the stock attack runs and calls
                 the entry for each evaluation.  Combines with `many`, not with `wide`
  Returns:
    List of the registered names
  """
  if wide and many_distance:
    raise ValueError("install takes wide=True or many_distance=True, not both: both register krum, bulyan, aksel and cge")
  done = []
  for name in (names or gars.keys()):
    if many_distance and name in many_distance_gars:
      rule = many_distance_gars[name]
    else:
      rule = wide_gars[name] if wide and name in wide_gars else many_gars[name] if many and name in many_gars else gars[name]
    if override:
      wrapped = aggregators.make_gar(rule.unchecked, rule.check, upper_bound=rule.upper_bound, influence=rule.influence)
      aggregators.gars[name] = wrapped
      setattr(aggregators, name, wrapped)
      _record(aggregators, name, name, rule)
      done.append(name)
    else:
      target = prefix + name
      if target not in aggregators.gars:
        aggregators.register(target, rule.unchecked, rule.check, upper_bound=rule.upper_bound, influence=rule.influence)
      _record(aggregators, target, name, rule)
      done.append(target)
  return done

def install_tools(tools, many=False):
  """ Replace `tools.compute_avg_dev_max` (tools/pytorch.py:97, used by attack.py:846-848 for the
  study metrics) with the CUDA version when the samples live on a GPU.  CPU samples keep the
  reference's own function: this is a device kernel, not a CPU reimplementation.
  Args:
    tools  The imported reference `tools` package
    many   Take up to 1024 CUDA samples on the device (`engine.compute_avg_dev_max(..., many=True)`) instead of 128
  Returns:
    The previous function
  """
  from . import engine, _lib
  stock = tools.compute_avg_dev_max
  limit = _lib.MAX_N_MANY if many else _lib.MAX_N_COORDINATE
  def compute_avg_dev_max(samples):
    if len(samples) > 0 and samples[0].is_cuda and len(samples) <= limit:
      return engine.compute_avg_dev_max(samples, many=True) if many else engine.compute_avg_dev_max(samples)
    return stock(samples)
  compute_avg_dev_max.__doc__ = stock.__doc__
  tools.compute_avg_dev_max = compute_avg_dev_max
  return stock

# ---------------------------------------------------------------------------- #
# The attacks' line search on the device

def _is_cuda(tensors):
  return all(t.is_cuda for t in tensors)

def _device_rule(defense, grad_honests, f_real, f_decl, model, many=False, many_distance=False):
  """ The name of the rule here that `defense` is, when the attack's search can run on the device:
  `defense` is an entry `install` registered, there are Byzantine rows to generate, every honest
  gradient is a float32 CUDA vector, the rule's input fits the search's row limit for that entry
  (128 rows for a wide entry of `install(..., wide=True)`; with `many`, 1024 rows for an entry of
  `install(..., many=True)`; with `many_distance`, 1024 rows for an entry of `install(..., many_distance=True)`; otherwise `engine.search_max_rows`: 128 rows for the coordinate-wise rules, 64 for
  the distance rules), and the rule accepts its parameters.  None otherwise: the stock attack then runs (and
  fails, if it must, as it always did). """
  import torch
  try:
    installed = _installed.get(defense)
  except TypeError:                            # unhashable: not one of ours
    return None
  if installed is None or not isinstance(f_real, int) or f_real < 1 or not isinstance(grad_honests, list) or not grad_honests:
    return None
  name, limit = installed
  if (many and defense in _many_installed) or (many_distance and defense in _many_distance_installed):
    from . import _lib
    limit = _lib.MAX_N_MANY
  if len(grad_honests) + f_real > limit or not _is_cuda(grad_honests):
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

def _search(backend, rule, grad_honests, f_real, *args, **kwargs):
  """ `backend.line_search(rule, grad_honests, f_real, *args, **kwargs)`, above MAX_N_COORDINATE rows with `many=True`
  for a coordinate-wise rule (only an entry of `install(..., many=True)` gets there, through
  `install_attacks(..., many=True)`) and `many_distance=True` for krum, bulyan, aksel and cge (only an entry of
  `install(..., many_distance=True)` gets there, through `install_attacks(..., many_distance=True)`). """
  from . import _lib
  if len(grad_honests) + f_real > _lib.MAX_N_COORDINATE:
    kwargs["many_distance" if rule in many_distance_gars else "many"] = True
  return backend.line_search(rule, grad_honests, f_real, *args, **kwargs)

def _identical(stock, direction, backend, many=False, many_distance=False):
  """ attacks/identical.py:46-86 with the factor search on the device. """
  def attack(grad_honests, f_real, f_decl, defense, model, factor=-16, negative=False, **kwargs):
    rule = _device_rule(defense, grad_honests, f_real, f_decl, model, many, many_distance) if factor < 0 else None
    if rule is None:
      return stock(grad_honests=grad_honests, f_real=f_real, f_decl=f_decl, defense=defense, model=model,
                   factor=factor, negative=negative, **kwargs)
    import torch
    grad_stck = torch.stack(grad_honests)
    grad_avg = grad_stck.mean(dim=0)
    grad_att = direction(grad_stck, grad_avg, **kwargs)
    _, byz = _search(backend, rule, grad_honests, f_real, f_decl, grad_avg, grad_att, math.ceil(-factor),
                     negative=negative, kind="identical")
    return [byz] * f_real
  return attack

def _empire_strict(stock, backend, many=False, many_distance=False):
  """ attacks/empire.py:29-65 with the epsilon search on the device. """
  def attack(grad_honests, f_real, f_decl, defense, model, epsilon=1, **kwargs):
    rule = _device_rule(defense, grad_honests, f_real, f_decl, model, many, many_distance) if epsilon < 0 else None
    if rule is None:
      return stock(grad_honests=grad_honests, f_real=f_real, f_decl=f_decl, defense=defense, model=model,
                   epsilon=epsilon, **kwargs)
    grad_avg = grad_honests[0].clone().detach()
    for grad in grad_honests[1:]:
      grad_avg.add_(grad)
    grad_avg.div_(len(grad_honests))
    _, byz = _search(backend, rule, grad_honests, f_real, f_decl, grad_avg, None, math.ceil(-epsilon), kind="empire-strict")
    return [byz] * f_real
  return attack

def _anticge(stock, backend):
  """ attacks/anticge.py:49-78 on the device (`engine.anticge`) when the honest rows are fp32 CUDA vectors and
  `bz_anticge` takes the arguments (`engine.anticge_takes`: 1..128 rows, 0 <= nh - f_decl < nh, f_real >= 0);
  the stock attack, with its arguments unchanged, otherwise. """
  def attack(grad_honests, f_decl, f_real, **kwargs):
    import torch
    from . import engine
    if (engine.anticge_takes(grad_honests, f_decl, f_real) and _is_cuda(grad_honests)
        and all(g.dtype == torch.float32 and g.dim() == 1 for g in grad_honests)):
      return backend.anticge(grad_honests, f_decl, f_real)
    return stock(grad_honests=grad_honests, f_decl=f_decl, f_real=f_real, **kwargs)
  return attack

_ATTACK_NAMES = ("little", "empire", "bulyan", "empire-strict")

def install_attacks(attacks, backend=None, names=None, many=False, many_distance=False):
  """ Replace `little`, `empire`, `bulyan` and `empire-strict` in the reference's `attacks` registry
  (attacks/__init__.py: `attacks`, `register`) with versions that, when the factor (epsilon) is negative
  and `defense` is a rule `install` registered, run the whole `line_maximize` search on the device and
  read its outcome once (`engine.line_search`).  The attack direction is computed with the reference's
  torch statements.  Every other call — positive factors, a `--gars` mixture, a stock rule, CPU tensors,
  more rows than the search takes against the entry (128 for a wide entry, `engine.search_max_rows` otherwise) —
  runs the stock attack unchanged.  The reference's `register` builds the
  checked wrappers, with the stock checks.
  `names` may also list "anticge": the attack against CGE then runs on the device (`engine.anticge`) whenever
  its honest rows are fp32 CUDA vectors and `bz_anticge` takes its arguments, whatever the defense.
  Args:
    attacks  The imported reference `attacks` package
    backend  Provider of `line_search` and `anticge` (default: `engine`; tests substitute a stand-in)
    names    Attacks to replace (default: the four line-searching ones)
    many     Against an entry of `install(..., many=True)`, search on the device up to 1024 rows, above 128 through
             `backend.line_search(..., many=True)`.  The default, False, keeps the search at 128 rows there
    many_distance  Against an entry of `install(..., many_distance=True)`, search on the device up to 1024 rows, above
             128 through `backend.line_search(..., many_distance=True)`.  The default, False, keeps the search at
             128 rows there.  Combines with `many`
  Returns:
    List of the replaced names """
  if backend is None:
    from . import engine as backend
  directions = {"little": _little, "empire": _empire, "bulyan": _bulyan}
  done = []
  for name in (_ATTACK_NAMES if names is None else names):
    stock = attacks.attacks.get(name)
    if stock is None:
      continue
    if name == "anticge":
      attack = _anticge(stock.unchecked, backend)
    elif name == "empire-strict":
      attack = _empire_strict(stock.unchecked, backend, many, many_distance)
    elif name in directions:
      attack = _identical(stock.unchecked, directions[name], backend, many, many_distance)
    else:
      raise KeyError(f"no device version of the attack {name!r}")
    del attacks.attacks[name]                  # `register` refuses duplicates
    attacks.register(name, attack, stock.check)
    setattr(attacks, name, attacks.attacks[name])
    done.append(name)
  return done
