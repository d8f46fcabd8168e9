# coding: utf-8
"""The aggregation rules behind the reference's plugin interface.

Mirrors `aggregators/__init__.py:15-86` of LPD-EPFL/ByzantineMomentum: every rule is a
callable taking keyword arguments only (`gradients`, `f`, `model`, plus rule specific ones;
unknown keywords are accepted and ignored), returning a NEW tensor, and carrying the members
`check`, `checked`, `unchecked`, `upper_bound`, `influence`.  `gars` maps the reference's
names (average, median, trmean, phocas, meamed, krum, bulyan, brute, aksel, cge) to them.
`wide_gars` holds krum, bulyan, aksel and cge again, built the same way, for 1 to 128 gradients
(`BZ_MAX_N_DISTANCE`): up to 64 they make exactly the call of their `gars` entry, above it they run
`bz_distance`.  `plugin.install(..., wide=True)` registers them.  `many_gars` holds the five coordinate-wise
rules again, for 1 to 1024 gradients (`BZ_MAX_N_MANY`): up to 128 they make exactly the call of their `gars`
entry, above it they run `bz_coordinate_many`.  `plugin.install(..., many=True)` registers them.
`many_distance_gars` holds krum, bulyan, aksel and cge once more, for 1 to 1024 gradients: up to 128 they make
exactly the call of their `wide_gars` entry, above it they run `bz_distance_many`.
`plugin.install(..., many_distance=True)` registers them.
The arithmetic runs in `libbyzagg.so` (see `engine.py`); this module only holds the
argument checks, the closed-form bounds and the selection bookkeeping for `influence`.

Differences with the reference, all deliberate:
  * `influence(honests, attacks, ...)` right after an aggregation over the same tensors
    reuses the selection computed on the device instead of recomputing all distances
    (attack.py:822 always follows attack.py:821);
  * the coordinate-wise rules (average, median, trmean, phocas, meamed) take up to 128 gradients
    (`BZ_MAX_N_COORDINATE`), and those of `many_gars` up to 1024 (`BZ_MAX_N_MANY`); with more than 64 gradients the distance-based rules of `gars` raise
    (`BZ_MAX_N`), with a message saying so, and those of `wide_gars` take up to 128.  Above 64
    gradients a `wide_gars` call reuses no distance of the previous call.
"""

import math

from . import _lib, engine
from .engine import _Memo as _Selection, _rule

__all__ = ["gars", "wide_gars", "many_gars", "many_distance_gars", "make_gar", "register", "UserException", "last_selection"]

class UserException(RuntimeError):
  """ Raised by `checked` on invalid parameters (the reference raises tools.UserException). """

# ---------------------------------------------------------------------------- #
# Wrapper (aggregators/__init__.py:42-69)

def make_gar(unchecked, check, upper_bound=None, influence=None, name=None, user_exception=None):
  label = name or getattr(unchecked, "__name__", "?")
  exc = user_exception or UserException
  def checked(**kwargs):
    message = check(**kwargs)
    if message is not None:
      raise exc(f"Aggregation rule {label!r} cannot be used with the given parameters: {message}")
    return unchecked(**kwargs)
  func = checked if __debug__ else unchecked
  func.check = check
  func.checked = checked
  func.unchecked = unchecked
  func.upper_bound = upper_bound
  func.influence = influence
  return func

gars = dict()

def register(name, unchecked, check, upper_bound=None, influence=None):
  if name in gars:
    raise KeyError(f"GAR name {name!r} already in use")
  gars[name] = make_gar(unchecked, check, upper_bound=upper_bound, influence=influence, name=name)

# ---------------------------------------------------------------------------- #
# Shared checks

def _bad_list(gradients):
  if not isinstance(gradients, list) or len(gradients) < 1:
    return f"Expected a list of at least one gradient to aggregate, got {gradients!r}"
  return None

def _bad_f(gradients, f, per_f, offset):
  """ f must be an int >= 1 with n >= per_f * f + offset. """
  n = len(gradients)
  if not isinstance(f, int) or f < 1 or n < per_f * f + offset:
    return f"Invalid number of Byzantine gradients to tolerate, got f = {f!r}, expected 1 ≤ f ≤ {(n - offset) // per_f}"
  return None

def _bad_m(gradients, f, m):
  limit = len(gradients) - f - 2
  if m is not None and (not isinstance(m, int) or m < 1 or m > limit):
    return f"Invalid number of selected gradients, got m = {m!r}, expected 1 ≤ m ≤ {limit}"
  return None

# ---------------------------------------------------------------------------- #
# Selection bookkeeping for `influence`

_last = _Selection()          # the last device-side selection of a rule with its parameters

def last_selection():
  """ Indices selected by the last distance-based aggregation (host list), or None. """
  return None if _last.value is None else _last.value.tolist()

def _accepted_ratio(indices, nb_honests, count):
  """ Share of the selected slots held by attack gradients: the reference tests object
  identity against the attack list (krum.py:145-149); honests come first, attacks last. """
  picked = indices.tolist()[:count]
  return sum(1 for i in picked if i >= nb_honests) / count

# ---------------------------------------------------------------------------- #
# average (aggregators/average.py)

def _average(gradients, **kwargs):
  return engine.average(gradients)

def _average_check(gradients, **kwargs):
  return _bad_list(gradients)

def _average_influence(honests, attacks, **kwargs):
  return len(attacks) / (len(honests) + len(attacks))

register("average", _average, _average_check, influence=_average_influence)

# ---------------------------------------------------------------------------- #
# median (aggregators/median.py)

def _median(gradients, **kwargs):
  return engine.median(gradients)

def _median_check(gradients, **kwargs):
  return _bad_list(gradients)

def _median_bound(n, f, d):
  return 1 / math.sqrt(n - f)

register("median", _median, _median_check, upper_bound=_median_bound)

# ---------------------------------------------------------------------------- #
# trmean / phocas / meamed (aggregators/trmean.py)

def _trim_check(gradients, f, **kwargs):
  return _bad_list(gradients) or _bad_f(gradients, f, 2, 1)

def _trmean(gradients, f, **kwargs):
  return engine.trmean(gradients, f)

def _phocas(gradients, f, **kwargs):
  return engine.phocas(gradients, f)

def _meamed(gradients, f, **kwargs):
  return engine.meamed(gradients, f)

register("trmean", _trmean, _trim_check)
register("phocas", _phocas, _trim_check)
register("meamed", _meamed, _trim_check)

# ---------------------------------------------------------------------------- #
# Multi-Krum (aggregators/krum.py)

def _krum(gradients, f, m=None, **kwargs):
  out, order = engine.krum(gradients, f, m)
  _last.store("krum", (f,), gradients, order)
  return out

def _krum_check(gradients, f, m=None, **kwargs):
  return _bad_list(gradients) or _bad_f(gradients, f, 2, 3) or _bad_m(gradients, f, m)

def _krum_bound(n, f, d):
  return 1 / math.sqrt(2 * (n - f + f * (n + f * (n - f - 2) - 2) / (n - 2 * f - 2)))

def _krum_influence(honests, attacks, f, m=None, **kwargs):
  gradients = honests + attacks
  order = _last.lookup("krum", (f,), gradients)
  if order is None:
    _, order = engine.krum(gradients, f, m)
  return _accepted_ratio(order, len(honests), _rule("krum", len(gradients), f, m).count)

register("krum", _krum, _krum_check, upper_bound=_krum_bound, influence=_krum_influence)

# ---------------------------------------------------------------------------- #
# Bulyan over Multi-Krum (aggregators/bulyan.py)

def _bulyan(gradients, f, m=None, **kwargs):
  out, _ = engine.bulyan(gradients, f, m)
  return out

def _bulyan_check(gradients, f, m=None, **kwargs):
  return _bad_list(gradients) or _bad_f(gradients, f, 4, 3) or _bad_m(gradients, f, m)

register("bulyan", _bulyan, _bulyan_check, upper_bound=_krum_bound)

# ---------------------------------------------------------------------------- #
# brute (aggregators/brute.py)

def _brute(gradients, f, **kwargs):
  out, sel = engine.brute(gradients, f)
  _last.store("brute", (f,), gradients, sel)
  return out

def _brute_check(gradients, f, **kwargs):
  return _bad_list(gradients) or _bad_f(gradients, f, 2, 1)

def _brute_bound(n, f, d):
  return (n - f) / (math.sqrt(8) * f)

def _brute_influence(honests, attacks, f, **kwargs):
  gradients = honests + attacks
  sel = _last.lookup("brute", (f,), gradients)
  if sel is None:
    _, sel = engine.brute(gradients, f)
  return _accepted_ratio(sel, len(honests), len(gradients) - f)

register("brute", _brute, _brute_check, upper_bound=_brute_bound, influence=_brute_influence)

# ---------------------------------------------------------------------------- #
# aksel (aggregators/aksel.py)

def _aksel(gradients, f, mode="mid", **kwargs):
  out, order = engine.aksel(gradients, f, mode)
  _last.store("aksel", (), gradients, order)
  return out

def _aksel_check(gradients, f, mode="mid", **kwargs):
  message = _bad_list(gradients) or _bad_f(gradients, f, 2, 1)
  if message is None and mode not in ("mid", "n-f"):
    message = f"Invalid operation mode {mode!r}"
  return message

def _aksel_influence(honests, attacks, f, mode="mid", **kwargs):
  gradients = honests + attacks
  count = _rule("aksel", len(gradients), f, mode=mode).count
  order = _last.lookup("aksel", (), gradients)
  if order is None:
    _, order = engine.aksel(gradients, f, mode)
  return _accepted_ratio(order, len(honests), count)

register("aksel", _aksel, _aksel_check, influence=_aksel_influence)

# ---------------------------------------------------------------------------- #
# CGE (aggregators/cge.py)

def _cge(gradients, f, **kwargs):
  out, order = engine.cge(gradients, f)
  _last.store("cge", (), gradients, order)
  return out

def _cge_check(gradients, f, m=None, **kwargs):
  return _bad_list(gradients)    # cge.py:59-70 validates nothing else

def _cge_influence(honests, attacks, f, **kwargs):
  gradients = honests + attacks
  order = _last.lookup("cge", (), gradients)
  if order is None:
    _, order = engine.cge(gradients, f)
  return _accepted_ratio(order, len(honests), len(gradients) - f)

register("cge", _cge, _cge_check, influence=_cge_influence)

# ---------------------------------------------------------------------------- #
# Multi-Krum, Bulyan, Aksel and CGE for up to 128 gradients

def _wide(name):
  """ The `wide_gars` entry of `name`: the check, bound and influence of `gars[name]`; up to MAX_N gradients its
  call, above it `engine.wide_distance` (`bz_distance`), which stores the selection for `influence` as it does. """
  narrow = gars[name]
  def unchecked(gradients, f, m=None, mode="mid", **kwargs):
    if not isinstance(gradients, list) or len(gradients) <= _lib.MAX_N:
      return narrow.unchecked(gradients=gradients, f=f, m=m, mode=mode, **kwargs)
    out, order = engine.wide_distance(name, gradients, f, m if name in ("krum", "bulyan") else None,
                                      mode if name == "aksel" else "mid")
    if name != "bulyan":
      _last.store(name, (f,) if name == "krum" else (), gradients, order)
    return out
  unchecked.__name__ = narrow.unchecked.__name__
  influence = None
  if narrow.influence is not None:
    def influence(honests, attacks, f, m=None, mode="mid", **kwargs):
      gradients = honests + attacks
      if len(gradients) > _lib.MAX_N and _last.lookup(name, (f,) if name == "krum" else (), gradients) is None:
        unchecked(gradients=gradients, f=f, m=m, mode=mode)
      return narrow.influence(honests, attacks, f=f, m=m, mode=mode, **kwargs)
  return make_gar(unchecked, narrow.check, upper_bound=narrow.upper_bound, influence=influence, name=name)

wide_gars = {name: _wide(name) for name in engine.WIDE_DISTANCE}

# ---------------------------------------------------------------------------- #
# The coordinate-wise rules for up to 1024 gradients

def _many(name):
  """ The `many_gars` entry of `name`: the check, bound and influence of `gars[name]`, the call of
  `engine.coordinate_many` (which is `gars[name]`'s call up to MAX_N_COORDINATE gradients). """
  narrow = gars[name]
  takes_f = name in ("trmean", "phocas", "meamed")
  def unchecked(gradients, f=None, **kwargs):
    return engine.coordinate_many(name, gradients, f if takes_f else None)
  unchecked.__name__ = narrow.unchecked.__name__
  return make_gar(unchecked, narrow.check, upper_bound=narrow.upper_bound, influence=narrow.influence, name=name)

many_gars = {name: _many(name) for name in ("average", "median", "trmean", "phocas", "meamed")}

# ---------------------------------------------------------------------------- #
# Multi-Krum, Bulyan, Aksel and CGE for up to 1024 gradients

def _many_distance(name):
  """ The `many_distance_gars` entry of `name`: the check, bound and influence of `gars[name]`; up to MAX_N_DISTANCE
  gradients the call of `wide_gars[name]`, above it `engine.distance_many` (`bz_distance_many`), which stores the
  selection for `influence` as `_wide` does. """
  narrow, wide = gars[name], wide_gars[name]
  def unchecked(gradients, f, m=None, mode="mid", **kwargs):
    if not isinstance(gradients, list) or len(gradients) <= _lib.MAX_N_DISTANCE:
      return wide.unchecked(gradients=gradients, f=f, m=m, mode=mode, **kwargs)
    out, order = engine.distance_many(name, gradients, f, m if name in ("krum", "bulyan") else None,
                                      mode if name == "aksel" else "mid")
    if name != "bulyan":
      _last.store(name, (f,) if name == "krum" else (), gradients, order)
    return out
  unchecked.__name__ = narrow.unchecked.__name__
  influence = None
  if narrow.influence is not None:
    def influence(honests, attacks, f, m=None, mode="mid", **kwargs):
      gradients = honests + attacks
      if len(gradients) > _lib.MAX_N and _last.lookup(name, (f,) if name == "krum" else (), gradients) is None:
        unchecked(gradients=gradients, f=f, m=m, mode=mode)
      return narrow.influence(honests, attacks, f=f, m=m, mode=mode, **kwargs)
  return make_gar(unchecked, narrow.check, upper_bound=narrow.upper_bound, influence=influence, name=name)

many_distance_gars = {name: _many_distance(name) for name in engine.WIDE_DISTANCE}
