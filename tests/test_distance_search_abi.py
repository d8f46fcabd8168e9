# coding: utf-8
"""The line search against Multi-Krum, Bulyan, Aksel and CGE up to 128 rows on the CPU: the header
`include/byzagg_distance_search.h` and its ctypes table, the argument checks of `bz_distance_line_search` (before
any CUDA call, with host addresses), its workspace size, the checks and bounds of `gars.wide_gars`, and which attacks
`plugin.install_attacks` sends to the device search once `plugin.install(..., wide=True)` registered the rules (with
a stand-in search).  No compute calls here."""

import ctypes
import pathlib
import re
import types

import pytest

ROOT = pathlib.Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "byzagg_distance_search.h"
NAMES = ["bz_distance_line_search", "bz_distance_line_search_workspace_bytes"]
KRUM, BULYAN, BRUTE, AKSEL, CGE = 5, 6, 7, 8, 9

def declared(path):
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", path.read_text())))

def test_header_declares_the_calls_and_byzagg_h_leaves_them_out():
  assert declared(HEADER) == NAMES
  for other in (ROOT / "include").glob("byzagg*.h"):
    if other != HEADER:
      assert "byzagg_distance_search.h" not in other.read_text(), other.name
      assert not set(declared(other)) & set(NAMES), other.name
  makefile = (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  assert "../../include/byzagg_distance_search.h" in makefile and "api_distance_search.inc" in makefile

def test_library_exports_the_calls_and_the_table_is_its_own():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.library_path()))
  for name in NAMES:
    assert hasattr(handle, name), name
  assert sorted(_lib.DISTANCE_SEARCH_SIGNATURES) == NAMES
  others = [_lib.SIGNATURES, _lib.SHARD_SIGNATURES, _lib.ATTACK_SIGNATURES, _lib.SEARCH_SHARD_SIGNATURES,
            _lib.SEARCH_PEER_SIGNATURES, _lib.COORDINATE_SIGNATURES, _lib.PEER_NEXT_SIGNATURES, _lib.DISTANCE_SIGNATURES,
            _lib.DISTANCE_SHARD_SIGNATURES, _lib.ANTICGE_SIGNATURES, _lib.ANTICGE_PEER_SIGNATURES,
            _lib.DISTANCE_PEER_SIGNATURES]
  assert not set(_lib.DISTANCE_SEARCH_SIGNATURES) & set().union(*others)
  for name, (restype, argtypes) in _lib.DISTANCE_SEARCH_SIGNATURES.items():
    fn = getattr(_lib.lib(), name)
    assert fn.argtypes == argtypes and fn.restype == restype
  # the same arguments as bz_line_search
  assert _lib.DISTANCE_SEARCH_SIGNATURES["bz_distance_line_search"] == _lib.ATTACK_SIGNATURES["bz_line_search"]

def test_workspace_is_the_search_s_up_to_64_rows_and_bz_distance_s_plus_the_state_above():
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  for n in range(1, 65):
    assert lib.bz_distance_line_search_workspace_bytes(n) == lib.bz_line_search_workspace_bytes(n), n
  sizes = {lib.bz_distance_line_search_workspace_bytes(n) for n in range(65, 129)}
  assert len(sizes) == 1
  size = sizes.pop()
  assert size >= lib.bz_distance_workspace_bytes(128) + 64 and size % 256 == 0
  assert lib.bz_line_search_workspace_bytes(128) == lib.bz_line_search_workspace_bytes(64)

def test_search_rejects_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here: a valid one would launch on host memory. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  bufs = [(ctypes.c_float * 64)() for _ in range(5)]
  h, avg, att, byz, out = (ctypes.addressof(b) for b in bufs)
  trace = ctypes.addressof((ctypes.c_double * 64)())
  status = ctypes.addressof((ctypes.c_int32 * 2)())
  ws_buf = (ctypes.c_double * 8)()
  ws = ctypes.addressof(ws_buf)
  def call(rule=KRUM, honest=None, nh=90, f_real=10, f_decl=10, kind=0, avg=avg, att=att, d=64, evals=16, byz=byz,
           out=out, trace=trace, status=status, ws=ws + 4, ws_bytes=1 << 40):
    rows = (ctypes.c_void_p * max(nh, 1))(*([h] * max(nh, 1))) if honest is None else honest
    return lib.bz_distance_line_search(rule, rows, nh, f_real, f_decl, kind, 0, avg, att, d, evals, byz, out, trace,
                                       status, ws, ws_bytes, None)
  def err():
    return lib.bz_last_error().decode()
  assert lib.bz_distance_line_search(KRUM, None, 90, 10, 10, 0, 0, avg, att, 64, 16, byz, out, trace, status, ws, 1 << 40,
                                     None) == -1
  assert "honest is NULL" in err()
  for rule in range(5):                                   # the coordinate-wise rules go through bz_line_search
    assert call(rule=rule) == -1 and "coordinate-wise" in err() and "bz_line_search" in err(), rule
  assert call(rule=10) == -1 and "unknown rule" in err()
  assert call(rule=-1) == -1 and "unknown rule" in err()
  assert call(nh=0) == -1 and call(f_real=0) == -1 and "f_real" in err()
  for rule in (KRUM, BULYAN, AKSEL, CGE):
    assert call(rule=rule, nh=120, f_real=9, f_decl=9) == -2 and "BZ_MAX_N_DISTANCE = 128" in err(), rule
  assert call(rule=BRUTE, nh=60, f_real=5, f_decl=5) == -2 and "brute" in err() and "64" in err()
  assert call(d=0) == -1 and "d = 0" in err()
  assert call(evals=0) == -1 and "evals" in err()
  assert call(kind=2) == -1 and "kind" in err()
  for what in ("avg", "byz", "out", "trace", "status"):
    assert call(**{what: None}) == -1 and "NULL" in err(), what
  assert call(att=None) == -1
  assert call(byz=avg) == -1 and "distinct" in err()
  assert call(out=byz) == -1 and "distinct" in err()
  assert call(avg=avg + 2) == -1 and "aligned" in err()
  for bad in (byz, out):
    assert call(honest=(ctypes.c_void_p * 90)(*([h] * 89 + [bad]))) == -1 and "honest[89] is byz or out" in err()
  assert call(honest=(ctypes.c_void_p * 90)(*([h] * 70 + [None] + [h] * 19))) == -1 and "rows[70] is NULL" in err()
  assert call(honest=(ctypes.c_void_p * 90)(*([h] * 70 + [h + 2] + [h] * 19))) == -1 and "rows[70]" in err()
  # the rule's own checks, with f = f_decl and the attack's defaults
  assert call(f_decl=99) == -1 and "f = 99" in err()
  assert call(rule=BULYAN, f_decl=25) == -1 and "4f + 3" in err()
  assert call(rule=BRUTE, nh=40, f_real=10, f_decl=20) == -2 and "subsets" in err()
  # the workspace, checked last
  need = lib.bz_distance_line_search_workspace_bytes(100)
  for rule in (KRUM, BULYAN, AKSEL, CGE):
    assert call(rule=rule, ws=ws, ws_bytes=need - 1) == -4 and "workspace" in err() and str(need) in err(), rule
  assert call(ws=ws + 4) == -4 and call(ws=None) == -4
  small = lib.bz_distance_line_search_workspace_bytes(25)
  assert small == lib.bz_line_search_workspace_bytes(25)
  assert call(nh=20, f_real=5, f_decl=5, ws=ws, ws_bytes=small - 1) == -4 and str(small) in err()
  assert call(kind=1, att=None, ws=ws, ws_bytes=need - 1) == -4     # empire-strict reads no direction

# ---- gars.wide_gars ------------------------------------------------------------------------------------------------

def test_wide_gars_mirror_the_checks_and_bounds_of_gars():
  torch = pytest.importorskip("torch")
  import byzantinemomentum_b200 as bz
  assert sorted(bz.wide_gars) == ["aksel", "bulyan", "cge", "krum"]
  assert len(bz.gars) == 10 and all(bz.wide_gars[name] is not bz.gars[name] for name in bz.wide_gars)
  rows = [torch.zeros(3) for _ in range(128)]
  for name, rule in bz.wide_gars.items():
    narrow = bz.gars[name]
    assert rule.check is narrow.check and rule.upper_bound is narrow.upper_bound, name
    assert (rule.influence is None) == (narrow.influence is None), name
    assert rule.unchecked is not narrow.unchecked and rule.checked is not narrow.checked, name
    for n in (1, 7, 25, 64, 65, 100, 128):
      for f in (-1, 0, 1, 5, 10, 31, 32, 60):
        for extra in ({}, {"m": 3}, {"m": 0}, {"mode": "n-f"}, {"mode": "bad"}):
          assert rule.check(gradients=rows[:n], f=f, **extra) == narrow.check(gradients=rows[:n], f=f, **extra), (name, n, f)
  assert bz.wide_gars["krum"].check(gradients=rows[:100], f=10) is None
  assert bz.wide_gars["bulyan"].check(gradients=rows[:128], f=31) is None
  assert bz.wide_gars["bulyan"].check(gradients=rows[:128], f=32) is not None
  assert bz.wide_gars["krum"].upper_bound(100, 10, 1000) == bz.gars["krum"].upper_bound(100, 10, 1000)

# ---- the plugin with wide entries ---------------------------------------------------------------------------------

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
  return ns

def _attacks():
  ns = types.SimpleNamespace(attacks={})
  def register(name, unchecked, check):
    if name in ns.attacks:
      raise KeyError(name)
    def checked(f_real, **kwargs):
      message = check(f_real=f_real, **kwargs)
      if message is not None:
        raise RuntimeError(message)
      return unchecked(f_real=f_real, **kwargs)
    checked.check, checked.checked, checked.unchecked = check, checked, unchecked
    ns.attacks[name] = checked
  ns.register = register
  for name in ("little", "empire", "bulyan", "empire-strict"):
    register(name, (lambda name: lambda **kw: ("stock", name))(name), lambda **kw: None)
  return ns

class SearchStandIn:
  """ Records the calls; returns a fixed factor and its Byzantine gradient. """
  def __init__(self):
    self.calls = []
  def line_search(self, gar, grad_honests, f_real, f_decl, grad_avg, grad_att, evals, negative=False, kind="identical"):
    self.calls.append(dict(gar=gar, nh=len(grad_honests), f_real=f_real, f_decl=f_decl, evals=evals, kind=kind))
    return 3., grad_avg.mul(-3.) if grad_att is None else grad_avg + 3. * grad_att

@pytest.fixture
def plugin_setup(monkeypatch):
  torch = pytest.importorskip("torch")
  from byzantinemomentum_b200 import plugin
  monkeypatch.setattr(plugin, "_installed", {})
  monkeypatch.setattr(plugin, "_is_cuda", lambda tensors: all(t.device.type == "cpu" for t in tensors))   # CPU rows stand for CUDA rows
  gen = torch.Generator().manual_seed(5)
  honest = [torch.randn(17, generator=gen) for _ in range(120)]
  return plugin, honest

def test_wide_install_registers_the_four_wide_entries_and_keeps_the_other_six(plugin_setup):
  import byzantinemomentum_b200 as bz
  plugin, _ = plugin_setup
  wide, default = _aggregators(), _aggregators()
  assert plugin.install(wide, wide=True) == plugin.install(default) == ["b200-" + name for name in bz.gars]
  for name in bz.gars:
    expected = bz.wide_gars.get(name, bz.gars[name])
    assert wide.gars["b200-" + name].unchecked is expected.unchecked, name
    assert default.gars["b200-" + name].unchecked is bz.gars[name].unchecked, name
    limit = 128 if name in bz.wide_gars or name in ("average", "median", "trmean", "phocas", "meamed") else 64
    assert plugin._installed[wide.gars["b200-" + name]] == (name, limit), name
    assert plugin._installed[default.gars["b200-" + name]] == (name, 64 if name in bz.wide_gars or name == "brute" else 128)
  over = _aggregators()
  assert plugin.install(over, override=True, names=["krum", "median"], wide=True) == ["krum", "median"]
  assert over.gars["krum"].unchecked is bz.wide_gars["krum"].unchecked and over.krum is over.gars["krum"]
  assert plugin._installed[over.gars["krum"]] == ("krum", 128)

@pytest.mark.parametrize("gar", ["krum", "cge"])
def test_attacks_against_a_wide_entry_run_the_device_search_up_to_128_rows(plugin_setup, gar):
  plugin, honest = plugin_setup
  wide, default, attacks, backend = _aggregators(), _aggregators(), _attacks(), SearchStandIn()
  plugin.install(wide, wide=True, names=[gar])
  plugin.install(default, names=[gar])
  plugin.install_attacks(attacks, backend=backend)
  def run(name, defense, nh, f_real=10, **kwargs):
    return attacks.attacks[name].checked(grad_honests=honest[:nh], f_real=f_real, f_decl=f_real, defense=defense,
                                         model=None, **kwargs)
  got = run("empire", wide.gars["b200-" + gar], 90, factor=-16)
  assert len(got) == 10 and all(g is got[0] for g in got)
  assert backend.calls[-1] == dict(gar=gar, nh=90, f_real=10, f_decl=10, evals=16, kind="identical")
  run("little", wide.gars["b200-" + gar], 118, f_real=10, factor=-4)
  assert backend.calls[-1]["nh"] == 118 and backend.calls[-1]["evals"] == 4
  run("empire-strict", wide.gars["b200-" + gar], 100, f_real=28, epsilon=-2)
  assert backend.calls[-1]["kind"] == "empire-strict" and backend.calls[-1]["nh"] == 100
  calls = len(backend.calls)
  # past 128 rows, against the default entry above 64 rows, and a positive factor: the stock attack
  assert run("empire", wide.gars["b200-" + gar], 119, factor=-16) == ("stock", "empire")
  assert run("empire", default.gars["b200-" + gar], 90, factor=-16) == ("stock", "empire")
  assert run("empire", wide.gars["b200-" + gar], 90, factor=2) == ("stock", "empire")
  assert len(backend.calls) == calls
  # at 64 rows and below both entries run the device search
  run("empire", default.gars["b200-" + gar], 54, factor=-16)
  run("empire", wide.gars["b200-" + gar], 54, factor=-16)
  assert len(backend.calls) == calls + 2
