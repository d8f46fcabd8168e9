# coding: utf-8
"""`bz_distance_many` (include/byzagg_distance_many.h), Multi-Krum, Bulyan, Aksel and CGE for up to 1024 rows, on the
CPU: the header and its binding, the sixth library's exports, the argument checks (each fails before any CUDA call),
the register budget of its kernels, and the row limits of the Python layers."""

import ctypes
import pathlib
import re
import shutil
import subprocess
import types

import numpy as np
import pytest

from conftest import Golden, canon_alias
import parity
from oracle import byzoracle as orc

ROOT = pathlib.Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "byzagg_distance_many.h"
MD_DIR = ROOT / "tests" / "golden" / "many_distance"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
SYMBOLS = ["bz_distance_many", "bz_distance_many_last_error", "bz_distance_many_workspace_bytes"]
KRUM, BULYAN, BRUTE, AKSEL, CGE = 5, 6, 7, 8, 9

def md_calls():
  out = []
  for path in sorted(MD_DIR.glob("golden_md_*.npz")):
    g = Golden(path)
    for call in g.calls:
      out.append(pytest.param(g, call, id=f"{g.name}:{call['tag']}"))
  return out

def declared_symbols():
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", HEADER.read_text())))

def other_libraries(_lib):
  return (_lib.library_path(), _lib.peers_library_path(), _lib.star_library_path(), _lib.many_library_path(),
          _lib.many_tools_library_path())

def test_header_declares_the_three_symbols_and_stays_out_of_the_other_headers():
  assert declared_symbols() == SYMBOLS
  for header in (ROOT / "include").glob("*.h"):
    if header != HEADER:
      assert "byzagg_distance_many.h" not in header.read_text(), header.name
  makefile = (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  assert "byzagg_distance_many.h" in makefile and re.search(r"^all: \$\(MANY_DISTANCE_OUT\)$", makefile, re.M)

def test_the_sixth_library_exports_the_symbols_and_no_other_library_does():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.many_distance_library_path()))
  for name in SYMBOLS:
    assert hasattr(handle, name), name
  for path in other_libraries(_lib):
    other = ctypes.CDLL(str(path))
    assert not any(hasattr(other, name) for name in SYMBOLS), path.name
  assert _lib.many_distance_library_path().parent == _lib.library_path().parent
  assert sorted(_lib.MANY_DISTANCE_SIGNATURES) == SYMBOLS
  lib = _lib.many_distance_lib()
  for name, (restype, argtypes) in _lib.MANY_DISTANCE_SIGNATURES.items():
    assert getattr(lib, name).argtypes == argtypes and getattr(lib, name).restype == restype, name
  assert _lib.MANY_DISTANCE_SIGNATURES["bz_distance_many"] == _lib.DISTANCE_SIGNATURES["bz_distance"]
  assert _lib.MANY_DISTANCE_SIGNATURES["bz_distance_many_workspace_bytes"] == _lib.DISTANCE_SIGNATURES["bz_distance_workspace_bytes"]

def test_library_path_override(monkeypatch):
  from byzantinemomentum_b200 import _lib
  monkeypatch.setenv("BYZAGG_MANY_DISTANCE_LIBRARY", "/somewhere/else.so")
  assert str(_lib.many_distance_library_path()) == "/somewhere/else.so"

def test_bad_arguments_fail_before_touching_the_gpu():
  """ Only invalid calls here (each fails before any CUDA call): the pointers are fake addresses. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.many_distance_lib()
  main = _lib.lib()
  message = lambda: lib.bz_distance_many_last_error().decode()
  rows = lambda n, address=0x100000: (ctypes.c_void_p * n)(*[address + 0x1000 * i for i in range(n)])
  out, ws = ctypes.c_void_p(0x90000000), ctypes.c_void_p(0xa0000000)
  big = 1 << 40
  def call(rule, n, f=0, m=1, mode=0, d=16, table=None, dest=out, ws_bytes=big, space=ws):
    return lib.bz_distance_many(rule, rows(max(n, 1)) if table is None else table, n, f, m, mode, d, dest, None, None,
                                space, ws_bytes, None)
  # the row count and the rule
  assert call(KRUM, 0) == -1 and "n = 0" in message()
  for rule in (KRUM, BULYAN, AKSEL, CGE):
    assert call(rule, 1025) == -2 and "BZ_MAX_N_MANY = 1024" in message(), rule
  assert call(BRUTE, 65) == -2 and "brute" in message()
  assert call(4, 300) == -1 and "unknown rule" in message()
  assert call(10, 300) == -1 and "unknown rule" in message()
  # f, m and mode above 128 rows: bz_distance's verdicts
  assert call(KRUM, 300, f=299) == -1 and "n - f - 1" in message()
  assert call(KRUM, 300, f=-1) == -1
  assert call(KRUM, 300, f=10, m=0) == -1 and "m = 0" in message()
  assert call(KRUM, 300, f=10, m=301) == -1 and "expected 1..300" in message()
  assert call(BULYAN, 300, f=75) == -1 and "4f + 3" in message()
  assert call(BULYAN, 300, f=74, m=225) == -1 and "expected 1..224" in message()
  assert call(AKSEL, 300, mode=2) == -1 and "mode = 2" in message()
  assert call(AKSEL, 300, f=300, mode=1) == -1 and "not executable" in message()
  # the rows, the output and the workspace
  assert call(KRUM, 300, f=10, table=rows(300, address=0x100002)) == -1 and "4-byte aligned" in message()
  with_null = rows(1024)
  with_null[1000] = None
  assert call(CGE, 1024, table=with_null) == -1 and "rows[1000] is NULL" in message()
  assert call(CGE, 300, dest=None) == -1 and "output" in message()
  overlap = rows(300)
  assert call(KRUM, 300, f=10, dest=ctypes.c_void_p(overlap[7] + 8)) == -1 and "overlaps rows[7]" in message()
  assert call(KRUM, 100, f=10, dest=ctypes.c_void_p(overlap[7] + 8)) == -1 and "overlaps rows[7]" in message()
  for rule in (KRUM, BULYAN, AKSEL, CGE):
    for n in (129, 300, 1024):
      assert call(rule, n, f=10, ws_bytes=64) == -4 and "workspace" in message(), (rule, n)
      need = lib.bz_distance_many_workspace_bytes(n)
      assert call(rule, n, f=10, ws_bytes=need - 1) == -4, (rule, n)
    assert call(rule, 300, f=10, space=ctypes.c_void_p(0xa0000004)) == -4 and "misaligned" in message()
  # up to 128 rows the call is bz_distance's, whose message comes through
  assert call(KRUM, 100, f=10, ws_bytes=64) == -4 and "bz_distance" in message()
  assert call(BRUTE, 64, f=70) == -1
  # d = 0 is a no-op once the arguments pass; a workspace at 8 mod 16 bytes passes (8-byte alignment is the contract)
  assert call(KRUM, 300, f=10, d=0) == 0 and call(CGE, 1024, d=0) == 0
  for rule in (KRUM, BULYAN, AKSEL, CGE):
    assert call(rule, 300, f=10, d=0, space=ctypes.c_void_p(0xa0000008)) == 0, rule
  # the sizes: bz_distance's up to 128 rows, above a size that grows with n and never falls below it
  for n in (1, 64, 65, 128):
    assert lib.bz_distance_many_workspace_bytes(n) == main.bz_distance_workspace_bytes(n)
  sizes = [lib.bz_distance_many_workspace_bytes(n) for n in (128, 129, 512, 1024)]
  assert sizes == sorted(sizes) and all(s % 256 == 0 for s in sizes)
  with pytest.raises(ValueError, match="bz_distance_many.*BZ_MAX_N_MANY = 1024"):
    call(KRUM, 2000)
    _lib.check(-2, "bz_distance_many")

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_the_new_kernels_fit_the_budget_and_live_in_the_sixth_library_only():
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.many_distance_library_path())], capture_output=True, text=True,
                        timeout=600).stdout
  usage = {name: (int(regs), int(stack)) for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text)}
  families = ("k2_pairdist_many", "k2_pairsum_many", "k2_rowkeys_many", "k5_select_many", "k3_average_many", "k4_bulyan_many")
  for family in families:
    assert any(family in name for name in usage), family
  assert all(any(family in name for family in families) for name in usage), sorted(usage)
  for name, (regs, stack) in usage.items():
    assert regs <= 255 and stack == 0, (name, regs, stack)
  sass = subprocess.run([CUOBJDUMP, "-sass", str(_lib.many_distance_library_path())], capture_output=True, text=True,
                        timeout=600).stdout
  for block in re.split(r"\n\s*Function : ", sass)[1:]:
    name = block.split("\n", 1)[0]
    assert "STL" not in block and "LDL" not in block, name
    # 16-byte global accesses only where K3's geometry found the rows and the output 16-byte aligned: the workspace
    # is only required to be 8-byte aligned
    if "k3_average_many" not in name:
      assert not re.search(r"\b(STG|LDG)\.E[.\w]*\.128\b", block), name
  for path in other_libraries(_lib):
    other = subprocess.run([CUOBJDUMP, "-res-usage", str(path)], capture_output=True, text=True, timeout=600).stdout
    assert not any(family in other for family in families), path.name

def test_the_row_limits_of_the_python_layers():
  torch = pytest.importorskip("torch")
  from byzantinemomentum_b200 import engine
  rows = [torch.zeros(4)] * 1025
  with pytest.raises(ValueError, match="maximum of 128"):
    engine.Plan("krum", rows[:129], f=1)
  with pytest.raises(ValueError, match="maximum of 1024"):
    engine.Plan("krum", rows, f=1, many=True)
  with pytest.raises(ValueError, match="maximum of 64"):
    engine.Plan("brute", rows[:129], f=1, many=True)
  with pytest.raises(ValueError, match="maximum of 1024"):
    engine.distance_many("cge", rows, 1)
  with pytest.raises(ValueError, match="maximum of 128"):
    engine.wide_distance("cge", rows[:129], 1)
  with pytest.raises(KeyError):
    engine.distance_many("brute", rows[:10], 1)

def test_many_distance_gars_carry_the_check_bound_and_influence_of_gars():
  import byzantinemomentum_b200 as bz
  assert sorted(bz.many_distance_gars) == ["aksel", "bulyan", "cge", "krum"]
  assert sorted(bz.wide_gars) == ["aksel", "bulyan", "cge", "krum"]
  assert sorted(bz.many_gars) == ["average", "meamed", "median", "phocas", "trmean"]
  for name, entry in bz.many_distance_gars.items():
    narrow = bz.gars[name]
    assert entry.check is narrow.check and entry.upper_bound is narrow.upper_bound, name
    assert (entry.influence is None) == (narrow.influence is None), name
    assert entry.unchecked.__name__ == narrow.unchecked.__name__
    assert entry is not bz.wide_gars[name]

def _registry():
  class Entry:
    def __init__(self, unchecked, check):
      self.unchecked, self.check = unchecked, check
  aggregators = types.SimpleNamespace(gars={})
  def register(name, unchecked, check, upper_bound=None, influence=None):
    aggregators.gars[name] = Entry(unchecked, check)
  aggregators.register = register
  return aggregators

def test_plugin_installs_the_many_distance_entries():
  pytest.importorskip("torch")
  from byzantinemomentum_b200 import plugin
  from byzantinemomentum_b200.gars import gars, many_gars, many_distance_gars
  aggregators = _registry()
  names = plugin.install(aggregators, prefix="md-", many_distance=True, many=True)
  assert sorted(names) == sorted("md-" + name for name in gars)
  for name in gars:
    want = many_distance_gars.get(name) or many_gars.get(name) or gars[name]
    entry = aggregators.gars["md-" + name]
    assert entry.unchecked is want.unchecked, name
  for name in many_distance_gars:
    assert plugin._installed[aggregators.gars["md-" + name]] == (name, 128), name
  assert plugin._installed[aggregators.gars["md-brute"]] == ("brute", 64)
  with pytest.raises(ValueError, match="wide"):
    plugin.install(_registry(), wide=True, many_distance=True)
  # without the new argument nothing changes
  plain = _registry()
  plugin.install(plain, prefix="p-")
  assert plain.gars["p-krum"].unchecked is gars["krum"].unchecked

def test_fixture_covers_the_stacks_and_is_small():
  names = sorted(p.name for p in MD_DIR.glob("golden_md_*.npz"))
  goldens = [Golden(MD_DIR / name) for name in names]
  assert sorted(g.n for g in goldens) == [129, 200, 256, 257, 511, 512, 777, 1024]
  assert {call["gar"] for g in goldens for call in g.calls} == {"krum", "bulyan", "aksel", "cge"}
  assert {g.manifest["kind"] for g in goldens} >= {"iid", "empire", "little", "nan", "inf", "quant", "tiny80", "nearmax"}
  assert any(g.nh == g.n for g in goldens)                          # one stack without an alias
  assert any("raises" in call for g in goldens for call in g.calls)   # the degenerate Bulyan
  assert sum((MD_DIR / name).stat().st_size for name in names) < 2.5 * 1024 * 1024

@pytest.mark.parametrize("g,call", md_calls())
def test_oracle_matches_the_reference_above_128_rows(g, call):
  """ The NumPy oracle against the reference's recorded calls at these n, as test_distance_wide_abi checks it up to
  128 rows: the selection (where recorded) and the output bit for bit, Bulyan within its closest-m bar. """
  gar, params, tag = call["gar"], call["params"], call["tag"]
  rows = [g.rows[i] for i in range(g.n)]
  if "raises" in call:
    assert gar == "bulyan"
    with pytest.raises(Exception):
      orc.bulyan(rows, **params)
    return
  ref = g.get(tag, "out")
  got, info = orc.GARS[gar](rows, return_info=True, **params)
  if gar == "bulyan":
    parity.assert_close_scaled(got, ref, parity.column_scale(info["stage1"]), tag, exempt=info["ambiguous"])
    parity.assert_in_hull(got, info["stage1"], info["ambiguous"], tag)
    return
  count = {"krum": params.get("m") or (g.n - params["f"] - 2), "cge": g.n - params["f"]}.get(gar, call.get("c"))
  if gar == "aksel" and np.isnan(g.get(tag, "dists")).any():     # NaN keys: the reference's order is undefined
    return
  assert canon_alias(info["order"][:count], g.nh) == canon_alias(g.get(tag, "order")[:count], g.nh), f"{tag}: selection differs"
  parity.assert_bit_exact(got, ref, tag)
