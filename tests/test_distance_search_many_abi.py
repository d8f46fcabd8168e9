# coding: utf-8
"""`bz_distance_line_search_many` (include/byzagg_distance_search_many.h) and `bz_distance_many_select`
(include/byzagg_distance_many_table.h) on the CPU: the headers and their bindings, the seventh library's exports, the
argument checks (each fails before any CUDA call), the workspace sizes, the resources of K2-star-many, the sixth
library's kernel set, the Python limits and the plugin's routing."""

import ctypes
import pathlib
import re
import shutil
import subprocess
import types

import pytest

ROOT = pathlib.Path(__file__).resolve().parent.parent
INCLUDE = ROOT / "include"
SEARCH_HEADER = INCLUDE / "byzagg_distance_search_many.h"
TABLE_HEADER = INCLUDE / "byzagg_distance_many_table.h"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
SEARCH_SYMBOLS = ["bz_distance_line_search_many", "bz_distance_line_search_many_last_error",
                  "bz_distance_line_search_many_workspace_bytes"]
TABLE_SYMBOLS = ["bz_distance_many_select"]
KRUM, BULYAN, BRUTE, AKSEL, CGE = 5, 6, 7, 8, 9

def declared_symbols(header):
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", header.read_text())))

def test_headers_declare_exactly_their_symbols_and_no_other_header_includes_them():
  assert declared_symbols(SEARCH_HEADER) == SEARCH_SYMBOLS
  assert declared_symbols(TABLE_HEADER) == TABLE_SYMBOLS
  for header in INCLUDE.glob("*.h"):
    text = header.read_text()
    for own in (SEARCH_HEADER, TABLE_HEADER):
      if header != own:
        assert f"#include \"{own.name}\"" not in text, (header.name, own.name)
    if header in (SEARCH_HEADER, TABLE_HEADER):
      assert "byzagg_distance_many.h" not in text, header.name
  makefile = (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  assert re.search(r"^all: \$\(MANY_SEARCH_OUT\)$", makefile, re.M)
  assert re.search(r"#define BZ_DISTANCE_MANY_TABLE_OFFSET (\d+)", TABLE_HEADER.read_text()).group(1) == "12544"

def _libraries(_lib):
  return {"libbyzagg": _lib.library_path(), "peers": _lib.peers_library_path(), "star": _lib.star_library_path(),
          "many": _lib.many_library_path(), "many_tools": _lib.many_tools_library_path(),
          "many_distance": _lib.many_distance_library_path(), "many_search": _lib.many_search_library_path()}

@pytest.mark.skipif(shutil.which("nm") is None, reason="nm not available")
def test_the_exports_live_in_their_library_only_and_the_bindings_match():
  from byzantinemomentum_b200 import _lib
  paths = _libraries(_lib)
  for owner, symbols in (("many_search", SEARCH_SYMBOLS), ("many_distance", TABLE_SYMBOLS)):
    for key, path in paths.items():
      # the dynamic symbols the library defines itself (dlsym would also find those of the libraries it links against)
      defined = set(subprocess.run(["nm", "-D", "--defined-only", str(path)], capture_output=True, text=True,
                                   check=True).stdout.split())
      assert all((name in defined) == (key == owner) for name in symbols), (key, symbols)
  assert _lib.many_search_library_path().parent == _lib.library_path().parent
  assert sorted(_lib.MANY_SEARCH_SIGNATURES) == SEARCH_SYMBOLS
  assert sorted(_lib.MANY_DISTANCE_TABLE_SIGNATURES) == TABLE_SYMBOLS
  assert sorted(_lib.MANY_DISTANCE_SIGNATURES) == ["bz_distance_many", "bz_distance_many_last_error",
                                                   "bz_distance_many_workspace_bytes"]
  assert _lib.MANY_SEARCH_SIGNATURES["bz_distance_line_search_many"] == _lib.DISTANCE_SEARCH_SIGNATURES["bz_distance_line_search"]
  assert (_lib.MANY_SEARCH_SIGNATURES["bz_distance_line_search_many_workspace_bytes"]
          == _lib.DISTANCE_SEARCH_SIGNATURES["bz_distance_line_search_workspace_bytes"])
  search = _lib.many_search_lib()
  for name, (restype, argtypes) in _lib.MANY_SEARCH_SIGNATURES.items():
    assert getattr(search, name).argtypes == argtypes and getattr(search, name).restype == restype, name
  table = _lib.many_distance_lib()
  assert table.bz_distance_many_select.argtypes == _lib.MANY_DISTANCE_TABLE_SIGNATURES["bz_distance_many_select"][1]

def test_library_path_override(monkeypatch):
  from byzantinemomentum_b200 import _lib
  monkeypatch.setenv("BYZAGG_MANY_SEARCH_LIBRARY", "/somewhere/else.so")
  assert str(_lib.many_search_library_path()) == "/somewhere/else.so"

def _fake_rows(n, address=0x100000):
  return (ctypes.c_void_p * n)(*[address + 0x10000 * i for i in range(n)])

def test_bad_arguments_fail_before_touching_the_gpu():
  """ Only invalid calls here (each fails before any CUDA call): the pointers are fake addresses. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.many_search_lib()
  main = _lib.lib()
  message = lambda: lib.bz_distance_line_search_many_last_error().decode()
  avg, att, byz, out = (ctypes.c_void_p(0x80000000 + 0x1000000 * k) for k in range(4))
  trace, status, ws = ctypes.c_void_p(0x90000000), ctypes.c_void_p(0x91000000), ctypes.c_void_p(0xa0000000)
  big = 1 << 40
  def call(rule, nh, f_real, f_decl=1, honest=None, kind=0, d=64, evals=4, b=byz, o=out, space=ws, ws_bytes=big):
    table = _fake_rows(max(nh, 1)) if honest is None else honest
    return lib.bz_distance_line_search_many(rule, table, nh, f_real, f_decl, kind, 0, avg, att, d, evals, b, o, trace, status,
                                            space, ws_bytes, None)
  # the rules
  for rule in range(5):
    assert call(rule, 200, 20) == -1 and "coordinate-wise" in message() and "bz_line_search_many" in message(), rule
  assert call(10, 200, 20) == -1 and "unknown rule" in message()
  assert call(BRUTE, 60, 5) == -2 and "brute" in message()
  for rule in (KRUM, BULYAN, AKSEL, CGE):
    assert call(rule, 1000, 25) == -2 and "BZ_MAX_N_MANY = 1024" in message(), rule
  # the counts and f
  assert call(KRUM, 0, 5) == -1 and "nh = 0" in message()
  assert call(KRUM, 200, 0) == -1 and "f_real = 0" in message()
  assert call(BULYAN, 280, 20, f_decl=75) == -1 and "4f + 3" in message()
  assert call(KRUM, 280, 20, f_decl=298) == -1 and "bz_distance_line_search_many" in message()
  # the vectors and the rows
  assert call(KRUM, 200, 20, d=0) == -1 and "d = 0" in message()
  assert call(KRUM, 200, 20, evals=0) == -1 and "evals" in message()
  assert call(KRUM, 200, 20, kind=2) == -1 and "kind" in message()
  assert call(KRUM, 200, 20, honest=ctypes.cast(None, ctypes.POINTER(ctypes.c_void_p))) == -1 and "honest is NULL" in message()
  assert call(KRUM, 200, 20, b=None) == -1 and "NULL" in message()
  assert call(KRUM, 200, 20, o=ctypes.c_void_p(0x83000002)) == -1 and "4-byte aligned" in message()
  assert call(KRUM, 200, 20, b=avg) == -1 and "distinct" in message()
  with_null = _fake_rows(200)
  with_null[150] = None
  assert call(KRUM, 200, 20, honest=with_null) == -1 and "honest[150] is NULL" in message()
  assert call(KRUM, 200, 20, honest=_fake_rows(200, address=0x100002)) == -1 and "4-byte aligned" in message()
  aliased = _fake_rows(200)
  aliased[7] = byz.value
  assert call(KRUM, 200, 20, honest=aliased) == -1 and "honest[7] is byz or out" in message()
  overlap = _fake_rows(200)
  assert call(KRUM, 200, 20, o=ctypes.c_void_p(overlap[9] + 8)) == -1 and "overlaps honest[9]" in message()
  # the workspace
  for rule in (KRUM, BULYAN, AKSEL, CGE):
    for nh, f_real in ((120, 9), (280, 20), (1000, 24)):
      need = lib.bz_distance_line_search_many_workspace_bytes(nh + f_real)
      assert call(rule, nh, f_real, ws_bytes=need - 1) == -4 and "workspace" in message(), (rule, nh)
    assert call(rule, 280, 20, space=ctypes.c_void_p(0xa0000004)) == -4 and "misaligned" in message()
  # up to 128 rows the call is bz_distance_line_search's, whose message comes through
  assert call(KRUM, 100, 20, ws_bytes=64) == -4 and "bz_distance_line_search" in message()
  # the sizes: bz_distance_line_search's up to 128 rows, above a size that grows with n
  for n in (1, 64, 65, 128):
    assert lib.bz_distance_line_search_many_workspace_bytes(n) == main.bz_distance_line_search_workspace_bytes(n)
  sizes = [lib.bz_distance_line_search_many_workspace_bytes(n) for n in (128, 129, 200, 512, 1000, 1024)]
  assert sizes == sorted(sizes) and all(s % 256 == 0 for s in sizes)
  assert lib.bz_distance_line_search_many_workspace_bytes(1024) >= _lib.many_distance_lib().bz_distance_many_workspace_bytes(1024)
  with pytest.raises(ValueError, match="bz_distance_line_search_many.*coordinate-wise"):
    call(1, 200, 20)
    _lib.check(-1, "bz_distance_line_search_many")

def test_select_rejects_bad_arguments_before_touching_the_gpu():
  from byzantinemomentum_b200 import _lib
  lib = _lib.many_distance_lib()
  message = lambda: lib.bz_distance_many_last_error().decode()
  out, ws = ctypes.c_void_p(0x90000000), ctypes.c_void_p(0xa0000000)
  need = lib.bz_distance_many_workspace_bytes(300)
  def call(rule, n, f=10, m=1, space=ws, ws_bytes=need):
    return lib.bz_distance_many_select(rule, _fake_rows(n), n, f, m, 64, out, None, None, space, ws_bytes, None)
  for rule in (AKSEL, CGE, BRUTE, 1):
    assert call(rule, 300) == -1 and "BZ_RULE_KRUM or BZ_RULE_BULYAN" in message(), rule
  assert call(KRUM, 100) == -2 and "BZ_MAX_N_DISTANCE" in message()
  assert call(KRUM, 1025) == -2 and "BZ_MAX_N_MANY" in message()
  assert call(BULYAN, 300, f=75) == -1 and "4f + 3" in message()
  assert call(KRUM, 300, m=301) == -1 and "m = 301" in message()
  assert call(KRUM, 300, ws_bytes=need - 1) == -4 and "bz_distance_many_select" in message()
  assert call(KRUM, 300, space=ctypes.c_void_p(0xa0000004)) == -4
  with pytest.raises(ValueError, match="bz_distance_many_select"):
    call(CGE, 300)
    _lib.check(-1, "bz_distance_many_select")

def _usage(path):
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(path)], capture_output=True, text=True, timeout=600).stdout
  return {name: (int(regs), int(stack)) for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text)}

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_the_star_kernel_lives_in_the_seventh_library_only_without_stack_spills_or_wide_global_access():
  from byzantinemomentum_b200 import _lib
  paths = _libraries(_lib)
  usage = _usage(paths["many_search"])
  assert any("k2_star_many" in name for name in usage) and any("k2_starfold_many" in name for name in usage), sorted(usage)
  assert all("k2_star" in name for name in usage), sorted(usage)
  for name, (regs, stack) in usage.items():
    assert regs <= 255 and stack == 0, (name, regs, stack)
  sass = subprocess.run([CUOBJDUMP, "-sass", str(paths["many_search"])], capture_output=True, text=True, timeout=600).stdout
  for block in re.split(r"\n\s*Function : ", sass)[1:]:
    name = block.split("\n", 1)[0]
    assert "STL" not in block and "LDL" not in block, name
    assert not re.search(r"\b(STG|LDG)\.E[.\w]*\.128\b", block), name
  for key, path in paths.items():
    if key != "many_search":
      assert not any("k2_star" in name for name in _usage(path)), key

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_the_sixth_library_keeps_its_13_kernels():
  from byzantinemomentum_b200 import _lib
  assert len(_usage(_lib.many_distance_library_path())) == 13

def test_the_python_limits_and_messages():
  torch = pytest.importorskip("torch")
  from byzantinemomentum_b200 import engine, sharded
  rows = [torch.zeros(4)] * 1025
  for gar in ("median", "trmean", "brute"):
    with pytest.raises(ValueError, match="many_distance=True takes the distance rules"):
      engine.LineSearch(gar, rows[:10], 2, 1, rows[0], rows[0], 4, many_distance=True)
  with pytest.raises(ValueError, match="coordinate-wise"):
    engine.LineSearch("krum", rows[:10], 2, 1, rows[0], rows[0], 4, many=True)
  with pytest.raises(ValueError, match="maximum of 1024"):
    engine.LineSearch("krum", rows, 2, 1, rows[0], rows[0], 4, many_distance=True)
  with pytest.raises(ValueError, match="maximum of 128"):
    engine.LineSearch("krum", rows[:129], 2, 1, rows[0], rows[0], 4)
  for gar in ("krum", "bulyan", "aksel", "cge"):
    assert sharded.search_rows(gar, many=True) == 64

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

def test_the_plugin_routes_many_distance_searches(monkeypatch):
  torch = pytest.importorskip("torch")
  from byzantinemomentum_b200 import plugin
  aggregators = _registry()
  plugin.install(aggregators, prefix="md-", many_distance=True, many=True)
  plugin.install(aggregators)
  monkeypatch.setattr(plugin, "_is_cuda", lambda tensors: True)          # CPU rows stand for CUDA rows
  for name in ("krum", "bulyan", "aksel", "cge"):
    assert plugin._installed[aggregators.gars["md-" + name]] == (name, 128)
    assert aggregators.gars["md-" + name] in plugin._many_distance_installed
    assert aggregators.gars["b200-" + name] not in plugin._many_distance_installed
  assert aggregators.gars["md-median"] not in plugin._many_distance_installed
  calls = []
  class Backend:
    @staticmethod
    def line_search(*args, **kwargs):
      calls.append((args[0], len(args[1]) + args[2], kwargs))
      return 0., args[1][0]
  rows = [torch.ones(8) for _ in range(1024)]
  default, md, both = _attacks(), _attacks(), _attacks()
  plugin.install_attacks(default, backend=Backend)
  plugin.install_attacks(md, backend=Backend, many_distance=True)
  plugin.install_attacks(both, backend=Backend, many=True, many_distance=True)
  def run(attacks, name, gar, nh, f_real=20, prefix="md-", **kw):
    return attacks.attacks[name].unchecked(grad_honests=rows[:nh], f_real=f_real, f_decl=5,
                                           defense=aggregators.gars[prefix + gar], model=None, **kw)
  # many_distance above 128 rows
  assert run(md, "empire", "krum", 280, factor=-4)[0] is rows[0]
  assert calls[-1] == ("krum", 300, dict(negative=False, kind="identical", many_distance=True))
  assert run(md, "empire-strict", "cge", 1000, f_real=24, epsilon=-4)[0] is rows[0]
  assert calls[-1] == ("cge", 1024, dict(kind="empire-strict", many_distance=True))
  assert run(md, "little", "krum", 1000, f_real=25, factor=-4) == "stock"      # 1025 rows
  assert run(md, "little", "median", 280, factor=-4) == "stock"                # a many entry needs many=True
  assert run(md, "little", "krum", 280, prefix="b200-", factor=-4) == "stock"  # a default entry keeps 64
  # the default route unchanged
  count = len(calls)
  assert run(default, "empire", "krum", 280, factor=-4) == "stock" and len(calls) == count
  assert run(default, "little", "krum", 100, factor=-4)[0] is rows[0]         # 120 rows against a 128-row entry
  assert calls[-1] == ("krum", 120, dict(negative=False, kind="identical"))
  assert run(md, "little", "krum", 100, factor=-4)[0] is rows[0]
  assert calls[-1] == ("krum", 120, dict(negative=False, kind="identical"))
  # many and many_distance combine; median's many=True call is unchanged
  assert run(both, "empire", "median", 280, factor=-4)[0] is rows[0]
  assert calls[-1] == ("median", 300, dict(negative=False, kind="identical", many=True))
  assert run(both, "empire", "bulyan", 280, factor=-4)[0] is rows[0]
  assert calls[-1] == ("bulyan", 300, dict(negative=False, kind="identical", many_distance=True))
