# coding: utf-8
"""`bz_coordinate_many` (include/byzagg_coordinate_many.h), the coordinate-wise rules for up to 1024 rows,
on the CPU: the header and its binding, the argument checks (before any CUDA call), the limits that stay
where they were, the register budget of the new kernels, and the NumPy oracle against the reference's
recorded outputs at n = 129..1024 (`tests/golden/many/`).  No compute calls here."""

import ctypes
import pathlib
import re
import shutil
import subprocess

import pytest

from conftest import Golden
import parity
from oracle import byzoracle as orc
from test_coordinate_abi import closest_rtol

ROOT = pathlib.Path(__file__).resolve().parent.parent
MANY_DIR = ROOT / "tests" / "golden" / "many"
HEADER = ROOT / "include" / "byzagg_coordinate_many.h"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
MANY_NS = [129, 200, 256, 257, 511, 512, 777, 1024]

def declared_symbols():
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", HEADER.read_text())))

def many_calls():
  out = []
  for path in sorted(MANY_DIR.glob("golden_many_*.npz")):
    g = Golden(path)
    for call in g.calls:
      out.append(pytest.param(g, call, id=f"{g.name}:{call['tag']}"))
  return out

def test_header_declares_bz_coordinate_many_and_byzagg_h_includes_it():
  assert declared_symbols() == ["bz_coordinate_many", "bz_coordinate_many_last_error"]
  assert re.search(r"#define BZ_MAX_N_MANY 1024\b", HEADER.read_text())
  byzagg = (ROOT / "include" / "byzagg.h").read_text()
  includes = re.findall(r'#include "(byzagg_\w+\.h)"', byzagg)
  assert includes.count("byzagg_coordinate_many.h") == 1
  assert includes.index("byzagg_coordinate_many.h") == includes.index("byzagg_coordinate.h") + 1
  assert "byzagg_coordinate_many.h" in (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()

def test_the_fourth_library_exports_bz_coordinate_many_and_libbyzagg_does_not():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.many_library_path()))
  for name in declared_symbols():
    assert hasattr(handle, name), name
  main = ctypes.CDLL(str(_lib.library_path()))
  assert not any(hasattr(main, name) for name in declared_symbols())
  assert _lib.many_library_path().parent == _lib.library_path().parent
  assert sorted(_lib.COORDINATE_MANY_SIGNATURES) == declared_symbols()
  assert not set(_lib.COORDINATE_MANY_SIGNATURES) & (set(_lib.SIGNATURES) | set(_lib.COORDINATE_SIGNATURES))
  fn = _lib.many_lib().bz_coordinate_many
  assert fn.argtypes == _lib.COORDINATE_MANY_SIGNATURES["bz_coordinate_many"][1]
  assert fn.argtypes == _lib.COORDINATE_SIGNATURES["bz_coordinate"][1]
  assert _lib.MAX_N_MANY == 1024 and _lib.MAX_N_COORDINATE == 128 and _lib.lib().bz_max_n() == _lib.MAX_N == 64

def test_bz_coordinate_many_rejects_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here (and d = 0, which launches nothing): the pointers are fake addresses. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.many_lib()
  rows = lambda n, address=0x1000: (ctypes.c_void_p * n)(*[address + 0x100 * i for i in range(n)])
  out = ctypes.c_void_p(0x900000)
  def call(rule=2, table=None, n=300, f=10, d=16, dest=out):
    return lib.bz_coordinate_many(rule, rows(max(n, 1)) if table is None else table, n, f, d, dest, None)
  def message():
    return lib.bz_coordinate_many_last_error().decode()
  assert call(n=0) == -1 and "n = 0" in message()
  assert call(n=1025, f=1) == -2 and "BZ_MAX_N_MANY = 1024" in message() and "bz_coordinate_many" in message()
  for rule in (-1, 5):
    assert call(rule=rule) == -1 and "unknown rule" in message()
  assert call(f=150) == -1 and "n - 2f" in message()
  assert call(n=1024, f=512) == -1 and "n - 2f" in message()
  assert call(f=-1) == -1
  assert lib.bz_coordinate_many(1, None, 300, 0, 16, out, None) == -1 and "rows is NULL" in message()
  assert call(dest=None) == -1 and "output" in message()
  assert call(table=rows(300, address=0x1002)) == -1 and "aligned" in message()
  with_null = rows(1024)
  with_null[700] = None
  assert call(table=with_null, n=1024) == -1 and "rows[700] is NULL" in message()
  assert call(dest=ctypes.c_void_p(0x900002)) == -1 and "aligned" in message()
  # f is not checked for average and median; d = 0 is a no-op for every rule
  assert call(rule=0, f=999, d=0) == 0 and call(rule=1, f=-5, d=0) == 0
  for rule in range(5):
    assert call(rule=rule, n=1024, f=511, d=0, dest=None) == 0
    assert call(rule=rule, n=129, f=64, d=0, dest=None) == 0
  # the message reaches Python from this library
  assert call(n=2000) == -2
  with pytest.raises(ValueError, match="bz_coordinate_many.*BZ_MAX_N_MANY = 1024"):
    _lib.check(-2, "bz_coordinate_many")

def test_bz_coordinate_keeps_its_128_row_limit():
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  table = (ctypes.c_void_p * 129)(*[0x1000 + 0x100 * i for i in range(129)])
  assert lib.bz_coordinate(1, table, 129, 0, 16, ctypes.c_void_p(0x900000), None) == -2
  assert "BZ_MAX_N_COORDINATE = 128" in lib.bz_last_error().decode()

def test_the_row_limits_of_the_python_layers():
  torch = pytest.importorskip("torch")
  from byzantinemomentum_b200 import _lib, engine
  rows = [torch.zeros(4)] * 1024
  engine._validate(rows, limit=_lib.MAX_N_MANY)
  with pytest.raises(ValueError, match="maximum of 1024"):
    engine._validate(rows + rows[:1], limit=_lib.MAX_N_MANY)
  with pytest.raises(ValueError, match="maximum of 128"):
    engine._validate(rows[:129], limit=_lib.MAX_N_COORDINATE)
  # the device line search keeps its limits
  assert engine.search_max_rows("median") == _lib.MAX_N_COORDINATE
  assert engine.search_max_rows("krum") == _lib.MAX_N

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_many_row_kernels_fit_the_register_budget():
  """ libbyzagg_many.so: one sorting kernel per bucket of n (256, 512, 1024 rows) and K3's average over the
  1024-pointer table, all with no stack and no spill, and nothing else; libbyzagg.so has none of them. """
  from byzantinemomentum_b200 import _lib
  main = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout
  assert "ManyRowTable" not in main and "k1_many" not in main
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.many_library_path())], capture_output=True, text=True, timeout=600).stdout
  usage = {name: (int(regs), int(stack)) for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text)}
  many = {name: v for name, v in usage.items() if "ManyRowTable" in name}
  buckets = sorted(int(m.group(1)) for name in many for m in [re.search(r"k1_manyILi(\d+)E", name)] if m)
  assert buckets == [256, 512, 1024], buckets
  assert sorted(name for name in many if "k3_many_average" in name) == sorted(
    f"_ZN2bz15k3_many_averageILi{v}EEEvNS_12ManyRowTableENS_4GeomEifPf" for v in (1, 2, 4))
  assert len(many) == len(usage) == 6, sorted(usage)
  for name, (regs, stack) in many.items():
    assert regs <= 255 and stack == 0, (name, regs, stack)
  sass = subprocess.run([CUOBJDUMP, "-sass", str(_lib.many_library_path())], capture_output=True, text=True, timeout=600).stdout
  for block in re.split(r"\n\s*Function : ", sass)[1:]:
    if "ManyRowTable" in block.split("\n", 1)[0]:
      assert "STL" not in block and "LDL" not in block, block.split("\n", 1)[0]

@pytest.mark.parametrize("g,call", many_calls())
def test_oracle_matches_the_reference_above_128_rows(g, call):
  """ Pins the oracle, and with it the trimmed mean's summation cascade at n - 2f up to 1022. """
  gar, params, tag = call["gar"], call["params"], call["tag"]
  assert "raises" not in call and gar in ("average", "median", "trmean", "phocas", "meamed")
  rows = [g.rows[i] for i in range(g.n)]
  ref = g.get(tag, "out")
  got = orc.GARS[gar](rows, **params)
  if gar in ("average", "median"):
    parity.assert_bit_exact(got, ref, tag)
  elif gar == "trmean":
    parity.assert_trmean(got, ref, g.rows, tag)
  else:
    f = params["f"]
    center = orc.trmean(rows, f) if gar == "phocas" else orc.median(rows)
    amb = parity.closest_ambiguous(g.rows, g.n - f, center)
    parity.assert_close_scaled(got, ref, parity.column_scale(g.rows), tag, rtol=closest_rtol(g.n - f), exempt=amb)
    parity.assert_in_hull(got, g.rows, amb, tag)

def test_many_goldens_cover_the_new_range():
  paths = sorted(MANY_DIR.glob("golden_many_*.npz"))
  goldens = [Golden(p) for p in paths]
  assert sorted(g.n for g in goldens) == MANY_NS
  assert {g.manifest["kind"] for g in goldens} == {"iid", "nan", "inf", "quant", "nearmax", "tiny80"}
  for g in goldens:
    fs = sorted({c["params"]["f"] for c in g.calls if "f" in c["params"]})
    assert fs == sorted({1, (g.n - 1) // 4, (g.n - 1) // 2}), (g.name, fs)
    assert {c["gar"] for c in g.calls} == {"average", "median", "trmean", "phocas", "meamed"}
  assert sum(p.stat().st_size for p in paths) < 2.5 * 1024 * 1024
  assert not any(p.parent == MANY_DIR for p in (ROOT / "tests" / "golden").glob("golden_*.npz"))

# ---- gars.many_gars and the plugin ------------------------------------------------------------------------------------

def test_many_gars_mirror_gars_and_gars_keep_128_rows():
  torch = pytest.importorskip("torch")
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine
  assert sorted(bz.many_gars) == ["average", "meamed", "median", "phocas", "trmean"]
  assert len(bz.gars) == 10 and all(bz.many_gars[name] is not bz.gars[name] for name in bz.many_gars)
  rows = [torch.zeros(8)] * 1025
  for name, rule in bz.many_gars.items():
    assert rule.check is not None and rule.upper_bound is bz.gars[name].upper_bound and rule.influence is bz.gars[name].influence
  assert bz.many_gars["trmean"].check(gradients=rows[:300], f=149) is None
  assert bz.many_gars["trmean"].check(gradients=rows[:300], f=150) is not None
  # the rows limits, checked before any CUDA call
  with pytest.raises(ValueError, match=r"maximum of 128 \(`gars.many_gars`"):
    bz.gars["median"](gradients=rows[:129])
  with pytest.raises(ValueError, match="maximum of 128"):
    engine.trmean(rows[:300], 10)
  with pytest.raises(ValueError, match="maximum of 1024"):
    bz.many_gars["median"](gradients=rows)
  with pytest.raises(ValueError, match="maximum of 1024"):
    engine.coordinate_many("trmean", rows, 10)
  with pytest.raises(ValueError, match="unknown coordinate-wise rule"):
    engine.coordinate_many("krum", rows[:10], 1)

def test_many_install_registers_the_five_many_entries_and_keeps_the_search_at_128(monkeypatch):
  pytest.importorskip("torch")
  import types
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import plugin
  monkeypatch.setattr(plugin, "_installed", {})
  def aggregators():
    class Entry:
      def __init__(self, unchecked, check):
        self.unchecked, self.check = unchecked, check
    agg = types.SimpleNamespace(gars={})
    def register(name, unchecked, check, upper_bound=None, influence=None):
      agg.gars[name] = Entry(unchecked, check)
    agg.register = register
    return agg
  many, both = aggregators(), aggregators()
  assert plugin.install(many, many=True) == plugin.install(both, many=True, wide=True) == ["b200-" + name for name in bz.gars]
  for name in bz.gars:
    assert many.gars["b200-" + name].unchecked is bz.many_gars.get(name, bz.gars[name]).unchecked, name
    expected = bz.many_gars.get(name, bz.wide_gars.get(name, bz.gars[name]))
    assert both.gars["b200-" + name].unchecked is expected.unchecked, name
    if name in bz.many_gars:
      assert plugin._installed[many.gars["b200-" + name]] == (name, 128), name
