# coding: utf-8
"""`bz_avg_dev_max_many` and `bz_line_search_many` (include/byzagg_many_tools.h), the study metrics and the line
search against the coordinate-wise rules for up to 1024 rows, on the CPU: the header and its binding, the argument
checks (before any CUDA call), the register budget of the K6-many kernels, the host-side limits of the Python
layers, and the NumPy oracle against the reference's recorded `tools.compute_avg_dev_max` on the 129-1024-row
fixtures (tests/golden/many/study_avg_dev_max_many.npz, made by tests/golden/make_study_many_golden.py)."""

import ctypes
import json
import pathlib
import re
import shutil
import subprocess
import types

import numpy as np
import pytest

from oracle import byzoracle as orc
from test_wide_study_abi import check

ROOT = pathlib.Path(__file__).resolve().parent.parent
MANY_DIR = ROOT / "tests" / "golden" / "many"
GOLDEN = MANY_DIR / "study_avg_dev_max_many.npz"
HEADER = ROOT / "include" / "byzagg_many_tools.h"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
SYMBOLS = ["bz_avg_dev_max_many", "bz_avg_dev_max_many_workspace_bytes", "bz_line_search_many",
           "bz_line_search_many_workspace_bytes", "bz_many_tools_last_error"]

def declared_symbols():
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", HEADER.read_text())))

def cases():
  z = np.load(GOLDEN, allow_pickle=False)
  return [pytest.param(c, id=c["tag"]) for c in json.loads(str(z["manifest"]))["cases"]]

def load(case):
  """ (rows, avg or None, norm_avg, norm_dev, norm_max) of one recorded call. """
  z = np.load(GOLDEN, allow_pickle=False)
  rows = np.load(MANY_DIR / case["fixture"], allow_pickle=False)["rows"][case["lo"]:case["hi"]]
  avg = z[case["tag"] + "/avg"] if case["has_avg"] else None
  return rows, avg, float(case["norm_avg"]), float(case["norm_dev"]), float(case["norm_max"])

def test_header_declares_the_five_symbols_and_stays_out_of_byzagg_h():
  assert declared_symbols() == SYMBOLS
  for header in (ROOT / "include").glob("*.h"):
    if header != HEADER:
      assert "byzagg_many_tools.h" not in header.read_text(), header.name
  makefile = (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  assert "byzagg_many_tools.h" in makefile and re.search(r"^all: \$\(MANY_TOOLS_OUT\)$", makefile, re.M)

def test_the_fifth_library_exports_the_symbols_and_no_other_library_does():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.many_tools_library_path()))
  for name in SYMBOLS:
    assert hasattr(handle, name), name
  for path in (_lib.library_path(), _lib.peers_library_path(), _lib.star_library_path(), _lib.many_library_path()):
    other = ctypes.CDLL(str(path))
    assert not any(hasattr(other, name) for name in SYMBOLS), path.name
  assert _lib.many_tools_library_path().parent == _lib.library_path().parent
  assert sorted(_lib.MANY_TOOLS_SIGNATURES) == SYMBOLS
  tools = _lib.many_tools_lib()
  for name, (restype, argtypes) in _lib.MANY_TOOLS_SIGNATURES.items():
    assert getattr(tools, name).argtypes == argtypes and getattr(tools, name).restype == restype, name
  assert _lib.MANY_TOOLS_SIGNATURES["bz_avg_dev_max_many"] == _lib.SIGNATURES["bz_avg_dev_max"]
  assert _lib.MANY_TOOLS_SIGNATURES["bz_line_search_many"] == _lib.ATTACK_SIGNATURES["bz_line_search"]

def test_library_path_override(monkeypatch):
  from byzantinemomentum_b200 import _lib
  monkeypatch.setenv("BYZAGG_MANY_TOOLS_LIBRARY", "/somewhere/else.so")
  assert str(_lib.many_tools_library_path()) == "/somewhere/else.so"

def test_avg_dev_max_many_rejects_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here (each fails before any CUDA call): the pointers are fake addresses. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.many_tools_lib()
  rows = lambda n, address=0x1000: (ctypes.c_void_p * n)(*[address + 0x100 * i for i in range(n)])
  avg, stats, ws = ctypes.c_void_p(0x900000), ctypes.c_void_p(0xa00000), ctypes.c_void_p(0xb00000)
  message = lambda: lib.bz_many_tools_last_error().decode()
  def call(n, ws_bytes=64, table=None, dest=avg, out=stats):
    return lib.bz_avg_dev_max_many(rows(max(n, 1)) if table is None else table, n, 16, dest, out, ws, ws_bytes, None)
  assert call(1025) == -2 and "bz_avg_dev_max_many" in message() and "BZ_MAX_N_MANY = 1024" in message()
  assert call(0) == -1 and "n = 0" in message()
  for n in (1, 128, 129, 300, 1024):               # past the row check: the small workspace is what fails
    assert call(n) == -4 and "workspace" in message(), n
    assert call(n, ws_bytes=1 << 40, out=None) == -1 and "stats is NULL" in message(), n
  assert call(300, ws_bytes=1 << 40, dest=None) == -1 and "output" in message()
  assert call(300, ws_bytes=1 << 40, table=rows(300, address=0x1002)) == -1 and "aligned" in message()
  with_null = rows(1024)
  with_null[900] = None
  assert call(1024, ws_bytes=1 << 40, table=with_null) == -1 and "rows[900] is NULL" in message()
  # up to 128 rows the workspace is bz_avg_dev_max's; above, a block per CTA, growing with n
  main = _lib.lib()
  for n in (1, 64, 128):
    assert lib.bz_avg_dev_max_many_workspace_bytes(n) == main.bz_workspace_bytes(n)
  sizes = [lib.bz_avg_dev_max_many_workspace_bytes(n) for n in (129, 512, 1024)]
  assert sizes == sorted(sizes) and all(s % 256 == 0 for s in sizes)
  # the message reaches Python from this library
  assert call(2000) == -2
  with pytest.raises(ValueError, match="bz_avg_dev_max_many.*BZ_MAX_N_MANY = 1024"):
    _lib.check(-2, "bz_avg_dev_max_many")

def test_the_128_row_entry_points_keep_their_limits():
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  table = (ctypes.c_void_p * 129)(*[0x1000 + 0x100 * i for i in range(129)])
  assert lib.bz_avg_dev_max(table, 129, 16, ctypes.c_void_p(0x90000), ctypes.c_void_p(0xa0000), ctypes.c_void_p(0xb0000),
                            1 << 40, None) == -2
  assert "BZ_MAX_N_COORDINATE = 128" in lib.bz_last_error().decode()

def test_line_search_many_rejects_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here: a valid one would launch on host memory. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.many_tools_lib()
  bufs = [(ctypes.c_float * 64)() for _ in range(5)]
  h, avg, att, byz, out = (ctypes.addressof(b) for b in bufs)
  trace = ctypes.addressof((ctypes.c_double * 64)())
  status = ctypes.addressof((ctypes.c_int32 * 2)())
  ws = ctypes.addressof((ctypes.c_double * 8)())
  def call(rule, nh, f_real, f_decl=5, evals=16, ws_bytes=1 << 40, honest=None, dest=None, b=None):
    rows = (ctypes.c_void_p * nh)(*([h] * nh)) if honest is None else honest
    return lib.bz_line_search_many(rule, rows, nh, f_real, f_decl, 0, 0, avg, att, 64, evals, b or byz, dest or out, trace,
                                   status, ws, ws_bytes, None)
  message = lambda: lib.bz_many_tools_last_error().decode()
  for rule in range(5):                            # average .. meamed: 1024 rows pass the row check
    assert call(rule, 1000, 24, evals=0) == -1 and "evals" in message(), rule
    assert call(rule, 1000, 24, ws_bytes=64) == -4 and "workspace" in message(), rule
    assert call(rule, 1000, 25) == -2 and "nh + f_real = 1025 exceeds BZ_MAX_N_MANY = 1024" in message(), rule
    assert call(rule, 100, 20, ws_bytes=64) == -4, rule    # the workspace of bz_line_search up to 128 rows
  for rule in range(5, 10):                        # the distance rules: bz_line_search / bz_distance_line_search
    assert call(rule, 60, 5) == -1 and "bz_line_search" in message() and "bz_distance_line_search" in message(), rule
    assert call(rule, 300, 5) == -1, rule
  assert call(10, 60, 5) == -1 and "unknown rule" in message()
  assert call(2, 1000, 24, f_decl=512) == -1 and "n - 2f" in message()      # trmean's n - 2f >= 1 at n = 1024
  assert call(2, 1000, 24, f_decl=511, ws_bytes=64) == -4                    # 1024 - 1022 = 2 rows kept: past it
  assert call(3, 300, 5, f_decl=-1) == -1 and "n - 2f" in message()
  assert call(1, 300, 0) == -1 and "f_real" in message()
  assert call(1, 300, 5, b=h) == -1 and "honest[0] is byz or out" in message()
  assert call(1, 300, 5, dest=avg) == -1 and "distinct" in message()
  assert call(1, 300, 5, dest=byz) == -1 and "distinct" in message()
  assert call(1, 300, 5, b=att) == -1 and "distinct" in message()
  with_null = (ctypes.c_void_p * 300)(*([h] * 300))
  with_null[250] = None
  assert call(1, 300, 5, honest=with_null) == -1 and "rows[250] is NULL" in message()
  main = _lib.lib()
  for n in (2, 64, 128):
    assert lib.bz_line_search_many_workspace_bytes(n) == main.bz_line_search_workspace_bytes(n)
  assert lib.bz_line_search_many_workspace_bytes(1024) % 256 == 0

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_study_many_kernels_fit_the_register_budget():
  """ libbyzagg_many_tools.so: one K6-many kernel per bucket of n (256, 512, 1024 rows), <= 255 registers, no stack,
  no spill, and nothing else; no other library has them. """
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.many_tools_library_path())], capture_output=True, text=True,
                        timeout=600).stdout
  usage = {name: (int(regs), int(stack)) for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text)}
  buckets = sorted(int(m.group(1)) for name in usage for m in [re.search(r"k6_manyILi(\d+)E", name)] if m)
  assert buckets == [256, 512, 1024] and len(usage) == 3, sorted(usage)
  for name, (regs, stack) in usage.items():
    assert "ManyRowTable" in name and regs <= 255 and stack == 0, (name, regs, stack)
  sass = subprocess.run([CUOBJDUMP, "-sass", str(_lib.many_tools_library_path())], capture_output=True, text=True,
                        timeout=600).stdout
  for block in re.split(r"\n\s*Function : ", sass)[1:]:
    assert "STL" not in block and "LDL" not in block, block.split("\n", 1)[0]
  for path in (_lib.library_path(), _lib.peers_library_path(), _lib.star_library_path(), _lib.many_library_path()):
    other = subprocess.run([CUOBJDUMP, "-res-usage", str(path)], capture_output=True, text=True, timeout=600).stdout
    assert "k6_many" not in other, path.name

def test_the_row_limits_of_the_python_layers():
  torch = pytest.importorskip("torch")
  from byzantinemomentum_b200 import _lib, engine, sharded
  rows = [torch.zeros(4)] * 1025
  with pytest.raises(ValueError, match="maximum of 1024"):
    engine.avg_dev_max_many_async(rows)
  with pytest.raises(ValueError, match="maximum of 128"):
    engine.avg_dev_max_async(rows[:129])
  for gar in ("average", "median", "trmean", "phocas", "meamed"):
    assert sharded.search_rows(gar, many=True) == _lib.MAX_N_MANY == 1024
    assert sharded.search_rows(gar) == sharded.search_rows(gar, wide=True) == 128
    assert engine.search_max_rows(gar) == 128
  for gar in ("krum", "bulyan", "brute", "aksel", "cge"):
    assert sharded.search_rows(gar, many=True) == sharded.search_rows(gar) == 64
  for gar in ("krum", "bulyan", "aksel", "cge"):
    assert sharded.search_rows(gar, wide=True, many=True) == 128
  # many=True takes the coordinate-wise rules only
  with pytest.raises(ValueError, match="coordinate-wise"):
    engine.LineSearch("krum", rows[:10], 2, 1, rows[0], rows[0], 4, many=True)
  with pytest.raises(ValueError, match="coordinate-wise"):
    sharded.ShardedLineSearch("cge", rows[:10], 2, 1, rows[0], rows[0], 4, many=True)

def _registry():
  class Entry:                                    # hashable, like the reference's checked functions
    def __init__(self, unchecked, check):
      self.unchecked, self.check = unchecked, check
  aggregators = types.SimpleNamespace(gars={})
  def register(name, unchecked, check, upper_bound=None, influence=None):
    aggregators.gars[name] = Entry(unchecked, check)
  aggregators.register = register
  return aggregators

def test_device_rule_takes_1024_rows_against_a_many_entry_only_when_asked(monkeypatch):
  torch = pytest.importorskip("torch")
  from byzantinemomentum_b200 import plugin
  aggregators = _registry()
  plugin.install(aggregators, prefix="many-", many=True)
  plugin.install(aggregators)
  monkeypatch.setattr(plugin, "_is_cuda", lambda tensors: True)          # CPU rows stand for CUDA rows
  rows = [torch.zeros(8) for _ in range(1024)]
  def rule(prefix, gar, nh, f_real, f_decl, many):
    return plugin._device_rule(aggregators.gars[prefix + gar], rows[:nh], f_real, f_decl, None, many)
  for many in (False, True):
    assert rule("many-", "median", 100, 28, 5, many) == "median"             # 128 rows either way
  assert rule("many-", "median", 100, 29, 5, False) is None                # 129 rows: only with many
  assert rule("many-", "median", 100, 29, 5, True) == "median"
  assert rule("many-", "trmean", 1000, 24, 100, True) == "trmean"
  assert rule("many-", "average", 1000, 25, 0, True) is None               # 1025 rows
  assert rule("b200-", "median", 200, 20, 5, True) is None                 # a default entry keeps 128
  assert rule("b200-", "krum", 40, 25, 5, True) is None                    # a distance rule keeps 64
  # the record of the registry is unchanged: the many entries keep their 128-row value
  assert plugin._installed[aggregators.gars["many-median"]] == ("median", 128)
  assert aggregators.gars["many-median"] in plugin._many_installed
  assert aggregators.gars["b200-median"] not in plugin._many_installed

def test_install_attacks_passes_many_above_128_rows_only(monkeypatch):
  torch = pytest.importorskip("torch")
  from byzantinemomentum_b200 import plugin
  aggregators = _registry()
  plugin.install(aggregators, prefix="many-", many=True)
  monkeypatch.setattr(plugin, "_is_cuda", lambda tensors: True)
  calls = []
  class Backend:
    @staticmethod
    def line_search(*args, **kwargs):
      calls.append((len(args[1]) + args[2], kwargs))
      return 0., args[1][0]
  def registry():
    attacks = types.SimpleNamespace(attacks={})
    stock = types.SimpleNamespace(unchecked=lambda **kwargs: "stock", check=None)
    for name in ("little", "empire", "bulyan", "empire-strict"):
      attacks.attacks[name] = stock
    def register(name, unchecked, check):
      attacks.attacks[name] = types.SimpleNamespace(unchecked=unchecked, check=check)
    attacks.register = register
    return attacks
  defense = aggregators.gars["many-median"]
  rows = [torch.ones(8) for _ in range(300)]
  default, many = registry(), registry()
  plugin.install_attacks(default, backend=Backend)
  plugin.install_attacks(many, backend=Backend, many=True)
  run = lambda attacks, name, nh, **kw: attacks.attacks[name].unchecked(grad_honests=rows[:nh], f_real=20, f_decl=5,
                                                                        defense=defense, model=None, **kw)
  assert run(default, "empire", 280, factor=-4) == "stock" and not calls
  assert run(many, "empire", 280, factor=-4)[0] is rows[0]
  assert calls[-1] == (300, dict(negative=False, kind="identical", many=True))
  assert run(many, "empire-strict", 280, epsilon=-4)[0] is rows[0]
  assert calls[-1] == (300, dict(kind="empire-strict", many=True))
  assert run(many, "little", 100, factor=-4)[0] is rows[0]                 # 120 rows: today's call
  assert calls[-1] == (120, dict(negative=False, kind="identical"))
  assert run(default, "little", 100, factor=-4)[0] is rows[0]
  assert calls[-1] == (120, dict(negative=False, kind="identical"))

def test_install_tools_takes_the_device_path_up_to_1024_samples_with_many(monkeypatch):
  pytest.importorskip("torch")
  import byzantinemomentum_b200 as bz
  monkeypatch.setattr(bz.engine, "compute_avg_dev_max", lambda samples, many=False: ("device", len(samples), many))
  tools = types.SimpleNamespace(compute_avg_dev_max=lambda samples: ("stock", len(samples)))
  bz.plugin.install_tools(tools, many=True)
  cuda = types.SimpleNamespace(is_cuda=True)
  assert tools.compute_avg_dev_max([cuda] * 1) == ("device", 1, True)
  assert tools.compute_avg_dev_max([cuda] * 129) == ("device", 129, True)
  assert tools.compute_avg_dev_max([cuda] * 1024) == ("device", 1024, True)
  assert tools.compute_avg_dev_max([cuda] * 1025) == ("stock", 1025)
  assert tools.compute_avg_dev_max([types.SimpleNamespace(is_cuda=False)] * 300) == ("stock", 300)

def test_golden_covers_the_many_fixtures_and_is_small():
  z = np.load(GOLDEN, allow_pickle=False)
  recorded = json.loads(str(z["manifest"]))["cases"]
  fixtures = sorted(p.name for p in MANY_DIR.glob("golden_many_*.npz"))
  assert sorted({c["fixture"] for c in recorded}) == fixtures and len(recorded) == 3 * len(fixtures)
  assert max(c["hi"] - c["lo"] for c in recorded) == 1024
  assert any(c["hi"] - c["lo"] > 128 for c in recorded if c["split"] == "honest")
  assert GOLDEN.stat().st_size < 1024 * 1024

@pytest.mark.parametrize("case", cases())
def test_oracle_matches_the_reference_above_128_rows(case):
  rows, avg, norm_avg, norm_dev, norm_max = load(case)
  check(orc.compute_avg_dev_max(list(rows)), avg, norm_avg, norm_dev, norm_max)
