# coding: utf-8
"""`bz_distance` (include/byzagg_distance.h), Multi-Krum, Bulyan, Aksel and CGE for up to 128 rows, on the
CPU: the header and its binding, the argument checks (before any CUDA call, with fake pointers), the
register and stack budgets of the kernels above 64 rows, and the NumPy oracle against the reference's
recorded outputs and selections at n = 65..128 (`tests/golden/wide_distance/`).  No compute calls here."""

import ctypes
import pathlib
import re
import shutil
import subprocess

import numpy as np
import pytest

from conftest import Golden, canon_alias
import parity
from oracle import byzoracle as orc

ROOT = pathlib.Path(__file__).resolve().parent.parent
WD_DIR = ROOT / "tests" / "golden" / "wide_distance"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
KRUM, BULYAN, BRUTE, AKSEL, CGE = 5, 6, 7, 8, 9

def declared_symbols():
  text = (ROOT / "include" / "byzagg_distance.h").read_text()
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", text)))

def wd_calls():
  out = []
  for path in sorted(WD_DIR.glob("golden_wd_*.npz")):
    g = Golden(path)
    for call in g.calls:
      out.append(pytest.param(g, call, id=f"{g.name}:{call['tag']}"))
  return out

def test_header_declares_bz_distance_and_byzagg_h_includes_it():
  assert declared_symbols() == ["bz_distance", "bz_distance_workspace_bytes"]
  assert re.search(r"#define BZ_MAX_N_DISTANCE 128\b", (ROOT / "include" / "byzagg_distance.h").read_text())
  assert '#include "byzagg_distance.h"' in (ROOT / "include" / "byzagg.h").read_text()
  assert "byzagg_distance.h" in (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()

def test_library_exports_bz_distance_and_the_table_matches():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.library_path()))
  for name in declared_symbols():
    assert hasattr(handle, name), name
  assert sorted(_lib.DISTANCE_SIGNATURES) == declared_symbols()
  others = set(_lib.SIGNATURES) | set(_lib.COORDINATE_SIGNATURES)
  assert not set(_lib.DISTANCE_SIGNATURES) & others
  for name, (restype, argtypes) in _lib.DISTANCE_SIGNATURES.items():
    assert getattr(_lib.lib(), name).argtypes == argtypes
  assert _lib.MAX_N_DISTANCE == 128 and _lib.lib().bz_max_n() == _lib.MAX_N == 64

def test_workspace_sizes():
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  for n in range(1, 65):
    assert lib.bz_distance_workspace_bytes(n) == lib.bz_workspace_bytes(n), n
  wide = lib.bz_distance_workspace_bytes(65)
  assert wide > lib.bz_workspace_bytes(64) and wide % 256 == 0
  assert all(lib.bz_distance_workspace_bytes(n) == wide for n in (100, 128))
  assert lib.bz_workspace_bytes(128) == lib.bz_workspace_bytes(64)        # unchanged

def test_bz_distance_rejects_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here (and d = 0, which launches nothing): the pointers are fake addresses. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  rows = lambda n, address=0x1000: (ctypes.c_void_p * n)(*[address + 0x100 * i for i in range(n)])
  out, order, status = ctypes.c_void_p(0x90000), ctypes.c_void_p(0xa0000), ctypes.c_void_p(0xb0000)
  big = 1 << 40
  def call(rule=KRUM, table=None, n=100, f=10, m=20, mode=0, d=16, dest=out, ws=0xc0000, ws_bytes=big):
    return lib.bz_distance(rule, rows(max(n, 1)) if table is None else table, n, f, m, mode, d, dest, order, status,
                           ctypes.c_void_p(ws), ws_bytes, None)
  def message():
    return lib.bz_last_error().decode()
  assert call(n=0) == -1 and "n = 0" in message()
  assert call(n=129) == -2 and "BZ_MAX_N_DISTANCE = 128" in message()
  for rule in (0, 1, 2, 3, 4, 10, -1):
    assert call(rule=rule) == -1 and "unknown rule" in message(), rule
  assert call(rule=BRUTE, n=65) == -2 and "brute" in message()
  assert call(rule=BRUTE, n=128, d=0) == -2
  # Multi-Krum: n - f - 1 >= 1, 1 <= m <= n
  assert call(f=99) == -1 and "n - f - 1" in message()
  assert call(f=-1) == -1
  assert call(m=0) == -1 and "m = 0" in message()
  assert call(m=101) == -1 and "expected 1..100" in message()
  # Bulyan: n >= 4f + 3, 1 <= m <= n - f - 2
  assert call(rule=BULYAN, f=25) == -1 and "4f + 3" in message()
  assert call(rule=BULYAN, n=65, f=16, m=1) == -1
  assert call(rule=BULYAN, f=24, m=75) == -1 and "expected 1..74" in message()
  assert call(rule=BULYAN, f=24, m=0) == -1
  # Aksel: its mode, and c in 1..n
  assert call(rule=AKSEL, mode=2) == -1 and "mode = 2" in message()
  assert call(rule=AKSEL, mode=1, f=100) == -1 and "not executable" in message()
  # the rows and the output
  assert lib.bz_distance(KRUM, None, 100, 10, 20, 0, 16, out, None, None, ctypes.c_void_p(0xc0000), big, None) == -1 and "rows is NULL" in message()
  assert call(dest=None) == -1 and "output" in message()
  assert call(table=rows(100, address=0x1002)) == -1 and "aligned" in message()
  with_null = rows(100)
  with_null[70] = None
  assert call(table=with_null) == -1 and "rows[70] is NULL" in message()
  # the workspace: bz_distance_workspace_bytes(n), 8-byte aligned
  need = lib.bz_distance_workspace_bytes(100)
  for rule in (KRUM, BULYAN, AKSEL, CGE):
    assert call(rule=rule, f=20, m=10, ws_bytes=need - 1) == -4 and "workspace" in message(), rule
    assert call(rule=rule, f=20, m=10, ws=0xc0004) == -4, rule
    assert call(rule=rule, f=20, m=10, ws=0) == -4, rule
  assert call(n=64, ws_bytes=lib.bz_workspace_bytes(64) - 1) == -4
  # d = 0 is a no-op for every rule, at every n
  for n in (7, 64, 65, 128):
    for rule in (KRUM, BULYAN, AKSEL, CGE):
      f = (n - 3) // 4
      assert call(rule=rule, n=n, f=f, m=1, d=0, dest=None, ws_bytes=need) == 0, (rule, n)
  # CGE checks no f (cge.py does not either)
  assert call(rule=CGE, f=200, d=0) == 0 and call(rule=CGE, f=-5, d=0) == 0

def test_plan_limits_stay_where_they_were():
  torch = pytest.importorskip("torch")
  from byzantinemomentum_b200 import _lib, engine
  rows = [torch.zeros(4)] * 65
  with pytest.raises(ValueError, match="coordinate-wise rules accept up to 128"):
    engine._validate(rows)                       # the default limit and its message are unchanged
  assert engine.WIDE_DISTANCE == ("krum", "bulyan", "aksel", "cge")
  assert engine.search_max_rows("krum") == _lib.MAX_N == 64

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_kernels_above_64_rows_fit_the_register_budget():
  """ The kernels bz_distance adds: K5 over the pass tables, K2' and the 12 K4 buckets over the 128-pointer
  table; no stack, no spill. """
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout
  usage = {name: (int(regs), int(stack)) for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text)}
  k5 = [name for name in usage if "k5_score_select_wide" in name]
  k2 = [name for name in usage if "k2_rowdist_wide" in name]
  k4 = sorted(int(m.group(1)) for name in usage for m in [re.search(r"k4_bulyan_wideILi(\d+)E", name)] if m)
  assert len(k5) == 1 and len(k2) == 2
  assert k4 == list(range(40, 129, 8)), k4
  for name in k5 + k2 + [name for name in usage if "k4_bulyan_wide" in name]:
    regs, stack = usage[name]
    assert regs <= 255 and stack == 0, (name, regs, stack)

def test_wide_distance_goldens_cover_the_range_and_stay_apart():
  names = sorted(p.name for p in WD_DIR.glob("golden_wd_*.npz"))
  assert len(names) >= 6
  goldens = [Golden(WD_DIR / name) for name in names]
  ns = {g.n for g in goldens}
  assert min(ns) == 65 and max(ns) == 128
  gars = {call["gar"] for g in goldens for call in g.calls}
  assert gars == {"krum", "bulyan", "aksel", "cge"}
  assert {g.manifest["kind"] for g in goldens} >= {"iid", "empire", "little", "nan", "inf", "quant",
                                                   "tiny80", "tiny110", "huge", "mixed", "hugebyz", "nearmax"}
  assert sum((WD_DIR / name).stat().st_size for name in names) < 2 * 1024 * 1024
  assert not list((ROOT / "tests" / "golden").glob("golden_wd_*.npz"))
  assert not list((ROOT / "tests" / "golden" / "wide").glob("golden_wd_*.npz"))

@pytest.mark.parametrize("g,call", wd_calls())
def test_oracle_matches_the_reference_above_64_rows(g, call):
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
  ref_order = g.get(tag, "order")
  if gar == "aksel" and np.isnan(g.get(tag, "dists")).any():     # NaN keys: the reference's order is undefined
    return
  assert canon_alias(info["order"][:count], g.nh) == canon_alias(ref_order[:count], g.nh), f"{tag}: selection differs"
  parity.assert_bit_exact(got, ref, tag)
