# coding: utf-8
"""`bz_coordinate` (include/byzagg_coordinate.h), the coordinate-wise rules for up to 128 rows, on
the CPU: the header and its binding, the argument checks (before any CUDA call), the host-side
row limit, the register budget of the kernels above 64 rows, and the NumPy oracle against the
reference's recorded outputs at n = 65..128 (`tests/golden/wide/`).  No compute calls here."""

import ctypes
import pathlib
import re
import shutil
import subprocess

import numpy as np
import pytest

from conftest import Golden
import parity
from oracle import byzoracle as orc

ROOT = pathlib.Path(__file__).resolve().parent.parent
WIDE_DIR = ROOT / "tests" / "golden" / "wide"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

def declared_symbols():
  text = (ROOT / "include" / "byzagg_coordinate.h").read_text()
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", text)))

def closest_rtol(m):
  """ The bar for Phocas / MeaMed: the reference sums the m selected values in `topk`'s unspecified
  order, so the rounding it may differ by grows with m; the 1e-6 of tests/parity.py, set for
  m <= 64, is scaled by m / 64 above. """
  return parity.RTOL * max(1., m / 64)

def wide_calls():
  out = []
  for path in sorted(WIDE_DIR.glob("golden_wide_*.npz")):
    g = Golden(path)
    for call in g.calls:
      out.append(pytest.param(g, call, id=f"{g.name}:{call['tag']}"))
  return out

def test_header_declares_bz_coordinate_and_byzagg_h_includes_it():
  assert declared_symbols() == ["bz_coordinate"]
  header = (ROOT / "include" / "byzagg_coordinate.h").read_text()
  assert re.search(r"#define BZ_MAX_N_COORDINATE 128\b", header)
  assert '#include "byzagg_coordinate.h"' in (ROOT / "include" / "byzagg.h").read_text()
  assert "byzagg_coordinate.h" in (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()

def test_library_exports_bz_coordinate_and_the_table_matches():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.library_path()))
  for name in declared_symbols():
    assert hasattr(handle, name), name
  assert sorted(_lib.COORDINATE_SIGNATURES) == declared_symbols()
  assert not set(_lib.COORDINATE_SIGNATURES) & set(_lib.SIGNATURES)
  assert getattr(_lib.lib(), "bz_coordinate").argtypes == _lib.COORDINATE_SIGNATURES["bz_coordinate"][1]
  assert _lib.MAX_N_COORDINATE == 128 and _lib.lib().bz_max_n() == _lib.MAX_N == 64

def test_bz_coordinate_rejects_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here (and d = 0, which launches nothing): the pointers are fake addresses. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  rows = lambda n, address=0x1000: (ctypes.c_void_p * n)(*[address + 0x100 * i for i in range(n)])
  out = ctypes.c_void_p(0x90000)
  def call(rule=2, table=None, n=100, f=10, d=16, dest=out):
    return lib.bz_coordinate(rule, rows(max(n, 1)) if table is None else table, n, f, d, dest, None)
  def message():
    return lib.bz_last_error().decode()
  assert call(n=0) == -1 and "n = 0" in message()
  assert call(n=129) == -2 and "BZ_MAX_N_COORDINATE" in message()
  for rule in (-1, 5):
    assert call(rule=rule) == -1 and "unknown rule" in message()
  assert call(f=50) == -1 and "n - 2f" in message()
  assert call(f=-1) == -1
  assert call(n=65, f=33) == -1
  assert lib.bz_coordinate(1, None, 100, 0, 16, out, None) == -1 and "rows is NULL" in message()
  assert call(dest=None) == -1 and "output" in message()
  assert call(table=rows(100, address=0x1002)) == -1 and "aligned" in message()
  with_null = rows(100)
  with_null[70] = None
  assert call(table=with_null) == -1 and "rows[70] is NULL" in message()
  assert call(dest=ctypes.c_void_p(0x90002)) == -1 and "aligned" in message()
  # f is not checked for average and median; d = 0 is a no-op for every rule
  assert call(rule=0, f=99, d=0) == 0 and call(rule=1, f=-5, d=0) == 0
  for rule in range(5):
    assert call(rule=rule, n=128, f=63, d=0, dest=None) == 0
  assert call(rule=4, n=3, f=1, d=0) == 0

def test_validate_takes_a_limit():
  torch = pytest.importorskip("torch")
  from byzantinemomentum_b200 import _lib, engine
  rows = [torch.zeros(4)] * 128
  engine._validate(rows, limit=_lib.MAX_N_COORDINATE)
  with pytest.raises(ValueError, match="maximum of 128"):
    engine._validate(rows + rows[:1], limit=_lib.MAX_N_COORDINATE)
  with pytest.raises(ValueError, match="coordinate-wise rules accept up to 128"):
    engine._validate(rows[:65])

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_kernels_above_64_rows_fit_the_register_budget():
  """ VEC = 1, two 128-thread CTAs per SM (<= 255 registers): the median keeps no stack, the
  sorted kernels no more than the 32-byte frame some n = 51 kernels keep. """
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout
  usage = {name: (int(regs), int(stack)) for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text)}
  wide = {name: v for name, v in usage.items() if "WideRowTable" in name}
  for kind in ("k1_median", "k1_sorted"):
    found = sorted(int(m.group(1)) for name in wide for m in [re.search(kind + r"ILi(\d+)ELi1E", name)] if m)
    assert found == list(range(65, 129)), (kind, found)
  assert sum("k3_average" in name for name in wide) == 3
  for name, (regs, stack) in wide.items():
    assert regs <= 255, (name, regs)
    assert stack <= (32 if "k1_sorted" in name else 0), (name, stack)

@pytest.mark.parametrize("g,call", wide_calls())
def test_oracle_matches_the_reference_above_64_rows(g, call):
  """ Pins the oracle, and with it the trimmed mean's summation cascade at n - 2f up to 126. """
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

def test_wide_goldens_cover_the_new_range():
  names = sorted(p.name for p in WIDE_DIR.glob("golden_wide_*.npz"))
  assert len(names) == 8
  ns = {Golden(WIDE_DIR / name).n for name in names}
  assert min(ns) == 65 and max(ns) == 128
  assert sum((WIDE_DIR / name).stat().st_size for name in names) < 2 * 1024 * 1024
  assert not any(p.parent == WIDE_DIR for p in (ROOT / "tests" / "golden").glob("golden_*.npz"))
