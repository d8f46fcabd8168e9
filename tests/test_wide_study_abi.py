# coding: utf-8
"""The study metrics and the attacks' line search above 64 rows, on the CPU: the NumPy oracle against
the reference's recorded `tools.compute_avg_dev_max` on the 65-128-row fixtures
(tests/golden/wide/study_avg_dev_max_wide.npz, made by tests/golden/make_study_wide_golden.py), the
row limits of `bz_avg_dev_max` and `bz_line_search` (checked before any CUDA call), the register budget
of the K6 kernels over the 128-pointer table, and the host-side limits of the plugin."""

import ctypes
import json
import math
import pathlib
import re
import shutil
import subprocess
import types

import numpy as np
import pytest

from oracle import byzoracle as orc
from parity import assert_bit_exact

ROOT = pathlib.Path(__file__).resolve().parent.parent
WIDE_DIR = ROOT / "tests" / "golden" / "wide"
GOLDEN = WIDE_DIR / "study_avg_dev_max_wide.npz"
SCALAR_RTOL = 2e-6     # the bar of tests/test_study_metrics.py
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

def cases():
  z = np.load(GOLDEN, allow_pickle=False)
  return [pytest.param(c, id=c["tag"]) for c in json.loads(str(z["manifest"]))["cases"]]

def load(case):
  """ (rows, avg or None, norm_avg, norm_dev, norm_max) of one recorded call. """
  z = np.load(GOLDEN, allow_pickle=False)
  rows = np.load(WIDE_DIR / case["fixture"], allow_pickle=False)["rows"][case["lo"]:case["hi"]]
  avg = z[case["tag"] + "/avg"] if case["has_avg"] else None
  return rows, avg, float(case["norm_avg"]), float(case["norm_dev"]), float(case["norm_max"])

def same_scalar(got, want, what):
  if math.isnan(want):
    assert math.isnan(got), f"{what}: {got} instead of nan"
  elif math.isinf(want):
    assert got == want, f"{what}: {got} instead of {want}"
  else:
    assert abs(got - want) <= SCALAR_RTOL * abs(want) + 1e-30, f"{what}: {got} vs {want}"

def check(result, avg, norm_avg, norm_dev, norm_max):
  got_avg, got_norm, got_dev, got_max = result
  if avg is None:
    assert got_avg is None
  else:
    assert_bit_exact(np.asarray(got_avg), avg)
  same_scalar(got_norm, norm_avg, "norm_avg")
  same_scalar(got_dev, norm_dev, "norm_dev")
  same_scalar(got_max, norm_max, "norm_max")

def test_golden_covers_the_wide_fixtures_and_is_small():
  z = np.load(GOLDEN, allow_pickle=False)
  recorded = json.loads(str(z["manifest"]))["cases"]
  fixtures = sorted(p.name for p in WIDE_DIR.glob("golden_wide_*.npz"))
  assert sorted({c["fixture"] for c in recorded}) == fixtures and len(recorded) == 3 * len(fixtures)
  assert max(c["hi"] - c["lo"] for c in recorded) == 128 and any(c["hi"] - c["lo"] > 64 for c in recorded if c["split"] == "honest")
  assert GOLDEN.stat().st_size < 1024 * 1024

@pytest.mark.parametrize("case", cases())
def test_oracle_matches_the_reference_above_64_rows(case):
  rows, avg, norm_avg, norm_dev, norm_max = load(case)
  check(orc.compute_avg_dev_max(list(rows)), avg, norm_avg, norm_dev, norm_max)

def test_avg_dev_max_takes_128_rows_and_names_the_limit_above():
  """ Only invalid calls here (each fails before any CUDA call): the pointers are fake addresses. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  rows = lambda n: (ctypes.c_void_p * n)(*[0x1000 + 0x100 * i for i in range(n)])
  avg, stats, ws = ctypes.c_void_p(0x90000), ctypes.c_void_p(0xa0000), ctypes.c_void_p(0xb0000)
  def call(n, ws_bytes=64):
    return lib.bz_avg_dev_max(rows(n), n, 16, avg, stats, ws, ws_bytes, None)
  message = lambda: lib.bz_last_error().decode()
  assert call(129) == -2 and "BZ_MAX_N_COORDINATE = 128" in message()
  for n in (64, 65, 100, 128):                      # past the row check: the small workspace is what fails
    assert call(n) == -4 and "workspace" in message(), n
  assert lib.bz_avg_dev_max(rows(128), 128, 16, avg, None, ws, 1 << 30, None) == -1 and "stats is NULL" in message()
  # the workspace of 64 rows serves up to 128
  assert lib.bz_workspace_bytes(128) == lib.bz_workspace_bytes(64)

def test_line_search_limit_depends_on_the_rule():
  """ Only invalid calls here: a valid one would launch on host memory. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  bufs = [(ctypes.c_float * 64)() for _ in range(5)]
  h, avg, att, byz, out = (ctypes.addressof(b) for b in bufs)
  trace = ctypes.addressof((ctypes.c_double * 64)())
  status = ctypes.addressof((ctypes.c_int32 * 2)())
  ws = ctypes.addressof((ctypes.c_double * 8)())
  def call(rule, nh, f_real, f_decl=5, evals=16, ws_bytes=1 << 40):
    rows = (ctypes.c_void_p * nh)(*([h] * nh))
    return lib.bz_line_search(rule, rows, nh, f_real, f_decl, 0, 0, avg, att, 64, evals, byz, out, trace, status,
                              ws, ws_bytes, None)
  message = lambda: lib.bz_last_error().decode()
  for rule in range(5):                             # average .. meamed: 128 rows pass the row check
    assert call(rule, 100, 28, evals=0) == -1 and "evals" in message(), rule
    assert call(rule, 100, 28, ws_bytes=64) == -4 and "workspace" in message(), rule
    assert call(rule, 100, 29) == -2 and "nh + f_real = 129 exceeds BZ_MAX_N_COORDINATE = 128" in message(), rule
  assert call(2, 100, 28, f_decl=64) == -1 and "n - 2f" in message()      # trmean's own check at n = 128
  for rule in range(5, 10):                         # the distance rules keep 64
    assert call(rule, 60, 5) == -2 and "nh + f_real = 65 exceeds BZ_MAX_N = 64" in message(), rule
  assert lib.bz_line_search_workspace_bytes(128) == lib.bz_line_search_workspace_bytes(64)

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_wide_study_kernels_fit_the_register_budget():
  """ One K6 kernel per bucket over the 128-pointer table, VEC = 1, <= 255 registers and no stack. """
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout
  usage = {name: (int(regs), int(stack)) for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text)}
  wide = {name: v for name, v in usage.items() if "k6_study" in name and "WideRowTable" in name}
  buckets = sorted(int(m.group(1)) for name in wide for m in [re.search(r"k6_studyILi(\d+)ELi1E", name)] if m)
  assert buckets == [80, 96, 112, 128] and len(wide) == 4, sorted(wide)
  for name, (regs, stack) in wide.items():
    assert regs <= 255 and stack == 0, (name, regs, stack)

def test_search_rows_limit_lives_in_the_engine():
  pytest.importorskip("torch")
  from byzantinemomentum_b200 import _lib, engine
  for gar in ("average", "median", "trmean", "phocas", "meamed"):
    assert engine.search_max_rows(gar) == _lib.MAX_N_COORDINATE == 128
  for gar in ("krum", "bulyan", "brute", "aksel", "cge"):
    assert engine.search_max_rows(gar) == _lib.MAX_N == 64

def test_device_rule_applies_the_rule_limit(monkeypatch):
  torch = pytest.importorskip("torch")
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import plugin
  class Entry:                                    # hashable, like the reference's checked functions
    def __init__(self, unchecked, check):
      self.unchecked, self.check = unchecked, check
  aggregators = types.SimpleNamespace(gars={})
  def register(name, unchecked, check, upper_bound=None, influence=None):
    aggregators.gars[name] = Entry(unchecked, check)
  aggregators.register = register
  bz.plugin.install(aggregators)
  monkeypatch.setattr(plugin, "_is_cuda", lambda tensors: True)          # CPU rows stand for CUDA rows
  rows = [torch.zeros(8) for _ in range(100)]
  rule = lambda gar, nh, f_real, f_decl: plugin._device_rule(aggregators.gars["b200-" + gar], rows[:nh], f_real, f_decl, None)
  assert rule("median", 100, 28, 5) == "median"
  assert rule("median", 100, 29, 5) is None                                # 129 rows
  assert rule("trmean", 100, 28, 40) == "trmean"
  assert rule("average", 65, 1, 0) == "average"
  assert rule("krum", 40, 24, 5) == "krum"                                 # 64 rows
  assert rule("krum", 40, 25, 5) is None                                   # 65 rows: a distance rule keeps 64
  assert rule("bulyan", 60, 5, 5) is None

def test_install_tools_takes_the_device_path_up_to_128_samples(monkeypatch):
  pytest.importorskip("torch")
  import byzantinemomentum_b200 as bz
  monkeypatch.setattr(bz.engine, "compute_avg_dev_max", lambda samples: ("device", len(samples)))
  tools = types.SimpleNamespace(compute_avg_dev_max=lambda samples: ("stock", len(samples)))
  bz.plugin.install_tools(tools)
  cuda = types.SimpleNamespace(is_cuda=True)
  assert tools.compute_avg_dev_max([cuda] * 65) == ("device", 65)
  assert tools.compute_avg_dev_max([cuda] * 128) == ("device", 128)
  assert tools.compute_avg_dev_max([cuda] * 129) == ("stock", 129)
