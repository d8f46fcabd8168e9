# coding: utf-8
"""GPU: Phocas and MeaMed column by column against K1's closest epilogue restated in NumPy
(tests/closest_columns.py), value for value (NaN == NaN), on stacks of constructed columns (infinities,
NaN of every sign and payload, NaN and infinite centres, key ties, plateaus, subnormals, overflow)
among random ones, and against the oracle where the chosen values are unique.  Every n from 3 to 128:
aligned rows (VEC = 4, 2 and 1, and the compile-time (n, f) kernels at n = 11, 25, 51), rows at mixed
4-byte offsets (the generic scalar kernel) and rows at one shared offset (the shifted vector path);
`bz_phocas` / `bz_meamed` up to 64 rows, `bz_coordinate` above.  Then one stack per rule through
`bz.gars` and `engine.Plan`."""

import ctypes

import numpy as np
import pytest

import closest_columns as cc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RULES = {"phocas": 3, "meamed": 4}      # BZ_RULE_*
LAYOUTS = {"aligned": [0], "mixed offsets": [0, 1, 2, 3, 1], "shared offset": [3]}

def _lib():
  from byzantinemomentum_b200 import _lib
  return _lib.lib()

def _device_rows(x, offsets):
  """ Row i of x at float offset offsets[i % len(offsets)] of its own 16-byte aligned stretch of one buffer. """
  n, d = x.shape
  pitch = (d + 8 + 3) // 4 * 4
  buf = torch.empty((n, pitch), device=DEV)
  host = torch.full((n, pitch), float("nan"))
  offs = [offsets[i % len(offsets)] for i in range(n)]
  for i in range(n):
    host[i, offs[i]:offs[i] + d] = torch.from_numpy(x[i])
  buf.copy_(host)
  return [buf[i, offs[i]:offs[i] + d] for i in range(n)]

def _call(mode, rows, f, d, offset=0):
  """ bz_<mode> up to 64 rows, bz_coordinate above, into a NaN-filled output at `offset`. """
  lib = _lib()
  n = len(rows)
  big = torch.full((d + 8,), float("nan"), device=DEV)
  out = big[offset:offset + d]
  ptrs = (ctypes.c_void_p * n)(*[r.data_ptr() for r in rows])
  stream = torch.cuda.current_stream().cuda_stream
  if n <= 64:
    rc = getattr(lib, "bz_" + mode)(ptrs, n, f, d, out.data_ptr(), stream)
  else:
    rc = lib.bz_coordinate(RULES[mode], ptrs, n, f, d, out.data_ptr(), stream)
  assert rc == 0, lib.bz_last_error()
  assert torch.isnan(big[:offset]).all() and torch.isnan(big[offset + d:]).all()
  return out.cpu().numpy()

def _check(n, fs, layouts, d, seed):
  for f in fs:
    x = cc.stack(n, f, d, seed + 131 * f)
    want = {mode: cc.k1_closest(x, f, mode)[0] for mode in cc.MODES}
    for layout in layouts:
      offsets = LAYOUTS[layout]
      rows = _device_rows(x, offsets)
      out_offset = offsets[0] if layout == "shared offset" else 0
      for mode in cc.MODES:
        got = _call(mode, rows, f, d, out_offset)
        cc.check_kernel(got, x, f, mode, f"{mode} n={n} f={f} {layout}", want=want[mode])

def _fs(n):
  return sorted({1, (n - 1) // 4, (n - 1) // 2} - {0})

@pytest.mark.parametrize("n", list(range(3, 129)))
def test_every_n(n):
  _check(n, _fs(n), LAYOUTS, 645 + 3 * n, 40_000 + n)

@pytest.mark.parametrize("n", [11, 25, 51])
def test_every_f_of_the_compile_time_kernels(n):
  """ Aligned rows and one shared offset take the (n, f) kernels with literal partners; mixed offsets the generic one. """
  _check(n, range(1, (n - 1) // 2 + 1), LAYOUTS, 1031, 41_000 + n)

@pytest.mark.parametrize("n", [25, 100])
@pytest.mark.parametrize("gar", cc.MODES)
def test_plugin_and_plan(n, gar):
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine
  f = (n - 1) // 4
  d = 2053
  x = cc.stack(n, f, d, 42_000 + n)
  rows = [torch.from_numpy(x[i].copy()).to(DEV) for i in range(n)]
  want = cc.k1_closest(x, f, gar)[0]
  plain = bz.gars[gar](gradients=rows, f=f)
  cc.check_kernel(plain.cpu().numpy(), x, f, gar, f"{gar} n={n} plugin", want=want)
  plan = engine.Plan(gar, rows, f=f)
  cc.check_kernel(plan().cpu().numpy(), x, f, gar, f"{gar} n={n} Plan", want=want)
