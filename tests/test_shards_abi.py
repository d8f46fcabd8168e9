# coding: utf-8
"""The entry points of `include/byzagg_shards.h` (gradient delivery for a d-sharded trainer): the header
declares them, `byzagg.h` includes it, the library exports them, the second ctypes table of
`_lib.py` matches, the argument checks run before any CUDA call, and the kernel compiles without
spilling.  No compute calls here (CPU suite)."""

import ctypes
import pathlib
import re
import shutil
import subprocess

import pytest

ROOT = pathlib.Path(__file__).resolve().parent.parent
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

def declared_symbols():
  text = (ROOT / "include" / "byzagg_shards.h").read_text()
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", text)))

def test_header_declares_the_delivery_and_byzagg_h_includes_it():
  assert declared_symbols() == ["bz_gradient_momentum", "bz_gradient_scatter"]
  main = (ROOT / "include" / "byzagg.h").read_text()
  assert '#include "byzagg_shards.h"' in main
  assert "byzagg_shards.h" in (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()

def test_library_exports_the_delivery_and_the_table_matches():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.library_path()))
  for name in declared_symbols():
    assert hasattr(handle, name), name
  assert sorted(_lib.SHARD_SIGNATURES) == declared_symbols()
  assert not set(_lib.SHARD_SIGNATURES) & set(_lib.SIGNATURES)
  for name in declared_symbols():
    assert getattr(_lib.lib(), name).argtypes == _lib.SHARD_SIGNATURES[name][1]

def test_gradient_scatter_rejects_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here: a valid one would launch on host memory. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  buf = (ctypes.c_float * 256)()
  a = ctypes.addressof(buf)
  dest = lambda *p: (ctypes.c_void_p * len(p))(*p)
  def call(grad=a, d=64, clip=0., nranks=2, slots=None):
    return lib.bz_gradient_scatter(grad, d, clip, nranks, dest(a, a) if slots is None else slots, None, 0, None)
  assert call(grad=None) == -1 and b"grad is NULL" in lib.bz_last_error()
  assert call(d=-1) == -1
  assert call(nranks=0) == -1 and b"nranks" in lib.bz_last_error()
  assert call(nranks=17, slots=dest(*[a] * 17)) == -1
  assert lib.bz_gradient_scatter(a, 64, 0., 2, None, None, 0, None) == -1 and b"dest is NULL" in lib.bz_last_error()
  assert call(slots=dest(a, None)) == -1 and b"dest[1] is NULL" in lib.bz_last_error()
  assert call(d=1, slots=dest(None, a)) == -1 and b"dest[0]" in lib.bz_last_error()    # rank 0 owns the only column
  assert call(slots=dest(a + 4, a)) == -1 and b"16-byte" in lib.bz_last_error()

def test_gradient_momentum_rejects_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here (and d = 0, which launches nothing): a valid one would launch on host memory. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  bufs = [(ctypes.c_float * 64)() for _ in range(3)]
  a, b, c = (ctypes.addressof(x) for x in bufs)
  table = lambda *p: (ctypes.c_void_p * len(p))(*p)
  def call(rows=None, n=2, d=64, mode=1, mom=None, server=None, honest=None):
    return lib.bz_gradient_momentum(table(a, a) if rows is None else rows, n, d, mode, mom, server, 0.9, 1., honest, None)
  assert lib.bz_gradient_momentum(None, 2, 64, 1, table(b, c), None, 0.9, 1., None, None) == -1 and b"rows is NULL" in lib.bz_last_error()
  assert call(d=-1, mom=table(b, c)) == -1
  assert call(n=0, mom=table(b, c)) == -1 and b"n = 0" in lib.bz_last_error()
  assert call(n=65, rows=table(*[a] * 65), mom=table(*[b] * 65)) == -1
  assert call(mode=0, mom=table(b, c)) == -1 and b"mode" in lib.bz_last_error()
  assert call(mode=1) == -1 and b"momentum is NULL" in lib.bz_last_error()
  assert call(mode=2, server=c) == -1 and b"honest is NULL" in lib.bz_last_error()
  assert call(mode=2, honest=table(b, c)) == -1 and b"server is NULL" in lib.bz_last_error()
  assert call(mom=table(b, b)) == -1 and b"same vector" in lib.bz_last_error()
  assert call(mom=table(b, None)) == -1 and b"momentum[1] is NULL" in lib.bz_last_error()
  assert call(rows=table(a, None), mom=table(b, c)) == -1 and b"rows[1] is NULL" in lib.bz_last_error()
  assert call(mode=2, server=c, honest=table(None, b)) == -1 and b"honest[0] is NULL" in lib.bz_last_error()
  assert call(d=0, rows=table(None, None), mom=table(None, None)) == 0      # an empty shard: nothing to do

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_delivery_kernels_do_not_spill():
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout
  found = re.findall(r"Function (\S*k7_(?:scatter|momentum)\S*):\s*\n\s*REG:(\d+) STACK:(\d+)", text)
  assert sum("k7_scatter" in f[0] for f in found) == 1 and sum("k7_momentum" in f[0] for f in found) == 2, found
  for name, regs, stack in found:
    assert int(stack) == 0 and int(regs) <= 64, (name, regs, stack)
