# coding: utf-8
"""The d-sharded phases of Multi-Krum, Bulyan, Aksel and CGE up to 128 rows (include/byzagg_distance_shards.h) on
the CPU: the header and its binding, the argument checks (before any CUDA call, with fake pointers), the register
and stack budgets of the kernels they add, and the exchange `ShardedPlan` resolves above and below 64 rows.  No
compute calls here."""

import ctypes
import pathlib
import re
import shutil
import subprocess

import pytest

ROOT = pathlib.Path(__file__).resolve().parent.parent
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
NAMES = ["bz_distance_partial", "bz_distance_reduce", "bz_distance_select"]
KRUM, BULYAN, BRUTE, AKSEL, CGE = 5, 6, 7, 8, 9
NEW_KERNELS = ("k2_pairshare_wide", "k2_rowshare_wide", "k5_blocks_select_wide", "k5_rowkeys_select_wide")

def declared_symbols(header):
  text = (ROOT / "include" / header).read_text()
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", text)))

def test_header_declares_the_phases_and_byzagg_h_includes_it():
  assert declared_symbols("byzagg_distance_shards.h") == NAMES
  main = (ROOT / "include" / "byzagg.h").read_text()
  assert '#include "byzagg_distance_shards.h"' in main
  assert main.index('#include "byzagg_distance_shards.h"') > main.index('#include "byzagg_distance.h"')     # at the end
  assert "byzagg_distance_shards.h" in (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  for header in ("byzagg.h", "byzagg_distance.h"):
    assert not set(NAMES) & set(declared_symbols(header))

def test_library_exports_them_and_the_table_is_disjoint():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.library_path()))
  for name in NAMES:
    assert hasattr(handle, name), name
  assert sorted(_lib.DISTANCE_SHARD_SIGNATURES) == NAMES
  others = [_lib.SIGNATURES, _lib.SHARD_SIGNATURES, _lib.ATTACK_SIGNATURES, _lib.SEARCH_SHARD_SIGNATURES,
            _lib.SEARCH_PEER_SIGNATURES, _lib.COORDINATE_SIGNATURES, _lib.PEER_NEXT_SIGNATURES, _lib.DISTANCE_SIGNATURES]
  for table in others:
    assert not set(_lib.DISTANCE_SHARD_SIGNATURES) & set(table)
  for name, (restype, argtypes) in _lib.DISTANCE_SHARD_SIGNATURES.items():
    assert getattr(_lib.lib(), name).argtypes == argtypes

def _fakes():
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  rows = lambda n, address=0x1000: (ctypes.c_void_p * max(n, 1))(*[address + 0x100 * i for i in range(max(n, 1))])
  message = lambda: lib.bz_last_error().decode()
  return lib, rows, message

def test_partial_rejects_bad_arguments_before_touching_the_gpu():
  lib, rows, message = _fakes()
  part, center = ctypes.c_void_p(0x90000), ctypes.c_void_p(0xa0000)
  big = 1 << 40
  def call(rule=KRUM, table=None, n=100, c=center, d=16, dest=part, ws=0xc0000, ws_bytes=big):
    return lib.bz_distance_partial(rule, rows(n) if table is None else table, n, c, d, dest, ctypes.c_void_p(ws), ws_bytes, None)
  assert call(n=0) == -1 and "n = 0" in message()
  assert call(n=129) == -2 and "BZ_MAX_N_DISTANCE = 128" in message()
  for rule in (0, 4, 10, -1):
    assert call(rule=rule) == -1 and "unknown rule" in message(), rule
  assert call(rule=BRUTE, n=65) == -2 and "brute" in message()
  assert call(rule=BRUTE, n=128, d=0) == -2
  assert lib.bz_distance_partial(KRUM, None, 100, None, 16, part, ctypes.c_void_p(0xc0000), big, None) == -1 and "rows is NULL" in message()
  assert call(dest=None) == -1 and "output" in message()
  assert call(dest=None, d=0) == -1 and "part is NULL" in message()
  assert call(table=rows(100, address=0x1002)) == -1 and "aligned" in message()
  assert call(rule=AKSEL, c=None) == -1 and "center" in message()
  # the workspace: bz_distance_workspace_bytes(n), 8-byte aligned, at every n
  for n in (25, 64, 65, 100, 128):
    need = lib.bz_distance_workspace_bytes(n)
    for rule in (KRUM, BULYAN, AKSEL, CGE):
      assert call(rule=rule, n=n, ws_bytes=need - 1) == -4 and "workspace" in message(), (rule, n)
      assert call(rule=rule, n=n, ws=0xc0004) == -4 and "misaligned" in message(), (rule, n)
      assert call(rule=rule, n=n, ws=0) == -4, (rule, n)

def test_select_rejects_bad_arguments_before_touching_the_gpu():
  lib, _, message = _fakes()
  parts, order, status = ctypes.c_void_p(0x90000), ctypes.c_void_p(0xa0000), ctypes.c_void_p(0xb0000)
  def call(rule=KRUM, p=parts, nparts=2, n=100, f=10, m=20, mode=0, o=order):
    return lib.bz_distance_select(rule, p, nparts, n, f, m, mode, o, status, None)
  assert call(n=0) == -1 and "n = 0" in message()
  assert call(n=129) == -2 and "BZ_MAX_N_DISTANCE = 128" in message()
  assert call(rule=3) == -1 and "unknown rule" in message()
  assert call(rule=BRUTE, n=65) == -2 and "brute" in message()
  assert call(p=None) == -1 and "parts / order is NULL" in message()
  assert call(o=None) == -1 and "parts / order is NULL" in message()
  for nparts in (0, -1):
    assert call(nparts=nparts) == -1 and f"nparts = {nparts}" in message()
  for n in (64, 100):
    assert call(n=n, f=n - 1) == -1 and "n - f - 1" in message(), n
    assert call(n=n, m=0) == -1 and "m = 0" in message(), n
    assert call(n=n, m=n + 1) == -1 and f"expected 1..{n}" in message(), n
    assert call(rule=BULYAN, n=n, f=n // 4) == -1 and "4f + 3" in message(), n
    assert call(rule=BULYAN, n=n, f=5, m=n - 6) == -1 and f"expected 1..{n - 7}" in message(), n
    assert call(rule=AKSEL, n=n, mode=2) == -1 and "mode = 2" in message(), n
    assert call(rule=AKSEL, n=n, mode=1, f=n) == -1 and "not executable" in message(), n

def test_reduce_rejects_bad_arguments_and_d_0_is_a_no_op():
  lib, rows, message = _fakes()
  out, order, status = ctypes.c_void_p(0x90000), ctypes.c_void_p(0xa0000), ctypes.c_void_p(0xb0000)
  def call(rule=KRUM, table=None, n=100, f=10, m=20, mode=0, o=order, d=16, dest=out):
    return lib.bz_distance_reduce(rule, rows(n) if table is None else table, n, f, m, mode, o, status, d, dest, None)
  assert call(n=0) == -1 and "n = 0" in message()
  assert call(n=129) == -2 and "BZ_MAX_N_DISTANCE = 128" in message()
  assert call(rule=11) == -1 and "unknown rule" in message()
  assert call(rule=BRUTE, n=65, f=1) == -2 and "brute" in message()
  assert call(o=None) == -1 and "order is NULL" in message()
  assert call(dest=None) == -1 and "output" in message()
  assert call(table=rows(100, address=0x1002)) == -1 and "aligned" in message()
  assert call(f=99) == -1 and "n - f - 1" in message()
  assert call(m=101) == -1 and "expected 1..100" in message()
  assert call(rule=BULYAN, f=25) == -1 and "4f + 3" in message()
  assert call(rule=BULYAN, f=24, m=75) == -1 and "expected 1..74" in message()
  assert call(rule=AKSEL, mode=5) == -1 and "mode = 5" in message()
  # d = 0 launches nothing, for every rule at every n (the pointers are fake)
  for n in (7, 64, 65, 128):
    f = (n - 3) // 4
    for rule in (KRUM, BULYAN, AKSEL, CGE) + ((BRUTE,) if n <= 64 else ()):
      assert call(rule=rule, n=n, f=f, m=1, d=0, dest=None) == 0, (rule, n)
  assert call(rule=CGE, f=200, d=0) == 0        # CGE checks no f (cge.py does not either)

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_new_kernels_fit_the_register_budget():
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout
  usage = {name: (int(regs), int(stack)) for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text)}
  counts = {kernel: [name for name in usage if kernel in name] for kernel in NEW_KERNELS}
  assert {kernel: len(names) for kernel, names in counts.items()} == {
    "k2_pairshare_wide": 1, "k2_rowshare_wide": 2, "k5_blocks_select_wide": 1, "k5_rowkeys_select_wide": 1}
  for names in counts.values():
    for name in names:
      regs, stack = usage[name]
      assert regs <= 255 and stack == 0, (name, regs, stack)

def test_exchange_above_and_below_64_rows():
  pytest.importorskip("torch")
  from byzantinemomentum_b200 import sharded
  for exchange in ("auto", "nccl", "p2p", "fused"):
    for n in (1, 25, 64):
      assert sharded.rows_exchange(exchange, n) == exchange, (exchange, n)
  for n in (65, 100, 128):
    assert sharded.rows_exchange("auto", n) == "nccl"
    assert sharded.rows_exchange("nccl", n) == "nccl"
    for exchange in ("p2p", "fused"):
      with pytest.raises(ValueError, match=f"at most MAX_N = 64 rows, not n = {n}"):
        sharded.rows_exchange(exchange, n)
  with pytest.raises(ValueError, match="unknown exchange"):
    sharded.rows_exchange("nvlink", 100)
