# coding: utf-8
"""The entry points of `include/byzagg_search_shards.h` (the line search on a d-sharded trainer): the
header declares them, `byzagg.h` includes it, the library exports them, the fourth ctypes table of
`_lib.py` matches, the argument checks reject bad input before any CUDA call, and the new kernels compile
without spilling.  No compute calls here (CPU suite)."""

import ctypes
import pathlib
import re
import shutil
import subprocess

import pytest

ROOT = pathlib.Path(__file__).resolve().parent.parent
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
NAMES = ["bz_pairdist_partial_reuse", "bz_search_candidate", "bz_search_score_partial", "bz_search_step"]

def declared_symbols():
  text = (ROOT / "include" / "byzagg_search_shards.h").read_text()
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", text)))

def test_header_declares_the_entry_points_and_byzagg_h_includes_it():
  assert declared_symbols() == NAMES
  assert '#include "byzagg_search_shards.h"' in (ROOT / "include" / "byzagg.h").read_text()
  assert "byzagg_search_shards.h" in (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  text = (ROOT / "include" / "byzagg_search_shards.h").read_text()
  from byzantinemomentum_b200 import _lib
  assert f"#define BZ_SEARCH_STATE_BYTES {_lib.SEARCH_STATE_BYTES}" in text
  for name, value in (("FIRST", _lib.CANDIDATE_FIRST), ("NEXT", _lib.CANDIDATE_NEXT), ("FINAL", _lib.CANDIDATE_FINAL)):
    assert re.search(rf"#define BZ_CANDIDATE_{name}\s+{value}\b", text), name

def test_library_exports_them_and_the_table_matches():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.library_path()))
  for name in NAMES:
    assert hasattr(handle, name), name
  assert sorted(_lib.SEARCH_SHARD_SIGNATURES) == NAMES
  others = set(_lib.SIGNATURES) | set(_lib.SHARD_SIGNATURES) | set(_lib.ATTACK_SIGNATURES)
  assert not set(_lib.SEARCH_SHARD_SIGNATURES) & others
  for name in NAMES:
    assert getattr(_lib.lib(), name).argtypes == _lib.SEARCH_SHARD_SIGNATURES[name][1]

def test_bad_arguments_are_rejected_before_touching_the_gpu():
  """ Only invalid calls here: a valid one would launch on host memory. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  err = lib.bz_last_error
  buf = (ctypes.c_double * 64)()
  p = ctypes.addressof(buf)
  small = (ctypes.c_double * 8)()
  ws = ctypes.addressof(small)
  rows = (ctypes.c_void_p * 25)(*([p] * 25))
  mode = ctypes.c_int(7)
  def phase_a(rows=rows, n=25, d=64, part=p, cache_in=None, u_old=0, cache_out=p + 256, mode_out=ctypes.byref(mode), ws=ws, ws_bytes=64):
    return lib.bz_pairdist_partial_reuse(rows, n, d, part, None, cache_in, u_old, cache_out, mode_out, ws, ws_bytes, None)
  assert phase_a(rows=None) == -1 and b"rows is NULL" in err()
  assert phase_a(n=65) == -2 and b"BZ_MAX_N" in err()
  assert phase_a(d=-1) == -1
  assert phase_a(part=None) == -1
  assert phase_a(cache_out=None) == -1 and b"cache_out" in err()
  assert phase_a(mode_out=None) == -1
  assert phase_a(cache_in=p + 256) == -1 and b"differ" in err()
  assert phase_a(cache_in=p + 512, u_old=65) == -1 and b"u_old" in err()
  assert phase_a() == -4 and b"workspace" in err()              # reached the workspace check: nothing launched
  assert mode.value == 7                                         # and nothing written
  def candidate(avg=p, att=p + 8, byz=p + 16, d=64, state=p, which=0, kind=0):
    return lib.bz_search_candidate(avg, att, byz, d, state, which, 0, kind, None)
  assert candidate(d=-1) == -1
  assert candidate(state=None) == -1 and b"state" in err()
  assert candidate(state=p + 4) == -1 and b"aligned" in err()
  assert candidate(which=3) == -1 and b"which" in err()
  assert candidate(kind=2) == -1 and b"kind" in err()
  assert candidate(att=None) == -1 and b"NULL" in err()
  assert candidate(byz=p) == -1 and b"distinct" in err()
  assert candidate(byz=p + 2) == -1 and b"aligned" in err()
  def score(out=p, avg=p + 8, d=64, state=p + 16, partial=p + 24, ws=ws, ws_bytes=64):
    return lib.bz_search_score_partial(out, avg, d, state, partial, ws, ws_bytes, None)
  assert score(d=-1) == -1
  assert score(state=None) == -1
  assert score(partial=None) == -1 and b"partial" in err()
  assert score(out=None) == -1 and b"NULL" in err()
  assert score(avg=p + 2) == -1 and b"aligned" in err()
  assert score() == -4 and b"workspace" in err()
  def step(partials=p, nparts=2, state=p + 64, trace=p + 128, status=p + 256, k=0, evals=16):
    return lib.bz_search_step(partials, nparts, state, trace, None, status, k, evals, None)
  assert step(partials=None) == -1 and step(nparts=0) == -1 and b"nparts" in err()
  assert step(state=None) == -1
  assert step(trace=None) == -1 and step(status=None) == -1
  assert step(k=16) == -1 and step(k=-1) == -1 and step(evals=0) == -1 and b"evals" in err()

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_the_new_kernels_do_not_spill():
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout
  found = re.findall(r"Function (\S*k9_search_step\S*):\s*\n\s*REG:(\d+) STACK:(\d+)", text)
  assert len(found) == 1, found
  for name, regs, stack in found:
    assert int(stack) == 0, (name, regs, stack)
  # the kind-4 tail with reuse lives in the existing ring kernels: still one kernel per shape, within budget
  ring = re.findall(r"Function (\S*k2_ring\S*):\s*\n\s*REG:(\d+) STACK:(\d+)", text)
  assert len(ring) == 8, ring
  for name, regs, _ in ring:
    assert int(regs) <= (128 if "ELi16E" in name else 168), (name, regs)
