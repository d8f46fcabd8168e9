# coding: utf-8
"""The entry points of `include/byzagg_attack.h` (the attacks' line search): the header declares them,
`byzagg.h` includes it, the library exports them, the third ctypes table of `_lib.py` matches, the
argument checks run before any CUDA call, and the candidate kernel compiles without spilling.  No
compute calls here (CPU suite)."""

import ctypes
import pathlib
import re
import shutil
import subprocess

import pytest

ROOT = pathlib.Path(__file__).resolve().parent.parent
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

def declared_symbols():
  text = (ROOT / "include" / "byzagg_attack.h").read_text()
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", text)))

def test_header_declares_the_search_and_byzagg_h_includes_it():
  assert declared_symbols() == ["bz_line_search", "bz_line_search_workspace_bytes"]
  main = (ROOT / "include" / "byzagg.h").read_text()
  assert '#include "byzagg_attack.h"' in main
  assert "byzagg_attack.h" in (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()

def test_library_exports_the_search_and_the_table_matches():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.library_path()))
  for name in declared_symbols():
    assert hasattr(handle, name), name
  assert sorted(_lib.ATTACK_SIGNATURES) == declared_symbols()
  assert not set(_lib.ATTACK_SIGNATURES) & (set(_lib.SIGNATURES) | set(_lib.SHARD_SIGNATURES))
  for name in declared_symbols():
    assert getattr(_lib.lib(), name).argtypes == _lib.ATTACK_SIGNATURES[name][1]
  lib = _lib.lib()
  # the rule's workspace, then two 64 x 64 distance tables and the search state
  assert lib.bz_line_search_workspace_bytes(25) >= lib.bz_workspace_bytes(25) + 2 * 64 * 64 * 8
  assert lib.bz_line_search_workspace_bytes(25) % 256 == 0

def test_line_search_rejects_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here: a valid one would launch on host memory. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  bufs = [(ctypes.c_float * 64)() for _ in range(5)]
  h, avg, att, byz, out = (ctypes.addressof(b) for b in bufs)
  trace = ctypes.addressof((ctypes.c_double * 64)())
  status = ctypes.addressof((ctypes.c_int32 * 2)())
  ws_buf = (ctypes.c_double * 8)()                  # far too small for any n
  ws = ctypes.addressof(ws_buf)
  def call(rule=5, honest=None, nh=20, f_real=5, f_decl=5, kind=0, avg=avg, att=att, d=64, evals=16, byz=byz, out=out,
           trace=trace, status=status, ws=ws, ws_bytes=1 << 40):
    rows = (ctypes.c_void_p * max(nh, 1))(*([h] * max(nh, 1))) if honest is None else honest
    return lib.bz_line_search(rule, rows, nh, f_real, f_decl, kind, 0, avg, att, d, evals, byz, out, trace, status,
                              ws, ws_bytes, None)
  err = lib.bz_last_error
  assert lib.bz_line_search(5, None, 20, 5, 5, 0, 0, avg, att, 64, 16, byz, out, trace, status, ws, 1 << 40, None) == -1
  assert b"honest is NULL" in err()
  assert call(nh=0) == -1 and call(f_real=0) == -1 and b"f_real" in err()
  assert call(nh=60) == -2 and b"BZ_MAX_N" in err()
  assert call(d=0) == -1 and b"d = 0" in err()
  assert call(evals=0) == -1 and b"evals" in err()
  assert call(kind=2) == -1 and b"kind" in err()
  for what in ("avg", "byz", "out", "trace", "status"):
    assert call(**{what: None}) == -1 and b"NULL" in err(), what
  assert call(att=None) == -1
  assert call(byz=avg) == -1 and b"distinct" in err()
  assert call(honest=(ctypes.c_void_p * 20)(*([h] * 19 + [byz]))) == -1 and b"honest[19]" in err()
  assert call(honest=(ctypes.c_void_p * 20)(*([h] * 19 + [None]))) == -1 and b"rows[19] is NULL" in err()
  assert call(rule=10) == -1 and b"unknown rule" in err()
  assert call(rule=2, f_decl=13) == -1                   # trmean: n - 2f < 1
  assert call(rule=6, f_decl=6) == -1 and b"4f + 3" in err()   # bulyan needs n >= 4f + 3
  assert call(rule=7, nh=40, f_real=10, f_decl=20) == -2 and b"subsets" in err()
  assert call(ws_bytes=64) == -4 and b"workspace" in err()
  assert call(ws=None) == -4
  assert call(kind=1, att=None, ws_bytes=64) == -4       # empire-strict reads no direction: got to the workspace check

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_candidate_and_score_kernels_do_not_spill():
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout
  found = re.findall(r"Function (\S*k8_candidate\S*):\s*\n\s*REG:(\d+) STACK:(\d+)", text)
  assert len(found) == 2, found                          # VEC = 4 and the scalar variant
  for name, regs, stack in found:
    assert int(stack) == 0 and int(regs) <= 32, (name, regs, stack)
  score = re.findall(r"Function (\S*k2_rowdist\S*Lb0ELb1E\S*):\s*\n\s*REG:(\d+) STACK:(\d+)", text)
  assert len(score) == 2, score                          # the SEARCH variants of K2'
  for name, regs, stack in score:
    assert int(regs) <= 128, (name, regs, stack)         # two 256-thread CTAs per SM, as K2'
