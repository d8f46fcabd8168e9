# coding: utf-8
"""The entry points of `include/byzagg_search_peers.h` (the d-sharded line search with its exchanges over
peer memory): the header declares them, `byzagg.h` includes it, the library exports them, their ctypes
table in `_lib.py` matches and is loaded, every argument check returns its code and message before any
CUDA call, and the new K2' kernels compile without spilling.  No compute calls here (CPU suite)."""

import ctypes
import pathlib
import re
import shutil
import subprocess

import pytest

ROOT = pathlib.Path(__file__).resolve().parent.parent
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
NAMES = ["bz_pairdist_reuse_peers", "bz_rowdist_peers", "bz_search_score_peers"]
KRUM, BULYAN, BRUTE, AKSEL, CGE = 5, 6, 7, 8, 9

def declared_symbols(header):
  text = (ROOT / "include" / header).read_text()
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", text)))

def test_header_declares_the_entry_points_and_byzagg_h_includes_it():
  assert declared_symbols("byzagg_search_peers.h") == NAMES
  assert '#include "byzagg_search_peers.h"' in (ROOT / "include" / "byzagg.h").read_text()
  assert "byzagg_search_peers.h" in (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  assert not set(NAMES) & set(declared_symbols("byzagg.h"))

def test_library_exports_them_and_the_table_matches():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.library_path()))
  for name in NAMES:
    assert hasattr(handle, name), name
  assert sorted(_lib.SEARCH_PEER_SIGNATURES) == NAMES
  others = set(_lib.SIGNATURES) | set(_lib.SHARD_SIGNATURES) | set(_lib.ATTACK_SIGNATURES) | set(_lib.SEARCH_SHARD_SIGNATURES)
  assert not set(_lib.SEARCH_PEER_SIGNATURES) & others
  for name in NAMES:
    assert getattr(_lib.lib(), name).argtypes == _lib.SEARCH_PEER_SIGNATURES[name][1]

class _Host:
  """ Host buffers standing in for device pointers: only invalid calls are made, which return before any
  CUDA call. """
  def __init__(self):
    self.buf = (ctypes.c_double * 256)()
    self.p = ctypes.addressof(self.buf)
    self.rows = (ctypes.c_void_p * 25)(*([self.p] * 25))
    self.blocks = (ctypes.c_void_p * 2)(self.p, self.p + 64)
    self.flags = (ctypes.c_void_p * 2)(self.p + 128, self.p + 192)
    self.mode = ctypes.c_int(7)

def test_pairdist_reuse_peers_rejects_bad_arguments():
  from byzantinemomentum_b200 import _lib
  lib, h = _lib.lib(), _Host()
  err = lib.bz_last_error
  p = h.p
  def call(rule=KRUM, rows=h.rows, n=25, f=5, m=18, d=64, out=p + 512, order=p, status=p + 256, cache_in=None, u_old=0,
           cache_out=p + 1024, mode_out=ctypes.byref(h.mode), rank=0, nranks=2, blocks=h.blocks, flags=h.flags, ws=p, ws_bytes=64):
    return lib.bz_pairdist_reuse_peers(rule, rows, n, f, m, d, out, order, status, None, cache_in, u_old, cache_out, mode_out,
                                       rank, nranks, blocks, flags, 1, ws, ws_bytes, None)
  assert call(rule=AKSEL) == -1 and b"BZ_RULE_KRUM" in err()
  assert call(rule=4) == -1 and b"rule 4" in err()
  assert call(rows=None) == -1 and b"rows is NULL" in err()
  assert call(n=65) == -2 and b"BZ_MAX_N" in err()
  assert call(d=-1) == -1 and b"d = -1" in err()
  assert call(out=None) == -1 and b"output pointer is NULL" in err()
  assert call(nranks=0) == -1 and b"rank 0 of 0" in err()
  assert call(nranks=17) == -1 and b"rank 0 of 17" in err()
  assert call(rank=2) == -1 and b"rank 2 of 2" in err()
  assert call(rank=-1) == -1 and b"rank -1 of 2" in err()
  assert call(blocks=None) == -1 and b"NULL peer table or status" in err()
  assert call(flags=None) == -1 and b"NULL peer table or status" in err()
  assert call(status=None) == -1 and b"NULL peer table or status" in err()
  assert call(blocks=(ctypes.c_void_p * 2)(p, None)) == -1 and b"peer 1: NULL or misaligned" in err()
  assert call(blocks=(ctypes.c_void_p * 2)(p, p + 4)) == -1 and b"peer 1: NULL or misaligned" in err()
  assert call(flags=(ctypes.c_void_p * 2)(p + 2, p)) == -1 and b"peer 0: NULL or misaligned" in err()
  assert call(cache_out=None) == -1 and b"cache_out / mode_out is NULL" in err()
  assert call(mode_out=None) == -1 and b"cache_out / mode_out is NULL" in err()
  assert call(cache_in=p + 1024) == -1 and b"must differ" in err()
  assert call(cache_in=p + 2048, u_old=0) == -1 and b"u_old = 0" in err()
  assert call(cache_in=p + 2048, u_old=65) == -1 and b"u_old = 65" in err()
  unaligned = (ctypes.c_void_p * 25)(*([p] * 24 + [p + 4]))
  assert call(rows=unaligned) == -1 and b"rows[24] is not 16-byte aligned" in err()
  assert call(f=24) == -1 and b"f = 24 not executable" in err()           # the rule's own checks
  assert call(m=26) == -1 and b"m = 26" in err()
  assert call(rule=BULYAN, f=6, m=1) == -1 and b"n >= 4f + 3" in err()
  assert call() == -4 and b"workspace" in err()                            # reached the workspace check: nothing launched
  assert call(rule=BRUTE, m=-7) == -4                                        # brute ignores m
  assert h.mode.value == -1                                                  # reset before the rule's checks, as bz_krum_reuse

def test_rowdist_peers_rejects_bad_arguments():
  from byzantinemomentum_b200 import _lib
  lib, h = _lib.lib(), _Host()
  err = lib.bz_last_error
  p = h.p
  def call(rule=AKSEL, rows=h.rows, n=25, f=5, mode=0, center=p + 1024, d=64, out=p + 512, order=p, status=p + 256, rank=1,
           nranks=2, blocks=h.blocks, flags=h.flags, ws=p, ws_bytes=64):
    return lib.bz_rowdist_peers(rule, rows, n, f, mode, center, d, out, order, status, rank, nranks, blocks, flags, 3, ws, ws_bytes, None)
  assert call(rule=KRUM) == -1 and b"BZ_RULE_AKSEL" in err()
  assert call(rows=None) == -1 and b"rows is NULL" in err()
  assert call(n=65) == -2 and b"BZ_MAX_N" in err()
  assert call(n=0) == -1
  assert call(d=-1) == -1
  assert call(rank=2) == -1 and b"rank 2 of 2" in err()
  assert call(nranks=17, rank=0) == -1 and b"of 17" in err()
  assert call(status=None) == -1 and b"NULL peer table or status" in err()
  assert call(flags=(ctypes.c_void_p * 2)(p, None)) == -1 and b"peer 1" in err()
  assert call(mode=2) == -1 and b"mode = 2" in err()
  assert call(mode=1, f=25) == -1 and b"f = 25 not executable" in err()
  assert call(center=None) == -1 and b"center" in err()
  assert call(center=p + 2) == -1 and b"center" in err()
  assert call(rule=CGE) == -1 and b"cge takes no center" in err()
  assert call(rule=CGE, center=None) == -4 and b"workspace" in err()
  assert call() == -4 and b"workspace" in err()
  assert call(d=0, center=None) == -4                                       # an empty shard needs no centre

def test_search_score_peers_rejects_bad_arguments():
  from byzantinemomentum_b200 import _lib
  lib, h = _lib.lib(), _Host()
  err = lib.bz_last_error
  p = h.p
  def call(out=p, avg=p + 8, d=64, state=p + 64, trace=p + 128, status=p + 256, k=0, evals=16, rank=0, nranks=2,
           blocks=h.blocks, flags=h.flags, ws=p, ws_bytes=64):
    return lib.bz_search_score_peers(out, avg, d, state, trace, None, status, k, evals, rank, nranks, blocks, flags, 9, ws, ws_bytes, None)
  assert call(d=-1) == -1 and b"d = -1" in err()
  assert call(state=None) == -1 and b"state" in err()
  assert call(state=p + 4) == -1 and b"aligned" in err()
  assert call(trace=None) == -1 and b"trace or status is NULL" in err()
  assert call(status=None) == -1 and b"trace or status is NULL" in err()
  assert call(k=16) == -1 and call(k=-1) == -1 and call(evals=0) == -1 and b"evals" in err()
  assert call(rank=5) == -1 and b"rank 5 of 2" in err()
  assert call(blocks=None) == -1 and b"NULL peer table" in err()
  assert call(out=None) == -1 and b"out or avg is NULL" in err()
  assert call(avg=p + 2) == -1 and b"4-byte aligned" in err()
  assert call() == -4 and b"workspace" in err()
  assert call(d=0, out=None, avg=None) == -4                                # an empty shard needs no vectors

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_the_new_kernels_do_not_spill():
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout
  found = re.findall(r"Function (\S*k2_rowdist_peers\S*):\s*\n\s*REG:(\d+) STACK:(\d+)", text)
  assert len(found) == 6, found                                    # CENTER x VEC for the rowdist mode, VEC for the score
  for name, regs, stack in found:
    assert int(regs) <= 128 and int(stack) <= 32, (name, regs, stack)   # two CTAs of 256 threads per SM, as the plain K2'
  ring = re.findall(r"Function (\S*k2_ring\S*):", text)
  assert len(ring) == 8, ring                                       # the exchange with reuse adds no ring kernel
