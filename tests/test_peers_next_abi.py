# coding: utf-8
"""The entry points of `include/byzagg_peers_next.h` (the exchanges over peer memory with the epoch taken from
the exchange buffer): the header declares them, `byzagg.h` includes it, the library exports them, their
ctypes table in `_lib.py` matches and is loaded, and every argument check — rank, both slots' tables, the
status word, alignment — returns its code and message before any CUDA call.  No compute calls here (CPU
suite)."""

import ctypes
import pathlib
import re
import shutil
import subprocess

import pytest

ROOT = pathlib.Path(__file__).resolve().parent.parent
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
NAMES = ["bz_bulyan_peers_next", "bz_krum_peers_next", "bz_pairdist_reuse_peers_next", "bz_rowdist_peers_next",
         "bz_search_score_peers_next"]
KRUM, BULYAN, BRUTE, AKSEL, CGE = 5, 6, 7, 8, 9

def declared_symbols(header):
  text = (ROOT / "include" / header).read_text()
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", text)))

def test_header_declares_the_entry_points_and_byzagg_h_includes_it():
  assert declared_symbols("byzagg_peers_next.h") == NAMES
  main = (ROOT / "include" / "byzagg.h").read_text()
  assert '#include "byzagg_peers_next.h"' in main
  assert main.index('#include "byzagg_peers_next.h"') > main.index('#include "byzagg_coordinate.h"')     # at the end
  assert "byzagg_peers_next.h" in (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  for header in ("byzagg.h", "byzagg_search_peers.h"):
    assert not set(NAMES) & set(declared_symbols(header))

def test_library_exports_them_and_the_table_matches():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.library_path()))
  for name in NAMES:
    assert hasattr(handle, name), name
  assert sorted(_lib.PEER_NEXT_SIGNATURES) == NAMES
  others = (set(_lib.SIGNATURES) | set(_lib.SHARD_SIGNATURES) | set(_lib.ATTACK_SIGNATURES) | set(_lib.SEARCH_SHARD_SIGNATURES)
            | set(_lib.SEARCH_PEER_SIGNATURES) | set(_lib.COORDINATE_SIGNATURES))
  assert not set(_lib.PEER_NEXT_SIGNATURES) & others
  for name in NAMES:
    assert getattr(_lib.lib(), name).argtypes == _lib.PEER_NEXT_SIGNATURES[name][1]
  # each is its by-value twin without the epoch
  twins = dict(_lib.SIGNATURES, **_lib.SEARCH_PEER_SIGNATURES)
  for name in NAMES:
    args = list(twins[name[:-len("_next")]][1])
    args.remove(ctypes.c_uint)
    assert _lib.PEER_NEXT_SIGNATURES[name][1] == args, name

class _Host:
  """ Host buffers standing in for device pointers: only invalid calls are made, which return before any
  CUDA call.  Two ranks: the tables hold 2 * 2 pointers, slot 0's then slot 1's. """
  def __init__(self):
    self.buf = (ctypes.c_double * 512)()
    self.p = ctypes.addressof(self.buf)
    self.rows = (ctypes.c_void_p * 25)(*([self.p] * 25))
    self.blocks = (ctypes.c_void_p * 4)(self.p, self.p + 64, self.p + 1536, self.p + 1600)
    self.flags = (ctypes.c_void_p * 4)(self.p + 128, self.p + 192, self.p + 1664, self.p + 1728)
    self.mode = ctypes.c_int(7)
  def tables(self, which, index, value):
    """ A copy of the blocks ("blocks") or flags ("flags") table with entry `index` replaced. """
    table = list(getattr(self, which))
    table[index] = value
    return (ctypes.c_void_p * 4)(*table)

def _check_exchange_arguments(call, err, h, name, status_message=b"NULL peer table or status"):
  """ The checks every _next call shares: rank, both slots' tables, the status word (the score's checks it with
  the trace, before the tables, as its by-value twin does). """
  p = h.p
  assert call(rank=0, nranks=0) == -1 and b"rank 0 of 0" in err()
  assert call(rank=0, nranks=17) == -1 and b"rank 0 of 17" in err()
  assert call(rank=2) == -1 and b"rank 2 of 2" in err()
  assert call(rank=-1) == -1 and b"rank -1 of 2" in err()
  assert call(blocks=None) == -1 and b"NULL peer table or status" in err()
  assert call(flags=None) == -1 and b"NULL peer table or status" in err()
  assert call(status=None) == -1 and status_message in err()
  assert call(blocks=h.tables("blocks", 1, None)) == -1 and b"peer 1: NULL or misaligned" in err()
  assert call(blocks=h.tables("blocks", 0, p + 4)) == -1 and b"peer 0: NULL or misaligned" in err()
  assert call(flags=h.tables("flags", 1, p + 2)) == -1 and b"peer 1: NULL or misaligned" in err()
  # slot 1's entries are checked too, and named
  for which, index, value, peer in (("blocks", 2, None, 0), ("blocks", 3, p + 4, 1), ("flags", 2, p + 1, 0), ("flags", 3, None, 1)):
    assert call(**{which: h.tables(which, index, value)}) == -1, (name, which, index)
    message = err()
    assert name.encode() in message and b"(slot 1)" in message and f"peer {peer}: NULL or misaligned".encode() in message, message

def test_krum_and_bulyan_peers_next_reject_bad_arguments():
  from byzantinemomentum_b200 import _lib
  lib, h = _lib.lib(), _Host()
  err = lib.bz_last_error
  p = h.p
  for name, m in (("bz_krum_peers_next", 18), ("bz_bulyan_peers_next", 1)):
    fn = getattr(lib, name)
    def call(rows=h.rows, n=25, f=5, m=m, d=64, out=p + 512, order=p, status=p + 256, rank=0, nranks=2, blocks=h.blocks,
             flags=h.flags, ws=p, ws_bytes=64):
      return fn(rows, n, f, m, d, out, order, status, rank, nranks, blocks, flags, ws, ws_bytes, None)
    _check_exchange_arguments(call, err, h, name)
    assert call(rows=None) == -1 and b"rows is NULL" in err()
    assert call(n=65) == -2 and b"BZ_MAX_N" in err()
    assert call(d=-1) == -1 and b"d = -1" in err()
    assert call(f=24) == -1 and b"f = 24 not executable" in err()
    assert call() == -4 and b"workspace" in err()                           # reached the workspace check: nothing launched

def test_pairdist_reuse_peers_next_rejects_bad_arguments():
  from byzantinemomentum_b200 import _lib
  lib, h = _lib.lib(), _Host()
  err = lib.bz_last_error
  p = h.p
  def call(rule=KRUM, rows=h.rows, n=25, f=5, m=18, d=64, out=p + 512, order=p, status=p + 256, cache_in=None, u_old=0,
           cache_out=p + 1024, mode_out=ctypes.byref(h.mode), rank=0, nranks=2, blocks=h.blocks, flags=h.flags, ws=p, ws_bytes=64):
    return lib.bz_pairdist_reuse_peers_next(rule, rows, n, f, m, d, out, order, status, None, cache_in, u_old, cache_out, mode_out,
                                            rank, nranks, blocks, flags, ws, ws_bytes, None)
  _check_exchange_arguments(call, err, h, "bz_pairdist_reuse_peers_next")
  assert call(rule=AKSEL) == -1 and b"BZ_RULE_KRUM" in err()
  assert call(n=65) == -2 and b"BZ_MAX_N" in err()
  assert call(cache_out=None) == -1 and b"cache_out / mode_out is NULL" in err()
  assert call(cache_in=p + 1024) == -1 and b"must differ" in err()
  assert call(cache_in=p + 2048, u_old=65) == -1 and b"u_old = 65" in err()
  unaligned = (ctypes.c_void_p * 25)(*([p] * 24 + [p + 4]))
  assert call(rows=unaligned) == -1 and b"rows[24] is not 16-byte aligned" in err()
  assert call(rows=unaligned, d=0) == -4                                    # an empty shard reads no row
  assert call(rule=BULYAN, f=6, m=1) == -1 and b"n >= 4f + 3" in err()
  assert call() == -4 and b"workspace" in err()
  assert call(rule=BRUTE, m=-7) == -4
  assert h.mode.value == -1

def test_rowdist_peers_next_rejects_bad_arguments():
  from byzantinemomentum_b200 import _lib
  lib, h = _lib.lib(), _Host()
  err = lib.bz_last_error
  p = h.p
  def call(rule=AKSEL, rows=h.rows, n=25, f=5, mode=0, center=p + 1024, d=64, out=p + 512, order=p, status=p + 256, rank=1,
           nranks=2, blocks=h.blocks, flags=h.flags, ws=p, ws_bytes=64):
    return lib.bz_rowdist_peers_next(rule, rows, n, f, mode, center, d, out, order, status, rank, nranks, blocks, flags, ws, ws_bytes, None)
  _check_exchange_arguments(call, err, h, "bz_rowdist_peers_next")
  assert call(rule=KRUM) == -1 and b"BZ_RULE_AKSEL" in err()
  assert call(n=65) == -2 and b"BZ_MAX_N" in err()
  assert call(mode=2) == -1 and b"mode = 2" in err()
  assert call(center=p + 2) == -1 and b"center" in err()                   # aksel's centre: 4-byte aligned
  assert call(rule=CGE) == -1 and b"cge takes no center" in err()
  assert call(rule=CGE, center=None) == -4 and b"workspace" in err()
  assert call() == -4 and b"workspace" in err()
  assert call(d=0, center=None) == -4

def test_search_score_peers_next_rejects_bad_arguments():
  from byzantinemomentum_b200 import _lib
  lib, h = _lib.lib(), _Host()
  err = lib.bz_last_error
  p = h.p
  def call(out=p, avg=p + 8, d=64, state=p + 64, trace=p + 128, status=p + 256, k=0, evals=16, rank=0, nranks=2,
           blocks=h.blocks, flags=h.flags, ws=p, ws_bytes=64):
    return lib.bz_search_score_peers_next(out, avg, d, state, trace, None, status, k, evals, rank, nranks, blocks, flags, ws, ws_bytes, None)
  _check_exchange_arguments(call, err, h, "bz_search_score_peers_next", status_message=b"trace or status is NULL")
  assert call(d=-1) == -1 and b"d = -1" in err()
  assert call(state=p + 4) == -1 and b"aligned" in err()
  assert call(k=16) == -1 and call(evals=0) == -1 and b"evals" in err()
  assert call(out=None) == -1 and b"out or avg is NULL" in err()
  assert call(avg=p + 2) == -1 and b"4-byte aligned" in err()                # alignment of the vectors
  assert call() == -4 and b"workspace" in err()
  assert call(d=0, out=None, avg=None) == -4

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_the_next_mode_adds_no_kernel():
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout
  assert len(re.findall(r"Function (\S*k2_rowdist_peers\S*):", text)) == 6       # a runtime flag in the tail, no instantiation
  assert len(re.findall(r"Function (\S*k2_ring\S*):", text)) == 8
