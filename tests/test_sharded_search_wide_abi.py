# coding: utf-8
"""The d-sharded line search against Multi-Krum, Bulyan, Aksel and CGE above 64 rows on the CPU
(`ShardedLineSearch(..., wide=True)`, include/byzagg_distance_search_shards.h):
  * the header, its ctypes table and the library's exports; the size of the pass tables;
  * every argument check of `bz_distance_partial_reuse`, before any CUDA call, with host addresses;
  * the row limits with `wide` and without it (unchanged), and their messages;
  * the exchange above 64 rows under `gloo` with 2 ranks: "auto" is "nccl", an explicit "fused" takes rows of any
    alignment, and both ranks agree;
  * the fused search on a stand-in: 2 epochs per evaluation above 64 rows;
  * two `gloo` ranks taking the same factor above 64 rows on the NumPy stand-in of tests/test_sharded_search_gloo.py;
  * the third library, libbyzagg_star.so (include/byzagg_rowshare_star.h): its header, Makefile line, table, exports
    (`nm`, `readelf`), its kernel's register and stack budget (`cuobjdump`), its workspace size and every argument
    check of `bz_rowshare_star`, with fake addresses.
No compute calls on the device here."""

import ctypes
import os
import pathlib
import re
import socket

import numpy as np
import pytest

torch = pytest.importorskip("torch")

ROOT = pathlib.Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "byzagg_distance_search_shards.h"
NAMES = ["bz_distance_partial_reuse", "bz_distance_pass_tables_bytes"]
KRUM, BULYAN, BRUTE, AKSEL, CGE = 5, 6, 7, 8, 9

def declared(path):
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", path.read_text())))

def test_header_declares_the_calls_and_byzagg_h_leaves_them_out():
  assert declared(HEADER) == NAMES
  for other in (ROOT / "include").glob("byzagg*.h"):
    if other != HEADER:
      assert "byzagg_distance_search_shards.h" not in other.read_text(), other.name
      assert not set(declared(other)) & set(NAMES), other.name
  makefile = (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  assert "../../include/byzagg_distance_search_shards.h" in makefile and "api_distance_search_shards.inc" in makefile

def test_library_exports_the_calls_and_the_table_is_its_own():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.library_path()))
  for name in NAMES:
    assert hasattr(handle, name), name
  assert sorted(_lib.DISTANCE_SEARCH_SHARD_SIGNATURES) == NAMES
  others = [_lib.SIGNATURES, _lib.SHARD_SIGNATURES, _lib.ATTACK_SIGNATURES, _lib.SEARCH_SHARD_SIGNATURES,
            _lib.SEARCH_PEER_SIGNATURES, _lib.COORDINATE_SIGNATURES, _lib.PEER_NEXT_SIGNATURES, _lib.DISTANCE_SIGNATURES,
            _lib.DISTANCE_SHARD_SIGNATURES, _lib.ANTICGE_SIGNATURES, _lib.ANTICGE_PEER_SIGNATURES,
            _lib.DISTANCE_SEARCH_SIGNATURES, _lib.DISTANCE_PEER_SIGNATURES]
  assert not set(_lib.DISTANCE_SEARCH_SHARD_SIGNATURES) & set().union(*others)
  for name, (restype, argtypes) in _lib.DISTANCE_SEARCH_SHARD_SIGNATURES.items():
    fn = getattr(_lib.lib(), name)
    assert fn.argtypes == argtypes and fn.restype == restype

def test_pass_tables_are_bz_distance_s():
  """ 6 passes of 64 x 64 doubles: the tables bz_distance keeps behind the 64-row workspace. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  size = lib.bz_distance_pass_tables_bytes()
  assert size == 6 * 64 * 64 * 8
  assert lib.bz_distance_workspace_bytes(100) == lib.bz_workspace_bytes(64) + size

def test_partial_reuse_rejects_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here: a valid one would launch on host memory. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  rows_buf = (ctypes.c_float * 64)()
  h = ctypes.addressof(rows_buf)
  part = ctypes.addressof((ctypes.c_double * 64)())
  tables = ctypes.addressof((ctypes.c_double * 64)())
  ws = ctypes.addressof((ctypes.c_double * 8)())
  mode = ctypes.c_int(-9)
  def call(rule=KRUM, n=100, rows=None, d=64, part=part, old_index=None, tables_in=tables, u_old=91, tables_out=tables,
           mode_out=ctypes.byref(mode), ws=ws, ws_bytes=1 << 40):
    table = (ctypes.c_void_p * max(n, 1))(*([h] * max(n, 1))) if rows is None else rows
    index = (ctypes.c_int32 * max(n, 1))(*(list(range(90)) + [-1] * 10 if n == 100 else [0] * max(n, 1))) if old_index is None else old_index
    return lib.bz_distance_partial_reuse(rule, table, n, d, part, index, tables_in, u_old, tables_out, mode_out, ws, ws_bytes,
                                         None)
  def err():
    return lib.bz_last_error().decode()
  for rule in (0, 4, BRUTE, AKSEL, CGE, 10):
    assert call(rule=rule) == -1 and "BZ_RULE_KRUM or BZ_RULE_BULYAN" in err(), rule
  for n in (1, 25, 64):
    assert call(n=n) == -2 and "bz_pairdist_partial_reuse" in err() and f"n = {n}" in err(), n
  assert call(n=129) == -2 and "BZ_MAX_N_DISTANCE = 128" in err()
  assert call(n=0) == -1 and "n = 0" in err()
  assert lib.bz_distance_partial_reuse(KRUM, None, 100, 64, part, None, None, 0, tables, ctypes.byref(mode), ws, 1 << 40,
                                       None) == -1 and "rows is NULL" in err()
  assert call(rows=(ctypes.c_void_p * 100)(*([h] * 70 + [None] + [h] * 29))) == -1 and "rows[70] is NULL" in err()
  assert call(rows=(ctypes.c_void_p * 100)(*([h] * 70 + [h + 2] + [h] * 29))) == -1 and "rows[70]" in err()
  assert call(d=-1) == -1 and "d = -1" in err()
  assert call(part=None) == -1 and "NULL" in err()
  assert call(tables_out=None) == -1 and "tables_out" in err()
  assert call(tables_out=tables + 4) == -1 and "tables_out" in err()
  assert call(mode_out=None) == -1 and "mode_out" in err()
  assert call(tables_in=tables + 4) == -1 and "tables_in" in err()
  for u_old in (0, 129):
    assert call(u_old=u_old) == -1 and f"u_old = {u_old}" in err(), u_old
  for bad in (-2, 128):
    index = (ctypes.c_int32 * 100)(*([0] * 99 + [bad]))
    assert call(old_index=index) == -1 and f"old_index[99] = {bad}" in err(), bad
  need = lib.bz_distance_workspace_bytes(100)
  assert call(ws_bytes=need - 1) == -4 and "workspace" in err() and str(need) in err()
  assert call(ws=ws + 4) == -4 and call(ws=None) == -4
  assert mode.value == -9                                  # nothing written by a rejected call
  # without previous tables nothing about them is checked
  assert call(tables_in=None, u_old=0, ws=None) == -4

# ---- the row limits -------------------------------------------------------------------------------------------------

def test_search_rows():
  from byzantinemomentum_b200 import engine, sharded
  for gar in ("krum", "bulyan", "aksel", "cge"):
    assert sharded.search_rows(gar) == engine.search_max_rows(gar) == 64
    assert sharded.search_rows(gar, wide=True) == 128
  assert sharded.search_rows("brute") == sharded.search_rows("brute", wide=True) == 64
  for gar in ("average", "median", "trmean", "phocas", "meamed"):
    assert sharded.search_rows(gar) == sharded.search_rows(gar, wide=True) == 128

# a search within the limit on CPU tensors stops at the device: no CUDA device here, or CPU tensors on a GPU machine
_PAST_THE_LIMIT = (ValueError, RuntimeError)

def _rows(nh, d=8):
  return [torch.full((d,), float(i)) for i in range(nh)], torch.zeros(d), torch.ones(d)

@pytest.mark.parametrize("gar", ["krum", "bulyan", "aksel", "cge"])
def test_wide_takes_the_four_rules_to_128_rows(gar):
  """ CPU tensors: a search within the limit gets past it and stops at the device check. """
  from byzantinemomentum_b200 import sharded
  honest, avg, att = _rows(120)
  with pytest.raises(ValueError, match="at most 64 rows"):
    sharded.ShardedLineSearch(gar, honest[:60], 5, 5, avg, att, 4)
  with pytest.raises(ValueError, match="at most 64 rows"):
    sharded.line_search(gar, honest[:60], 5, 5, avg, att, 4)
  with pytest.raises(ValueError, match="at most 128 rows"):
    sharded.ShardedLineSearch(gar, honest, 9, 9, avg, att, 4, wide=True)
  for nh, f_real in ((60, 5), (100, 20), (127, 1)):
    with pytest.raises(_PAST_THE_LIMIT, match="CUDA"):
      sharded.ShardedLineSearch(gar, honest[:nh], f_real, 5, avg, att, 4, wide=True)
  with pytest.raises(_PAST_THE_LIMIT, match="CUDA"):
    sharded.line_search(gar, honest[:100], 20, 5, avg, att, 4, wide=True)

def test_wide_keeps_brute_at_64_and_the_coordinate_rules_at_128():
  from byzantinemomentum_b200 import sharded
  honest, avg, att = _rows(130)
  with pytest.raises(ValueError, match="at most 64 rows"):
    sharded.ShardedLineSearch("brute", honest[:60], 5, 5, avg, att, 4, wide=True)
  for gar in ("average", "median", "trmean", "phocas", "meamed"):
    for wide in (False, True):
      with pytest.raises(ValueError, match="at most 128 rows"):
        sharded.ShardedLineSearch(gar, honest[:120], 9, 9, avg, att, 4, wide=wide)
      with pytest.raises(_PAST_THE_LIMIT, match="CUDA"):
        sharded.ShardedLineSearch(gar, honest[:100], 20, 20, avg, att, 4, wide=wide)

# ---- the exchange above 64 rows -------------------------------------------------------------------------------------

# (facts of rank 0, facts of rank 1, gar, n, exchange, wide) -> what both ranks get; facts: (aligned, symmetric, engine)
ALL = (1, 1, 1)
SCENARIOS = [
  (ALL, ALL, "krum", 100, "auto", True, "nccl"),
  (ALL, ALL, "cge", 128, "auto", True, "nccl"),
  (ALL, ALL, "bulyan", 65, "nccl", True, "nccl"),
  (ALL, ALL, "krum", 100, "fused", True, "fused"),
  ((0, 1, 1), (0, 1, 1), "bulyan", 100, "fused", True, "fused"),       # rows of any alignment above 64
  ((0, 1, 1), ALL, "krum", 100, "auto", True, "nccl"),
  (ALL, (1, 0, 1), "aksel", 100, "fused", True, "raise"),
  ((1, 0, 1), ALL, "krum", 100, "fused", True, "raise"),
  (ALL, ALL, "krum", 64, "auto", True, "fused"),                       # up to 64 rows: choose_search_exchange's
  ((0, 1, 1), ALL, "krum", 64, "fused", True, "raise"),
  (ALL, ALL, "krum", 100, "auto", False, "fused"),                     # without wide: choose_search_exchange's
  ((0, 1, 1), ALL, "krum", 100, "fused", False, "raise"),
]

def _exchange_worker(rank, world, port, queue):
  import sys
  sys.path.insert(0, str(ROOT))
  import torch.distributed as dist
  from byzantinemomentum_b200 import sharded
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    got = []
    for facts0, facts1, gar, n, exchange, wide, _ in SCENARIOS:
      aligned, symmetric, engine = facts0 if rank == 0 else facts1
      try:
        got.append(sharded.search_exchange(gar, n, exchange, aligned, symmetric, engine, wide=wide))
      except ValueError:
        got.append("raise")
    queue.put((rank, got))
  finally:
    dist.destroy_process_group()

def _spawn(target, world=2):
  import torch.multiprocessing as mp
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
  ctx = mp.get_context("spawn")
  queue = ctx.Queue()
  procs = [ctx.Process(target=target, args=(r, world, port, queue)) for r in range(world)]
  for p in procs:
    p.start()
  got = dict(queue.get(timeout=300) for _ in procs)
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  return got

def test_two_ranks_agree_on_the_exchange_above_64_rows():
  got = _spawn(_exchange_worker)
  assert got[0] == got[1] == [want for *_, want in SCENARIOS]

def test_one_rank_exchange_above_64_rows():
  from byzantinemomentum_b200 import sharded
  assert sharded.search_exchange("krum", 100, "auto", True, True, True, wide=True) == "nccl"
  assert sharded.search_exchange("krum", 100, "fused", False, False, True, wide=True) == "fused"
  with pytest.raises(ValueError):
    sharded.search_exchange("brute", 64, "fused", False, True, True, wide=True)
  with pytest.raises(ValueError, match="unknown exchange"):
    sharded.search_exchange("krum", 100, "p2p", True, True, True, wide=True)

class _Recorder:
  """ The fused stages of one rank, recording what they are given. """
  def __init__(self, gar, honest, f_real, f_decl, avg, att, evals, negative, kind, world, wide=False):
    self.device = avg.device
    self.distance, self.wide = True, wide
    self.byz = torch.zeros(avg.numel())
    self.record = torch.zeros(2 * evals + 2, dtype=torch.float64)
    self.calls = []
  def fuse(self, fx):
    self.calls.append(("fuse", fx.n, fx.world, fx.rank))
  def evaluate_fused(self, k, epoch):
    self.calls.append(("rule", k, epoch))
  def score_fused(self, k, epoch):
    self.calls.append(("score", k, epoch))
  def finish(self):
    self.calls.append(("finish",))
    return self.byz

class _Backend:
  def __init__(self):
    self.made = []
  def search_shard(self, *args, **kw):
    self.made.append((len(args), kw))
    return _Recorder(*args, **kw)

@pytest.mark.parametrize("gar", ["krum", "bulyan", "aksel", "cge"])
def test_fused_search_above_64_rows_issues_two_epochs_per_evaluation(gar):
  from byzantinemomentum_b200 import sharded
  nh, f, evals = 90, 10, 5
  for d, start in ((601, 0), (0, 0), (33, 2**32 - 3)):
    honest = [torch.full((d + 1,), float(i))[1:] for i in range(nh)]    # unaligned views
    avg, att = torch.zeros(d), torch.ones(d)
    backend = _Backend()
    assert sharded.ShardedLineSearch(gar, honest, f, f, avg, att, evals, backend=backend, wide=True).exchange == "nccl"
    search = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, evals, backend=backend, exchange="fused", wide=True)
    assert backend.made == [(10, {"wide": True})] * 2
    assert search.exchange == "fused" and search._fx.world == 1 and search._fx.n == nh + f
    search._fx.epoch = start
    search()
    search()
    calls = search._shard.calls
    assert calls[0] == ("fuse", nh + f, 1, 0)
    epochs = [c[2] for c in calls if c[0] in ("rule", "score")]
    assert epochs == list(range(start + 1, start + 1 + 4 * evals)), (gar, d, epochs)
    order = [c[:2] for c in calls[1:]]
    assert order == 2 * ([x for k in range(evals) for x in (("rule", k), ("score", k))] + [("finish",)])

def test_without_wide_the_backend_gets_the_ten_arguments():
  from byzantinemomentum_b200 import sharded
  backend = _Backend()
  honest, avg, att = _rows(20)
  sharded.ShardedLineSearch("krum", honest, 5, 5, avg, att, 3, backend=backend)
  assert backend.made == [(10, {})]

# ---- two ranks on the NumPy stand-in --------------------------------------------------------------------------------

CASES = (("krum", 601, 90, 10), ("bulyan", 601, 60, 10), ("aksel", 601, 80, 20), ("cge", 1, 99, 1))
EVALS = 7

def _inputs(d, nh):
  gen = torch.Generator().manual_seed(d + nh + 3)
  honest = [torch.randn(d, generator=gen) * (0.5 + i / 40.) for i in range(nh)]
  stck = torch.stack(honest)
  return honest, stck.mean(dim=0), stck.var(dim=0).sqrt_()

def _factor_worker(rank, world, port, queue):
  import sys
  sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
  import torch.distributed as dist
  from byzantinemomentum_b200 import sharded
  from fake_backend import OracleBackend
  from test_sharded_search_gloo import _Shard

  class SearchBackend(OracleBackend):
    def search_shard(self, *args, wide=False):
      assert wide
      return _Shard(self, *args)

  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    got = {}
    for gar, d, nh, f in CASES:
      honest, avg, att = _inputs(d, nh)
      lo, hi = sharded.shard_bounds(d, world, rank)
      cut = lambda v: v[lo:hi].contiguous()
      search = sharded.ShardedLineSearch(gar, [cut(g) for g in honest], f, f, cut(avg), cut(att), EVALS, negative=True,
                                         backend=SearchBackend(), wide=True)
      assert search.exchange == "nccl"
      byz = search()
      factor, trace = search.result()
      got[gar] = (factor, trace, byz.numpy().copy())
    queue.put((rank, got))
  finally:
    dist.destroy_process_group()

def test_two_ranks_take_the_same_factor_above_64_rows():
  import sys
  sys.path.insert(0, str(ROOT / "tests"))
  import line_oracle
  got = _spawn(_factor_worker)
  for gar, d, nh, f in CASES:
    (f0, t0, b0), (f1, t1, b1) = got[0][gar], got[1][gar]
    assert f0 == f1 and [(x.hex(), y.hex()) for x, y in t0] == [(x.hex(), y.hex()) for x, y in t1], gar
    ys = [y for _, y in t0]
    xs = []
    want = line_oracle.line_maximize(lambda x: (xs.append(x), ys[len(xs) - 1])[1], EVALS)
    assert [x for x, _ in t0] == xs and f0 == want, gar
    if d == 1:
      assert b1.size == 0                                  # rank 1's shard is empty and it still joined
    honest, avg, att = _inputs(d, nh)
    np.testing.assert_array_equal(np.concatenate([b0, b1]), (avg + f0 * att).numpy())

# ---- libbyzagg_star.so: CGE's candidate-only phase A ------------------------------------------------------------------

import shutil
import subprocess

STAR_HEADER = ROOT / "include" / "byzagg_rowshare_star.h"
STAR_CALLS = ["bz_rowshare_star", "bz_rowshare_star_workspace_bytes"]
STAR_NAMES = sorted(["bz_rowshare_star_last_error"] + STAR_CALLS)

def test_star_header_declares_the_calls_and_byzagg_h_leaves_it_out():
  assert declared(STAR_HEADER) == STAR_NAMES
  for other in (ROOT / "include").glob("byzagg*.h"):
    if other != STAR_HEADER:
      assert "byzagg_rowshare_star.h" not in other.read_text(), other.name
      assert not set(declared(other)) & set(STAR_NAMES), other.name

def test_makefile_builds_the_third_library():
  makefile = (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  assert re.search(r"^all: \$\(OUT\) \$\(PEERS_OUT\)$", makefile, re.M)
  assert re.search(r"^all: \$\(STAR_OUT\)$", makefile, re.M)
  assert "STAR_OUT  := ../libbyzagg_star" in makefile
  assert "STAR_OBJS := $(BUILD)/api_rowshare_star.o $(BUILD)/k2_rowshare_star.o" in makefile
  rule = re.search(r"^\$\(STAR_OUT\): \$\(STAR_OBJS\)\n\t(.*)$", makefile, re.M).group(1)
  assert "-shared" in rule and "-cudart static" in rule and "$(ARCH)" in rule and "$(OBJS)" not in rule
  assert "$(PEERS_OBJS)" not in rule and "-lbyzagg" not in rule and "libbyzagg" not in rule
  assert "../../include/byzagg_rowshare_star.h" in makefile

def test_star_table_is_its_own_and_the_library_exports_it():
  from byzantinemomentum_b200 import _lib
  assert sorted(_lib.ROWSHARE_STAR_SIGNATURES) == STAR_NAMES
  others = [_lib.SIGNATURES, _lib.SHARD_SIGNATURES, _lib.ATTACK_SIGNATURES, _lib.SEARCH_SHARD_SIGNATURES,
            _lib.SEARCH_PEER_SIGNATURES, _lib.COORDINATE_SIGNATURES, _lib.PEER_NEXT_SIGNATURES, _lib.DISTANCE_SIGNATURES,
            _lib.DISTANCE_SHARD_SIGNATURES, _lib.ANTICGE_SIGNATURES, _lib.ANTICGE_PEER_SIGNATURES,
            _lib.DISTANCE_SEARCH_SIGNATURES, _lib.DISTANCE_SEARCH_SHARD_SIGNATURES, _lib.DISTANCE_PEER_SIGNATURES]
  assert not set(_lib.ROWSHARE_STAR_SIGNATURES) & set().union(*others)
  assert _lib.star_library_path() == _lib.library_path().parent / "libbyzagg_star.so"
  for other in (_lib.library_path(), _lib.peers_library_path()):
    handle = ctypes.CDLL(str(other))
    for name in STAR_NAMES:
      assert not hasattr(handle, name), (other.name, name)
  for name, (restype, argtypes) in _lib.ROWSHARE_STAR_SIGNATURES.items():
    fn = getattr(_lib.star_lib(), name)
    assert fn.argtypes == argtypes and fn.restype == restype

@pytest.mark.skipif(shutil.which("nm") is None, reason="nm not available")
def test_third_library_exports_only_its_calls_and_needs_nothing_of_the_others():
  from byzantinemomentum_b200 import _lib
  path = str(_lib.star_library_path())
  defined = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True).stdout
  assert sorted(re.findall(r" T (\S+)", defined)) == STAR_NAMES
  undefined = subprocess.run(["nm", "-D", "--undefined-only", path], capture_output=True, text=True).stdout
  assert "bz" not in undefined and "byzagg" not in undefined
  needed = subprocess.run(["readelf", "-d", path], capture_output=True, text=True).stdout if shutil.which("readelf") else ""
  assert "libbyzagg" not in needed and "libcudart" not in needed

def test_missing_third_library_raises_with_the_build_hint(monkeypatch, tmp_path):
  from byzantinemomentum_b200 import _lib
  monkeypatch.setenv("BYZAGG_STAR_LIBRARY", str(tmp_path / "nowhere.so"))
  monkeypatch.setattr(_lib, "_star_lib", None)
  with pytest.raises(_lib.LibraryError, match="build the CUDA extension"):
    _lib.star_lib()

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_the_star_kernel_fits_its_budget():
  """ One kernel, 256 threads and two CTAs per SM: at most 128 registers, no stack. """
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.star_library_path())], capture_output=True, text=True,
                        timeout=600).stdout
  usage = {name: (int(regs), int(stack)) for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text)}
  assert list(usage) == ["_ZN2bz16k2_rowshare_starEPKfiilPdPjS2_"], usage
  regs, stack = usage["_ZN2bz16k2_rowshare_starEPKfiilPdPjS2_"]
  assert regs <= 128 and stack == 0, (regs, stack)

def test_star_workspace_sizes():
  from byzantinemomentum_b200 import _lib
  lib = _lib.star_lib()
  for n in range(1, 129):
    size = lib.bz_rowshare_star_workspace_bytes(n)
    assert size % 256 == 0 and size >= 256 + 336 * n * 8, n
  assert lib.bz_rowshare_star_workspace_bytes(200) == lib.bz_rowshare_star_workspace_bytes(128)

def test_star_rejects_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here: fake addresses. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.star_lib()
  def err():
    return lib.bz_rowshare_star_last_error().decode()
  honest, cand, part, ws = 0x100000, 0x900000, 0xa00000, 0xb00000
  def call(n=100, c0=90, d=64, rows=None, part=part, ws=ws, ws_bytes=1 << 30):
    k = min(max(c0, 0), n)
    table = rows if rows is not None else (ctypes.c_void_p * max(n, 1))(*([honest + 4096 * i for i in range(k)] +
                                                                           [cand] * (max(n, 1) - k)))
    return lib.bz_rowshare_star(table, n, c0, d, part, ws, ws_bytes, None)
  assert lib.bz_rowshare_star(None, 100, 90, 64, part, ws, 1 << 30, None) == -1 and "rows is NULL" in err()
  assert call(n=0, c0=0) == -1 and "n = 0" in err()
  for n in (1, 25, 64, 129):
    assert call(n=n, c0=n - 1) == -2 and f"n = {n}" in err() and "BZ_MAX_N_DISTANCE = 128" in err(), n
  for c0 in (0, 100, -1):
    assert call(c0=c0) == -1 and f"c0 = {c0}" in err(), c0
  assert call(d=-1) == -1 and "d = -1" in err()
  rows = (ctypes.c_void_p * 100)(*([honest + 4096 * i for i in range(90)] + [cand] * 9 + [cand + 4096]))
  assert call(rows=rows) == -1 and "rows[99] differs from rows[90]" in err()
  rows = (ctypes.c_void_p * 100)(*([honest + 4096 * i for i in range(89)] + [cand] * 11))
  assert call(rows=rows) == -1 and "rows[89] is the candidate" in err()
  rows = (ctypes.c_void_p * 100)(*([honest + 4096 * i for i in range(89)] + [None] + [cand] * 10))
  assert call(rows=rows) == -1 and "rows[89] is NULL" in err()
  assert call(rows=rows, d=0, ws=None) == -4                 # an empty shard reads no row
  rows = (ctypes.c_void_p * 100)(*([honest + 4096 * i for i in range(90)] + [cand + 2] * 10))
  assert call(rows=rows) == -1 and "rows[90] is not 4-byte aligned" in err()
  assert call(part=None) == -1 and "part" in err()
  assert call(part=part + 4) == -1 and "part" in err()
  need = lib.bz_rowshare_star_workspace_bytes(100)
  assert call(ws_bytes=need - 1) == -4 and "workspace" in err() and str(need) in err()
  assert call(ws=None) == -4 and call(ws=ws + 4) == -4
  assert call(d=0, ws=None) == -4 and call(d=0, ws_bytes=need - 1) == -4
  same = (ctypes.c_void_p * 100)(*([cand] * 100))             # an empty shard: every row may share one address
  assert call(rows=same, d=0, ws=None) == -4 and call(rows=same, d=64) == -1 and "rows[0] is the candidate" in err()
