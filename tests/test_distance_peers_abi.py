# coding: utf-8
"""Phase B of the d-sharded Multi-Krum, Bulyan, Aksel and CGE above 64 rows with its exchange over peer memory
(include/byzagg_distance_peers.h, libbyzagg_peers.so) on the CPU: the header and the second library's binding, the
argument checks (before any CUDA call, with fake pointers), the register and stack budgets of its kernels, every
kernel of libbyzagg.so unchanged in resources and SASS, and the choice of `ShardedPlan`'s exchange
(`sharded.plan_exchange`) under gloo with two ranks.  No compute calls here.

`tests/golden/kernels_before_distance_peers.json` records, for every kernel of libbyzagg.so as it was before the
second library, its registers, its stack and a digest of its SASS (`kernel_table` of test_anticge_peers_abi.py); it
was written with `python tests/test_distance_peers_abi.py --record byzantinemomentum_b200/libbyzagg.so` on that
library.  The entries of `k1_sorted<18, 1, -1, -1>` and `k1_sorted<18, 4, -1, -1>` were recorded later, when the
18-row trimmed mean at f = 0 began to sum in ATen's cascade order (`trmean_sorted` in k1_select.cuh)."""

import ctypes
import json
import os
import pathlib
import re
import shutil
import socket
import subprocess
import sys

import pytest

from test_anticge_peers_abi import CUOBJDUMP, declared, kernel_table

ROOT = pathlib.Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "byzagg_distance_peers.h"
BEFORE = ROOT / "tests" / "golden" / "kernels_before_distance_peers.json"
CALLS = ["bz_distance_select_peers", "bz_distance_select_peers_next"]
NAMES = ["bz_distance_peers_last_error"] + CALLS
# the kernels of libbyzagg_peers.so: (pattern of the mangled name, count, register budget, stack budget).  The pairs
# kernel runs 1024 threads in one CTA, so it must stay within 64 registers; the keys kernel runs 128.
NEW_KERNELS = [(r"k5_blocks_select_peers", 1, 64, 0),
               (r"k5_rowkeys_select_peers", 1, 128, 0)]
KRUM, BULYAN, BRUTE, AKSEL, CGE = 5, 6, 7, 8, 9

def test_header_declares_the_calls_and_byzagg_h_leaves_it_out():
  assert declared(HEADER) == sorted(NAMES)
  text = HEADER.read_text()
  assert '#include "byzagg.h"' in text
  byzagg = (ROOT / "include" / "byzagg.h").read_text()
  includes = re.findall(r'#include "(byzagg_\w+\.h)"', byzagg)
  assert "byzagg_distance_peers.h" not in includes and includes[-1] == "byzagg_anticge_peers.h"
  assert not set(declared(ROOT / "include" / "byzagg.h")) & set(NAMES)
  for other in (ROOT / "include").glob("byzagg*.h"):
    if other != HEADER:
      assert "byzagg_distance_peers.h" not in other.read_text(), other.name
      assert not set(declared(other)) & set(NAMES), other.name

def test_makefile_builds_the_second_library():
  makefile = (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  assert re.search(r"^all: \$\(OUT\) \$\(PEERS_OUT\)$", makefile, re.M)
  assert "PEERS_OUT := ../libbyzagg_peers" in makefile
  assert "PEERS_OBJS := $(BUILD)/api_distance_peers.o $(BUILD)/k5_select_peers.o" in makefile
  rule = re.search(r"^\$\(PEERS_OUT\): \$\(PEERS_OBJS\)\n\t(.*)$", makefile, re.M).group(1)
  assert "-shared" in rule and "-cudart static" in rule and "$(ARCH)" in rule and "$(OBJS)" not in rule
  assert "-lbyzagg" not in rule and "libbyzagg.so" not in rule
  assert "-fvisibility=hidden" in makefile and "code=sm_90a" in makefile
  assert "../../include/byzagg_distance_peers.h" in makefile

def test_table_is_its_own_and_the_library_exports_it():
  from byzantinemomentum_b200 import _lib
  assert sorted(_lib.DISTANCE_PEER_SIGNATURES) == sorted(NAMES)
  others = [_lib.SIGNATURES, _lib.SHARD_SIGNATURES, _lib.ATTACK_SIGNATURES, _lib.SEARCH_SHARD_SIGNATURES,
            _lib.SEARCH_PEER_SIGNATURES, _lib.COORDINATE_SIGNATURES, _lib.PEER_NEXT_SIGNATURES, _lib.DISTANCE_SIGNATURES,
            _lib.DISTANCE_SHARD_SIGNATURES, _lib.ANTICGE_SIGNATURES, _lib.ANTICGE_PEER_SIGNATURES]
  assert not set(_lib.DISTANCE_PEER_SIGNATURES) & set().union(*others)
  assert _lib.peers_library_path() == _lib.library_path().parent / "libbyzagg_peers.so"
  main = ctypes.CDLL(str(_lib.library_path()))
  for name in NAMES:
    assert not hasattr(main, name), name                  # libbyzagg.so does not carry them
  for name, (restype, argtypes) in _lib.DISTANCE_PEER_SIGNATURES.items():
    fn = getattr(_lib.peers_lib(), name)
    assert fn.argtypes == argtypes and fn.restype == restype

@pytest.mark.skipif(shutil.which("nm") is None, reason="nm not available")
def test_second_library_exports_only_its_calls_and_needs_nothing_of_the_first():
  from byzantinemomentum_b200 import _lib
  path = str(_lib.peers_library_path())
  defined = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True).stdout
  assert sorted(re.findall(r" T (\S+)", defined)) == sorted(NAMES)
  undefined = subprocess.run(["nm", "-D", "--undefined-only", path], capture_output=True, text=True).stdout
  assert "bz" not in undefined and "byzagg" not in undefined
  needed = subprocess.run(["readelf", "-d", path], capture_output=True, text=True).stdout if shutil.which("readelf") else ""
  assert "libbyzagg" not in needed and "libcudart" not in needed

def test_missing_library_raises_with_the_build_hint(monkeypatch, tmp_path):
  from byzantinemomentum_b200 import _lib
  monkeypatch.setenv("BYZAGG_PEERS_LIBRARY", str(tmp_path / "nowhere.so"))
  monkeypatch.setattr(_lib, "_peers_lib", None)
  with pytest.raises(_lib.LibraryError, match="build the CUDA extension"):
    _lib.peers_lib()

def test_calls_reject_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here: fake addresses. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.peers_lib()
  def tables(R, slots, blocks=0x200000, flags=0x300000):
    return ((ctypes.c_void_p * (slots * R))(*[blocks + 0x20000 * i for i in range(slots * R)]),
            (ctypes.c_void_p * (slots * R))(*[flags + 0x100 * i for i in range(slots * R)]))
  def message():
    return lib.bz_distance_peers_last_error().decode()
  for next_ in (False, True):
    slots = 2 if next_ else 1
    def call(rule=KRUM, part=0x100000, n=100, f=10, m=50, mode=0, order=0x90000, status=0xa0000, rank=0, R=2, peers=None):
      blocks, flags = tables(R, slots) if peers is None else peers
      head = (rule, ctypes.c_void_p(part) if part else None, n, f, m, mode, ctypes.c_void_p(order) if order else None,
              ctypes.c_void_p(status) if status else None, rank, R, blocks, flags)
      return lib.bz_distance_select_peers_next(*head, None) if next_ else lib.bz_distance_select_peers(*head, 7, None)
    assert call(rule=4) == -1 and "unknown rule" in message()
    assert call(rule=10) == -1 and "unknown rule" in message()
    assert call(n=0) == -1 and "n = 0" in message()
    assert call(n=129) == -2 and "128" in message()
    assert call(rule=BRUTE, n=100) == -2 and "brute" in message()
    for rule in (KRUM, BULYAN, BRUTE, AKSEL, CGE):
      for n in (1, 25, 64):
        assert call(rule=rule, n=n, f=0, m=1) == -2, (rule, n)
        text = message()
        assert all(name in text for name in ("bz_krum_peers", "bz_bulyan_peers", "bz_rowdist_peers")), text
    assert call(part=0) == -1 and "part" in message()
    assert call(part=0x100004) == -1 and "aligned" in message()
    assert call(order=0) == -1 and "order" in message()
    # the counts of bz_distance_select
    assert call(f=99) == -1 and "f = 99" in message()
    assert call(f=-1) == -1
    assert call(m=0) == -1 and "m = 0" in message()
    assert call(m=101) == -1 and "m = 101" in message()
    assert call(rule=BULYAN, f=25) == -1 and "4f + 3" in message()
    assert call(rule=BULYAN, f=10, m=89) == -1 and "m = 89" in message()
    assert call(rule=AKSEL, mode=2) == -1 and "mode = 2" in message()
    assert call(rule=AKSEL, mode=1, f=100) == -1 and "f = 100" in message()
    # the exchange: ranks, tables, status
    assert call(R=0) == -1 and "rank" in message()
    assert call(R=17) == -1 and "rank" in message()
    assert call(rank=2, R=2) == -1 and call(rank=-1) == -1
    assert call(status=0) == -1 and "status" in message()
    assert call(rule=CGE, status=0) == -1
    assert call(peers=(None, tables(2, slots)[1])) == -1 and "NULL peer table" in message()
    blocks, flags = tables(3, slots)
    flags[2] = 0x300002                                    # misaligned flag array, slot 0 of rank 2
    assert call(R=3, peers=(blocks, flags)) == -1 and "peer 2" in message()
    blocks, flags = tables(2, slots)
    blocks[1] = 0x200004                                   # misaligned block
    assert call(peers=(blocks, flags)) == -1 and "peer 1" in message()
    if next_:
      blocks, flags = tables(3, 2)
      blocks[4] = None                                     # slot 1 of rank 1
      assert call(R=3, peers=(blocks, flags)) == -1 and "slot 1" in message()
  # the message reaches Python from the library that failed
  assert lib.bz_distance_select_peers(KRUM, None, 100, 10, 50, 0, None, None, 0, 1, None, None, 1, None) == -1
  with pytest.raises(ValueError, match="bz_distance_select_peers.*part / order is NULL"):
    _lib.check(-1, "bz_distance_select_peers")

def _usage():
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.peers_library_path())], capture_output=True, text=True, timeout=600).stdout
  return {name: (int(regs), int(stack)) for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text)}

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_kernels_of_the_second_library_fit_their_budgets():
  usage = _usage()
  assert len(usage) == sum(count for _, count, *_ in NEW_KERNELS), sorted(usage)
  for pattern, count, budget, frame in NEW_KERNELS:
    names = [name for name in usage if re.search(pattern, name)]
    assert len(names) == count, (pattern, names)
    for name in names:
      regs, stack = usage[name]
      assert regs <= budget and stack <= frame, (name, regs, stack)

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_every_kernel_of_libbyzagg_is_unchanged():
  from byzantinemomentum_b200 import _lib
  before = json.loads(BEFORE.read_text())
  now = kernel_table(_lib.library_path())
  assert len(before) > 400
  assert sorted(set(before) ^ set(now)) == []
  changed = [name for name in before if now[name] != before[name]]
  assert not changed, [(name, before[name], now[name]) for name in changed[:5]]

# ---- the choice of the exchange ------------------------------------------------------------------------------------

GARS = ["krum", "bulyan", "brute", "aksel", "cge"]
SIZES = [25, 64, 65, 128]
# (aligned on rank 0, aligned on rank 1, symmetric on rank 0, symmetric on rank 1)
FACTS = [(1, 1, 1, 1), (1, 0, 1, 1), (0, 0, 1, 1), (1, 1, 1, 0), (1, 1, 0, 0)]

def _want_fused(gar, n, aligned, symmetric):
  """ What an explicit "fused" gives on two ranks whose agreed facts are `aligned` and `symmetric`. """
  if gar in ("krum", "bulyan") and n <= 64:
    return "fused" if aligned and symmetric else "raise"     # the ring's exchange, as before
  if gar in ("krum", "bulyan", "aksel", "cge"):
    return "fused" if symmetric else "raise"                 # any alignment
  return "raise"

def _worker(rank, world, port, queue):
  sys.path.insert(0, str(ROOT))
  import torch.distributed as dist
  from byzantinemomentum_b200 import sharded
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  def outcome(fn):
    try:
      return fn()
    except ValueError:
      return "raise"
  try:
    got = []
    for a0, a1, s0, s1 in FACTS:
      aligned, symmetric = (a0, s0) if rank == 0 else (a1, s1)
      for gar in GARS:
        for n in SIZES:
          for exchange in ("auto", "nccl", "p2p", "fused"):
            new = outcome(lambda: sharded.plan_exchange(gar, n, exchange, aligned, symmetric))
            old = outcome(lambda: sharded.choose_exchange(gar, sharded.rows_exchange(exchange, n), aligned, symmetric))
            got.append((a0, a1, s0, s1, gar, n, exchange, new, old))
    queue.put((rank, got))
  finally:
    dist.destroy_process_group()

def test_two_ranks_agree_on_the_plan_exchange():
  pytest.importorskip("torch")
  import torch.multiprocessing as mp
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
  ctx = mp.get_context("spawn")
  queue = ctx.Queue()
  procs = [ctx.Process(target=_worker, args=(r, 2, port, queue)) for r in range(2)]
  for p in procs:
    p.start()
  got = dict(queue.get(timeout=300) for _ in procs)
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  assert got[0] == got[1]
  fused_new = 0
  for a0, a1, s0, s1, gar, n, exchange, new, old in got[0]:
    what = (a0, a1, s0, s1, gar, n, exchange)
    if exchange != "fused":
      assert new == old, what                                # "auto", "nccl" and "p2p" keep today's choice
    else:
      assert new == _want_fused(gar, n, a0 and a1, s0 and s1), (what, new)
      fused_new += new == "fused" and old == "raise"
  assert fused_new > 0
  # spot checks of the table above
  table = {(a0, a1, s0, s1, gar, n, ex): new for a0, a1, s0, s1, gar, n, ex, new, _ in got[0]}
  assert table[(1, 1, 1, 1, "krum", 128, "auto")] == "nccl"
  assert table[(1, 1, 1, 1, "krum", 128, "p2p")] == "raise"
  assert table[(1, 0, 1, 1, "krum", 128, "fused")] == "fused"                 # one rank unaligned
  assert table[(1, 0, 1, 1, "krum", 25, "fused")] == "raise"
  assert table[(1, 0, 1, 1, "cge", 25, "fused")] == "fused"
  assert table[(1, 1, 1, 0, "aksel", 65, "fused")] == "raise"                     # one rank without symmetric memory
  assert table[(1, 1, 1, 1, "aksel", 25, "auto")] == "p2p"

def test_one_rank_and_too_many_ranks(monkeypatch):
  pytest.importorskip("torch")
  from byzantinemomentum_b200 import sharded
  for gar, n in (("aksel", 1), ("cge", 64), ("krum", 65), ("bulyan", 128), ("cge", 100)):
    assert sharded.plan_exchange(gar, n, "fused", False, False) == "fused"    # one rank: a plain buffer
    assert sharded.plan_exchange(gar, n, "auto", True, True) == "nccl"
  with pytest.raises(ValueError):
    sharded.plan_exchange("krum", 25, "fused", False, True)                   # the ring's rule
  with pytest.raises(ValueError):
    sharded.plan_exchange("brute", 25, "fused", True, True)
  with pytest.raises(ValueError, match="unknown exchange"):
    sharded.plan_exchange("cge", 100, "ring", True, True)
  monkeypatch.setattr(sharded.dist, "is_initialized", lambda: True)
  monkeypatch.setattr(sharded.dist, "get_world_size", lambda group=None: 17)
  monkeypatch.setattr(sharded, "_agree", lambda facts, group: list(facts))
  with pytest.raises(ValueError, match="symmetric memory"):
    sharded.plan_exchange("cge", 100, "fused", True, True)
  monkeypatch.setattr(sharded.dist, "get_world_size", lambda group=None: 16)
  assert sharded.plan_exchange("cge", 100, "fused", False, True) == "fused"
  with pytest.raises(ValueError, match="symmetric memory"):
    sharded.plan_exchange("krum", 100, "fused", True, False)

if __name__ == "__main__":
  if len(sys.argv) == 3 and sys.argv[1] == "--record":
    table = kernel_table(sys.argv[2])
    BEFORE.write_text("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v)}" for k, v in table.items()) + "\n}\n")
  else:
    sys.exit("usage: test_distance_peers_abi.py --record LIBRARY")
