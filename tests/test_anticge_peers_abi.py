# coding: utf-8
"""The d-sharded attack against CGE with its exchanges over peer memory (include/byzagg_anticge_peers.h) on the CPU:
the header and its binding, the argument checks (before any CUDA call, with fake pointers), the register and stack
budgets of the new kernels, every kernel that existed before them unchanged in resources and SASS, and the choice of
the exchange (`sharded.choose_anticge_exchange`) under gloo with two ranks.  No compute calls here.

`tests/golden/kernels_before_anticge_peers.json` records, for every kernel of the library as it was before these
entry points, its registers, its stack and a digest of its SASS (`kernel_table`); it was written with
`python tests/test_anticge_peers_abi.py --record byzantinemomentum_b200/libbyzagg.so` on that library.  The entries of
`k1_sorted<18, 1, -1, -1>` and `k1_sorted<18, 4, -1, -1>` were recorded later, when the 18-row trimmed mean at f = 0
began to sum in ATen's cascade order (`trmean_sorted` in k1_select.cuh)."""

import ctypes
import hashlib
import json
import os
import pathlib
import re
import shutil
import socket
import subprocess
import sys

import pytest

ROOT = pathlib.Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "byzagg_anticge_peers.h"
BEFORE = ROOT / "tests" / "golden" / "kernels_before_anticge_peers.json"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
NAMES = ["bz_anticge_peers", "bz_anticge_peers_next"]
# the kernels these entry points add: (pattern of the mangled name, count, register budget, stack budget).  K2'-norms
# runs two 256-thread CTAs per SM, as K2'.  Up to 64 rows it is the body of k2_rowdist_peers, whose VEC = 4 form
# keeps the 24-byte frame that k2_rowdist<VEC = 4> and k2_rowdist_peers<VEC = 4> keep (the blocks must be phase A's
# bits, so the vector width and the occupancy stay theirs); every other new kernel has no stack.
NEW_KERNELS = [(r"k2_anticge_normsILi4E", 1, 128, 24),
               (r"k2_anticge_normsILi1E", 1, 128, 0),
               (r"k2_anticge_norms_wide", 1, 128, 0),
               (r"k10_anticge_peers", 4, 255, 0)]

def declared(path):
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", path.read_text())))

def test_header_declares_the_calls_and_byzagg_h_includes_it_last():
  assert declared(HEADER) == NAMES
  byzagg = (ROOT / "include" / "byzagg.h").read_text()
  includes = re.findall(r'#include "(byzagg_\w+\.h)"', byzagg)
  assert includes[-1] == "byzagg_anticge_peers.h" and includes.count("byzagg_anticge_peers.h") == 1
  assert not set(declared(ROOT / "include" / "byzagg.h")) & set(NAMES)
  makefile = (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  assert "../../include/byzagg_anticge_peers.h" in makefile and "api_anticge_peers.inc" in makefile

def test_library_exports_the_calls_and_the_table_is_its_own():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.library_path()))
  for name in NAMES:
    assert hasattr(handle, name), name
  assert sorted(_lib.ANTICGE_PEER_SIGNATURES) == NAMES
  others = [_lib.SIGNATURES, _lib.SHARD_SIGNATURES, _lib.ATTACK_SIGNATURES, _lib.SEARCH_SHARD_SIGNATURES,
            _lib.SEARCH_PEER_SIGNATURES, _lib.COORDINATE_SIGNATURES, _lib.PEER_NEXT_SIGNATURES, _lib.DISTANCE_SIGNATURES,
            _lib.DISTANCE_SHARD_SIGNATURES, _lib.ANTICGE_SIGNATURES]
  assert not set(_lib.ANTICGE_PEER_SIGNATURES) & set().union(*others)
  for name, (restype, argtypes) in _lib.ANTICGE_PEER_SIGNATURES.items():
    fn = getattr(_lib.lib(), name)
    assert fn.argtypes == argtypes and fn.restype == restype

def test_calls_reject_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here, and the calls that launch nothing (d = 0 with the NaN fill): fake addresses. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  big = 1 << 40
  def rows(n, address=0x1000):
    return (ctypes.c_void_p * n)(*[address + 0x100 * i for i in range(n)])
  def tables(R, blocks=0x200000, flags=0x300000):
    return ((ctypes.c_void_p * (2 * R))(*[blocks + 0x1000 * i for i in range(2 * R)]),
            (ctypes.c_void_p * (2 * R))(*[flags + 0x100 * i for i in range(2 * R)]))
  def message():
    return lib.bz_last_error().decode()
  for next_ in (False, True):
    def call(table=None, nh=25, f_decl=5, f_real=5, d=16, out=0x90000, status=0xa0000, rank=0, R=2, peers=None, ws=0xc0000,
             ws_bytes=big):
      blocks, flags = tables(R) if peers is None else peers
      head = (rows(max(nh, 1)) if table is None else table, nh, f_decl, f_real, d, ctypes.c_void_p(out) if out else None,
              ctypes.c_void_p(status) if status else None, rank, R, blocks, flags)
      tail = (ctypes.c_void_p(ws) if ws else None, ws_bytes, None)
      return lib.bz_anticge_peers_next(*head, *tail) if next_ else lib.bz_anticge_peers(*head, 7, *tail)
    assert call(nh=0) == -1 and "n = 0" in message()
    assert call(nh=129) == -2 and "128" in message()
    for f_decl in (0, -1, 26):
      assert call(f_decl=f_decl) == -1 and "f_decl" in message(), f_decl
    assert call(f_real=-1) == -1 and "f_real" in message()
    assert call(table=rows(25, address=0x1002)) == -1 and "aligned" in message()
    with_null = rows(100)
    with_null[70] = None
    assert call(table=with_null, nh=100, f_decl=10) == -1 and "rows[70] is NULL" in message()
    assert call(out=0) == -1 and "output" in message()
    assert call(ws_bytes=lib.bz_anticge_workspace_bytes(25) - 1) == -4 and "workspace" in message()
    assert call(ws=0xc0004) == -4 and call(ws=0) == -4
    # the exchange: ranks, tables of both slots, status
    assert call(R=0) == -1 and "rank" in message()
    assert call(R=17) == -1 and "rank" in message()
    assert call(rank=2, R=2) == -1 and call(rank=-1) == -1
    assert call(status=0) == -1 and "status" in message()
    blocks, flags = tables(3)
    blocks[4] = None                                       # slot 1 of rank 1
    assert call(R=3, peers=(blocks, flags)) == -1 and "slot 1" in message()
    blocks, flags = tables(3)
    flags[2] = 0x300002                                    # misaligned flag array, slot 0 of rank 2
    assert call(R=3, peers=(blocks, flags)) == -1 and "peer 2" in message()
    blocks, _ = tables(2)
    blocks[1] = 0x200004                                   # misaligned block
    assert call(peers=(blocks, tables(2)[1])) == -1
    assert call(peers=(None, tables(2)[1])) == -1 and "NULL peer table" in message()
    # the checks run before the NaN fill's shortcut, and d = 0 with the fill launches nothing
    assert call(f_real=6, status=0) == -1
    for nh in (1, 64, 65, 128):
      assert call(nh=nh, f_decl=1, f_real=3, d=0, out=0) == 0, nh

def _usage():
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout
  return {name: (int(regs), int(stack)) for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text)}

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_new_kernels_fit_their_register_and_stack_budgets():
  usage = _usage()
  for pattern, count, budget, frame in NEW_KERNELS:
    names = [name for name in usage if re.search(pattern, name)]
    assert len(names) == count, (pattern, names)
    for name in names:
      regs, stack = usage[name]
      assert regs <= budget and stack <= frame, (name, regs, stack)

def kernel_table(library):
  """ {kernel: [registers, stack, digest of its SASS]} of every kernel in `library`. """
  usage = {name: (int(regs), int(stack)) for name, regs, stack in
           re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)",
                      subprocess.run([CUOBJDUMP, "-res-usage", str(library)], capture_output=True, text=True, timeout=600).stdout)}
  sass = subprocess.run([CUOBJDUMP, "-sass", str(library)], capture_output=True, text=True, timeout=1200).stdout
  code = {}
  for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
    name, _, body = chunk.partition("\n")
    # the instructions with their encodings; the dump pads its columns to the widest line of the whole library
    lines = [" ".join(line.split()) for line in body.splitlines() if re.match(r"\s*/\*[0-9a-f]{4,}\*/", line)]
    code[name.strip()] = hashlib.sha256("\n".join(lines).encode()).hexdigest()[:20]
  assert set(code) == set(usage), sorted(set(code) ^ set(usage))[:5]
  return {name: [regs, stack, code[name]] for name, (regs, stack) in sorted(usage.items())}

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_every_kernel_that_existed_before_is_unchanged():
  from byzantinemomentum_b200 import _lib
  before = json.loads(BEFORE.read_text())
  now = kernel_table(_lib.library_path())
  assert len(before) > 400
  missing = sorted(set(before) - set(now))
  assert not missing, missing[:5]
  changed = [name for name in before if now[name] != before[name]]
  assert not changed, [(name, before[name], now[name]) for name in changed[:5]]
  added = set(now) - set(before)
  assert all(any(re.search(pattern, name) for pattern, *_ in NEW_KERNELS) for name in added), sorted(added)
  assert len(added) == sum(count for _, count, *_ in NEW_KERNELS)

# ---- the choice of the exchange ------------------------------------------------------------------------------------

# (symmetric on rank 0, symmetric on rank 1, exchange) -> what both ranks get ("raise": ValueError on both)
SCENARIOS = [
  (1, 1, "auto", "fused"),
  (1, 0, "auto", "nccl"),
  (0, 1, "auto", "nccl"),
  (1, 1, "nccl", "nccl"),
  (1, 1, "fused", "fused"),
  (1, 0, "fused", "raise"),
  (0, 1, "fused", "raise"),
]

def _worker(rank, world, port, queue):
  sys.path.insert(0, str(ROOT))
  import torch.distributed as dist
  from byzantinemomentum_b200 import sharded
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    got = []
    for sym0, sym1, exchange, _ in SCENARIOS:
      try:
        got.append(sharded.choose_anticge_exchange(exchange, sym0 if rank == 0 else sym1))
      except ValueError:
        got.append("raise")
    queue.put((rank, got))
  finally:
    dist.destroy_process_group()

def test_two_ranks_agree_on_the_exchange():
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
  assert got[0] == got[1] == [want for *_, want in SCENARIOS]

def test_one_rank_and_too_many_ranks(monkeypatch):
  pytest.importorskip("torch")
  from byzantinemomentum_b200 import sharded
  assert sharded.choose_anticge_exchange("auto", True) == "nccl"            # one rank keeps the collective stages
  assert sharded.choose_anticge_exchange("fused", False) == "fused"         # a plain buffer serves one rank
  with pytest.raises(ValueError, match="unknown exchange"):
    sharded.choose_anticge_exchange("p2p", True)
  monkeypatch.setattr(sharded.dist, "is_initialized", lambda: True)
  monkeypatch.setattr(sharded.dist, "get_world_size", lambda group=None: 17)
  monkeypatch.setattr(sharded, "_agree", lambda facts, group: list(facts))
  assert sharded.choose_anticge_exchange("auto", True) == "nccl"
  with pytest.raises(ValueError, match="symmetric memory"):
    sharded.choose_anticge_exchange("fused", True)
  monkeypatch.setattr(sharded.dist, "get_world_size", lambda group=None: 16)
  assert sharded.choose_anticge_exchange("auto", True) == "fused"
  assert sharded.choose_anticge_exchange("auto", False) == "nccl"

if __name__ == "__main__":
  if len(sys.argv) == 3 and sys.argv[1] == "--record":
    table = kernel_table(sys.argv[2])
    BEFORE.write_text("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v)}" for k, v in table.items()) + "\n}\n")
  else:
    sys.exit("usage: test_anticge_peers_abi.py --record LIBRARY")
