# coding: utf-8
"""How `sharded.ShardedLineSearch` picks its exchange, and the epochs its fused search issues (CPU suite).

  * `choose_search_exchange` under `gloo`, world_size 2, with stand-in facts per rank: "auto" takes "fused"
    only when both ranks have every fact, and the two ranks always agree; one rank without symmetric
    memory, with unaligned rows or with a stand-in backend moves both to "nccl"; an explicit "fused" that
    one rank cannot serve raises on both.
  * One rank, and more than 16 ranks, without a process group.
  * The fused search on a backend stand-in issues 2 epochs per evaluation for a distance rule and 1 for
    the others, in issue order from the shared counter, whatever the rank's columns (an empty shard too)."""

import os
import socket

import pytest

torch = pytest.importorskip("torch")

# (facts of rank 0, facts of rank 1, exchange) -> what both ranks get ("raise": ValueError on both).
# facts: (aligned, symmetric, engine)
ALL = (1, 1, 1)
SCENARIOS = [
  (ALL, ALL, "auto", "fused"),
  (ALL, (1, 0, 1), "auto", "nccl"),
  ((0, 1, 1), ALL, "auto", "nccl"),
  (ALL, (1, 1, 0), "auto", "nccl"),
  (ALL, ALL, "nccl", "nccl"),
  (ALL, ALL, "fused", "fused"),
  (ALL, (1, 1, 0), "fused", "fused"),         # an explicit request with a backend that provides the stages
  (ALL, (0, 1, 1), "fused", "raise"),
  ((1, 0, 1), ALL, "fused", "raise"),
]

def _worker(rank, world, port, queue):
  import sys, pathlib
  root = pathlib.Path(__file__).resolve().parent.parent
  sys.path.insert(0, str(root))
  import torch.distributed as dist
  from byzantinemomentum_b200 import sharded
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    got = []
    for facts0, facts1, exchange, _ in SCENARIOS:
      aligned, symmetric, engine = facts0 if rank == 0 else facts1
      try:
        got.append(sharded.choose_search_exchange(exchange, aligned, symmetric, engine))
      except ValueError:
        got.append("raise")
    queue.put((rank, got))
  finally:
    dist.destroy_process_group()

def test_two_ranks_agree_on_the_exchange():
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
  from byzantinemomentum_b200 import sharded
  assert sharded.choose_search_exchange("auto", True, True, True) == "nccl"          # one rank keeps the collective path
  assert sharded.choose_search_exchange("fused", True, False, False) == "fused"      # a plain buffer serves one rank
  with pytest.raises(ValueError):
    sharded.choose_search_exchange("fused", False, True, True)
  with pytest.raises(ValueError, match="unknown exchange"):
    sharded.choose_search_exchange("p2p", True, True, True)
  monkeypatch.setattr(sharded.dist, "is_initialized", lambda: True)
  monkeypatch.setattr(sharded.dist, "get_world_size", lambda group=None: 17)
  monkeypatch.setattr(sharded, "_agree", lambda facts, group: list(facts))
  assert sharded.choose_search_exchange("auto", True, True, True) == "nccl"
  with pytest.raises(ValueError):
    sharded.choose_search_exchange("fused", True, True, True)
  monkeypatch.setattr(sharded.dist, "get_world_size", lambda group=None: 16)
  assert sharded.choose_search_exchange("auto", True, True, True) == "fused"

class _Recorder:
  """ The fused stages of one rank, recording what they are given. """
  def __init__(self, gar, honest, f_real, f_decl, avg, att, evals, negative, kind, world):
    from byzantinemomentum_b200 import sharded
    self.device = avg.device
    self.distance = gar in sharded.DISTANCE_BASED
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
  def search_shard(self, *args):
    return _Recorder(*args)

@pytest.mark.parametrize("gar", ["average", "median", "trmean", "phocas", "meamed", "krum", "bulyan", "brute", "aksel", "cge"])
def test_fused_search_issues_its_epochs_in_order(gar):
  from byzantinemomentum_b200 import sharded
  nh, f, evals = 9, 2, 5
  distance = gar in sharded.DISTANCE_BASED
  sequences = []
  for d, start in ((601, 0), (0, 0), (33, 2**32 - 3)):           # an empty shard; across the 32-bit wrap
    honest = [torch.full((d,), float(i)) for i in range(nh)]
    avg, att = torch.zeros(d), torch.ones(d)
    assert sharded.ShardedLineSearch(gar, honest, f, f, avg, att, evals, backend=_Backend()).exchange == "nccl"
    search = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, evals, backend=_Backend(), exchange="fused")
    assert search.exchange == "fused" and search._fx.world == 1 and search._fx.n == nh + f
    search._fx.epoch = start
    search()
    search()                                                       # a second search continues the counter
    calls = search._shard.calls
    assert calls[0] == ("fuse", nh + f, 1, 0)
    epochs = [c[2] for c in calls if c[0] in ("rule", "score") and c[2] is not None]
    per = 2 if distance else 1
    assert epochs == list(range(start + 1, start + 1 + 2 * per * evals)), (gar, d, epochs)
    assert search._fx.epoch == start + 2 * per * evals
    if not distance:
      assert all(c[2] is None for c in calls if c[0] == "rule")
    order = [c[:2] for c in calls[1:]]
    assert order == 2 * ([x for k in range(evals) for x in (("rule", k), ("score", k))] + [("finish",)])
    sequences.append([e - start for e in epochs])
  assert sequences[0] == sequences[1] == sequences[2]
