# coding: utf-8
"""Host logic of `sharded.GradientShards` (gradient delivery to the d-sharded path) on CPU: under
`gloo` with world_size 2 and the collective exchange, and in-process on one rank.  The scatter and
the momentum placement run on a torch stand-in (`TorchDelivery`) with the same per-coordinate
semantics as the CUDA calls; the CUDA calls themselves are covered by the `-m gpu` tests.

Every rank regenerates the seeded full gradients, pushes its own workers (i % R == rank), delivers,
and places momentum on its columns; its delivered and honest rows must equal columns [lo_r, hi_r)
of what one process computes on the full gradients, bit for bit."""

import math
import os
import socket

import numpy as np
import pytest

torch = pytest.importorskip("torch")

MU, DAMPENING = 0.9, 0.1
STEPS = 3
# (n, d, clip, momentum placement): ragged d, d = 1 (rank 1's shard is empty), n not a multiple of R,
# no clip / a clip that does not trigger / one that does, worker and server momentum
CASES = [(5, 601, None, "worker"), (5, 601, 1e9, "server"), (6, 601, 2.0, "worker"), (5, 1, 0.5, "server"),
         (4, 600, 2.0, "update"), (3, 37, 3.0, "server")]

class TorchDelivery:
  """ Stand-in for the engine's `gradient_scatter` / `momentum_rows`: elementwise operations only
  (no fused multiply-add, no order-dependent reduction but the norm, computed once per gradient in
  fp64 by NumPy), so a shard of the result has exactly the bits of the same columns of the full
  computation. """
  @staticmethod
  def clipped(grad, clip):
    g = grad.clone()
    if clip is not None and clip > 0:
      norm = float(np.float32(math.sqrt(float(np.sum(g.numpy().astype(np.float64) ** 2)))))
      if norm > clip:
        g = g.mul(float(np.float32(clip / norm)))
    return g
  def gradient_scatter(self, grad, clip, slots):
    from byzantinemomentum_b200.sharded import shard_bounds
    g = self.clipped(grad, clip)
    for r, slot in enumerate(slots):
      lo, hi = shard_bounds(g.numel(), len(slots), r)
      assert slot.numel() == hi - lo
      slot.copy_(g[lo:hi])
  @staticmethod
  def momentum_row(row, momentum, mu, dampening, honest=None):
    if honest is None:
      momentum.copy_((momentum.double() * mu + row.double() * (1. - dampening)).float())
      return momentum
    honest.copy_((row.double() * (1. - dampening) + momentum.double() * mu).float())
    return honest
  def momentum_rows(self, rows, mu, dampening, momentums=None, server=None, honests=None):
    if momentums is not None:
      return [self.momentum_row(r, m, mu, dampening) for r, m in zip(rows, momentums, strict=True)]
    return [self.momentum_row(r, server, mu, dampening, honest=h) for r, h in zip(rows, honests, strict=True)]

def _grad(case, step, i, d):
  gen = torch.Generator().manual_seed(10_000 * case + 100 * step + i)
  return torch.randn(d, generator=gen) * (0.2 + 0.3 * i)

def _momenta(case, n, d):
  gen = torch.Generator().manual_seed(777 + case)
  return [torch.randn(d, generator=gen) for _ in range(n)], torch.randn(d, generator=gen)

def _run_case(shards, case, n, d, clip, placement, lo, hi):
  """ STEPS steps on one rank; returns [(delivered rows, honest rows)] per step as arrays. """
  workers, server = _momenta(case, n, d)
  workers = [w[lo:hi].clone() for w in workers[:n - 1]]       # the last worker is not honest: no momentum
  server = server[lo:hi].clone()
  out = []
  for step in range(STEPS):
    for i in shards.workers():
      shards.push(i, _grad(case, step, i, d), clip=clip)
    rows = shards.deliver()
    assert len(rows) == n and all(r.numel() == hi - lo for r in rows)
    if placement == "worker":
      honest = shards.honests_worker(workers, MU, DAMPENING)
    elif placement == "server":
      honest = shards.honests_server(server, MU, DAMPENING, count=n - 1)
    else:
      honest = rows
    out.append((np.stack([r.numpy().copy() for r in rows]), np.stack([h.numpy().copy() for h in honest])))
  return out

def _expected(case, n, d, clip, placement):
  be = TorchDelivery()
  workers, server = _momenta(case, n, d)
  workers = workers[:n - 1]
  out = []
  for step in range(STEPS):
    rows = [be.clipped(_grad(case, step, i, d), clip) for i in range(n)]
    if placement == "worker":
      honest = [be.momentum_row(r, m, MU, DAMPENING) for r, m in zip(rows, workers)]
    elif placement == "server":
      honest = [be.momentum_row(r, server, MU, DAMPENING, honest=torch.empty(d)) for r in rows[:n - 1]]
    else:
      honest = rows
    out.append((np.stack([r.numpy() for r in rows]), np.stack([h.numpy().copy() for h in honest])))
  return out

def _worker(rank, world, port, queue):
  import sys, pathlib
  root = pathlib.Path(__file__).resolve().parent.parent
  sys.path.insert(0, str(root)); sys.path.insert(0, str(root / "tests"))
  import torch.distributed as dist
  from byzantinemomentum_b200 import sharded
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    got = {}
    for case, (n, d, clip, placement) in enumerate(CASES):
      shards = sharded.GradientShards(n, d, "cpu", exchange="collective", backend=TorchDelivery())
      assert shards.exchange == "collective" and shards.slots == 1
      assert list(shards.workers()) == list(range(rank, n, world))
      lo, hi = sharded.shard_bounds(d, world, rank)
      assert (shards.lo, shards.hi) == (lo, hi)
      got[case] = (lo, hi, _run_case(shards, case, n, d, clip, placement, lo, hi))
    # misuse: both raise before any collective, so the ranks stay in step
    shards = sharded.GradientShards(5, 601, "cpu", exchange="collective", backend=TorchDelivery())
    errors = []
    try:
      shards.deliver()                                   # nothing pushed
    except RuntimeError as err:
      errors.append(("missing", str(err)))
    try:
      shards.push(1 - rank, torch.zeros(601))            # the other rank's worker
    except ValueError as err:
      errors.append(("foreign", str(err)))
    shards.push(rank, torch.zeros(601))
    try:
      shards.deliver()                                   # rank 0 still owes workers 2 and 4, rank 1 worker 3
    except RuntimeError as err:
      errors.append(("partial", str(err)))
    got["errors"] = errors
    # the ranks agree on the exchange: symmetric memory on rank 0 only
    agreed = {}
    for request in ("auto", "p2p", "collective"):
      try:
        agreed[request] = sharded.choose_delivery(request, rank == 0)
      except ValueError:
        agreed[request] = "refused"
    agreed["both"] = sharded.choose_delivery("auto", True)
    got["agreed"] = agreed
    queue.put((rank, got))
  finally:
    dist.destroy_process_group()

def test_two_rank_delivery_matches_single_process():
  import torch.multiprocessing as mp
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
  ctx = mp.get_context("spawn")
  queue = ctx.Queue()
  procs = [ctx.Process(target=_worker, args=(r, 2, port, queue)) for r in range(2)]
  for p in procs:
    p.start()
  got = dict(queue.get(timeout=180) for _ in procs)
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  for case, (n, d, clip, placement) in enumerate(CASES):
    want = _expected(case, n, d, clip, placement)
    for rank in (0, 1):
      lo, hi, steps = got[rank][case]
      for step, ((rows, honest), (want_rows, want_honest)) in enumerate(zip(steps, want)):
        where = f"case {CASES[case]} rank {rank} step {step}"
        assert np.array_equal(rows.view(np.int32), want_rows[:, lo:hi].view(np.int32)), f"delivered rows, {where}"
        assert np.array_equal(honest.view(np.int32), want_honest[:, lo:hi].view(np.int32)), f"honest rows, {where}"
  assert got[1][3][:2] == (1, 1)                          # d = 1: rank 1's shard is empty
  for rank in (0, 1):
    kinds = [k for k, _ in got[rank]["errors"]]
    assert kinds == ["missing", "foreign", "partial"], got[rank]["errors"]
    assert got[rank]["agreed"] == {"auto": "collective", "p2p": "refused", "collective": "collective", "both": "p2p"}

def test_one_rank_without_a_process_group():
  from byzantinemomentum_b200 import sharded
  for case, (n, d, clip, placement) in enumerate(CASES):
    shards = sharded.GradientShards(n, d, "cpu", backend=TorchDelivery())
    assert shards.exchange == "collective" and list(shards.workers()) == list(range(n))
    assert shards.pitch % 64 == 0 and shards.pitch >= d
    workers, server = _momenta(case, n, d)
    workers = workers[:n - 1]
    steps = []
    for step in range(STEPS):
      for i in shards.workers():
        shards.push(i, _grad(case, step, i, d), clip=clip)
      before = shards.rows(0)[0]._version
      rows = shards.deliver()
      assert rows[0]._version > before                  # the delivery bumps the rows' version counter
      if placement == "worker":
        honest = shards.honests_worker(workers, MU, DAMPENING)
      elif placement == "server":
        honest = shards.honests_server(server, MU, DAMPENING, count=n - 1)
      else:
        honest = rows
      steps.append((np.stack([r.numpy().copy() for r in rows]), np.stack([h.numpy().copy() for h in honest])))
    for (rows, honest), (want_rows, want_honest) in zip(steps, _expected(case, n, d, clip, placement)):
      assert np.array_equal(rows.view(np.int32), want_rows.view(np.int32)), CASES[case]
      assert np.array_equal(honest.view(np.int32), want_honest.view(np.int32)), CASES[case]

def test_world_above_the_peer_limit_is_refused(monkeypatch):
  from byzantinemomentum_b200 import _lib, sharded
  monkeypatch.setattr(sharded.dist, "is_initialized", lambda: True)
  monkeypatch.setattr(sharded.dist, "get_world_size", lambda group=None: _lib.MAX_PEERS + 1)
  monkeypatch.setattr(sharded.dist, "get_rank", lambda group=None: 0)
  with pytest.raises(ValueError, match="at most 16 ranks"):
    sharded.GradientShards(25, 1000, "cpu", backend=TorchDelivery())

def test_unknown_exchange_is_refused():
  from byzantinemomentum_b200 import sharded
  with pytest.raises(ValueError, match="unknown exchange"):
    sharded.GradientShards(5, 10, "cpu", exchange="nccl", backend=TorchDelivery())

def test_misplaced_tensors_are_refused_before_any_launch(monkeypatch):
  """ A gradient on another device than the shards', a slot that is not CUDA memory and the p2p exchange
  without a process group raise ValueError instead of reaching a kernel. """
  from byzantinemomentum_b200 import engine, sharded
  shards = sharded.GradientShards(3, 10, "meta", exchange="collective")
  with pytest.raises(ValueError, match="on meta"):
    shards.push(0, torch.zeros(10))
  with pytest.raises(ValueError, match="slot 0 must be a contiguous float32 CUDA vector"):
    engine.gradient_scatter(torch.zeros(10), None, [torch.zeros(5), torch.zeros(5)])     # host memory
  monkeypatch.setattr(sharded, "_symmetric_memory_importable", lambda: True)
  with pytest.raises(ValueError, match="initialised process group"):
    sharded.GradientShards(3, 10, "cpu", exchange="p2p", backend=TorchDelivery())
  with pytest.raises(ValueError, match="momentum vectors for 3 workers"):
    shards = sharded.GradientShards(3, 10, "cpu", backend=TorchDelivery())
    for i in shards.workers():
      shards.push(i, torch.zeros(10))
    shards.deliver()
    shards.honests_worker([torch.zeros(10)] * 4, 0.9, 0.)

def test_rows_of_one_rank_survive_the_next_steps_pushes():
  """ The collective exchange on a single rank: the pushes of step t+1 go to the send buffer, so the
  rows `deliver()` returned for step t stay as they were until the next `deliver()`. """
  from byzantinemomentum_b200 import sharded
  shards = sharded.GradientShards(3, 50, "cpu", backend=TorchDelivery())
  for i in shards.workers():
    shards.push(i, torch.full((50,), float(i)))
  delivered = [r.clone() for r in shards.deliver()]
  for i in shards.workers():
    shards.push(i, torch.full((50,), 10. + i))
  assert all(torch.equal(a, b) for a, b in zip(shards.rows(), delivered))
  assert all(torch.equal(r, torch.full((50,), 10. + i)) for i, r in enumerate(shards.deliver()))
