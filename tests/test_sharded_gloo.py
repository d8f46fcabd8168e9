# coding: utf-8
"""Multi-rank host logic of the d-sharded path under `gloo`, world_size 2, on CPU: each rank
holds half of the columns; the concatenated shards must reproduce the single-process oracle.
(The phases themselves run on the NumPy stand-in `tests/fake_backend.py`; the CUDA phases are
covered by the `-m gpu` tests.)"""

import os
import socket

import numpy as np
import pytest

torch = pytest.importorskip("torch")

CASES = [("average", {}), ("median", {}), ("trmean", dict(f=3)), ("phocas", dict(f=3)), ("meamed", dict(f=3)),
         ("krum", dict(f=3)), ("krum", dict(f=3, m=2)), ("bulyan", dict(f=2)), ("brute", dict(f=3)),
         ("aksel", dict(f=3)), ("aksel", dict(f=3, mode="n-f")), ("cge", dict(f=3))]

def _inputs():
  n, nb, d = 11, 3, 601
  gen = torch.Generator().manual_seed(2024)
  mu = torch.randn(d, generator=gen)
  honest = mu[None, :] + torch.linspace(0.5, 1.5, n - nb)[:, None] * torch.randn(n - nb, d, generator=gen)
  byz = honest.mean(dim=0).mul(-1.1)
  return [honest[i] for i in range(n - nb)] + [byz] * nb

def _worker(rank, world, port, queue):
  import sys, pathlib
  root = pathlib.Path(__file__).resolve().parent.parent
  sys.path.insert(0, str(root)); sys.path.insert(0, str(root / "tests"))
  import torch.distributed as dist
  from byzantinemomentum_b200 import sharded
  from fake_backend import OracleBackend
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    rows = _inputs()
    d = rows[0].shape[0]
    per = (d + world - 1) // world
    lo, hi = rank * per, min(d, (rank + 1) * per)
    shard = [r[lo:hi].contiguous() for r in rows]
    out = {}
    for i, (gar, params) in enumerate(CASES):
      res, sel = sharded.aggregate(gar, shard, backend=OracleBackend(), return_selection=True, **params)
      out[i] = (res.numpy().copy(), None if sel is None else sel.numpy().copy())
    study = {}
    for tag, samples in (("all", shard), ("one", shard[:1]), ("none", [])):
      avg, norm_avg, norm_dev, norm_max = sharded.compute_avg_dev_max(samples, backend=OracleBackend())
      study[tag] = (None if avg is None else avg.numpy().copy(), norm_avg, norm_dev, norm_max)
    if rank == 1:                                       # a NaN on one rank only must reach every rank
      poisoned = [r.clone() for r in shard]
      poisoned[2][5] = float("nan")
    else:
      poisoned = shard
    study["nan"] = sharded.compute_avg_dev_max(poisoned, backend=OracleBackend())[1:]
    out["study"] = study
    # model update on the shard + all-gather of the parameters (ragged and even splits)
    upd = {}
    for dd in (d, d - 1):
      params = torch.linspace(-1., 1., dd)
      grad = torch.sin(torch.arange(dd, dtype=torch.float32))
      l, h = sharded.shard_bounds(dd, world, rank)
      for wd in (0., 0.01):
        mine = params.clone()
        sharded.apply_update(mine, grad[l:h].clone(), 0.05, weight_decay=wd)
        upd[(dd, wd)] = mine.numpy().copy()
    out["update"] = upd
    out["replicated"] = sharded.replicate(sharded.aggregate("trmean", shard, f=3, backend=OracleBackend())).numpy().copy()
    queue.put((rank, lo, hi, out))
  finally:
    dist.destroy_process_group()

def _exchange_worker(rank, world, port, queue):
  """ Rank 0 holds aligned rows, rank 1 views that start one float in (as `shard_bounds` gives an odd
  shard start); symmetric memory counts as available on both. """
  import sys, pathlib
  root = pathlib.Path(__file__).resolve().parent.parent
  sys.path.insert(0, str(root))
  import torch.distributed as dist
  from byzantinemomentum_b200 import sharded
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    base = [torch.zeros(65) for _ in range(7)]
    rows = [b[:64] for b in base] if rank == 0 else [b[1:] for b in base]
    aligned = sharded.rows_aligned(rows)
    got = {"aligned": aligned}
    for gar in ("krum", "bulyan", "cge"):
      for request in ("auto", "fused", "p2p", "nccl"):
        try:
          got[(gar, request)] = sharded.choose_exchange(gar, request, aligned, True)
        except ValueError:
          got[(gar, request)] = "refused"
    got["no symmetric memory"] = sharded.choose_exchange("krum", "auto", True, rank == 0)
    got["both aligned"] = sharded.choose_exchange("krum", "auto", True, True)
    queue.put((rank, got))
  finally:
    dist.destroy_process_group()

def test_ranks_agree_on_the_exchange():
  """ Each rank's own rows would pick "fused" on rank 0 and "p2p" on rank 1: two protocols that never
  meet.  The choice is agreed across the group, and an infeasible explicit request fails everywhere. """
  import torch.multiprocessing as mp
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
  ctx = mp.get_context("spawn")
  queue = ctx.Queue()
  procs = [ctx.Process(target=_exchange_worker, args=(r, 2, port, queue)) for r in range(2)]
  for p in procs:
    p.start()
  got = dict(queue.get(timeout=180) for _ in procs)
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  assert got[0]["aligned"] and not got[1]["aligned"]
  assert got[0] == dict(got[1], aligned=True), "the ranks chose different exchanges"
  for gar in ("krum", "bulyan", "cge"):
    assert got[0][(gar, "auto")] == "p2p"
    assert got[0][(gar, "fused")] == "refused"
    assert got[0][(gar, "p2p")] == "p2p" and got[0][(gar, "nccl")] == "nccl"
  assert got[0]["no symmetric memory"] == "nccl"
  assert got[0]["both aligned"] == "fused"

def test_two_rank_sharding_matches_single_process():
  import torch.multiprocessing as mp
  from oracle import byzoracle as orc
  import parity
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
  ctx = mp.get_context("spawn")
  queue = ctx.Queue()
  procs = [ctx.Process(target=_worker, args=(r, 2, port, queue)) for r in range(2)]
  for p in procs:
    p.start()
  got = [queue.get(timeout=180) for _ in procs]
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  got.sort(key=lambda x: x[0])
  rows = [r.numpy() for r in _inputs()]
  for i, (gar, params) in enumerate(CASES):
    full = np.concatenate([g[3][i][0] for g in got])
    sels = [g[3][i][1] for g in got]
    ref = orc.GARS[gar](rows, **params)
    if gar in ("phocas", "meamed", "bulyan"):
      parity.assert_close_scaled(full, ref, parity.column_scale(np.stack(rows)), f"{gar} sharded")
    else:
      parity.assert_bit_exact(full, ref, f"{gar} sharded")
    if sels[0] is not None:
      assert np.array_equal(sels[0], sels[1]), f"{gar}: ranks derived different selections"

  # study metrics: shards of the average concatenate to the oracle's, scalars agree on every rank
  import math
  for tag, samples in (("all", rows), ("one", rows[:1]), ("none", [])):
    ref_avg, ref_norm, ref_dev, ref_max = orc.compute_avg_dev_max(samples)
    per_rank = [g[3]["study"][tag] for g in got]
    if ref_avg is None:
      assert all(r[0] is None for r in per_rank)
    else:
      parity.assert_bit_exact(np.concatenate([r[0] for r in per_rank]), ref_avg, f"sharded average ({tag})")
    assert per_rank[0][1:] == per_rank[1][1:] or all(math.isnan(a) and math.isnan(b) for a, b in zip(per_rank[0][1:], per_rank[1][1:]) if a != b)
    for got_value, ref_value in zip(per_rank[0][1:], (ref_norm, ref_dev, ref_max)):
      if math.isnan(ref_value):
        assert math.isnan(got_value)
      else:
        assert abs(got_value - ref_value) <= 1e-12 * abs(ref_value)
  for r in (0, 1):
    norm_avg, norm_dev, norm_max = got[r][3]["study"]["nan"]
    assert math.isnan(norm_avg) and math.isnan(norm_dev) and math.isnan(norm_max)
  # sharded model update: every rank ends with the parameters a replicated torch SGD step gives
  for dd in (601, 600):
    for wd in (0., 0.01):
      params = torch.nn.Parameter(torch.linspace(-1., 1., dd))
      params.grad = torch.sin(torch.arange(dd, dtype=torch.float32))
      torch.optim.SGD([params], lr=0.05, momentum=0., dampening=0., weight_decay=wd).step()
      for r in range(2):
        parity.assert_bit_exact(got[r][3]["update"][(dd, wd)], params.detach().numpy(), f"sharded SGD step d={dd} wd={wd} on rank {r}")
  # replicated output: every rank ends with the full vector (shards of 301 and 300 columns)
  for r in (0, 1):
    parity.assert_bit_exact(got[r][3]["replicated"], orc.trmean(rows, 3), f"replicated output on rank {r}")
