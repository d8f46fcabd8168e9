#!/usr/bin/env python3
# coding: utf-8
"""Under torchrun (N >= 2): gradient delivery to the d-sharded path (`sharded.GradientShards`).
Every rank regenerates the seeded full gradients and checks that both exchanges ("p2p" through
symmetric memory, "collective" through one all_to_all_single) deliver exactly its columns of
`GradientStack.push`'s rows, bit-identical between the exchanges; that `ShardedPlan` over the delivered
rows selects what the single-GPU `Plan` selects; and prints the per-step time of this rank's pushes
plus `deliver` for both exchanges, next to one `GradientStack` pass over all n workers on one GPU.

  torchrun --nproc-per-node 8 tools/shards_check.py
"""
import datetime, os, subprocess, sys, pathlib
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
import torch.distributed as dist
import byzantinemomentum_b200 as bz
from byzantinemomentum_b200 import sharded

CASES = [(25, 5, 1_310_922), (51, 12, 36_489_290)]       # (n, f, d)
CLIP = 1500.

def grad(i, d, dev):
  gen = torch.Generator(device=dev).manual_seed(1000 + i)
  return torch.randn(d, device=dev, generator=gen) * (0.5 + i / 25)

def timeit(fn, K, warmup=3):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  dist.barrier()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(K):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / K * 1e3

def card():
  name = torch.cuda.get_device_name()
  try:
    limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip()
  except Exception as err:
    limit = f"unknown ({err})"
  return f"{name}, power limit {limit}"

def main():
  rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
  torch.cuda.set_device(local)
  dev = torch.device("cuda", local)
  dist.init_process_group("nccl", device_id=dev, timeout=datetime.timedelta(seconds=300))
  ok = True
  auto = sharded.choose_delivery("auto", sharded._symmetric_memory_importable())
  if rank == 0:
    print(f"{world} ranks on {card()}; exchange='auto' picks {auto!r}", flush=True)
  for n, f, d in CASES:
    lo, hi = sharded.shard_bounds(d, world, rank)
    stack = bz.GradientStack(n, d, dev)                       # the single-GPU rows every rank checks against
    for i in range(n):
      stack.push(i, grad(i, d, dev), clip=CLIP)
    mine = {i: grad(i, d, dev) for i in range(rank, n, world)}
    delivered, times = {}, {}
    for exchange in ("p2p", "collective"):
      shards = sharded.GradientShards(n, d, dev, exchange=exchange)
      def step():
        for i, g in mine.items():
          shards.push(i, g, clip=CLIP)
        return shards.deliver()
      rows = step()
      delivered[exchange] = [r.clone() for r in rows]
      same = all(torch.equal(r.view(torch.int32), stack.sampled()[i][lo:hi].view(torch.int32)) for i, r in enumerate(rows))
      ok = ok and same
      # ShardedPlan over the delivered rows selects what one GPU selects over the full rows
      for gar in ("krum", "bulyan"):
        plans = [sharded.ShardedPlan(gar, shards.rows(s), f=f) for s in range(shards.slots)]
        step()
        plans[shards.slot]()
        single = bz.Plan(gar, stack.sampled(), f=f)
        single()
        picked = torch.equal(plans[shards.slot].selection, single.selection)
        ok = ok and picked
        if rank == 0:
          print(f"n={n} d={d} {exchange:10s} {gar:6s}: columns exact={same} selection as one GPU={picked} ({plans[0].exchange})", flush=True)
      times[exchange] = timeit(step, 20)
      del shards
    ok = ok and all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(delivered["p2p"], delivered["collective"]))
    grads = [grad(i, d, dev) for i in range(n)] if rank == 0 else None
    t_stack = float("nan")
    if rank == 0:
      def stack_pass():
        for i, g in enumerate(grads):
          stack.push(i, g, clip=CLIP)
      for _ in range(3):
        stack_pass()
      torch.cuda.synchronize()
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(20):
        stack_pass()
      e1.record()
      torch.cuda.synchronize()
      t_stack = e0.elapsed_time(e1) / 20 * 1e3
    worst = torch.tensor([times["p2p"], times["collective"]], device=dev)
    dist.all_reduce(worst, op=dist.ReduceOp.MAX)
    if rank == 0:
      print(f"n={n} d={d} R={world}: push + deliver per step (slowest rank) p2p {worst[0]:9.1f} us, collective {worst[1]:9.1f} us | "
            f"GradientStack, all n on one GPU {t_stack:9.1f} us", flush=True)
    del stack, grads, mine
    torch.cuda.empty_cache()
  flag = torch.tensor([1 if ok else 0], device=dev)
  dist.all_reduce(flag, op=dist.ReduceOp.MIN)
  if rank == 0:
    print("ALL RANKS IDENTICAL" if int(flag.item()) == 1 else "MISMATCH", flush=True)
  dist.destroy_process_group()

if __name__ == "__main__":
  main()
