#!/usr/bin/env python3
# coding: utf-8
"""Under torchrun (N >= 2): the line search on the d-sharded path with its exchanges inside the kernels
(`ShardedLineSearch(exchange="fused")`, peer memory) against the same search with collectives
("nccl").  Every rank regenerates the seeded full vectors, takes its `shard_bounds` columns in 64-float
pitched (16-byte aligned) rows, runs both searches for every rule and checks that the trace, the factor,
the status word, its shard of the Byzantine gradient and of the rule's last output are bit-identical
between the exchanges and across the ranks; it also prints the per-search time of both (slowest rank),
with the card's name and power limit.
--graph: the fused search is also captured (`ShardedLineSearch.graph()`, whose exchanges take their epoch
from the buffer) and replayed around an eager search on the same buffer; the replays must give the eager
fused search's bits on every rank, and their time (slowest rank) is printed too.

  torchrun --nproc-per-node 8 tools/search_peers_check.py [--graph]
"""
import datetime, os, subprocess, sys, pathlib
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
import torch.distributed as dist
from byzantinemomentum_b200 import engine, sharded

GARS = ["average", "median", "trmean", "phocas", "meamed", "krum", "bulyan", "brute", "aksel", "cge"]
CASES = [(25, 1_310_922), (25, 7)]          # (n, d): a real shard, and d < R (empty shards) at R = 8
F = {"brute": 2}                            # f = 5 otherwise; brute: C(n, n - f) <= 2^31
EVALS = 16
GRAPH = "--graph" in sys.argv                # also replay the fused search from `ShardedLineSearch.graph()`

def card():
  name = torch.cuda.get_device_name()
  try:
    limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip()
  except Exception as err:
    limit = f"unknown ({err})"
  return f"{name}, power limit {limit}"

def timeit(search, K=10):
  for _ in range(2):
    search()
  torch.cuda.synchronize()
  dist.barrier()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(K):
    search()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / K * 1e3

def main():
  rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
  torch.cuda.set_device(local)
  dev = torch.device("cuda", local)
  dist.init_process_group("nccl", device_id=dev, timeout=datetime.timedelta(seconds=300))
  engine.config.strict_status = False
  ok = True
  if rank == 0:
    print(f"{world} ranks on {card()}", flush=True)
  for n, d in CASES:
    gen = torch.Generator(device=dev).manual_seed(n + d)
    mu = torch.randn(d, device=dev, generator=gen)
    lo, hi = sharded.shard_bounds(d, world, rank)
    pitch = ((hi - lo) + 63) // 64 * 64 or 64
    for gar in GARS:
      f = F.get(gar, 5)
      full = [mu + (0.5 + i / (n - f)) * torch.randn(d, device=dev, generator=gen) for i in range(n - f)]
      stck = torch.stack(full)
      vectors = full + [stck.mean(dim=0), stck.var(dim=0).sqrt_()]
      buf = torch.zeros((len(vectors), pitch), device=dev)
      rows = [buf[i, :hi - lo].copy_(v[lo:hi]) for i, v in enumerate(vectors)]
      honest, avg, att = rows[:n - f], rows[n - f], rows[n - f + 1]
      runs = {}
      for exchange in ("nccl", "fused"):
        search = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, EVALS, negative=True, exchange=exchange)
        search()
        torch.cuda.synchronize()
        runs[exchange] = (search.record.clone(), search.byz.clone(), search._shard.out.clone(), timeit(search) if d > 1000 else 0.)
        if exchange == "fused" and GRAPH:
          # the captured search (after graph()'s own eager warm-up), then an eager one between two replays
          replay = search.graph()
          replay()
          search()
          replay()
          torch.cuda.synchronize()
          runs["graph"] = (search.record.clone(), search.byz.clone(), search._shard.out.clone(), timeit(replay) if d > 1000 else 0.)
      if GRAPH:
        (rec_g, byz_g, out_g, t_g), (rec_f, byz_f, out_f, _) = runs["graph"], runs["fused"]
        same_g = (torch.equal(rec_g.view(torch.int64), rec_f.view(torch.int64)) and torch.equal(byz_g.view(torch.int32), byz_f.view(torch.int32))
                  and torch.equal(out_g.view(torch.int32), out_f.view(torch.int32)))
        ok = ok and same_g
        worst_g = torch.tensor([t_g], device=dev)
        dist.all_reduce(worst_g, op=dist.ReduceOp.MAX)
        if rank == 0:
          print(f"n={n} d={d} {gar:7s}: fused graph replay == eager fused on every rank: {same_g}; per replay (slowest rank) "
                f"{worst_g[0]:9.1f} us", flush=True)
      (rec_c, byz_c, out_c, t_c), (rec_f, byz_f, out_f, t_f) = runs["nccl"], runs["fused"]
      same = (torch.equal(rec_c.view(torch.int64), rec_f.view(torch.int64)) and torch.equal(byz_c.view(torch.int32), byz_f.view(torch.int32))
              and torch.equal(out_c.view(torch.int32), out_f.view(torch.int32)))
      gathered = [torch.empty_like(rec_f) for _ in range(world)]
      dist.all_gather(gathered, rec_f)
      same = same and all(torch.equal(g.view(torch.int64), rec_f.view(torch.int64)) for g in gathered)
      ok = ok and same
      worst = torch.tensor([t_c, t_f], device=dev)
      dist.all_reduce(worst, op=dist.ReduceOp.MAX)
      if rank == 0:
        print(f"n={n} d={d} {gar:7s}: fused == nccl on every rank: {same}; per search (slowest rank) nccl {worst[0]:9.1f} us, "
              f"fused {worst[1]:9.1f} us", flush=True)
  flag = torch.tensor([1 if ok else 0], device=dev)
  dist.all_reduce(flag, op=dist.ReduceOp.MIN)
  if rank == 0:
    print("ALL RANKS IDENTICAL" if int(flag.item()) == 1 else "MISMATCH", flush=True)
  dist.destroy_process_group()

if __name__ == "__main__":
  main()
