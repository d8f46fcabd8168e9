#!/usr/bin/env python3
# coding: utf-8
"""Eager against CUDA-graph replay of the d-sharded line search, on one GPU (one JSON line per shape):
`sharded.ShardedLineSearch(exchange="fused")` on one rank (a plain device buffer in the FusedExchange
layout) called eagerly and replayed from `graph()`, next to `engine.LineSearch` eagerly and from its
`graph()`: n = 25, f = 5, 16 evaluations of `little`'s direction (`negative`), for Multi-Krum, the trimmed
mean and the median, at d = 163,866 (rank 0's shard of the headline model at R = 8) and d = 1,310,922.
The four runs alternate after a warm-up; CUDA events around each run (issued, not read back), median of
REPS.  The records of the four are checked bit-identical.  The card's name and power limit are read in the
same run.  Multi-GPU gains need a node with several GPUs (tools/search_peers_check.py --graph)."""
import json, pathlib, subprocess, sys
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
from byzantinemomentum_b200 import engine, sharded
dev = torch.device("cuda", 0)
REPS = 30

def card():
  query = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
  return query[0] if query else torch.cuda.get_device_name(dev)

def event_ms(fn):
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  fn()
  end.record()
  end.synchronize()
  return start.elapsed_time(end)

def alternate(*fns, warm=3):
  """ Median ms of each of `fns`, run in turns after `warm` runs of each. """
  for _ in range(warm):
    for fn in fns:
      fn()
  torch.cuda.synchronize()
  times = [[] for _ in fns]
  for _ in range(REPS):
    for fn, t in zip(fns, times):
      t.append(event_ms(fn))
  return tuple(sorted(t)[REPS // 2] for t in times)

def rows(n, d, seed):
  gen = torch.Generator(device=dev).manual_seed(seed)
  buf = torch.randn((n, (d + 63) // 64 * 64), device=dev, generator=gen)
  return [buf[i, :d] for i in range(n)]

def main():
  tag = card()
  n, f, evals = 25, 5, 16
  for d in (163_866, 1_310_922):
    honest = rows(n - f, d, 1)
    stck = torch.stack(honest)
    avg, att = stck.mean(dim=0), stck.var(dim=0).sqrt_()
    for gar in ("krum", "trmean", "median"):
      single = engine.LineSearch(gar, honest, f, f, avg, att, evals, negative=True)
      fused = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, evals, negative=True, exchange="fused")
      single_graph, fused_graph = single.graph(), fused.graph()
      t = alternate(fused, fused_graph, single, single_graph)
      torch.cuda.synchronize()
      same = torch.equal(fused.record[:-1].view(torch.int64), single.record[:-1].view(torch.int64))
      print(json.dumps(dict(card=tag, gar=gar, n=n, d=d, evals=evals, fused_eager_ms=round(t[0], 4), fused_graph_ms=round(t[1], 4),
                            line_search_eager_ms=round(t[2], 4), line_search_graph_ms=round(t[3], 4),
                            epoch=fused._fx.epoch, records_identical=bool(same))), flush=True)

if __name__ == "__main__":
  if not torch.cuda.is_available():
    sys.exit("sharded_graph_time.py measures on a GPU: none found")
  engine.config.strict_status = False
  main()
