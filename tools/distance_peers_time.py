#!/usr/bin/env python3
# coding: utf-8
"""Time the d-sharded Multi-Krum, Bulyan, Aksel and CGE above 64 rows on ONE GPU, with CUDA events: one rank of
`sharded.ShardedPlan` with the fused exchange (`bz_distance_partial`, `bz_distance_select_peers` over a plain device
buffer registered as the exchange of n rows, `bz_distance_reduce`), the same rank with "nccl" (its three phases and a copy, no collective on one rank),
the single-GPU `engine.Plan` (`bz_distance`), and the fused plan's CUDA graph replay (`bz_distance_select_peers_next`).
The four calls are timed in alternation, `--rounds` times each, and the median round is reported.  The fused call,
its replay and "nccl" must give the same bits at every timed size (checked first).  Prints one JSON line per (n, d,
rule) with the card's name and power limit, read in the same run.  Several GPUs cannot be measured this way: what
the fused exchange costs there (one CTA reading R blocks over NVLink) and saves (one all-gather) is not measured.

    python tools/distance_peers_time.py [--n 65 100 128] [--d 1310922 36489290] [--rounds 3] [--out results/x.json]
"""

import argparse
import json
import pathlib
import statistics
import sys

import torch

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import byzantinemomentum_b200 as bz  # noqa: E402
from byzantinemomentum_b200 import sharded  # noqa: E402
from anticge_time import card, time_us  # noqa: E402

RULES = ("krum", "bulyan", "aksel", "cge")

def main():
  parser = argparse.ArgumentParser()
  parser.add_argument("--n", type=int, nargs="+", default=[65, 100, 128])
  parser.add_argument("--d", type=int, nargs="+", default=[1310922, 36489290])
  parser.add_argument("--rounds", type=int, default=3)
  parser.add_argument("--out", default=None)
  args = parser.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("no CUDA device: this tool times the H100 and has nothing to measure here")
  info = card()
  lines = []
  for d in args.d:
    for n in args.n:
      gen = torch.Generator(device="cuda").manual_seed(n + d)
      block = torch.randn(n, d, device="cuda", generator=gen)
      block.mul_(torch.linspace(0.5, 1.5, n, device="cuda")[:, None])
      rows = list(block)
      iters = max(3, min(50, int(3e10 // (n * d))))
      # one rank without a process group: the fused plans share a plain device buffer registered for them
      sharded._registered(sharded._fused, lambda n, device, group: sharded.FusedExchange.local(n, device), n, block.device, None)
      for gar in RULES:
        f = (n - 3) // 4
        fused = sharded.ShardedPlan(gar, rows, f=f, exchange="fused")
        nccl = sharded.ShardedPlan(gar, rows, f=f, exchange="nccl")
        single = bz.engine.Plan(gar, rows, f=f)
        captured = sharded.ShardedPlan(gar, rows, f=f, exchange="fused")      # holds what the graph reads and writes
        replay = captured.graph()
        outs = [fused(), replay(), nccl(), single()]
        torch.cuda.synchronize()
        same = all(torch.equal(o.view(torch.int32), outs[2].view(torch.int32)) for o in outs[:2])
        same = same and torch.equal(fused.selection, nccl.selection)
        calls = dict(fused_us=fused, nccl_us=nccl, plan_us=single, fused_graph_us=replay)
        times = {name: [] for name in calls}
        for _ in range(args.rounds):
          for name, fn in calls.items():
            times[name].append(time_us(fn, iters))
        line = dict(gar=gar, n=n, f=f, d=d, ranks=1, rounds=args.rounds, iters=iters,
                    **{name: round(statistics.median(t), 1) for name, t in times.items()},
                    spread_us={name: round(max(t) - min(t), 1) for name, t in times.items()},
                    fused_equals_nccl_bits=same, plan_equals_nccl_bits=torch.equal(outs[3].view(torch.int32), outs[2].view(torch.int32)),
                    multi_gpu="not measured", **info)
        print(json.dumps(line), flush=True)
        lines.append(line)
        del fused, nccl, single, captured, replay
      del rows, block
      sharded._fused.clear()
      torch.cuda.empty_cache()
  if args.out:
    pathlib.Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    pathlib.Path(args.out).write_text("\n".join(json.dumps(x) for x in lines) + "\n")
  if not all(x["fused_equals_nccl_bits"] for x in lines):
    raise SystemExit("the fused exchange and \"nccl\" gave different bits")

if __name__ == "__main__":
  main()
