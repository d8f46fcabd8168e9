#!/usr/bin/env python3
# coding: utf-8
"""Time the d-sharded attack against CGE on ONE GPU, with CUDA events: one rank of `sharded.ShardedAntiCGE` with
the fused exchange (`bz_anticge_peers`: K2'-norms, K10 with the exchange, K11, over a plain device buffer), the same
rank with "nccl" (its four stages, no collective on one rank), the single-GPU `engine.AntiCGE` (`bz_anticge`), and
the fused call's CUDA graph replay (`bz_anticge_peers_next`).  The calls are timed in alternation, `--rounds` times
each, and the median round is reported.  The four rows must be the same bits (checked first).  Prints one JSON line
per nh with the card's name and power limit, read in the same run.  Several GPUs cannot be measured this way: what
the fused exchange saves there (two all-gathers per step) is not measured here.

    python tools/anticge_peers_time.py [--n 25 100] [--d 1310720] [--iters 200] [--rounds 5] [--out results/x.json]
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

def main():
  parser = argparse.ArgumentParser()
  parser.add_argument("--n", type=int, nargs="+", default=[25, 100])
  parser.add_argument("--d", type=int, default=1310720)
  parser.add_argument("--iters", type=int, default=200)
  parser.add_argument("--rounds", type=int, default=5)
  parser.add_argument("--out", default=None)
  args = parser.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("no CUDA device: this tool times the H100 and has nothing to measure here")
  info = card()
  lines = []
  for nh in args.n:
    f_decl = nh // 4
    gen = torch.Generator(device="cuda").manual_seed(nh)
    rows = [torch.randn(args.d, device="cuda", generator=gen) * (0.5 + i / nh) for i in range(nh)]
    fused = sharded.ShardedAntiCGE(rows, f_decl, f_decl, exchange="fused")
    nccl = sharded.ShardedAntiCGE(rows, f_decl, f_decl, exchange="nccl")
    single = bz.engine.AntiCGE(rows, f_decl, f_decl)
    replay = sharded.ShardedAntiCGE(rows, f_decl, f_decl, exchange="fused").graph()
    outs = [fused()[0], nccl()[0], replay()[0], single()[0]]
    torch.cuda.synchronize()
    same = all(torch.equal(o.view(torch.int32), outs[0].view(torch.int32)) for o in outs[:3])
    rel = ((outs[0] - outs[3]).abs() / outs[3].abs()).max().item()
    calls = dict(fused_us=fused, nccl_us=nccl, single_gpu_us=single, fused_graph_us=replay)
    times = {name: [] for name in calls}
    for _ in range(args.rounds):
      for name, fn in calls.items():
        times[name].append(time_us(fn, args.iters))
    line = dict(nh=nh, f_decl=f_decl, d=args.d, ranks=1, rounds=args.rounds, iters=args.iters,
                **{name: round(statistics.median(t), 1) for name, t in times.items()},
                spread_us={name: round(max(t) - min(t), 1) for name, t in times.items()},
                sharded_paths_bit_equal=same, max_rel_diff_vs_single_gpu=rel, multi_gpu="not measured", **info)
    print(json.dumps(line), flush=True)
    lines.append(line)
  if args.out:
    pathlib.Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    pathlib.Path(args.out).write_text("\n".join(json.dumps(x) for x in lines) + "\n")

if __name__ == "__main__":
  main()
