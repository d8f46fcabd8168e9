#!/usr/bin/env python3
# coding: utf-8
"""Time the d-sharded factor search against Multi-Krum, Bulyan, Aksel and CGE above 64 rows on ONE rank.

n in {65, 100, 128} with f = (n - 3) / 4 aliased Byzantine rows, 16 evaluations of `little`'s direction, and two shard
widths: d = 1,310,922 and d = 4,561,162 (a 36.5M-parameter model over 8 ranks).  Per rule, n and d:
  nccl_us         `ShardedLineSearch(..., exchange="nccl", wide=True)`, eager (one rank: the gathers are copies);
  fused_us        the same with exchange="fused" (one rank: a plain device buffer);
  graph_us        the fused search captured in a CUDA graph, one replay;
  one_gpu_us      `engine.LineSearch` (`bz_distance_line_search`) on the same rows;
  plan_loop_us    16 calls of `ShardedPlan(..., exchange="nccl")` on the same rows: the rule alone, with every
                  distance pass at every call;
  first_eval_us, later_eval_us   the "nccl" search of 1 evaluation, and what each evaluation after the first adds
                  ((16 evaluations - 1 evaluation) / 15).
CUDA events around one call, median of REPS.  Only one rank is measured: the exchanges over several GPUs are not.
The card's name, power limit and maximum SM clock are read in the same run.

    python tools/sharded_search_wide_time.py [--out FILE.json]
"""
import json, pathlib, sys
ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import torch
from byzantinemomentum_b200 import engine, sharded
from distance_wide_time import card, events_us

DS = (1_310_922, 4_561_162)
NS = (65, 100, 128)
EVALS = 16
GARS = ("krum", "bulyan", "aksel", "cge")
dev = torch.device("cuda", 0)

def main():
  result = dict(card=card(), torch=torch.__version__, evals=EVALS, cases=[])
  print("card:", result["card"], flush=True)
  for d in DS:
    for n in NS:
      f = (n - 3) // 4
      gen = torch.Generator(device=dev).manual_seed(n)
      buf = engine._row_buffer(n - f, d, dev)
      buf[:, :d] = torch.randn(n - f, d, device=dev, generator=gen) * torch.linspace(0.5, 1.5, n - f, device=dev)[:, None]
      honest = [buf[i, :d] for i in range(n - f)]
      stck = torch.stack(honest)
      avg, att = stck.mean(dim=0), stck.var(dim=0).sqrt_()
      del stck
      for gar in GARS:
        def search(exchange, evals=EVALS):
          return sharded.ShardedLineSearch(gar, honest, f, f, avg, att, evals, exchange=exchange, wide=True)
        nccl, fused, one = search("nccl"), search("fused"), search("nccl", 1)
        single = engine.LineSearch(gar, honest, f, f, avg, att, EVALS)
        byz = avg + att
        plan = sharded.ShardedPlan(gar, honest + [byz] * f, f=f, exchange="nccl")
        def plan_loop():
          for _ in range(EVALS):
            plan()
        case = dict(gar=gar, n=n, d=d, f=f, nccl_us=events_us(nccl), fused_us=events_us(fused),
                    graph_us=events_us(fused.graph()), one_gpu_us=events_us(single), plan_loop_us=events_us(plan_loop),
                    first_eval_us=events_us(one))
        case["later_eval_us"] = (case["nccl_us"] - case["first_eval_us"]) / (EVALS - 1)
        case = {k: round(v, 1) if isinstance(v, float) else v for k, v in case.items()}
        result["cases"].append(case)
        print(json.dumps(case), flush=True)
        del nccl, fused, one, single, plan
      del honest, buf, avg, att
      torch.cuda.empty_cache()
  if "--out" in sys.argv:
    path = pathlib.Path(sys.argv[sys.argv.index("--out") + 1])
    path.parent.mkdir(parents=True, exist_ok=True)
    path.write_text(json.dumps(result, indent=1) + "\n")

if __name__ == "__main__":
  main()
