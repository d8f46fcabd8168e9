#!/usr/bin/env python3
# coding: utf-8
"""Time one step's factor search against Multi-Krum, Bulyan, Aksel and CGE above 64 rows.

n in {65, 100, 128} with f = (n - 3) / 4 (the largest f Bulyan takes) aliased Byzantine rows, d = 1,310,922, and the
16 evaluations of `little`'s direction (attacks/identical.py:67-77, factor -16).  Per rule and n:
  search_us      `engine.LineSearch` (`bz_distance_line_search`), eager: CUDA events around one call, median of REPS;
  graph_us       the same search captured in a CUDA graph, one replay;
  plan_loop_us   the same 16 evaluations as a host loop of `line_maximize` in which every evaluation is a full
                 `engine.Plan` call (`bz_distance`, every distance pass) plus the torch score read back to the host:
                 what the search's star passes and its device-side transitions save; wall clock, median of 5.
For Multi-Krum at n = 100 the reference's torch statements (tools/distance_wide_time.py's restatement) run a few
evaluations of the same loop: ref_eval_us is the median wall clock of one evaluation (candidate, rule, score).
The card's name, power limit and maximum SM clock are read in the same run.

    python tools/distance_search_time.py [--out FILE.json]
"""
import json, pathlib, sys, time
ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
import torch
from byzantinemomentum_b200 import engine
import line_oracle
from distance_wide_time import card, events_us, ref_krum, wall_us

D = 1_310_922
NS = (65, 100, 128)
EVALS = 16
GARS = ("krum", "bulyan", "aksel", "cge")
dev = torch.device("cuda", 0)

def main():
  result = dict(card=card(), torch=torch.__version__, d=D, evals=EVALS, cases=[])
  print("card:", result["card"], flush=True)
  for n in NS:
    f = (n - 3) // 4
    gen = torch.Generator(device=dev).manual_seed(n)
    buf = engine._row_buffer(n - f, D, dev)                 # 256-byte aligned rows, as the ring reads them
    buf[:, :D] = torch.randn(n - f, D, device=dev, generator=gen) * torch.linspace(0.5, 1.5, n - f, device=dev)[:, None]
    honest = [buf[i, :D] for i in range(n - f)]
    stck = torch.stack(honest)
    avg, att = stck.mean(dim=0), stck.var(dim=0).sqrt_()
    del stck
    for gar in GARS:
      search = engine.LineSearch(gar, honest, f, f, avg, att, EVALS)
      search_us = events_us(search)
      graph_us = events_us(search.graph())
      byz = torch.empty_like(avg)
      plan = engine.Plan(gar, honest + [byz] * f, f=f)
      def scape(x):
        torch.add(avg, att, alpha=x, out=byz)
        diff = plan().sub(avg)
        return diff.dot(diff).item()
      loop = lambda: line_oracle.line_maximize(scape, EVALS)
      loop()
      case = dict(gar=gar, n=n, f=f, unique_rows=n - f + 1, search_us=round(search_us, 1), graph_us=round(graph_us, 1),
                  plan_loop_us=round(wall_us(loop, 5), 1))
      case["plan_loop_over_search"] = round(case["plan_loop_us"] / search_us, 2)
      if gar == "krum" and n == 100:
        rows = honest + [byz] * f
        def ref_eval(x=1.0):
          torch.add(avg, att, alpha=x, out=byz)
          diff = ref_krum(rows, f).sub_(avg)
          return diff.dot(diff).item()
        ref_eval()
        case["ref_eval_us"] = round(wall_us(ref_eval, 3), 1)
        case["ref_search_us_derived"] = round(case["ref_eval_us"] * EVALS, 1)
      result["cases"].append(case)
      print(json.dumps(case), flush=True)
      del search, plan
    del honest, buf, avg, att
    torch.cuda.empty_cache()
  if "--out" in sys.argv:
    path = pathlib.Path(sys.argv[sys.argv.index("--out") + 1])
    path.parent.mkdir(parents=True, exist_ok=True)
    path.write_text(json.dumps(result, indent=1) + "\n")

if __name__ == "__main__":
  main()
