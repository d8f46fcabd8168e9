#!/usr/bin/env python3
# coding: utf-8
"""Time of the attacks' line search against Multi-Krum, Bulyan, Aksel and CGE above 128 rows
(`LineSearch(..., many_distance=True)`, `bz_distance_line_search_many`, libbyzagg_many_search.so).

At n in {129, 256, 512, 1024}, d = 1,310,922, f_real = f_decl = (n - 3) // 4 (Bulyan's largest f), nh = n - f_real
honest rows, so u = nh + 1 unique rows:
  search16_us     one search of 16 evaluations (CUDA events, median of REPS after a warm-up);
  next_eval_us    (time at 16 evaluations - time at 1) / 15: the cost of an evaluation after the first;
  plan_us         one `Plan(gar, rows, f, many=True)` call on the same rows, the cost of the stock route's evaluation;
  star_us         K2-star-many's device time per launch (torch.profiler, in a run of its own), Multi-Krum only,
                  against its HBM floor (u - 1) * d * 4 bytes at the 3.35 TB/s of the H100 SXM data sheet.
The card's name, power limit and maximum SM clock are read in the same run.

    python tools/distance_search_many_time.py [--quick] [--out FILE.json]
"""
import json, pathlib, statistics, subprocess, sys
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
from byzantinemomentum_b200 import engine

HBM_BYTES_PER_S = 3.35e12
QUICK = "--quick" in sys.argv
REPS = 3 if QUICK else 7
D = 200_003 if QUICK else 1_310_922
NS = (129, 256, 512, 1024)
GARS = ("krum", "bulyan", "aksel", "cge")
dev = torch.device("cuda", 0)

def card():
  query = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip().splitlines()
  name, watts, mhz = [s.strip() for s in query[0].split(",")]
  return name, float(watts), float(mhz)

def call_us(fn, reps=REPS):
  """ Median over `reps` calls of one call's time (CUDA events around it), after one warm-up call. """
  fn()
  torch.cuda.synchronize()
  times = []
  for _ in range(reps):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    times.append(start.elapsed_time(stop) * 1e3)
  return statistics.median(times)

def star_us(search, evals):
  """ K2-star-many's device time per launch over one search (torch.profiler). """
  from torch.profiler import profile, ProfilerActivity
  search()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    search()
    torch.cuda.synchronize()
  total = sum(ev.device_time_total for ev in prof.key_averages()
              if ev.device_type == torch.autograd.DeviceType.CUDA and "k2_star_many" in ev.key and "fold" not in ev.key)
  return total / (evals - 1)

def main():
  name, watts, mhz = card()
  gen = torch.Generator(device=dev).manual_seed(5)
  results = []
  for n in NS:
    f = (n - 3) // 4
    nh = n - f
    honest = [torch.randn(D, device=dev, generator=gen) for _ in range(nh)]
    stck = torch.stack(honest)
    avg, att = stck.mean(dim=0), stck.var(dim=0).sqrt_()
    del stck
    u = nh + 1
    for gar in GARS:
      searches = {evals: engine.LineSearch(gar, honest, f, f, avg, att, evals, many_distance=True) for evals in (1, 16)}
      t16, t1 = call_us(searches[16]), call_us(searches[1])
      byz = searches[16].byz.clone()
      plan = engine.Plan(gar, honest + [byz] * f, f=f, many=True)
      row = dict(n=n, u=u, f=f, d=D, gar=gar, search16_us=round(t16, 1), next_eval_us=round((t16 - t1) / 15, 1),
                 plan_us=round(call_us(plan), 1))
      row["next_eval_over_plan"] = round(row["next_eval_us"] / row["plan_us"], 3)
      if gar == "krum":
        floor = (u - 1) * D * 4 / HBM_BYTES_PER_S * 1e6
        star = star_us(searches[16], 16)
        row.update(star_us=round(star, 1), star_floor_us=round(floor, 1), star_over_floor=round(star / floor, 2))
      print(json.dumps(row), flush=True)
      results.append(row)
      del searches, plan
    del honest, avg, att
    torch.cuda.empty_cache()
  report = dict(card=name, power_limit_w=watts, max_sm_clock_mhz=mhz, d=D, reps=REPS, results=results)
  if "--out" in sys.argv:
    out = pathlib.Path(sys.argv[sys.argv.index("--out") + 1])
    out.parent.mkdir(parents=True, exist_ok=True)
    out.write_text(json.dumps(report, indent=1))
  print(json.dumps(dict(card=name, power_limit_w=watts, max_sm_clock_mhz=mhz)))

if __name__ == "__main__":
  main()
