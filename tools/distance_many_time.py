#!/usr/bin/env python3
# coding: utf-8
"""Time of Multi-Krum, Bulyan, Aksel and CGE above 128 rows (`bz_distance_many`, libbyzagg_many_distance.so).

`Plan(many=True)` calls at n in {129, 256, 512, 1024}, d = 1,310,922, f = (n - 3) // 4 aliased Byzantine rows (one
tensor), so u = n - f + 1 unique rows; each call timed alone with CUDA events, median of REPS calls after a warm-up.
In the same run: `bz_distance` at n = 128 (u = 98), Multi-Krum, the bar for n = 129; and one torch.profiler pass per
(rule, n) that splits the call into its kernels (K2-many and its slice sum, K5-many, K2'-many, the reduce).
Floors, computed, not measured:
  fp32_floor_us   K2-many: u (u - 1) d lane operations over 132 SMs x 128 lanes at the card's maximum SM clock;
  hbm_floor_us    K2'-many: n * d * 4 bytes at the 3.35 TB/s of the H100 SXM data sheet.
The card's name, power limit and maximum SM clock are read in the same run.

    python tools/distance_many_time.py [--quick] [--out FILE.json]
"""
import json, pathlib, statistics, subprocess, sys
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
from byzantinemomentum_b200 import engine

HBM_BYTES_PER_S = 3.35e12
QUICK = "--quick" in sys.argv
REPS = 5 if QUICK else 21
D = 200_003 if QUICK else 1_310_922
NS = (129, 256, 512, 1024)
RULES = (("krum", "mid"), ("bulyan", "mid"), ("aksel", "mid"), ("cge", "mid"))
dev = torch.device("cuda", 0)

def card():
  query = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip().splitlines()
  name, watts, mhz = [s.strip() for s in query[0].split(",")]
  return name, float(watts), float(mhz)

def call_us(fn, reps=REPS):
  """ Median over `reps` calls of one call's time (CUDA events around it), after two warm-up calls. """
  fn(); fn()
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

def kernels_us(fn, calls=3):
  """ Per kernel name (up to its template arguments): device time per call, from torch.profiler. """
  from torch.profiler import profile, ProfilerActivity
  fn()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(calls):
      fn()
    torch.cuda.synchronize()
  out = {}
  for ev in prof.key_averages():
    if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time_total > 0:
      name = ev.key.split("(")[0].split("<")[0].replace("void ", "").replace("bz::", "")
      out[name] = out.get(name, 0.) + ev.device_time_total / calls
  return {k: round(v, 1) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}

def rows_for(n, f, d):
  gen = torch.Generator(device=dev).manual_seed(n)
  nh = n - f
  honest = torch.randn(nh, d, generator=gen, device=dev)
  byz = honest[:8].mean(dim=0).mul(-1.1)
  return honest, [honest[i] for i in range(nh)] + [byz] * f

def main():
  name, watts, mhz = card()
  result = dict(card=name, power_limit_w=watts, max_sm_mhz=mhz, d=D, reps=REPS, calls={}, kernels={}, floors={})
  print(f"{name}, power limit {watts:.0f} W, max SM clock {mhz:.0f} MHz, d = {D}", flush=True)
  lanes_per_s = 132 * 128 * mhz * 1e6
  # the bar: bz_distance at 128 rows (u = 98), timed in this run
  honest, rows = rows_for(128, 31, D)
  plan = engine.Plan("krum", rows, f=31)
  result["calls"]["krum n=128 bz_distance"] = round(call_us(plan), 1)
  del plan, rows, honest
  for n in NS:
    f = (n - 3) // 4
    u = n - f + 1
    honest, rows = rows_for(n, f, D)
    result["floors"][f"n={n}"] = dict(u=u, fp32_floor_us=round(u * (u - 1) * D / lanes_per_s * 1e6, 1),
                                      hbm_floor_us=round(n * D * 4 / HBM_BYTES_PER_S * 1e6, 1))
    for gar, mode in RULES:
      plan = engine.Plan(gar, rows, f=f, mode=mode, many=True)
      key = f"{gar} n={n}"
      result["calls"][key] = round(call_us(plan), 1)
      result["kernels"][key] = kernels_us(plan)
      print(key, result["calls"][key], result["kernels"][key], flush=True)
      del plan
    del rows, honest
    torch.cuda.empty_cache()
  print(json.dumps(result["floors"]))
  text = json.dumps(result, indent=1)
  if "--out" in sys.argv:
    pathlib.Path(sys.argv[sys.argv.index("--out") + 1]).write_text(text)
  print(text)

if __name__ == "__main__":
  main()
