#!/usr/bin/env python3
# coding: utf-8
"""Per-call time of the coordinate-wise rules above 128 rows (`bz_coordinate_many`, through `engine.Plan`):
n in {129, 256, 512, 1024}, f = n // 4, d = 1,310,922, every row a distinct vector.

Per call: microseconds from CUDA events around each call (every shape warmed up first, median of REPS
calls), and beside it the HBM floor of the call: n * d * 4 bytes read at the 3.35 TB/s of the H100 SXM
data sheet (arithmetic, not measured: 0.40 ms at n = 256, 1.60 ms at n = 1024).  The card's name and
power limit are read in the same run.  Nothing gates on these numbers; they record what the kernels reach.

    python tools/coordinate_many_time.py [--quick] [--out FILE.json]
"""
import json, pathlib, statistics, subprocess, sys
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
from byzantinemomentum_b200 import engine

HBM_BYTES_PER_S = 3.35e12
QUICK = "--quick" in sys.argv
REPS = 5 if QUICK else 20
NS = (129, 256, 512, 1024)
D = 1_310_922
RULES = ("average", "median", "trmean", "phocas", "meamed")
dev = torch.device("cuda", 0)

def card():
  query = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
  return query[0] if query else torch.cuda.get_device_name(dev)

def time_plan(plan):
  plan()
  plan()
  torch.cuda.synchronize(dev)
  times = []
  for _ in range(REPS):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    plan()
    stop.record()
    stop.synchronize()
    times.append(start.elapsed_time(stop) * 1e3)
  return statistics.median(times)

def main():
  results = dict(card=card(), d=D, reps=REPS, rows=[])
  print(f"card: {results['card']}   d = {D:,}")
  print(f"{'n':>5} {'rule':>8} {'us/call':>10} {'HBM floor us':>13} {'floor/time':>10}")
  for n in NS:
    rows = [torch.randn(D, device=dev) for _ in range(n)]
    floor_us = n * D * 4 / HBM_BYTES_PER_S * 1e6
    for rule in RULES:
      plan = engine.Plan(rule, rows, f=None if rule in ("average", "median") else n // 4)
      us = time_plan(plan)
      results["rows"].append(dict(n=n, rule=rule, us=round(us, 1), hbm_floor_us=round(floor_us, 1)))
      print(f"{n:>5} {rule:>8} {us:>10.1f} {floor_us:>13.1f} {floor_us / us:>10.2f}", flush=True)
    del rows, plan
    torch.cuda.empty_cache()
  if "--out" in sys.argv:
    pathlib.Path(sys.argv[sys.argv.index("--out") + 1]).write_text(json.dumps(results, indent=1))

if __name__ == "__main__":
  main()
