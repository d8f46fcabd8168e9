#!/usr/bin/env python3
# coding: utf-8
"""Time per rank of the d-sharded phases of Multi-Krum, Bulyan, Aksel and CGE above 64 rows
(`bz_distance_partial`, `bz_distance_select`, `bz_distance_reduce`), next to `engine.Plan` at full d.

n in {65, 100, 128} with f = (n - 3) / 4 aliased Byzantine rows; d in {1,310,922; 36,489,290}.  For R in
{1, 2, 4, 8} one rank's work is timed on this GPU: phase A and phase C over rank 0's d/R columns (views of the
full rows), phase B over R gathered blocks (copies of rank 0's block: the cost of B does not depend on their
content).  Aksel's phase A includes the shard's coordinate-wise median, as `ShardedPlan` issues it.  The
exchange between A and B cannot be timed on one GPU: the multi-GPU step time is not measured here.  Every call
is warmed up, then timed with CUDA events; the median of REPS = 30 is kept.  The card's name and power limit
are read in the same run.

    python tools/distance_shards_time.py [--quick] [--out FILE.json]
"""
import ctypes, json, pathlib, subprocess, sys
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
from byzantinemomentum_b200 import _lib, engine, sharded

QUICK = "--quick" in sys.argv
REPS = 5 if QUICK else 30
NS = (65, 100, 128)
DS = (1_310_922,) if QUICK else (1_310_922, 36_489_290)
RANKS = (1, 2, 4, 8)
RULES = ("krum", "bulyan", "aksel", "cge")
dev = torch.device("cuda", 0)

def card():
  query = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
  return query[0] if query else torch.cuda.get_device_name(dev)

def events_us(fn):
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  times = []
  for _ in range(REPS):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    times.append(start.elapsed_time(stop) * 1e3)
  times.sort()
  return times[len(times) // 2]

def issue(fn, args):
  code = fn(*args)
  if code != 0:
    _lib.check(code, fn.__name__)

def main():
  line = card()
  result = dict(card=line, torch=torch.__version__, reps=REPS, cases=[])
  print("card:", line, flush=True)
  lib = _lib.lib()
  stream = torch.cuda.current_stream(dev).cuda_stream
  for d in DS:
    for n in NS:
      f = (n - 3) // 4
      gen = torch.Generator(device=dev).manual_seed(n)
      honest = torch.randn(n - f, d, device=dev, generator=gen) * torch.linspace(0.5, 1.5, n - f, device=dev)[:, None]
      byz = honest.mean(dim=0).mul_(-1.1)
      rows = list(honest.unbind(0)) + [byz] * f
      ws = torch.empty(lib.bz_distance_workspace_bytes(n), dtype=torch.uint8, device=dev)
      for gar in RULES:
        plan = engine.Plan(gar, rows, f=f)
        plan_us = events_us(plan)
        del plan
        rule = engine._rule(gar, n, f)
        for R in RANKS:
          lo, hi = sharded.shard_bounds(d, R, 0)
          shard = [g[lo:hi] for g in rows]
          ptrs = (ctypes.c_void_p * n)(*[g.data_ptr() for g in shard])
          width = n * n if rule.pair else n
          part = torch.zeros(width, dtype=torch.float64, device=dev)
          out = torch.empty(hi - lo, dtype=torch.float32, device=dev)
          meta = torch.zeros(n + 1, dtype=torch.int32, device=dev)
          median = engine.Plan("median", shard) if rule.center else None
          center = None if median is None else median.out.data_ptr()
          a, b, c = rule.phase_entries(ptrs, hi - lo, center, part.data_ptr(), 0, R, out.data_ptr(), meta.data_ptr(), ws, stream)
          def phase_a():
            if median is not None:
              median()
            issue(*a)
          phase_a()
          blocks = part.unsqueeze(0).repeat(R, 1)
          b = (b[0], (b[1][0], blocks.data_ptr()) + b[1][2:])
          issue(*b)
          case = dict(gar=gar, n=n, f=f, d=d, ranks=R, shard_d=hi - lo,
                      a_us=round(events_us(phase_a), 1), b_us=round(events_us(lambda: issue(*b)), 1),
                      c_us=round(events_us(lambda: issue(*c)), 1), plan_full_d_us=round(plan_us, 1))
          result["cases"].append(case)
          print(json.dumps(case), flush=True)
          del median, blocks
      del rows, honest, byz, ws
      torch.cuda.empty_cache()
  if "--out" in sys.argv:
    path = pathlib.Path(sys.argv[sys.argv.index("--out") + 1])
    path.parent.mkdir(parents=True, exist_ok=True)
    path.write_text(json.dumps(result, indent=1) + "\n")

if __name__ == "__main__":
  main()
