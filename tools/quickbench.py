#!/usr/bin/env python3
# coding: utf-8
"""Quick kernel timing on one GPU (development aid; bench.py is the contract)."""
import sys, time, pathlib
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
import byzantinemomentum_b200 as bz
from byzantinemomentum_b200 import engine

def timeit(fn, iters=20, warmup=3):
  for _ in range(warmup): fn()
  torch.cuda.synchronize()
  evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
  for a, b in evs:
    a.record(); fn(); b.record()
  torch.cuda.synchronize()
  ts = sorted(a.elapsed_time(b) for a, b in evs)
  return ts[len(ts) // 2], ts[0]

def main():
  from bench import peak_hbm
  peak = peak_hbm()[0]          # MEASURED_PEAKS.json, else the H100 SXM data sheet
  dev = torch.device("cuda", 0)
  bz.config.strict_status = "--nostrict" not in sys.argv
  cases = []
  for d in (79_510, 1_310_922, 36_489_290):
    for n, f in ((11, 5), (25, 10), (51, 12)):
      if n * d * 4 > 40e9: continue
      cases.append((n, f, d))
  flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
  for n, f, d in cases:
    rows = [torch.randn(d, device=dev) for _ in range(n)]
    fk = min(f, (n - 3) // 4) if n >= 7 else 1
    rules = [("average", lambda: engine.average(rows), n + 1),
             ("median", lambda: engine.median(rows), n + 1),
             ("trmean", lambda: engine.trmean(rows, f), n + 1),
             ("phocas", lambda: engine.phocas(rows, f), n + 1),
             ("meamed", lambda: engine.meamed(rows, f), n + 1),
             ("krum", lambda: engine.krum(rows, fk, n - fk - 2), n + (n - fk - 2) + 1),
             ("bulyan", lambda: engine.bulyan(rows, fk, n - fk - 2), n + (n - fk - 2) + 1),
             ("aksel", lambda: engine.aksel(rows, fk), 2 * n + (n + 1) // 2 + 3),
             ("cge", lambda: engine.cge(rows, fk), n + (n - fk) + 1)]
    if n <= 11: rules.append(("brute", lambda: engine.brute(rows, 3), n + (n - 3) + 1))
    for name, fn, units in rules:
      def step():
        flush.zero_() if d * n * 4 < 512e6 else None
        return fn()
      # time only fn: flush outside the event pair
      for _ in range(3): fn()
      torch.cuda.synchronize()
      ts = []
      for _ in range(10 if d > 5e6 else 30):
        if d * n * 4 < 512e6: flush.zero_()
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
      ts.sort()
      med = ts[len(ts) // 2]
      gbs = units * d * 4 / (med * 1e-3) / 1e9
      print(f"{name:8s} n={n:2d} f={f:2d} d={d:9d}  {med*1e3:9.1f} us (min {ts[0]*1e3:9.1f})  {gbs:8.1f} GB/s  {gbs/peak*100:5.1f}% of measured HBM peak  read-only {n*d*4/(med*1e-3)/1e9/peak*100:5.1f}%", flush=True)
    del rows
    torch.cuda.empty_cache()

if __name__ == "__main__":
  main()
