#!/usr/bin/env python3
# coding: utf-8
"""One GPU: cost of gradient delivery's kernels with R ranks emulated by R plain device buffers.
  * `bz_gradient_scatter` of one gradient into R slots against `GradientStack.push` of the same
    gradient (one row), with and without a clip that triggers: the same d*4 bytes read and written;
  * the owner's momentum placement of its n rows on d/R columns in one `bz_gradient_momentum` launch
    (`engine.momentum_rows`, worker and server side), against the HBM time of its bytes.
CUDA events around K back-to-back calls after a warm-up; prints one line per measurement, the card
name and its power limit first.

  python tools/shards_time.py
"""
import subprocess, sys, pathlib
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
from byzantinemomentum_b200 import engine, sharded

def per_call_us(fn, K=50):
  for _ in range(5):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(K):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / K * 1e3

def main():
  dev = torch.device("cuda", 0)
  limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
  print(f"{torch.cuda.get_device_name(dev)}, power limit {limit}", flush=True)
  for d in (1_310_922, 36_489_290):
    g = torch.randn(d, device=dev)
    stack = engine.GradientStack(1, d, dev)
    for clip in (None, 1.0):
      t_stack = per_call_us(lambda: stack.push(0, g, clip=clip))
      line = f"d={d:>10} clip={'none' if clip is None else 'on  '} GradientStack.push {t_stack:8.1f} us |"
      for R in (1, 8):
        bounds = [sharded.shard_bounds(d, R, r) for r in range(R)]
        bufs = [engine._row_buffer(1, hi - lo, dev)[0, :hi - lo] for lo, hi in bounds]
        line += f" scatter R={R} {per_call_us(lambda: engine.gradient_scatter(g, clip, bufs)):8.1f} us"
      print(line, flush=True)
  for n, d, R in ((25, 1_310_922, 8), (51, 36_489_290, 8)):
    lo, hi = sharded.shard_bounds(d, R, 0)
    buf = engine._row_buffer(n, hi - lo, dev)
    rows = [buf[i, :hi - lo] for i in range(n)]
    moms = [torch.randn(hi - lo, device=dev) for _ in range(n)]
    server = torch.randn(hi - lo, device=dev)
    honests = [torch.empty(hi - lo, device=dev) for _ in range(n)]
    t_worker = per_call_us(lambda: engine.momentum_rows(rows, 0.9, 0.1, momentums=moms), 20)
    t_server = per_call_us(lambda: engine.momentum_rows(rows, 0.9, 0.1, server=server, honests=honests), 20)
    floor_worker = n * 3 * (hi - lo) * 4 / 3.35e12 * 1e6          # read row + momentum, write momentum
    floor_server = (2 * n + 1) * (hi - lo) * 4 / 3.35e12 * 1e6    # read rows, write honest rows, read server
    print(f"momentum n={n} on {hi - lo} columns (d={d}, R={R}), one launch: worker {t_worker:8.1f} us "
          f"(HBM floor at 3.35 TB/s {floor_worker:7.1f} us), server {t_server:8.1f} us (floor {floor_server:7.1f} us)", flush=True)

if __name__ == "__main__":
  main()
