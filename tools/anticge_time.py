#!/usr/bin/env python3
# coding: utf-8
"""Time the attack against CGE on one GPU: `engine.AntiCGE` (K2' + K10 + K11), its CUDA graph replay, and the
reference's statements (attacks/anticge.py:59-78, restated with the same torch calls: n + 1 host reads of a
norm, n norm reductions and maxpos + 1 `add_` passes) on the same rows, with CUDA events.  Prints one JSON line
per (n, d) with the card's name and power limit, read in the same run, and the HBM floor
(nh + maxpos + 3)·4·d / 3.35 TB/s (K2' reads the rows, K10 reads maxpos of them and writes the row, K11 reads and
writes it again).

    python tools/anticge_time.py [--n 25 100] [--d 1310720] [--iters 200] [--out results/anticge_time.json]
"""

import argparse
import json
import math
import pathlib
import subprocess
import sys

import torch

sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import byzantinemomentum_b200 as bz  # noqa: E402

HBM = 3.35e12

def reference(grad_honests, f_decl, f_real):
  if f_real > f_decl:
    byz = torch.empty_like(grad_honests[0])
    byz.copy_(torch.tensor((math.nan,), dtype=byz.dtype))
    return [byz] * f_real
  def byznorm(grad):
    norm = grad.norm().item()
    return norm if math.isfinite(norm) else math.inf
  normed = sorted(((byznorm(grad), grad) for grad in grad_honests), key=lambda pair: pair[0])
  maxpos = len(grad_honests) - f_decl
  maxnorm = math.nextafter(normed[maxpos][0], 0)
  attack = normed[0][1].clone().detach_()
  for _, grad in normed[:maxpos]:
    attack.add_(grad)
  attnorm = attack.norm().item()
  if attnorm > 0:
    attack.mul_(-maxnorm / attnorm)
  return [attack] * f_real

def card():
  try:
    text = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in text.split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)
  except Exception as err:                       # the number is still a number; say what is missing
    return dict(gpu=torch.cuda.get_device_name(), power_limit=f"unavailable ({err})")

def time_us(fn, iters):
  for _ in range(5):
    fn()
  torch.cuda.synchronize()
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(iters):
    fn()
  stop.record()
  stop.synchronize()
  return start.elapsed_time(stop) * 1e3 / iters

def main():
  parser = argparse.ArgumentParser()
  parser.add_argument("--n", type=int, nargs="+", default=[25, 100])
  parser.add_argument("--d", type=int, default=1310720)
  parser.add_argument("--iters", type=int, default=200)
  parser.add_argument("--out", default=None)
  args = parser.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("no CUDA device: this tool times the H100 and has nothing to measure here")
  info = card()
  lines = []
  for nh in args.n:
    f_decl = nh // 4
    maxpos = nh - f_decl
    gen = torch.Generator(device="cuda").manual_seed(nh)
    rows = [torch.randn(args.d, device="cuda", generator=gen) * (0.5 + i / nh) for i in range(nh)]
    attack = bz.engine.AntiCGE(rows, f_decl, f_decl)
    replay = attack.graph()
    ours = attack()[0].clone()
    ref = reference(rows, f_decl, f_decl)[0]
    rel = ((ours - ref).abs() / ref.abs()).max().item()
    device_us = time_us(attack, args.iters)
    graph_us = time_us(replay, args.iters)
    ref_us = time_us(lambda: reference(rows, f_decl, f_decl), max(10, args.iters // 10))
    floor_us = (nh + maxpos + 3) * 4 * args.d / HBM * 1e6
    line = dict(nh=nh, f_decl=f_decl, maxpos=maxpos, d=args.d, device_us=round(device_us, 1), graph_us=round(graph_us, 1),
                reference_us=round(ref_us, 1), hbm_floor_us=round(floor_us, 1), max_rel_diff_vs_reference=rel, **info)
    print(json.dumps(line), flush=True)
    lines.append(line)
  if args.out:
    pathlib.Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    pathlib.Path(args.out).write_text("\n".join(json.dumps(x) for x in lines) + "\n")

if __name__ == "__main__":
  main()
