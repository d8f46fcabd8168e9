#!/usr/bin/env python3
# coding: utf-8
""" Time of the study step (attack.py:846-866) per training step on CUDA gradients:
  stock     the reference's statements as they are (library kernels, one `.item()` per quantity);
            taken from the installed reference (`tools.compute_avg_dev_max`) when it is there
  k6        stock statements with `tools.compute_avg_dev_max` swapped (`plugin.install_tools`)
  fused     `engine.study_step`: K6 x (2 or 3) + three `bz_rowdots` passes, ONE host read
Wall clock around a synchronised step (the block is host-sync bound): python tools/study_time.py [n d pasts] """
import math
import pathlib
import sys
import time

import torch

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import byzantinemomentum_b200 as bz
from byzantinemomentum_b200 import engine

def stock_block(avg_dev_max, sampleds, honests, attacks, defense, pasts, momentum):
  s_avg, s_norm, _, _ = avg_dev_max(sampleds)
  h_avg, h_norm, _, _ = avg_dev_max(honests)
  a_avg, a_norm, _, _ = avg_dev_max(attacks)
  d_norm = defense.norm().item()
  defense.abs().max().item()
  out = [torch.dot(s_avg, h_avg).div_(s_norm).div_(h_norm).item(), torch.dot(s_avg, a_avg).div_(s_norm).div_(a_norm).item(),
         torch.dot(s_avg, defense).div_(s_norm).div_(d_norm).item(), torch.dot(h_avg, a_avg).div_(h_norm).div_(a_norm).item(),
         torch.dot(h_avg, defense).div_(h_norm).div_(d_norm).item(), torch.dot(a_avg, defense).div_(a_norm).div_(d_norm).item()]
  if pasts:
    out.append(torch.dot(s_avg, pasts[0][0]).div_(s_norm).div_(pasts[0][1]).item())
    out.append(momentum * sum(momentum ** i * torch.dot(s_avg, g).item() for i, (g, _) in enumerate(pasts)))
  return out

def library_avg_dev_max(samples):      # what tools/pytorch.py:97-125 does, with library calls
  avg = samples[0].clone()
  for s in samples[1:]:
    avg.add_(s)
  avg.div_(len(samples))
  norm = avg.norm().item()
  var = 0.
  for s in samples:
    var += s.sub(avg).norm().item() ** 2
  return avg, norm, math.sqrt(var / (len(samples) - 1)), avg.abs().max().item()

def main():
  n, d, npast = (int(x) for x in sys.argv[1:4]) if len(sys.argv) >= 4 else (25, 1310922, 2)
  f = 5
  dev = "cuda:0"
  sampleds = [torch.randn(d, device=dev) for _ in range(n - f)]
  honests = [g * 0.1 + 1. for g in sampleds]           # momentum placement: other tensors (attack.py:799-808)
  attacks = [torch.randn(d, device=dev) for _ in range(f)]
  defense = torch.randn(d, device=dev)
  pasts = [(g, g.norm().item()) for g in (torch.randn(d, device=dev) for _ in range(npast))]
  stock = library_avg_dev_max
  try:
    import os
    places = ([pathlib.Path(os.environ["BYZ_REFERENCE"])] if os.environ.get("BYZ_REFERENCE") else [])
    ref = next((q.resolve() for q in places if (q / "tools" / "__init__.py").exists() and (q / "attack.py").exists()), None)
    if ref is not None:
      sys.path.insert(0, str(ref))
      import tools as reftools
      stock = reftools.compute_avg_dev_max
  except Exception:
    pass
  arms = {
    "stock": lambda: stock_block(stock, sampleds, honests, attacks, defense, pasts, 0.9),
    "k6": lambda: stock_block(bz.compute_avg_dev_max, sampleds, honests, attacks, defense, pasts, 0.9),
    "fused": lambda: engine.study_step(sampleds, honests, attacks, defense, pasts, 0.9),
  }
  print(f"study step, n_study={n - f} attacks={f} d={d} pasts={npast}; stock compute_avg_dev_max: {'reference' if stock is not library_avg_dev_max else 'library restatement'}")
  for name, fn in arms.items():
    for _ in range(5):
      fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(30):
      t0 = time.perf_counter()
      fn()
      torch.cuda.synchronize()
      times.append(time.perf_counter() - t0)
    times.sort()
    print(f"  {name:6s} median {times[len(times) // 2] * 1e3:8.3f} ms   min {times[0] * 1e3:8.3f} ms")

if __name__ == "__main__":
  main()
