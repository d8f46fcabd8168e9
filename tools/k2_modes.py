#!/usr/bin/env python3
# coding: utf-8
"""Experiment (not run yet: the round-1 GPU budget ended): time per tile of the producer-warp
TMA K2 of tools/experiments/k2_producer_warp_and_row_blocks.patch under its issue/wait modes
(env BYZAGG_K2_MODE, read at every launch): bit 0 = only lane 0 waits on `empty`, bit 1 = lane 0
issues every copy, bit 2 = the producer is warp 0 (the oldest warp, scheduler priority) instead of
the last warp.  2 and 4 tiles per CTA need no `empty` wait at all (4 stages), so the step from
4 to 5 tiles isolates that wait.  Apply the patch, rebuild, then:
    python tools/k2_modes.py
"""
import os, sys, pathlib, time
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
import byzantinemomentum_b200 as bz
dev = torch.device("cuda", 0)
n = 25
sms = torch.cuda.get_device_properties(dev).multi_processor_count
for tiles in (2, 4, 5, 8, 16):
  d = sms * 512 * tiles
  rows = [torch.randn(d, device=dev) for _ in range(n)]
  for mode in (0, 1, 2, 3, 4, 5):
    os.environ["BYZAGG_K2_MODE"] = str(mode)
    bz.engine.pairdist_partial(rows); torch.cuda.synchronize()
    t0 = time.perf_counter()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); bz.engine.pairdist_partial(rows); b.record(); torch.cuda.synchronize()
    print("tiles/CTA %2d mode %d: %10.1f us (wall %.3f s)" % (tiles, mode, a.elapsed_time(b) * 1e3, time.perf_counter() - t0), flush=True)
