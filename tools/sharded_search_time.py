#!/usr/bin/env python3
# coding: utf-8
"""Times of the line search on the d-sharded path, on one GPU (one JSON line per measurement):

  search     `sharded.ShardedLineSearch` at world size 1, with its collective exchange ("nccl") and with the
             exchange inside its kernels ("fused", on a plain device buffer), against `engine.LineSearch`:
             16 evaluations of `little`'s direction (factor -16, `negative`), n = 25 (f = 5), for
             Multi-Krum, the trimmed mean and the median, at d = 1,310,922 and at d_r = 163,866 (rank 0's
             shard at R = 8).  The searches issued and finished on the device (no result() read), CUDA
             events around each; the three records are checked bit-identical.
  phase_a    phase A of one evaluation on that shard, n = 25 and n = 51: `bz_pairdist_partial_reuse`
             with the previous evaluation's table (only the candidate's pairs) and without a table.
The two runs of a pair alternate, every shape is warmed up first; medians of REPS.  The card's name and
power limit are read in the same run.  Multi-GPU times need a node with several GPUs: not measured here."""
import ctypes, json, pathlib, subprocess, sys
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
from byzantinemomentum_b200 import _lib, engine, sharded
dev = torch.device("cuda", 0)
REPS = 30

def card():
  query = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
  return query[0] if query else torch.cuda.get_device_name(dev)

def event_ms(fn):
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  fn()
  end.record()
  end.synchronize()
  return start.elapsed_time(end)

def alternate(*fns, warm=3):
  """ Median ms of each of `fns`, run in turns after `warm` runs of each. """
  for _ in range(warm):
    for fn in fns:
      fn()
  torch.cuda.synchronize()
  times = [[] for _ in fns]
  for _ in range(REPS):
    for fn, t in zip(fns, times):
      t.append(event_ms(fn))
  return tuple(sorted(t)[REPS // 2] for t in times)

def rows(n, d, seed):
  gen = torch.Generator(device=dev).manual_seed(seed)
  buf = torch.randn((n, (d + 63) // 64 * 64), device=dev, generator=gen)
  return [buf[i, :d] for i in range(n)]

def search_times(tag):
  n, f = 25, 5
  for d in (1_310_922, 163_866):
    honest = rows(n - f, d, 1)
    stck = torch.stack(honest)
    avg, att = stck.mean(dim=0), stck.var(dim=0).sqrt_()
    for gar in ("krum", "trmean", "median"):
      single = engine.LineSearch(gar, honest, f, f, avg, att, 16, negative=True)
      shard = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, 16, negative=True, exchange="nccl")
      fused = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, 16, negative=True, exchange="fused")
      t_single, t_shard, t_fused = alternate(single, shard, fused)
      same = all(torch.equal(single.record[:-1].view(torch.int64), s.record[:-1].view(torch.int64)) for s in (shard, fused))
      print(json.dumps(dict(what="search", card=tag, gar=gar, n=n, d=d, evals=16, line_search_ms=round(t_single, 4),
                            sharded_world1_ms=round(t_shard, 4), fused_world1_ms=round(t_fused, 4),
                            sharded_per_eval_extra_us=round((t_shard - t_single) / 16 * 1e3, 2),
                            fused_per_eval_extra_us=round((t_fused - t_single) / 16 * 1e3, 2), records_identical=same)), flush=True)

def phase_a_times(tag):
  lib = _lib.lib()
  d = 163_866
  stream = torch.cuda.current_stream().cuda_stream
  for n in (25, 51):
    f = 5 if n == 25 else 12
    honest = rows(n - f, d, 2)
    byz = torch.empty((d + 63) // 64 * 64, device=dev)[:d]
    ptrs = (ctypes.c_void_p * n)(*[g.data_ptr() for g in honest + [byz] * f])
    old_index = (ctypes.c_int32 * n)(*(list(range(n - f)) + [-1] * f))
    ws = torch.empty(int(lib.bz_workspace_bytes(n)), dtype=torch.uint8, device=dev)
    part = torch.empty((n, n), dtype=torch.float64, device=dev)
    tables = torch.empty((2, 64 * 64), dtype=torch.float64, device=dev)
    mode = ctypes.c_int(-1)
    def call(cache_in, u_old, index):
      rc = lib.bz_pairdist_partial_reuse(ptrs, n, d, part.data_ptr(), index, cache_in, u_old, tables[1].data_ptr(),
                                         ctypes.byref(mode), ws.data_ptr(), ws.numel(), stream)
      _lib.check(rc, "bz_pairdist_partial_reuse")
    byz.copy_(honest[0])
    rc = lib.bz_pairdist_partial_reuse(ptrs, n, d, part.data_ptr(), None, None, 0, tables[0].data_ptr(),
                                       ctypes.byref(mode), ws.data_ptr(), ws.numel(), stream)
    _lib.check(rc, "bz_pairdist_partial_reuse")
    modes = []
    reuse = lambda: (call(tables[0].data_ptr(), n - f + 1, old_index), modes.append(mode.value))
    full = lambda: call(None, 0, None)
    t_reuse, t_full = alternate(reuse, full)
    assert set(modes) == {1}, modes
    print(json.dumps(dict(what="phase_a", card=tag, n=n, d_r=d, reuse_us=round(t_reuse * 1e3, 2), full_us=round(t_full * 1e3, 2),
                          speedup=round(t_full / t_reuse, 2))), flush=True)

if __name__ == "__main__":
  if not torch.cuda.is_available():
    sys.exit("sharded_search_time.py measures on a GPU: none found")
  engine.config.strict_status = False
  tag = card()
  search_times(tag)
  phase_a_times(tag)
