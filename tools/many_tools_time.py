#!/usr/bin/env python3
# coding: utf-8
"""Time of the study metrics and of the attacks' line search against the coordinate-wise rules above 128 rows.

K6-many (`bz_avg_dev_max_many`, libbyzagg_many_tools.so) at n in {129, 256, 512, 1024}, d = 1,310,922, every
row a distinct vector, against:
  floor_us     the HBM floor (n + 1) * 4 * d bytes at the 3.35 TB/s of the H100 SXM data sheet;
  average_us   `bz_coordinate_many`'s average over the same rows, which moves the same bytes;
  torch_us     the reference's `tools.compute_avg_dev_max` statements (tools/pytorch.py:97-125: clone,
               add_, div_, norm, abs().max(), then per row sub + dot + `.item()`), on the same GPU.
K6 and the average are timed with CUDA events around CALLS back-to-back calls of the C entry points
(median of REPS samples after a warm-up); the torch statements with a wall clock around one call that
ends in its own host reads.

--search: one step's whole search (`little`'s direction, factor -16, 16 evaluations) at n = 300
(280 honest rows, f_real = f_decl = 20), d = 1,310,922, median and trimmed mean: the host loop of the
reference's statements over the `many_gars` entry against `engine.LineSearch(..., many=True)` read once.

The card's name and power limit are read in the same run.

    python tools/many_tools_time.py [--quick] [--search] [--out FILE.json]
"""
import ctypes, json, math, pathlib, subprocess, sys, time
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
import byzantinemomentum_b200 as bz
from byzantinemomentum_b200 import _lib, engine

HBM_BYTES_PER_S = 3.35e12
QUICK = "--quick" in sys.argv
REPS = 5 if QUICK else 31
CALLS = 10
NS = (129, 256, 512, 1024)
DS = (1_310_922,)
dev = torch.device("cuda", 0)

def card():
  query = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
  return query[0] if query else torch.cuda.get_device_name(dev)

def events_us(fn, calls=CALLS, reps=REPS):
  """ Median over `reps` samples of the time per call of `calls` back-to-back calls (CUDA events). """
  fn()                                                   # warm-up: module loading, attributes
  torch.cuda.synchronize()
  times = []
  for _ in range(reps):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(calls):
      fn()
    stop.record()
    stop.synchronize()
    times.append(start.elapsed_time(stop) * 1e3 / calls)
  times.sort()
  return times[len(times) // 2]

def wall_ms(fn, reps):
  fn()
  times = []
  for _ in range(reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    times.append((time.perf_counter() - t0) * 1e3)
  times.sort()
  return times[len(times) // 2]

def reference_statements(samples):
  """ tools/pytorch.py:97-125, statement for statement. """
  grad_avg = samples[0].clone().detach_()
  for grad in samples[1:]:
    grad_avg.add_(grad)
  grad_avg.div_(len(samples))
  norm_avg = grad_avg.norm().item()
  norm_max = grad_avg.abs().max().item()
  norm_var = 0.
  for grad in samples:
    grad = grad.sub(grad_avg)
    norm_var += grad.dot(grad).item()
  norm_var /= len(samples) - 1
  return grad_avg, norm_avg, math.sqrt(norm_var), norm_max

def study_times():
  lib, many, tools = _lib.lib(), _lib.many_lib(), _lib.many_tools_lib()
  cases = []
  for d in DS:
    for n in NS:
      gen = torch.Generator(device=dev).manual_seed(n)
      stack = torch.randn(n, d, device=dev, generator=gen)
      rows = list(stack.unbind(0))
      ptrs = (ctypes.c_void_p * n)(*[r.data_ptr() for r in rows])
      avg = torch.empty(d, device=dev)
      out = torch.empty(d, device=dev)
      stats = torch.empty(2 + n, dtype=torch.float64, device=dev)
      ws = torch.empty(int(tools.bz_avg_dev_max_many_workspace_bytes(n)), dtype=torch.uint8, device=dev)
      stream = torch.cuda.current_stream(dev).cuda_stream
      def k6():
        rc = tools.bz_avg_dev_max_many(ptrs, n, d, avg.data_ptr(), stats.data_ptr(), ws.data_ptr(), ws.numel(), stream)
        assert rc == 0, tools.bz_many_tools_last_error()
      def average():
        rc = many.bz_coordinate_many(0, ptrs, n, 0, d, out.data_ptr(), stream)
        assert rc == 0, many.bz_coordinate_many_last_error()
      moved = (n + 1) * d * 4
      k6_us, avg_us = events_us(k6), events_us(average)
      # the same average, bit for bit, from both entry points
      k6(); average()
      torch.cuda.synchronize()
      case = dict(n=n, d=d, k6_many_us=round(k6_us, 1), average_us=round(avg_us, 1), floor_us=round(moved / HBM_BYTES_PER_S * 1e6, 1),
                  k6_many_hbm_fraction=round(moved / k6_us * 1e6 / HBM_BYTES_PER_S, 3),
                  average_hbm_fraction=round(moved / avg_us * 1e6 / HBM_BYTES_PER_S, 3),
                  k6_many_over_average=round(k6_us / avg_us, 3), same_average=bool(torch.equal(avg, out)))
      torch_ms = wall_ms(lambda: reference_statements(rows), 3 if QUICK else 7)
      case["torch_us"] = round(torch_ms * 1e3, 1)
      case["speedup_vs_torch"] = round(torch_ms * 1e3 / k6_us, 2)
      cases.append(case)
      print(json.dumps(case), flush=True)
      del rows, stack, ptrs, avg, out, stats, ws
      torch.cuda.empty_cache()
  return cases

def search_times():
  reps = 5 if QUICK else 21
  n, f, d = 300, 20, 1_310_922
  cases = []
  for gar in ("median", "trmean"):
    gen = torch.Generator(device=dev).manual_seed(2)
    honest = [torch.randn(d, device=dev, generator=gen) * (1 + i / n) for i in range(n - f)]
    stck = torch.stack(honest)
    avg, att = stck.mean(dim=0), stck.var(dim=0).sqrt_()
    search = engine.LineSearch(gar, honest, f, f, avg, att, 16, many=True)
    search()
    factor, trace = search.result()
    xs = [x for x, _ in trace]
    def host():
      for x in xs:                                       # identical.py:67-74 at the visited factors
        grad_attack = avg + x * att
        aggregated = bz.many_gars[gar](gradients=honest + [grad_attack] * f, f=f)
        aggregated.sub_(avg)
        aggregated.dot(aggregated).item()
      byz = avg.clone()
      byz.add_(att.mul(factor))
    def device():
      search()
      search.result()
    rec = dict(gar=gar, n=n, f=f, d=d, evals=16, host_ms=round(wall_ms(host, reps), 3), device_ms=round(wall_ms(device, reps), 3))
    rec["speedup"] = round(rec["host_ms"] / rec["device_ms"], 3)
    cases.append(rec)
    print(json.dumps(rec), flush=True)
  return cases

def main():
  result = dict(card=card(), torch=torch.__version__, reps=REPS, calls=CALLS, hbm_tb_s=HBM_BYTES_PER_S / 1e12)
  print("card:", result["card"], flush=True)
  result["study"] = study_times()
  if "--search" in sys.argv:
    result["search"] = search_times()
  if "--out" in sys.argv:
    path = pathlib.Path(sys.argv[sys.argv.index("--out") + 1])
    path.parent.mkdir(parents=True, exist_ok=True)
    path.write_text(json.dumps(result, indent=1) + "\n")

if __name__ == "__main__":
  main()
