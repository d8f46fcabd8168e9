#!/usr/bin/env python3
# coding: utf-8
"""Per-call time of the coordinate-wise rules above 64 rows (`bz_coordinate`, through `engine.Plan`):
n in {65, 100, 128}, f = n // 4, d in {1,310,922; 36,489,290}, every row a distinct vector.

Per call: microseconds from CUDA events around each call (every shape warmed up first, median of
REPS calls), GB/s over the (n + 1) * d * 4 bytes a call must move, and that rate as a fraction of the
3.35 TB/s HBM3 bandwidth of the H100 SXM data sheet.  At d = 1,310,922 the reference's own torch
statements run on the same rows and GPU for comparison (with their `torch.stack`):
  median   torch.stack(rows).median(dim=0).values                           (aggregators/median.py:39)
  trmean   stack.sort(dim=0).values[f:-f].mean(dim=0)                       (trmean.py:33)
  phocas   the trimmed mean, then the closest-m statements of trmean.py:45-50
  meamed   the median, then the same closest-m statements
(the closest-m statements are written out here: tools/ do not import oracle/), and the outputs
compared: the largest difference relative to the column's magnitude, for Phocas and MeaMed away from
the columns where an exact tie makes the closest-m choice ambiguous (for Phocas, under the torch
statements' trimmed mean or the library's).  At d = 36.5M the
stack, and the sort's int64 indices (~37 GB at n = 128), rule the statements out: new path only.
The card's name and power limit are read in the same run.

    python tools/coordinate_time.py [--quick] [--out FILE.json]
"""
import json, pathlib, subprocess, sys
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
from byzantinemomentum_b200 import engine

HBM_BYTES_PER_S = 3.35e12
QUICK = "--quick" in sys.argv
REPS = 5 if QUICK else 30
NS = (65, 100, 128)
DS = (1_310_922,) if QUICK else (1_310_922, 36_489_290)
RULES = ("average", "median", "trmean", "phocas", "meamed")
dev = torch.device("cuda", 0)

def card():
  query = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
  return query[0] if query else torch.cuda.get_device_name(dev)

def median_us(fn, reps=REPS):
  fn()                                                   # warm-up: module loading, attributes, allocator
  torch.cuda.synchronize()
  times = []
  for _ in range(reps):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    times.append(start.elapsed_time(stop) * 1e3)
  times.sort()
  return times[len(times) // 2]

def closest(g, f, c):
  """ trmean.py:45-50: mean of the n - f values of each column closest to c. """
  n, d = g.shape
  p = g.clone().sub_(c).abs_().topk(n - f, dim=0, largest=False, sorted=False).indices
  p.mul_(d).add_(torch.arange(0, d, dtype=p.dtype, device=p.device))
  return g.take(p).mean(dim=0)

def trmean(g, f):
  return g.sort(dim=0).values[f:-f].mean(dim=0)

def tie_columns(g, f, c):
  """ Columns whose n - f closest values are not unique (an exact tie of |x - c| across the boundary):
  `topk` may take either value there, and the means differ by design. """
  key = (g - c).abs().sort(dim=0).values
  m = g.shape[0] - f
  return key[m - 1] == key[m]

def compare(rule, rows, f, got, ref):
  """ Largest difference to the torch statements relative to the column's magnitude, outside tie columns. """
  g = torch.stack(rows)
  scale = torch.maximum(ref.abs(), g.abs().mean(dim=0))
  rel = (got - ref).abs() / scale
  out = {}
  if rule in ("phocas", "meamed"):
    # Phocas' centre is the trimmed mean, whose last bit depends on the summation order (torch's on
    # the GPU is not ATen's CPU cascade that the kernels follow): ties under either centre count
    ties = tie_columns(g, f, g.median(dim=0).values) if rule == "meamed" else \
           tie_columns(g, f, trmean(g, f)) | tie_columns(g, f, engine.trmean(rows, f))
    rel = rel[~ties]
    out["tie_columns"] = int(ties.sum())
  out["max_rel_diff_vs_torch"] = float(rel.max())
  return out

TORCH = {
  "median": lambda rows, f: torch.stack(rows).median(dim=0).values,
  "trmean": lambda rows, f: trmean(torch.stack(rows), f),
  "phocas": lambda rows, f: (lambda g: closest(g, f, trmean(g, f)))(torch.stack(rows)),
  "meamed": lambda rows, f: (lambda g: closest(g, f, g.median(dim=0).values))(torch.stack(rows)),
}

def main():
  result = dict(card=card(), torch=torch.__version__, reps=REPS, hbm_tb_s=HBM_BYTES_PER_S / 1e12, cases=[])
  print("card:", result["card"], flush=True)
  for d in DS:
    for n in NS:
      f = n // 4
      gen = torch.Generator(device=dev).manual_seed(n)
      stack = torch.randn(n, d, device=dev, generator=gen)
      rows = list(stack.unbind(0))
      moved = (n + 1) * d * 4
      for rule in RULES:
        plan = engine.Plan(rule, rows, f=None if rule in ("average", "median") else f)
        us = median_us(plan)
        case = dict(rule=rule, n=n, f=f, d=d, us=round(us, 1), gb_s=round(moved / us / 1e3, 1),
                    hbm_fraction=round(moved / us * 1e6 / HBM_BYTES_PER_S, 3))
        if rule in TORCH and d == DS[0]:
          ref = TORCH[rule](rows, f)
          got = plan()
          case["torch_us"] = round(median_us(lambda: TORCH[rule](rows, f), max(5, REPS // 3)), 1)
          case["speedup"] = round(case["torch_us"] / us, 2)
          # same numbers: median exact, the means within fp32 summation-order differences
          case.update(compare(rule, rows, f, got, ref))
          del ref, got
        result["cases"].append(case)
        print(json.dumps(case), flush=True)
        del plan
      del rows, stack
      torch.cuda.empty_cache()
  if "--out" in sys.argv:
    path = pathlib.Path(sys.argv[sys.argv.index("--out") + 1])
    path.parent.mkdir(parents=True, exist_ok=True)
    path.write_text(json.dumps(result, indent=1) + "\n")

if __name__ == "__main__":
  main()
