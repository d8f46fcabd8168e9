#!/usr/bin/env python3
# coding: utf-8
"""Time per `Plan` call of Multi-Krum, Bulyan, Aksel and CGE above 64 rows (`bz_distance`).

n in {65, 100, 128} with f = (n - 3) / 4 (the largest f Bulyan takes) aliased Byzantine rows, so that the
distance passes run over the n - f + 1 unique rows; d in {1,310,922; 36,489,290}.  Every shape is warmed
up, then each call is timed with CUDA events and the median of REPS = 30 calls is kept.  Beside each time:
  pair_floor_us  (krum, bulyan) the FP32 floor of the distance passes: the sum over the passes of
                 u_p (u_p - 1) lane operations per coordinate (2 FP32 operations on packed pairs, as DESIGN §4.2
                 counts them), over 132 SMs x 128 lanes at the card's maximum SM clock;
  hbm_floor_us   one read of the unique rows (pairwise rules) or of all n rows (aksel, cge) at the 3.35 TB/s
                 of the H100 SXM data sheet;
  torch_us       at d = 1,310,922 only: the reference's torch statements (krum.py:44-62,80, bulyan.py:49-84,
                 aksel.py:37-49,64, cge.py:36-38,53-56, restated below) on the same GPU, wall clock around one
                 call, median of 3.
The card's name, power limit and maximum SM clock are read in the same run.

    python tools/distance_wide_time.py [--quick] [--out FILE.json]
"""
import json, math, pathlib, subprocess, sys, time
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
from byzantinemomentum_b200 import engine

HBM_BYTES_PER_S = 3.35e12
SMS, LANES = 132, 128
QUICK = "--quick" in sys.argv
REPS = 5 if QUICK else 30
NS = (65, 100, 128)
DS = (1_310_922,) if QUICK else (1_310_922, 36_489_290)
RULES = (("krum", "mid"), ("bulyan", "mid"), ("aksel", "mid"), ("cge", "mid"))
dev = torch.device("cuda", 0)

def card():
  query = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
  return query[0] if query else torch.cuda.get_device_name(dev)

def max_sm_hz(card_line):
  try:
    return float(card_line.split(",")[2].strip().split()[0]) * 1e6
  except (IndexError, ValueError):
    return 1.98e9

def pass_sizes(u):
  """ The row counts of the distance passes over u unique rows (dist.cuh, PassTables). """
  if u <= 64:
    return [u]
  k = (u + 31) // 32
  start = [b * u // k for b in range(k + 1)]
  size = [start[b + 1] - start[b] for b in range(k)]
  return [size[a] + size[b] for a in range(k) for b in range(a + 1, k)]

# ---- the reference's statements, on the rows' device ----

def _mean_of(rows):
  return sum(rows).div_(len(rows))

def _distances(rows):
  n = len(rows)
  table = [[math.inf] * n for _ in range(n)]
  for a in range(n - 1):
    for b in range(a + 1, n):
      value = rows[a].sub(rows[b]).norm().item()
      table[a][b] = table[b][a] = value if math.isfinite(value) else math.inf
  return table

def ref_krum(rows, f):
  n = len(rows)
  table = _distances(rows)
  scored = sorted(((sum(sorted(table[i][j] for j in range(n) if j != i)[:n - f - 1]), i) for i in range(n)), key=lambda p: p[0])
  return _mean_of([rows[i] for _, i in scored[:n - f - 2]])

def ref_bulyan(rows, f):
  n = len(rows)
  m = m_max = n - f - 2
  table = _distances(rows)
  order = [i for _, i in sorted(((sum(sorted(table[i])[:m]), i) for i in range(n)), key=lambda p: p[0])]
  theta = n - 2 * f - 2
  selected = []
  for it in range(theta):
    m = min(m, m_max - it)
    selected.append(_mean_of([rows[i] for i in order[it:it + m]]))
  stacked = torch.stack(selected)
  med = stacked.median(dim=0).values
  picks = stacked.clone().sub_(med).abs_().topk(theta - 2 * f, dim=0, largest=False, sorted=False).indices
  picks.mul_(stacked.shape[1]).add_(torch.arange(0, stacked.shape[1], dtype=picks.dtype, device=picks.device))
  return stacked.take(picks).mean(dim=0)

def ref_aksel(rows, f):
  center = torch.stack(rows).median(dim=0)[0]
  keyed = sorted((((x - center).pow_(2).sum().item(), i) for i, x in enumerate(rows)), key=lambda p: p[0])
  return _mean_of([rows[i] for _, i in keyed[:(len(rows) + 1) // 2]])

def ref_cge(rows, f):
  ranked = sorted(((row.norm().item(), i) for i, row in enumerate(rows)), key=lambda p: p[0] if math.isfinite(p[0]) else math.inf)
  m = len(rows) - f
  total = rows[ranked[0][1]].clone()
  for _, i in ranked[1:m]:
    total.add_(rows[i])
  return total.div_(m)

REFERENCE = dict(krum=ref_krum, bulyan=ref_bulyan, aksel=ref_aksel, cge=ref_cge)

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

def wall_us(fn, reps=3):
  times = []
  for _ in range(reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    times.append((time.perf_counter() - t0) * 1e6)
  times.sort()
  return times[len(times) // 2]

def main():
  line = card()
  clock = max_sm_hz(line)
  result = dict(card=line, torch=torch.__version__, reps=REPS, hbm_tb_s=HBM_BYTES_PER_S / 1e12, sm_clock_hz=clock, cases=[])
  print("card:", line, flush=True)
  for d in DS:
    for n in NS:
      f = (n - 3) // 4
      gen = torch.Generator(device=dev).manual_seed(n)
      honest = torch.randn(n - f, d, device=dev, generator=gen) * torch.linspace(0.5, 1.5, n - f, device=dev)[:, None]
      byz = honest.mean(dim=0).mul_(-1.1)
      rows = list(honest.unbind(0)) + [byz] * f
      u = n - f + 1
      for gar, mode in RULES:
        plan = engine.Plan(gar, rows, f=f, mode=mode)
        us = events_us(plan)
        pair = gar in ("krum", "bulyan")
        case = dict(gar=gar, n=n, f=f, d=d, us=round(us, 1),
                    hbm_floor_us=round((u if pair else n) * d * 4 / HBM_BYTES_PER_S * 1e6, 1))
        if pair:
          lane_ops = sum(s * (s - 1) for s in pass_sizes(u))
          case["passes"] = len(pass_sizes(u))
          case["pair_floor_us"] = round(lane_ops * d / (SMS * LANES * clock) * 1e6, 1)
        if d < 2_000_000:
          ref = lambda: REFERENCE[gar](rows, f)
          ref()
          case["torch_us"] = round(wall_us(ref), 1)
          case["speedup_vs_torch"] = round(case["torch_us"] / us, 1)
        result["cases"].append(case)
        print(json.dumps(case), flush=True)
        del plan
      del rows, honest, byz
      torch.cuda.empty_cache()
  if "--out" in sys.argv:
    path = pathlib.Path(sys.argv[sys.argv.index("--out") + 1])
    path.parent.mkdir(parents=True, exist_ok=True)
    path.write_text(json.dumps(result, indent=1) + "\n")

if __name__ == "__main__":
  main()
