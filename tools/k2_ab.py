#!/usr/bin/env python3
# coding: utf-8
"""K2 A/B on one GPU: the ring kernel (k2_ring.cu) against the round-1 kernel (k2_pairdist.cu),
same inputs — correctness of the [n, n] block against an fp64 reference computed on the device,
then device time of `bz_pairdist_partial` (K2 + the fixed-order block reduction) by CUDA events.
    python tools/k2_ab.py [--quick] [--json out.json]
BYZAGG_K2_LEGACY=1 (read per call) selects the round-1 kernel."""
import argparse, json, os, pathlib, sys
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
import byzantinemomentum_b200 as bz
from byzantinemomentum_b200 import engine

dev = torch.device("cuda", 0)

def block(rows):
  return engine.pairdist_partial(rows)

def reference(rows, chunk=1 << 20):
  n, d = len(rows), rows[0].numel()
  out = torch.zeros((n, n), dtype=torch.float64, device=dev)
  for a in range(0, d, chunk):
    x = torch.stack([r[a:a + chunk] for r in rows]).double()
    # direct differences in fp64: sum (xi - xj)^2
    for i in range(n):
      out[i] += ((x[i][None, :] - x) ** 2).sum(dim=1)
  return out

def timed(fn, sets, reps):
  for k in range(3): fn(k % sets)
  torch.cuda.synchronize()
  best = None
  for _ in range(3):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for k in range(reps): fn(k % sets)
    b.record(); torch.cuda.synchronize()
    t = a.elapsed_time(b) / reps * 1e3
    best = t if best is None else min(best, t)
  return best

def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--quick", action="store_true")
  ap.add_argument("--json", default=None)
  ap.add_argument("--cases", default=None, help="n:d,n:d,...")
  ap.add_argument("--no-alias", action="store_true")
  ap.add_argument("--only", default=None, choices=("legacy", "ring"))
  args = ap.parse_args()
  from bench import peak_hbm
  peak = peak_hbm()[0]          # MEASURED_PEAKS.json, else the H100 SXM data sheet
  if args.cases:
    cases = [tuple(int(v) for v in c.split(":")) for c in args.cases.split(",")]
  elif args.quick:
    cases = [(25, 1_310_922), (51, 1_310_922)]
  else:
    cases = [(25, 1_310_922), (25, 36_489_290), (21, 1_310_922), (11, 1_310_922), (25, 79_510), (30, 1_310_922), (36, 1_310_922),
             (40, 1_310_922), (51, 4_568_373), (51, 79_510), (64, 1_310_922)]
  results = []
  for n, d in cases:
    sets = max(1, min(6, -(-3 * 126 * 2**20 // (n * d * 4))))
    gen = torch.Generator(device=dev).manual_seed(3)
    stacks = [[torch.randn(d, device=dev, generator=gen) for _ in range(n)] for _ in range(sets)]
    rows = stacks[0]
    ref = reference(rows) if n * d <= 51 * 5_000_000 else None
    rec = dict(n=n, d=d)
    for mode in (("legacy", "ring") if args.only is None else (args.only,)):
      os.environ["BYZAGG_K2_LEGACY"] = "1" if mode == "legacy" else "0"
      got = block(rows)
      torch.cuda.synchronize()
      if ref is not None:
        iu = torch.triu_indices(n, n, 1, device=dev)
        rel = ((got[iu[0], iu[1]] - ref[iu[0], iu[1]]).abs() / ref[iu[0], iu[1]]).max().item()
        rec[mode + "_max_rel_err_sq"] = rel
      reps = 50 if n * d < 2e8 else 10
      rec[mode + "_us"] = timed(lambda k: block(stacks[k]), sets, reps)
      rec[mode + "_hbm_frac"] = n * d * 4 / (rec[mode + "_us"] * 1e-6) / 1e9 / peak
    # FP32 pipe floor: n(n-1) lane-ops per coordinate at 128 lanes/clk/SM, 132 SMs, 1.98 GHz (H100 SXM)
    rec["fp_floor_us"] = n * (n - 1) * d / (132 * 128 * 1.98e9) * 1e6
    rec["hbm_floor_us"] = n * d * 4 / (peak * 1e9) * 1e6
    results.append(rec)
    print(json.dumps(rec), flush=True)
    del stacks, rows
    torch.cuda.empty_cache()
  os.environ["BYZAGG_K2_LEGACY"] = "0"
  if args.no_alias:
    return
  # aliases: the self flag path (f Byzantine rows are one tensor), incl. a NaN / inf aliased row
  for n, nb, d, poison in ((25, 5, 1_310_922, None), (25, 5, 1_310_922, "nan"), (25, 5, 1_310_922, "inf"), (51, 12, 500_003, None), (51, 12, 500_003, "inf")):
    gen = torch.Generator(device=dev).manual_seed(5)
    honest = [torch.randn(d, device=dev, generator=gen) for _ in range(n - nb)]
    byz = torch.randn(d, device=dev, generator=gen)
    if poison == "nan": byz[12345] = float("nan")
    if poison == "inf": byz[12345] = float("inf")
    rows = honest + [byz] * nb
    f = nb if n >= 2 * nb + 3 else 1
    outs = {}
    for mode in ("legacy", "ring"):
      os.environ["BYZAGG_K2_LEGACY"] = "1" if mode == "legacy" else "0"
      out, sel = engine.krum(rows, f, n - f - 2)
      outs[mode] = (out.clone(), sel.clone())
    same_sel = bool((outs["legacy"][1] == outs["ring"][1]).all())
    same_out = bool(torch.equal(outs["legacy"][0], outs["ring"][0]) or (outs["legacy"][0].isnan() & outs["ring"][0].isnan()).all())
    rec = dict(alias_case=f"n={n} nb={nb} d={d} poison={poison}", same_selection=same_sel, same_output=same_out, selection=outs["ring"][1].tolist())
    results.append(rec)
    print(json.dumps(rec), flush=True)
  os.environ["BYZAGG_K2_LEGACY"] = "0"
  if args.json:
    pathlib.Path(args.json).write_text(json.dumps(results, indent=1))

if __name__ == "__main__":
  main()
