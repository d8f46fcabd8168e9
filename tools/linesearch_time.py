#!/usr/bin/env python3
# coding: utf-8
"""Per-evaluation time of the attacks' line search (attacks/identical.py:68-77): 16 evaluations of
the rule on the same honest rows with a new Byzantine row each, with and without distance reuse.

With --search: the time of one step's whole search instead (`little`'s direction, factor -16):
  host_ms    the reference's statements (identical.py:67-77) over `bz.gars`: per evaluation the
             candidate row, the rule, `sub_`, `dot(...).item()` (one host sync each), at the x values
             the device search visits (the host search makes the same choices up to score ties);
  device_ms  `engine.LineSearch` issued and read once (`result()`), eager;
  graph_ms   the same search replayed from a CUDA graph, then read once.
Wall clock around work that ends in a synchronisation, median of REPS, after warm-up.  The card's name
and power limit are read in the same run."""
import json, pathlib, subprocess, sys, time
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
import byzantinemomentum_b200 as bz
from byzantinemomentum_b200 import engine
dev = torch.device("cuda", 0)
bz.config.strict_status = False
out = []
QUICK = "--quick" in sys.argv

def card():
  query = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
  return query[0] if query else torch.cuda.get_device_name(dev)

def median_ms(fn, reps):
  times = []
  for _ in range(reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    times.append((time.perf_counter() - t0) * 1e3)
  times.sort()
  return times[len(times) // 2]

def search_times():
  """ One step's whole search, old host loop vs the device search (eager and graph-replayed). """
  reps = 5 if QUICK else 21
  cases = (("trmean", 51, 12, 79_510), ("median", 51, 12, 79_510), ("krum", 25, 5, 79_510),
           ("trmean", 25, 5, 1_310_922), ("median", 25, 5, 1_310_922), ("krum", 25, 5, 1_310_922))
  result = dict(card=card(), cases=[])
  for gar, n, f, d in cases[:1] if QUICK else cases:
    gen = torch.Generator(device=dev).manual_seed(2)
    honest = [torch.randn(d, device=dev, generator=gen) * (1 + i / n) for i in range(n - f)]
    stck = torch.stack(honest)
    avg, att = stck.mean(dim=0), stck.var(dim=0).sqrt_()
    search = engine.LineSearch(gar, honest, f, f, avg, att, 16)
    search()
    factor, trace = search.result()
    xs = [x for x, _ in trace]
    def host():
      for x in xs:                                       # identical.py:67-74 at the visited factors
        grad_attack = avg + x * att
        aggregated = bz.gars[gar](gradients=honest + [grad_attack] * f, f=f)
        aggregated.sub_(avg)
        aggregated.dot(aggregated).item()
      byz = avg.clone()
      byz.add_(att.mul(factor))
    def device():
      search()
      search.result()
    replay = search.graph()
    def graphed():
      replay()
      search.result()
    for fn in (host, device, graphed):
      fn()                                               # warm-up: modules, allocator, distance table
    rec = dict(gar=gar, n=n, f=f, d=d, evals=16, factor=factor)
    for name, fn in (("host_ms", host), ("device_ms", device), ("graph_ms", graphed)):
      rec[name] = round(median_ms(fn, reps), 4)
    rec["device_speedup"] = round(rec["host_ms"] / rec["device_ms"], 3)
    rec["graph_speedup"] = round(rec["host_ms"] / rec["graph_ms"], 3)
    result["cases"].append(rec)
    print(json.dumps(rec), flush=True)
  return result

if "--search" in sys.argv:
  result = search_times()
  print(json.dumps(dict(card=result["card"])), flush=True)
  if len(sys.argv) > 1 and not sys.argv[1].startswith("--"):
    pathlib.Path(sys.argv[1]).write_text(json.dumps(result, indent=1))
  sys.exit(0)
REPS = 5
CASES = (("krum", 25, 5, 5, 1_310_922),) if QUICK else (("krum", 25, 5, 5, 1_310_922), ("bulyan", 25, 5, 5, 1_310_922), ("krum", 51, 12, 12, 1_310_922), ("krum", 11, 3, 3, 1_310_922),
                         ("krum", 25, 5, 5, 79_510), ("krum", 51, 12, 12, 79_510))
for gar, n, nb, f, d in CASES:
  gen = torch.Generator(device=dev).manual_seed(1)
  honest = [torch.randn(d, device=dev, generator=gen) for _ in range(n - nb)]
  attacks = [torch.randn(d, device=dev, generator=gen) for _ in range(17)]
  rec = dict(gar=gar, n=n, f=f, d=d)
  for reuse in (False, True):
    engine.config.reuse_distances = reuse
    best = None
    for rep in range(REPS):
      bz.gars[gar].unchecked(gradients=honest + [attacks[16]] * nb, f=f)          # the step's first call (fills the table)
      torch.cuda.synchronize()
      a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      a.record()
      for k in range(16):
        bz.gars[gar].unchecked(gradients=honest + [attacks[k]] * nb, f=f)
      b.record(); torch.cuda.synchronize()
      t = a.elapsed_time(b) / 16 * 1e3
      best = t if best is None else min(best, t)
    rec["reuse_us" if reuse else "full_us"] = best
  rec["ratio"] = rec["reuse_us"] / rec["full_us"]
  # the same 16 evaluations through the C ABI with every argument prepared (no Python bookkeeping in
  # the timed loop): what the library itself gains
  if gar == "krum":
    import ctypes
    from byzantinemomentum_b200 import _lib
    lib = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    ws = engine._workspace(dev, st)
    outb = torch.empty(d, device=dev); order = torch.empty(n, dtype=torch.int32, device=dev)
    tabs = [torch.empty(64 * 64, dtype=torch.float64, device=dev) for _ in range(2)]
    lists = [honest + [attacks[k]] * nb for k in range(17)]
    ptrs = [(ctypes.c_void_p * n)(*[g.data_ptr() for g in l]) for l in lists]
    old = (ctypes.c_int32 * n)(*([i for i in range(n - nb)] + [-1] * nb))
    mode = ctypes.c_int(0)
    m = n - f - 2
    def full(k):
      return lib.bz_krum(ptrs[k], n, f, m, d, outb.data_ptr(), order.data_ptr(), ws.data_ptr(), ws.numel(), st)
    def reuse(k, cur):
      return lib.bz_krum_reuse(ptrs[k], n, f, m, d, outb.data_ptr(), order.data_ptr(), old, tabs[cur].data_ptr(), n - nb + 1,
                               tabs[cur ^ 1].data_ptr(), ctypes.byref(mode), ws.data_ptr(), ws.numel(), st)
    for name in ("abi_full_us", "abi_reuse_us"):
      best = None
      for rep in range(5):
        lib.bz_krum_reuse(ptrs[16], n, f, m, d, outb.data_ptr(), order.data_ptr(), None, None, 0, tabs[0].data_ptr(), ctypes.byref(mode),
                          ws.data_ptr(), ws.numel(), st)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        cur = 0
        for k in range(16):
          if name == "abi_full_us": full(k)
          else:
            reuse(k, cur); cur ^= 1
        b.record(); torch.cuda.synchronize()
        t = a.elapsed_time(b) / 16 * 1e3
        best = t if best is None else min(best, t)
      rec[name] = best
    rec["abi_ratio"] = rec["abi_reuse_us"] / rec["abi_full_us"]
    rec["abi_last_mode"] = mode.value
  out.append(rec)
  print(json.dumps(rec), flush=True)
engine.config.reuse_distances = True
if len(sys.argv) > 1 and not sys.argv[1].startswith("--"):
  pathlib.Path(sys.argv[1]).write_text(json.dumps(out, indent=1))
