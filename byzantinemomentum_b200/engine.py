# coding: utf-8
"""Host side of the CUDA path: turns a list of n flat fp32 tensors into ONE call of the C ABI.

PyTorch is plumbing here (device memory, the current stream, the caching allocator); every
numeric operation happens in `libbyzagg.so`.  The gradients are never stacked: the library
receives the n row pointers (`tensor.data_ptr()`) and reads the rows where they live.

CPU tensors (`--device-gar cpu` in the reference's attack.py:66-69) are staged to the
current CUDA device — each distinct tensor object once, so the f aliased Byzantine entries
(attacks/identical.py:86) cost one copy — and the result is copied back: that is the
"host buffers" end-to-end path `bench.py` times.  Without a CUDA device or without the
compiled library every entry point raises; there is no CPU fallback.
"""

import ctypes
import math
import time
import weakref

import torch

from . import _lib, hostmem

__all__ = ["average", "median", "trmean", "phocas", "meamed", "krum", "bulyan", "brute", "aksel", "cge",
           "pairdist_partial", "rowdist_partial", "krum_select", "bulyan_select", "brute_select",
           "rowdist_select", "average_selected", "bulyan_reduce", "avg_dev_max_async", "compute_avg_dev_max", "rowdots_async", "study_step",
           "config", "Plan", "pair_cache_stats", "GradientStack", "host_path_report"]

class _Config:
  """ strict_status: after brute / bulyan, read the device status word (one 4-byte D2H copy,
  i.e. a stream sync) and raise where the reference raises (brute.py:67, bulyan.py:70).
  When False the call stays asynchronous and a failed rule yields an all-NaN vector.
  reuse_distances: Multi-Krum / Bulyan / brute on CUDA tensors keep the table of squared pairwise
  distances of their last call; a following call whose rows are, but for 1..4 of them, the very
  same unmodified tensor objects (identity, address and in-place version all equal) only
  computes the distances of the new rows — the attacks' line search, attacks/identical.py:68-77,
  evaluates the rule up to 16 times per step on the same honest gradients.  Results are
  bit-identical either way.  A caller that rewrites a gradient behind PyTorch's back (`.data`,
  raw pointers, external kernels: no version bump) must switch this off. """
  strict_status = True
  reuse_distances = True
config = _Config()

# ---------------------------------------------------------------------------- #
# Argument plumbing

class _Prepared:
  __slots__ = ("rows", "n", "d", "device", "ptrs", "stream", "to_cpu", "keep", "host_mode", "host_t0")

_workspaces = {}
_staging = {}

_MAX_WORKSPACES = 16

def _workspace(device, stream):
  """ One scratch buffer per (device, stream), sized for MAX_N (~10 MB).  At most
  `_MAX_WORKSPACES` are kept (least recently used dropped; the caching allocator keeps a dropped
  buffer alive until the launches already queued on its stream have run). """
  key = (device.index, stream)
  ws = _workspaces.pop(key, None)
  if ws is None:
    nbytes = int(_lib.lib().bz_workspace_bytes(_lib.MAX_N))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
    while len(_workspaces) >= _MAX_WORKSPACES:
      _workspaces.pop(next(iter(_workspaces)))
  _workspaces[key] = ws          # most recently used last
  return ws

_F32 = torch.float32

_COPY_LANES = 4
_copy_lanes = {}

class _HostPath:
  """ How host rows reach the GPU is decided by MEASUREMENT, per device: the right answer differs between
  boxes of the same model (pinned rows on the far socket can copy several times faster over four streams
  than over one; on other boxes four streams are the slow ones).  Candidates:
    "lanes"     the row copies spread over 4 streams,
    "lane"      the row copies on the current stream,
    "batch"     `bz_stage_rows`: the row copies as ONE cudaMemcpyBatchAsync on a copy stream (a separate
                cudaMemcpyAsync per row costs ~5.7 us of copy-engine time each),
    "pipeline"  (coordinate-wise rules only) `bz_coordinate_host`: the vector cut into column chunks, the
                H2D copy of chunk c+1, the kernel of chunk c and the D2H copy of chunk c-1 running at once.
  (A third one — no staging, the kernel reading the pinned rows in place over PCIe — measured the same
  2.7 ms as the copies and needs `Tensor.is_pinned()`, which costs ~1 ms PER TENSOR on some boxes: dropped.)
  The first calls try each candidate three times (wall clock of the whole call: it ends with a
  synchronisation); the first sample pays one-time costs, the slower of the other two ranks the candidate. """
  def __init__(self):
    self.times = {}
    self.best = {}
  def choose(self, single_pass, pinned):
    key = (single_pass, pinned)
    if key in self.best:
      return self.best[key]
    candidates = ["lanes", "lane"] + (["pipeline"] if single_pass else ["batch"])
    if forced_host_path is not None and forced_host_path in candidates:
      self.best[key] = forced_host_path
      return forced_host_path
    seen = self.times.setdefault(key, {})
    for mode in candidates:
      if len(seen.get(mode, ())) < 3:          # three samples each: the first one pays one-time costs
        return mode
    # the median of the last two samples: a path that is fast once and slow the next time is not "the fastest"
    self.best[key] = min(candidates, key=lambda mode: max(seen[mode][1:]))
    return self.best[key]
  def record(self, single_pass, pinned, mode, seconds):
    key = (single_pass, pinned)
    if key not in self.best:
      self.times.setdefault(key, {}).setdefault(mode, []).append(seconds)

_host_paths = {}
forced_host_path = None      # tests / A-B runs: pin the host path ("lanes", "lane", "pipeline") instead of measuring
_PIPELINE_CHUNKS = 4       # column chunks of the host pipeline: H2D, kernel and D2H of three chunks overlap
_RULE_CODES = dict(average=0, median=1, trmean=2, phocas=3, meamed=4)      # BZ_RULE_*

def host_path_report(device_index=None):
  """ What the measurement found (bench / tests): {(single_pass, pinned): {"best": mode, "ms": {mode: best ms}}}. """
  if device_index is None:
    device_index = torch.cuda.current_device()
  hp = _host_paths.get(device_index)
  if hp is None:
    return {}
  keys = list(dict.fromkeys(list(hp.times) + list(hp.best)))
  return {f"single_pass={k[0]},pinned={k[1]}": dict(best=hp.best.get(k), ms={m: round(min(v) * 1e3, 3) for m, v in hp.times.get(k, {}).items() if v},
                                                           samples_ms={m: [round(x * 1e3, 3) for x in v] for m, v in hp.times.get(k, {}).items() if v}) for k in keys}

def _copy_streams(device):
  lanes = _copy_lanes.get(device.index)
  if lanes is None:
    lanes = _copy_lanes[device.index] = [torch.cuda.Stream(device) for _ in range(_COPY_LANES)]
  return lanes

def _validate(gradients):
  """ One pass over the list: types, dtype, rank, length; returns (first, all_contiguous). """
  if not isinstance(gradients, (list, tuple)) or len(gradients) < 1:
    raise ValueError(f"expected a non-empty list of gradients, got {type(gradients).__name__} of length {len(gradients) if hasattr(gradients, '__len__') else '?'}")
  first = gradients[0]
  if not isinstance(first, torch.Tensor):
    raise TypeError(f"gradients must be torch tensors, got {type(first).__name__}")
  if len(gradients) > _lib.MAX_N:
    raise ValueError(f"{len(gradients)} gradients exceed the supported maximum of {_lib.MAX_N}")
  if first.dim() != 1:
    raise ValueError("gradients must be 1-D tensors")
  d = first.numel()
  cuda = first.is_cuda
  index = first.get_device()
  contiguous = True
  for grad in gradients:
    if grad.dtype is not _F32:
      raise TypeError(f"gradients must be float32 (attack.py:461 fixes the dtype), got {grad.dtype}")
    if grad.dim() != 1 or grad.numel() != d or grad.is_cuda != cuda or grad.get_device() != index:
      raise ValueError("gradients must be 1-D tensors of one shape on one device")
    contiguous = contiguous and grad.is_contiguous()
  return first, contiguous

class _CallCache:
  """ Small cache of prepared arguments for calls on CUDA tensors, keyed by the identity of the
  tensor objects (held through weak references) and re-validated against their current data
  pointers: a trainer that aggregates the same momentum buffers every step (attack.py:800-804)
  pays for the list validation once.  At most `capacity` lists, oldest evicted first. """
  capacity = 8
  def __init__(self):
    self.entries = {}          # ids tuple -> (refs, addresses, prep)
  def lookup(self, gradients):
    if not self.entries or type(gradients) is not list:
      return None
    entry = self.entries.get(tuple(map(id, gradients)))
    if entry is None:
      return None
    refs, addresses, prep = entry
    for ref, grad in zip(refs, gradients):
      if ref() is not grad:
        return None
    if tuple([g.data_ptr() for g in gradients]) != addresses or gradients[0].numel() != prep.d:
      return None
    return prep
  def store(self, gradients, addresses, prep):
    try:
      refs = [weakref.ref(g) for g in gradients]
    except TypeError:
      return
    if len(self.entries) >= self.capacity:
      self.entries.pop(next(iter(self.entries)))
    self.entries[tuple(map(id, gradients))] = (refs, addresses, prep)

_call_cache = _CallCache()

def _prepare(gradients, single_pass=False):
  prep = _call_cache.lookup(gradients)
  if prep is not None:
    prep.stream = torch.cuda.current_stream(prep.device).cuda_stream
    return prep
  first, contiguous = _validate(gradients)
  if not torch.cuda.is_available():
    raise _lib.LibraryError("no CUDA device available: byzantinemomentum_b200 runs on H100 (sm_90a) GPUs only (no CPU fallback)")
  _lib.lib()
  prep = _Prepared()
  prep.host_mode = None
  n, d = len(gradients), first.shape[0]
  keep = None
  if first.device.type == "cuda":
    device = first.device
    rows = gradients if contiguous else [g if g.is_contiguous() else g.contiguous() for g in gradients]
    prep.to_cpu = False
  elif first.device.type == "cpu":
    # Stage every distinct tensor object once into a cached [k, d] device buffer
    device = torch.device("cuda", torch.cuda.current_device())
    uniq = {}
    for g in gradients:
      uniq.setdefault(id(g), g)
    pinned = False          # never asked: Tensor.is_pinned() is a slow driver query on some boxes
    path = _host_paths.get(device.index)
    if path is None:
      path = _host_paths[device.index] = _HostPath()
    mode = path.choose(single_pass, pinned)
    prep.host_mode = (single_pass, pinned, mode)
    torch.cuda.current_stream(device).synchronize()        # the clock below times this call only
    prep.host_t0 = time.perf_counter()
    key = (device.index, len(uniq), d)
    buf = _staging.get(key)
    if buf is None:
      _staging.clear()
      pitch = (d + 63) // 64 * 64       # rows 256-byte aligned: keeps the vector-load path
      buf = torch.empty((len(uniq), pitch), dtype=torch.float32, device=device)
      _staging[key] = buf
    # The row copies go out on several streams.  Measured (tools/h2d_probe2.py, two-socket host):
    # pinned rows that live on the OTHER socket's memory copy at 8.5 GB/s on one stream and at
    # 53 GB/s on two or more — with one stream the e2e step took 12.5 ms, 2.5x the box's own PCIe
    # floor, and varied 4x between boxes depending on where the caller's pages happened to be.
    current = torch.cuda.current_stream(device)
    if mode == "batch" and not all(g.is_contiguous() for g in uniq.values()):
      mode = "lane"
    lanes = _copy_streams(device) if mode == "lanes" else ([_copy_streams(device)[0]] if mode == "batch" else [current])
    if mode in ("lanes", "batch"):
      for lane in lanes:
        lane.wait_stream(current)        # the previous call's kernels have finished with the staging buffer
    slot = {}
    if mode == "batch":
      hosts = (ctypes.c_void_p * len(uniq))(*[g.data_ptr() for g in uniq.values()])
      with _on(device):
        code = _lib.lib().bz_stage_rows(hosts, len(uniq), d, buf.data_ptr(), buf.stride(0), lanes[0].cuda_stream)
      _lib.check(code, "bz_stage_rows")
      for k, ident in enumerate(uniq):
        slot[ident] = buf[k, :d]
    else:
      for k, (ident, g) in enumerate(uniq.items()):
        row = buf[k, :d]
        with torch.cuda.stream(lanes[k % len(lanes)]):
          row.copy_(g, non_blocking=True)
        slot[ident] = row
    if mode in ("lanes", "batch"):
      for lane in lanes:
        current.wait_stream(lane)
    rows = [slot[id(g)] for g in gradients]
    keep = buf
    prep.to_cpu = True
  else:
    raise ValueError(f"unsupported device {first.device}")
  addresses = tuple([g.data_ptr() for g in rows])
  prep.rows, prep.n, prep.d, prep.device, prep.keep = rows, n, d, device, keep
  prep.ptrs = (ctypes.c_void_p * n)(*addresses)
  prep.stream = torch.cuda.current_stream(device).cuda_stream
  if not prep.to_cpu and contiguous and type(gradients) is list:
    prep.rows = None            # the cache must not keep the gradients alive
    _call_cache.store(gradients, addresses, prep)
  return prep

class _on:
  """ Make `device` current for the launches (cheap when it already is). """
  __slots__ = ("device", "prev")
  def __init__(self, device):
    self.device = device
    self.prev = None
  def __enter__(self):
    cur = torch.cuda.current_device()
    if cur != self.device.index:
      self.prev = cur
      torch.cuda.set_device(self.device)
  def __exit__(self, *exc):
    if self.prev is not None:
      torch.cuda.set_device(self.prev)

_host_out = {}

def _finish(prep, out):
  """ Device result for device inputs; for staged host inputs, a NEW host tensor (the copy goes
  through a cached pinned buffer so that the D2H transfer runs at full PCIe rate). """
  if not prep.to_cpu:
    return out
  # The result goes straight into a NEW pinned tensor, which the caller owns: PyTorch's caching host
  # allocator recycles such blocks, so after the first steps this costs neither a cudaHostAlloc nor page
  # faults — the former `cached pinned buffer + clone()` paid a fresh 5 MB of page faults per call.
  result = torch.empty(prep.d, dtype=torch.float32, pin_memory=True)
  result.copy_(out, non_blocking=True)
  torch.cuda.current_stream(prep.device).synchronize()
  if prep.host_mode is not None:
    single_pass, was_pinned, mode = prep.host_mode
    _host_paths[prep.device.index].record(single_pass, was_pinned, mode, time.perf_counter() - prep.host_t0)
  return result

def _raise_status(code):
  if code == _lib.STATUS_NO_FINITE_SET:
    raise AssertionError(_lib.STATUS_MESSAGES[code])        # brute.py:67
  if code == _lib.STATUS_DEGENERATE:
    raise TypeError(_lib.STATUS_MESSAGES[code])             # bulyan.py:70 (`gradients[None]`)

# ---------------------------------------------------------------------------- #
# Coordinate-wise rules

def _coordinate_pipeline(name, gradients, f, path, device):
  """ Host rows in, host vector out through `bz_coordinate_host` (column chunks; copies and kernels overlap). """
  t0 = time.perf_counter()
  n, d = len(gradients), gradients[0].shape[0]
  rows = [g if g.is_contiguous() else g.contiguous() for g in gradients]
  pitch = (d + 63) // 64 * 64
  key = (device.index, n, d)
  buf = _staging.get(key)
  if buf is None or buf.shape[0] < n:
    _staging.clear()
    buf = _staging[key] = torch.empty((n, pitch), dtype=torch.float32, device=device)
  out = torch.empty(d, dtype=torch.float32, device=device)
  result = torch.empty(d, dtype=torch.float32, pin_memory=True)
  current = torch.cuda.current_stream(device)
  lanes = _copy_streams(device)
  ptrs = (ctypes.c_void_p * n)(*[g.data_ptr() for g in rows])
  with _on(device):
    code = _lib.lib().bz_coordinate_host(_RULE_CODES[name], ptrs, n, 0 if f is None else int(f), d, result.data_ptr(),
                                         buf.data_ptr(), pitch, out.data_ptr(), _PIPELINE_CHUNKS,
                                         current.cuda_stream, lanes[0].cuda_stream, lanes[1].cuda_stream)
  _lib.check(code, "bz_coordinate_host")
  current.synchronize()           # the host rows, `out` and the staging rows stay alive until here
  path.record(True, False, "pipeline", time.perf_counter() - t0)
  return result

def _coordinate(name, gradients, f=None):
  if type(gradients) in (list, tuple) and len(gradients) > 0 and isinstance(gradients[0], torch.Tensor) and gradients[0].device.type == "cpu" and torch.cuda.is_available():
    _validate(gradients)
    _lib.lib()
    device = torch.device("cuda", torch.cuda.current_device())
    path = _host_paths.get(device.index)
    if path is None:
      path = _host_paths[device.index] = _HostPath()
    if path.choose(True, False) == "pipeline":
      torch.cuda.current_stream(device).synchronize()        # the clock times this call only
      return _coordinate_pipeline(name, gradients, f, path, device)
  prep = _prepare(gradients, single_pass=True)
  out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  fn = getattr(_lib.lib(), "bz_" + name)
  with _on(prep.device):
    if f is None:
      code = fn(prep.ptrs, prep.n, prep.d, out.data_ptr(), prep.stream)
    else:
      code = fn(prep.ptrs, prep.n, int(f), prep.d, out.data_ptr(), prep.stream)
  _lib.check(code, "bz_" + name)
  return _finish(prep, out)

def average(gradients):
  return _coordinate("average", gradients)

def median(gradients):
  return _coordinate("median", gradients)

def trmean(gradients, f):
  return _coordinate("trmean", gradients, f)

def phocas(gradients, f):
  return _coordinate("phocas", gradients, f)

def meamed(gradients, f):
  return _coordinate("meamed", gradients, f)

# ---------------------------------------------------------------------------- #
# Distance reuse across calls (SURVEY.md §8(f) row 1)

class _PairCache:
  """ Per device: the unique rows of the last Multi-Krum / Bulyan / brute call (weak references,
  addresses, versions, their positions in the table) and two device buffers holding the table of
  squared distances (the library reads one, writes the other). """
  def __init__(self, device):
    self.buffers = [torch.empty(_lib.MAX_N * _lib.MAX_N, dtype=torch.float64, device=device) for _ in range(2)]
    self.current = 0          # buffer holding the last table
    self.rows = {}            # id(tensor) -> (weakref, data_ptr, version, index)
    self.u = 0
    self.d = -1
    self.stream = None
    self.mode = ctypes.c_int(-1)
    self.stats = dict(full=0, star=0, off=0)
  def old_index(self, gradients, d, stream):
    """ (ctypes int32[n] or None, cache_in ptr or None, u_old) for this call.  One pass over the
    rows; the addresses / versions read here are kept for `update`. """
    self._ptrs = ptrs = [g.data_ptr() for g in gradients]
    self._vers = vers = [g._version for g in gradients]
    if self.u == 0 or self.d != d or self.stream != stream:
      return None, None, 0
    n = len(gradients)
    table = (ctypes.c_int32 * n)()
    hits = 0
    get = self.rows.get
    for i, g in enumerate(gradients):
      entry = get(id(g))
      if entry is not None and entry[1] == ptrs[i] and entry[2] == vers[i] and entry[0]() is g:
        table[i] = entry[3]
        hits += 1
      else:
        table[i] = -1
    if hits == 0:
      return None, None, 0
    return table, self.buffers[self.current].data_ptr(), self.u
  def update(self, gradients, d, stream):
    """ After a call that wrote its table: remember its unique rows (pointer equality, first
    appearance: the library's order). """
    mode = self.mode.value
    if mode < 0:
      self.rows, self.u = {}, 0
      self.stats["off"] += 1
      return
    self.stats["star" if mode == 1 else "full"] += 1
    index, rows = {}, {}
    ref = weakref.ref
    try:
      for g, ptr, ver in zip(gradients, self._ptrs, self._vers):
        k = index.get(ptr)
        if k is None:
          k = index[ptr] = len(index)
        key = id(g)
        if key not in rows:
          rows[key] = (ref(g), ptr, ver, k)
    except TypeError:
      rows, index = {}, {}
    self.rows, self.u, self.d, self.stream = rows, len(index), d, stream
    self.current ^= 1
  def out_buffer(self):
    return self.buffers[self.current ^ 1].data_ptr()

_pair_caches = {}

def _pair_cache(prep, gradients):
  """ The cache to use for this call, or None (reuse switched off, staged host rows, packed copies). """
  if not config.reuse_distances or prep.to_cpu or prep.rows is not None and prep.rows is not gradients:
    return None
  cache = _pair_caches.get(prep.device.index)
  if cache is None:
    cache = _pair_caches[prep.device.index] = _PairCache(prep.device)
  return cache

def pair_cache_stats(device_index=None):
  """ Calls served per mode ({"full", "star", "off"}) by the distance cache of a device (tests, bench). """
  if device_index is None:
    device_index = torch.cuda.current_device()
  cache = _pair_caches.get(device_index)
  return dict(cache.stats) if cache is not None else dict(full=0, star=0, off=0)

# ---------------------------------------------------------------------------- #
# Distance-based rules (single device).  Each returns (out, selection) where `selection` is a
# DEVICE int32 tensor (all n indices by increasing score/distance; brute: the n-f subset).

def _aux(prep):
  ws = _workspace(prep.device, prep.stream)
  meta = torch.empty(prep.n + 1, dtype=torch.int32, device=prep.device)   # order[n] + status
  return ws, meta

def krum(gradients, f, m):
  prep = _prepare(gradients)
  out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  ws, meta = _aux(prep)
  cache = _pair_cache(prep, gradients)
  with _on(prep.device):
    if cache is None:
      code = _lib.lib().bz_krum(prep.ptrs, prep.n, int(f), int(m), prep.d, out.data_ptr(), meta.data_ptr(),
                                ws.data_ptr(), ws.numel(), prep.stream)
    else:
      old, cache_in, u_old = cache.old_index(gradients, prep.d, prep.stream)
      code = _lib.lib().bz_krum_reuse(prep.ptrs, prep.n, int(f), int(m), prep.d, out.data_ptr(), meta.data_ptr(), old, cache_in, u_old,
                                      cache.out_buffer(), ctypes.byref(cache.mode), ws.data_ptr(), ws.numel(), prep.stream)
  _lib.check(code, "bz_krum")
  if cache is not None:
    cache.update(gradients, prep.d, prep.stream)
  return _finish(prep, out), meta[:prep.n]

def bulyan(gradients, f, m):
  prep = _prepare(gradients)
  out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  ws, meta = _aux(prep)
  status = meta[prep.n:]
  cache = _pair_cache(prep, gradients)
  with _on(prep.device):
    if cache is None:
      code = _lib.lib().bz_bulyan(prep.ptrs, prep.n, int(f), int(m), prep.d, out.data_ptr(), meta.data_ptr(),
                                  status.data_ptr(), ws.data_ptr(), ws.numel(), prep.stream)
    else:
      old, cache_in, u_old = cache.old_index(gradients, prep.d, prep.stream)
      code = _lib.lib().bz_bulyan_reuse(prep.ptrs, prep.n, int(f), int(m), prep.d, out.data_ptr(), meta.data_ptr(), status.data_ptr(),
                                        old, cache_in, u_old, cache.out_buffer(), ctypes.byref(cache.mode), ws.data_ptr(), ws.numel(), prep.stream)
  _lib.check(code, "bz_bulyan")
  if cache is not None:
    cache.update(gradients, prep.d, prep.stream)
  if config.strict_status:
    _raise_status(int(status.item()))
  return _finish(prep, out), meta[:prep.n]

def brute(gradients, f):
  prep = _prepare(gradients)
  out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  ws, meta = _aux(prep)
  status = meta[prep.n:]
  cache = _pair_cache(prep, gradients)
  with _on(prep.device):
    if cache is None:
      code = _lib.lib().bz_brute(prep.ptrs, prep.n, int(f), prep.d, out.data_ptr(), meta.data_ptr(),
                                 status.data_ptr(), ws.data_ptr(), ws.numel(), prep.stream)
    else:
      old, cache_in, u_old = cache.old_index(gradients, prep.d, prep.stream)
      code = _lib.lib().bz_brute_reuse(prep.ptrs, prep.n, int(f), prep.d, out.data_ptr(), meta.data_ptr(), status.data_ptr(),
                                       old, cache_in, u_old, cache.out_buffer(), ctypes.byref(cache.mode), ws.data_ptr(), ws.numel(), prep.stream)
  _lib.check(code, "bz_brute")
  if cache is not None:
    cache.update(gradients, prep.d, prep.stream)
  if config.strict_status:
    _raise_status(int(status.item()))
  return _finish(prep, out), meta[:prep.n - int(f)]

def aksel(gradients, f, mode="mid"):
  if mode not in _lib.AKSEL_MODES:
    raise NotImplementedError(mode)      # aksel.py:47-48
  prep = _prepare(gradients)
  out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  ws, meta = _aux(prep)
  with _on(prep.device):
    code = _lib.lib().bz_aksel(prep.ptrs, prep.n, int(f), _lib.AKSEL_MODES[mode], prep.d, out.data_ptr(),
                               meta.data_ptr(), ws.data_ptr(), ws.numel(), prep.stream)
  _lib.check(code, "bz_aksel")
  return _finish(prep, out), meta[:prep.n]

def cge(gradients, f):
  prep = _prepare(gradients)
  out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  ws, meta = _aux(prep)
  with _on(prep.device):
    code = _lib.lib().bz_cge(prep.ptrs, prep.n, int(f), prep.d, out.data_ptr(), meta.data_ptr(),
                             ws.data_ptr(), ws.numel(), prep.stream)
  _lib.check(code, "bz_cge")
  return _finish(prep, out), meta[:prep.n]

# ---------------------------------------------------------------------------- #
# Study metrics on the same stack (tools/pytorch.py:97-125, attack.py:846-848)

def avg_dev_max_async(samples):
  """ (avg, stats): the average of the rows and a DEVICE fp64 vector [2 + n]:
  stats[0] = ||avg||^2, stats[1] = max |avg|, stats[2 + i] = ||samples[i] - avg||^2.  No sync. """
  prep = _prepare_device(samples, "the study metrics take CUDA tensors (tools.compute_avg_dev_max handles CPU samples)")
  avg = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  stats = torch.empty(2 + prep.n, dtype=torch.float64, device=prep.device)
  ws = _workspace(prep.device, prep.stream)
  with _on(prep.device):
    code = _lib.lib().bz_avg_dev_max(prep.ptrs, prep.n, prep.d, avg.data_ptr(), stats.data_ptr(),
                                     ws.data_ptr(), ws.numel(), prep.stream)
  _lib.check(code, "bz_avg_dev_max")
  return avg, stats

class _StudyMemo:
  """ Last `compute_avg_dev_max` result, valid for the very same tensor objects at the same
  addresses and in-place versions (weak references: a dead or different tensor never matches).
  attack.py:846-847 asks for the sampled and for the honest gradients; without worker/server-side
  momentum and with nb_for_study = nb_honests those are the SAME tensors (`grad_honests =
  grad_sampleds[:nb_honests]`, attack.py:808): the second pass over n x d is saved. """
  def __init__(self):
    self.refs = self.state = self.result = None
  def lookup(self, samples):
    if self.refs is None or len(self.refs) != len(samples):
      return None
    for ref, g in zip(self.refs, samples):
      if ref() is not g:
        return None
    if tuple((g.data_ptr(), g._version) for g in samples) != self.state:
      return None
    avg, a, b, c = self.result
    return avg.clone(), a, b, c                               # callers own the average they get (grad_pasts keeps it)
  def store(self, samples, result):
    try:
      self.refs = tuple(weakref.ref(g) for g in samples)
    except TypeError:
      self.refs = None
      return
    self.state = tuple((g.data_ptr(), g._version) for g in samples)
    self.result = result

_study_memo = _StudyMemo()

def compute_avg_dev_max(samples):
  """ Drop-in for `tools.compute_avg_dev_max(samples)` (tools/pytorch.py:97-125): returns
  (average gradient or None, norm of the average, norm standard deviation, max |coordinate| of the
  average).  One device->host read of 2 + n doubles instead of the reference's n + 2 `.item()`s. """
  n = len(samples)
  if n == 0:
    return None, math.nan, math.nan, math.nan                 # :105-106
  hit = _study_memo.lookup(samples)
  if hit is not None:
    return hit
  result = _compute_avg_dev_max(samples, n)
  _study_memo.store(samples, (result[0].clone(),) + result[1:])
  return result

def _compute_avg_dev_max(samples, n):
  avg, stats = avg_dev_max_async(samples)
  return _study_tuple(avg, stats.tolist(), n)                 # the only synchronisation

def _study_tuple(avg, host, n):
  norm_avg = ctypes.c_float(math.sqrt(host[0])).value      # :110 returns an fp32 norm: same rounding in the logs
  norm_max = host[1]
  if n >= 2:
    norm_var = 0.
    for value in host[2:]:                                    # :116-120: same left-to-right sum
      norm_var += value
    norm_dev = math.sqrt(norm_var / (n - 1))
  else:
    norm_dev = math.nan                                       # :122-123
  return avg, norm_avg, norm_dev, norm_max

def rowdots_async(center, rows):
  """ DEVICE fp64 vector: out[i] = <rows[i], center>, all rows in one pass (`bz_rowdots`).  No sync. """
  rows = list(rows)
  if len(rows) > _lib.MAX_N:
    return torch.cat([rowdots_async(center, rows[k:k + _lib.MAX_N]) for k in range(0, len(rows), _lib.MAX_N)])
  prep = _prepare_device(rows, "the study dot products take CUDA tensors")
  if center.dtype != torch.float32 or center.shape != (prep.d,) or center.device != prep.device or not center.is_contiguous():
    raise ValueError("center must be a contiguous float32 vector like the rows")
  out = torch.empty(prep.n, dtype=torch.float64, device=prep.device)
  ws = _workspace(prep.device, prep.stream)
  with _on(prep.device):
    code = _lib.lib().bz_rowdots(prep.ptrs, prep.n, center.data_ptr(), prep.d, out.data_ptr(), ws.data_ptr(), ws.numel(), prep.stream)
  _lib.check(code, "bz_rowdots")
  return out

def study_step(grad_sampleds, grad_honests, grad_attacks, grad_defense, pasts, momentum):
  """ Everything attack.py:846-866 computes for one line of the study file, on the device:
    * the three `tools.compute_avg_dev_max` calls (K6, one pass each; a repeated list is computed once),
    * the norm and the largest |coordinate| of the defense gradient,
    * the six cosines between the sampled / honest / attack averages and the defense gradient,
    * the cosine with the last past gradient and the curvature sum over all past gradients
  with THREE passes of `bz_rowdots` (one vector against many) instead of 7 + len(pasts) `torch.dot(...).item()`
  and ONE device->host read for the whole step (the reference: 9 + len(samples) + len(pasts) `.item()`s).
  Args:
    grad_sampleds, grad_honests, grad_attacks  Lists of CUDA gradients (the attack list may be empty)
    grad_defense  The aggregated gradient
    pasts         Iterable of (gradient, norm) of the past sampled averages, most recent first
    momentum      args.momentum
  Returns:
    dict with the reference's variable names (attack.py:846-866) """
  nan = math.nan
  pasts = list(pasts)
  ns, nh, na = len(grad_sampleds), len(grad_honests), len(grad_attacks)
  s_avg, s_stats = avg_dev_max_async(grad_sampleds)
  same = nh == ns and all(a is b for a, b in zip(grad_sampleds, grad_honests))      # attack.py:808 without momentum placement
  h_avg, h_stats = (s_avg, s_stats) if same else avg_dev_max_async(grad_honests)
  have_attack = na > 0
  a_avg, a_stats = avg_dev_max_async(grad_attacks) if have_attack else (None, s_stats[:0])
  # one vector against many, three times; every result lands in one device vector read once
  first = [h_avg] + ([a_avg] if have_attack else []) + [grad_defense] + [g for g, _ in pasts]
  second = ([a_avg] if have_attack else []) + [grad_defense]
  host = torch.cat([s_stats, h_stats, a_stats, rowdots_async(s_avg, first), rowdots_async(h_avg, second),
                    rowdots_async(grad_defense, second), grad_defense.abs().max().double().reshape(1)]).tolist()    # the only synchronisation
  _, s_norm, s_dev, s_max = _study_tuple(None, host[:2 + ns], ns)
  _, h_norm, h_dev, h_max = _study_tuple(None, host[2 + ns:4 + ns + nh], nh)
  if have_attack:
    _, a_norm, a_dev, a_max = _study_tuple(None, host[4 + ns + nh:6 + ns + nh + na], na)
    dots = host[6 + ns + nh + na:]
  else:
    a_norm = a_dev = a_max = nan
    dots = host[4 + ns + nh:]
  k = 0
  sh = dots[k]; k += 1
  sa = dots[k] if have_attack else nan; k += 1 if have_attack else 0
  sd = dots[k]; k += 1
  past_dots = dots[k:k + len(pasts)]; k += len(pasts)
  ha = dots[k] if have_attack else nan; k += 1 if have_attack else 0
  hd = dots[k]; k += 1
  ad = dots[k] if have_attack else nan; k += 1 if have_attack else 0
  dd = dots[k]; k += 1
  d_max = dots[k]
  d_norm = ctypes.c_float(math.sqrt(dd)).value            # Tensor.norm() is an fp32 value (attack.py:851)
  f32 = lambda x: ctypes.c_float(x).value                 # torch.dot(...).div_().div_().item(): fp32 arithmetic
  def div(a, b):                                          # IEEE division (a zero norm gives inf / nan, as div_ does)
    try:
      return f32(a / b)
    except ZeroDivisionError:
      return nan if a == 0 or math.isnan(a) else math.copysign(math.inf, a) * math.copysign(1., b)
  cos = lambda dot, na, nb: div(div(f32(dot), na), nb)
  out = dict(sampled_grad_avg=s_avg, sampled_norm_avg=s_norm, sampled_norm_dev=s_dev, sampled_norm_max=s_max,
             honest_grad_avg=h_avg, honest_norm_avg=h_norm, honest_norm_dev=h_dev, honest_norm_max=h_max,
             attack_grad_avg=a_avg, attack_norm_avg=a_norm, attack_norm_dev=a_dev, attack_norm_max=a_max,
             defense_norm_avg=d_norm, defense_norm_max=f32(d_max),
             cosin_splhon=cos(sh, s_norm, h_norm), cosin_splatt=cos(sa, s_norm, a_norm) if have_attack else nan,
             cosin_spldef=cos(sd, s_norm, d_norm), cosin_honatt=cos(ha, h_norm, a_norm) if have_attack else nan,
             cosin_hondef=cos(hd, h_norm, d_norm), cosin_attdef=cos(ad, a_norm, d_norm) if have_attack else nan)
  if pasts:
    out["cosin_sampled"] = cos(past_dots[0], s_norm, pasts[0][1])
    out["curv_sampled"] = momentum * sum((momentum ** i) * f32(dot) for i, dot in enumerate(past_dots))
  else:
    out["cosin_sampled"] = nan
    out["curv_sampled"] = nan
  return out

# ---------------------------------------------------------------------------- #
# Phases of the d-sharded multi-GPU path (device tensors only)

def _prepare_device(gradients, message="the sharded phases take CUDA tensors"):
  prep = _prepare(gradients)
  if prep.to_cpu:
    raise ValueError(message)
  return prep

def pairdist_partial(gradients):
  """ [n, n] fp64: this shard's share of the squared pairwise distances (entries i < j). """
  prep = _prepare_device(gradients)
  part = torch.empty((prep.n, prep.n), dtype=torch.float64, device=prep.device)
  ws = _workspace(prep.device, prep.stream)
  with _on(prep.device):
    code = _lib.lib().bz_pairdist_partial(prep.ptrs, prep.n, prep.d, part.data_ptr(), ws.data_ptr(), ws.numel(), prep.stream)
  _lib.check(code, "bz_pairdist_partial")
  return part

def rowdist_partial(gradients, center=None):
  """ [n] fp64: this shard's share of the squared distance of every row to `center` (None: origin). """
  prep = _prepare_device(gradients)
  part = torch.empty(prep.n, dtype=torch.float64, device=prep.device)
  ws = _workspace(prep.device, prep.stream)
  cptr = None
  if center is not None:
    if center.dtype != torch.float32 or center.shape != (prep.d,) or center.device != prep.device or not center.is_contiguous():
      raise ValueError("center must be a contiguous float32 vector like the rows")
    cptr = center.data_ptr()
  with _on(prep.device):
    code = _lib.lib().bz_rowdist_partial(prep.ptrs, prep.n, cptr, prep.d, part.data_ptr(), ws.data_ptr(), ws.numel(), prep.stream)
  _lib.check(code, "bz_rowdist_partial")
  return part

def _select_common(parts, n):
  if parts.dtype != torch.float64 or not parts.is_contiguous() or parts.device.type != "cuda":
    raise ValueError("parts must be a contiguous float64 CUDA tensor")
  nparts = parts.shape[0]
  meta = torch.empty(n + 1, dtype=torch.int32, device=parts.device)
  stream = torch.cuda.current_stream(parts.device).cuda_stream
  return nparts, meta, stream

def krum_select(parts, n, f):
  """ parts: [R, n, n] gathered partial blocks -> order (device int32[n]). """
  nparts, meta, stream = _select_common(parts, n)
  with _on(parts.device):
    code = _lib.lib().bz_krum_select(parts.data_ptr(), nparts, n, int(f), meta.data_ptr(), stream)
  _lib.check(code, "bz_krum_select")
  return meta[:n]

def bulyan_select(parts, n, f, m):
  nparts, meta, stream = _select_common(parts, n)
  with _on(parts.device):
    code = _lib.lib().bz_bulyan_select(parts.data_ptr(), nparts, n, int(f), int(m), meta.data_ptr(), meta[n:].data_ptr(), stream)
  _lib.check(code, "bz_bulyan_select")
  return meta[:n], meta[n:]

def brute_select(parts, n, f):
  nparts, meta, stream = _select_common(parts, n)
  with _on(parts.device):
    code = _lib.lib().bz_brute_select(parts.data_ptr(), nparts, n, int(f), meta.data_ptr(), meta[n:].data_ptr(), stream)
  _lib.check(code, "bz_brute_select")
  return meta[:n - int(f)], meta[n:]

def rowdist_select(parts, n, sqrt_norm):
  nparts, meta, stream = _select_common(parts, n)
  with _on(parts.device):
    code = _lib.lib().bz_rowdist_select(parts.data_ptr(), nparts, n, 1 if sqrt_norm else 0, meta.data_ptr(), stream)
  _lib.check(code, "bz_rowdist_select")
  return meta[:n]

# Peer-memory variants of phase B: `peer_ptrs` is a list of R device addresses (one per rank, rank
# order) of the ranks' partial blocks, mapped over NVLink; the blocks are read in place.

def _peers(peer_ptrs, n, device):
  if not 1 <= len(peer_ptrs) <= _lib.MAX_PEERS:
    raise ValueError(f"{len(peer_ptrs)} peers, expected 1..{_lib.MAX_PEERS}")
  table = (ctypes.c_void_p * len(peer_ptrs))(*[int(p) for p in peer_ptrs])
  meta = torch.empty(n + 1, dtype=torch.int32, device=device)
  return table, meta, torch.cuda.current_stream(device).cuda_stream

def krum_select_peers(peer_ptrs, n, f, device):
  table, meta, stream = _peers(peer_ptrs, n, device)
  with _on(device):
    code = _lib.lib().bz_krum_select_peers(table, len(peer_ptrs), n, int(f), meta.data_ptr(), stream)
  _lib.check(code, "bz_krum_select_peers")
  return meta[:n]

def bulyan_select_peers(peer_ptrs, n, f, m, device):
  table, meta, stream = _peers(peer_ptrs, n, device)
  with _on(device):
    code = _lib.lib().bz_bulyan_select_peers(table, len(peer_ptrs), n, int(f), int(m), meta.data_ptr(), meta[n:].data_ptr(), stream)
  _lib.check(code, "bz_bulyan_select_peers")
  return meta[:n], meta[n:]

def brute_select_peers(peer_ptrs, n, f, device):
  table, meta, stream = _peers(peer_ptrs, n, device)
  with _on(device):
    code = _lib.lib().bz_brute_select_peers(table, len(peer_ptrs), n, int(f), meta.data_ptr(), meta[n:].data_ptr(), stream)
  _lib.check(code, "bz_brute_select_peers")
  return meta[:n - int(f)], meta[n:]

def rowdist_select_peers(peer_ptrs, n, sqrt_norm, device):
  table, meta, stream = _peers(peer_ptrs, n, device)
  with _on(device):
    code = _lib.lib().bz_rowdist_select_peers(table, len(peer_ptrs), n, 1 if sqrt_norm else 0, meta.data_ptr(), stream)
  _lib.check(code, "bz_rowdist_select_peers")
  return meta[:n]

def pairdist_partial_into(gradients, part):
  """ Phase A writing straight into `part` (e.g. this rank's slot of a symmetric buffer). """
  prep = _prepare_device(gradients)
  ws = _workspace(prep.device, prep.stream)
  with _on(prep.device):
    code = _lib.lib().bz_pairdist_partial(prep.ptrs, prep.n, prep.d, part.data_ptr(), ws.data_ptr(), ws.numel(), prep.stream)
  _lib.check(code, "bz_pairdist_partial")
  return part

def rowdist_partial_into(gradients, center, part):
  prep = _prepare_device(gradients)
  ws = _workspace(prep.device, prep.stream)
  cptr = None if center is None else center.data_ptr()
  with _on(prep.device):
    code = _lib.lib().bz_rowdist_partial(prep.ptrs, prep.n, cptr, prep.d, part.data_ptr(), ws.data_ptr(), ws.numel(), prep.stream)
  _lib.check(code, "bz_rowdist_partial")
  return part

def average_selected(gradients, selection, count, zero_init=True, divisor=None, status=None):
  """ Ordered-subset average of the local shard; `selection` is a device int32 tensor or None. """
  prep = _prepare_device(gradients)
  out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  sel_ptr = None if selection is None else selection.data_ptr()
  st_ptr = None if status is None else status.data_ptr()
  with _on(prep.device):
    code = _lib.lib().bz_average_selected(prep.ptrs, prep.n, sel_ptr, int(count), 1 if zero_init else 0,
                                          float(count if divisor is None else divisor), st_ptr, prep.d, out.data_ptr(), prep.stream)
  _lib.check(code, "bz_average_selected")
  return out

def bulyan_reduce(gradients, f, m, order, status=None):
  prep = _prepare_device(gradients)
  out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  st_ptr = None if status is None else status.data_ptr()
  with _on(prep.device):
    code = _lib.lib().bz_bulyan_reduce(prep.ptrs, prep.n, int(f), int(m), order.data_ptr(), st_ptr, prep.d, out.data_ptr(), prep.stream)
  _lib.check(code, "bz_bulyan_reduce")
  return out

# ---------------------------------------------------------------------------- #
# Gradient production (SURVEY.md §8(f) row 2; attack.py:776-780, 791-795, 799-810)

class GradientStack:
  """ The n worker gradients of a step as rows of ONE preallocated [n, d] device buffer, filled by
  `bz_gradient_row`: per worker, one pass that clips (norm and scale stay on the device: no
  `.item()`), writes the sampled row (the reference's `grad.clone()`) and applies the momentum
  placement — instead of norm + mul_ + clone + mul_ + add_ (7 vector passes and a host sync).

      stack = GradientStack(n_sampled, d, device)            # once
      for i in range(n_sampled):                             # every step
        grad, loss = model.backprop(outloss=True)
        stack.push(i, grad, clip=args.gradient_clip)                              # momentum at "update"
        stack.push(i, grad, clip, worker_momentum=gmtm[i], mu=0.9, dampening=0.)   # at "worker": gmtm[i] updated in place
        stack.push(i, grad, clip, server_momentum=gserver, mu=0.9, dampening=0.)   # at "server": honest row i written
      rows = stack.sampled(k)  /  stack.honest(k)             # lists of row views for the rule

  Bit-exact with the ATen sequence (tests/test_cuda_gradient_rows.py); when clipping occurs the
  scale factor may differ by 1 ulp (ATen's fp32 norm order is build specific). """
  def __init__(self, n, d, device):
    self.n, self.d, self.device = n, d, torch.device(device)
    pitch = (d + 63) // 64 * 64                     # rows 256-byte aligned: vector loads, TMA bulk copies
    self._sampled = torch.empty((n, pitch), dtype=torch.float32, device=self.device)
    self._honest = None
    self._pitch = pitch
    self._lib = _lib.lib()
  def _honest_buffer(self):
    if self._honest is None:
      self._honest = torch.empty((self.n, self._pitch), dtype=torch.float32, device=self.device)
    return self._honest
  def push(self, i, grad, clip=None, worker_momentum=None, server_momentum=None, mu=0., dampening=0.):
    """ Row i <- this worker's gradient.  Returns the sampled row (a view of the buffer). """
    if grad.dtype != torch.float32 or grad.dim() != 1 or grad.numel() != self.d or not grad.is_contiguous() or grad.device != self.device:
      raise ValueError("grad must be a contiguous float32 vector of d elements on the stack's device")
    if worker_momentum is not None and server_momentum is not None:
      raise ValueError("worker-side and server-side momentum are exclusive (attack.py:799-810)")
    row = self._sampled[i, :self.d]
    mode, mom, honest = 0, None, None
    if worker_momentum is not None:
      mode, mom = 1, worker_momentum
    elif server_momentum is not None:
      mode, mom, honest = 2, server_momentum, self._honest_buffer()[i, :self.d]
    if mom is not None and (mom.dtype != torch.float32 or mom.shape != (self.d,) or not mom.is_contiguous() or mom.device != self.device):
      raise ValueError("momentum must be a contiguous float32 vector like the gradient")
    stream = torch.cuda.current_stream(self.device).cuda_stream
    ws = _workspace(self.device, stream)
    with _on(self.device):
      code = self._lib.bz_gradient_row(grad.data_ptr(), self.d, float(clip) if clip is not None else 0., row.data_ptr(), mode,
                                       None if mom is None else mom.data_ptr(), float(mu), 1. - float(dampening),
                                       None if honest is None else honest.data_ptr(), ws.data_ptr(), ws.numel(), stream)
    _lib.check(code, "bz_gradient_row")
    # the kernel wrote through raw pointers: tell PyTorch (the identity/version keyed caches of this
    # package — prepared arguments, selection, distance table, study memo — rely on the counter;
    # views share it with their base, so every row of the buffer is invalidated: conservative)
    _bump = torch.autograd.graph.increment_version
    _bump(row)
    if mode == 1:
      _bump(mom)
    elif mode == 2:
      _bump(honest)
    return row
  def sampled(self, count=None):
    return [self._sampled[i, :self.d] for i in range(self.n if count is None else count)]
  def honest(self, count=None):
    buf = self._honest_buffer()
    return [buf[i, :self.d] for i in range(self.n if count is None else count)]

# ---------------------------------------------------------------------------- #
# Prepared calls

class Plan:
  """ A prepared aggregation: every argument of the C-ABI call is resolved once (row pointers,
  output, workspace, stream), `plan()` then only issues the call — a few microseconds of host
  time, no allocation, no host/device synchronisation — so the call can run back to back at
  kernel rate or be captured in a CUDA graph.  The row tensors and the output are held by the
  plan; their CONTENT may change between calls (e.g. momentum buffers updated in place).
      plan = engine.Plan("krum", gradients, f=5)
      aggregated = plan()          # same tensor every time: plan.out
      plan.selection               # device int32 (distance-based rules)
  For brute / bulyan the device status word is NOT checked here (that would synchronise);
  read `plan.status` when needed: non-zero means the rule is undefined on this data and `out`
  is NaN. """
  def __init__(self, gar, gradients, f=None, m=None, mode="mid", out=None):
    prep = _prepare(list(gradients))
    if prep.to_cpu:
      raise ValueError("Plan takes CUDA tensors (host tensors go through the plain call, which stages them)")
    lib = _lib.lib()
    n, d = prep.n, prep.d
    self.gar, self.n, self.d, self.device = gar, n, d, prep.device
    self.rows = list(gradients)
    if not all(g.is_contiguous() for g in self.rows):
      # a packed copy would neither stay alive nor follow in-place updates of the originals
      raise ValueError("Plan takes contiguous rows (the plain call accepts strided views and packs them)")
    self.out = torch.empty(d, dtype=torch.float32, device=prep.device) if out is None else out
    if self.out.dtype != torch.float32 or self.out.shape != (d,) or self.out.device != prep.device or not self.out.is_contiguous():
      raise ValueError("out must be a contiguous float32 vector like the rows")
    self._ptrs = (ctypes.c_void_p * n)(*[g.data_ptr() for g in self.rows])
    self._stream = prep.stream
    self.selection = None
    self.status = None
    o, st = self.out.data_ptr(), self._stream
    if gar in ("average", "median"):
      fn, args = getattr(lib, "bz_" + gar), (self._ptrs, n, d, o, st)
    elif gar in ("trmean", "phocas", "meamed"):
      fn, args = getattr(lib, "bz_" + gar), (self._ptrs, n, int(f), d, o, st)
    else:
      self._ws = _workspace(prep.device, prep.stream)
      self._meta = torch.empty(n + 1, dtype=torch.int32, device=prep.device)
      ws, wn, meta, status = self._ws.data_ptr(), self._ws.numel(), self._meta.data_ptr(), self._meta[n:].data_ptr()
      self.selection = self._meta[:n]
      if gar == "krum":
        m = n - f - 2 if m is None else m
        fn, args = lib.bz_krum, (self._ptrs, n, int(f), int(m), d, o, meta, ws, wn, st)
      elif gar == "bulyan":
        m = n - f - 2 if m is None else m
        self.status = self._meta[n:]
        fn, args = lib.bz_bulyan, (self._ptrs, n, int(f), int(m), d, o, meta, status, ws, wn, st)
      elif gar == "brute":
        self.status = self._meta[n:]
        self.selection = self._meta[:n - int(f)]
        fn, args = lib.bz_brute, (self._ptrs, n, int(f), d, o, meta, status, ws, wn, st)
      elif gar == "aksel":
        fn, args = lib.bz_aksel, (self._ptrs, n, int(f), _lib.AKSEL_MODES[mode], d, o, meta, ws, wn, st)
      elif gar == "cge":
        fn, args = lib.bz_cge, (self._ptrs, n, int(f), d, o, meta, ws, wn, st)
      else:
        raise KeyError(f"unknown aggregation rule {gar!r}")
    self._fn, self._args, self._what = fn, args, "bz_" + gar
    self._graph = None
  def graph(self):
    """ Capture the prepared call in a CUDA graph and return `replay`: a callable that launches the
    whole rule (memset + distance pass with its fused scoring + reduce pass, with their
    programmatic-dependent-launch edges) as ONE graph launch and returns `plan.out`.  Every launch
    of the library is capturable (it never synchronises and allocates nothing).  Worth it where
    launch latency shows: small d, or a host loop that cannot stay ahead of the GPU. """
    if self._graph is None:
      with _on(self.device):
        self()                                           # warm-up outside the capture (module loading, attributes)
        torch.cuda.synchronize(self.device)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
          stream = torch.cuda.current_stream(self.device).cuda_stream      # the capture stream
          code = self._fn(*(self._args[:-1] + (stream,)))
        if code != 0:
          _lib.check(code, self._what)
      self._graph = graph
    graph, out = self._graph, self.out
    def replay():
      graph.replay()
      return out
    return replay
  def __call__(self):
    if torch.cuda.current_device() == self.device.index:
      code = self._fn(*self._args)
    else:
      with _on(self.device):           # the launches go to the device that owns the rows
        code = self._fn(*self._args)
    if code != 0:
      _lib.check(code, self._what)
    return self.out
