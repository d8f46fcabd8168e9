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
import functools
import math
import time
import weakref

import torch

from . import _lib, hostmem

__all__ = ["average", "median", "trmean", "phocas", "meamed", "krum", "bulyan", "brute", "aksel", "cge",
           "pairdist_partial", "rowdist_partial", "select", "krum_select", "bulyan_select", "brute_select",
           "rowdist_select", "average_selected", "bulyan_reduce", "avg_dev_max_async", "compute_avg_dev_max", "rowdots_async", "study_step",
           "StudyPartials", "study_partials", "study_finish",
           "LineSearch", "line_search", "config", "Plan", "pair_cache_stats", "GradientStack", "gradient_scatter", "momentum_rows", "host_path_report"]

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

def _row_buffer(rows, d, device):
  """ [rows, pitch] fp32 device buffer whose rows start 256-byte aligned (vector loads, TMA bulk copies). """
  return torch.empty((rows, (d + 63) // 64 * 64), dtype=torch.float32, device=device)

def _staging_buffer(device, rows, d):
  """ The device buffer host rows are staged into; one shape is kept at a time. """
  key = (device.index, rows, d)
  buf = _staging.get(key)
  if buf is None:
    _staging.clear()
    buf = _staging[key] = _row_buffer(rows, d, device)
  return buf

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

def _host_path(device):
  path = _host_paths.get(device.index)
  if path is None:
    path = _host_paths[device.index] = _HostPath()
  return path

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
    mode = _host_path(device).choose(single_pass, pinned)
    prep.host_mode = (single_pass, pinned, mode)
    torch.cuda.current_stream(device).synchronize()        # the clock below times this call only
    prep.host_t0 = time.perf_counter()
    buf = _staging_buffer(device, len(uniq), d)
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
      _run(device, _lib.lib().bz_stage_rows, (hosts, len(uniq), d, buf.data_ptr(), buf.stride(0), lanes[0].cuda_stream))
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

def _call(fn, args):
  """ One C-ABI call; raises on a non-zero return code. """
  code = fn(*args)
  if code != 0:
    _lib.check(code, fn.__name__)

def _run(device, fn, args):
  """ `_call` with `device` current. """
  with _on(device):
    _call(fn, args)

def _check_like_rows(vector, prep, what):
  if vector.dtype != torch.float32 or vector.shape != (prep.d,) or vector.device != prep.device or not vector.is_contiguous():
    raise ValueError(f"{what} must be a contiguous float32 vector like the rows")

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
  buf = _staging_buffer(device, n, d)
  out = torch.empty(d, dtype=torch.float32, device=device)
  result = torch.empty(d, dtype=torch.float32, pin_memory=True)
  current = torch.cuda.current_stream(device)
  lanes = _copy_streams(device)
  ptrs = (ctypes.c_void_p * n)(*[g.data_ptr() for g in rows])
  _run(device, _lib.lib().bz_coordinate_host, (_RULE_CODES[name], ptrs, n, 0 if f is None else int(f), d, result.data_ptr(),
                                               buf.data_ptr(), buf.stride(0), out.data_ptr(), _PIPELINE_CHUNKS,
                                               current.cuda_stream, lanes[0].cuda_stream, lanes[1].cuda_stream))
  current.synchronize()           # the host rows, `out` and the staging rows stay alive until here
  path.record(True, False, "pipeline", time.perf_counter() - t0)
  return result

def _coordinate_call(name, prep, f, out):
  """ (fn, args) of the coordinate-wise rule `name` writing to the address `out`. """
  head = (prep.ptrs, prep.n, int(f)) if name in ("trmean", "phocas", "meamed") else (prep.ptrs, prep.n)
  return getattr(_lib.lib(), "bz_" + name), head + (prep.d, out, prep.stream)

def _coordinate(name, gradients, f=None):
  if type(gradients) in (list, tuple) and len(gradients) > 0 and isinstance(gradients[0], torch.Tensor) and gradients[0].device.type == "cpu" and torch.cuda.is_available():
    _validate(gradients)
    _lib.lib()
    device = torch.device("cuda", torch.cuda.current_device())
    path = _host_path(device)
    if path.choose(True, False) == "pipeline":
      torch.cuda.current_stream(device).synchronize()        # the clock times this call only
      return _coordinate_pipeline(name, gradients, f, path, device)
  prep = _prepare(gradients, single_pass=True)
  out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  _run(prep.device, *_coordinate_call(name, prep, f, out.data_ptr()))
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
# Distance-based rules: what each one runs, resolved once for the plain call, `Plan` and the
# phases of the d-sharded path

DISTANCE_BASED = ("krum", "bulyan", "brute", "aksel", "cge")

class _Rule:
  """ The facts of a distance-based rule for (gar, n, f, m, mode):
    m              Multi-Krum selection size (krum, bulyan; default n - f - 2)
    params         its arguments after (rows, n) in `bz_<gar>`
    pair           the distances are pairwise (else from every row to `center`)
    center         the distances are to the coordinate-wise median (aksel; else cge: to the origin)
    select, select_params   phase B: `bz_<select>_select[_peers]`, its arguments after (blocks, R, n)
                            (those of `<select>_select[_peers]` after (blocks, n))
    status         the rule reports a status word, after the n-entry order (bulyan, brute)
    count, zero_init        phase C of all but bulyan: average of the first `count` selected rows
    length         length of the selection returned """
  __slots__ = ("gar", "n", "f", "m", "params", "pair", "center", "select", "select_params", "status", "count", "zero_init", "length")
  def __init__(self, gar, n, f, m, mode):
    if gar not in DISTANCE_BASED:
      raise KeyError(f"unknown aggregation rule {gar!r}")
    f = int(f)
    m = n - f - 2 if m is None else int(m)
    self.gar, self.n, self.f, self.m = gar, n, f, m
    self.pair = gar in ("krum", "bulyan", "brute")
    self.center = gar == "aksel"
    self.status = gar in ("bulyan", "brute")
    self.zero_init = gar != "cge"
    self.length = n - f if gar == "brute" else n
    if gar == "aksel":
      if mode not in _lib.AKSEL_MODES:
        raise NotImplementedError(mode)      # aksel.py:47-48
      self.params = (f, _lib.AKSEL_MODES[mode])
      self.count = (n + 1) // 2 if mode == "mid" else n - f
    else:
      self.params = (f, m) if gar in ("krum", "bulyan") else (f,)
      self.count = m if gar == "krum" else n - f
    self.select = gar if self.pair else "rowdist"
    self.select_params = (f, m) if gar == "bulyan" else (f,) if self.pair else (int(gar == "cge"),)
  def entry(self, ptrs, d, out, meta, ws, stream, reuse=()):
    """ (fn, args) of the single-GPU call `bz_<gar>` writing to the addresses `out` and `meta`
    (order[n] + status), or of `bz_<gar>_reuse` given the distance cache's `reuse` arguments. """
    status = (meta + 4 * self.n,) if self.status else ()
    fn = getattr(_lib.lib(), "bz_" + self.gar + ("_reuse" if reuse else ""))
    return fn, (ptrs, self.n) + self.params + (d, out, meta) + status + reuse + (ws.data_ptr(), ws.numel(), stream)

@functools.lru_cache(maxsize=256)
def _rule(gar, n, f, m=None, mode="mid"):
  """ The `_Rule` of these arguments; KeyError for an unknown rule, NotImplementedError for an unknown aksel mode. """
  return _Rule(gar, n, f, m, mode)

def _distance(gar, gradients, f, m=None, mode="mid"):
  """ The single-device call: (out, selection) where `selection` is a DEVICE int32 tensor (all n
  indices by increasing score/distance; brute: the n-f subset). """
  rule = _rule(gar, len(gradients) if isinstance(gradients, (list, tuple)) else 0, f, m, mode)    # before the device is touched
  prep = _prepare(gradients)
  out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  ws = _workspace(prep.device, prep.stream)
  meta = torch.empty(prep.n + 1, dtype=torch.int32, device=prep.device)   # order[n] + status
  cache = _pair_cache(prep, gradients) if rule.pair else None
  reuse = () if cache is None else cache.old_index(gradients, prep.d, prep.stream) + (cache.out_buffer(), ctypes.byref(cache.mode))
  _run(prep.device, *rule.entry(prep.ptrs, prep.d, out.data_ptr(), meta.data_ptr(), ws, prep.stream, reuse))
  if cache is not None:
    cache.update(gradients, prep.d, prep.stream)
  if rule.status and config.strict_status:
    _raise_status(int(meta[prep.n].item()))
  return _finish(prep, out), meta[:rule.length]

def krum(gradients, f, m=None):
  return _distance("krum", gradients, f, m)

def bulyan(gradients, f, m=None):
  return _distance("bulyan", gradients, f, m)

def brute(gradients, f):
  return _distance("brute", gradients, f)

def aksel(gradients, f, mode="mid"):
  return _distance("aksel", gradients, f, mode=mode)

def cge(gradients, f):
  return _distance("cge", gradients, f)

# ---------------------------------------------------------------------------- #
# The attacks' line search (attacks/identical.py:67-77, attacks/empire.py:51-59, tools/misc.py:468-513)

_SEARCH_RULES = dict(_RULE_CODES, krum=5, bulyan=6, brute=7, aksel=8, cge=9)      # BZ_RULE_*
_SEARCH_KINDS = {"identical": 0, "empire-strict": 1}                             # BZ_ATTACK_*

class LineSearch:
  """ A prepared `bz_line_search`: `line_maximize(eval_factor, evals)` of the identical-family attacks
  (kind "identical": candidate `grad_avg + s * grad_att`, s = -x when `negative`) or of empire-strict
  (kind "empire-strict": `grad_avg.mul(-x)`) against the rule `gar` with its defaults and f = f_decl,
  every evaluation, score and next factor computed on the device.  Like `Plan`, `search()` only issues
  the call (no allocation, no synchronisation; `graph()` captures it) and holds what it reads and writes:
      byz     the candidate row; after the call the attack's Byzantine gradient for the chosen factor
      record  fp64 [2 * evals + 2]: (x_k, y_k) per evaluation, the chosen factor, then the status word
  `result()` reads `record` once and returns (factor, trace), raising where the plain rule raises. """
  def __init__(self, gar, grad_honests, f_real, f_decl, grad_avg, grad_att, evals, negative=False, kind="identical"):
    if gar not in _SEARCH_RULES:
      raise KeyError(f"unknown aggregation rule {gar!r}")
    if kind not in _SEARCH_KINDS:
      raise ValueError(f"unknown attack kind {kind!r}, expected one of {sorted(_SEARCH_KINDS)}")
    honest = list(grad_honests)
    prep = _prepare(honest)
    if prep.to_cpu:
      raise ValueError("the line search takes CUDA tensors")
    if not all(g.is_contiguous() for g in honest):
      raise ValueError("the line search takes contiguous honest gradients")
    self.gar, self.evals, self.device = gar, int(evals), prep.device
    self.rows = honest
    self.vectors = [grad_avg] if grad_att is None else [grad_avg, grad_att]
    for vector in self.vectors:
      _check_like_rows(vector, prep, "grad_avg and grad_att")
    self.byz = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
    self._out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
    self.record = torch.empty(2 * max(self.evals, 0) + 2, dtype=torch.float64, device=prep.device)
    n = prep.n + int(f_real)
    self._ws = torch.empty(int(_lib.lib().bz_line_search_workspace_bytes(min(max(n, 1), _lib.MAX_N))), dtype=torch.uint8, device=prep.device)
    status = self.record.data_ptr() + 8 * (self.record.numel() - 1)
    self._fn = _lib.lib().bz_line_search
    self._args = (_SEARCH_RULES[gar], prep.ptrs, prep.n, int(f_real), int(f_decl), _SEARCH_KINDS[kind], int(bool(negative)),
                  grad_avg.data_ptr(), None if grad_att is None else grad_att.data_ptr(), prep.d, self.evals,
                  self.byz.data_ptr(), self._out.data_ptr(), self.record.data_ptr(), status,
                  self._ws.data_ptr(), self._ws.numel(), prep.stream)
    self._graph = None
  def __call__(self):
    """ Enqueue the search on the current stream of the rows' device. """
    with _on(self.device):
      _call(self._fn, self._args[:-1] + (torch.cuda.current_stream(self.device).cuda_stream,))
    return self.byz
  def graph(self):
    """ Capture the search in a CUDA graph; returns `replay`, which launches it and returns `byz`. """
    if self._graph is None:
      with _on(self.device):
        self()                                           # warm-up outside the capture
        torch.cuda.synchronize(self.device)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
          code = self._fn(*(self._args[:-1] + (torch.cuda.current_stream(self.device).cuda_stream,)))
        if code != 0:
          _lib.check(code, self._fn.__name__)
      self._graph = graph
    graph, byz = self._graph, self.byz
    def replay():
      graph.replay()
      return byz
    return replay
  def result(self):
    """ (factor, trace) from ONE device->host read: trace = [(x_k, y_k), ...].  With
    `config.strict_status`, a failed evaluation of Bulyan or brute raises what the plain call raises. """
    host = self.record.cpu()
    code = int(host[-1:].view(torch.int32)[0])
    if config.strict_status:
      _raise_status(code)
    values = host.tolist()
    return values[2 * self.evals], [(values[2 * k], values[2 * k + 1]) for k in range(self.evals)]

def line_search(gar, grad_honests, f_real, f_decl, grad_avg, grad_att, evals, negative=False, kind="identical"):
  """ The attacks' factor search on the device (see `LineSearch`).  Returns (factor, byz): the factor
  `tools.line_maximize` picks, a Python float, and the Byzantine gradient the attack returns for it, a
  device tensor (the reference returns it `f_real` times, aliased). """
  search = LineSearch(gar, grad_honests, f_real, f_decl, grad_avg, grad_att, evals, negative, kind)
  byz = search()
  factor, _ = search.result()
  return factor, byz

# ---------------------------------------------------------------------------- #
# Study metrics on the same stack (tools/pytorch.py:97-125, attack.py:846-848)

def avg_dev_max_async(samples):
  """ (avg, stats): the average of the rows and a DEVICE fp64 vector [2 + n]:
  stats[0] = ||avg||^2, stats[1] = max |avg|, stats[2 + i] = ||samples[i] - avg||^2.  No sync. """
  prep = _prepare_device(samples, "the study metrics take CUDA tensors (tools.compute_avg_dev_max handles CPU samples)")
  avg = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  stats = torch.empty(2 + prep.n, dtype=torch.float64, device=prep.device)
  ws = _workspace(prep.device, prep.stream)
  _run(prep.device, _lib.lib().bz_avg_dev_max, (prep.ptrs, prep.n, prep.d, avg.data_ptr(), stats.data_ptr(), ws.data_ptr(), ws.numel(), prep.stream))
  return avg, stats

class _Memo:
  """ One result of a computation `what` with parameters `params`, valid only for the very tensor
  OBJECTS it was computed on (held through weak references, compared with `is`, like `_CallCache`),
  at the same addresses and in-place versions: a freed list whose ids / addresses are reused by new
  tensors can never match, and a dead reference drops the entry. """
  def __init__(self):
    self.clear()
  def clear(self):
    self.what = self.params = self.refs = self.state = self.value = None
  @staticmethod
  def _state(tensors):
    return tuple((g.data_ptr(), g._version) for g in tensors)
  def store(self, what, params, tensors, value):
    try:
      refs = tuple(weakref.ref(g) for g in tensors)
    except TypeError:
      self.clear()
      return
    self.what, self.params, self.refs, self.state, self.value = what, params, refs, self._state(tensors), value
  def lookup(self, what, params, tensors):
    if self.refs is None or self.what != what or self.params != params or len(self.refs) != len(tensors):
      return None
    for ref, g in zip(self.refs, tensors):
      if ref() is not g:
        if ref() is None:
          self.clear()
        return None
    if self._state(tensors) != self.state:
      return None
    return self.value

# attack.py:846-847 asks for the sampled and for the honest gradients; without worker/server-side
# momentum and with nb_for_study = nb_honests those are the SAME tensors (`grad_honests =
# grad_sampleds[:nb_honests]`, attack.py:808): the second pass over n x d is saved.
_study_memo = _Memo()

def compute_avg_dev_max(samples):
  """ Drop-in for `tools.compute_avg_dev_max(samples)` (tools/pytorch.py:97-125): returns
  (average gradient or None, norm of the average, norm standard deviation, max |coordinate| of the
  average).  One device->host read of 2 + n doubles instead of the reference's n + 2 `.item()`s. """
  n = len(samples)
  if n == 0:
    return None, math.nan, math.nan, math.nan                 # :105-106
  hit = _study_memo.lookup("avg_dev_max", (), samples)
  if hit is not None:
    avg, a, b, c = hit
    return avg.clone(), a, b, c                               # callers own the average they get (grad_pasts keeps it)
  result = _compute_avg_dev_max(samples, n)
  _study_memo.store("avg_dev_max", (), samples, (result[0].clone(),) + result[1:])
  return result

def _compute_avg_dev_max(samples, n):
  avg, stats = avg_dev_max_async(samples)
  return _study_tuple(avg, stats.tolist(), n)                 # the only synchronisation

def _merge_ranks(parts, maxima):
  """ One host vector from the R ranks' fp64 partial vectors `parts` (rank order, equal lengths) —
  the rule of every sharded study scalar.  Entry k is ((p0[k] + p1[k]) + p2[k]) + ..., started from
  rank 0's value rather than from 0.0, so that one rank's vector comes back unchanged (0.0 + (-0.0)
  would turn a negative-zero dot product into +0.0); at the indices in `maxima` it is the largest
  value instead, NaN when any rank has a NaN (torch's max propagates it, Python's max() may drop it). """
  total = list(parts[0])
  for part in parts[1:]:
    for k, value in enumerate(part):
      if k not in maxima:
        total[k] += value
      elif math.isnan(value) or math.isnan(total[k]):
        total[k] = math.nan
      elif value > total[k]:
        total[k] = value
  return total

def fp32_overflow(sum_sq):
  """ +inf where an fp64 sum of squares rounds to +inf in fp32 (where ATen's fp32 `norm()` / `dot()`
  accumulator overflows), else the sum itself. """
  return math.inf if ctypes.c_float(sum_sq).value == math.inf else sum_sq

def fp32_norm(sum_sq):
  """ The fp32 `Tensor.norm()` of a vector from the fp64 sum of its squares (+inf on overflow). """
  return ctypes.c_float(math.sqrt(fp32_overflow(sum_sq))).value

def _study_tuple(avg, host, n):
  norm_avg = fp32_norm(host[0])                              # :110 returns an fp32 norm: same rounding in the logs
  norm_max = host[1]
  if n >= 2:
    norm_var = 0.
    for value in host[2:]:                                    # :116-120: same left-to-right sum of fp32 dot()s
      norm_var += fp32_overflow(value)
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
  _check_like_rows(center, prep, "center")
  out = torch.empty(prep.n, dtype=torch.float64, device=prep.device)
  ws = _workspace(prep.device, prep.stream)
  _run(prep.device, _lib.lib().bz_rowdots, (prep.ptrs, prep.n, center.data_ptr(), prep.d, out.data_ptr(), ws.data_ptr(), ws.numel(), prep.stream))
  return out

class StudyPartials:
  """ One shard's share of attack.py:846-866 (`study_partials`): the shard of the three averages
  (`attack_avg` is None without attack gradients), the list lengths `counts` = (ns, nh, na), the norms of
  the past gradients, and `vector`: ONE fp64 device vector of sums and maxima over the shard's columns,
      [0, 2 + ns)             K6 stats of the sampled gradients: ||avg||^2, max |avg|, ||g_i - avg||^2 per row
      then 2 + nh             the same for the honest gradients
      then 2 + na (na > 0)    the same for the attack gradients
      then 2 + a + P          <s_avg, x> for x in (h_avg, [a_avg], defense, the P pasts)   (a = 1 if na > 0 else 0)
      then a + 1              <h_avg, x> for x in ([a_avg], defense)
      then a + 1              <defense, x> for x in ([a_avg], defense)
      last                    max |defense| (0 for an empty shard: |x| >= 0, so 0 is no value)
  The length depends on (ns, nh, na, P) only, so every rank of a d-sharded step has the same layout.  The
  entries at `maxima()` merge across shards by max, every other one by addition. """
  __slots__ = ("sampled_avg", "honest_avg", "attack_avg", "vector", "counts", "past_norms")
  def maxima(self):
    ns, nh, na = self.counts
    return (1, 3 + ns) + ((5 + ns + nh,) if na else ()) + (self.vector.numel() - 1,)

def study_partials(grad_sampleds, grad_honests, grad_attacks, grad_defense, pasts, backend=None):
  """ The device half of `study_step` on one shard of the columns (the whole vectors on one GPU):
  K6 over each list (the honest pass is skipped when `grad_honests` holds the very same tensors as
  `grad_sampleds`, attack.py:808 without momentum placement; none without attack gradients), three
  `bz_rowdots` passes and the defense's max |x|, all into one device vector.  No sync.
  Args:
    grad_sampleds, grad_honests, grad_attacks, grad_defense  As `study_step`, or this rank's columns of them
    pasts    Iterable of (gradient or its shard, norm of the WHOLE gradient), most recent first
    backend  Provider of `avg_dev_max_async` and `rowdots_async` (default: this module)
  Returns:
    StudyPartials """
  avg_dev_max = avg_dev_max_async if backend is None else backend.avg_dev_max_async
  rowdots = rowdots_async if backend is None else backend.rowdots_async
  pasts = list(pasts)
  ns, nh, na = len(grad_sampleds), len(grad_honests), len(grad_attacks)
  s_avg, s_stats = avg_dev_max(grad_sampleds)
  same = nh == ns and all(a is b for a, b in zip(grad_sampleds, grad_honests))
  h_avg, h_stats = (s_avg, s_stats) if same else avg_dev_max(grad_honests)
  have_attack = na > 0
  a_avg, a_stats = avg_dev_max(grad_attacks) if have_attack else (None, s_stats[:0])
  # one vector against many, three times; every result lands in one device vector
  first = [h_avg] + ([a_avg] if have_attack else []) + [grad_defense] + [g for g, _ in pasts]
  second = ([a_avg] if have_attack else []) + [grad_defense]
  d_max = grad_defense.abs().max().double().reshape(1) if grad_defense.numel() else s_stats.new_zeros(1)
  out = StudyPartials()
  out.sampled_avg, out.honest_avg, out.attack_avg = s_avg, h_avg, a_avg
  out.vector = torch.cat([s_stats, h_stats, a_stats, rowdots(s_avg, first), rowdots(h_avg, second), rowdots(grad_defense, second), d_max])
  out.counts = (ns, nh, na)
  out.past_norms = [norm for _, norm in pasts]
  return out

def study_finish(partials, parts, momentum):
  """ The host half of `study_step`: the dict of attack.py:846-866 from the R shards' partial vectors.
  Every additive entry is summed across the shards in rank order in fp64, the maxima are merged
  (`_merge_ranks`), and only then come the fp32 overflow rule, the norms and the fp32 divisions — so
  every rank that holds the same R vectors returns bitwise the same scalars, and one shard gives
  exactly the one-GPU result.
  Args:
    partials  This shard's StudyPartials (its averages, list lengths and past norms)
    parts     R host sequences of floats, the shards' `vector`s in rank order (one: [vector.tolist()])
    momentum  args.momentum
  Returns:
    dict with the reference's variable names; the averages are this shard's """
  nan = math.nan
  ns, nh, na = partials.counts
  past_norms = partials.past_norms
  host = _merge_ranks(parts, partials.maxima())
  _, s_norm, s_dev, s_max = _study_tuple(None, host[:2 + ns], ns)
  _, h_norm, h_dev, h_max = _study_tuple(None, host[2 + ns:4 + ns + nh], nh)
  have_attack = na > 0
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
  past_dots = dots[k:k + len(past_norms)]; k += len(past_norms)
  ha = dots[k] if have_attack else nan; k += 1 if have_attack else 0
  hd = dots[k]; k += 1
  ad = dots[k] if have_attack else nan; k += 1 if have_attack else 0
  dd = dots[k]; k += 1
  d_max = dots[k]
  d_norm = fp32_norm(dd)                                  # Tensor.norm() is an fp32 value (attack.py:851)
  f32 = lambda x: ctypes.c_float(x).value                 # torch.dot(...).div_().div_().item(): fp32 arithmetic
  def div(a, b):                                          # IEEE division (a zero norm gives inf / nan, as div_ does)
    try:
      return f32(a / b)
    except ZeroDivisionError:
      return nan if a == 0 or math.isnan(a) else math.copysign(math.inf, a) * math.copysign(1., b)
  cos = lambda dot, na, nb: div(div(f32(dot), na), nb)
  out = dict(sampled_grad_avg=partials.sampled_avg, sampled_norm_avg=s_norm, sampled_norm_dev=s_dev, sampled_norm_max=s_max,
             honest_grad_avg=partials.honest_avg, honest_norm_avg=h_norm, honest_norm_dev=h_dev, honest_norm_max=h_max,
             attack_grad_avg=partials.attack_avg, attack_norm_avg=a_norm, attack_norm_dev=a_dev, attack_norm_max=a_max,
             defense_norm_avg=d_norm, defense_norm_max=f32(d_max),
             cosin_splhon=cos(sh, s_norm, h_norm), cosin_splatt=cos(sa, s_norm, a_norm) if have_attack else nan,
             cosin_spldef=cos(sd, s_norm, d_norm), cosin_honatt=cos(ha, h_norm, a_norm) if have_attack else nan,
             cosin_hondef=cos(hd, h_norm, d_norm), cosin_attdef=cos(ad, a_norm, d_norm) if have_attack else nan)
  if past_norms:
    out["cosin_sampled"] = cos(past_dots[0], s_norm, past_norms[0])
    out["curv_sampled"] = momentum * sum((momentum ** i) * f32(dot) for i, dot in enumerate(past_dots))
  else:
    out["cosin_sampled"] = nan
    out["curv_sampled"] = nan
  return out

def study_step(grad_sampleds, grad_honests, grad_attacks, grad_defense, pasts, momentum):
  """ Everything attack.py:846-866 computes for one line of the study file, on the device:
    * the three `tools.compute_avg_dev_max` calls (K6, one pass each; a repeated list is computed once),
    * the norm and the largest |coordinate| of the defense gradient,
    * the six cosines between the sampled / honest / attack averages and the defense gradient,
    * the cosine with the last past gradient and the curvature sum over all past gradients
  with THREE passes of `bz_rowdots` (one vector against many) instead of 7 + len(pasts) `torch.dot(...).item()`
  and ONE device->host read for the whole step (the reference: 9 + len(samples) + len(pasts) `.item()`s).
  `study_partials` + `study_finish` over one shard; `sharded.study_step` is the d-sharded form.
  Args:
    grad_sampleds, grad_honests, grad_attacks  Lists of CUDA gradients (the attack list may be empty)
    grad_defense  The aggregated gradient
    pasts         Iterable of (gradient, norm) of the past sampled averages, most recent first
    momentum      args.momentum
  Returns:
    dict with the reference's variable names (attack.py:846-866) """
  partials = study_partials(grad_sampleds, grad_honests, grad_attacks, grad_defense, pasts)
  return study_finish(partials, [partials.vector.tolist()], momentum)            # the only synchronisation

# ---------------------------------------------------------------------------- #
# Phases of the d-sharded multi-GPU path (device tensors only)

def _prepare_device(gradients, message="the sharded phases take CUDA tensors"):
  prep = _prepare(gradients)
  if prep.to_cpu:
    raise ValueError(message)
  return prep

def _partial_call(prep, pair, center, part, ws):
  """ (fn, args) of phase A: this shard's share of the squared pairwise distances (`pair`), or of the
  squared distances of the rows to the address `center` (None: the origin), written to `part`. """
  lib = _lib.lib()
  if pair:
    return lib.bz_pairdist_partial, (prep.ptrs, prep.n, prep.d, part, ws.data_ptr(), ws.numel(), prep.stream)
  return lib.bz_rowdist_partial, (prep.ptrs, prep.n, center, prep.d, part, ws.data_ptr(), ws.numel(), prep.stream)

def _partial(gradients, pair, center, out):
  prep = _prepare_device(gradients)
  if center is not None:
    _check_like_rows(center, prep, "center")
    center = center.data_ptr()
  if out is None:
    out = torch.empty((prep.n, prep.n) if pair else prep.n, dtype=torch.float64, device=prep.device)
  _run(prep.device, *_partial_call(prep, pair, center, out.data_ptr(), _workspace(prep.device, prep.stream)))
  return out

def pairdist_partial(gradients, out=None):
  """ [n, n] fp64: this shard's share of the squared pairwise distances (entries i < j); written
  into `out` when given (e.g. this rank's slot of a symmetric buffer). """
  return _partial(gradients, True, None, out)

def rowdist_partial(gradients, center=None, out=None):
  """ [n] fp64: this shard's share of the squared distance of every row to `center` (None: origin);
  written into `out` when given. """
  return _partial(gradients, False, center, out)

def _select_call(rule, blocks, meta, stream):
  """ (fn, args) of phase B writing the order (and status word) to the address `meta`: `bz_<rule>_select`
  on the gathered blocks (a [R, ...] fp64 CUDA tensor), or `bz_<rule>_select_peers` on a list of R
  device addresses of the ranks' blocks (rank order, mapped over NVLink: read in place). """
  if isinstance(blocks, torch.Tensor):
    if blocks.dtype != torch.float64 or not blocks.is_contiguous() or blocks.device.type != "cuda":
      raise ValueError("parts must be a contiguous float64 CUDA tensor")
    suffix, nparts, table = "", blocks.shape[0], blocks.data_ptr()
  else:
    if not 1 <= len(blocks) <= _lib.MAX_PEERS:
      raise ValueError(f"{len(blocks)} peers, expected 1..{_lib.MAX_PEERS}")
    suffix, nparts, table = "_peers", len(blocks), (ctypes.c_void_p * len(blocks))(*[int(p) for p in blocks])
  status = (meta + 4 * rule.n,) if rule.status else ()
  fn = getattr(_lib.lib(), "bz_" + rule.select + "_select" + suffix)
  return fn, (table, nparts, rule.n) + rule.select_params + (meta,) + status + (stream,)

def select(gar, blocks, n, f, m=None, device=None):
  """ Phase B of a distance-based rule from the R partial blocks, `blocks` as in `_select_call`
  (peer addresses: the selection goes to `device`).  Returns the selection at the rule's length (a
  device int32 tensor), with the status word for bulyan and brute. """
  rule = _rule(gar, n, f, m)
  if isinstance(blocks, torch.Tensor):
    device = blocks.device
  meta = torch.empty(n + 1, dtype=torch.int32, device=device)
  _run(device, *_select_call(rule, blocks, meta.data_ptr(), torch.cuda.current_stream(device).cuda_stream))
  return (meta[:rule.length], meta[n:]) if rule.status else meta[:n]

def krum_select(parts, n, f):
  return select("krum", parts, n, f)

def bulyan_select(parts, n, f, m):
  return select("bulyan", parts, n, f, m)

def brute_select(parts, n, f):
  return select("brute", parts, n, f)

def rowdist_select(parts, n, sqrt_norm):
  return select("cge" if sqrt_norm else "aksel", parts, n, 0)     # the order of the row distances: f plays no part

def krum_select_peers(peer_ptrs, n, f, device):
  return select("krum", peer_ptrs, n, f, device=device)

def bulyan_select_peers(peer_ptrs, n, f, m, device):
  return select("bulyan", peer_ptrs, n, f, m, device=device)

def brute_select_peers(peer_ptrs, n, f, device):
  return select("brute", peer_ptrs, n, f, device=device)

def rowdist_select_peers(peer_ptrs, n, sqrt_norm, device):
  return select("cge" if sqrt_norm else "aksel", peer_ptrs, n, 0, device=device)

def _average_call(prep, selection, count, zero_init, divisor, status, out):
  return _lib.lib().bz_average_selected, (prep.ptrs, prep.n, selection, int(count), 1 if zero_init else 0, float(divisor), status, prep.d, out, prep.stream)

def _reduce_call(prep, rule, selection, status, out):
  """ (fn, args) of phase C: the rule's reduce of the local shard over the selection, all addresses. """
  if rule.gar == "bulyan":
    return _lib.lib().bz_bulyan_reduce, (prep.ptrs, prep.n, rule.f, rule.m, selection, status, prep.d, out, prep.stream)
  return _average_call(prep, selection, rule.count, rule.zero_init, rule.count, status if rule.status else None, out)

def _ptr(tensor):
  return None if tensor is None else tensor.data_ptr()

def average_selected(gradients, selection, count, zero_init=True, divisor=None, status=None):
  """ Ordered-subset average of the local shard; `selection` is a device int32 tensor or None. """
  prep = _prepare_device(gradients)
  out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  _run(prep.device, *_average_call(prep, _ptr(selection), count, zero_init, count if divisor is None else divisor, _ptr(status), out.data_ptr()))
  return out

def bulyan_reduce(gradients, f, m, order, status=None):
  prep = _prepare_device(gradients)
  out = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
  _run(prep.device, *_reduce_call(prep, _rule("bulyan", prep.n, f, m), order.data_ptr(), _ptr(status), out.data_ptr()))
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
    self._sampled = _row_buffer(n, d, self.device)
    self._pitch = self._sampled.stride(0)
    self._honest = None
    self._lib = _lib.lib()
  def _honest_buffer(self):
    if self._honest is None:
      self._honest = _row_buffer(self.n, self.d, self.device)
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
    _run(self.device, self._lib.bz_gradient_row, (grad.data_ptr(), self.d, float(clip) if clip is not None else 0., row.data_ptr(), mode,
                                                  _ptr(mom), float(mu), 1. - float(dampening), _ptr(honest), ws.data_ptr(), ws.numel(), stream))
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

def gradient_scatter(grad, clip, slots):
  """ `bz_gradient_scatter`: clip `grad` as `GradientStack.push` does (clip None or <= 0: no clipping)
  and write columns [lo_r, hi_r) of the result into `slots[r]` (`sharded.shard_bounds` over R =
  len(slots) ranks), in one pass.  The slots are contiguous fp32 CUDA vectors of hi_r - lo_r
  elements, 16-byte aligned, addressable from `grad`'s GPU: its own memory or another GPU's mapped into
  it (symmetric memory).  Their version counters are not bumped here, that is for the rank that owns
  them to do. """
  d, R = grad.numel(), len(slots)
  if not 1 <= R <= _lib.MAX_PEERS:
    raise ValueError(f"{R} slots, expected 1..{_lib.MAX_PEERS}")
  per = (d + R - 1) // R
  ptrs = []
  for r, slot in enumerate(slots):
    lo = min(d, r * per)
    width = min(d, lo + per) - lo
    if slot.dtype != torch.float32 or slot.numel() != width or not slot.is_contiguous() or slot.device.type != "cuda":
      raise ValueError(f"slot {r} must be a contiguous float32 CUDA vector of the {width} columns of rank {r}")
    ptrs.append(slot.data_ptr() if slot.numel() else None)
  if grad.dtype != torch.float32 or grad.dim() != 1 or not grad.is_contiguous() or grad.device.type != "cuda":
    raise ValueError("grad must be a contiguous float32 CUDA vector")
  stream = torch.cuda.current_stream(grad.device).cuda_stream
  ws = _workspace(grad.device, stream)
  _run(grad.device, _lib.lib().bz_gradient_scatter, (grad.data_ptr(), d, float(clip) if clip is not None else 0., R,
                                                     (ctypes.c_void_p * R)(*ptrs), ws.data_ptr(), ws.numel(), stream))

def momentum_rows(rows, mu, dampening, momentums=None, server=None, honests=None):
  """ The momentum placement of attack.py:799-810 on rows that are already clipped, one launch per 64
  rows (`bz_gradient_momentum`): the arithmetic `GradientStack.push` applies after the clip, so the
  results have the same bits.
    momentums given       worker side: momentums[k] <- momentums[k] * mu + (1 - dampening) * rows[k],
                          in place (:802); distinct vectors, one per row
    server and honests    server side: honests[k] <- rows[k] * (1 - dampening) + mu * server (:807)
  Every vector is a contiguous fp32 CUDA vector of the rows' length, all on one GPU; rows of zero
  columns (an empty shard) are a no-op.  Bumps the version counter of what it writes.
  Returns the honest rows (`momentums` on the worker side). """
  rows = list(rows)
  worker = momentums is not None
  if worker == (server is not None or honests is not None):
    raise ValueError("give either momentums (worker side) or server and honests (server side)")
  if not worker and (server is None or honests is None):
    raise ValueError("the server side needs both server and honests")
  outs = list(momentums if worker else honests)
  if len(outs) != len(rows) or not rows:
    raise ValueError(f"{len(outs)} output vectors for {len(rows)} rows")
  shape, device = rows[0].shape, rows[0].device
  for what, vs in (("row", rows), ("momentum" if worker else "honest", outs), ("server", [] if worker else [server])):
    for v in vs:
      if v.dtype != torch.float32 or v.dim() != 1 or v.shape != shape or not v.is_contiguous() or v.device != device or device.type != "cuda":
        raise ValueError(f"every {what} must be a contiguous float32 CUDA vector like the first row")
  if shape[0] == 0:
    return outs                                    # an empty tensor's address may be 0: nothing to launch
  lib, table = _lib.lib(), ctypes.c_void_p * _lib.MAX_N
  stream = torch.cuda.current_stream(device).cuda_stream
  for k in range(0, len(rows), _lib.MAX_N):
    part = slice(k, k + _lib.MAX_N)
    ptrs = table(*[r.data_ptr() for r in rows[part]])
    written = table(*[o.data_ptr() for o in outs[part]])
    _run(device, lib.bz_gradient_momentum, (ptrs, len(rows[part]), shape[0], 1 if worker else 2, written if worker else None,
                                            None if worker else server.data_ptr(), float(mu), 1. - float(dampening),
                                            None if worker else written, stream))
  for o in outs:
    torch.autograd.graph.increment_version(o)
  return outs

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
    n, d = prep.n, prep.d
    self.gar, self.n, self.d, self.device = gar, n, d, prep.device
    self.rows = list(gradients)
    if not all(g.is_contiguous() for g in self.rows):
      # a packed copy would neither stay alive nor follow in-place updates of the originals
      raise ValueError("Plan takes contiguous rows (the plain call accepts strided views and packs them)")
    self.out = torch.empty(d, dtype=torch.float32, device=prep.device) if out is None else out
    _check_like_rows(self.out, prep, "out")
    self.selection = None
    self.status = None
    if gar in _RULE_CODES:
      fn, args = _coordinate_call(gar, prep, f, self.out.data_ptr())
    else:
      rule = _rule(gar, n, f, m, mode)
      self._ws = _workspace(prep.device, prep.stream)
      self._meta = torch.empty(n + 1, dtype=torch.int32, device=prep.device)
      self.selection = self._meta[:rule.length]
      if rule.status:
        self.status = self._meta[n:]
      fn, args = rule.entry(prep.ptrs, d, self.out.data_ptr(), self._meta.data_ptr(), self._ws, prep.stream)
    self._fn, self._args = fn, args
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
        if code != 0:                                    # raised after the capture has ended
          _lib.check(code, self._fn.__name__)
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
      _lib.check(code, self._fn.__name__)
    return self.out
