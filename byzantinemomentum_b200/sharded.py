# coding: utf-8
"""d-sharded aggregation across GPUs (one process per GPU, `torch.distributed`).

Rank r holds the columns of its shard of every worker gradient — a list of n fp32 vectors of
length d_r — and produces the matching shard of the aggregated gradient (SURVEY.md §8(e)).

  * average / median / trmean / phocas / meamed are coordinate-wise: NO collective.
  * krum / bulyan / brute / aksel / cge select whole rows from global distances: each rank
    computes the fp64 partial sums of squares over its shard (phase A), ONE all-gather
    exchanges the R small blocks (n*n or n doubles per rank: 5 KB at n = 25), every rank sums
    them in rank order — bitwise the same result everywhere, so every rank derives the
    identical selection (phase B) — and reduces its own shard with it (phase C).
    An all-reduce would leave the summation order to the collective; all-gather + fixed
    order does not.

The reference has no distributed path at all (SURVEY.md §2 #28); this module is the new
multi-GPU form of its `aggregate(gradients, f, ...)`.

`backend` is the object providing the phases; it defaults to `byzantinemomentum_b200.engine`
(the CUDA library).  The CPU tests inject a NumPy stand-in to exercise this host logic under
`gloo` with world_size 2; there is no fallback: with the default backend and no GPU the
phases raise.
"""

import math

import torch
import torch.distributed as dist

from . import _lib
from . import engine as _engine

__all__ = ["aggregate", "aggregate_p2p", "compute_avg_dev_max", "replicate", "apply_update", "shard_bounds", "rows_aligned", "choose_exchange", "PeerExchange", "FusedExchange", "ShardedPlan", "COORDINATE_WISE", "DISTANCE_BASED"]

COORDINATE_WISE = ("average", "median", "trmean", "phocas", "meamed")
DISTANCE_BASED = ("krum", "bulyan", "brute", "aksel", "cge")

def _gather(part, group):
  """ All-gather one small fp64 block per rank -> [R, *part.shape], rank order. """
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  if world == 1:
    return part.unsqueeze(0).contiguous()
  gathered = torch.empty((world,) + tuple(part.shape), dtype=part.dtype, device=part.device)
  dist.all_gather([gathered[r] for r in range(world)], part.contiguous(), group=group)
  return gathered

class PeerExchange:
  """ Exchange of the partial blocks through NVLink peer memory instead of a collective.

  Every rank owns two slots of n*n doubles in a SYMMETRIC buffer (torch symmetric memory: the
  same allocation mapped into every rank's address space over NVLink/NVSwitch).  A step writes
  its block into slot `step % 2` (phase A writes there directly), crosses ONE device-side
  barrier, and the selection kernel then reads the R blocks in place from the R ranks
  (`bz_*_select_peers`): gather and scoring are one kernel.  Two slots make one barrier per
  step enough: a rank can only reach the barrier of step t+1 after its reads of step t, so by
  the time slot t%2 is rewritten (step t+2) every peer has finished reading it.
  Needs CUDA peer access between the ranks' GPUs (one NVSwitch domain) and <= 16 ranks. """
  def __init__(self, n, device, group=None):
    import torch.distributed._symmetric_memory as symm_mem
    self.n = n
    self.device = device
    self.group = group if group is not None else dist.group.WORLD
    self.world = dist.get_world_size(self.group)
    self.buffer = symm_mem.empty(2 * n * n, dtype=torch.float64, device=device)
    self.handle = symm_mem.rendezvous(self.buffer, self.group)
    self.peer_base = [int(p) for p in self.handle.buffer_ptrs]
    self.step = 0
  def slot(self):
    """ (this rank's slot as a tensor, the R peers' addresses of the same slot) for this step. """
    off = (self.step % 2) * self.n * self.n
    mine = self.buffer[off:off + self.n * self.n]
    return mine, [base + off * 8 for base in self.peer_base]
  def publish(self):
    """ Order every rank's phase-A writes before anyone's reads (stream-ordered device barrier). """
    self.handle.barrier(channel=0)
    self.step += 1

_exchanges = {}

def peer_exchange(n, device, group=None):
  key = (n, device.index, id(group))
  ex = _exchanges.get(key)
  if ex is None:
    ex = _exchanges[key] = PeerExchange(n, device, group)
  return ex

class FusedExchange:
  """ Symmetric buffer for the exchange that runs INSIDE the distance pass (`bz_krum_peers`,
  `bz_bulyan_peers`): per rank two slots of n*n doubles plus, per slot, a flag array of 16 words.  The
  last CTA of each rank's distance pass writes its block into its slot, raises its flag on every GPU,
  waits for the R flags, and adds the R blocks in place over NVLink — no barrier op, no collective, no
  separate selection kernel.  `epoch` (the step number) tells this step's flags from older ones; two
  slots make that enough (a rank rewrites slot s only after every peer has signalled the step in
  between, i.e. finished reading s). """
  FLAG_WORDS = 16
  def __init__(self, n, device, group=None):
    import torch.distributed._symmetric_memory as symm_mem
    self.n, self.device = n, device
    self.group = group if group is not None else dist.group.WORLD
    self.world = dist.get_world_size(self.group)
    self.rank = dist.get_rank(self.group)
    words = 2 * n * n + 2 * self.FLAG_WORDS // 2             # doubles; the flags are uint32 pairs in the tail
    self.buffer = symm_mem.empty(words, dtype=torch.float64, device=device)
    self.buffer.zero_()
    self.handle = symm_mem.rendezvous(self.buffer, self.group)
    torch.cuda.synchronize(device)
    self.handle.barrier(channel=0)                           # every rank's flags are zero before anyone signals
    torch.cuda.synchronize(device)
    self.peer_base = [int(p) for p in self.handle.buffer_ptrs]
    self.epoch = 0
  def tables(self, slot):
    """ (ctypes array of the R block pointers, ctypes array of the R flag-array pointers) of a slot. """
    import ctypes
    block = slot * self.n * self.n * 8
    flags = 2 * self.n * self.n * 8 + slot * self.FLAG_WORDS * 4
    return ((ctypes.c_void_p * self.world)(*[b + block for b in self.peer_base]),
            (ctypes.c_void_p * self.world)(*[b + flags for b in self.peer_base]))

_fused = {}

def fused_exchange(n, device, group=None):
  key = (n, device.index, id(group))
  ex = _fused.get(key)
  if ex is None:
    ex = _fused[key] = FusedExchange(n, device, group)
  return ex

def rows_aligned(rows):
  """ Whether the ring kernel takes these rows: every non-empty row 16-byte aligned (an empty shard
  reads nothing). """
  return all(g.numel() == 0 or g.data_ptr() % 16 == 0 for g in rows)

def _symmetric_memory_importable():
  try:
    import torch.distributed._symmetric_memory  # noqa: F401
  except Exception:
    return False
  return True

EXCHANGES = ("auto", "fused", "p2p", "nccl")

def choose_exchange(gar, exchange, aligned, symmetric, group=None):
  """ The exchange of `ShardedPlan`, the same on every rank of `group`.  The two ranks' protocols do
  not mix (different symmetric buffers, flags nobody raises), so the local facts — `aligned`: this
  rank's rows are 16-byte aligned; `symmetric`: symmetric memory can be set up here — are agreed on
  with one all-reduce (MIN) before the choice: a shard that starts mid-vector on one rank moves every
  rank to "p2p".  An explicit request that some rank cannot serve raises on every rank.
  Returns "fused", "p2p" or "nccl". """
  if exchange not in EXCHANGES:
    raise ValueError(f"unknown exchange {exchange!r}")
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  facts = [int(bool(aligned)), int(bool(symmetric))]
  if world > 1:
    device = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")
    agreed = torch.tensor(facts, dtype=torch.int32, device=device)
    dist.all_reduce(agreed, op=dist.ReduceOp.MIN, group=group)
    facts = agreed.tolist()
  aligned, symmetric = bool(facts[0]), bool(facts[1])
  fusable = gar in ("krum", "bulyan") and aligned
  if exchange == "auto":
    if world == 1 or world > _lib.MAX_PEERS or not symmetric:
      return "nccl"
    return "fused" if fusable else "p2p"
  if exchange == "fused" and not (fusable and symmetric and world <= _lib.MAX_PEERS):
    raise ValueError(f"the fused exchange serves krum / bulyan on 16-byte aligned rows, with symmetric memory, on every one of at most {_lib.MAX_PEERS} ranks")
  if exchange == "p2p" and not symmetric:
    raise ValueError("the p2p exchange needs symmetric memory on every rank")
  return exchange

def aggregate_p2p(gar, gradients, f=None, m=None, mode="mid", group=None, return_selection=False):
  """ `aggregate` for the distance-based rules with the exchange fused into the selection kernel
  (peer memory over NVLink, see PeerExchange).  CUDA engine only. """
  be = _engine
  n = len(gradients)
  if gar in COORDINATE_WISE:
    return aggregate(gar, gradients, f=f, m=m, mode=mode, group=group, return_selection=return_selection)
  device = gradients[0].device
  ex = peer_exchange(n, device, group)
  mine, peers = ex.slot()
  if gar in ("krum", "bulyan", "brute"):
    be.pairdist_partial_into(gradients, mine)
    ex.publish()
    if gar == "krum":
      m = n - f - 2 if m is None else m
      sel = be.krum_select_peers(peers, n, f, device)
      out = be.average_selected(gradients, sel, m)
    elif gar == "bulyan":
      m = n - f - 2 if m is None else m
      sel, status = be.bulyan_select_peers(peers, n, f, m, device)
      out = be.bulyan_reduce(gradients, f, m, sel, status)
    else:
      sel, status = be.brute_select_peers(peers, n, f, device)
      out = be.average_selected(gradients, sel, n - f, status=status)
  elif gar == "aksel":
    count = (n + 1) // 2 if mode == "mid" else n - f
    center = be.median(gradients)
    be.rowdist_partial_into(gradients, center, mine[:n])
    ex.publish()
    sel = be.rowdist_select_peers(peers, n, False, device)
    out = be.average_selected(gradients, sel, count)
  elif gar == "cge":
    be.rowdist_partial_into(gradients, None, mine[:n])
    ex.publish()
    sel = be.rowdist_select_peers(peers, n, True, device)
    out = be.average_selected(gradients, sel, n - f, zero_init=False)
  else:
    raise KeyError(f"unknown aggregation rule {gar!r}")
  return (out, sel) if return_selection else out

class ShardedPlan:
  """ Prepared d-sharded aggregation (the multi-GPU counterpart of `engine.Plan`): every argument
  of the three phases is resolved once — row pointers, this rank's partial block, the gathered
  [R, n, n] buffer (or the peers' addresses of the symmetric slots), selection, output, workspace —
  so that a step is 3 C-ABI calls plus ONE exchange, with no allocation and no host/device
  synchronisation.  The rows and the output are held; their CONTENT may change between calls.

      plan = sharded.ShardedPlan("krum", shard_rows, f=5)          # exchange="auto": peer memory when available
      out_shard = plan()                                            # plan.out, plan.selection (device int32)

  exchange: "nccl"  one `all_gather_into_tensor` of the R blocks (n*n*8 B each), then the selection
                    kernel sums them in rank order;
            "p2p"   the block is written straight into this rank's slot of a SYMMETRIC buffer, one
                    device-side barrier, and the selection kernel reads the R blocks in place from
                    the R peers over NVLink (`bz_*_select_peers`): gather + scoring in one kernel;
            "fused" (krum, bulyan) the exchange runs INSIDE the distance pass: its last CTA publishes the
                    block in the symmetric buffer, flags the peers, waits for theirs and scores — a step
                    is the single-GPU rule's two launches, nothing else (`bz_krum_peers`);
            "auto"  "fused" where it applies on every rank, else "p2p", when every rank of the group
                    has symmetric memory; else "nccl".  The ranks agree on the choice
                    (`choose_exchange`); a failing symmetric-memory setup raises.
  Both exchanges use the same fixed summation order: bitwise identical selections on every rank.
  Coordinate-wise rules need no exchange and simply wrap `engine.Plan`. """
  def __init__(self, gar, gradients, f=None, m=None, mode="mid", group=None, exchange="auto"):
    import ctypes
    from . import _lib
    self.gar, self.group = gar, group
    self.rows = list(gradients)
    n = self.n = len(self.rows)
    self.world = dist.get_world_size(group) if dist.is_initialized() else 1
    self.selection = None
    self.status = None
    if gar in COORDINATE_WISE:
      self._local = _engine.Plan(gar, self.rows, f=f)
      self.out = self._local.out
      self.exchange = "none"
      return
    if gar not in DISTANCE_BASED:
      raise KeyError(f"unknown aggregation rule {gar!r}")
    self._local = None
    lib = _lib.lib()
    prep = _engine._prepare_device(self.rows)
    if not all(g.is_contiguous() for g in self.rows):
      raise ValueError("ShardedPlan takes contiguous rows")
    device = self.device = prep.device
    d = self.d = prep.d
    self._ptrs = (ctypes.c_void_p * n)(*[g.data_ptr() for g in self.rows])
    self._stream = prep.stream
    self._ws = _engine._workspace(device, prep.stream)
    ws, wn, st = self._ws.data_ptr(), self._ws.numel(), self._stream
    self.out = torch.empty(d, dtype=torch.float32, device=device)
    self._meta = torch.empty(n + 1, dtype=torch.int32, device=device)
    meta, status = self._meta.data_ptr(), self._meta[n:].data_ptr()
    self.selection = self._meta[:n]
    o = self.out.data_ptr()
    pair = gar in ("krum", "bulyan", "brute")
    width = n * n if pair else n
    # ---- exchange: one choice for the whole group ------------------------------------------------
    exchange = choose_exchange(gar, exchange, rows_aligned(self.rows), _symmetric_memory_importable(), group)
    if exchange == "fused":
      self._fx = fused_exchange(n, device, group)
    elif exchange == "p2p":
      self._ex = peer_exchange(n, device, group)
    self.exchange = exchange
    if exchange == "fused":
      fx = self._fx
      mm = n - f - 2 if m is None else m
      self.status = self._meta[n:]
      fn = lib.bz_krum_peers if gar == "krum" else lib.bz_bulyan_peers
      self._fused_fn = fn
      self._fused_tables = [fx.tables(0), fx.tables(1)]
      self._fused_head = (self._ptrs, n, int(f), int(mm), d, o, meta, status, fx.rank, fx.world)
      self._fused_tail = (ws, wn, st)
      self._check = _lib.check
      self._pre = None
      return
    if exchange == "p2p":
      ex = self._ex
      # two slots -> two prepared argument sets; the step counter of the exchange picks one
      self._slots = []
      for slot in range(2):
        off = slot * n * n
        mine = ex.buffer[off:off + width]
        table = (ctypes.c_void_p * self.world)(*[base + off * 8 for base in ex.peer_base])
        self._slots.append((mine, table))
    else:
      self._part = torch.empty(width, dtype=torch.float64, device=device)
      self._gathered = torch.empty((self.world, width), dtype=torch.float64, device=device)
    # ---- phases ---------------------------------------------------------------------------------
    if gar == "aksel":
      self._center = torch.empty(d, dtype=torch.float32, device=device)
      self._pre = (lib.bz_median, (self._ptrs, n, d, self._center.data_ptr(), st))
      center = self._center.data_ptr()
    else:
      self._pre = None
      center = None
    def phase_a(part_ptr):
      if pair:
        return lib.bz_pairdist_partial, (self._ptrs, n, d, part_ptr, ws, wn, st)
      return lib.bz_rowdist_partial, (self._ptrs, n, center, d, part_ptr, ws, wn, st)
    def phase_b(parts_ptr, peers):
      R = self.world
      if gar == "krum":
        return (lib.bz_krum_select_peers if peers else lib.bz_krum_select), (parts_ptr, R, n, int(f), meta, st)
      if gar == "bulyan":
        return (lib.bz_bulyan_select_peers if peers else lib.bz_bulyan_select), (parts_ptr, R, n, int(f), int(mm), meta, status, st)
      if gar == "brute":
        return (lib.bz_brute_select_peers if peers else lib.bz_brute_select), (parts_ptr, R, n, int(f), meta, status, st)
      return (lib.bz_rowdist_select_peers if peers else lib.bz_rowdist_select), (parts_ptr, R, n, 1 if gar == "cge" else 0, meta, st)
    mm = (n - f - 2 if m is None else m) if gar in ("krum", "bulyan") else None
    if gar == "krum":
      self._c = (lib.bz_average_selected, (self._ptrs, n, meta, int(mm), 1, float(mm), None, d, o, st))
    elif gar == "bulyan":
      self.status = self._meta[n:]
      self._c = (lib.bz_bulyan_reduce, (self._ptrs, n, int(f), int(mm), meta, status, d, o, st))
    elif gar == "brute":
      self.status = self._meta[n:]
      self.selection = self._meta[:n - int(f)]
      self._c = (lib.bz_average_selected, (self._ptrs, n, meta, n - int(f), 1, float(n - int(f)), status, d, o, st))
    elif gar == "aksel":
      if mode not in _lib.AKSEL_MODES:
        raise NotImplementedError(mode)
      count = (n + 1) // 2 if mode == "mid" else n - int(f)
      self._c = (lib.bz_average_selected, (self._ptrs, n, meta, count, 1, float(count), None, d, o, st))
    else:  # cge
      count = n - int(f)
      self._c = (lib.bz_average_selected, (self._ptrs, n, meta, count, 0, float(count), None, d, o, st))
    if exchange == "p2p":
      self._ab = [(phase_a(mine.data_ptr()), phase_b(table, True)) for mine, table in self._slots]
    else:
      self._ab = [(phase_a(self._part.data_ptr()), phase_b(self._gathered.data_ptr(), False))]
    self._check = _lib.check
  def __call__(self):
    if self._local is not None:
      return self._local()
    check = self._check
    if self.exchange == "fused":
      fx = self._fx
      fx.epoch += 1
      blocks, flags = self._fused_tables[fx.epoch % 2]
      with _engine._on(self.device):
        check(self._fused_fn(*self._fused_head, blocks, flags, fx.epoch, *self._fused_tail), "bz_*_peers")
      return self.out
    with _engine._on(self.device):
      if self._pre is not None:
        check(self._pre[0](*self._pre[1]), "bz_median")
      if self.exchange == "p2p":
        ex = self._ex
        (fa, aa), (fb, ab) = self._ab[ex.step % 2]
        check(fa(*aa), "phase A")
        ex.publish()
      else:
        (fa, aa), (fb, ab) = self._ab[0]
        check(fa(*aa), "phase A")
        if self.world > 1:
          dist.all_gather_into_tensor(self._gathered, self._part, group=self.group)
        else:
          self._gathered.copy_(self._part.unsqueeze(0))
      check(fb(*ab), "phase B")
      check(self._c[0](*self._c[1]), "phase C")
    return self.out

def aggregate(gar, gradients, f=None, m=None, mode="mid", group=None, backend=None, return_selection=False):
  """ Aggregate this rank's shard.
  Args:
    gar        Rule name (one of COORDINATE_WISE + DISTANCE_BASED)
    gradients  List of n fp32 CUDA vectors: this rank's columns of the n worker gradients
    f          Number of Byzantine gradients to tolerate (ignored by average / median)
    m          Multi-Krum selection size (krum / bulyan; default n - f - 2)
    mode       Aksel mode ("mid" or "n-f")
    group      Process group (default: the world)
    backend    Provider of the phases (default: the CUDA engine)
  Returns:
    This rank's shard of the aggregated gradient (and the device-side selection if asked)
  """
  be = backend or _engine
  n = len(gradients)
  if gar in COORDINATE_WISE:
    if gar == "average":
      out = be.average(gradients)
    elif gar == "median":
      out = be.median(gradients)
    else:
      out = getattr(be, gar)(gradients, f)
    return (out, None) if return_selection else out
  if gar == "krum":
    m = n - f - 2 if m is None else m
    parts = _gather(be.pairdist_partial(gradients), group)
    order = be.krum_select(parts, n, f)
    out = be.average_selected(gradients, order, m)
    sel = order
  elif gar == "bulyan":
    m = n - f - 2 if m is None else m
    parts = _gather(be.pairdist_partial(gradients), group)
    order, status = be.bulyan_select(parts, n, f, m)
    out = be.bulyan_reduce(gradients, f, m, order, status)
    sel = order
  elif gar == "brute":
    parts = _gather(be.pairdist_partial(gradients), group)
    sel, status = be.brute_select(parts, n, f)
    out = be.average_selected(gradients, sel, n - f, status=status)
  elif gar == "aksel":
    count = (n + 1) // 2 if mode == "mid" else n - f
    center = be.median(gradients)                                   # coordinate-wise: local
    parts = _gather(be.rowdist_partial(gradients, center), group)
    sel = be.rowdist_select(parts, n, False)
    out = be.average_selected(gradients, sel, count)
  elif gar == "cge":
    count = n - f
    parts = _gather(be.rowdist_partial(gradients, None), group)
    sel = be.rowdist_select(parts, n, True)
    out = be.average_selected(gradients, sel, count, zero_init=False)
  else:
    raise KeyError(f"unknown aggregation rule {gar!r}")
  return (out, sel) if return_selection else out

def compute_avg_dev_max(samples, group=None, backend=None):
  """ `tools.compute_avg_dev_max` (tools/pytorch.py:97-125) over d-sharded samples: every rank
  passes its columns of the n samples and gets its shard of the average plus the GLOBAL scalars.
  One pass over the local shard (`avg_dev_max_async`), then ONE all-gather of 2 + n doubles; the
  sums of squares are added in rank order and the maxima compared, so every rank returns
  bitwise the same three numbers.
  Returns:
    (this rank's shard of the average or None, norm of the average, norm standard deviation,
     max |coordinate| of the average)
  """
  be = backend or _engine
  n = len(samples)
  if n == 0:
    return None, math.nan, math.nan, math.nan
  avg, stats = be.avg_dev_max_async(samples)
  gathered = _gather(stats, group).tolist()            # [R][2 + n]; the only synchronisation
  norm_sq, norm_max, norm_var = 0., 0., 0.
  for rank_stats in gathered:                          # rank order
    norm_sq += rank_stats[0]
    if math.isnan(rank_stats[1]) or math.isnan(norm_max):
      norm_max = math.nan                              # torch's max propagates a NaN; Python's max() may drop it
    elif rank_stats[1] > norm_max:
      norm_max = rank_stats[1]
  if n >= 2:
    for i in range(n):                                 # sample order, ranks inside
      dev = 0.
      for rank_stats in gathered:
        dev += rank_stats[2 + i]
      norm_var += _engine.fp32_overflow(dev)           # the reference's fp32 dot(): +inf past FLT_MAX
    norm_dev = math.sqrt(norm_var / (n - 1))
  else:
    norm_dev = math.nan
  return avg, _engine.fp32_norm(norm_sq), norm_dev, norm_max          # an fp32 norm, as on one GPU

def replicate(shard, group=None):
  """ All-gather the ranks' output shards into the full aggregated gradient on every rank
  (SURVEY.md §8(e): what a trainer that keeps a replicated model needs before
  `model.set_gradient`, experiments/model.py:368-380).  Shards may differ in length (the last
  rank's is shorter when R does not divide d): lengths are exchanged first, shards padded to
  the longest for the collective and trimmed after it.
  Args:
    shard  This rank's [d_r] slice of the result
    group  Process group (default: the world)
  Returns:
    [sum of d_r] vector, the shards in rank order
  """
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  if world == 1:
    return shard.clone()
  length = torch.tensor([shard.numel()], dtype=torch.int64, device=shard.device)
  lengths = torch.empty(world, dtype=torch.int64, device=shard.device)
  dist.all_gather_into_tensor(lengths, length, group=group)
  lengths = lengths.tolist()
  longest = max(lengths)
  padded = shard if shard.numel() == longest else torch.cat([shard, shard.new_zeros(longest - shard.numel())])
  gathered = torch.empty(world * longest, dtype=shard.dtype, device=shard.device)
  dist.all_gather_into_tensor(gathered, padded.contiguous(), group=group)
  if all(l == longest for l in lengths):
    return gathered
  return torch.cat([gathered[r * longest:r * longest + lengths[r]] for r in range(world)])


def shard_bounds(d, world, rank):
  """ [lo, hi) of rank's columns under the even split used throughout (the last shards may be shorter). """
  per = (d + world - 1) // world
  lo = min(d, rank * per)
  return lo, min(d, lo + per)

def apply_update(params, shard, lr, weight_decay=0., group=None):
  """ Close the d-sharded loop (SURVEY.md §8(f) row 4): the model update of `experiments/model.py:368-380`
  — `set_gradient(aggregated)` + `optimizer.step()` of the reference's plain SGD (attack.py:544:
  momentum 0, dampening 0, weight decay w) — done by every rank ON ITS SHARD of the flat parameter
  vector, followed by ONE all-gather of the updated parameters.  Against `replicate(shard)` + a
  replicated update this moves the same d*4 bytes over NVLink but does the update arithmetic once
  instead of R times and never materialises the full aggregated gradient.
  The arithmetic is torch's SGD: g' = g + w p (only when w != 0), p <- p - lr g', in place, fp32.
  Args:
    params        Flat fp32 parameter vector [d], replicated on every rank (updated in place)
    shard         This rank's [hi - lo] slice of the aggregated gradient (`ShardedPlan.out`)
    lr            Learning rate
    weight_decay  L2 coefficient w
    group         Process group (default: the world)
  Returns:
    `params`
  """
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  rank = dist.get_rank(group) if dist.is_initialized() else 0
  d = params.numel()
  lo, hi = shard_bounds(d, world, rank)
  if shard.numel() != hi - lo:
    raise ValueError(f"shard of {shard.numel()} elements, expected {hi - lo} (columns {lo}..{hi} of {d})")
  mine = params[lo:hi]
  if weight_decay != 0.:
    mine.add_(shard.add(mine, alpha=weight_decay), alpha=-lr)
  else:
    mine.add_(shard, alpha=-lr)
  if world == 1:
    return params
  per = (d + world - 1) // world
  if per * world == d:
    # in place with NCCL (rank r's slot of the output IS its shard); other backends get a copy
    dist.all_gather_into_tensor(params, mine if dist.get_backend(group) == "nccl" else mine.clone(), group=group)
    return params
  # ragged split: pad the shards to `per` for the collective, trim after it
  padded = mine if mine.numel() == per else torch.cat([mine, mine.new_zeros(per - mine.numel())])
  gathered = torch.empty(world * per, dtype=params.dtype, device=params.device)
  dist.all_gather_into_tensor(gathered, padded.contiguous(), group=group)
  params.copy_(gathered[:d])
  return params
