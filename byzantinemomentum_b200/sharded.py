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

import collections
import ctypes
import math

import torch
import torch.distributed as dist

from . import _lib
from . import engine as _engine

__all__ = ["aggregate", "aggregate_p2p", "compute_avg_dev_max", "study_step", "replicate", "apply_update", "shard_bounds", "rows_aligned", "choose_exchange", "rows_exchange", "plan_exchange", "choose_search_exchange", "PeerExchange", "FusedExchange", "ShardedPlan", "GradientShards", "choose_delivery", "ShardedLineSearch", "line_search", "search_rows", "search_exchange", "choose_anticge_exchange", "ShardedAntiCGE", "anticge", "COORDINATE_WISE", "DISTANCE_BASED"]

COORDINATE_WISE = ("average", "median", "trmean", "phocas", "meamed")
DISTANCE_BASED = _engine.DISTANCE_BASED

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
  def slot(self, step=None):
    """ (this rank's slot as a tensor, the R peers' addresses of the same slot) for `step` (default: this step). """
    off = ((self.step if step is None else step) % 2) * self.n * self.n
    mine = self.buffer[off:off + self.n * self.n]
    return mine, [base + off * 8 for base in self.peer_base]
  def publish(self):
    """ Order every rank's phase-A writes before anyone's reads (stream-ordered device barrier). """
    self.handle.barrier(channel=0)
    self.step += 1

_exchanges = {}

def _registered(registry, kind, n, device, group):
  """ The exchange of this kind for (n, device, group), set up on first use. """
  key = (n, device.index, id(group))
  ex = registry.get(key)
  if ex is None:
    ex = registry[key] = kind(n, device, group)
  return ex

def peer_exchange(n, device, group=None):
  return _registered(_exchanges, PeerExchange, n, device, group)

class FusedExchange:
  """ Symmetric buffer for the exchange that runs INSIDE the distance pass (`bz_krum_peers`,
  `bz_bulyan_peers`): per rank two slots of n*n doubles plus, per slot, a flag array of 16 words.  The
  last CTA of each rank's distance pass writes its block into its slot, raises its flag on every GPU,
  waits for the R flags, and adds the R blocks in place over NVLink — no barrier op, no collective, no
  separate selection kernel.  `epoch` (the step number) tells this step's flags from older ones; two
  slots make that enough (a rank rewrites slot s only after every peer has signalled the step in
  between, i.e. finished reading s).
  `ShardedLineSearch(exchange="fused")` runs its exchanges (the rule's block, the score's share) over the
  same buffer: one per call here, each advancing `epoch` by one; above MAX_N rows (`wide=True`) the rule's block goes
  through `bz_distance_select_peers`, as `ShardedPlan`'s does.  That relies on one condition: the calls
  that share a FusedExchange (the search and the `ShardedPlan` of the same n) are issued on ONE stream, in
  the same order on every rank.
  `ShardedAntiCGE(exchange="fused")` of nh honest rows runs its two exchanges (the nh norm sums, then the
  attack's sum of squares) over the buffer of n = nh in one `bz_anticge_peers` call, advancing `epoch` by two
  (by none when f_real > f_decl: the NaN fill exchanges nothing).  It shares the buffer with a `ShardedPlan`
  or `ShardedLineSearch` of the same n on the same condition: one stream, the same order on every rank.
  `ShardedPlan(exchange="fused")` of Aksel and CGE up to MAX_N rows runs its exchange in K2′'s last CTA
  (`bz_rowdist_peers`); above MAX_N rows, for all four rules, in phase B's kernel (`bz_distance_select_peers`,
  which copies the plan's staged phase-A block into the slot first): one exchange per call or replay either way,
  on the same condition of sharing.  So a buffer of n rows serves a `ShardedPlan`, a `ShardedAntiCGE` and a
  `ShardedLineSearch` of those n rows at any n, above MAX_N rows the search with `wide=True`.
  The epoch rule, kept here alone: `epoch` is the host's count of the exchanges issued so far (unbounded; the
  kernels see it modulo 2^32), and the flags hold the same count on the device (this rank's own entry [rank]
  of its flag array, in the slot of its last epoch).  An eager call of k exchanges takes `epoch + 1` as its
  first epoch, passes it by value with the tables of slot `epoch % 2` (`bz_anticge_peers`: of both slots),
  and leaves `epoch` k higher (`_reserve`).  A captured call cannot pass it: its `bz_*_peers_next` twin takes
  both slots' tables and the epoch from the flags (one past the later of the two own entries, wrap-aware; 1
  on a zeroed buffer), and each replay reserves the graph's exchanges, so that eager calls and replays can
  interleave on one buffer.  `_args` forms the arguments either way. """
  FLAG_WORDS = 16
  _slot_tables = None                                          # (slot 0's, slot 1's, both()), built on first use
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
  @classmethod
  def local(cls, n, device):
    """ The same layout on a plain device buffer, for one rank: no process group, no symmetric memory. """
    fx = cls.__new__(cls)
    fx.n, fx.device, fx.group, fx.world, fx.rank, fx.epoch = n, device, None, 1, 0, 0
    fx.buffer = torch.zeros(2 * n * n + cls.FLAG_WORDS, dtype=torch.float64, device=device)
    fx.handle = None
    fx.peer_base = [fx.buffer.data_ptr()]
    return fx
  def tables(self, slot):
    """ (ctypes array of the R block pointers, ctypes array of the R flag-array pointers) of a slot. """
    block = slot * self.n * self.n * 8
    flags = 2 * self.n * self.n * 8 + slot * self.FLAG_WORDS * 4
    return ((ctypes.c_void_p * self.world)(*[b + block for b in self.peer_base]),
            (ctypes.c_void_p * self.world)(*[b + flags for b in self.peer_base]))
  def both(self):
    """ The tables of both slots, as the `bz_*_peers_next` calls take them: (2R block pointers, 2R flag-array
    pointers), slot 0's then slot 1's. """
    (b0, f0), (b1, f1) = self.tables(0), self.tables(1)
    return ((ctypes.c_void_p * (2 * self.world))(*b0, *b1), (ctypes.c_void_p * (2 * self.world))(*f0, *f1))
  def _reserve(self, k):
    """ The first epoch of a call of k exchanges; `epoch` is left k higher. """
    first = self.epoch + 1
    self.epoch += k
    return first
  def _args(self, exchanging, epoch):
    """ (fn, args) of the `_Exchanging` call by value at `epoch`, or (None) of its `_next` twin. """
    if self._slot_tables is None:
      self._slot_tables = (self.tables(0), self.tables(1), self.both())
    fn, fn_next, head, tail, both = exchanging
    if epoch is None:
      return fn_next, head + self._slot_tables[2] + tail
    return fn, head + self._slot_tables[2 if both else epoch % 2] + (epoch % (1 << 32),) + tail

# A call that exchanges over a `FusedExchange`: its by-value entry point, its `_next` twin, its arguments before the
# slot tables (`head`) and after the epoch (`tail`); `both`: the by-value call takes both slots' tables.
_Exchanging = collections.namedtuple("_Exchanging", "fn fn_next head tail both", defaults=(False,))

_fused = {}

def fused_exchange(n, device, group=None):
  return _registered(_fused, FusedExchange, n, device, group)

def _capturable(exchange, world, what):
  """ Raise unless `what` can capture `exchange` on `world` ranks: "fused" anywhere, any exchange on one rank. """
  if exchange == "p2p" or (exchange == "nccl" and world > 1):
    raise ValueError(f"{what}.graph() captures the fused exchange on any number of ranks, or any exchange on one rank: "
                     f"not {exchange!r} on {world} ranks")

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

def _agree(facts, group):
  """ The element-wise minimum over the ranks of `group` of every rank's list of local facts (ints):
  one all-reduce (MIN), none on a single rank. """
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  if world == 1:
    return list(facts)
  device = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")
  agreed = torch.tensor(facts, dtype=torch.int32, device=device)
  dist.all_reduce(agreed, op=dist.ReduceOp.MIN, group=group)
  return agreed.tolist()

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
  aligned, symmetric = map(bool, _agree([int(bool(aligned)), int(bool(symmetric))], group))
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

def rows_exchange(exchange, n):
  """ The exchange `ShardedPlan` of n rows asks `choose_exchange` for.  The "p2p" and "fused" exchanges
  serve up to MAX_N rows; above, "auto" is "nccl" and an explicit "p2p" or "fused" raises.  Every rank has
  the same n, so every rank resolves the same way, before any collective. """
  if exchange not in EXCHANGES:
    raise ValueError(f"unknown exchange {exchange!r}")
  if n <= _lib.MAX_N or exchange in ("auto", "nccl"):
    return "nccl" if n > _lib.MAX_N else exchange
  raise ValueError(f"the {exchange} exchange serves at most MAX_N = {_lib.MAX_N} rows, not n = {n}: "
                   f"above, ShardedPlan exchanges through \"nccl\"")

def plan_exchange(gar, n, exchange, aligned, symmetric, group=None):
  """ The exchange of a `ShardedPlan` of n rows, the same on every rank of `group`.  "auto", "nccl" and "p2p"
  resolve as `rows_exchange` then `choose_exchange` do.  An explicit "fused" is served wherever the rule's exchange
  can run inside a kernel: krum and bulyan up to MAX_N rows keep `choose_exchange`'s rule (the distance ring's
  exchange, 16-byte aligned rows); aksel and cge at every n (`bz_rowdist_peers` up to MAX_N rows), and krum and
  bulyan above MAX_N rows, take rows of any alignment (above MAX_N rows, `bz_distance_select_peers` after phase A).
  Those need symmetric memory on every one of at most MAX_PEERS ranks, agreed on with one all-reduce (MIN), or a
  single rank.  A request some rank cannot serve raises on every rank.  Returns "fused",
  "p2p" or "nccl". """
  if exchange != "fused" or gar not in _engine.WIDE_DISTANCE or (gar in ("krum", "bulyan") and n <= _lib.MAX_N):
    return choose_exchange(gar, rows_exchange(exchange, n), aligned, symmetric, group)
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  (symmetric,) = map(bool, _agree([int(bool(symmetric))], group))
  if not (world == 1 or (symmetric and world <= _lib.MAX_PEERS)):
    raise ValueError(f"the fused exchange of {gar} on {n} rows needs symmetric memory on every one of at most "
                     f"{_lib.MAX_PEERS} ranks")
  return "fused"

def _phases(be, gar, gradients, f, m, mode, group, p2p):
  """ (this rank's shard of the result, the selection) of a distance-based rule.  Phase A computes
  this rank's partial block; the R blocks are all-gathered into [R, ...] in rank order, or (`p2p`)
  written into this rank's slot of the PeerExchange and read in place by phase B, which derives the
  selection; phase C reduces the local shard with it.  Phase B is the backend's
  `<select>_select(blocks, n, *select_params)` or `<select>_select_peers(peers, n, *select_params, device)`. """
  n = len(gradients)
  rule = _engine._rule(gar, n, f, m, mode)
  center = be.median(gradients) if rule.center else None           # coordinate-wise: local
  into = {}
  if p2p:
    ex = peer_exchange(n, gradients[0].device, group)
    mine, peers = ex.slot()
    into = dict(out=mine if rule.pair else mine[:n])
  part = be.pairdist_partial(gradients, **into) if rule.pair else be.rowdist_partial(gradients, center, **into)
  if p2p:
    ex.publish()
    picked = getattr(be, rule.select + "_select_peers")(peers, n, *rule.select_params, part.device)
  else:
    picked = getattr(be, rule.select + "_select")(_gather(part, group), n, *rule.select_params)
  sel, status = picked if rule.status else (picked, None)
  if gar == "bulyan":
    return be.bulyan_reduce(gradients, rule.f, rule.m, sel, status), sel
  return be.average_selected(gradients, sel, rule.count, rule.zero_init, status=status), sel

def aggregate_p2p(gar, gradients, f=None, m=None, mode="mid", group=None, return_selection=False):
  """ `aggregate` for the distance-based rules with the exchange fused into the selection kernel
  (peer memory over NVLink, see PeerExchange).  CUDA engine only. """
  if gar in COORDINATE_WISE:
    return aggregate(gar, gradients, f=f, m=m, mode=mode, group=group, return_selection=return_selection)
  out, sel = _phases(_engine, gar, gradients, f, m, mode, group, True)
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
            "fused" the exchange runs inside a kernel, over the symmetric buffer of `fused_exchange(n, ...)`
                    (which needs an initialised process group, or a buffer registered for it), one exchange
                    per call: krum and bulyan up to MAX_N rows in the distance pass, whose last CTA
                    publishes the block, flags the peers, waits for theirs and scores — a step is the single-GPU rule's two launches (`bz_krum_peers`,
                    16-byte aligned rows); aksel and cge up to MAX_N rows in K2′'s last CTA
                    (`bz_rowdist_peers`: [median], one call); the four rules above MAX_N rows in phase B
                    (`bz_distance_partial` into a staging buffer, `bz_distance_select_peers` of the second
                    library, `bz_distance_reduce`).  Rows of any alignment except for krum / bulyan up to
                    MAX_N rows;
            "auto"  "fused" where it applies on every rank (krum and bulyan up to MAX_N rows), else "p2p",
                    when every rank of the group has symmetric memory; else "nccl".  The ranks agree on
                    the choice (`plan_exchange`); a failing symmetric-memory setup raises.
  Every exchange uses the same fixed summation order: bitwise identical selections on every rank, and the
  fused exchange gives "nccl"'s bits.  `status` is always present with "fused" (0, or a peer that did not show up).
  Coordinate-wise rules need no exchange and simply wrap `engine.Plan`.
  Rows: up to MAX_N_DISTANCE for krum, bulyan, aksel and cge, MAX_N for brute.  Above MAX_N the exchange is
  "nccl" or an explicit "fused" (`plan_exchange`: "auto" resolves to "nccl", "p2p" raises); "nccl"'s phases are
  `bz_distance_partial`, `bz_distance_select` and `bz_distance_reduce` at every n: the n x n block of 128 rows
  is 131 KB per rank.  One rank gives `engine.Plan`'s output, selection and status bit for bit.
  With "fused" the buffer of `fused_exchange(n, ...)` can be shared with a `ShardedAntiCGE` of n honest rows and a
  `ShardedLineSearch` of n rows (above MAX_N rows with `wide=True`), their calls on one stream in the same order on
  every rank.

  `graph()` captures a step in a CUDA graph, as `engine.Plan.graph()` does: "fused" on any number of ranks
  (the captured kernel takes its epoch from the exchange buffer, the `_next` calls), any exchange on one
  rank; a coordinate-wise plan returns `engine.Plan.graph()`.  Like a call, `graph()` and every replay are
  collective: every rank issues them at the same point of its stream order. """
  def __init__(self, gar, gradients, f=None, m=None, mode="mid", group=None, exchange="auto"):
    self.gar, self.group = gar, group
    self.rows = list(gradients)
    n = self.n = len(self.rows)
    self.world = dist.get_world_size(group) if dist.is_initialized() else 1
    self.selection = None
    self.status = None
    self._graph = None
    if gar in COORDINATE_WISE:
      self._local = _engine.Plan(gar, self.rows, f=f)
      self.out = self._local.out
      self.exchange = "none"
      return
    rule = _engine._rule(gar, n, f, m, mode)
    self._local = None
    if exchange not in EXCHANGES:
      raise ValueError(f"unknown exchange {exchange!r}")
    limit = _lib.MAX_N_DISTANCE if gar in _engine.WIDE_DISTANCE else _lib.MAX_N
    prep = _engine._prepare_device(self.rows, limit=limit)
    if not all(g.is_contiguous() for g in self.rows):
      raise ValueError("ShardedPlan takes contiguous rows")
    device = self.device = prep.device
    self.d = prep.d
    if n > _lib.MAX_N:
      # the pass tables of bz_distance_partial, held by the plan, as `engine.Plan` holds them
      ws = self._ws = torch.empty(int(_lib.lib().bz_distance_workspace_bytes(n)), dtype=torch.uint8, device=device)
    else:
      ws = self._ws = _engine._workspace(device, prep.stream)
    self.out = torch.empty(prep.d, dtype=torch.float32, device=device)
    self._meta = torch.empty(n + 1, dtype=torch.int32, device=device)
    meta, status, out = self._meta.data_ptr(), self._meta[n:].data_ptr(), self.out.data_ptr()
    self.selection = self._meta[:rule.length]
    if rule.status:
      self.status = self._meta[n:]
    facts = (rows_aligned(self.rows), _symmetric_memory_importable(), group)
    if exchange == "fused" and not (dist.is_initialized() or (n, device.index, id(group)) in _fused):
      # no process group to set the fused buffer up over and none registered (`fused_exchange`): resolved as before
      exchange = self.exchange = choose_exchange(gar, rows_exchange(exchange, n), *facts)
    else:
      exchange = self.exchange = plan_exchange(gar, n, exchange, *facts)
    if exchange == "fused" and rule.pair and n <= _lib.MAX_N:
      fx = self._fx = fused_exchange(n, device, group)
      self.status = self._meta[n:]                          # krum too: a peer that never signals
      lib = _lib.lib()
      self._exchanging = _Exchanging(getattr(lib, f"bz_{gar}_peers"), getattr(lib, f"bz_{gar}_peers_next"),
                                     (prep.ptrs, n) + rule.params + (prep.d, out, meta, status, fx.rank, fx.world),
                                     (ws.data_ptr(), ws.numel(), prep.stream))
      self._fused_around = ([], [])
      return
    # aksel: the coordinate-wise median of the local shard is the center of phase A
    self._median = _engine.Plan("median", self.rows) if rule.center else None
    center = None if self._median is None else self._median.out.data_ptr()
    width = n * n if rule.pair else n
    if exchange == "fused":
      self._fuse(rule, prep, center, ws, out, meta, status)
      return
    if exchange == "p2p":
      def phases(part, blocks):
        return _engine._partial_call(prep, rule.pair, center, part, ws), _engine._select_call(rule, blocks, meta, prep.stream)
      # two slots -> two prepared argument sets; the step counter of the exchange picks one
      self._ex = peer_exchange(n, device, group)
      self._ab = [phases(mine.data_ptr(), peers) for mine, peers in map(self._ex.slot, range(2))]
      self._c = _engine._reduce_call(prep, rule, meta, status if rule.status else None, out)
    else:
      # bz_distance_partial / _select / _reduce: one dispatch for 1 to MAX_N_DISTANCE rows
      self._part = torch.empty(width, dtype=torch.float64, device=device)
      self._gathered = torch.empty((self.world, width), dtype=torch.float64, device=device)
      a, b, self._c = rule.phase_entries(prep.ptrs, prep.d, center, self._part.data_ptr(), self._gathered.data_ptr(),
                                         self.world, out, meta, ws, prep.stream)
      self._ab = [(a, b)]
  def _fuse(self, rule, prep, center, ws, out, meta, status):
    """ The fused exchange of Aksel and CGE up to MAX_N rows (`bz_rowdist_peers`: phase A, the exchange, the
    selection and the reduce in its kernels), and of the four rules above (`bz_distance_partial` into a staging
    buffer, `bz_distance_select_peers` of the second library, `bz_distance_reduce`). """
    n, device, gar = self.n, self.device, self.gar
    fx = self._fx = fused_exchange(n, device, self.group)
    self.status = self._meta[n:]
    code, (m, mode) = _engine._SEARCH_RULES[gar], rule._m_mode()
    before = [(self._median._fn, self._median._args)] if self._median is not None else []
    if n <= _lib.MAX_N:
      lib = _lib.lib()
      self._exchanging = _Exchanging(lib.bz_rowdist_peers, lib.bz_rowdist_peers_next,
                                     (code, prep.ptrs, n, rule.f, mode, center, prep.d, out, meta, status, fx.rank, fx.world),
                                     (ws.data_ptr(), ws.numel(), prep.stream))
      self._fused_around = (before, [])
    else:
      peers = _lib.peers_lib()
      self._part = torch.empty(n * n if rule.pair else n, dtype=torch.float64, device=device)
      a, _, c = rule.phase_entries(prep.ptrs, prep.d, center, self._part.data_ptr(), None, 1, out, meta, ws, prep.stream)
      self._exchanging = _Exchanging(peers.bz_distance_select_peers, peers.bz_distance_select_peers_next,
                                     (code, self._part.data_ptr(), n, rule.f, m, mode, meta, status, fx.rank, fx.world),
                                     (prep.stream,))
      self._fused_around = (before + [a], [c])
  def __call__(self):
    if self._local is not None:
      return self._local()
    with _engine._on(self.device):
      self._issue()
    return self.out
  def graph(self):
    """ Capture a step in a CUDA graph (after one eager step, the warm-up) and return `replay`: a callable
    that launches it and returns `plan.out`.  With "fused", each replay advances the exchange's epoch by one. """
    if self._local is not None:
      return self._local.graph()
    _capturable(self.exchange, self.world, "ShardedPlan")
    fx = self._fx if self.exchange == "fused" else None
    return _engine._capture(self, self.device, lambda call: self._issue(call, captured=True), lambda: self.out, fx, 1)
  def _issue(self, call=_engine._call, captured=False):
    """ One step's calls through `call(fn, args)`; `captured`: the fused exchange takes its epoch from the buffer. """
    if self.exchange == "fused":
      before, after = self._fused_around
      for step in before:
        call(*step)
      fx = self._fx
      call(*fx._args(self._exchanging, None if captured else fx._reserve(1)))
      for step in after:
        call(*step)
      return
    if self._median is not None:
      call(self._median._fn, self._median._args)
    if self.exchange == "p2p":
      ex = self._ex
      a, b = self._ab[ex.step % 2]
      call(*a)
      ex.publish()
    else:
      a, b = self._ab[0]
      call(*a)
      if self.world > 1:
        dist.all_gather_into_tensor(self._gathered, self._part, group=self.group)
      else:
        self._gathered.copy_(self._part.unsqueeze(0))
    call(*b)
    call(*self._c)

SEARCH_EXCHANGES = ("auto", "fused", "nccl")

def search_rows(gar, wide=False, many=False):
  """ The most rows (honest + f_real) `ShardedLineSearch` takes against the rule `gar`: `engine.search_max_rows(gar)`,
  with `wide` MAX_N_DISTANCE for krum, bulyan, aksel and cge (brute stays at MAX_N), and with `many` MAX_N_MANY for
  the coordinate-wise rules (without it they stay at MAX_N_COORDINATE). """
  if wide and gar in _engine.WIDE_DISTANCE:
    return _lib.MAX_N_DISTANCE
  if many and gar in COORDINATE_WISE:
    return _lib.MAX_N_MANY
  return _engine.search_max_rows(gar)

def choose_search_exchange(exchange, aligned, symmetric, engine, group=None):
  """ The exchange of `ShardedLineSearch`, the same on every rank of `group`: the local facts — `aligned`:
  this rank's rows suit the rule's fused call (16-byte aligned for Multi-Krum, Bulyan and brute, any for
  the others); `symmetric`: symmetric memory can be set up here; `engine`: the CUDA library runs the
  stages — are agreed on with one all-reduce (MIN), as in `choose_exchange`.  "auto" takes "fused" on 2 to
  16 ranks that all have the facts, else "nccl" (one rank, or a stand-in backend, keeps the collective
  path).  An explicit "fused" needs `aligned` on every rank, and symmetric memory on every one of at most
  16 ranks unless there is one rank (its buffer is then plain device memory); otherwise it raises on every
  rank.  Returns "fused" or "nccl". """
  if exchange not in SEARCH_EXCHANGES:
    raise ValueError(f"unknown exchange {exchange!r}")
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  aligned, symmetric, engine = map(bool, _agree([int(bool(aligned)), int(bool(symmetric)), int(bool(engine))], group))
  fusable = aligned and (world == 1 or (symmetric and world <= _lib.MAX_PEERS))
  if exchange == "auto":
    return "fused" if world > 1 and engine and fusable else "nccl"
  if exchange == "fused" and not fusable:
    raise ValueError(f"the fused exchange of the line search needs 16-byte aligned rows for krum / bulyan / brute on every rank, "
                     f"and symmetric memory on every one of at most {_lib.MAX_PEERS} ranks")
  return exchange

def search_exchange(gar, n, exchange, aligned, symmetric, engine, group=None, wide=False):
  """ The exchange of a `ShardedLineSearch` of n rows against `gar`, the same on every rank of `group`:
  `choose_search_exchange`'s, except with `wide` for krum, bulyan, aksel and cge above MAX_N rows.  There the
  exchange runs in phase B's kernel (`bz_distance_select_peers`), so rows of any alignment are served, and "auto"
  resolves to "nccl", as `ShardedPlan` resolves it above MAX_N rows.  The ranks still agree through
  `choose_search_exchange`'s one all-reduce. """
  if wide and gar in _engine.WIDE_DISTANCE and n > _lib.MAX_N:
    return choose_search_exchange("nccl" if exchange == "auto" else exchange, True, symmetric, engine, group)
  return choose_search_exchange(exchange, aligned, symmetric, engine, group)

DELIVERIES = ("auto", "p2p", "collective")

def choose_delivery(exchange, symmetric, group=None):
  """ The exchange of `GradientShards`, the same on every rank of `group`: the local fact `symmetric`
  (symmetric memory can be set up here) is agreed on with one all-reduce (MIN), as in
  `choose_exchange`.  "auto" takes "p2p" on several ranks that all have symmetric memory, else
  "collective"; an explicit "p2p" that some rank cannot serve raises on every rank. """
  if exchange not in DELIVERIES:
    raise ValueError(f"unknown exchange {exchange!r}")
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  (symmetric,) = map(bool, _agree([int(bool(symmetric))], group))
  if exchange == "auto":
    return "p2p" if world > 1 and symmetric else "collective"
  if exchange == "p2p" and not symmetric:
    raise ValueError("the p2p exchange needs symmetric memory on every rank")
  return exchange

class _SymmetricRows:
  """ A fp32 buffer of `shape` in symmetric memory (one allocation mapped into every rank of the group
  over NVLink / NVSwitch), `peers[r]`: rank r's buffer as a tensor on this GPU, `barrier()`: the
  stream-ordered device barrier of the group. """
  def __init__(self, shape, device, group):
    if not dist.is_initialized():
      raise ValueError("the p2p exchange needs an initialised process group: its symmetric buffer is set up across the group's ranks")
    import torch.distributed._symmetric_memory as symm_mem
    group = group if group is not None else dist.group.WORLD
    self.buffer = symm_mem.empty(*shape, dtype=torch.float32, device=device)
    self.handle = symm_mem.rendezvous(self.buffer, group)
    self.peers = [self.handle.get_buffer(r, tuple(shape), torch.float32) for r in range(dist.get_world_size(group))]
  def barrier(self):
    self.handle.barrier(channel=0)

def _symmetric_rows(shape, device, group):
  return _SymmetricRows(shape, device, group)

class GradientShards:
  """ Delivery of the worker gradients to the d-sharded path (the multi-GPU counterpart of
  `engine.GradientStack`).  Worker i is backpropagated on rank i % R, where it is one full [d] vector;
  the rules need columns [lo_r, hi_r) (`shard_bounds`) of all n workers on every rank r.  `push` clips
  the gradient and writes each rank's columns straight into that rank's memory in ONE pass
  (`bz_gradient_scatter`); `deliver` makes them visible to their owners.

      shards = sharded.GradientShards(n, d, device)            # once; exchange="auto"
      for i in shards.workers():                              # this rank's workers: i % R == rank
        grad, loss = model.backprop(outloss=True)
        shards.push(i, grad, clip=args.gradient_clip)
      sampled = shards.deliver()                              # n rows of this rank's hi - lo columns
      honest = shards.honests_worker(gmtm_shards, mu, dampening)   # or honests_server(server_shard, ...), or `sampled`
      out = plans[shards.slot]()                              # a ShardedPlan per slot over shards.rows(slot)

  exchange: "p2p"         every rank owns a SYMMETRIC buffer of two slots of [n, pitch] fp32 (pitch:
                          ceil(d / R) rounded up to 64 floats); `push` writes slot `step % 2` of every
                          rank over NVLink and `deliver` crosses one device-side barrier.  Two slots make
                          that barrier enough: a producer rewrites slot s only after the barrier of the
                          step in between, which every owner reaches only after its reads of slot s.
            "collective"  `push` writes into this rank's [R, ceil(n / R), pitch] send buffer, `deliver`
                          does one `all_to_all_single` into the matching receive buffer (a copy on a
                          single rank); row i is `recv[i % R, i // R, :hi - lo]`.
            "auto"        "p2p" when every rank of several has symmetric memory, else "collective"; the
                          ranks agree on it (`choose_delivery`).
  Both exchanges deliver the same bits: those of `GradientStack.push`'s sampled row, sliced.
  Momentum is placed by the owner on its columns, all rows in one launch (`honests_worker` /
  `honests_server`, `bz_gradient_momentum`: the arithmetic of `GradientStack.push` after the clip):
  only the clipped gradient crosses NVLink, and the momentum buffers stay local shards.

  Contract: the rows of a step stay valid until this rank calls `deliver()` of the next step.  A rank
  whose shard is empty (rank r * ceil(d / R) >= d: when d < R, but also e.g. rank 3 for d = 9, R = 4)
  has rows of zero columns and still joins every barrier and collective.
  `push` of a worker this rank does not produce raises, and so does `deliver` while one of this rank's
  workers has not been pushed.  Build one `ShardedPlan` per slot (`slots` of them) over `rows(slot)`.

  `backend` provides `gradient_scatter` and `momentum_rows` (default: the CUDA engine). """
  def __init__(self, n, d, device, group=None, exchange="auto", backend=None):
    self.n, self.d, self.group = int(n), int(d), group
    self.device = torch.device(device)
    if self.device.type == "cuda" and self.device.index is None:
      self.device = torch.device("cuda", torch.cuda.current_device())
    self.world = dist.get_world_size(group) if dist.is_initialized() else 1
    self.rank = dist.get_rank(group) if dist.is_initialized() else 0
    if self.world > _lib.MAX_PEERS:
      raise ValueError(f"GradientShards serves at most {_lib.MAX_PEERS} ranks (BZ_MAX_PEERS): the group has {self.world}")
    self._be = backend or _engine
    self.lo, self.hi = shard_bounds(self.d, self.world, self.rank)
    width = self.hi - self.lo
    self.pitch = ((self.d + self.world - 1) // self.world + 63) // 64 * 64
    bounds = [shard_bounds(self.d, self.world, r) for r in range(self.world)]
    self.exchange = choose_delivery(exchange, _symmetric_memory_importable(), group)
    R = self.world
    if self.exchange == "p2p":
      sym = self._sym = _symmetric_rows((2, self.n, self.pitch), self.device, group)
      self.slots = 2
      self._local = sym.buffer
      self._dest = {(s, i): [sym.peers[r][s, i, :hi - lo] for r, (lo, hi) in enumerate(bounds)]
                    for s in range(2) for i in self.workers()}
      self._rows = [[sym.buffer[s, i, :width] for i in range(self.n)] for s in range(2)]
    else:
      self._local = torch.empty((R, (self.n + R - 1) // R, self.pitch), dtype=torch.float32, device=self.device)
      self._send = torch.empty_like(self._local)     # also on one rank: a push must not overwrite delivered rows
      self.slots = 1
      self._dest = {(0, i): [self._send[r, i // R, :hi - lo] for r, (lo, hi) in enumerate(bounds)] for i in self.workers()}
      self._rows = [[self._local[i % R, i // R, :width] for i in range(self.n)]]
    self._honest = None
    self._pushed = set()
    self.step = 0
  def workers(self):
    """ The workers this rank produces: i % R == rank. """
    return range(self.rank, self.n, self.world)
  @property
  def slot(self):
    """ The slot of the last delivered step (0 with the collective exchange). """
    if self.step == 0:
      raise RuntimeError("nothing delivered yet")
    return (self.step - 1) % self.slots
  def rows(self, slot=None):
    """ This rank's columns of the n workers in `slot` (default: the last delivered step's), as views. """
    return list(self._rows[self.slot if slot is None else slot])
  def push(self, i, grad, clip=None):
    """ Clip worker i's full gradient (clip None or <= 0: no clipping) and write every rank's columns
    of it into that rank's row i of this step. """
    if not 0 <= i < self.n or i % self.world != self.rank:
      raise ValueError(f"worker {i} is produced on rank {i % self.world} of {self.world}, not on rank {self.rank}")
    if grad.numel() != self.d or grad.device != self.device:
      raise ValueError(f"grad must hold d = {self.d} elements on {self.device}: it has {grad.numel()} on {grad.device}")
    self._be.gradient_scatter(grad, clip, self._dest[(self.step % self.slots, i)])
    self._pushed.add(i)
  def deliver(self):
    """ Finish the step: every rank's pushes reach their owners.  Returns this rank's n rows. """
    missing = [i for i in self.workers() if i not in self._pushed]
    if missing:
      raise RuntimeError(f"workers {missing} of rank {self.rank} were not pushed this step")
    if self.exchange == "p2p":
      self._sym.barrier()
    elif self.world > 1:
      dist.all_to_all_single(self._local, self._send, group=self.group)
    else:
      self._local.copy_(self._send)
    # other GPUs' kernels (or the collective) wrote the rows: tell PyTorch, whose version counter the
    # identity / version keyed caches of this package rely on (views share their base's counter)
    torch.autograd.graph.increment_version(self._local)
    self._pushed.clear()
    self.step += 1
    return self.rows()
  def honests_worker(self, momentums, mu, dampening):
    """ Worker-side momentum (attack.py:799-803) on this rank's columns: momentums[k] <- momentums[k] *
    mu + (1 - dampening) * row k, in place, for the first len(momentums) rows.  Returns `momentums`. """
    momentums = list(momentums)
    if len(momentums) > self.n:
      raise ValueError(f"{len(momentums)} momentum vectors for {self.n} workers")
    if momentums:
      self._be.momentum_rows(self.rows()[:len(momentums)], mu, dampening, momentums=momentums)
    return momentums
  def honests_server(self, server, mu, dampening, count=None):
    """ Server-side momentum (attack.py:805-808) on this rank's columns: honest row k = row k * (1 -
    dampening) + mu * server, for the first `count` rows (default n), into a buffer of this object
    (rewritten by the next call).  `server` is this rank's shard of the server momentum (the previous
    `ShardedPlan.out`).  Returns the honest rows. """
    rows = self.rows()[:self.n if count is None else count]
    if self._honest is None:
      self._honest = _engine._row_buffer(self.n, self.hi - self.lo, self.device)
    honest = [self._honest[k, :self.hi - self.lo] for k in range(len(rows))]
    if rows:
      self._be.momentum_rows(rows, mu, dampening, server=server, honests=honest)
    return honest

_CACHE_DOUBLES = _lib.MAX_N * _lib.MAX_N            # BZ_CACHE_DOUBLES

class _SearchShard:
  """ One rank's device side of `ShardedLineSearch`: the calls of every stage resolved once (row pointers,
  buffers, workspace, the current stream at construction), for `world` ranks.
    blocks, part   [world, width] gathered partial blocks of the rule / this rank's block (blocks[0] on one rank)
    scores, score  [world] gathered score shares / this rank's share (scores[:1] on one rank)
  `fuse(fx)` prepares the stages of the fused exchange over the FusedExchange `fx` as well. """
  def __init__(self, gar, grad_honests, f_real, f_decl, grad_avg, grad_att, evals, negative, kind, world, wide=False, many=False):
    honest = list(grad_honests)
    f_real = int(f_real)
    n = len(honest) + f_real
    limit = search_rows(gar, wide, many)
    if f_real < 1 or n > limit:
      raise ValueError(f"f_real = {f_real} with {len(honest)} honest rows: expected f_real >= 1 and at most {limit} rows")
    prep = _engine._prepare_device(honest, "the line search takes CUDA tensors", limit=limit)
    if not all(g.is_contiguous() for g in honest):
      raise ValueError("the line search takes contiguous honest gradients")
    for vector in [grad_avg] if grad_att is None else [grad_avg, grad_att]:
      _engine._check_like_rows(vector, prep, "grad_avg and grad_att")
    device, d, stream = prep.device, prep.d, prep.stream
    self.device, self.evals = device, evals
    self.byz = torch.empty(d, dtype=torch.float32, device=device)
    self.out = torch.empty(d, dtype=torch.float32, device=device)
    self.record = torch.zeros(2 * evals + 2, dtype=torch.float64, device=device)
    self._state = torch.zeros(_lib.SEARCH_STATE_BYTES // 8, dtype=torch.float64, device=device)
    self.scores = torch.zeros(world, dtype=torch.float64, device=device)
    self.score = self.scores[:1] if world == 1 else torch.zeros(1, dtype=torch.float64, device=device)
    inputs = honest + [self.byz] * f_real
    rows = self._rows = _engine._prepare_device(inputs, limit=limit)
    ws = self._ws = _engine._workspace(device, stream)
    lib = _lib.lib()
    state, out, avg = self._state.data_ptr(), self.out.data_ptr(), grad_avg.data_ptr()
    self._avg = avg
    att = None if grad_att is None else grad_att.data_ptr()
    self._candidates = [(lib.bz_search_candidate, (avg, att, self.byz.data_ptr(), d, state, which, int(bool(negative)),
                                                   _engine._SEARCH_KINDS[kind], stream))
                        for which in (_lib.CANDIDATE_FIRST, _lib.CANDIDATE_NEXT, _lib.CANDIDATE_FINAL)]
    self._score = (lib.bz_search_score_partial, (out, avg, d, state, self.score.data_ptr(), ws.data_ptr(), ws.numel(), stream))
    self._stream = stream
    self.call = _engine._call           # every stage's calls go through it (`ShardedLineSearch._issue` sets it)
    self.distance = gar in DISTANCE_BASED
    self.wide = self.distance and n > _lib.MAX_N
    eval_status = None
    self._pair = False
    if self.wide:
      eval_status = self._wide(gar, n, f_decl, honest, inputs, world)
    elif not self.distance:
      self._coordinate = _engine._coordinate_call(gar, rows, f_decl, out)
    else:
      rule = self._rule = _engine._rule(gar, n, f_decl)
      width = n * n if rule.pair else n
      self.blocks = torch.zeros((world, width), dtype=torch.float64, device=device)
      self.part = self.blocks[0] if world == 1 else torch.zeros(width, dtype=torch.float64, device=device)
      self._meta = torch.zeros(n + 1, dtype=torch.int32, device=device)      # order[n] + status
      meta = self._meta.data_ptr()
      status = meta + 4 * n if rule.status else None
      eval_status = None if rule.gar == "krum" else status
      part = self.part.data_ptr()
      self._pair = rule.pair
      if rule.pair:
        # the honest rows keep their place in the table from one evaluation to the next, the candidate row
        # (one tensor f_real times, new content) is new at every evaluation; an empty shard's rows are all
        # distinct, as bz_pairdist_partial_reuse counts them
        first = {}
        to_unique = [first.setdefault(g.data_ptr() if d > 0 else i, len(first)) for i, g in enumerate(inputs)]
        u = len(first)
        old_index = (ctypes.c_int32 * n)(*[to_unique[i] if i < len(honest) else -1 for i in range(n)])
        self._tables = torch.empty((2, _CACHE_DOUBLES), dtype=torch.float64, device=device)
        self._mode = ctypes.c_int(-1)
        tables = [t.data_ptr() for t in self._tables]
        # the reuse arguments of evaluation k writing table k % 2, after one reading table (k - 1) % 2 or not
        self._reuse = [[((old_index, tables[1 - s], u) if reused else (None, None, 0)) + (tables[s], ctypes.byref(self._mode))
                        for reused in (False, True)] for s in (0, 1)]
        def phase_a(reuse):
          return lib.bz_pairdist_partial_reuse, (rows.ptrs, n, d, part) + reuse + (ws.data_ptr(), ws.numel(), stream)
        # [k % 2][reuse]
        self._phase_a = [[phase_a(reuse) for reuse in self._reuse[s]] for s in (0, 1)]
      else:
        # aksel: the local coordinate-wise median is the centre; it goes to `out`, which the reduce rewrites (bz_aksel's order)
        self._median = _engine._coordinate_call("median", rows, None, out) if rule.center else None
        self._phase_a = _engine._partial_call(rows, False, out if rule.center else None, part, ws)
      self._select = _engine._select_call(rule, self.blocks, meta, stream)
      self._reduce = _engine._reduce_call(rows, rule, meta, status, out)
    record = self.record.data_ptr()
    self._steps = [(lib.bz_search_step, (self.scores.data_ptr(), world, state, record, eval_status, record + 8 * (2 * evals + 1),
                                         k, evals, stream)) for k in range(evals)]
  def _wide(self, gar, n, f_decl, honest, inputs, world):
    """ The stages of a distance rule above MAX_N rows (krum, bulyan, aksel, cge): phase A through
    `bz_distance_partial_reuse` (krum, bulyan: the honest rows' pass tables kept in two tables the evaluations
    alternate between), `bz_distance_partial` (aksel after its local median; cge at the first evaluation, then
    `bz_rowshare_star` of the third library, which rewrites only the candidate's sums), phases B and C through
    `bz_distance_select` and `bz_distance_reduce`.  The search owns its workspace and tables, so nothing else on the
    stream rewrites them between two evaluations.  Returns the evaluation's status word for the transition. """
    lib = _lib.lib()
    rows, device, stream, d = self._rows, self.device, self._stream, self._rows.d
    out = self.out.data_ptr()
    rule = self._rule = _engine._rule(gar, n, f_decl)
    width = n * n if rule.pair else n
    self.blocks = torch.zeros((world, width), dtype=torch.float64, device=device)
    self.part = self.blocks[0] if world == 1 else torch.zeros(width, dtype=torch.float64, device=device)
    self._meta = torch.zeros(n + 1, dtype=torch.int32, device=device)      # order[n] + status
    meta = self._meta.data_ptr()
    ws = self._ws = torch.empty(int(lib.bz_distance_workspace_bytes(n)), dtype=torch.uint8, device=device)
    fn, args = self._score
    self._score = fn, args[:5] + (ws.data_ptr(), ws.numel(), stream)
    self._median = _engine._coordinate_call("median", rows, None, out) if rule.center else None
    part = self.part.data_ptr()
    full, select, self._reduce = rule.phase_entries(rows.ptrs, d, out if rule.center else None, part, self.blocks.data_ptr(),
                                                    world, out, meta, ws, stream)
    self._select = select
    self._pair = rule.pair
    if rule.pair:
      # as up to MAX_N rows: the honest rows keep their unique rows, the candidate (one tensor f_real times) is the
      # last unique row; evaluation k writes table k % 2, reading table (k - 1) % 2 after the first
      first = {}
      for g in inputs:
        first.setdefault(g.data_ptr(), len(first))
      u = len(first)
      old_index = (ctypes.c_int32 * n)(*[first[g.data_ptr()] if i < len(honest) else -1 for i, g in enumerate(inputs)])
      self._tables = torch.empty((2, int(lib.bz_distance_pass_tables_bytes()) // 8), dtype=torch.float64, device=device)
      self._mode = ctypes.c_int(-1)
      tables = [t.data_ptr() for t in self._tables]
      code = _engine._SEARCH_RULES[gar]
      def phase_a(s, reused):
        reuse = (old_index, tables[1 - s], u) if reused else (None, None, 0)
        return lib.bz_distance_partial_reuse, ((code, rows.ptrs, n, d, part) + reuse + (tables[s], ctypes.byref(self._mode))
                                               + (ws.data_ptr(), ws.numel(), stream))
      self._phase_a = [[phase_a(s, reused) for reused in (False, True)] for s in (0, 1)]
    elif gar == "cge":
      # after the first evaluation only the candidate's sums change: K2'-star (libbyzagg_star) rewrites part[nh, n)
      star = _lib.star_lib()
      self._star_ws = torch.empty(int(star.bz_rowshare_star_workspace_bytes(n)), dtype=torch.uint8, device=device)
      self._phase_a = [full, (star.bz_rowshare_star, (rows.ptrs, n, len(honest), d, part, self._star_ws.data_ptr(),
                                                      self._star_ws.numel(), stream))]
    else:
      self._phase_a = full
    status = meta + 4 * n if rule.status else None
    return None if gar == "krum" else status
  def fuse(self, fx):
    """ Prepare the stages of the fused exchange over `fx` (a `FusedExchange` of n rows): per evaluation the
    rule's `*_peers` call (distance rules) and `bz_search_score_peers`, every argument but the slot's
    tables and the epoch resolved here (and of their `bz_*_peers_next` twins, which take both slots' tables
    and no epoch).  Every distance rule then reports a status word (0, or a peer that did not show up), which
    the score's transition folds into the search's. """
    lib = _lib.lib()
    rows, ws, stream = self._rows, self._ws, self._stream
    n, d, state, out, record = rows.n, rows.d, self._state.data_ptr(), self.out.data_ptr(), self.record.data_ptr()
    self._fx = fx
    tail = (ws.data_ptr(), ws.numel(), stream)
    peers = (fx.rank, fx.world)
    eval_status = None
    if self.distance:
      rule, meta = self._rule, self._meta.data_ptr()
      code = _engine._SEARCH_RULES[rule.gar]
      eval_status = meta + 4 * n
      if self.wide:
        # above MAX_N rows: phase A into the staging block `part`, then phase B's kernel copies it into the slot and
        # exchanges it (libbyzagg_peers), then phase C
        peers_lib, (m, mode) = _lib.peers_lib(), rule._m_mode()
        self._rule_peers = _Exchanging(peers_lib.bz_distance_select_peers, peers_lib.bz_distance_select_peers_next,
                                       (code, self.part.data_ptr(), n, rule.f, m, mode, meta, eval_status) + peers, (stream,))
      elif self._pair:
        head = (code, rows.ptrs, n, rule.f, rule.m, d, out, meta, eval_status)
        self._rule_peers = [[_Exchanging(lib.bz_pairdist_reuse_peers, lib.bz_pairdist_reuse_peers_next, head + reuse + peers, tail)
                             for reuse in self._reuse[s]] for s in (0, 1)]
      else:
        mode = _lib.AKSEL_MODES["mid"] if rule.center else 0
        self._rule_peers = _Exchanging(lib.bz_rowdist_peers, lib.bz_rowdist_peers_next,
                                       (code, rows.ptrs, n, rule.f, mode, out if rule.center else None, d, out, meta,
                                        eval_status) + peers, tail)
    self._score_peers = [_Exchanging(lib.bz_search_score_peers, lib.bz_search_score_peers_next,
                                     (out, self._avg, d, state, record, eval_status, record + 8 * (2 * self.evals + 1), k,
                                      self.evals) + peers, tail)
                         for k in range(self.evals)]
  def _phase_a_call(self, k):
    """ (fn, args) of evaluation k's phase A on the distance-rule paths that reuse pair distances or take no reuse. """
    if self.wide and self._rule.gar == "cge":
      return self._phase_a[int(k > 0)]
    if not self._pair:
      return self._phase_a
    if self.wide:
      return self._phase_a[k % 2][int(k > 0)]
    return self._phase_a[k % 2][int(k > 0 and self._mode.value >= 0)]
  def evaluate_fused(self, k, epoch):
    """ Evaluation k up to its score with the fused exchange: the candidate row, then the rule (distance
    rules: its exchange at `epoch`, or None: at the epoch the flags give; coordinate-wise rules: no exchange). """
    with _engine._on(self.device):
      self.call(*self._candidates[_lib.CANDIDATE_FIRST if k == 0 else _lib.CANDIDATE_NEXT])
      if not self.distance:
        self.call(*self._coordinate)
      elif self.wide:
        if self._median is not None:
          self.call(*self._median)
        self.call(*self._phase_a_call(k))
        self.call(*self._fx._args(self._rule_peers, epoch))
        self.call(*self._reduce)
      elif self._pair:
        self.call(*self._fx._args(self._rule_peers[k % 2][int(k > 0 and self._mode.value >= 0)], epoch))
      else:
        if self._median is not None:
          self.call(*self._median)
        self.call(*self._fx._args(self._rule_peers, epoch))
  def score_fused(self, k, epoch):
    """ The score of evaluation k, its exchange at `epoch` (None: at the epoch the flags give) and the transition. """
    with _engine._on(self.device):
      self.call(*self._fx._args(self._score_peers[k], epoch))
  def evaluate(self, k):
    call = self.call
    with _engine._on(self.device):
      call(*self._candidates[_lib.CANDIDATE_FIRST if k == 0 else _lib.CANDIDATE_NEXT])
      if not self.distance:
        call(*self._coordinate)
        call(*self._score)
        return self.score
      if not self._pair and self._median is not None:
        call(*self._median)
      call(*self._phase_a_call(k))
    return self.part
  def conclude(self, blocks):
    if blocks is self.blocks:
      select = self._select
    elif self.wide:
      fn, args = self._select
      select = fn, args[:1] + (blocks.data_ptr(), blocks.shape[0]) + args[3:]
    else:
      select = _engine._select_call(self._rule, blocks, self._meta.data_ptr(), self._stream)
    with _engine._on(self.device):
      self.call(*select)
      self.call(*self._reduce)
      self.call(*self._score)
    return self.score
  def step(self, k, scores):
    fn, args = self._steps[k]
    if scores is not self.scores:
      args = (scores.data_ptr(), scores.numel()) + args[2:]
    with _engine._on(self.device):
      self.call(fn, args)
  def finish(self):
    with _engine._on(self.device):
      self.call(*self._candidates[_lib.CANDIDATE_FINAL])
    return self.byz

class ShardedLineSearch:
  """ The attacks' line search (`engine.LineSearch`: `line_maximize(eval_factor, evals)` of the identical-family
  attacks or of empire-strict against the rule `gar` with its defaults and f = f_decl) on a d-sharded
  trainer.  Every rank passes its columns of the honest rows, of `grad_avg` and of `grad_att`; a score is
  a sum over all d columns, so each evaluation is, on every rank:
    1. the candidate row of the current factor (this rank's columns);
    2. the rule on honest + [byz] * f_real: coordinate-wise rules locally, with no exchange; Multi-Krum,
       Bulyan and brute: phase A with distance reuse (only the candidate's pairs after the first
       evaluation), ONE `all_gather_into_tensor` of the n x n blocks, phases B and C; Aksel (its local
       median) and CGE: the row distances, one all-gather of n doubles, phases B and C;
    3. this rank's fp64 share of the score, one all-gather of R doubles;
    4. the transition: y = fl32 of the R shares added in rank order, then the next factor, bitwise the
       same on every rank.
  A last candidate writes this rank's shard of the Byzantine gradient (`byz`) for the chosen factor.
  `evals` is fixed in advance, so every rank issues the same launches and collectives and no host-side
  decision is shared; a rank with an empty shard joins every collective.  On one rank there is no
  collective, and the trace, the factor, `byz` and the rule's last output are those of `engine.LineSearch`.
  Like `ShardedPlan`, `search()` only issues the work on the stream that was current at construction (no
  allocation, no synchronisation), and holds what it reads and writes; `result()` reads `record` once.

  The caller forms the shard of the attack direction: for `little` and `empire` the columns of the
  full-vector direction; for `bulyan` (a one-hot vector at `target_idx`) that column lies on exactly one
  rank (shard_bounds), every other rank's shard of it is zero.

  Each evaluation's work between two exchanges is one stage method (`evaluate`, `conclude`, `step`,
  `finish`), so that `search()` is those stages plus the collectives.  `backend`, for tests, provides
  `search_shard(gar, grad_honests, f_real, f_decl, grad_avg, grad_att, evals, negative, kind, world)`, an
  object with the stages (default: the CUDA library).

  exchange: "nccl"   the collectives above;
            "fused"  no collective: every exchange runs inside the kernel that needs it, over the symmetric
                     buffer of `fused_exchange(n, ...)` (the one `ShardedPlan(exchange="fused")` of the same n
                     uses; a plain device buffer on one rank).  An evaluation is the candidate, [Aksel: the
                     local median], the rule's `*_peers` call (`bz_pairdist_reuse_peers`: distances with
                     reuse, exchange, scoring and reduce; `bz_rowdist_peers`), and `bz_search_score_peers`
                     (the share's exchange and the transition): 2 exchanges per evaluation for a distance
                     rule, 1 for the others, each advancing the buffer's epoch by one.  The same bits as
                     "nccl".  The calls that share the buffer must be issued on one stream, in the same
                     order on every rank.  The eager calls pass the epoch by value; `graph()` captures
                     the `_next` calls, which take it from the buffer;
            "auto"   "fused" on 2..16 ranks with symmetric memory, the CUDA engine and (Multi-Krum, Bulyan,
                     brute) 16-byte aligned rows on every rank, else "nccl"; the ranks agree on it
                     (`choose_search_exchange`).
  wide:     False (default): the limits of `engine.search_max_rows` (64 rows against a distance rule), as before.
            True: krum, bulyan, aksel and cge up to MAX_N_DISTANCE rows (`search_rows`; brute stays at MAX_N).
            Above MAX_N rows phase A is `bz_distance_partial_reuse` (krum, bulyan: star passes of the candidate
            after the first evaluation, over two pass tables the search owns), `bz_distance_partial` (aksel after
            its local median; cge at the first evaluation, then `bz_rowshare_star` of libbyzagg_star.so, which reads
            the candidate row alone), phases B and C `bz_distance_select` and `bz_distance_reduce`; "fused" exchanges
            the block in `bz_distance_select_peers` (libbyzagg_peers.so, rows of any alignment), 2 exchanges per
            evaluation; "auto" resolves to "nccl" there (`search_exchange`).  A stand-in backend gets
            `wide=True` as a keyword after its 10 arguments.
  many:     False (default): the coordinate-wise rules up to MAX_N_COORDINATE rows, as before.  True: up to MAX_N_MANY
            (`search_rows`); above MAX_N_COORDINATE rows the rule is `bz_coordinate_many` (`engine._coordinate_call`),
            and the trace, the factor and `byz` on one rank are those of `engine.LineSearch(..., many=True)`.  The
            fused exchange carries only the score's share for these rules, at any n.  The distance rules raise
            ValueError.  A stand-in backend gets `many=True` as a keyword after its 10 arguments.
  `graph()` captures the whole search in a CUDA graph, as `engine.LineSearch.graph()` does: "fused" on any
  number of ranks, "nccl" on one rank (no collective).  Like a search, `graph()` and every replay are
  collective: every rank issues them at the same point of its stream order. """
  def __init__(self, gar, grad_honests, f_real, f_decl, grad_avg, grad_att, evals, negative=False, kind="identical",
               group=None, backend=None, exchange="auto", wide=False, many=False):
    if gar not in _engine._SEARCH_RULES:
      raise KeyError(f"unknown aggregation rule {gar!r}")
    if many and gar not in COORDINATE_WISE:
      raise ValueError(f"many=True takes the coordinate-wise rules {list(COORDINATE_WISE)}, not {gar!r}")
    if kind not in _engine._SEARCH_KINDS:
      raise ValueError(f"unknown attack kind {kind!r}, expected one of {sorted(_engine._SEARCH_KINDS)}")
    if int(evals) < 1:
      raise ValueError(f"evals = {evals}, expected evals >= 1")
    self.gar, self.evals, self.group = gar, int(evals), group
    self.world = dist.get_world_size(group) if dist.is_initialized() else 1
    honest = list(grad_honests)
    pair = gar in ("krum", "bulyan", "brute")
    self.exchange = search_exchange(gar, len(honest) + int(f_real), exchange, not pair or rows_aligned(honest),
                                    _symmetric_memory_importable(), backend is None, group, wide)
    make = _SearchShard if backend is None else backend.search_shard
    self._backend, self._graph = backend, None
    extra = dict({"wide": True} if wide else {}, **({"many": True} if many else {}))
    self._shard = make(gar, honest, f_real, f_decl, grad_avg, grad_att, self.evals, negative, kind, self.world, **extra)
    self.byz, self.record = self._shard.byz, self._shard.record
    if self.exchange == "fused":
      n, device = len(honest) + int(f_real), self._shard.device
      self._fx = FusedExchange.local(n, device) if self.world == 1 else fused_exchange(n, device, group)
      self._shard.fuse(self._fx)
  def evaluate(self, k):
    """ Evaluation k up to its first exchange: the candidate row, then the rule's phase A (distance rules:
    returns this rank's partial block) or the whole rule and the score share (coordinate-wise rules:
    returns the share). """
    return self._shard.evaluate(k)
  def conclude(self, blocks):
    """ Distance rules, between the two exchanges: phases B and C on the [R, ...] gathered blocks, then the
    score share (returned). """
    return self._shard.conclude(blocks)
  def step(self, k, scores):
    """ The transition of evaluation k from the [R] gathered score shares. """
    self._shard.step(k, scores)
  def finish(self):
    """ The Byzantine gradient's shard for the chosen factor (returned). """
    return self._shard.finish()
  def _exchange(self, gathered, part):
    if self.world > 1:
      dist.all_gather_into_tensor(gathered.view(-1), part, group=self.group)
    return gathered
  def graph(self):
    """ Capture the whole search (every evaluation and the last candidate) in a CUDA graph, after one eager
    search (the warm-up), and return `replay`: a callable that launches it and returns `byz`.  With "fused",
    each replay advances the exchange's epoch by the graph's exchanges: 2 per evaluation for a distance rule,
    1 for the others.  CUDA engine only. """
    if self._backend is not None:
      raise ValueError("ShardedLineSearch.graph() needs the CUDA engine, not a stand-in backend")
    _capturable(self.exchange, self.world, "ShardedLineSearch")
    shard = self._shard
    fx = self._fx if self.exchange == "fused" else None
    return _engine._capture(self, shard.device, lambda call: self._issue(call, captured=True), lambda: self.byz, fx,
                            (2 if shard.distance else 1) * self.evals)
  def __call__(self):
    return self._issue()
  def _issue(self, call=_engine._call, captured=False):
    """ The search's stages and exchanges, every C call of the CUDA engine's stages through `call(fn, args)`;
    `captured`: the fused exchanges take their epochs from the buffer. """
    shard = self._shard
    shard.call = call
    try:
      if self.exchange == "fused":
        fx = self._fx
        def epoch():
          return None if captured else fx._reserve(1)
        for k in range(self.evals):
          shard.evaluate_fused(k, epoch() if shard.distance else None)
          shard.score_fused(k, epoch())
        return self.finish()
      for k in range(self.evals):
        part = self.evaluate(k)
        if shard.distance:
          part = self.conclude(self._exchange(shard.blocks, part))
        self.step(k, self._exchange(shard.scores, part))
      return self.finish()
    finally:
      shard.call = _engine._call
  def result(self):
    """ (factor, trace) from ONE device->host read, the same on every rank; with `engine.config.strict_status`,
    a failed evaluation of Bulyan or brute raises what the plain call raises. """
    return _engine._search_outcome(self.record, self.evals)

def line_search(gar, grad_honests, f_real, f_decl, grad_avg, grad_att, evals, negative=False, kind="identical", group=None,
                exchange="auto", wide=False, many=False):
  """ `engine.line_search` on a d-sharded trainer (see `ShardedLineSearch`, its `wide` for krum, bulyan, aksel
  and cge above MAX_N rows and its `many` for the coordinate-wise rules above MAX_N_COORDINATE rows): returns (factor,
  this rank's shard of the Byzantine gradient), the factor the same Python float on every rank. """
  search = ShardedLineSearch(gar, grad_honests, f_real, f_decl, grad_avg, grad_att, evals, negative, kind, group,
                             exchange=exchange, wide=wide, many=many)
  byz = search()
  factor, _ = search.result()
  return factor, byz

def choose_anticge_exchange(exchange, symmetric, group=None):
  """ The exchange of `ShardedAntiCGE`, the same on every rank of `group`: the local fact `symmetric` (symmetric
  memory can be set up here) is agreed on with one all-reduce (MIN), as in `choose_search_exchange`.  "auto" takes
  "fused" on 2 to 16 ranks that all have symmetric memory, else "nccl" (one rank keeps the collective stages).  An
  explicit "fused" needs symmetric memory on every one of at most 16 ranks unless there is one rank (its buffer is
  then plain device memory); otherwise it raises on every rank.  Rows may have any alignment.  Returns "fused" or
  "nccl". """
  if exchange not in SEARCH_EXCHANGES:
    raise ValueError(f"unknown exchange {exchange!r}")
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  (symmetric,) = map(bool, _agree([int(bool(symmetric))], group))
  fusable = world == 1 or (symmetric and world <= _lib.MAX_PEERS)
  if exchange == "auto":
    return "fused" if world > 1 and fusable else "nccl"
  if exchange == "fused" and not fusable:
    raise ValueError(f"the fused exchange of the attack against CGE needs symmetric memory on every one of at most "
                     f"{_lib.MAX_PEERS} ranks")
  return exchange

class ShardedAntiCGE:
  """ `engine.AntiCGE` on a d-sharded trainer: this rank's columns of the honest rows in, this rank's shard of the
  attack row out, with the same order and the same factor on every rank.  Its stages, each enqueue only:
    `norms()`            phase A of CGE (`bz_distance_partial`): this shard's sums of squares, nh doubles;
    `sum(blocks)`        on the R gathered blocks [R, nh]: phase B of CGE (`bz_distance_select`, the order), then
                         `bz_anticge_partial` (this shard of the unscaled attack); returns its fp64 sum of squares;
    `scale(partials)`    on the R gathered sums [R]: `bz_anticge_scale`; returns [byz] * f_real.
  The caller all-gathers between the stages.  f_real > f_decl needs no exchange: `engine.AntiCGE` fills the shard
  with NaN.

  `attack()` issues a whole step on the current stream, with no host read, and returns [byz] * f_real:
  exchange: "nccl"   the stages and the two all-gathers (of nh doubles, then of one double per rank);
            "fused"  one `bz_anticge_peers` call over the buffer of `fused_exchange(nh, ...)` (a plain device buffer
                     on one rank): both exchanges run inside its kernels, over peer memory, and each call advances
                     the buffer's `epoch` by two.  The same bits as "nccl".  The buffer may be shared with a
                     `ShardedPlan` or `ShardedLineSearch` of the same n, whose calls are then issued on the same
                     stream, in the same order on every rank;
            "auto"   "fused" on 2..16 ranks that all have symmetric memory, else "nccl"; the ranks agree on it
                     (`choose_anticge_exchange`).
  `graph()` captures a step in a CUDA graph: "fused" on any number of ranks (the captured call takes its epoch from
  the buffer, `bz_anticge_peers_next`), "nccl" on one rank.  Like a call, `graph()` and every replay are collective:
  every rank issues them at the same point of its stream order. """
  def __init__(self, grad_honests, f_decl, f_real, group=None, exchange="auto"):
    honest = list(grad_honests)
    if not _engine.anticge_takes(honest, f_decl, f_real):
      raise ValueError(f"the attack against CGE takes 1..{_lib.MAX_N_DISTANCE} honest rows, 1 <= f_decl <= nh and "
                       f"f_real >= 0, got nh = {len(honest)}, f_decl = {f_decl!r}, f_real = {f_real!r}")
    prep = self._prep = _engine._prepare_device(honest, "the sharded attack takes CUDA tensors", limit=_lib.MAX_N_DISTANCE)
    self.rows, self.f_decl, self.f_real, self.device = honest, f_decl, f_real, prep.device
    self.group = group
    self.world = dist.get_world_size(group) if dist.is_initialized() else 1
    lib = _lib.lib()
    self._dws = torch.empty(int(lib.bz_distance_workspace_bytes(prep.n)), dtype=torch.uint8, device=prep.device)
    self._ws = torch.empty(int(lib.bz_anticge_workspace_bytes(prep.n)), dtype=torch.uint8, device=prep.device)
    self.part = torch.empty(prep.n, dtype=torch.float64, device=prep.device)
    self.order = torch.empty(prep.n, dtype=torch.int32, device=prep.device)
    self.partial = torch.empty(1, dtype=torch.float64, device=prep.device)
    self.byz = torch.empty(prep.d, dtype=torch.float32, device=prep.device)
    self._graph, self.status = None, None
    self.exchange = choose_anticge_exchange(exchange, _symmetric_memory_importable(), group)
    if self.exchange == "fused":
      self.status = torch.zeros(1, dtype=torch.int32, device=prep.device)
      self._fuse(FusedExchange.local(prep.n, prep.device) if self.world == 1 else fused_exchange(prep.n, prep.device, group))
  def _fuse(self, fx):
    """ Run the fused exchanges over `fx`, a FusedExchange of n = nh. """
    p, lib = self._prep, _lib.lib()
    self._fx = fx
    self._exchanging = _Exchanging(lib.bz_anticge_peers, lib.bz_anticge_peers_next,
                                   (p.ptrs, p.n, self.f_decl, self.f_real, p.d, self.byz.data_ptr(), self.status.data_ptr(),
                                    fx.rank, fx.world), (self._ws.data_ptr(), self._ws.numel()), both=True)
  def _stream(self):
    return torch.cuda.current_stream(self.device).cuda_stream
  def norms(self):
    p, lib = self._prep, _lib.lib()
    _engine._run(self.device, lib.bz_distance_partial, (_engine._SEARCH_RULES["cge"], p.ptrs, p.n, None, p.d, self.part.data_ptr(),
                                                        self._dws.data_ptr(), self._dws.numel(), self._stream()))
    return self.part
  def sum(self, blocks):
    p, lib = self._prep, _lib.lib()
    self._blocks = blocks = blocks.contiguous()
    _engine._run(self.device, lib.bz_distance_select, (_engine._SEARCH_RULES["cge"], blocks.data_ptr(), blocks.shape[0], p.n, 0, 0, 0,
                                                       self.order.data_ptr(), None, self._stream()))
    _engine._run(self.device, lib.bz_anticge_partial, (p.ptrs, p.n, self.f_decl, self.order.data_ptr(), p.d, self.byz.data_ptr(),
                                                       self.partial.data_ptr(), self._ws.data_ptr(), self._ws.numel(), self._stream()))
    return self.partial
  def scale(self, partials):
    p, lib = self._prep, _lib.lib()
    self._partials = partials = partials.contiguous()
    _engine._run(self.device, lib.bz_anticge_scale, (self._blocks.data_ptr(), self.order.data_ptr(), partials.data_ptr(),
                                                     partials.numel(), p.n, self.f_decl, p.d, self.byz.data_ptr(), self._stream()))
    return [self.byz] * self.f_real
  def __call__(self):
    """ One step on the current stream of the rows' device; returns [byz] * f_real. """
    with _engine._on(self.device):
      self._issue()
    return [self.byz] * self.f_real
  def graph(self):
    """ Capture a step in a CUDA graph (after one eager step, the warm-up) and return `replay`: a callable that
    launches it and returns [byz] * f_real.  With "fused", each replay advances the exchange's epoch by two. """
    _capturable(self.exchange, self.world, "ShardedAntiCGE")
    fx = self._fx if self.exchange == "fused" else None
    return _engine._capture(self, self.device, lambda call: self._issue(call, captured=True), lambda: [self.byz] * self.f_real,
                            fx, 0 if self.f_real > self.f_decl else 2)
  def _issue(self, call=_engine._call, captured=False):
    """ A step's calls, the fused one and the NaN fill's through `call(fn, args)`; `captured`: the fused call takes
    its epoch from the buffer. """
    if self.exchange == "fused":
      fx = self._fx
      # two exchanges, none for the NaN fill of f_real > f_decl
      fn, args = fx._args(self._exchanging, None if captured else fx._reserve(0 if self.f_real > self.f_decl else 2))
      call(fn, args + (self._stream(),))
      return
    if self.f_real > self.f_decl:
      p = self._prep
      call(_lib.lib().bz_anticge, (p.ptrs, p.n, self.f_decl, self.f_real, p.d, self.byz.data_ptr(), self._ws.data_ptr(),
                                   self._ws.numel(), self._stream()))
      return
    blocks = _gather(self.norms(), self.group)
    self.scale(_gather(self.sum(blocks), self.group).reshape(-1))

def anticge(grad_honests, f_decl, f_real, group=None, exchange="auto"):
  """ attacks/anticge.py's attack on a d-sharded trainer (see `ShardedAntiCGE`): every rank passes its columns of
  the nh honest gradients and gets its shard of the attack row, f_real times, aliased.  "nccl": two all-gathers, of
  nh and of one double per rank; "fused": one call that exchanges over peer memory; no host read. """
  if isinstance(f_real, int) and isinstance(f_decl, int) and f_real > f_decl:
    return _engine.anticge(grad_honests, f_decl, f_real)
  return ShardedAntiCGE(grad_honests, f_decl, f_real, group, exchange)()

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
  if gar in COORDINATE_WISE:
    out = getattr(be, gar)(gradients) if gar in ("average", "median") else getattr(be, gar)(gradients, f)
    return (out, None) if return_selection else out
  out, sel = _phases(be, gar, gradients, f, m, mode, group, False)
  return (out, sel) if return_selection else out

def compute_avg_dev_max(samples, group=None, backend=None, many=False):
  """ `tools.compute_avg_dev_max` (tools/pytorch.py:97-125) over d-sharded samples: every rank
  passes its columns of the n samples and gets its shard of the average plus the GLOBAL scalars.
  One pass over the local shard (`avg_dev_max_async`), then ONE all-gather of 2 + n doubles; the
  sums of squares are added in rank order and the maxima compared, so every rank returns
  bitwise the same three numbers.  With `many`, up to MAX_N_MANY samples (`avg_dev_max_many_async`).
  Returns:
    (this rank's shard of the average or None, norm of the average, norm standard deviation,
     max |coordinate| of the average)
  """
  be = backend or _engine
  n = len(samples)
  if n == 0:
    return None, math.nan, math.nan, math.nan
  avg, stats = be.avg_dev_max_many_async(samples) if many else be.avg_dev_max_async(samples)
  gathered = _gather(stats, group).tolist()            # [R][2 + n]; the only synchronisation
  return _engine._study_tuple(avg, _engine._merge_ranks(gathered, (1,)), n)      # fp32 overflow rule after the sums

def study_step(grad_sampleds, grad_honests, grad_attacks, grad_defense, pasts, momentum, group=None, backend=None, many=False):
  """ `engine.study_step` (attack.py:846-866) over d-sharded vectors: every rank passes its columns
  and gets its shards of the three averages plus the GLOBAL scalars, bitwise the same on every rank.
  One `engine.study_partials` pass over the local shard, then ONE all-gather of its fp64 vector
  (14 + ns + nh + na + P doubles with P past gradients, 9 + ns + nh + P without attack gradients: the
  same length on every rank), then `engine.study_finish`: sums added in rank order, maxima merged, and
  only then the fp32 overflow rule, the norms and the fp32 divisions.  A rank whose shard is empty
  (d < R) still joins.
  Against one GPU the averages are bit-identical per coordinate; the scalars differ only by the
  order of the fp64 additions (the R per-rank blocks added in rank order).
  Args:
    grad_sampleds, grad_honests, grad_attacks, grad_defense  This rank's columns of them
    pasts     Iterable of (this rank's shard of a past sampled average, its GLOBAL norm), most recent
              first: (`sampled_grad_avg`, `sampled_norm_avg`) of an earlier call
    momentum  args.momentum
    group     Process group (default: the world)
    backend   Provider of `avg_dev_max_async` and `rowdots_async` (default: the CUDA engine), and of
              `avg_dev_max_many_async` with `many`
    many      Lists of up to MAX_N_MANY gradients (`avg_dev_max_many_async`) instead of MAX_N_COORDINATE
  Returns:
    dict with the reference's variable names
  """
  partials = _engine.study_partials(grad_sampleds, grad_honests, grad_attacks, grad_defense, pasts, backend=backend, many=many)
  return _engine.study_finish(partials, _gather(partials.vector, group).tolist(), momentum)    # the only synchronisation

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
