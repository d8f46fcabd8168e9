# coding: utf-8
"""GPU tests of the exchange fused into the distance pass of Krum and Bulyan (`bz_krum_peers`,
`bz_bulyan_peers`, `ShardedPlan(exchange="fused")`), with R ranks emulated on ONE GPU.

Each emulated rank owns a buffer with the `sharded.FusedExchange` layout (two slots of n*n doubles,
then 16 uint32 flags per slot) and its own 16-byte aligned copy of its `shard_bounds` columns; the
Byzantine row stays one tensor repeated on every rank, as in the reference.  A step is emulated
without two grids ever running at once:
  1. every rank's block is published alone (`nranks = 1`: the call waits only on the flag it has
     just raised itself, in a scratch word);
  2. each rank r in turn makes the real call (`nranks = R`) after the test has set every flag that
     call waits on; the call must raise its flag on every rank, rewrite its slot with the same bits,
     sum the R slots in rank order, score, and reduce its shard.
Every rank must derive the same order; the orders, blocks and outputs are checked against the
phases of the d-sharded path (`bz_pairdist_partial`, `bz_*_select`, `bz_average_selected` /
`bz_bulyan_reduce`) and the oracle on the full rows.  Steps alternate slots over an epoch wrap, with
the rows changed in place between steps, so a wrong slot or epoch reads the previous step's blocks."""

import ctypes

import numpy as np
import pytest

import parity
from conftest import canon_alias
from oracle import byzoracle as orc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FLT_MAX = float(np.finfo(np.float32).max)
U32 = 1 << 32
EPOCHS = (0xFFFFFFFE, 0xFFFFFFFF, 0, 1)      # four steps across the wrap, slot = epoch % 2
FLAG_WORDS = 16

def _lib():
  from byzantinemomentum_b200 import _lib
  return _lib.lib()

def _ptrs(addrs):
  return (ctypes.c_void_p * len(addrs))(*addrs)

def _rows_ptrs(rows):
  return _ptrs([r.data_ptr() for r in rows])

def _stream():
  return torch.cuda.current_stream().cuda_stream

def _s32(v):
  """ uint32 flag value as the int32 the flag tensors hold. """
  v %= U32
  return v - U32 if v >= 1 << 31 else v

def _bits(t):
  """ Bit pattern of a float tensor (NaN payloads included) for bitwise comparisons. """
  return t.contiguous().view(torch.int64 if t.dtype == torch.float64 else torch.int32)

def _same_bits(a, b):
  return torch.equal(_bits(a), _bits(b))

def _sm_count():
  return torch.cuda.get_device_properties(0).multi_processor_count

class Ranks:
  """ R emulated ranks, each with its own buffer in the `FusedExchange` layout. """
  def __init__(self, R, n):
    self.R, self.n = R, n
    self.buf = [torch.zeros(2 * n * n + FLAG_WORDS, dtype=torch.float64, device=DEV) for _ in range(R)]
  def slot(self, p, s):
    nn = self.n * self.n
    return self.buf[p][s * nn:(s + 1) * nn]
  def flags(self, p, s):
    return self.buf[p][2 * self.n * self.n:].view(torch.int32)[FLAG_WORDS * s:FLAG_WORDS * (s + 1)]
  def tables(self, s):
    return (_ptrs([self.slot(p, s).data_ptr() for p in range(self.R)]),
            _ptrs([self.flags(p, s).data_ptr() for p in range(self.R)]))

class Call:
  """ Output, order, status and workspace of one rule call on d columns. """
  def __init__(self, rule, n, f, m, d):
    self.rule, self.n, self.f, self.m, self.d = rule, n, f, m, d
    self.out = torch.empty(max(d, 1), device=DEV)[:d]
    self.order = torch.empty(n, dtype=torch.int32, device=DEV)
    self.status = torch.empty(1, dtype=torch.int32, device=DEV)
    self.nbytes = _lib().bz_workspace_bytes(64)
    self.ws = torch.empty(self.nbytes, dtype=torch.uint8, device=DEV)
  def reset(self):
    self.out.fill_(float("nan"))
    self.order.fill_(-1)
    self.status.fill_(7)
  def peers(self, rows, rank, nranks, blocks, flags, epoch):
    lib = _lib()
    fn = lib.bz_krum_peers if self.rule == "krum" else lib.bz_bulyan_peers
    self.reset()
    rc = fn(_rows_ptrs(rows), self.n, self.f, self.m, self.d, self.out.data_ptr(), self.order.data_ptr(), self.status.data_ptr(),
            rank, nranks, blocks, flags, epoch, self.ws.data_ptr(), self.nbytes, _stream())
    torch.cuda.synchronize()
    return rc
  def single(self, rows):
    """ The single-GPU rule on the same rows. """
    lib = _lib()
    self.reset()
    if self.rule == "krum":
      rc = lib.bz_krum(_rows_ptrs(rows), self.n, self.f, self.m, self.d, self.out.data_ptr(), self.order.data_ptr(),
                       self.ws.data_ptr(), self.nbytes, _stream())
    else:
      rc = lib.bz_bulyan(_rows_ptrs(rows), self.n, self.f, self.m, self.d, self.out.data_ptr(), self.order.data_ptr(),
                         self.status.data_ptr(), self.ws.data_ptr(), self.nbytes, _stream())
    torch.cuda.synchronize()
    return rc

def _full_rows(n, nb, d, seed, kind, R):
  """ n rows on the device, the last nb one tensor.  kinds: "iid" (rows of distinct spread, the
  Byzantine row far out), "nan" (the Byzantine row holds a NaN in the shard of rank seed % R only),
  "nanrows" (the Byzantine row is all NaN), "overflow" (see test_overflow_applies_to_the_summed_table). """
  gen = torch.Generator(device=DEV).manual_seed(seed)
  nh = n - nb
  if kind == "overflow":
    idx = torch.arange(n, device=DEV)
    sigma = torch.where(idx % 8 == 7, 3.0 + 0.5 * (1. - idx / n), 0.8 * (1. - 0.01 * (idx % 7)))
    mu = torch.randn(d, device=DEV, generator=gen)
    x = (mu[None, :] + sigma[:, None] * torch.randn(n, d, device=DEV, generator=gen)) * float(np.sqrt(1e38 / d))
    return [x[i].clone() for i in range(n)]
  mu = torch.randn(d, device=DEV, generator=gen)
  honest = [mu + (0.5 + i / max(nh - 1, 1)) * torch.randn(d, device=DEV, generator=gen) for i in range(nh)]
  if nb == 0:
    return honest
  byz = torch.stack(honest).mean(dim=0) * -1.1
  if kind == "nan":
    from byzantinemomentum_b200.sharded import shard_bounds
    k = seed % R
    lo, hi = shard_bounds(d, R, k)
    while hi <= lo:                                   # an empty shard cannot hold it: the next one
      k = (k + 1) % R
      lo, hi = shard_bounds(d, R, k)
    byz[lo + (hi - lo) // 2] = float("nan")
  elif kind == "nanrows":
    byz.fill_(float("nan"))
  return honest + [byz] * nb

def _unique(rows):
  """ Distinct row tensors in first-occurrence order (the order the library dedupes them in). """
  seen, out = set(), []
  for r in rows:
    if r.data_ptr() not in seen:
      seen.add(r.data_ptr())
      out.append(r)
  return out

def _make_shards(full, R):
  """ Per rank, its columns of every row in a separate 16-byte aligned tensor (an empty shard too
  gets its own address), aliased rows still one tensor. """
  from byzantinemomentum_b200.sharded import shard_bounds
  d = full[0].numel()
  shards = []
  for r in range(R):
    lo, hi = shard_bounds(d, R, r)
    copies = {}
    rows = []
    for x in full:
      c = copies.get(id(x))
      if c is None:
        c = copies[id(x)] = torch.empty(max(hi - lo, 1), device=DEV)[:hi - lo]
      rows.append(c)
    assert all(c.data_ptr() % 16 == 0 for c in rows)
    shards.append(rows)
  _refill(shards, full)
  return shards

def _refill(shards, full):
  """ New row contents, same tensors (momentum buffers are updated in place between steps). """
  from byzantinemomentum_b200.sharded import shard_bounds
  d, R = full[0].numel(), len(shards)
  for r, rows in enumerate(shards):
    lo, hi = shard_bounds(d, R, r)
    for c, x in zip(rows, full):
      c.copy_(x[lo:hi])

def _pairdist(rows):
  part = torch.empty(len(rows), len(rows), dtype=torch.float64, device=DEV)
  lib = _lib()
  nbytes = lib.bz_workspace_bytes(64)
  ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
  rc = lib.bz_pairdist_partial(_rows_ptrs(rows), len(rows), rows[0].numel(), part.data_ptr(), ws.data_ptr(), nbytes, _stream())
  assert rc == 0, lib.bz_last_error()
  return part

def _phase_b(rule, parts, n, f, m):
  """ Order (and status) of the phase-B kernel over the R gathered blocks. """
  lib = _lib()
  order = torch.full((n,), -1, dtype=torch.int32, device=DEV)
  status = torch.full((1,), 7, dtype=torch.int32, device=DEV)
  if rule == "krum":
    rc = lib.bz_krum_select(parts.data_ptr(), parts.shape[0], n, f, order.data_ptr(), _stream())
    status.zero_()
  else:
    rc = lib.bz_bulyan_select(parts.data_ptr(), parts.shape[0], n, f, m, order.data_ptr(), status.data_ptr(), _stream())
  assert rc == 0, lib.bz_last_error()
  return order.cpu().tolist(), int(status.item())

def _phase_c(rule, rows, n, f, m, order, status):
  """ Phase C on one shard with the given order: what the fused call's reduce pass must give. """
  lib = _lib()
  d = rows[0].numel()
  out = torch.full((d,), float("nan"), device=DEV)
  if rule == "krum":
    rc = lib.bz_average_selected(_rows_ptrs(rows), n, order.data_ptr(), m, 1, float(m), None, d, out.data_ptr(), _stream())
  else:
    rc = lib.bz_bulyan_reduce(_rows_ptrs(rows), n, f, m, order.data_ptr(), status.data_ptr(), d, out.data_ptr(), _stream())
  assert rc == 0, lib.bz_last_error()
  return out

def _check_block(block, rows, tag):
  """ A published block: n x n over the rows.  Entry (i, j), i < j, is the pair of their distinct
  rows with the bits of the phase-A pass over the distinct rows, or, when both are one tensor, its
  alias flag (0, or NaN when the shard holds a NaN / inf); every other entry is 0. """
  n = len(rows)
  uniq = _unique(rows)
  u = len(uniq)
  a = torch.tensor([next(k for k, x in enumerate(uniq) if x.data_ptr() == r.data_ptr()) for r in rows], device=DEV)
  lo, hi = torch.minimum(a[:, None], a[None, :]), torch.maximum(a[:, None], a[None, :])
  pu = _pairdist(uniq) if rows[0].numel() > 0 else torch.zeros(u, u, dtype=torch.float64, device=DEV)
  flag = torch.tensor([0. if torch.isfinite(x).all() else float("nan") for x in uniq], dtype=torch.float64, device=DEV)
  upper = torch.ones(n, n, dtype=torch.bool, device=DEV).triu(1)
  alias = lo == hi
  want = torch.where(upper, torch.where(alias, flag[lo], pu[lo, hi]), torch.zeros_like(pu[lo, hi]))
  table = block.view(n, n)
  assert _same_bits(table[upper & ~alias], want[upper & ~alias]), f"{tag}: published pairs differ from phase A"
  assert torch.equal(table.isnan(), want.isnan()), f"{tag}: alias flags"
  assert torch.equal(table.nan_to_num(), want.nan_to_num()), f"{tag}: entries outside the pairs"

def _run(rule, n, f, nb, R, d, kind="iid", m=None, epochs=EPOCHS, seed=0, whole_order=False):
  from byzantinemomentum_b200.sharded import shard_bounds
  m_max = n - f - 2
  m = m_max if m is None else m
  nh = n - nb
  bounds = [shard_bounds(d, R, r) for r in range(R)]
  ranks = Ranks(R, n)
  scratch = torch.zeros(FLAG_WORDS, dtype=torch.int32, device=DEV)
  calls = [Call(rule, n, f, m, hi - lo) for lo, hi in bounds]
  use_oracle = n * d <= 20_000_000
  full = _full_rows(n, nb, d, seed, kind, R)
  shards = _make_shards(full, R)
  prev = None
  for step, epoch in enumerate(epochs):
    tag = f"{rule} n={n} f={f} R={R} d={d} {kind} epoch={epoch:#x}"
    if step > 0:
      full = _full_rows(n, nb, d, seed + 7919 * step, kind, R)
      _refill(shards, full)
    s = epoch % 2
    blocks, flags = ranks.tables(s)
    # 1. every rank's block alone
    pub = []
    for p in range(R):
      scratch.zero_()
      rc = calls[p].peers(shards[p], 0, 1, _ptrs([ranks.slot(p, s).data_ptr()]), _ptrs([scratch.data_ptr()]), epoch)
      assert rc == 0, _lib().bz_last_error()
      assert int(scratch[0].item()) == _s32(epoch) and not scratch[1:].any(), f"{tag}: rank {p} alone did not signal itself"
      pub.append(ranks.slot(p, s).clone())
      _check_block(pub[p], shards[p], f"{tag} rank {p}")
      if bounds[p][1] == bounds[p][0]:
        assert not pub[p].any(), f"{tag}: rank {p} has no columns and must publish zeros"
    if prev is not None:
      assert all(not _same_bits(ranks.slot(p, 1 - s), pub[p]) for p in range(R) if bounds[p][1] > bounds[p][0]), \
        f"{tag}: the previous step's blocks are not told apart from this one's"
    other = [ranks.slot(p, 1 - s).clone() for p in range(R)]
    # 2. the real call of every rank, its flags set beforehand
    got = []
    for r in range(R):
      for p in range(R):
        ranks.flags(p, s).fill_(_s32(epoch - 2))                    # the slot's previous use
      preset = [_s32(epoch - 2)] * FLAG_WORDS
      for t in range(R):
        if t != r:
          preset[t] = _s32(epoch + (1 if t == (r + 1) % R else 0))  # one peer is already a step further
          ranks.flags(r, s)[t] = preset[t]
      rc = calls[r].peers(shards[r], r, R, blocks, flags, epoch)
      assert rc == 0, _lib().bz_last_error()
      for p in range(R):
        fl = ranks.flags(p, s).cpu().tolist()
        assert fl[r] == _s32(epoch), f"{tag}: rank {r} did not signal rank {p}"
        for t in range(FLAG_WORDS):
          if t != r:
            assert fl[t] == (preset[t] if p == r else _s32(epoch - 2)), f"{tag}: rank {r} wrote flag {t} of rank {p}"
      assert _same_bits(ranks.slot(r, s), pub[r]), f"{tag}: rank {r} published other bits than alone"
      got.append((calls[r].order.clone(), int(calls[r].status.item()), calls[r].out.clone()))
    for p in range(R):
      assert _same_bits(ranks.slot(p, 1 - s), other[p]), f"{tag}: the other slot of rank {p} was written"
    # 3. one order everywhere, the phases' order and outputs
    order0 = got[0][0]
    for r, (order, status, _) in enumerate(got):
      assert torch.equal(order, order0), f"{tag}: rank {r} derived another order"
      assert status in (0, 2), f"{tag}: rank {r} status {status}"
      assert status == got[0][1]
    status = got[0][1]
    order = order0.cpu().tolist()
    assert sorted(order) == list(range(n)), f"{tag}: order {order}"
    parts = torch.stack([_pairdist(rows) for rows in shards])
    order_b, status_b = _phase_b(rule, parts, n, f, m)
    k = m if rule == "krum" else m_max
    assert canon_alias(order[:k], nh) == canon_alias(order_b[:k], nh), f"{tag}: fused order {order} vs phase B {order_b}"
    assert status == status_b, f"{tag}: status {status} vs phase B {status_b}"
    for r in range(R):
      if bounds[r][1] > bounds[r][0]:
        want = _phase_c(rule, shards[r], n, f, m, got[r][0], calls[r].status)
        assert _same_bits(got[r][2], want), f"{tag}: rank {r} output differs from phase C"
    out = torch.cat([g[2] for g in got])
    # 4. against the oracle on the full rows (the single-GPU rule where the oracle would be slow)
    if step == 0 or not use_oracle:
      one = Call(rule, n, f, m, d)
      slot1 = torch.zeros(n * n, dtype=torch.float64, device=DEV)
      assert one.peers(full, 0, 1, _ptrs([slot1.data_ptr()]), _ptrs([scratch.data_ptr()]), epoch) == 0
      fused1 = (one.order.clone(), int(one.status.item()), one.out.clone())
      assert one.single(full) == 0, _lib().bz_last_error()
      assert torch.equal(fused1[0], one.order), f"{tag}: nranks = 1 order differs from bz_{rule}"
      assert _same_bits(fused1[2], one.out), f"{tag}: nranks = 1 output differs from bz_{rule}"
      if rule == "bulyan":
        assert fused1[1] == int(one.status.item())
      if not use_oracle:
        assert canon_alias(order[:k], nh) == canon_alias(one.order.cpu().tolist()[:k], nh), tag
        assert _same_bits(out, one.out), f"{tag}: concatenated shards differ from the single-GPU rule"
    if use_oracle:
      host = [x.cpu().numpy() for x in full]
      if rule == "krum":
        ref, info = orc.krum(host, f, m=m, return_info=True)
        assert status == 0
        assert canon_alias(order[:m], nh) == canon_alias(info["selection"], nh), f"{tag}: order vs oracle"
        if whole_order:
          assert order == info["order"], f"{tag}: whole order vs oracle (ties included)"
        parity.assert_bit_exact(out.cpu().numpy(), ref, tag)
      else:
        try:
          ref, info = orc.bulyan(host, f, m=m, return_info=True)
        except TypeError:
          assert status == 2, f"{tag}: the oracle finds the stack degenerate"
          assert torch.isnan(out).all(), f"{tag}: a degenerate stack gives NaN"
        else:
          assert status == 0, tag
          assert canon_alias(order[:m_max], nh) == canon_alias(info["order"][:m_max], nh), f"{tag}: order vs oracle"
          parity.assert_close_scaled(out.cpu().numpy(), ref, parity.column_scale(info["stage1"]), tag, exempt=info["ambiguous"])
    prev = got
  return shards

# Launch shapes with a fused tail (ring_shape in k2_ring.cu, counted in DISTINCT rows u): u <= 15 six
# warps, 16-25 twelve warps in one CTA, 26-35 clusters of 12-warp CTAs, > 35 clusters of 16-warp CTAs.
# Shards: ragged, exact multiples of the 512 / 256-column tile, 1-3 columns, and many tiles per walker.
KRUM = [  # n, f, nb, R, d, kind, m
  (7, 1, 1, 2, 4099, "iid", None),          # u = 7
  (11, 2, 2, 1, 1001, "iid", None),         # u = 10, one rank
  (11, 2, 2, 3, 3 * 1024, "iid", None),     # u = 10, every shard 2 x 512 columns
  (15, 3, 3, 16, 10007, "iid", 1),          # u = 13, m = 1
  (25, 5, 5, 8, 20011, "nan", None),        # u = 21, NaN in one shard
  (33, 7, 0, 3, 6007, "iid", None),         # u = 33, clusters of 12-warp CTAs
  (51, 12, 12, 16, 16 * 256 * 7, "iid", None),   # u = 40, 16-warp clusters, 7 tiles of 256 per shard
  (64, 15, 0, 2, 5, "iid", None),           # u = 64, shards of 3 and 2 columns
  (64, 15, 15, 3, 30011, "nan", 3),         # u = 50
]
BULYAN = [  # n, f, nb, R, d, kind, m
  (11, 2, 2, 2, 4001, "iid", None),         # K4 compiled for (11, 2)
  (25, 5, 5, 8, 10007, "nan", None),        # K4 compiled for (25, 5)
  (51, 12, 12, 3, 3001, "iid", None),       # K4 compiled for (51, 12)
  (15, 3, 3, 16, 1031, "iid", None),        # n = 4f + 3
  (33, 5, 0, 2, 4 * 512, "iid", 10),        # m < n - f - 2: the generic K4
  (64, 15, 0, 1, 777, "iid", None),         # one rank
  (11, 2, 5, 3, 2003, "nanrows", None),     # more NaN rows than f: degenerate (status 2, NaN output)
  (7, 1, 1, 2, 3, "iid", None),             # shards of 2 and 1 columns
]

@pytest.mark.parametrize("n,f,nb,R,d,kind,m", KRUM)
def test_fused_krum(n, f, nb, R, d, kind, m):
  _run("krum", n, f, nb, R, d, kind, m, seed=31 * n + R)

@pytest.mark.parametrize("n,f,nb,R,d,kind,m", BULYAN)
def test_fused_bulyan(n, f, nb, R, d, kind, m):
  _run("bulyan", n, f, nb, R, d, kind, m, seed=37 * n + R)

def test_fused_exchange_at_full_ring_depth():
  """ Every walker of every rank goes round its stage ring and flushes several times (the rule of
  test_cuda_depth.py, with the SM count), two steps; checked against the single-GPU rules. """
  n, f, nb, R = 25, 5, 5, 2
  d = 2 * 1_250_003
  per_walker = (d // R // 512) // (2 * _sm_count())
  assert per_walker >= 2 * 4 + 1, f"{per_walker} full tiles per walker: the test no longer reaches ring depth"
  for rule in ("krum", "bulyan"):
    _run(rule, n, f, nb, R, d, "iid", epochs=EPOCHS[1:3], seed=5)
    torch.cuda.empty_cache()

def test_overflow_applies_to_the_summed_table():
  """ Rows s (mu + sigma_i z_i) as in test_cuda_extremes.py, over 16 shards: every shard's sum of
  squares stays below FLT_MAX / 2, while the pairs with a large row add up past 2 FLT_MAX across the
  ranks.  Those distances are +inf on every rank, and the +inf scores tie in index order, as in the
  oracle; small pairs stay below FLT_MAX / 2. """
  n, f, R, d = 17, 3, 16, 300_007
  full = _full_rows(n, 0, d, 17, "overflow", R)
  shards = _make_shards(full, R)
  parts = torch.stack([_pairdist(rows) for rows in shards]).cpu().numpy()
  iu = np.triu_indices(n, 1)
  assert (parts[:, iu[0], iu[1]] < FLT_MAX / 2).all()
  total = parts.sum(axis=0)[iu]
  assert ((total < FLT_MAX / 2) | (total > 2 * FLT_MAX)).all() and (total > 2 * FLT_MAX).any()
  _, scores = orc.krum_order(orc.pairwise_distances([x.cpu().numpy() for x in full]), f)
  assert np.isinf(scores).any() and sum(np.isfinite(scores)) >= n - f - 2
  del full, shards
  _run("krum", n, f, 0, R, d, "overflow", epochs=EPOCHS[:2], seed=17, whole_order=True)

def test_rank_with_an_empty_shard_joins_the_exchange():
  """ d = 9 over 4 ranks: rank 3 has no columns.  It must still publish (a zero block), raise its
  flag on every rank and derive the same order; the other ranks' shards give the oracle. """
  from byzantinemomentum_b200.sharded import shard_bounds
  assert shard_bounds(9, 4, 3) == (9, 9)
  for rule in ("krum", "bulyan"):
    _run(rule, 11, 2, 2, 4, 9, "iid", seed=9)

def test_unaligned_rows_are_unsupported():
  lib = _lib()
  n, f, d = 11, 2, 4001
  base = [torch.randn(d + 1, device=DEV) for _ in range(n)]
  rows = [b[1:] for b in base]
  block = torch.zeros(n * n, dtype=torch.float64, device=DEV)
  scratch = torch.zeros(FLAG_WORDS, dtype=torch.int32, device=DEV)
  for rule in ("krum", "bulyan"):
    call = Call(rule, n, f, n - f - 2, d)
    assert call.peers(rows, 0, 1, _ptrs([block.data_ptr()]), _ptrs([scratch.data_ptr()]), 5) == -2
    assert b"16-byte aligned" in lib.bz_last_error()
    assert not scratch.any() and not block.any()

@pytest.mark.parametrize("gar,kw", [("krum", dict(f=5)), ("krum", dict(f=5, m=3)), ("bulyan", dict(f=5))])
def test_sharded_plan_fused_on_one_rank(gar, kw):
  """ `ShardedPlan(exchange="fused")` on one rank, its symmetric buffer a plain device buffer: every
  call advances the epoch and alternates the slot, and must give the single-GPU rule bit for bit,
  also after in-place updates of the rows. """
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import sharded
  n, nb, d = 25, 5, 20011
  full = _full_rows(n, nb, d, 91, "iid", 1)
  device = full[0].device
  fx = sharded.FusedExchange.__new__(sharded.FusedExchange)
  fx.n, fx.device, fx.group = n, device, None
  fx.world, fx.rank, fx.epoch = 1, 0, 0
  fx.buffer = torch.zeros(2 * n * n + FLAG_WORDS, dtype=torch.float64, device=device)
  fx.peer_base = [fx.buffer.data_ptr()]
  key = (n, device.index, id(None))
  assert key not in sharded._fused
  sharded._fused[key] = fx
  try:
    plan = sharded.ShardedPlan(gar, full, exchange="fused", **kw)
    assert plan.exchange == "fused" and plan._fx is fx
    for step in range(6):
      got = plan().clone()
      want = bz.gars[gar](gradients=full, **kw)
      assert _same_bits(got, want), f"{gar} {kw}: call {step}"
      assert int(plan.status.item()) == 0
      if gar == "krum":
        assert plan.selection.cpu().tolist() == bz.last_selection()
      assert fx.epoch == step + 1
      flags = fx.buffer[2 * n * n:].view(torch.int32)
      assert int(flags[FLAG_WORDS * (fx.epoch % 2)].item()) == fx.epoch
      full[step % (n - nb)].mul_(-1.5)              # content changes, pointers do not
      full[-1].add_(0.25)
  finally:
    del sharded._fused[key]
