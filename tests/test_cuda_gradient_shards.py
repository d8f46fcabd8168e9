# coding: utf-8
"""GPU tests of gradient delivery to the d-sharded path (`bz_gradient_scatter`, `engine.gradient_scatter`,
`engine.momentum_rows`, `sharded.GradientShards`), with R ranks emulated on ONE GPU: every rank's slot is
a plain device buffer, as peer memory would be.

The bar is `GradientStack.push` on the same gradient: every slot must hold the matching columns of its
sampled row bit for bit (the clip scale comes from the same device norm), nothing outside a slot may
be written (canary fill), and the momentum placed on the shards must equal the stack's honest rows."""

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CANARY = 0x7FBADBAD                       # a signalling NaN no computation produces
PAD = 64                                  # floats of canary on each side of a slot (keeps it 256-byte aligned)

def _bits(t):
  return t.contiguous().view(torch.int32)

def _same_bits(a, b):
  return torch.equal(_bits(a), _bits(b))

def _grad(d, kind, seed):
  """ One gradient: "none" / "loose" / "tight" clips (no clip, one that does not trigger, one that
  does), "overflow" (the squared norm overflows fp32: scale 0), "nan" (one NaN entry: no scaling),
  "offset" (a view starting 4 bytes into its buffer). """
  gen = torch.Generator(device=DEV).manual_seed(seed)
  if kind == "offset":
    return torch.randn(d + 1, device=DEV, generator=gen)[1:], 2.0
  g = torch.randn(d, device=DEV, generator=gen)
  if kind == "overflow":
    return g * 1e30, 1.0
  if kind == "nan":
    g[d // 2] = float("nan")
    return g, 2.0
  return g, {"none": None, "loose": 1e30, "tight": 2.0}[kind]

KINDS = ("none", "loose", "tight", "overflow", "nan", "offset")

@pytest.mark.parametrize("d", [1, 3, 5, 9, 4099, 8 * 1021 + 3, 1_310_922])     # 5, 9: empty last shards with d >= R
@pytest.mark.parametrize("R", [1, 2, 3, 4, 8, 16])
def test_scatter_slots_are_the_stack_row_sliced(R, d):
  from byzantinemomentum_b200 import engine, sharded
  stack = engine.GradientStack(1, d, DEV)
  bounds = [sharded.shard_bounds(d, R, r) for r in range(R)]
  bufs = [torch.empty(hi - lo + 2 * PAD, device=DEV) for lo, hi in bounds]
  slots = [b[PAD:PAD + hi - lo] for b, (lo, hi) in zip(bufs, bounds)]
  for k, kind in enumerate(KINDS):
    grad, clip = _grad(d, kind, 1000 * R + k)
    want = stack.push(0, grad, clip=clip).clone()
    for b in bufs:
      _bits(b).fill_(CANARY)
    engine.gradient_scatter(grad, clip, slots)
    torch.cuda.synchronize()
    if kind == "overflow":
      assert torch.count_nonzero(want) == 0                        # norm +inf: scale 0, a zero row
    for r, ((lo, hi), b, s) in enumerate(zip(bounds, bufs, slots)):
      where = f"R={R} d={d} {kind} rank {r}"
      assert _same_bits(s, want[lo:hi]), where
      assert torch.all(_bits(b[:PAD]) == CANARY) and torch.all(_bits(b[PAD + hi - lo:]) == CANARY), f"{where}: wrote outside its slot"

@pytest.mark.parametrize("d", [4099, 1_310_922])
@pytest.mark.parametrize("placement", ["worker", "server"])
def test_momentum_on_the_shards_is_the_stack_honest_row(d, placement):
  from byzantinemomentum_b200 import engine, sharded
  R, n, mu, damp = 3, 4, 0.9, 0.1
  gen = torch.Generator(device=DEV).manual_seed(d)
  stack = engine.GradientStack(n, d, DEV)
  bounds = [sharded.shard_bounds(d, R, r) for r in range(R)]
  rows = [engine._row_buffer(n, hi - lo, DEV) for lo, hi in bounds]
  moms = [torch.randn(d, device=DEV, generator=gen) for _ in range(n)]
  server = torch.randn(d, device=DEV, generator=gen)
  mom_shards = [[m[lo:hi].clone() for m in moms] for lo, hi in bounds]
  server_shards = [server[lo:hi].clone() for lo, hi in bounds]
  honest_shards = [engine._row_buffer(n, hi - lo, DEV) for lo, hi in bounds]
  for step in range(2):
    for i in range(n):
      grad = torch.randn(d, device=DEV, generator=gen) * (0.5 + i)
      clip = 30.0 if i % 2 else None
      kw = dict(worker_momentum=moms[i]) if placement == "worker" else dict(server_momentum=server)
      stack.push(i, grad, clip=clip, mu=mu, dampening=damp, **kw)
      engine.gradient_scatter(grad, clip, [rows[r][i, :hi - lo] for r, (lo, hi) in enumerate(bounds)])
    for r, (lo, hi) in enumerate(bounds):                          # each owner: its n rows in one launch
      mine = [rows[r][i, :hi - lo] for i in range(n)]
      if placement == "worker":
        engine.momentum_rows(mine, mu, damp, momentums=mom_shards[r])
      else:
        engine.momentum_rows(mine, mu, damp, server=server_shards[r], honests=[honest_shards[r][i, :hi - lo] for i in range(n)])
    want = moms if placement == "worker" else stack.honest()
    for r, (lo, hi) in enumerate(bounds):
      for i in range(n):
        got = mom_shards[r][i] if placement == "worker" else honest_shards[r][i, :hi - lo]
        assert _same_bits(got, want[i][lo:hi]), (placement, d, step, r, i)
        assert _same_bits(rows[r][i, :hi - lo], stack.sampled()[i][lo:hi]), (placement, d, step, r, i)

@pytest.mark.parametrize("placement", ["worker", "server"])
def test_momentum_rows_beyond_one_launch(placement):
  """ More rows than one launch takes (64): `engine.momentum_rows` splits them, with the stack's bits. """
  from byzantinemomentum_b200 import engine
  n, d, mu, damp = 70, 1031, 0.9, 0.25
  gen = torch.Generator(device=DEV).manual_seed(70)
  stack = engine.GradientStack(n, d, DEV)
  moms = [torch.randn(d, device=DEV, generator=gen) for _ in range(n)]
  server = torch.randn(d, device=DEV, generator=gen)
  # every third vector starts 4 bytes into its buffer: those rows take the one-at-a-time path
  shifted = lambda v, i: torch.empty(d + 1, device=DEV)[1:].copy_(v) if i % 3 == 2 else v.clone()
  mine = [shifted(m, i) for i, m in enumerate(moms)]
  for i in range(n):
    kw = dict(worker_momentum=moms[i]) if placement == "worker" else dict(server_momentum=server)
    stack.push(i, torch.randn(d, device=DEV, generator=gen), clip=20.0, mu=mu, dampening=damp, **kw)
  versions = [m._version for m in mine]
  if placement == "worker":
    got = engine.momentum_rows(stack.sampled(), mu, damp, momentums=mine)
    want = moms
  else:
    want = stack.honest()
    got = engine.momentum_rows(stack.sampled(), mu, damp, server=server, honests=[shifted(torch.empty(d, device=DEV), i) for i in range(n)])
    assert all(_same_bits(a, b) for a, b in zip(got, want))
    got = engine.momentum_rows(stack.sampled(), mu, damp, server=shifted(server, 2), honests=[torch.empty(d, device=DEV) for _ in range(n)])
  assert all(_same_bits(a, b) for a, b in zip(got, want))
  if placement == "worker":
    assert all(m._version > v for m, v in zip(mine, versions))

class _PlainSymmetricRows:
  """ The symmetric buffer of a world of one: a plain device buffer, its own only peer. """
  def __init__(self, shape, device, group):
    self.buffer = torch.empty(shape, dtype=torch.float32, device=device)
    self.peers = [self.buffer]
    self.barriers = 0
  def barrier(self):
    self.barriers += 1

@pytest.mark.parametrize("exchange", ["p2p", "collective"])
def test_gradient_shards_on_one_rank(exchange, monkeypatch):
  """ `GradientShards` without a process group on both exchanges: several steps (both p2p slots),
  the rows bumped on every delivery, and the stack's rows bit for bit. """
  from byzantinemomentum_b200 import engine, sharded
  monkeypatch.setattr(sharded, "_symmetric_rows", _PlainSymmetricRows)
  monkeypatch.setattr(sharded, "_symmetric_memory_importable", lambda: True)
  n, d, mu, damp = 5, 50_021, 0.9, 0.0
  gen = torch.Generator(device=DEV).manual_seed(11)
  shards = sharded.GradientShards(n, d, DEV, exchange=exchange)
  assert shards.exchange == exchange and shards.slots == (2 if exchange == "p2p" else 1)
  stack = engine.GradientStack(n, d, DEV)
  moms = [torch.randn(d, device=DEV, generator=gen) for _ in range(n - 1)]
  mom_shards = [m.clone() for m in moms]
  seen = []
  for step in range(5):
    versions = [r._version for r in shards.rows(step % shards.slots)]
    for i in shards.workers():
      grad = torch.randn(d, device=DEV, generator=gen) * (1 + i)
      clip = 100.0 if i % 2 else None
      stack.push(i, grad, clip=clip, worker_momentum=moms[i] if i < n - 1 else None, mu=mu, dampening=damp)
      shards.push(i, grad, clip=clip)
    rows = shards.deliver()
    assert shards.slot == step % shards.slots and shards.step == step + 1
    assert all(r._version > v for r, v in zip(rows, versions))
    assert all(r.data_ptr() % 256 == 0 for r in rows)
    seen.append(rows[0].data_ptr())
    for i in range(n):
      assert _same_bits(rows[i], stack.sampled()[i]), (exchange, step, i)
    honest = shards.honests_worker(mom_shards, mu, damp)
    for i in range(n - 1):
      assert _same_bits(honest[i], moms[i]), (exchange, step, i)
  assert len(set(seen)) == shards.slots
  if exchange == "p2p":
    assert shards._sym.barriers == 5
  with pytest.raises(ValueError):
    sharded.GradientShards(n, d, DEV, exchange="nccl")

def _emulated_delivery(n, d, R, grads, clip):
  """ Each emulated rank's [n, pitch] rows, filled by one scatter per gradient. """
  from byzantinemomentum_b200 import engine, sharded
  bounds = [sharded.shard_bounds(d, R, r) for r in range(R)]
  bufs = [engine._row_buffer(n, hi - lo, DEV) for lo, hi in bounds]
  for i, g in enumerate(grads):
    engine.gradient_scatter(g, clip, [bufs[r][i, :hi - lo] for r, (lo, hi) in enumerate(bounds)])
  return [[b[i, :hi - lo] for i in range(n)] for b, (lo, hi) in zip(bufs, bounds)]

@pytest.mark.parametrize("R", [2, 3, 8])
def test_rules_over_delivered_shards_give_the_single_gpu_result(R):
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine
  n, nb, f, d, clip = 25, 5, 5, 100_003, 400.0
  gen = torch.Generator(device=DEV).manual_seed(R)
  honest = [torch.randn(d, device=DEV, generator=gen) * (0.5 + i / 19) for i in range(n - nb)]
  byz = torch.stack(honest).mean(dim=0).mul(-1.1)
  grads = honest + [byz] * nb
  stack = engine.GradientStack(n, d, DEV)
  for i, g in enumerate(grads):
    stack.push(i, g, clip=clip)
  full = stack.sampled()
  shards = _emulated_delivery(n, d, R, grads, clip)
  for gar, kw in (("average", {}), ("median", {}), ("trmean", dict(f=f)), ("phocas", dict(f=f)), ("meamed", dict(f=f))):
    want = bz.Plan(gar, full, **kw)().clone()
    got = torch.cat([bz.Plan(gar, s, **kw)() for s in shards])
    assert _same_bits(got, want), (gar, R)
  m = n - f - 2
  parts = torch.stack([engine.pairdist_partial(s) for s in shards])
  order = engine.krum_select(parts, n, f)
  plan = bz.Plan("krum", full, f=f)
  want = plan().clone()
  assert order[:plan.selection.numel()].tolist() == plan.selection.tolist()
  assert _same_bits(torch.cat([engine.average_selected(s, order, m) for s in shards]), want), ("krum", R)
  order_b, status = engine.bulyan_select(parts, n, f, m)
  plan_b = bz.Plan("bulyan", full, f=f)
  plan_b()
  assert int(status.item()) == 0 and order_b.tolist() == plan_b.selection.tolist(), ("bulyan", R)
  got_b = torch.cat([engine.bulyan_reduce(s, f, m, order_b, status) for s in shards])
  assert _same_bits(got_b, plan_b.out), ("bulyan", R)
