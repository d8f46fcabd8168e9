# coding: utf-8
"""The attack against CGE on the H100 (`bz_anticge`, `engine.AntiCGE`, `sharded.ShardedAntiCGE`): the order and the
unscaled sum bit for bit against the oracle and `bz_cge`, the row within the stated bound of the reference's
statements run on the same GPU, every recorded case of `tests/golden/anticge/`, misaligned rows, a CUDA graph,
and one and three ranks of the d-sharded path emulated on one GPU."""

import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import byzoracle as orc
import anticge_oracle as aorc
from test_anticge_abi import GOLDEN, RTOL, close, goldens

DEV = "cuda"

def _bits(t):
  return t.detach().cpu().contiguous().view(torch.int32)

def reference(grad_honests, f_decl, f_real):
  """ attacks/anticge.py:59-78, restated with the same torch statements. """
  if f_real > f_decl:
    byz = torch.empty_like(grad_honests[0])
    byz.copy_(torch.tensor((math.nan,), dtype=byz.dtype))
    return [byz] * f_real
  def byznorm(grad):
    norm = grad.norm().item()
    return norm if math.isfinite(norm) else math.inf
  normed = sorted(((byznorm(grad), grad) for grad in grad_honests), key=lambda pair: pair[0])
  maxpos = len(grad_honests) - f_decl
  maxnorm = math.nextafter(normed[maxpos][0], 0)
  attack = normed[0][1].clone().detach_()
  for _, grad in normed[:maxpos]:
    attack.add_(grad)
  attnorm = attack.norm().item()
  if attnorm > 0:
    attack.mul_(-maxnorm / attnorm)
  return [attack] * f_real

def _rows(nh, d, seed, views=False):
  gen = torch.Generator().manual_seed(seed)
  stack = torch.randn(nh, d, generator=gen) * (0.5 + torch.rand(nh, 1, generator=gen))
  if not views:
    return [r.to(DEV) for r in stack]
  buf = torch.zeros(nh, d + 5, device=DEV)
  return [buf[i, 1:d + 1].copy_(stack[i]) for i in range(nh)]        # 4-byte, not 16-byte, aligned

def _order(attack):
  return attack._ws[:4 * len(attack.rows)].view(torch.int32).cpu().tolist()

@pytest.mark.parametrize("path", goldens())
def test_goldens(path):
  import byzantinemomentum_b200 as bz
  z = np.load(path)
  rows = [torch.from_numpy(r.copy()).to(DEV) for r in z["rows"]]
  f_decl, f_real = int(z["f_decl"]), int(z["f_real"])
  attack = bz.engine.AntiCGE(rows, f_decl, f_real)
  out = attack()
  torch.cuda.synchronize()
  assert len(out) == f_real == int(z["count"]) and all(o is out[0] for o in out)
  if f_real == 0:
    return
  got = out[0].cpu().numpy()
  if f_real > f_decl:
    assert np.array_equal(got.view(np.uint32), np.full(got.size, 0x7fc00000, np.uint32))
    return
  assert _order(attack) == z["order"].tolist()
  assert close(got, z["out"]), np.nanmax(np.abs(got - z["out"]) / np.abs(z["out"]))

@pytest.mark.parametrize("nh,d,f_decl", [(1, 1000, 1), (7, 4099, 2), (25, 1 << 20, 5), (25, 3000, 25), (64, 70001, 16),
                                         (65, 5003, 16), (100, 65536, 24), (128, 9001, 31), (128, 2000, 1)])
def test_order_sum_and_row_against_the_oracle_bz_cge_and_the_reference(nh, d, f_decl):
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import sharded
  rows = _rows(nh, d, 100 + nh)
  host = [r.cpu().numpy() for r in rows]
  want, info = aorc.anticge(host, f_decl, f_decl, return_info=True)
  attack = bz.engine.AntiCGE(rows, f_decl, f_decl)
  got = attack()[0].cpu().numpy()
  assert _order(attack) == info["order"]
  if nh <= 64:
    _, selection = bz.engine.cge(rows, 0)
    assert selection.cpu().tolist() == info["order"]
  # the unscaled sum, from the same K10 through the one-rank d-sharded stages
  one = sharded.ShardedAntiCGE(rows, f_decl, f_decl)
  one.sum(one.norms().unsqueeze(0))
  assert one.order.cpu().tolist() == info["order"]
  assert np.array_equal(one.byz.cpu().numpy().view(np.uint32), info["presum"].view(np.uint32))
  assert close(got, want[0]), np.max(np.abs(got - want[0]) / np.abs(want[0]))
  ref = reference(rows, f_decl, f_decl)[0].cpu().numpy()
  assert close(got, ref), np.max(np.abs(got - ref) / np.abs(ref))

def test_misaligned_views_graph_replay_and_aliasing():
  import byzantinemomentum_b200 as bz
  rows, views = _rows(25, 100003, 7), _rows(25, 100003, 7, views=True)
  assert all(v.data_ptr() % 16 != 0 for v in views)
  plain = bz.engine.AntiCGE(rows, 5, 4)
  first = plain()[0].clone()
  out = bz.engine.anticge(views, 5, 4)
  assert len(out) == 4 and all(o is out[0] for o in out)
  assert torch.equal(_bits(out[0]), _bits(first))
  replay = plain.graph()                                  # captured: the call reads nothing back on the host
  plain.byz.zero_()
  out = replay()
  torch.cuda.synchronize()
  assert len(out) == 4 and out[0] is plain.byz and torch.equal(_bits(out[0]), _bits(first))
  fill = bz.engine.AntiCGE(rows, 3, 4).graph()()
  assert torch.equal(_bits(fill[0]), torch.full((100003,), 0x7fc00000, dtype=torch.int32))

def _shards(full, R):
  from byzantinemomentum_b200 import sharded
  d = full[0].numel()
  return [[v[lo:hi] for v in full] for lo, hi in (sharded.shard_bounds(d, R, r) for r in range(R))]

@pytest.mark.parametrize("R", [1, 3])
@pytest.mark.parametrize("nh,f_decl", [(25, 5), (100, 24)])
def test_emulated_ranks_agree_and_match_one_gpu(R, nh, f_decl):
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import sharded
  d = 300007
  rows = _rows(nh, d, 11 + R)
  single = bz.engine.anticge(rows, f_decl, 2)[0].cpu().numpy()
  inst = [sharded.ShardedAntiCGE(cols, f_decl, 2) for cols in _shards(rows, R)]
  blocks = torch.stack([a.norms() for a in inst])
  partials = torch.cat([a.sum(blocks) for a in inst])
  pre = [a.byz.clone() for a in inst]
  outs = [a.scale(partials) for a in inst]
  torch.cuda.synchronize()
  assert all(len(o) == 2 and o[0] is o[1] for o in outs)
  assert all(torch.equal(a.order, inst[0].order) for a in inst)
  # one factor, the same bits on every rank: fl32(-maxnorm / attnorm) from the gathered blocks and partials
  key = orc.fp32_norm(orc.sum_parts(blocks.cpu().numpy()))[inst[0].order[nh - f_decl].item()]
  key = float(key) if math.isfinite(key) else math.inf
  attnorm = float(orc.fp32_norm(orc.sum_parts(partials.cpu().numpy())))
  factor = torch.tensor(-math.nextafter(key, 0) / attnorm, dtype=torch.float32).to(DEV)
  for p, o in zip(pre, outs):
    assert torch.equal(_bits(o[0]), _bits(p * factor))
  assert close(torch.cat([o[0] for o in outs]).cpu().numpy(), single)
  if R == 1:                                              # the driver with its exchanges (one rank: no collective)
    assert torch.equal(_bits(sharded.anticge(rows, f_decl, 2)[0]), _bits(outs[0][0]))
