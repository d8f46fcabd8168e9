# coding: utf-8
"""The study block (attack.py:846-866) over R column shards, the ranks emulated on one GPU: the device
half (`engine.study_partials`) on each shard, the host half (`engine.study_finish`) over the R partial
vectors in rank order — what `sharded.study_step` does with one all-gather in the middle.  Against
`engine.study_step` on the whole vectors: the averages are bit-identical, the scalars agree within
the bar of `tests/test_cuda_study_step.py` (they differ only by the order of the fp64 additions),
one shard is bit-identical, and the fp32 overflow rule applies after the cross-rank sum."""

import math

import pytest
import torch

from byzantinemomentum_b200 import engine, sharded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MOMENTUM = 0.9
FLT_MAX = 3.4028234663852886e38
AVERAGES = ("sampled_grad_avg", "honest_grad_avg", "attack_grad_avg")

def _rows(n, d, seed, scale=1.):
  gen = torch.Generator(device="cpu").manual_seed(seed)
  return [(torch.randn(d, generator=gen) * scale).to(DEV) for _ in range(n)]

def _inputs(ns, nh, na, npast, d, shared, seed=11):
  sampleds = _rows(ns, d, seed)
  honests = sampleds[:nh] if shared else _rows(nh, d, seed + 1)
  attacks = [a.mul(-2.) for a in _rows(na, d, seed + 2)]
  defense = _rows(1, d, seed + 3, 0.3)[0]
  pasts = [(g, g.norm().item()) for g in _rows(npast, d, seed + 4)]
  return sampleds, honests, attacks, defense, pasts

def _emulate(sampleds, honests, attacks, defense, pasts, R):
  """ Every rank's dict, and every rank's partial vector, for R shards (unaligned views on purpose). """
  d = defense.numel()
  partials = []
  for r in range(R):
    lo, hi = sharded.shard_bounds(d, R, r)
    cut = lambda rows: [g[lo:hi] for g in rows]
    shard_s = cut(sampleds)
    shard_h = shard_s[:len(honests)] if all(h is s for h, s in zip(honests, sampleds)) else cut(honests)
    partials.append(engine.study_partials(shard_s, shard_h, cut(attacks), defense[lo:hi], [(g[lo:hi], norm) for g, norm in pasts]))
  vectors = [p.vector.tolist() for p in partials]
  return [engine.study_finish(p, vectors, MOMENTUM) for p in partials], vectors

def _same(a, b):
  return a == b or (math.isnan(a) and math.isnan(b))

def _bits(v):
  return v.view(torch.int32)

def _scalars(result):
  return {k: v for k, v in result.items() if k not in AVERAGES}

def _check(inputs, R):
  want = engine.study_step(*inputs, MOMENTUM)
  ranks, vectors = _emulate(*inputs, R)
  for res in ranks[1:]:                              # bitwise the same scalars on every rank
    for key, val in _scalars(ranks[0]).items():
      assert _same(res[key], val), (R, key, res[key], val)
  for key in AVERAGES:                               # per coordinate: the shards concatenate to the whole
    if want[key] is None:
      assert all(res[key] is None for res in ranks)
    else:
      assert torch.equal(_bits(torch.cat([res[key] for res in ranks])), _bits(want[key])), (R, key)
  got = _scalars(ranks[0])
  assert set(got) == set(_scalars(want))
  for key, ref in _scalars(want).items():
    val = got[key]
    if R == 1:
      assert _same(val, ref) and math.copysign(1., val) == math.copysign(1., ref), (key, val, ref)
    elif math.isnan(ref) or math.isinf(ref):
      assert _same(val, ref), (R, key, val, ref)
    else:
      assert abs(val - ref) <= 2e-5 * abs(ref) + 3e-6, (R, key, val, ref)
  return ranks, vectors

@pytest.mark.parametrize("R", [1, 2, 3, 8, 16])
@pytest.mark.parametrize("ns,nh,na,npast,d,shared", [(8, 8, 3, 2, 79510, True), (8, 6, 0, 3, 4099, False), (5, 5, 2, 70, 10007, False),
                                                     (3, 2, 1, 1, 5, False), (25, 25, 0, 25, 1310922, True)])
def test_shards_compose_to_the_one_gpu_study_step(ns, nh, na, npast, d, shared, R):
  ranks, vectors = _check(_inputs(ns, nh, na, npast, d, shared), R)
  assert len({len(v) for v in vectors}) == 1         # one layout on every rank, empty shards included (d = 5 < R)

def test_zero_vectors_and_a_nan_on_one_shard():
  d = 257
  zeros = [torch.zeros(d, device=DEV) for _ in range(3)]
  for R in (1, 2, 8):
    ranks, _ = _check((zeros, zeros, [], torch.zeros(d, device=DEV), []), R)
    assert ranks[0]["sampled_norm_avg"] == 0. and math.isnan(ranks[0]["cosin_splhon"]) and math.isnan(ranks[0]["cosin_sampled"])
  sampleds, honests, attacks, defense, pasts = _inputs(6, 6, 2, 2, 1001, False)
  sampleds[1][990] = float("nan")                    # in the last shard only
  for R in (2, 3, 8):
    ranks, _ = _check((sampleds, honests, attacks, defense, pasts), R)
    assert math.isnan(ranks[0]["sampled_norm_max"]) and math.isnan(ranks[0]["cosin_spldef"])

def test_overflow_applies_after_the_cross_rank_sum():
  """ Each shard's sum of squares stays below FLT_MAX / 2, the whole vector's passes 2 * FLT_MAX: the
  norms are +inf on every rank, as the reference's fp32 `norm()` of the whole vector is. """
  R, d = 8, 64
  big = torch.full((d,), 3.9e18, device=DEV)         # 64 * 3.9e18^2 = 9.7e38; per shard of 8: 1.2e38
  wiggle = _rows(4, d, 3, 1e16)
  sampleds = [big + w for w in wiggle]
  attacks = [big.neg()]
  defense = big.mul(1.01)
  inputs = (sampleds, sampleds[:3], attacks, defense, [(big, math.inf)])
  ranks, vectors = _check(inputs, R)
  for v in vectors:
    assert v[0] < FLT_MAX / 2                        # ||s_avg||^2 of the shard
  assert sum(v[0] for v in vectors) > 2 * FLT_MAX
  for res in ranks:
    for key in ("sampled_norm_avg", "honest_norm_avg", "attack_norm_avg", "defense_norm_avg"):
      assert res[key] == math.inf, key

def test_sharded_study_step_at_world_size_one_is_the_one_gpu_call():
  import torch.distributed as dist
  assert not dist.is_initialized()
  for case in [(8, 8, 3, 2, 79510, True), (8, 6, 0, 70, 4099, False), (1, 1, 1, 1, 33, True)]:
    inputs = _inputs(*case)
    want = engine.study_step(*inputs, MOMENTUM)
    got = sharded.study_step(*inputs, MOMENTUM)
    assert set(got) == set(want)
    for key, ref in want.items():
      if key in AVERAGES:
        assert (ref is None and got[key] is None) or torch.equal(_bits(got[key]), _bits(ref)), key
      else:
        assert _same(got[key], ref) and math.copysign(1., got[key]) == math.copysign(1., ref), (key, got[key], ref)
