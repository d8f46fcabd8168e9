# coding: utf-8
"""GPU parity: distance reuse across calls (SURVEY.md §8(f) row 1).

The attacks' line search (attacks/identical.py:68-77, `tools.line_maximize`) evaluates the rule up to
16 times per step on the SAME honest tensors plus one new Byzantine tensor repeated f times.  With
`engine.config.reuse_distances` (default on) Multi-Krum / Bulyan / brute keep the table of squared
distances of their last call and compute only the pairs of the new rows.  The bar: every evaluation
bit-identical — output AND selection — to the same call with reuse switched off."""

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"

def _honest(n_h, d, seed):
  gen = torch.Generator(device=DEV).manual_seed(seed)
  mu = torch.randn(d, device=DEV, generator=gen)
  return [mu + (0.5 + i / max(n_h - 1, 1)) * torch.randn(d, device=DEV, generator=gen) for i in range(n_h)]

def _attack(honest, factor):
  avg = torch.stack(honest).mean(dim=0)
  return avg.mul(-factor)                         # a NEW tensor per evaluation, like grad_avg + factor * grad_att

def _plain(bz, gar, rows, **kw):
  from byzantinemomentum_b200 import engine
  engine.config.reuse_distances = False
  try:
    out = bz.gars[gar](gradients=rows, **kw)
    sel = bz.last_selection()
  finally:
    engine.config.reuse_distances = True
  return out, sel

@pytest.mark.parametrize("gar,n,nb,f,d", [("krum", 25, 5, 5, 40_013), ("bulyan", 25, 5, 5, 40_013), ("brute", 11, 3, 3, 40_013),
                                          ("krum", 51, 12, 12, 20_011), ("bulyan", 51, 12, 12, 20_011), ("krum", 33, 6, 6, 30_011),
                                          ("krum", 25, 5, 5, 1_310_922)])
def test_line_search_evaluations_are_bit_identical_with_and_without_reuse(gar, n, nb, f, d):
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine
  honest = _honest(n - nb, d, 5)
  before = engine.pair_cache_stats()
  keep = []
  for k, factor in enumerate((1.1, 0.3, 7.0, 1.0, 0.0, 2.5, 1.5, 1.75, 1.6, 1.55, 30.0, 1.58, 1.57, 1.575, 1.5725, 1.57125)):
    byz = _attack(honest, factor)
    keep.append(byz)                              # keep the tensors alive: a freed one could be re-allocated at the same address
    rows = honest + [byz] * nb
    got = bz.gars[gar](gradients=rows, f=f)
    sel = bz.last_selection()
    want, want_sel = _plain(bz, gar, rows, f=f)
    assert torch.equal(got, want), (gar, k, factor)
    if gar != "bulyan":
      assert sel == want_sel, (gar, k)
    # the attack then edits the RESULT in place (identical.py:75) — never an input
    got.sub_(honest[0])
  after = engine.pair_cache_stats()
  assert after["star"] - before["star"] == 15, (before, after)      # first call fills the table, 15 reuse it
  assert after["full"] - before["full"] == 1

def test_reuse_follows_in_place_updates_and_replacements():
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine
  n, nb, f, d = 25, 5, 5, 30_011
  honest = _honest(n - nb, d, 6)
  byz = _attack(honest, 1.1)
  rows = honest + [byz] * nb
  bz.gars["krum"](gradients=rows, f=f)
  s0 = engine.pair_cache_stats()
  # an honest row modified in place: its version changed -> it is a new row (2 new with the attack)
  honest[3].mul_(1.5)
  rows = honest + [_attack(honest, 0.7)] * nb
  got = bz.gars["krum"](gradients=rows, f=f)
  want, _ = _plain(bz, "krum", rows, f=f)
  assert torch.equal(got, want)
  s1 = engine.pair_cache_stats()
  assert s1["star"] - s0["star"] == 1
  # six rows replaced: more than a star pass handles -> full pass, same result
  fresh = _honest(6, d, 7)
  rows = fresh + honest[6:] + [rows[-1]] * nb
  got = bz.gars["krum"](gradients=rows, f=f)
  want, _ = _plain(bz, "krum", rows, f=f)
  assert torch.equal(got, want)
  s2 = engine.pair_cache_stats()
  assert s2["full"] - s1["full"] == 1 and s2["star"] == s1["star"]
  # the very same list again: nothing is new -> full pass (no star task to run), still equal
  assert torch.equal(bz.gars["krum"](gradients=rows, f=f), want)
  # two DISTINCT new rows, not aliased
  rows2 = rows[:-nb] + [_attack(honest, 0.2), _attack(honest, 0.4)] + [rows[-1]] * (nb - 2)
  got = bz.gars["bulyan"](gradients=rows2, f=f)
  want, _ = _plain(bz, "bulyan", rows2, f=f)
  assert torch.equal(got, want)

def test_reuse_with_non_finite_attack_rows_and_other_streams():
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine
  n, nb, f, d = 25, 5, 5, 30_011
  honest = _honest(n - nb, d, 8)
  bz.gars["krum"](gradients=honest + [_attack(honest, 1.1)] * nb, f=f)
  for poison in (float("nan"), float("inf"), -float("inf")):
    byz = _attack(honest, 1.3)
    byz[777] = poison
    rows = honest + [byz] * nb
    got = bz.gars["krum"](gradients=rows, f=f)
    sel = bz.last_selection()
    want, want_sel = _plain(bz, "krum", rows, f=f)
    assert torch.equal(got, want) and sel == want_sel
    assert all(i < n - nb for i in sel[:n - f - 2])       # the poisoned rows score +inf: never selected
  # another stream: the table of the default stream is not reused (no cross-stream ordering)
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  s0 = engine.pair_cache_stats()
  with torch.cuda.stream(side):
    rows = honest + [_attack(honest, 0.9)] * nb
    got = bz.gars["krum"](gradients=rows, f=f)
  side.synchronize()
  assert engine.pair_cache_stats()["star"] == s0["star"]
  want, _ = _plain(bz, "krum", rows, f=f)
  assert torch.equal(got, want)

def test_reuse_takes_the_plain_pass_when_the_fused_tail_does_not_fit():
  """ 64 row entries over few distinct tensors: the fused scoring step works on a 64 x 64 table in the
  ring's shared memory.  Over 15 distinct rows (6-warp shape, 3 stages of 15 x 512 floats) it fits;
  over 10 (61,440 < 66,048 bytes) it does not, so the call with 1 new row among 10 takes no star pass:
  it must run the very kernels of the plain call, give its bits and write no table ("off"). """
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine
  from torch.profiler import ProfilerActivity, profile
  n, f, d = 64, 5, 30_011
  distinct = _honest(15, d, 9)
  before = engine.pair_cache_stats()
  bz.gars["krum"](gradients=(distinct * 5)[:n], f=f)
  s0 = engine.pair_cache_stats()
  assert s0["full"] - before["full"] == 1, (before, s0)      # the table of the 15 rows is there to reuse
  rows = ((distinct[:9] + [_attack(distinct, 0.8)]) * 7)[:n]

  def run(reuse):
    engine.config.reuse_distances = reuse
    try:
      with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = bz.gars["krum"](gradients=rows, f=f)
        torch.cuda.synchronize()
      sel = bz.last_selection()
    finally:
      engine.config.reuse_distances = True
    return out, sel, sorted({e.name for e in prof.events() if "bz::" in e.name})

  got, sel, got_kernels = run(True)
  s1 = engine.pair_cache_stats()
  want, want_sel, want_kernels = run(False)
  assert torch.equal(got, want) and sel == want_sel
  assert (s1["off"] - s0["off"], s1["star"] - s0["star"], s1["full"] - s0["full"]) == (1, 0, 0), (s0, s1)
  assert any("k2_ring" in k for k in want_kernels), want_kernels
  assert got_kernels == want_kernels, (got_kernels, want_kernels)
