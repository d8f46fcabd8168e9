# coding: utf-8
"""Host-side logic added in round 2 that needs no GPU: the measured choice of the host->device path, the
study-metrics memo, the identity/version keyed selection cache, the shard bounds of the sharded update."""

import gc
import importlib

import pytest

torch = pytest.importorskip("torch")

engine = importlib.import_module("byzantinemomentum_b200.engine")
gars = importlib.import_module("byzantinemomentum_b200.gars")
sharded = importlib.import_module("byzantinemomentum_b200.sharded")

def test_host_path_tries_every_candidate_three_times_then_keeps_the_fastest():
  path = engine._HostPath()
  seen = []
  costs = {"lanes": 3.0, "lane": 2.0, "pipeline": 2.5}
  for _ in range(9):
    mode = path.choose(True, False)
    seen.append(mode)
    path.record(True, False, mode, costs[mode])
  assert sorted(seen) == ["lane"] * 3 + ["lanes"] * 3 + ["pipeline"] * 3      # coordinate-wise rules: three candidates
  assert all(path.choose(True, False) == "lane" for _ in range(5))
  path.record(True, False, "lane", 99.)             # later samples do not reopen the decision
  assert path.choose(True, False) == "lane"
  seen = []
  for _ in range(9):                                # another kind of call is measured on its own, without the pipeline
    mode = path.choose(False, False)
    seen.append(mode)
    path.record(False, False, mode, 1.0)
  assert sorted(seen) == ["batch"] * 3 + ["lane"] * 3 + ["lanes"] * 3

def test_host_path_ranks_by_the_slower_of_the_late_samples():
  path = engine._HostPath()
  samples = {"lanes": [9., 3., 3.], "lane": [9., 2.6, 2.7], "pipeline": [9., 2.4, 3.5]}      # fast once, slow the next time
  for _ in range(9):
    mode = path.choose(True, False)
    path.record(True, False, mode, samples[mode].pop(0))
  assert path.choose(True, False) == "lane"

def test_forced_host_path_is_used_without_sampling():
  path = engine._HostPath()
  engine.forced_host_path = "pipeline"
  try:
    assert path.choose(True, False) == "pipeline"
    assert path.choose(False, False) == "lanes"     # not a candidate there: measured as usual
  finally:
    engine.forced_host_path = None

def test_study_metrics_memo_matches_only_the_same_unmodified_tensor_objects(monkeypatch):
  memo = engine._Memo()
  monkeypatch.setattr(engine, "_study_memo", memo)
  rows = [torch.arange(4.), torch.ones(4)]
  result = (torch.full((4,), 2.), 1., 2., 3.)
  assert memo.lookup("avg_dev_max", (), rows) is None
  memo.store("avg_dev_max", (), rows, result)
  hit = engine.compute_avg_dev_max(list(rows))       # another list object, the same tensors: served by the memo
  assert hit is not None and torch.equal(hit[0], result[0]) and hit[1:] == (1., 2., 3.)
  assert hit[0] is not result[0]                     # callers own the average they get
  assert memo.lookup("avg_dev_max", (), rows[:1]) is None
  assert memo.lookup("avg_dev_max", (), [rows[0], torch.ones(4)]) is None          # equal values, another object
  rows[1].add_(1.)                                   # in-place update bumps the version
  assert memo.lookup("avg_dev_max", (), rows) is None

def test_selection_cache_never_serves_a_recycled_identity():
  sel = gars._Selection()
  rows = [torch.zeros(3) for _ in range(4)]
  sel.store("krum", (1,), rows, "indices")
  assert sel.lookup("krum", (1,), rows) == "indices"
  assert sel.lookup("krum", (2,), rows) is None and sel.lookup("brute", (1,), rows) is None
  rows[2].mul_(2.)
  assert sel.lookup("krum", (1,), rows) is None
  sel.store("krum", (1,), rows, "again")
  del rows
  gc.collect()
  fresh = [torch.zeros(3) for _ in range(4)]         # may reuse ids / addresses of the dead tensors, at version 0
  assert sel.lookup("krum", (1,), fresh) is None
  assert sel.refs is None                            # a dead reference dropped the entry

def test_shard_bounds_cover_the_vector_without_overlap():
  for d, world in ((601, 2), (600, 2), (36_546_980, 8), (7, 8), (1, 4)):
    spans = [sharded.shard_bounds(d, world, r) for r in range(world)]
    assert spans[0][0] == 0 and spans[-1][1] == d
    assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
    assert all(lo <= hi for lo, hi in spans)

def test_study_step_bookkeeping_with_the_device_passes_replaced(monkeypatch):
  """ engine.study_step: which dot product lands in which cosine (attack.py:854-866), NaN columns without
  attack gradients, the curvature sum over the past gradients — checked on the CPU by replacing the two
  device passes (K6 and bz_rowdots) with plain tensor code.  (The CUDA passes themselves: -m gpu tests.) """
  import math
  def fake_avg_dev_max(samples):
    stack = torch.stack(samples).double()
    avg = stack.mean(dim=0)
    stats = torch.cat([avg.pow(2).sum().reshape(1), avg.abs().max().reshape(1), (stack - avg).pow(2).sum(dim=1)])
    return avg.float(), stats
  def fake_rowdots(center, rows):
    return torch.stack([torch.dot(r.double(), center.double()) for r in rows])
  monkeypatch.setattr(engine, "avg_dev_max_async", fake_avg_dev_max)
  monkeypatch.setattr(engine, "rowdots_async", fake_rowdots)
  gen = torch.Generator().manual_seed(5)
  d = 97
  for ns, nh, na, npast, shared in [(6, 6, 2, 2, True), (6, 4, 0, 3, False), (3, 3, 1, 0, False)]:
    sampleds = [torch.randn(d, generator=gen) for _ in range(ns)]
    honests = sampleds[:nh] if shared else [torch.randn(d, generator=gen) for _ in range(nh)]
    attacks = [torch.randn(d, generator=gen) for _ in range(na)]
    defense = torch.randn(d, generator=gen)
    pasts = [(g, g.norm().item()) for g in (torch.randn(d, generator=gen) for _ in range(npast))]
    got = engine.study_step(sampleds, honests, attacks, defense, pasts, 0.9)
    s_avg = torch.stack(sampleds).double().mean(dim=0)
    h_avg = torch.stack(honests).double().mean(dim=0)
    a_avg = torch.stack(attacks).double().mean(dim=0) if na else None
    dd = defense.double()
    cos = lambda a, b: math.nan if a is None or b is None else (torch.dot(a, b) / a.norm() / b.norm()).item()
    want = dict(cosin_splhon=cos(s_avg, h_avg), cosin_splatt=cos(s_avg, a_avg), cosin_spldef=cos(s_avg, dd),
                cosin_honatt=cos(h_avg, a_avg), cosin_hondef=cos(h_avg, dd), cosin_attdef=cos(a_avg, dd),
                sampled_norm_avg=s_avg.norm().item(), honest_norm_avg=h_avg.norm().item(), defense_norm_avg=dd.norm().item(),
                defense_norm_max=dd.abs().max().item(),
                sampled_norm_dev=math.sqrt(sum((g.double() - s_avg).pow(2).sum().item() for g in sampleds) / (ns - 1)),
                attack_norm_avg=a_avg.norm().item() if na else math.nan,
                attack_norm_dev=(math.sqrt(sum((g.double() - a_avg).pow(2).sum().item() for g in attacks) / (na - 1)) if na > 1 else math.nan))
    if npast:
      want["cosin_sampled"] = (torch.dot(s_avg, pasts[0][0].double()) / s_avg.norm() / pasts[0][1]).item()
      want["curv_sampled"] = 0.9 * sum(0.9 ** i * torch.dot(s_avg, g.double()).item() for i, (g, _) in enumerate(pasts))
    else:
      want["cosin_sampled"] = want["curv_sampled"] = math.nan
    for key, ref in want.items():
      if math.isnan(ref):
        assert math.isnan(got[key]), (key, got[key])
      else:
        assert abs(got[key] - ref) <= 1e-5 * abs(ref) + 1e-6, (key, got[key], ref)
    assert (got["attack_grad_avg"] is None) == (na == 0)
    assert torch.allclose(got["sampled_grad_avg"].double(), s_avg, atol=1e-6)

def test_nothing_outside_tests_smoke_and_bench_imports_the_oracle():
  """ oracle/ is the checker: the product (`byzantinemomentum_b200/`, `native/`) and the helper scripts
  (`tools/`) must not import it; `bench.py` and `__graft_entry__.py` may (CPU legs / smoke check). """
  import pathlib, re
  root = pathlib.Path(__file__).resolve().parent.parent
  pattern = re.compile(r"^\s*(from\s+oracle\b|import\s+oracle\b)", re.M)
  offenders = []
  for folder in ("byzantinemomentum_b200", "native", "tools"):
    for path in (root / folder).rglob("*.py"):
      if pattern.search(path.read_text()):
        offenders.append(str(path.relative_to(root)))
  assert offenders == []
