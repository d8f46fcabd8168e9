# coding: utf-8
"""GPU tests of the coordinate-wise rules above 128 rows (`bz_coordinate_many`, n = 129..1024): the
reference's recorded outputs (`tests/golden/many/`) through `gars.many_gars`, NaN / +-inf / ties column by
column, the same bits as `bz_coordinate` at 128 rows, row views at 4-byte offsets, strided and aliased rows,
the staging ring at full depth, the prepared, captured and sharded paths, host rows, and the limits of
`gars` (128) and `many_gars` (1024)."""

import ctypes

import numpy as np
import pytest

from conftest import Golden
import closest_columns as cc
import parity
from oracle import byzoracle as orc
from test_coordinate_abi import closest_rtol
from test_coordinate_many_abi import MANY_DIR
from test_cuda_k1_edges import _stack

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RULES = {"average": 0, "median": 1, "trmean": 2, "phocas": 3, "meamed": 4}      # BZ_RULE_*

def _ptrs(rows):
  return (ctypes.c_void_p * len(rows))(*[r.data_ptr() for r in rows])

def _many(name, rows, d, f=0, out=None, entry="bz_coordinate_many"):
  """ One bz_coordinate_many (libbyzagg_many.so) or bz_coordinate (libbyzagg.so) call into a NaN-filled output. """
  from byzantinemomentum_b200 import _lib
  out = torch.full((d,), float("nan"), device=DEV) if out is None else out
  lib = _lib.many_lib() if entry == "bz_coordinate_many" else _lib.lib()
  rc = getattr(lib, entry)(RULES[name], _ptrs(rows), len(rows), f, d, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
  if rc != 0:
    _lib.check(rc, entry)
  return out

def _device_rows(x, offsets):
  """ Row i of x at float offset offsets[i % len(offsets)] of its own buffer. """
  n, d = x.shape
  rows = []
  for i in range(n):
    off = offsets[i % len(offsets)]
    buf = torch.empty(d + 8, device=DEV)
    buf[off:off + d] = torch.from_numpy(x[i])
    rows.append(buf[off:off + d])
  return rows

def _check_all_rules(x, rows, what, fs=None):
  """ Every rule through bz_coordinate_many against the oracle: average, median and trimmed mean bit-exact,
  Phocas and MeaMed value for value against K1's closest epilogue and within the closest-means bar. """
  n, d = x.shape
  host = [x[i] for i in range(n)]
  parity.assert_bit_exact(_many("average", rows, d).cpu().numpy(), orc.average(host), f"average {what}")
  parity.assert_bit_exact(_many("median", rows, d).cpu().numpy(), orc.median(host), f"median {what}")
  for f in (fs or sorted({0, 1, (n - 1) // 4, (n - 1) // 2})):
    parity.assert_bit_exact(_many("trmean", rows, d, f).cpu().numpy(), orc.trmean(host, f), f"trmean {what} f={f}")
    if f >= 1:
      for name in cc.MODES:
        cc.check_kernel(_many(name, rows, d, f).cpu().numpy(), x, f, name, f"{name} {what} f={f}")

# ---------------------------------------------------------------------------- #
# The reference's outputs

def _many_calls():
  out = []
  for path in sorted(MANY_DIR.glob("golden_many_*.npz")):
    g = Golden(path)
    for call in g.calls:
      out.append(pytest.param(g, call, id=f"{g.name}:{call['tag']}"))
  return out

@pytest.mark.parametrize("g,call", _many_calls())
def test_matches_the_reference_above_128_rows(g, call):
  import byzantinemomentum_b200 as bz
  gar, params, tag = call["gar"], dict(call["params"]), call["tag"]
  honests = [torch.from_numpy(g.rows[i].copy()).to(DEV) for i in range(g.nh)]
  attacks = [torch.from_numpy(g.rows[g.nh].copy()).to(DEV)] * g.nb if g.nb else []
  rows = honests + attacks
  before = torch.stack(rows).clone()
  out = bz.many_gars[gar](gradients=rows, **params)
  assert out.device == rows[0].device and out.dtype == torch.float32 and out.shape == rows[0].shape
  assert torch.equal(torch.stack(rows).view(torch.int32), before.view(torch.int32)), "inputs modified"
  got = out.cpu().numpy()
  ref = g.get(tag, "out")
  np_rows = [g.rows[i] for i in range(g.n)]
  if gar in ("average", "median"):
    parity.assert_bit_exact(got, ref, tag)
  elif gar == "trmean":
    parity.assert_trmean(got, ref, g.rows, tag)
    parity.assert_bit_exact(got, orc.trmean(np_rows, **params), tag + " [oracle]")
  else:
    f = params["f"]
    center = orc.trmean(np_rows, f) if gar == "phocas" else orc.median(np_rows)
    amb = parity.closest_ambiguous(g.rows, g.n - f, center)
    parity.assert_close_scaled(got, ref, parity.column_scale(g.rows), tag, rtol=closest_rtol(g.n - f), exempt=amb)
    parity.assert_bit_exact(got, cc.k1_closest(g.rows, f, gar, center)[0], tag + " [K1's closest epilogue]")

# ---------------------------------------------------------------------------- #
# Column by column: NaN, +-inf, -0, subnormals, key ties, overflow

@pytest.mark.parametrize("n", [129, 131, 255, 256, 257, 300, 511, 512, 513, 800, 1023, 1024])
def test_special_values(n):
  d = 517 + n % 64
  x = _stack(n, d, 4100 + n)
  _check_all_rules(x, _device_rows(x, [0]), f"n={n} aligned")
  _check_all_rules(x, _device_rows(x, [0, 1, 2, 3, 1]), f"n={n} mixed offsets", fs=[(n - 1) // 3])

@pytest.mark.parametrize("n", [129, 256, 257, 512, 513, 1024])
def test_constructed_columns(n):
  """ The constructed columns of tests/closest_columns.py (infinities, NaN signs and payloads, key ties,
  plateaus, signed zeros, overflow, cancellation) at several f, every rule. """
  for f in sorted({1, (n - 1) // 4, (n - 1) // 2}):
    x = cc.stack(n, f, 700 + n % 7, seed=n * 3 + f)
    cc.check_restatement(x, f, "phocas", f"n={n} f={f}")
    _check_all_rules(x, _device_rows(x, [0, 3]), f"n={n} constructed", fs=[f])

# ---------------------------------------------------------------------------- #
# bz_coordinate's bits at 128 rows; input layouts; the ring at full depth

def test_128_rows_give_bz_coordinate_bits():
  n, d = 128, 4099
  x = _stack(n, d, 4300)
  for offsets in ([0], [1, 2]):
    rows = _device_rows(x, offsets)
    for name, fs in (("average", [0]), ("median", [0]), ("trmean", [1, 40, 63]), ("phocas", [1, 63]), ("meamed", [1, 31])):
      for f in fs:
        want = _many(name, rows, d, f, entry="bz_coordinate")
        got = _many(name, rows, d, f)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (name, f, offsets)

@pytest.mark.parametrize("n", [129, 700])
@pytest.mark.parametrize("offset", [1, 3])
def test_shared_offset_views(n, offset):
  """ Every row and the output at the same offset (the shifted vector path of the average). """
  d = 3001
  x = _stack(n, d, 4400 + n + offset)
  rows = _device_rows(x, [offset])
  _check_all_rules(x, rows, f"n={n} offset={offset}", fs=[n // 4])
  outbig = torch.full((d + 8,), float("nan"), device=DEV)
  for name in ("average", "median", "trmean"):
    _many(name, rows, d, f=n // 4, out=outbig[offset:offset + d])
    want = orc.trmean([x[i] for i in range(n)], n // 4) if name == "trmean" else orc.GARS[name]([x[i] for i in range(n)])
    parity.assert_bit_exact(outbig[offset:offset + d].cpu().numpy(), want, f"{name} offset output")
    assert torch.isnan(outbig[:offset]).all() and torch.isnan(outbig[offset + d:]).all()

def test_strided_and_aliased_rows():
  """ Column views of a matrix (the plain call packs them), and one tensor standing for many rows. """
  import byzantinemomentum_b200 as bz
  n, d = 300, 2053
  x = _stack(n, d, 4500)
  base = torch.from_numpy(np.ascontiguousarray(x.T)).to(DEV)          # [d, n]: row i is base[:, i], stride n
  strided = [base[:, i] for i in range(n)]
  host = [x[i] for i in range(n)]
  for gar, kw in (("average", {}), ("median", {}), ("trmean", dict(f=75))):
    want = orc.trmean(host, 75) if gar == "trmean" else orc.GARS[gar](host)
    parity.assert_bit_exact(bz.many_gars[gar](gradients=strided, **kw).cpu().numpy(), want, f"{gar} strided")
  honest = [torch.from_numpy(x[i]).to(DEV) for i in range(200)]
  byz = torch.from_numpy(x[200]).to(DEV)
  rows = honest + [byz] * 100
  xa = np.stack([x[i] for i in range(200)] + [x[200]] * 100)
  _check_all_rules(xa, rows, "aliased", fs=[99, 149])

@pytest.mark.parametrize("n,d", [(129, 132 * 64 * 5 + 37), (512, 132 * 32 * 5 + 5), (1024, 132 * 16 * 5 + 3), (1000, 1)])
def test_ring_wraps_at_full_depth(n, d):
  """ More tiles per CTA than the ring has stages (one CTA per SM), d not a multiple of the tile. """
  rng = np.random.default_rng(4600 + n)
  x = rng.standard_normal((n, d)).astype(np.float32)
  x[:, ::7] = np.round(x[:, ::7])
  rows = _device_rows(x, [0, 1])
  _check_all_rules(x, rows, f"n={n} d={d}", fs=[n // 5])

# ---------------------------------------------------------------------------- #
# Host layers

def _rows300(d=50_003, seed=51):
  gen = torch.Generator().manual_seed(seed)
  honest = [torch.randn(d, generator=gen) for _ in range(200)]
  byz = torch.randn(d, generator=gen) * 3
  return honest + [byz] * 100

@pytest.mark.parametrize("gar,f", [("average", None), ("median", None), ("trmean", 100), ("phocas", 120), ("meamed", 149)])
def test_plan_graph_and_sharded_plan_give_the_plain_bits(gar, f):
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine, sharded
  host = _rows300()
  rows = [r.to(DEV) for r in host[:200]]
  rows += [host[200].to(DEV)] * 100
  kw = {} if f is None else dict(f=f)
  plain = bz.many_gars[gar](gradients=rows, **kw)
  again = engine.coordinate_many(gar, rows, f)
  assert torch.equal(plain.view(torch.int32), again.view(torch.int32)), "two runs differ"
  plan = engine.Plan(gar, rows, f=f)
  assert plan._fn.__name__ == "bz_coordinate_many"
  assert torch.equal(plan().view(torch.int32), plain.view(torch.int32))
  replay = plan.graph()
  plan.out.fill_(float("nan"))
  assert torch.equal(replay().view(torch.int32), plain.view(torch.int32))
  plan.out.fill_(float("nan"))
  assert torch.equal(replay().view(torch.int32), plain.view(torch.int32))
  splan = sharded.ShardedPlan(gar, rows, f=f)
  assert splan.exchange == "none"
  assert torch.equal(splan().view(torch.int32), plain.view(torch.int32))
  # host rows in, host vector out, the same bits
  on_host = bz.many_gars[gar](gradients=host, **kw)
  assert on_host.device.type == "cpu"
  assert torch.equal(on_host.view(torch.int32), plain.cpu().view(torch.int32))

def test_median_of_1024_rows_through_a_captured_plan():
  import byzantinemomentum_b200 as bz
  n, d = 1024, 20_011
  x = _stack(n, d, 4700)
  rows = [torch.from_numpy(x[i]).to(DEV) for i in range(n)]
  replay = bz.Plan("median", rows).graph()
  parity.assert_bit_exact(replay().cpu().numpy(), orc.median([x[i] for i in range(n)]), "median n=1024 graph")

@pytest.mark.parametrize("shards", [1, 3])
def test_column_shards_concatenate_to_the_whole(shards):
  import byzantinemomentum_b200 as bz
  d = 40_009
  rows = [r.to(DEV) for r in _rows300(d, seed=57)]
  per = -(-d // shards)
  for gar, kw in (("average", {}), ("median", {}), ("trmean", dict(f=25)), ("phocas", dict(f=25)), ("meamed", dict(f=140))):
    whole = bz.many_gars[gar](gradients=rows, **kw)
    parts = [bz.many_gars[gar](gradients=[r[lo:min(d, lo + per)] for r in rows], **kw) for lo in range(0, d, per)]
    assert torch.equal(torch.cat(parts).view(torch.int32), whole.view(torch.int32)), (gar, shards)

def test_gars_keep_128_rows_and_many_gars_take_1024():
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine
  rows = [torch.randn(1000, device=DEV) for _ in range(65)]
  host = [r.cpu().numpy() for r in rows] * 2
  with pytest.raises(ValueError, match="maximum of 128 .*many_gars"):
    bz.gars["median"](gradients=rows * 2)            # 130 rows
  with pytest.raises(ValueError, match="maximum of 128"):
    engine.trmean(rows * 2, 10)
  parity.assert_bit_exact(bz.many_gars["median"](gradients=rows * 2).cpu().numpy(), orc.median(host), "130 rows")
  parity.assert_bit_exact(bz.Plan("median", rows * 2)().cpu().numpy(), orc.median(host), "130 rows, Plan")
  # up to 128 rows a many_gars entry makes its gars entry's call
  for gar, kw in (("average", {}), ("median", {}), ("trmean", dict(f=20)), ("phocas", dict(f=20)), ("meamed", dict(f=30))):
    assert torch.equal(bz.many_gars[gar](gradients=rows, **kw).view(torch.int32), bz.gars[gar](gradients=rows, **kw).view(torch.int32))
  with pytest.raises(ValueError, match="maximum of 1024"):
    bz.many_gars["median"](gradients=rows * 15 + rows[:51])   # 1026 rows
  with pytest.raises(ValueError, match="maximum of 1024"):
    bz.Plan("median", rows * 15 + rows[:51])
