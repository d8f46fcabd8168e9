# coding: utf-8
"""GPU tests of the coordinate-wise rules above 64 rows (`bz_coordinate`, n = 65..128): the
reference's recorded outputs (`tests/golden/wide/`), every n on the values sorting networks get
wrong, row views at 4-byte offsets, the same bits as `bz_<rule>` up to 64 rows, the prepared and
sharded paths, host rows, and the rules that still stop at 64 rows."""

import ctypes

import numpy as np
import pytest

from conftest import Golden
import closest_columns as cc
import parity
from oracle import byzoracle as orc
from test_coordinate_abi import WIDE_DIR, closest_rtol
from test_cuda_k1_edges import _stack

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RULES = {"average": 0, "median": 1, "trmean": 2, "phocas": 3, "meamed": 4}      # BZ_RULE_*

def _lib():
  from byzantinemomentum_b200 import _lib
  return _lib.lib()

def _ptrs(rows):
  return (ctypes.c_void_p * len(rows))(*[r.data_ptr() for r in rows])

def _coordinate(name, rows, d, f=0, out=None):
  """ One bz_coordinate call into a NaN-filled output. """
  lib = _lib()
  out = torch.full((d,), float("nan"), device=DEV) if out is None else out
  rc = lib.bz_coordinate(RULES[name], _ptrs(rows), len(rows), f, d, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
  assert rc == 0, lib.bz_last_error()
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
  """ Every rule through bz_coordinate against the oracle: average, median and trimmed mean bit-exact. """
  n, d = x.shape
  host = [x[i] for i in range(n)]
  parity.assert_bit_exact(_coordinate("average", rows, d).cpu().numpy(), orc.average(host), f"average {what}")
  parity.assert_bit_exact(_coordinate("median", rows, d).cpu().numpy(), orc.median(host), f"median {what}")
  for f in (fs or sorted({1, (n - 1) // 4, (n - 1) // 2})):
    parity.assert_bit_exact(_coordinate("trmean", rows, d, f).cpu().numpy(), orc.trmean(host, f), f"trmean {what} f={f}")
    for name in cc.MODES:
      cc.check_kernel(_coordinate(name, rows, d, f).cpu().numpy(), x, f, name, f"{name} {what} f={f}")

# ---------------------------------------------------------------------------- #
# The reference's outputs

def _wide_calls():
  out = []
  for path in sorted(WIDE_DIR.glob("golden_wide_*.npz")):
    g = Golden(path)
    for call in g.calls:
      out.append(pytest.param(g, call, id=f"{g.name}:{call['tag']}"))
  return out

@pytest.mark.parametrize("g,call", _wide_calls())
def test_matches_the_reference_above_64_rows(g, call):
  import byzantinemomentum_b200 as bz
  gar, params, tag = call["gar"], dict(call["params"]), call["tag"]
  honests = [torch.from_numpy(g.rows[i].copy()).to(DEV) for i in range(g.nh)]
  attacks = [torch.from_numpy(g.rows[g.nh].copy()).to(DEV)] * g.nb if g.nb else []
  rows = honests + attacks
  before = torch.stack(rows).clone()
  out = bz.gars[gar](gradients=rows, **params)
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
# Every n: NaN, +-inf, -0, subnormals, ties; aligned rows and 4-byte offsets

@pytest.mark.parametrize("n", list(range(65, 129)))
def test_special_values_every_n(n):
  d = 517 + 2 * n
  x = _stack(n, d, 2500 + n)
  _check_all_rules(x, _device_rows(x, [0]), f"n={n} aligned")
  _check_all_rules(x, _device_rows(x, [0, 1, 2, 3, 1]), f"n={n} mixed offsets", fs=[(n - 1) // 3])

@pytest.mark.parametrize("n", [65, 100, 128])
@pytest.mark.parametrize("offset", [1, 3])
def test_shared_offset_views(n, offset):
  """ Every row and the output at the same offset (the shifted vector path of the average). """
  d = 3001
  x = _stack(n, d, 2700 + n + offset)
  rows = _device_rows(x, [offset])
  _check_all_rules(x, rows, f"n={n} offset={offset}", fs=[n // 4])
  outbig = torch.full((d + 8,), float("nan"), device=DEV)
  for name in ("average", "median"):
    _coordinate(name, rows, d, out=outbig[offset:offset + d])
    parity.assert_bit_exact(outbig[offset:offset + d].cpu().numpy(), orc.GARS[name]([x[i] for i in range(n)]), f"{name} offset output")
    assert torch.isnan(outbig[:offset]).all() and torch.isnan(outbig[offset + d:]).all()

# ---------------------------------------------------------------------------- #
# Up to 64 rows: bz_coordinate is bz_<rule>

@pytest.mark.parametrize("n", [1, 11, 25, 51, 64])
def test_same_bits_as_the_per_rule_entry_points(n):
  lib = _lib()
  d = 4099
  x = _stack(n, d, 2900 + n)
  for offsets in ([0], [1, 2]):
    rows = _device_rows(x, offsets)
    stream = torch.cuda.current_stream().cuda_stream
    for name, fs in (("average", [0]), ("median", [0]), ("trmean", range(1, (n + 1) // 2)), ("phocas", [(n - 1) // 2]), ("meamed", [(n - 1) // 4])):
      for f in fs:
        if name in ("phocas", "meamed") and f < 1:
          continue
        want = torch.full((d,), float("nan"), device=DEV)
        fn = getattr(lib, "bz_" + name)
        rc = fn(_ptrs(rows), n, d, want.data_ptr(), stream) if name in ("average", "median") else fn(_ptrs(rows), n, f, d, want.data_ptr(), stream)
        assert rc == 0, lib.bz_last_error()
        got = _coordinate(name, rows, d, f)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (name, n, f, offsets)

# ---------------------------------------------------------------------------- #
# Host layers

def _rows100(d=50_003, seed=31):
  gen = torch.Generator().manual_seed(seed)
  honest = [torch.randn(d, generator=gen) for _ in range(80)]
  byz = torch.randn(d, generator=gen) * 3
  return honest + [byz] * 20

@pytest.mark.parametrize("gar,f", [("average", None), ("median", None), ("trmean", 20), ("phocas", 30), ("meamed", 49)])
def test_plan_graph_and_sharded_plan_give_the_plain_bits(gar, f):
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import engine, sharded
  host = _rows100()
  rows = [r.to(DEV) for r in host[:80]]
  rows += [host[80].to(DEV)] * 20
  kw = {} if f is None else dict(f=f)
  plain = bz.gars[gar](gradients=rows, **kw)
  plan = engine.Plan(gar, rows, f=f)
  assert torch.equal(plan().view(torch.int32), plain.view(torch.int32))
  replay = plan.graph()
  plan.out.fill_(float("nan"))
  assert torch.equal(replay().view(torch.int32), plain.view(torch.int32))
  splan = sharded.ShardedPlan(gar, rows, f=f)
  assert splan.exchange == "none"
  assert torch.equal(splan().view(torch.int32), plain.view(torch.int32))
  # host rows in, host vector out, the same bits
  on_host = bz.gars[gar](gradients=host, **kw)
  assert on_host.device.type == "cpu"
  assert torch.equal(on_host.view(torch.int32), plain.cpu().view(torch.int32))

@pytest.mark.parametrize("shards", [1, 3, 8])
def test_column_shards_concatenate_to_the_whole(shards):
  """ R ranks emulated on one GPU: each takes columns [lo_r, hi_r) of every row (views at any
  offset); the R results side by side are the single-GPU result. """
  import byzantinemomentum_b200 as bz
  d = 40_009
  rows = [r.to(DEV) for r in _rows100(d, seed=37)]
  per = -(-d // shards)
  for gar, kw in (("average", {}), ("median", {}), ("trmean", dict(f=25)), ("phocas", dict(f=25)), ("meamed", dict(f=40))):
    whole = bz.gars[gar](gradients=rows, **kw)
    parts = [bz.gars[gar](gradients=[r[lo:min(d, lo + per)] for r in rows], **kw) for lo in range(0, d, per)]
    assert torch.equal(torch.cat(parts).view(torch.int32), whole.view(torch.int32)), (gar, shards)

def test_native_median_takes_100_rows():
  import native
  import byzantinemomentum_b200 as bz
  rows = [r.to(DEV) for r in _rows100(10_007, seed=41)]
  got = native.median.aggregate(rows)
  parity.assert_bit_exact(got.cpu().numpy(), orc.median([r.cpu().numpy() for r in rows]), "native median")
  assert torch.equal(got, bz.gars["median"](gradients=rows))

def test_distance_rules_still_stop_at_64_rows():
  import byzantinemomentum_b200 as bz
  rows = [torch.randn(1000, device=DEV) for _ in range(65)]
  with pytest.raises(ValueError, match="coordinate-wise rules accept up to 128"):
    bz.gars["krum"](gradients=rows, f=5)
  bz.gars["median"](gradients=rows)                  # the same list through a coordinate-wise rule first
  with pytest.raises(ValueError, match="coordinate-wise rules accept up to 128"):
    bz.gars["krum"](gradients=rows, f=5)
  with pytest.raises(ValueError):
    bz.gars["median"](gradients=rows * 2)            # 130 rows
