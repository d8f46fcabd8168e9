# coding: utf-8
"""`bz_distance` and `Plan` above 64 rows on the GPU: Multi-Krum, Bulyan, Aksel and CGE at every n in
65..128 against the NumPy oracle on seeded stacks with aliased Byzantine rows, the reference's fixtures
(tests/golden/wide_distance/), the launches of bz_<rule> at n <= 64, rows that are not 16-byte aligned,
determinism, and `Plan` / `Plan.graph()` at n = 65, 100 and 128."""

import ctypes

import numpy as np
import pytest

from conftest import Golden, canon_alias
import bulyan_columns
import parity
from oracle import byzoracle as orc
from test_distance_wide_abi import WD_DIR

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

CODES = dict(krum=5, bulyan=6, brute=7, aksel=8, cge=9)
MIN_MARGIN = 1e-5         # selections closer than this (relative) are not compared: fp32-norm noise is ~1e-7

def _lib():
  from byzantinemomentum_b200 import _lib
  return _lib.lib()

def stack(n, nb, d, seed, kind="spread"):
  """ [n, d] fp32: n - nb honest rows mu + sigma_i z_i (sigma_i spread over [0.5, 1.5]), the nb Byzantine rows
  one row (aliased when put on the device); kind "nan": the Byzantine row is NaN. """
  rng = np.random.default_rng(seed)
  nh = n - nb
  mu = rng.standard_normal(d)
  honest = mu[None, :] + np.linspace(0.5, 1.5, nh)[:, None] * rng.standard_normal((nh, d))
  byz = np.full(d, np.nan) if kind == "nan" else -1.1 * honest.mean(axis=0)
  return np.concatenate([honest, np.repeat(byz[None, :], nb, axis=0)]).astype(np.float32), nh

def device_rows(x, nh, offset=0):
  """ The rows of x on cuda:0, the Byzantine rows ONE tensor; offset > 0: every row starts `offset` floats
  into its own buffer (4-byte but not 16-byte aligned). """
  dev = torch.device("cuda", 0)
  def put(row):
    buf = torch.empty(row.shape[0] + offset, dtype=torch.float32, device=dev)
    buf[offset:] = torch.from_numpy(row)
    return buf[offset:]
  rows = [put(x[i]) for i in range(nh)]
  if x.shape[0] > nh:
    byz = put(x[nh])
    rows += [byz] * (x.shape[0] - nh)
  return rows

def call(gar, rows, f, m=None, mode=0, ws=None):
  """ bz_distance on cuda:0: (out, order, status) as numpy after a synchronise. """
  n, d = len(rows), rows[0].numel()
  dev = rows[0].device
  lib = _lib()
  m = (n - f - 2 if m is None else m) if gar in ("krum", "bulyan") else 0
  out = torch.full((d,), 7., dtype=torch.float32, device=dev)
  meta = torch.full((n + 1,), -1, dtype=torch.int32, device=dev)
  if ws is None:
    ws = torch.empty(lib.bz_distance_workspace_bytes(n), dtype=torch.uint8, device=dev)
  ptrs = (ctypes.c_void_p * n)(*[r.data_ptr() for r in rows])
  stream = torch.cuda.current_stream(dev).cuda_stream
  code = lib.bz_distance(CODES[gar], ptrs, n, f, m, mode, d, out.data_ptr(), meta.data_ptr(), meta.data_ptr() + 4 * n,
                         ws.data_ptr(), ws.numel(), stream)
  assert code == 0, lib.bz_last_error().decode()
  torch.cuda.synchronize(dev)
  return out.cpu().numpy(), meta[:n].cpu().numpy(), int(meta[n].item())

def clear(keys, order, upto, nh):
  """ Whether the first upto + 1 keys in `order` are apart by MIN_MARGIN (relative), ties between aliased
  Byzantine rows (indices >= nh, the same tensor: the same key on both sides) aside. """
  for k in range(min(upto, len(order) - 1)):
    i, j = order[k], order[k + 1]
    if i >= nh and j >= nh:
      continue
    a, b = keys[i], keys[j]
    if np.isfinite(a) and np.isfinite(b):
      if (b - a) / max(abs(b), 1e-300) < MIN_MARGIN:
        return False
    elif a == b or np.isnan(a) or np.isnan(b):
      return False
  return True

def check_against_oracle(gar, x, nh, got, order, status, f, m=None, mode="mid", what=""):
  """ The selection (where its margin is clear) and the status bit-exact, the output bit-exact (Multi-Krum,
  Aksel, CGE) or within the closest-m bar (Bulyan; where the selection is compared, also K4's order bit for bit
  and within the bar of the exact mean of its window, tests/bulyan_columns.py).  Returns whether the selection
  was compared. """
  rows = [x[i] for i in range(x.shape[0])]
  n = len(rows)
  if gar == "bulyan":
    m = n - f - 2 if m is None else m
    try:
      ref, info = orc.bulyan(rows, f, m, return_info=True)
    except TypeError:                             # degenerate: the reference fails, the device sets the status word
      assert status == 2 and np.isnan(got).all(), what
      return True
    assert status == 0, what
    parity.assert_close_scaled(got, ref, parity.column_scale(info["stage1"]), what, exempt=info["ambiguous"])
    if not clear(info["scores"], info["order"], n - f - 2, nh):
      return False
    assert canon_alias(order[:n - f - 2], nh) == canon_alias(info["order"][:n - f - 2], nh), what
    bulyan_columns.check(got, info["stage1"], f, bulyan_columns.uses_wide(n, f), what)
    return True
  if gar == "krum":
    ref, info = orc.krum(rows, f, m, return_info=True)
    count, keys = n - f - 2 if m is None else m, info["scores"]
  elif gar == "aksel":
    ref, info = orc.aksel(rows, f, mode, return_info=True)
    count, keys = (n + 1) // 2 if mode == "mid" else n - f, info["distances"]
  else:
    ref, info = orc.cge(rows, f, return_info=True)
    count, keys = n - f, info["norms"]
  if not clear(keys, info["order"], count, nh):
    return False
  assert canon_alias(order[:count], nh) == canon_alias(info["order"][:count], nh), what
  parity.assert_bit_exact(got, ref, what)
  return True

@pytest.mark.parametrize("n", range(65, 129))
def test_every_n_against_the_oracle(n):
  nb = n // 5
  x, nh = stack(n, nb, 67 + 3 * n, seed=n)
  rows = device_rows(x, nh)
  f = (n - 3) // 4                               # the largest f Bulyan takes: theta = n - 2f - 2 down to 33
  m_max = n - f - 2
  compared = 0
  for gar, m, mode in (("krum", None, 0), ("krum", 3, 0), ("bulyan", None, 0), ("bulyan", 1, 0), ("bulyan", m_max // 2, 0),
                       ("aksel", None, 0), ("aksel", None, 1), ("cge", None, 0)):
    got, order, status = call(gar, rows, f, m, mode)
    compared += check_against_oracle(gar, x, nh, got, order, status, f, m, "mid" if mode == 0 else "n-f", f"{gar} n={n}")
  assert compared >= 2, n

@pytest.mark.parametrize("n,f", [(65, 0), (100, 1), (128, 0), (128, 31), (97, 23)])
def test_bulyan_theta_range_and_nan_rows(n, f):
  """ theta up to 126 (f = 0) and the degenerate case: NaN Byzantine rows with f below their count. """
  for kind, nb in (("spread", n // 4), ("nan", n // 4)):
    x, nh = stack(n, nb, 131, seed=1000 + n + f, kind=kind)
    got, order, status = call("bulyan", device_rows(x, nh), f)
    check_against_oracle("bulyan", x, nh, got, order, status, f, what=f"bulyan {kind} n={n} f={f}")

def wd_calls():
  return [pytest.param(path, id=path.stem) for path in sorted(WD_DIR.glob("golden_wd_*.npz"))]

@pytest.mark.parametrize("path", wd_calls())
def test_reference_fixtures(path):
  g = Golden(path)
  rows = device_rows(g.rows, g.nh)
  for c in g.calls:
    gar, params, tag = c["gar"], c["params"], c["tag"]
    f, m = params["f"], params.get("m")
    mode = params.get("mode", "mid")
    got, order, status = call(gar, rows, f, m, 1 if mode == "n-f" else 0)
    if "raises" in c:
      assert gar == "bulyan" and status == 2 and np.isnan(got).all(), tag
      continue
    ref = g.get(tag, "out")
    if gar == "bulyan":
      assert status == 0, tag
      _, info = orc.bulyan([g.rows[i] for i in range(g.n)], return_info=True, **params)
      parity.assert_close_scaled(got, ref, parity.column_scale(info["stage1"]), tag, exempt=info["ambiguous"])
      continue
    if gar == "aksel" and np.isnan(g.get(tag, "dists")).any():
      continue
    count = {"krum": m or (g.n - f - 2), "cge": g.n - f}.get(gar, c.get("c"))
    assert canon_alias(order[:count], g.nh) == canon_alias(g.get(tag, "order")[:count], g.nh), tag
    parity.assert_bit_exact(got, ref, tag)

@pytest.mark.parametrize("n", [7, 25, 51, 64])
def test_up_to_64_rows_bz_distance_is_bz_rule(n):
  lib = _lib()
  nb = n // 5
  x, nh = stack(n, nb, 1031, seed=77 + n)
  rows = device_rows(x, nh)
  dev = rows[0].device
  f = (n - 3) // 4
  ws = torch.empty(lib.bz_workspace_bytes(n), dtype=torch.uint8, device=dev)
  assert lib.bz_distance_workspace_bytes(n) == ws.numel()
  ptrs = (ctypes.c_void_p * n)(*[r.data_ptr() for r in rows])
  stream = torch.cuda.current_stream(dev).cuda_stream
  d = x.shape[1]
  for gar, mode in (("krum", 0), ("bulyan", 0), ("brute", 0), ("aksel", 0), ("aksel", 1), ("cge", 0)):
    if gar == "brute" and n > 7:
      continue
    got, order, status = call(gar, rows, f, None, mode, ws=ws)
    out = torch.empty(d, dtype=torch.float32, device=dev)
    meta = torch.full((n + 1,), -1, dtype=torch.int32, device=dev)
    o, s = meta.data_ptr(), meta.data_ptr() + 4 * n
    if gar == "krum":
      code = lib.bz_krum(ptrs, n, f, n - f - 2, d, out.data_ptr(), o, ws.data_ptr(), ws.numel(), stream)
    elif gar == "bulyan":
      code = lib.bz_bulyan(ptrs, n, f, n - f - 2, d, out.data_ptr(), o, s, ws.data_ptr(), ws.numel(), stream)
    elif gar == "brute":
      code = lib.bz_brute(ptrs, n, f, d, out.data_ptr(), o, s, ws.data_ptr(), ws.numel(), stream)
    elif gar == "aksel":
      code = lib.bz_aksel(ptrs, n, f, mode, d, out.data_ptr(), o, ws.data_ptr(), ws.numel(), stream)
    else:
      code = lib.bz_cge(ptrs, n, f, d, out.data_ptr(), o, ws.data_ptr(), ws.numel(), stream)
    assert code == 0
    torch.cuda.synchronize(dev)
    length = n - f if gar == "brute" else n
    assert np.array_equal(out.cpu().numpy().view(np.uint32), got.view(np.uint32)), (gar, n)
    assert np.array_equal(meta[:length].cpu().numpy(), order[:length]), (gar, n)
    if gar in ("bulyan", "brute"):
      assert int(meta[n].item()) == status

@pytest.mark.parametrize("n", [65, 100, 128])
def test_unaligned_rows_and_determinism(n):
  x, nh = stack(n, n // 4, 1000, seed=500 + n)
  aligned = device_rows(x, nh)
  shifted = device_rows(x, nh, offset=1)            # not 16-byte aligned: the cp.async distance kernel
  assert shifted[0].data_ptr() % 16 != 0
  f = (n - 3) // 4
  for gar, mode in (("krum", 0), ("bulyan", 0), ("aksel", 0), ("cge", 0)):
    first = call(gar, aligned, f, None, mode)
    again = call(gar, aligned, f, None, mode)
    assert np.array_equal(first[0].view(np.uint32), again[0].view(np.uint32)) and np.array_equal(first[1], again[1]), gar
    other = call(gar, shifted, f, None, mode)
    check_against_oracle(gar, x, nh, other[0], other[1], other[2], f, what=f"{gar} unaligned n={n}")
    if gar in ("aksel", "cge"):                       # K2' reads any alignment the same way
      assert np.array_equal(first[0].view(np.uint32), other[0].view(np.uint32)), gar

@pytest.mark.parametrize("n", [65, 100, 128])
def test_plan_and_graph(n):
  from byzantinemomentum_b200 import engine
  x, nh = stack(n, n // 5, 4099, seed=900 + n)
  rows = device_rows(x, nh)
  f = (n - 3) // 4
  for gar, mode in (("krum", "mid"), ("bulyan", "mid"), ("aksel", "n-f"), ("cge", "mid")):
    plan = engine.Plan(gar, rows, f=f, mode=mode)
    got = plan().cpu().numpy()
    sel = plan.selection.cpu().numpy()
    want = call(gar, rows, f, None, 1 if mode == "n-f" else 0)
    assert np.array_equal(got.view(np.uint32), want[0].view(np.uint32)), gar
    assert np.array_equal(sel, want[1]), gar
    if gar == "bulyan":
      assert int(plan.status.item()) == want[2] == 0
    else:
      assert plan.status is None
    check_against_oracle(gar, x, nh, got, sel, want[2], f, mode=mode, what=f"plan {gar} n={n}")
    plan.out.fill_(0.)
    replay = plan.graph()
    out = replay()
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want[0].view(np.uint32)), gar
  with pytest.raises(ValueError, match="maximum of 64"):
    engine.Plan("brute", rows, f=1)
  with pytest.raises(ValueError, match="maximum of 128"):
    engine.Plan("krum", rows + rows[:129 - n], f=1)
