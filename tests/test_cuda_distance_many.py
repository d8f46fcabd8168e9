# coding: utf-8
"""`bz_distance_many`, `engine.distance_many`, `Plan(many=True)`, `gars.many_distance_gars` and the plugin above 128
rows on the GPU: Multi-Krum, Bulyan, Aksel and CGE against the NumPy oracle (with test_cuda_distance_wide's rules) at
the bucket and tile edges of n and of the unique-row count u, Bulyan from its smallest theta to 1022, bz_distance's
bits up to 128 rows, rows at mixed 4-byte offsets, the ends of the fp32 range, determinism, and one full-depth call
per rule at n = 1024 replayed from a CUDA graph."""

import ctypes

import numpy as np
import pytest

from conftest import Golden, canon_alias
import parity
from oracle import byzoracle as orc
from test_cuda_distance_wide import CODES, check_against_oracle, device_rows, stack
from test_distance_many_abi import MD_DIR, _registry

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

RULES = (("krum", None, 0), ("krum", 3, 0), ("bulyan", None, 0), ("bulyan", 1, 0), ("aksel", None, 0), ("aksel", None, 1),
         ("cge", None, 0))

def _lib():
  from byzantinemomentum_b200 import _lib
  return _lib

_workspaces = {}

def workspace(n, dev):
  lib = _lib().many_distance_lib()
  nbytes = lib.bz_distance_many_workspace_bytes(n)
  if nbytes not in _workspaces:
    _workspaces[nbytes] = torch.empty(nbytes + 8, dtype=torch.uint8, device=dev)
  return _workspaces[nbytes]

def call(gar, rows, f, m=None, mode=0, fn="bz_distance_many", ws_offset=0):
  """ bz_distance_many (or bz_distance) on cuda:0: (out, order, status) as numpy after a synchronise; `ws_offset`
  bytes into the workspace. """
  n, d = len(rows), rows[0].numel()
  dev = rows[0].device
  lib = _lib().many_distance_lib() if fn == "bz_distance_many" else _lib().lib()
  m = (n - f - 2 if m is None else m) if gar in ("krum", "bulyan") else 0
  out = torch.full((d,), 7., dtype=torch.float32, device=dev)
  meta = torch.full((n + 1,), -1, dtype=torch.int32, device=dev)
  ws = workspace(n, dev) if fn == "bz_distance_many" else torch.empty(lib.bz_distance_workspace_bytes(n), dtype=torch.uint8, device=dev)
  ptrs = (ctypes.c_void_p * n)(*[r.data_ptr() for r in rows])
  stream = torch.cuda.current_stream(dev).cuda_stream
  code = getattr(lib, fn)(CODES[gar], ptrs, n, f, m, mode, d, out.data_ptr(), meta.data_ptr(), meta.data_ptr() + 4 * n,
                          ws.data_ptr() + ws_offset, ws.numel() - ws_offset, stream)
  assert code == 0, (lib.bz_distance_many_last_error() if fn == "bz_distance_many" else lib.bz_last_error()).decode()
  torch.cuda.synchronize(dev)
  return out.cpu().numpy(), meta[:n].cpu().numpy(), int(meta[n].item())

def run_rules(x, nh, rows, f, what, rules=RULES):
  compared = 0
  m_max = x.shape[0] - f - 2
  for gar, m, mode in rules:
    m = m_max // 2 if m == "half" else m
    got, order, status = call(gar, rows, f, m, mode)
    compared += check_against_oracle(gar, x, nh, got, order, status, f, m, "mid" if mode == 0 else "n-f", f"{what} {gar} m={m}")
  return compared

@pytest.mark.parametrize("n", [129, 255, 256, 257, 511, 512, 513, 1023, 1024, 130, 200, 300, 384, 700, 900])
def test_every_rule_against_the_oracle(n):
  nb = n // 5
  x, nh = stack(n, nb, 61 + n % 97, seed=n)
  f = (n - 3) // 4                               # the largest f Bulyan takes
  rules = RULES if n in (129, 256, 257, 512, 1024) else RULES + (("bulyan", "half", 0),)
  # above ~500 rows the adjacent scores of the first n - f rows come closer than MIN_MARGIN somewhere: fewer compare
  assert run_rules(x, nh, device_rows(x, nh), f, f"n={n}", rules) >= (2 if n <= 512 else 1), n

@pytest.mark.parametrize("u", [63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257])
def test_unique_rows_at_the_tile_edges(u):
  """ n = 300 rows of which n - u + 1 are one aliased tensor: u on both sides of every 64-row tile edge. """
  n = 300
  x, nh = stack(n, n - u + 1, 97, seed=4000 + u)
  f = min((n - 3) // 4, n - u + 1)
  compared = run_rules(x, nh, device_rows(x, nh), f, f"u={u}", (("krum", None, 0), ("bulyan", None, 0), ("krum", 5, 0)))
  assert compared >= 1, u

@pytest.mark.parametrize("n", [129, 500, 1024])
def test_one_unique_row_and_no_alias(n):
  dev = torch.device("cuda", 0)
  row = torch.from_numpy(np.random.default_rng(n).standard_normal(83).astype(np.float32)).to(dev)
  rows = [row] * n                                  # u = 1: every score is 0, the order is the index order
  f = (n - 3) // 4
  for gar in ("krum", "bulyan", "aksel", "cge"):
    got, order, status = call(gar, rows, f)
    ref = getattr(orc, gar)([row.cpu().numpy()] * n, f)
    parity.assert_bit_exact(got, ref, f"{gar} u=1 n={n}")
    assert list(order) == list(range(n)) and (status == 0 or gar != "bulyan"), gar
  x, nh = stack(n, 0, 75, seed=7 * n)               # u = n
  assert run_rules(x, nh, device_rows(x, nh), f, f"u=n={n}") >= 1

@pytest.mark.parametrize("n,f", [(129, 31), (129, 0), (300, 74), (1024, 255), (1024, 100), (1024, 0)])
def test_bulyan_theta_range_and_nan_rows(n, f):
  """ theta from its smallest value for the n (f = (n - 3) // 4) to 1022 (n = 1024, f = 0); NaN Byzantine rows with f
  below their count make the reference fail: status 2 and a NaN output. """
  for kind, nb in (("spread", n // 4), ("nan", n // 4)):
    x, nh = stack(n, nb, 53, seed=2000 + n + f, kind=kind)
    got, order, status = call("bulyan", device_rows(x, nh), f)
    check_against_oracle("bulyan", x, nh, got, order, status, f, what=f"bulyan {kind} n={n} f={f}")

@pytest.mark.parametrize("path", [pytest.param(p, id=p.stem) for p in sorted(MD_DIR.glob("golden_md_*.npz"))])
def test_reference_fixtures(path):
  """ Every recorded call of the reference above 128 rows: the selection and the output bit for bit (Multi-Krum,
  Aksel, CGE), Bulyan within its closest-m bar, the degenerate Bulyan as status 2 and a NaN output. """
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

def test_workspace_at_8_mod_16_bytes():
  """ The contract asks for an 8-byte aligned workspace: one at 8 mod 16 gives the bits of a 256-byte aligned one. """
  n = 300
  x, nh = stack(n, 60, 517, seed=77)
  rows = device_rows(x, nh)
  f = (n - 3) // 4
  assert workspace(n, rows[0].device).data_ptr() % 16 == 0
  for gar, m, mode in RULES:
    want = call(gar, rows, f, m, mode)
    got = call(gar, rows, f, m, mode, ws_offset=8)
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)), gar
    assert np.array_equal(got[1], want[1]) and got[2] == want[2], gar

@pytest.mark.parametrize("n", [65, 100, 128])
def test_up_to_128_rows_it_is_bz_distance(n):
  x, nh = stack(n, n // 5, 1031, seed=300 + n)
  rows = device_rows(x, nh)
  f = (n - 3) // 4
  assert _lib().many_distance_lib().bz_distance_many_workspace_bytes(n) == _lib().lib().bz_distance_workspace_bytes(n)
  for gar, m, mode in RULES:
    want = call(gar, rows, f, m, mode, fn="bz_distance")
    got = call(gar, rows, f, m, mode)
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)), (gar, n)
    assert np.array_equal(got[1], want[1]) and got[2] == want[2], (gar, n)

@pytest.mark.parametrize("n", [200, 777])
def test_mixed_offsets_aliases_and_determinism(n):
  x, nh = stack(n, n // 4, 333, seed=800 + n)
  dev = torch.device("cuda", 0)
  def put(row, offset):
    buf = torch.empty(row.shape[0] + offset, dtype=torch.float32, device=dev)
    buf[offset:] = torch.from_numpy(row)
    return buf[offset:]
  rows = [put(x[i], i % 4) for i in range(nh)]
  byz = put(x[nh], 3)
  rows += [byz] * (n - nh)
  assert len({r.data_ptr() % 16 for r in rows}) == 4
  aligned = device_rows(x, nh)
  f = (n - 3) // 4
  for gar, m, mode in RULES:
    first = call(gar, rows, f, m, mode)
    again = call(gar, rows, f, m, mode)
    assert np.array_equal(first[0].view(np.uint32), again[0].view(np.uint32)) and np.array_equal(first[1], again[1]), gar
    other = call(gar, aligned, f, m, mode)
    # the distances do not depend on where a row starts; the averages take the same order
    assert np.array_equal(first[1], other[1]) and np.array_equal(first[0].view(np.uint32), other[0].view(np.uint32)), gar
    check_against_oracle(gar, x, nh, first[0], first[1], first[2], f, m, "mid" if mode == 0 else "n-f", f"{gar} offsets")

def test_ends_of_the_fp32_range():
  """ Rows near FLT_MAX: pairs whose squared distance overflows fp32 score +inf; all-zero rows have key 0 and keep
  their index order; subnormal rows. """
  n, d = 300, 129
  rng = np.random.default_rng(11)
  x = rng.standard_normal((n, d)).astype(np.float32)
  x[:40] *= np.float32(3e37)                        # huge: every pair with them overflows
  x[40:80] = 0.                                     # zero rows: CGE keys 0, in index order
  x[80:120] = (rng.standard_normal((40, d)) * 1e-41).astype(np.float32)       # subnormal
  nh = n
  rows = device_rows(x, nh)
  f = 60
  for gar, m, mode in RULES:
    got, order, status = call(gar, rows, f, m, mode)
    check_against_oracle(gar, x, nh, got, order, status, f, m, "mid" if mode == 0 else "n-f", f"{gar} extremes")
  got, order, status = call("cge", rows, f)
  assert list(order[:40]) == list(range(40, 80))
  D = orc.pairwise_distances([x[i] for i in range(n)])
  assert np.isinf(D[0, 1]) and np.isinf(D[0, 200])

def test_full_depth_and_graph_replay():
  """ n = 1024 rows of d = 1,310,922 with f = 255 aliased Byzantine rows: every rule bitwise equal across two calls
  and its Plan(many=True).graph() replay. """
  from byzantinemomentum_b200 import engine
  n, d, f = 1024, 1_310_922, 255
  dev = torch.device("cuda", 0)
  gen = torch.Generator(device=dev).manual_seed(5)
  nh = n - f
  honest = torch.randn(nh, d, generator=gen, device=dev)
  rows = [honest[i] for i in range(nh)] + [honest[:8].mean(dim=0).mul(-1.1)] * f
  for gar, mode in (("krum", "mid"), ("bulyan", "mid"), ("aksel", "n-f"), ("cge", "mid")):
    first = call(gar, rows, f, None, 1 if mode == "n-f" else 0)
    again = call(gar, rows, f, None, 1 if mode == "n-f" else 0)
    assert np.array_equal(first[0].view(np.uint32), again[0].view(np.uint32)) and np.array_equal(first[1], again[1]), gar
    plan = engine.Plan(gar, rows, f=f, mode=mode, many=True)
    replay = plan.graph()
    plan.out.fill_(0.)
    out = replay()
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32), first[0].view(np.uint32)), gar
    assert np.array_equal(plan.selection.cpu().numpy(), first[1]), gar
    if gar == "krum":                               # the average of the selected rows, bit for bit
      sel = first[1][:n - f - 2].tolist()
      acc = torch.zeros(d, device=dev)
      for k in sel:
        acc = acc + rows[k]                         # fp32 adds in selection order, as K3
      mean = acc.cpu().numpy() / np.float32(len(sel))      # IEEE division (torch's scalar division multiplies)
      assert np.array_equal(mean.view(np.uint32), first[0].view(np.uint32)), gar
    del plan, replay
  torch.cuda.empty_cache()

def test_engine_host_rows_gars_and_plugin():
  import byzantinemomentum_b200 as bz
  n = 300
  x, nh = stack(n, 40, 211, seed=31)
  host = [torch.from_numpy(x[i]) for i in range(nh)]
  host += [torch.from_numpy(x[nh])] * (n - nh)
  rows = device_rows(x, nh)
  f = 50
  for gar, mode in (("krum", "mid"), ("bulyan", "mid"), ("aksel", "mid"), ("cge", "mid")):
    want = call(gar, rows, f)
    out, sel = bz.engine.distance_many(gar, host, f, mode=mode)
    assert out.device.type == "cpu" and np.array_equal(out.numpy().view(np.uint32), want[0].view(np.uint32)), gar
    assert np.array_equal(sel.cpu().numpy(), want[1]), gar
    got = bz.many_distance_gars[gar](gradients=rows, f=f)
    assert np.array_equal(got.cpu().numpy().view(np.uint32), want[0].view(np.uint32)), gar
  # influence reuses the stored selection and matches the oracle's
  for gar in ("krum", "aksel", "cge"):
    entry = bz.many_distance_gars[gar]
    if entry.influence is None:
      continue
    got = entry.influence(rows[:nh], rows[nh:], f=f)
    ref = orc.influence(gar, [x[i] for i in range(nh)], [x[nh]] * (n - nh), f=f)
    assert abs(got - ref) <= 1e-12, gar
  aggregators = _registry()
  bz.plugin.install(aggregators, many_distance=True)
  got = aggregators.gars["b200-krum"].unchecked(gradients=rows, f=f)
  assert np.array_equal(got.cpu().numpy().view(np.uint32), call("krum", rows, f)[0].view(np.uint32))
  with pytest.raises(TypeError):                    # the degenerate Bulyan raises as the reference does
    xn, nhn = stack(n, 80, 50, seed=3, kind="nan")
    bz.engine.distance_many("bulyan", device_rows(xn, nhn), 40)
