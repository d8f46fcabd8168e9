# coding: utf-8
"""GPU parity, part 2: the C ABI called directly through ctypes (the `-m gpu` parity tests
proper), on seeded inputs against the NumPy oracle: every n from 1 to 64, ragged sizes,
unaligned d-shard views, aliased rows, NaN / inf rows, error codes."""

import ctypes

import numpy as np
import pytest

import parity
from oracle import byzoracle as orc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

DEV = "cuda:0"

def _lib():
  from byzantinemomentum_b200 import _lib
  return _lib.lib()

def _ptrs(rows):
  return (ctypes.c_void_p * len(rows))(*[r.data_ptr() for r in rows])

def _stream():
  return torch.cuda.current_stream().cuda_stream

def _ws():
  nbytes = _lib().bz_workspace_bytes(64)
  return torch.empty(nbytes, dtype=torch.uint8, device=DEV), nbytes

def _rand_rows(n, d, seed, scale=None):
  gen = torch.Generator().manual_seed(seed)
  x = torch.randn(n, d, generator=gen)
  if scale is not None:
    x = x * scale[:, None]
  return x

def _call_coord(name, rows, f=None):
  lib = _lib()
  d = rows[0].shape[0]
  out = torch.full((d,), float("nan"), device=DEV)
  fn = getattr(lib, "bz_" + name)
  if f is None:
    rc = fn(_ptrs(rows), len(rows), d, out.data_ptr(), _stream())
  else:
    rc = fn(_ptrs(rows), len(rows), f, d, out.data_ptr(), _stream())
  assert rc == 0, lib.bz_last_error()
  return out.cpu().numpy()

# ---------------------------------------------------------------------------- #

@pytest.mark.parametrize("n", list(range(1, 65)))
def test_median_trmean_every_n(n):
  """ Sorting network of every size: median and trimmed means (f = 1, (n - 1) // 4, (n - 1) // 2; every f in
  test_cuda_every_f.py) vs the oracle, bit-exact. """
  d = 1000 + n
  x = _rand_rows(n, d, 1000 + n)
  rows = [x[i].to(DEV) for i in range(n)]
  host = [x[i].numpy() for i in range(n)]
  parity.assert_bit_exact(_call_coord("median", rows), orc.median(host), f"median n={n}")
  parity.assert_bit_exact(_call_coord("average", rows), orc.average(host), f"average n={n}")
  fs = sorted({1, (n - 1) // 4, (n - 1) // 2} - {0}) if n >= 3 else []
  for f in fs:
    parity.assert_bit_exact(_call_coord("trmean", rows, f), orc.trmean(host, f), f"trmean n={n} f={f}")
    for name, center in (("phocas", orc.trmean(host, f)), ("meamed", orc.median(host))):
      got = _call_coord(name, rows, f)
      ref = orc.GARS[name](host, f)
      amb = parity.closest_ambiguous(x.numpy(), n - f, center)
      parity.assert_close_scaled(got, ref, parity.column_scale(x.numpy()), f"{name} n={n} f={f}", exempt=amb)

@pytest.mark.parametrize("n,f", [(11, 1), (11, 2), (11, 4), (11, 5), (25, 1), (25, 5), (25, 7), (25, 10), (25, 11), (25, 12), (51, 1), (51, 12), (51, 17), (51, 24), (51, 25)])
def test_trmean_specialised_pairs(n, f):
  """ The (n, f) pairs with a compile-time pruned network, incl. NaN / inf columns. """
  d = 4096 + 37
  x = _rand_rows(n, d, 77 + n + f)
  x[0, ::7] = float("nan")
  x[1, ::11] = float("inf")
  x[2, ::13] = float("-inf")
  x[n - 1, 5::7] = float("nan")
  rows = [x[i].to(DEV) for i in range(n)]
  host = [x[i].numpy() for i in range(n)]
  parity.assert_bit_exact(_call_coord("trmean", rows, f), orc.trmean(host, f), f"trmean n={n} f={f}")

@pytest.mark.parametrize("n", [11, 25, 51])
def test_every_compile_time_f_of_the_hot_n(n):
  """ n = 11, 25, 51 have one trmean / phocas / meamed kernel PER f (pruned network, literal partner
  indices): run all of them, finite and non-finite columns. """
  d = 3001
  x = _rand_rows(n, d, 4242 + n)
  x[0, ::9] = float("nan")
  x[1, 3::9] = float("inf")
  x[n - 1, 6::9] = float("-inf")
  rows = [x[i].to(DEV) for i in range(n)]
  host = [x[i].numpy() for i in range(n)]
  xs = x.numpy()
  for f in range(1, (n - 1) // 2 + 1):
    parity.assert_bit_exact(_call_coord("trmean", rows, f), orc.trmean(host, f), f"trmean n={n} f={f}")
    for name, center in (("phocas", orc.trmean(host, f)), ("meamed", orc.median(host))):
      got = _call_coord(name, rows, f)
      ref = orc.GARS[name](host, f)
      amb = parity.closest_ambiguous(xs, n - f, center)
      parity.assert_close_scaled(got, ref, parity.column_scale(xs), f"{name} n={n} f={f}", exempt=amb)

@pytest.mark.parametrize("d", [1, 2, 3, 4, 5, 7, 8, 31, 127, 128, 129, 511, 513, 1025])
def test_ragged_sizes(d):
  n, f = 13, 3
  x = _rand_rows(n, d, 500 + d)
  rows = [x[i].to(DEV) for i in range(n)]
  host = [x[i].numpy() for i in range(n)]
  parity.assert_bit_exact(_call_coord("median", rows), orc.median(host), f"median d={d}")
  parity.assert_bit_exact(_call_coord("trmean", rows, f), orc.trmean(host, f), f"trmean d={d}")
  parity.assert_bit_exact(_call_coord("average", rows), orc.average(host), f"average d={d}")

@pytest.mark.parametrize("offsets", [[1], [2], [3], [0, 1, 2, 3], [4, 4, 8, 12], [1, 1, 1, 5]])
def test_unaligned_shard_views(offsets):
  """ d-shard views `row[off:off+d]` are only 4-byte aligned (SURVEY.md §7.2): same offset for all
  rows -> shifted vector path; mixed offsets -> scalar path.  Output view is offset too. """
  n, f, d = 12, 2, 2053
  x = _rand_rows(n, d + 16, 900 + sum(offsets))
  big = [x[i].to(DEV) for i in range(n)]
  offs = [offsets[i % len(offsets)] for i in range(n)]
  rows = [big[i][offs[i]:offs[i] + d] for i in range(n)]
  host = [x[i].numpy()[offs[i]:offs[i] + d] for i in range(n)]
  lib = _lib()
  outbig = torch.full((d + 16,), float("nan"), device=DEV)
  out = outbig[offs[0]:offs[0] + d]
  for name, args, ref in (("median", (), orc.median(host)), ("trmean", (f,), orc.trmean(host, f)), ("average", (), orc.average(host))):
    outbig.fill_(float("nan"))
    rc = getattr(lib, "bz_" + name)(_ptrs(rows), n, *args, d, out.data_ptr(), _stream())
    assert rc == 0, lib.bz_last_error()
    parity.assert_bit_exact(out.cpu().numpy(), ref, f"{name} offsets={offsets}")
    # nothing written outside the view
    assert torch.isnan(outbig[:offs[0]]).all() and torch.isnan(outbig[offs[0] + d:]).all()
  # distance-based rules on the same views
  ws, nbytes = _ws()
  order = torch.empty(n, dtype=torch.int32, device=DEV)
  rc = lib.bz_krum(_ptrs(rows), n, f, n - f - 2, d, out.data_ptr(), order.data_ptr(), ws.data_ptr(), nbytes, _stream())
  assert rc == 0, lib.bz_last_error()
  ref, info = orc.krum(host, f, return_info=True)
  assert order.cpu().tolist()[:n - f - 2] == info["selection"]
  parity.assert_bit_exact(out.cpu().numpy(), ref, f"krum offsets={offsets}")

def _distance_inputs(n, nb, d, seed, kind="empire"):
  gen = torch.Generator().manual_seed(seed)
  nh = n - nb
  mu = torch.randn(d, generator=gen)
  honest = mu[None, :] + torch.linspace(0.5, 1.5, nh)[:, None] * torch.randn(nh, d, generator=gen)
  byz = honest.mean(dim=0).mul(-1.1) if kind == "empire" else torch.full((d,), float("nan"))
  byz_dev = byz.to(DEV)
  rows = [honest[i].to(DEV) for i in range(nh)] + [byz_dev] * nb
  host = [honest[i].numpy() for i in range(nh)] + [byz.numpy()] * nb
  return rows, host

@pytest.mark.parametrize("n,nb,f,d", [(5, 1, 1, 300), (7, 2, 2, 1000), (11, 3, 3, 5000), (16, 3, 3, 777), (25, 5, 5, 20011),
                                      (26, 6, 5, 3000), (31, 6, 6, 1500), (40, 8, 8, 1200), (51, 12, 12, 2500), (64, 15, 15, 900)])
@pytest.mark.parametrize("kind", ["empire", "nan"])
def test_distance_rules_vs_oracle(n, nb, f, d, kind):
  """ krum / bulyan / brute / aksel / cge through the C ABI: selections bit-exact, values per parity.py. """
  lib = _lib()
  rows, host = _distance_inputs(n, nb, d, 4000 + n, kind)
  ws, nbytes = _ws()
  out = torch.empty(d, device=DEV)
  order = torch.empty(n, dtype=torch.int32, device=DEV)
  status = torch.zeros(1, dtype=torch.int32, device=DEV)
  # krum (default m and m = 1)
  for m in (n - f - 2, 1):
    rc = lib.bz_krum(_ptrs(rows), n, f, m, d, out.data_ptr(), order.data_ptr(), ws.data_ptr(), nbytes, _stream())
    assert rc == 0, lib.bz_last_error()
    ref, info = orc.krum(host, f, m=m, return_info=True)
    nh = n - nb
    canon = lambda idx: [min(int(i), nh) for i in idx]
    assert canon(order.cpu().tolist()[:m]) == canon(info["selection"]), f"krum m={m}"
    parity.assert_bit_exact(out.cpu().numpy(), ref, f"krum n={n} m={m}")
  # distances themselves (phase A) against the oracle's correctly rounded values
  part = torch.empty(n, n, dtype=torch.float64, device=DEV)
  rc = lib.bz_pairdist_partial(_ptrs(rows), n, d, part.data_ptr(), ws.data_ptr(), nbytes, _stream())
  assert rc == 0, lib.bz_last_error()
  got = np.sqrt(part.cpu().numpy())
  D = orc.pairwise_distances(host, map_nonfinite=False)
  iu = np.triu_indices(n, 1)
  fin = np.isfinite(D[iu])
  np.testing.assert_allclose(got[iu][fin], D[iu][fin], rtol=5e-7)
  assert np.array_equal(np.isfinite(got[iu]), fin)
  il = np.tril_indices(n, 0)
  assert (part.cpu().numpy()[il] == 0).all()
  # bulyan
  if n >= 4 * f + 3:
    rc = lib.bz_bulyan(_ptrs(rows), n, f, n - f - 2, d, out.data_ptr(), order.data_ptr(), status.data_ptr(), ws.data_ptr(), nbytes, _stream())
    assert rc == 0, lib.bz_last_error()
    ref, info = orc.bulyan(host, f, return_info=True)
    assert int(status.item()) == 0
    assert canon(order.cpu().tolist()[:n - f - 2]) == canon(info["order"][:n - f - 2])
    parity.assert_close_scaled(out.cpu().numpy(), ref, parity.column_scale(info["stage1"]), f"bulyan n={n}", exempt=info["ambiguous"])
  # brute (small subset counts only)
  import math
  if math.comb(n, n - f) <= 60000:
    sel = torch.empty(n, dtype=torch.int32, device=DEV)
    rc = lib.bz_brute(_ptrs(rows), n, f, d, out.data_ptr(), sel.data_ptr(), status.data_ptr(), ws.data_ptr(), nbytes, _stream())
    assert rc == 0, lib.bz_last_error()
    if kind == "nan" and nb > f:
      assert int(status.item()) == 1
    else:
      ref, info = orc.brute(host, f, return_info=True)
      assert int(status.item()) == 0
      assert canon(sel.cpu().tolist()[:n - f]) == canon(info["selection"]), "brute selection"
      parity.assert_bit_exact(out.cpu().numpy(), ref, f"brute n={n}")
  # cge
  rc = lib.bz_cge(_ptrs(rows), n, f, d, out.data_ptr(), order.data_ptr(), ws.data_ptr(), nbytes, _stream())
  assert rc == 0, lib.bz_last_error()
  ref, info = orc.cge(host, f, return_info=True)
  assert canon(order.cpu().tolist()[:n - f]) == canon(info["selection"])
  parity.assert_bit_exact(out.cpu().numpy(), ref, f"cge n={n}")
  # aksel (NaN rows make the reference's order undefined: finite case only)
  if kind == "empire":
    for mode, name in ((0, "mid"), (1, "n-f")):
      rc = lib.bz_aksel(_ptrs(rows), n, f, mode, d, out.data_ptr(), order.data_ptr(), ws.data_ptr(), nbytes, _stream())
      assert rc == 0, lib.bz_last_error()
      ref, info = orc.aksel(host, f, mode=name, return_info=True)
      c = len(info["selection"])
      assert canon(order.cpu().tolist()[:c]) == canon(info["selection"]), f"aksel {name}"
      parity.assert_bit_exact(out.cpu().numpy(), ref, f"aksel n={n} {name}")

def test_error_codes():
  lib = _lib()
  x = torch.randn(3, 16, device=DEV)
  rows = [x[i] for i in range(3)]
  out = torch.empty(16, device=DEV)
  assert lib.bz_median(None, 3, 16, out.data_ptr(), _stream()) == -1
  assert b"rows is NULL" in lib.bz_last_error()
  assert lib.bz_median(_ptrs(rows), 0, 16, out.data_ptr(), _stream()) == -1
  many = (ctypes.c_void_p * 65)(*([x[0].data_ptr()] * 65))
  assert lib.bz_median(many, 65, 16, out.data_ptr(), _stream()) == -2
  assert lib.bz_trmean(_ptrs(rows), 3, 2, 16, out.data_ptr(), _stream()) == -1          # n - 2f < 1
  assert lib.bz_median(_ptrs(rows), 3, 0, None, _stream()) == 0                          # d = 0: no-op
  ws, nbytes = _ws()
  assert lib.bz_krum(_ptrs(rows), 3, 1, 1, 16, out.data_ptr(), None, ws.data_ptr(), 16, _stream()) == -4   # workspace too small
  assert lib.bz_bulyan(_ptrs(rows), 3, 1, 1, 16, out.data_ptr(), None, None, ws.data_ptr(), nbytes, _stream()) == -1  # n < 4f+3
  # inputs are never modified, output never aliases
  before = x.clone()
  assert lib.bz_median(_ptrs(rows), 3, 16, out.data_ptr(), _stream()) == 0
  torch.cuda.synchronize()
  assert torch.equal(before, x)

def test_krum_peers_leaves_the_status_word_alone_when_a_check_fails():
  """ `bz_krum_peers` zeroes its status word only once every argument has passed: a bad f or an
  undersized workspace returns an error and writes no device memory. """
  lib = _lib()
  n, f, m, d = 11, 2, 3, 64
  x = torch.randn(n, d, device=DEV)
  out = torch.empty(d, device=DEV)
  order = torch.empty(n, dtype=torch.int32, device=DEV)
  status = torch.full((1,), 7, dtype=torch.int32, device=DEV)
  blocks = torch.zeros(2, n * n, dtype=torch.float64, device=DEV)
  flags = torch.zeros(2, 32, dtype=torch.int32, device=DEV)
  table = lambda t: (ctypes.c_void_p * 2)(*[t[r].data_ptr() for r in range(2)])
  ws, nbytes = _ws()
  for bad_f, ws_bytes, code in ((n - 1, nbytes, -1), (f, 16, -4)):
    rc = lib.bz_krum_peers(_ptrs([x[i] for i in range(n)]), n, bad_f, m, d, out.data_ptr(), order.data_ptr(), status.data_ptr(),
                           0, 2, table(blocks), table(flags), 1, ws.data_ptr(), ws_bytes, _stream())
    assert rc == code, lib.bz_last_error()
  torch.cuda.synchronize()
  assert status.item() == 7

def test_cpu_tensors_are_staged():
  """ Reference-facing call with HOST tensors (attack.py --device-gar cpu): staged, result on the CPU. """
  import byzantinemomentum_b200 as bz
  n, f, d = 11, 2, 3001
  x = _rand_rows(n - 2, d, 31337)
  byz = x.mean(dim=0) * -1.1
  rows = [x[i] for i in range(n - 2)] + [byz, byz]
  host = [r.numpy() for r in rows]
  out = bz.gars["median"](gradients=rows, f=f)
  assert out.device.type == "cpu"
  parity.assert_bit_exact(out.numpy(), orc.median(host), "median staged")
  out = bz.gars["krum"](gradients=rows, f=f)
  parity.assert_bit_exact(out.numpy(), orc.krum(host, f), "krum staged")
  assert bz.gars["krum"].influence(rows[:n - 2], rows[n - 2:], f=f) == orc.influence("krum", host[:n - 2], host[n - 2:], f=f)

@pytest.mark.parametrize("n,f", [(7, 1), (15, 3), (19, 4), (23, 5), (27, 6), (31, 7), (35, 8), (39, 9), (43, 10), (47, 11)])
def test_bulyan_register_resident_reduce_for_every_tight_configuration(n, f):
  """ n = 4f + 3 (the tightest n bulyan.py:104-105 accepts for each f) has a compile-time
  `k4_bulyan_static<N, F, VEC>`; unaligned shard views take its VEC = 1 form. """
  import byzantinemomentum_b200 as bz
  d = 6007
  rows, host = _distance_inputs(n, f, d, 7000 + n, "empire")
  ref, info = orc.bulyan(host, f, return_info=True)
  got = bz.gars["bulyan"](gradients=rows, f=f).cpu().numpy()
  parity.assert_close_scaled(got, ref, parity.column_scale(info["stage1"]), f"bulyan n={n} f={f}", exempt=info["ambiguous"])
  views = [r[1:] for r in rows[:n - f]] + [rows[-1][1:]] * f          # 4-byte aligned only
  ref_v, info_v = orc.bulyan([h[1:] for h in host], f, return_info=True)
  got_v = bz.gars["bulyan"](gradients=views, f=f).cpu().numpy()
  parity.assert_close_scaled(got_v, ref_v, parity.column_scale(info_v["stage1"]), f"bulyan n={n} f={f} (views)", exempt=info_v["ambiguous"])
