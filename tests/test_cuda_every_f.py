# coding: utf-8
"""GPU: the trimmed mean, Phocas and MeaMed at every f, on the three kernel paths of the coordinate-wise rules.

What f changes in a kernel is its epilogue: which ranks R = n - 2f are kept, where the trimmed mean's 16-row and
256-row cascade folds fall (`trmean_sorted` in k1_select.cuh, `many_trmean` in k1_many.cu), and how many
(s[l], s[l + m]) pairs the closest epilogue compares (`closest_pairs`, `many_closest`).  f = 0 is valid and keeps
the whole column.

  * every n from 1 to 128 at every f from 0 to (n - 1) // 2: `bz_<rule>` up to 64 rows, `bz_coordinate` above;
    16-byte aligned rows (the vector kernels, and at n = 11, 25, 51 the compile-time (n, f) kernels) and rows at
    mixed 4-byte offsets (the generic scalar kernel);
  * `bz_coordinate_many` at every f for the first and last n of each row bucket (129, 256 | 257, 512 | 513, 1023,
    1024: every R from 1 to 1024), the same two layouts;
  * `bz_coordinate_many`'s trimmed mean at every n from 129 to 1024, at f = 0, 1, (n - 1) // 2 and each f whose
    R is 15, 16, 17, 255, 256, 257, 511, 512 or 513;
  * the 18-row trimmed mean at f = 0, whose sequential sum once skipped the cascade, through every entry point.

For f >= 1 the rows are tests/closest_columns.py's `stack(n, f, ...)`: NaN, +-inf, key ties and signed zeros at
that f's trim boundary among random columns; for f = 0 they are test_cuda_k1_edges.py's special values.  The
trimmed mean is bit-exact against the oracle, and within `closest_columns.sum_bound` of the exact (fsum) mean of
sorted ranks [f, n - f), a bar that does not depend on the summation order.  Phocas and MeaMed are value for value
K1's closest epilogue (`closest_columns.check_kernel`) and, where the chosen values are unique, the oracle."""

import ctypes

import numpy as np
import pytest

import closest_columns as cc
import parity
from oracle import byzoracle as orc
from test_cuda_k1_edges import SPECIALS, _stack

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RULES = {"trmean": 2, "phocas": 3, "meamed": 4}      # BZ_RULE_*
LAYOUTS = {"aligned": [0], "mixed offsets": [0, 1, 2, 3, 1]}
F32 = np.float32

class _Rows:
  """ The rows of x on the device, row i at float offset offsets[i % len(offsets)] of its own 16-byte aligned
  stretch of one buffer (NaN around it), and the table of their addresses. """
  def __init__(self, x, offsets):
    n, d = x.shape
    pitch = (d + 8 + 3) // 4 * 4
    offs = np.array([offsets[i % len(offsets)] for i in range(n)])
    host = np.full((n, pitch), np.nan, dtype=F32)
    for o in set(offs.tolist()):
      host[offs == o, o:o + d] = x[offs == o]
    self.buf = torch.from_numpy(host).to(DEV)
    base = self.buf.data_ptr()
    self.ptrs = (ctypes.c_void_p * n)(*(base + 4 * (i * pitch + int(offs[i])) for i in range(n)))
    self.n, self.d = n, d

def _call(rule, rows, f):
  """ bz_<rule> up to 64 rows, bz_coordinate up to 128, bz_coordinate_many above, into a NaN-filled output. """
  from byzantinemomentum_b200 import _lib
  out = torch.full((rows.d,), float("nan"), device=DEV)
  stream = torch.cuda.current_stream().cuda_stream
  if rows.n <= 64:
    entry, rc = "bz_" + rule, getattr(_lib.lib(), "bz_" + rule)(rows.ptrs, rows.n, f, rows.d, out.data_ptr(), stream)
  elif rows.n <= _lib.MAX_N_COORDINATE:
    entry, rc = "bz_coordinate", _lib.lib().bz_coordinate(RULES[rule], rows.ptrs, rows.n, f, rows.d, out.data_ptr(), stream)
  else:
    entry, rc = "bz_coordinate_many", _lib.many_lib().bz_coordinate_many(RULES[rule], rows.ptrs, rows.n, f, rows.d, out.data_ptr(), stream)
  _lib.check(rc, entry)
  return out.cpu().numpy()

def _sorted(x):
  """ The columns sorted as the kernels sort them (-0 before +0, NaN last). """
  return cc.from_key(np.sort(cc.to_key(x), axis=0))

def check_trmean_exact(got, x, f, what):
  """ `got` against the exact mean of sorted ranks [f, n - f), whatever the order of the fp32 additions: within
  `sum_bound` where that mean is finite and so is `got`; NaN where a kept rank is NaN or they hold both infinities;
  the infinity they hold where they hold one.  Where the finite kept magnitudes add up past FLT_MAX a partial sum
  may overflow, to either infinity: then a finite mean may come out non-finite, and an infinite one NaN. """
  n = x.shape[0]
  kept = _sorted(x)[f:n - f]
  exact = cc.exact_mean(kept)
  got64 = np.asarray(got, dtype=np.float64)
  with np.errstate(invalid="ignore"):
    k64 = kept.astype(np.float64)
    err = np.abs(got64 - exact)
  mag = np.where(np.isfinite(k64), np.abs(k64), 0.).sum(axis=0)
  may_overflow = mag * (1 + kept.shape[0] * cc.U) > parity.FLT_MAX
  fin = np.isfinite(exact)
  inside = fin & np.isfinite(got64)
  bad = inside & ~(err <= cc.sum_bound(kept, exact))
  assert not bad.any(), f"{what}: {int(bad.sum())} columns out of the summation bound, first at {np.flatnonzero(bad)[:5]}"
  ok = np.where(fin, np.isfinite(got64) | may_overflow,
                parity.equal_values(got64, exact) | (np.isinf(exact) & np.isnan(got64) & may_overflow))
  assert ok.all(), f"{what}: non-finite means at {np.flatnonzero(~ok)[:5]}: got {got64[~ok][:5]}, exact {exact[~ok][:5]}"

def check_every_rule(x, f):
  """ The trimmed mean, Phocas and MeaMed of x at f through every layout: the first layout against the references,
  the others to the same values. """
  n = x.shape[0]
  trmean = orc.trmean(x, f)
  centres = {"phocas": trmean, "meamed": orc.median(x)}
  want = {mode: cc.k1_closest(x, f, mode, centres[mode])[0] for mode in cc.MODES}
  for i, (layout, offsets) in enumerate(LAYOUTS.items()):
    rows = _Rows(x, offsets)
    tag = f"n={n} f={f} {layout}"
    got = _call("trmean", rows, f)
    parity.assert_bit_exact(got, trmean, "trmean " + tag)
    if i == 0:
      check_trmean_exact(got, x, f, "trmean " + tag + " [exact]")
    for mode in cc.MODES:
      got = _call(mode, rows, f)
      if i == 0:
        cc.check_kernel(got, x, f, mode, f"{mode} {tag}", want=want[mode], c=centres[mode])
      else:
        parity.assert_bit_exact(got, want[mode], f"{mode} {tag} [K1's closest epilogue]")

def rows_at(n, f, d, seed):
  """ The special values of test_cuda_k1_edges.py at f = 0 (and below 3 rows), else the constructed columns at f. """
  return _stack(n, d, seed) if f == 0 or n < 3 else cc.stack(n, f, d, seed + 131 * f)

# ---------------------------------------------------------------------------- #
# 1 to 128 rows: K1, every f

D = 163      # two copies of the constructed columns (strides 1 and 2), and a tail of 3 after 40 groups of 4

@pytest.mark.parametrize("n", list(range(1, 129)))
def test_every_f_up_to_128_rows(n):
  for f in range(0, (n - 1) // 2 + 1):
    check_every_rule(rows_at(n, f, D, 60_000 + 1000 * n), f)

# ---------------------------------------------------------------------------- #
# 129 to 1024 rows: K1-many

D_MANY = 67  # one copy of the constructed columns (K1-many sorts each column alone), a tail after one tile of 64

@pytest.mark.parametrize("n", [129, 256, 257, 512, 513, 1023, 1024])
def test_every_f_above_128_rows(n):
  """ The first and last n of each bucket (P = 256, 512, 1024); n = 1023 and 1024 keep every R from 1 to 1024. """
  for f in range(0, (n - 1) // 2 + 1):
    check_every_rule(rows_at(n, f, D_MANY, 70_000 + 1000 * n), f)

def many_fs(n):
  """ f = 0, 1, (n - 1) // 2, and each f that keeps R = 15, 16, 17 (the first fold of ATen's cascade), 255, 256, 257
  (the fold of its 256-row level) or 511, 512, 513 (the second such fold). """
  fs = {0, 1, (n - 1) // 2}
  for r in (15, 16, 17, 255, 256, 257, 511, 512, 513):
    if r <= n and (n - r) % 2 == 0:
      fs.add((n - r) // 2)
  return sorted(fs)

def many_rows(n, d, seed):
  """ Noise over sixteen binades (the summation order shows in the last bits), ties, and NaN, +-inf, +-0,
  subnormals and +-FLT_MAX in every eighth column at a density low enough that most f trim them away. """
  rng = np.random.default_rng(seed)
  x = (rng.standard_normal((n, d)) * np.exp2(rng.integers(-8, 8, (n, d)))).astype(F32)
  x[:, 1::8] = np.round(x[:, 1::8])
  cols = np.arange(0, d, 8)
  mask = rng.random((n, cols.size)) < 0.02
  x[:, cols] = np.where(mask, SPECIALS[rng.integers(0, SPECIALS.size, (n, cols.size))], x[:, cols])
  return x

@pytest.mark.parametrize("n", list(range(129, 1025)))
def test_many_trmean_every_n(n):
  d = 61
  x = many_rows(n, d, 80_000 + n)
  rows = _Rows(x, LAYOUTS["aligned"])
  for f in many_fs(n):
    got = _call("trmean", rows, f)
    parity.assert_bit_exact(got, orc.trmean(x, f), f"trmean n={n} f={f}")
    check_trmean_exact(got, x, f, f"trmean n={n} f={f} [exact]")

# ---------------------------------------------------------------------------- #
# 18 rows at f = 0

def test_trmean_of_18_rows_at_f0_is_atens_mean():
  """ At n = 18 and f = 0 (R = 18) ATen sums the sorted column as (s16 + s17) + (s0 + ... + s15); a sequential
  ((s0 + ... + s15) + s16) + s17 gives other bits in many columns.  Every entry point must give ATen's bits:
  bz_trmean, bz_coordinate, engine.trmean, Plan and its graph, on aligned rows and rows at mixed offsets.
  Phocas and MeaMed at f = 0 average the whole column. """
  from byzantinemomentum_b200 import _lib, engine
  n, d = 18, 4096            # a multiple of 32: torch's CPU mean sums every column in the same order
  rng = np.random.default_rng(90_018)
  x = (rng.standard_normal((n, d)) * np.exp2(rng.integers(-8, 8, (n, d)))).astype(F32)
  s = np.sort(x, axis=0)
  seq = np.zeros(d, dtype=F32)
  for k in range(n):
    seq = (seq + s[k]).astype(F32)
  seq = (seq / F32(n)).astype(F32)
  want = orc.trmean(x, 0)
  differ = int((seq.view(np.int32) != want.view(np.int32)).sum())
  assert differ > 0, "the sequential order gives the cascade's bits on these rows: the test would not see it"
  threads = torch.get_num_threads()
  torch.set_num_threads(1)
  try:
    aten = torch.stack([torch.from_numpy(x[i]) for i in range(n)]).sort(dim=0).values.mean(dim=0).numpy()
  finally:
    torch.set_num_threads(threads)
  assert np.array_equal(want.view(np.int32), aten.view(np.int32)), "the oracle is not ATen's mean"
  def same_bits(got, what):
    got = np.asarray(got.cpu().numpy() if isinstance(got, torch.Tensor) else got, dtype=F32)
    bad = got.view(np.int32) != want.view(np.int32)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {d} columns differ from ATen's mean, first at {np.flatnonzero(bad)[:5]}"
  stream = torch.cuda.current_stream().cuda_stream
  for layout, offsets in LAYOUTS.items():
    rows = _Rows(x, offsets)
    same_bits(_call("trmean", rows, 0), f"bz_trmean {layout}")
    out = torch.full((d,), float("nan"), device=DEV)
    _lib.check(_lib.lib().bz_coordinate(RULES["trmean"], rows.ptrs, n, 0, d, out.data_ptr(), stream), "bz_coordinate")
    same_bits(out, f"bz_coordinate {layout}")
    for mode in cc.MODES:
      cc.check_kernel(_call(mode, rows, 0), x, 0, mode, f"{mode} n=18 f=0 {layout}")
  dev_rows = [torch.from_numpy(x[i].copy()).to(DEV) for i in range(n)]
  same_bits(engine.trmean(dev_rows, 0), "engine.trmean")
  plan = engine.Plan("trmean", dev_rows, f=0)
  same_bits(plan(), "Plan")
  replay = plan.graph()
  plan.out.fill_(float("nan"))
  same_bits(replay(), "Plan.graph")
