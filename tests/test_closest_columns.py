# coding: utf-8
"""CPU self-checks of the Phocas / MeaMed column reference (tests/closest_columns.py): the restated K1
epilogue always picks a valid closest set and stays within the summation bound of its exact mean, agrees
with the oracle wherever the chosen values are unique, gives each constructed column the outcome it is
built for, and the checks the GPU tests apply reject kernels that are subtly wrong on non-finite columns.
Also the value-aware exemption of tests/parity.py on the reference's recorded outputs."""

import pathlib
from fractions import Fraction

import numpy as np
import pytest

import closest_columns as cc
import parity
from conftest import Golden
from oracle import byzoracle as orc

F32 = np.float32
GOLDEN = pathlib.Path(__file__).resolve().parent / "golden"

def fs_of(n):
  return sorted({1, (n - 1) // 4, (n - 1) // 2} - {0})

def random_columns(n, d, seed):
  """ Small columns with heavy ties: small integers and halves, +-0, subnormals, +-1e30, +-inf and NaN of
  both signs, mixed with normal noise at a density drawn per column. """
  rng = np.random.default_rng(seed)
  pool = np.array([0., -0., 1., -1., 0.5, 2., -2., 2. ** -149, -2. ** -149, 2. ** -127, 1e30, -1e30,
                   np.inf, -np.inf, np.nan, -np.nan], dtype=F32)
  x = rng.standard_normal((n, d)).astype(F32)
  x[:, ::3] = np.round(x[:, ::3])
  density = rng.uniform(0., 1., d) ** 2
  mask = rng.random((n, d)) < density[None, :]
  return np.where(mask, pool[rng.integers(0, pool.size, (n, d))], x).astype(F32)

NS = list(range(3, 20)) + [24, 25, 26, 33, 40, 51, 64, 65, 77, 100, 127, 128]

@pytest.mark.parametrize("n", NS)
def test_random_columns_pick_a_closest_set_within_the_bound(n):
  """ A valid closest set and the summation bound on every column; where the chosen values are unique, the
  oracle's row-order sum within the same bound of the same exact mean. """
  x = random_columns(n, 3000, 17 * n)
  for f in range(1, (n - 1) // 2 + 1) if n <= 19 else fs_of(n):
    for mode in cc.MODES:
      what = f"n={n} f={f} {mode}"
      out, chosen, c = cc.check_restatement(x, f, mode, what)
      unique = ~cc.value_ambiguous(x, n - f, c) & ~np.isnan(c)
      vals = cc.chosen_values(x, chosen)
      exact = cc.exact_mean(vals)
      ref = orc.closest_mean(x, n - f, c)
      fin = unique & np.isfinite(exact) & np.isfinite(out) & np.isfinite(ref)
      with np.errstate(invalid="ignore"):
        err = np.abs(ref.astype(np.float64) - exact)
      assert (err[fin] <= cc.sum_bound(vals, exact)[fin]).all(), what + " [oracle]"
      nonfin = unique & ~np.isfinite(exact)
      assert parity.equal_values(ref[nonfin], out[nonfin]).all(), what + " [oracle, non-finite]"

@pytest.mark.parametrize("n", list(range(3, 129)))
def test_constructed_columns_get_their_outcomes(n):
  case = {name: j for j, name in enumerate(cc.CONSTRUCTED)}
  for f in fs_of(n):
    m = n - f
    x = cc.constructed_columns(n, f, seed=n * 131 + f)
    assert x.shape == (n, len(cc.CONSTRUCTED))
    for mode in cc.MODES:
      what = f"n={n} f={f} {mode}"
      out, chosen, c = cc.check_restatement(x, f, mode, what)
      # the documented outcomes, on every column
      live = ~np.isnan(c)
      assert np.isnan(out[~live]).all()
      pos = (chosen & np.isposinf(x)).any(axis=0)
      neg = (chosen & np.isneginf(x)).any(axis=0)
      assert np.isnan(out[live & pos & neg]).all(), what
      assert np.isposinf(out[live & pos & ~neg]).all(), what
      assert np.isneginf(out[live & neg & ~pos]).all(), what
      with np.errstate(invalid="ignore"):
        nan_key = np.isnan(x - c[None, :])
      room = (~nan_key).sum(axis=0) >= m
      assert not (chosen & nan_key)[:, live & room].any(), what + " [a NaN key chosen]"
      # each case reaches what it is built for
      if mode == "phocas":
        assert np.isposinf(c[case["+inf beyond f"]]) and np.isposinf(out[case["+inf beyond f"]])
        assert np.isfinite(c[case["nan within f"]]) and np.isfinite(out[case["nan within f"]])
        assert np.isfinite(out[case["nan signs and payloads"]])
        assert np.isnan(c[case["nan beyond f"]])
        assert np.isfinite(out[case["single nan"]])
      else:
        assert np.isnan(c[case["single nan"]]) and np.isnan(out[case["nan signs and payloads"]])
        if n >= 2 * f + 4:
          assert np.isnan(out[case["both infinities"]])
      assert np.isposinf(c[case["+inf majority"]]) and np.isposinf(out[case["+inf majority"]])
      for j in (case["+inf"], case["-inf"]):
        assert np.isfinite(c[j]) and np.isfinite(out[j])
      assert out[case["all equal"]] == F32(0.75)
      assert np.isposinf(out[case["overflow"]]) or m < 3
      assert not cc.value_ambiguous(x, m, c)[[case["plateau"], case["all equal"]]].any()
      j = case["key ties"]
      with np.errstate(all="ignore"):
        assert len(set(cc.abs_key(x[:, j] - c[j]).tolist())) <= n // 2 + 1

@pytest.mark.parametrize("n", [1, 2, 3, 16, 17, 18, 40, 129])
def test_f0_keeps_the_whole_column_in_rank_order(n):
  """ f = 0 (m = n): no pairs; every entry chosen, summed from +0.0 in rank order, divided by n. """
  x = random_columns(n, 2000, 19 * n)
  s = cc.from_key(np.sort(cc.to_key(x), axis=0))
  acc = np.zeros(x.shape[1], dtype=F32)
  with np.errstate(all="ignore"):
    for k in range(n):
      acc = (acc + s[k]).astype(F32)
    whole = (acc / F32(n)).astype(F32)
  for mode in cc.MODES:
    what = f"n={n} f=0 {mode}"
    out, chosen, c = cc.check_restatement(x, 0, mode, what)
    assert chosen.all(), what
    assert parity.equal_values(out, np.where(np.isnan(c), np.nan, whole)).all(), what
    cc.check_kernel(out, x, 0, mode, what)

def test_exact_mean_is_exact():
  rng = np.random.default_rng(1)
  v = (rng.standard_normal((37, 5)) * 10. ** rng.integers(-30, 30, (37, 5))).astype(F32)
  got = cc.exact_mean(v)
  for j in range(5):
    want = float(sum(Fraction(float(x)) for x in v[:, j]) / 37)
    assert abs(got[j] - want) <= 2. ** -52 * abs(want)
  assert np.isnan(cc.exact_mean(np.array([[np.inf], [-np.inf]]))[0])
  assert cc.exact_mean(np.array([[-np.inf], [1.]]))[0] == -np.inf

def test_value_ambiguity_is_about_values_not_keys():
  x = np.array([[1.], [2.], [2.], [3.], [5.]], dtype=F32)
  c = np.array([2.], dtype=F32)
  assert not cc.value_ambiguous(x, 2, c)[0]         # keys 1, 0, 0, 1, 3: the two 2s
  assert cc.value_ambiguous(x, 3, c)[0]             # 2, 2, then 1 or 3 at the same key
  assert not cc.value_ambiguous(x, 4, c)[0]         # both
  z = np.array([[-0.], [0.], [1.]], dtype=F32)
  assert not cc.value_ambiguous(z, 1, np.array([0.], dtype=F32))[0]
  inf = np.array([[np.inf], [np.inf], [1.], [2.]], dtype=F32)
  assert not cc.value_ambiguous(inf, 3, np.array([np.inf], dtype=F32))[0]   # NaN keys, all from +inf

# ---------------------------------------------------------------------------------------------- #
# Teeth: faults the GPU checks must reject

def _variant(x, f, mode, ties_up=False, inf_key_smallest=False):
  """ K1's epilogue with one step changed, as a faulty kernel would run it. """
  x = np.asarray(x, dtype=F32)
  n = x.shape[0]
  m = n - f
  c = cc.center(x, f, mode)
  s = cc.from_key(np.sort(cc.to_key(x), axis=0))
  def key(v):
    with np.errstate(all="ignore"):
      diff = v - c
    k = cc.abs_key(diff)
    return np.where(np.isinf(diff), 0, k) if inf_key_smallest else k
  acc = np.zeros(x.shape[1], dtype=F32)
  with np.errstate(all="ignore"):
    for l in range(f):
      dlo, dhi = key(s[l]), key(s[l + m])
      up = (dlo >= dhi) if ties_up else (dlo > dhi)
      acc = (acc + np.where(up, s[l + m], s[l])).astype(F32)
    for k in range(f, m):
      acc = (acc + s[k]).astype(F32)
    out = (acc / F32(m)).astype(F32)
  out[np.isnan(c)] = np.nan
  return out

@pytest.mark.parametrize("n", [11, 25, 51, 100])
def test_the_checks_reject_faulty_kernels(n):
  """ On the stacks the GPU tests feed, each fault changes outputs that `check_kernel` compares: the centre
  returned on columns holding NaN or +-inf, ties sent to the upper element, and an infinite key counted
  smallest.  The first and last are also caught by the oracle comparison alone (value-aware exemption). """
  for f in fs_of(n):
    x = cc.stack(n, f, 1031, seed=n + 7 * f)
    for mode in cc.MODES:
      what = f"n={n} f={f} {mode}"
      good = cc.k1_closest(x, f, mode)[0]
      assert parity.equal_values(_variant(x, f, mode), good).all()
      cc.check_kernel(good, x, f, mode, what)
      c = cc.center(x, f, mode)
      nonfinite = ~np.isfinite(x).all(axis=0)
      centre_out = np.where(nonfinite, c, good)
      for bad in (centre_out, _variant(x, f, mode, ties_up=True), _variant(x, f, mode, inf_key_smallest=True)):
        assert not parity.equal_values(bad, good).all(), what
        with pytest.raises(AssertionError):
          cc.check_kernel(bad, x, f, mode, what)
      exempt = parity.closest_ambiguous(x, n - f, c)
      ref = orc.closest_mean(x, n - f, c)
      for bad in (centre_out, _variant(x, f, mode, inf_key_smallest=True)):
        with pytest.raises(AssertionError):
          parity.assert_close_scaled(bad, ref, parity.column_scale(x), what, rtol=parity.RTOL * max(1., (n - f) / 64), exempt=exempt)

# ---------------------------------------------------------------------------------------------- #
# The reference's recorded outputs

def test_value_aware_exemption_on_the_goldens():
  """ Of the 143,676 columns of the 308 recorded Phocas / MeaMed calls (tests/golden, wide and live), the
  key-based exemption set aside 43,315; the value-aware one sets aside about 11,000.  The oracle's match on
  the columns now compared is asserted call by call by test_oracle_golden.py, test_oracle_live_reference.py
  and test_coordinate_abi.py. """
  paths = sorted(GOLDEN.glob("golden_*.npz")) + sorted((GOLDEN / "wide").glob("golden_wide_*.npz")) + sorted((GOLDEN / "live").glob("golden_*.npz"))
  calls = columns = exempt = 0
  for path in paths:
    g = Golden(path)
    for call in g.calls:
      if call["gar"] not in cc.MODES or "raises" in call:
        continue
      f = call["params"]["f"]
      c = cc.center(g.rows, f, call["gar"])
      calls += 1
      columns += g.rows.shape[1]
      exempt += int(parity.closest_ambiguous(g.rows, g.n - f, c).sum())
  print(f"value-aware exemption: {exempt} of {columns} columns in {calls} calls")
  assert calls == 308 and columns == 143_676
  assert exempt <= 11_200
