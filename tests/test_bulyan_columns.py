# coding: utf-8
"""CPU self-checks of Bulyan's column reference (tests/bulyan_columns.py): the restated K4 order always picks a
valid closest set and stays within bounds of its exact mean, the constructed columns reach the cases they
name, and the checks would notice a kernel whose window, median or sum were subtly off."""

import math
from fractions import Fraction

import numpy as np
import pytest

import bulyan_columns as bc
import parity
from test_cuda_distance_wide import stack

U = 2. ** -24

SIZES = [(1, 0), (2, 0), (3, 0), (4, 1), (7, 3), (25, 5), (33, 16), (40, 19), (60, 1), (62, 0), (73, 26), (112, 7),
         (121, 2), (124, 1), (126, 0)]

def sum_bound(win, exact, wide):
  """ A rigorous bound on |out - exact| for K4's order: the fp32 sum of beta terms errs by at most
  gamma_{beta-1} sum |w| (fp64: negligible, then one fp32 rounding), the division by one more rounding. """
  beta = win.shape[0]
  mag = np.abs(win.astype(np.float64)).sum(axis=0) / beta
  g = (beta - 1) * U / (1 - (beta - 1) * U)
  return (2.2 * U * np.abs(exact) + (1e-12 if wide else g) * mag * (1 + 2 * U)) + 2. ** -149

@pytest.mark.parametrize("theta,f", SIZES)
@pytest.mark.parametrize("wide", [False, True])
def test_random_columns_pick_a_closest_set_within_bounds(theta, f, wide):
  """ Normal, offset, Cauchy and aliased columns: a valid window, the summation bound, and the 1e-6 bar (the fp32
  order of the 64-row K4 only where it runs, theta <= 62). """
  rng = np.random.default_rng(theta * 7 + f)
  d = 300
  cols = [rng.standard_normal((theta, d)), 5. + rng.standard_normal((theta, d)), rng.standard_cauchy((theta, d))]
  # aliased rows: one value repeated in a third of the column
  alias = rng.standard_normal((theta, d))
  alias[: theta // 3] = alias[0]
  cols.append(alias)
  beta = theta - 2 * f
  for s in cols:
    s = s.astype(np.float32)
    out, srt, lstar, med = bc.k4_reduce(s, f, wide)
    assert bc.closest_set_valid(srt, med, bc.window_mask(srt, lstar, beta)).all()
    win = bc.window(srt, lstar, beta)
    exact = bc.exact_mean(win, beta)
    assert (np.abs(out - exact) <= sum_bound(win, exact, wide)).all()
    if wide or theta <= 62:
      rel = bc.check(out, s, f, wide)
      assert rel.max() <= (3 * U if wide else 1e-6)

@pytest.mark.parametrize("theta,f", SIZES)
def test_constructed_columns(theta, f):
  s = bc.constructed_columns(theta, f, seed=theta)
  assert s.shape == (theta, len(bc.CONSTRUCTED))
  case = {c: j for j, c in enumerate(bc.CONSTRUCTED)}
  for wide in (False, True):
    out = bc.k4_reduce(s, f, wide)[0]
    bc.check(out, s, f, wide, f"theta={theta} f={f}")
    assert math.isnan(out[case["nan"]])
    if theta - 2 * f >= 3:
      assert np.isposinf(out[case["overflow"]])       # FLT_MAX / 2 three times: the rounded sum overflows
  if f == 0 and theta >= 2:
    assert math.isnan(bc.k4_reduce(s, f, True)[0][case["infinities"]])     # the window holds +inf and -inf
  # the window moves along a plateau of equal keys, and key ties sit on both of its edges
  beta = theta - 2 * f
  srt = bc.k4_sorted(s)
  med = bc.k4_reduce(s, f, True)[3]
  key = bc.closeness(srt, med)
  if 2 * f >= 2:
    j = case["key ties"]
    assert len(set(key[:, j].tolist())) < theta

def test_exact_mean_is_exact():
  rng = np.random.default_rng(1)
  v = (rng.standard_normal((37, 5)) * 10. ** rng.integers(-30, 30, (37, 5))).astype(np.float32)
  got = bc.exact_mean(v, 37)
  for j in range(5):
    want = float(sum(Fraction(float(x)) for x in v[:, j]) / 37)
    assert abs(got[j] - want) <= 2. ** -52 * abs(want)
  assert np.isnan(bc.exact_mean(np.array([[np.inf], [-np.inf]]), 2)[0])
  assert bc.exact_mean(np.array([[np.inf], [1.]]), 2)[0] == np.inf

def test_to_key_orders_like_the_kernel():
  x = np.array([np.nan, np.inf, 1., 2. ** -149, 0., -0., -2. ** -149, -1., -np.inf], dtype=np.float32)
  k = bc.to_key(x)
  assert list(np.argsort(k)) == [8, 7, 6, 5, 4, 3, 2, 1, 0]
  back = bc.from_key(k)
  assert np.array_equal(back[1:].view(np.int32), x[1:].view(np.int32)) and math.isnan(back[0])
  assert bc.abs_key(np.float32(np.nan)) > bc.abs_key(np.float32(np.inf)) > bc.abs_key(np.float32(-3.))

def test_an_aliased_window_summed_in_fp32_drifts_past_the_bar():
  """ Why K4-wide adds its window in fp64: with f = 1 and m = 1 stage 1 is the rows themselves; at 124 values, 30
  of them one aliased row, an ascending fp32 sum of the 122-value window misses the exact mean by more than 1e-6
  of the column's scale at one coordinate, the fp64 sum rounded once by 5e-8. """
  x, _ = stack(128, 30, 2053, seed=3011)
  s = x[-124:, 475:476]
  rel = {}
  for wide in (False, True):
    out, srt, lstar, med = bc.k4_reduce(s, 1, wide)
    exact = bc.exact_mean(bc.window(srt, lstar, 122), 122)
    rel[wide] = bc.relative_error(out, exact, parity.column_scale(s))[0]
  assert rel[False] > 1e-6 and rel[True] < 1e-7, rel

def _variant(s, f, strict=True, median_at=None, pad=None):
  """ K4's stage 2 with one step changed, as a faulty kernel would run it. """
  s = np.asarray(s, dtype=np.float32)
  theta = s.shape[0]
  beta = theta - 2 * f
  srt = bc.k4_sorted(s)
  if pad is not None:                # theta values padded to `pad` with a key that sorts first
    srt = bc.from_key(np.sort(np.concatenate([bc.to_key(srt), np.zeros((pad - theta, s.shape[1]), np.int32)]), axis=0))[:theta]
  idx = (theta - 1) // 2 if median_at is None else median_at
  med = np.where(np.isnan(srt[theta - 1]), np.float32(np.nan), srt[idx]).astype(np.float32)
  lstar = np.zeros(s.shape[1], dtype=np.int64)
  with np.errstate(all="ignore"):
    for l in range(theta - beta):
      dlo, dhi = bc.abs_key(srt[l] - med), bc.abs_key(srt[l + beta] - med)
      lstar = np.where((dlo > dhi) if strict else (dlo >= dhi), l + 1, lstar)
    acc = bc.window(srt, lstar, beta).astype(np.float64).sum(axis=0)
    out = (acc.astype(np.float32) / np.float32(beta)).astype(np.float32)
  out[np.isnan(med)] = np.nan
  return out

@pytest.mark.parametrize("theta,f", [(t, f) for t, f in SIZES if f >= 1 and t >= 4])
def test_the_columns_tell_faulty_kernels_apart(theta, f):
  """ A `>=` in the window step, the upper median, or padding keys of 0 each change the output of some column the
  GPU tests feed (constructed, or random as they draw them). """
  s = np.concatenate([bc.constructed_columns(theta, f, seed=theta),
                      np.random.default_rng(theta).standard_normal((theta, 64)).astype(np.float32)], axis=1)
  good = bc.k4_reduce(s, f, True)[0]
  assert np.array_equal(_variant(s, f).view(np.int32), good.view(np.int32))
  for bad in (dict(strict=False), dict(median_at=theta // 2), dict(pad=-(-theta // 8) * 8)):
    if bad.get("median_at") == (theta - 1) // 2 or bad.get("pad") == theta:
      continue                                          # odd theta: the same median; theta a multiple of 8: no padding
    assert not parity.equal_values(_variant(s, f, **bad), good).all(), bad
