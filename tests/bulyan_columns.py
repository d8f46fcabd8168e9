# coding: utf-8
"""Bulyan's second stage (bulyan.py:78-84) column by column: an exact reference, and a restatement of the
order K4 (k4_bulyan.cu, k4_bulyan_wide.cu) adds in.  Test infrastructure only: plain NumPy, no GPU.

Stage 1 is `orc.bulyan_stage1`, bit exact: theta fp32 values per coordinate.  Stage 2 picks the beta =
theta - 2f values whose keys fl32|fl32(x - med)| are smallest, med the lower median (NaN when the column
holds a NaN; NaN keys count as largest), and averages them.  A set of beta smallest keys is not unique when
keys tie across its boundary, so the reference checks a set instead of choosing one:
  * `closest_set_valid`: every key inside the set is <= every key outside it;
  * `exact_mean`: the mean of a set, summed exactly (math.fsum) and rounded once.
`k4_reduce` restates the kernels step by step: the column sorted by key (-0 before +0, NaN last), the
median at (theta - 1) // 2, the window of beta sorted values that starts right after the last strict gain
(|s[l] - med| > |s[l + beta] - med|, compared as magnitude bits with NaN largest), the window added in
ascending order from 0.0 (in fp32 by the 64-row K4, in fp64 rounded once to fp32 by K4-wide) and one fp32
division by beta.  Where the window's fp32 sum overflows, any value
in the column's hull is acceptable (parity.assert_in_hull)."""

import math

import numpy as np

from oracle import byzoracle as orc

F32 = np.float32
I32 = np.int32
RTOL = 1e-6
NAN_KEY = np.int32(0x7fffffff)
# A mean in fp32's subnormal range is only good to its spacing, 2^-149: the bar's scale never drops below
# the magnitude at which RTOL of it is that spacing.
SUBNORMAL_FLOOR = 2. ** -149 / RTOL

def sizes(n, f):
  """ (m_max, theta, beta) of Bulyan at (n, f). """
  return n - f - 2, n - 2 * f - 2, n - 4 * f - 2

def uses_wide(n, f):
  """ Whether bz_distance's Bulyan reduces with K4-wide: above 64 rows, and at theta = 61 and 62 (n = 63 and 64,
  f = 0), past the last 64-row kernel. """
  return n > 64 or n - 2 * f - 2 > 60

def stage1(g, order, f, m):
  """ The theta x d stage-1 values (bulyan.py:64-73), no degenerate check: the rows of `order` in score order. """
  return orc.bulyan_stage1(np.asarray(g, dtype=F32), list(order), f, m)

# ---------------------------------------------------------------------------------------------- #
# Keys

def to_key(x):
  """ float_to_key: an int32 whose order is the fp32 order, -0 below +0, every NaN INT_MAX (largest). """
  x = np.asarray(x, dtype=F32)
  k = x.view(I32)
  k = k ^ ((k >> 31) & I32(0x7fffffff))
  return np.where(np.isnan(x), NAN_KEY, k).astype(I32)

def from_key(k):
  k = np.asarray(k, dtype=I32)
  return (k ^ ((k >> 31) & I32(0x7fffffff))).view(F32)

def abs_key(x):
  """ abs_key: the magnitude bits, NaN (any payload) largest. """
  x = np.asarray(x, dtype=F32)
  return np.where(np.isnan(x), NAN_KEY, x.view(I32) & I32(0x7fffffff)).astype(I32)

def closeness(s, med):
  """ The keys of stage 2, fl32|fl32(x - med)|, as ordered integers (NaN largest). """
  with np.errstate(all="ignore"):
    return abs_key(np.asarray(s, dtype=F32) - np.asarray(med, dtype=F32)[None, :])

# ---------------------------------------------------------------------------------------------- #
# The exact reference

def lower_median(s):
  """ torch's median(dim=0) of the theta x d values: rank (theta - 1) // 2, NaN if the column holds one. """
  s = np.asarray(s, dtype=F32)
  srt = np.sort(s, axis=0)
  med = srt[(s.shape[0] - 1) // 2].copy()
  med[np.isnan(s).any(axis=0)] = np.nan
  return med

def closest_set_valid(s, med, chosen):
  """ Per column: whether the boolean [theta, d] mask `chosen` holds beta values with the smallest keys, i.e.
  no key inside exceeds a key outside (NaN keys largest). """
  key = closeness(s, med).astype(np.int64)
  inside = np.where(chosen, key, -1).max(axis=0)
  outside = np.where(chosen, np.int64(1) << 40, key).min(axis=0)
  return inside <= outside

def exact_mean(values, beta):
  """ The mean of each column of `values` [beta, d], summed exactly and rounded once to fp64: NaN if a value is
  NaN or the column holds +inf and -inf, else +-inf if it holds one, else fsum / beta. """
  v = np.asarray(values, dtype=np.float64)
  out = np.empty(v.shape[1])
  for j in range(v.shape[1]):
    col = v[:, j]
    if np.isnan(col).any() or (np.isposinf(col).any() and np.isneginf(col).any()):
      out[j] = math.nan
    elif np.isinf(col).any():
      out[j] = col[np.isinf(col)][0]
    else:
      out[j] = math.fsum(col.tolist()) / beta
  return out

# ---------------------------------------------------------------------------------------------- #
# K4's order

def k4_sorted(s):
  return from_key(np.sort(to_key(s), axis=0))

def k4_window(srt, med, beta):
  """ The window start: right after the last strict gain of moving the window one place up. """
  theta = srt.shape[0]
  lstar = np.zeros(srt.shape[1], dtype=np.int64)
  with np.errstate(all="ignore"):
    for l in range(theta - beta):
      dlo = abs_key(srt[l] - med)
      dhi = abs_key(srt[l + beta] - med)
      lstar = np.where(dlo > dhi, l + 1, lstar)
  return lstar

def k4_reduce(s, f, wide):
  """ K4's stage 2 on the theta x d stage-1 values: (out fp32 [d], sorted column, window start, median).  The
  64-row K4 adds the window in fp32; K4-wide (`wide`, above 64 rows) adds it in fp64 and rounds the sum to
  fp32 once, before the division. """
  s = np.asarray(s, dtype=F32)
  theta = s.shape[0]
  beta = theta - 2 * f
  srt = k4_sorted(s)
  med = np.where(np.isnan(srt[theta - 1]), F32(np.nan), srt[(theta - 1) // 2]).astype(F32)
  lstar = k4_window(srt, med, beta)
  win = window(srt, lstar, beta)
  acc = np.zeros(s.shape[1], dtype=np.float64 if wide else F32)
  with np.errstate(all="ignore"):
    for q in range(beta):
      acc = acc + win[q].astype(acc.dtype)
    out = (acc.astype(F32) / F32(beta)).astype(F32)
  out[np.isnan(med)] = np.nan
  return out, srt, lstar, med

def window(srt, lstar, beta):
  """ The beta sorted values of each column's window [lstar, lstar + beta). """
  return np.take_along_axis(srt, lstar[None, :] + np.arange(beta)[:, None], axis=0)

def window_mask(srt, lstar, beta):
  pos = np.arange(srt.shape[0])[:, None]
  return (pos >= lstar[None, :]) & (pos < lstar[None, :] + beta)

# ---------------------------------------------------------------------------------------------- #
# Checking an output

def check(out, s, f, wide, what=""):
  """ `out` [d] against stage 2 of the theta x d values `s`: bit for bit K4's order; its window a valid
  closest set around the lower median; within RTOL * max(|exact|, column scale) of the exact mean of that
  window (the scale floored at SUBNORMAL_FLOOR), except where its fp32 sum overflows (then within the
  column's hull).  Returns the errors relative
  to max(|exact|, column scale) (0 where either side is not finite). """
  import parity
  s = np.asarray(s, dtype=F32)
  beta = s.shape[0] - 2 * f
  want, srt, lstar, med = k4_reduce(s, f, wide)
  got = np.asarray(out, dtype=F32)
  parity.assert_bit_exact(got, want, what + " [K4's order]")
  live = ~np.isnan(med)
  ref_med = lower_median(s)
  assert np.array_equal(np.isnan(ref_med), ~live) and np.array_equal(med[live], ref_med[live]), what + " [median]"
  assert closest_set_valid(srt, med, window_mask(srt, lstar, beta))[live].all(), what + " [not a closest set]"
  exact = exact_mean(window(srt, lstar, beta), beta)
  exact[~live] = np.nan
  scale = np.maximum(parity.column_scale(s), SUBNORMAL_FLOOR)
  overflow = np.isfinite(exact) & ~np.isfinite(got)
  parity.assert_close_scaled(got, exact, scale, what + " [exact mean]", exempt=overflow)
  if overflow.any():
    parity.assert_in_hull(got, s, overflow, what + " [overflow]")
  return relative_error(got, exact, scale)

def relative_error(got, exact, scale):
  got = np.asarray(got, dtype=np.float64)
  fin = np.isfinite(got) & np.isfinite(exact)
  rel = np.zeros(got.shape)
  rel[fin] = np.abs(got[fin] - exact[fin]) / np.maximum(np.abs(exact[fin]), scale[fin])
  return rel

# ---------------------------------------------------------------------------------------------- #
# Constructed columns

FLT_MAX = float(np.finfo(F32).max)
CONSTRUCTED = ("median ties", "plateau", "key ties", "signed zeros and subnormals", "infinities", "nan",
               "overflow", "cancellation")

def constructed_columns(theta, f, seed):
  """ theta x len(CONSTRUCTED) fp32 stage-1 values, one column per case, rows shuffled:
    median ties      half the column equal to its median, the rest spread either side;
    plateau          beta + 3 equal values (the window moves along equal keys), the rest spread;
    key ties         values med +- k for k = 1, 2, ...: every key but the median's ties across the window edges;
    signed zeros and subnormals  -0, +0 and +-2^-149 .. 2^-126 (stage 1 adds from 0.0: -0 reaches K4 as +0);
    infinities       one +inf and one -inf among finite values (with f = 0 the window holds both: NaN);
    nan              one NaN: the output is NaN;
    overflow         values near FLT_MAX / 2, all positive: the window's fp32 sum overflows;
    cancellation     +-1e30 in equal numbers around small values. """
  rng = np.random.default_rng(seed)
  beta = theta - 2 * f
  cols = []
  spread = lambda k: rng.uniform(-4., 4., k)
  c = spread(theta)
  c[: (theta + 1) // 2] = 1.
  cols.append(c)
  c = spread(theta)
  c[: min(theta, beta + 3)] = 2.5
  cols.append(c)
  k = np.arange(theta) - (theta - 1) // 2
  cols.append(3. + np.sign(k) * np.ceil(np.abs(k) / 2.))
  tiny = 2. ** -149
  cols.append(np.array([-0., 0., tiny, -tiny, 2. ** -130, -2. ** -127, 2. ** -126])[rng.integers(0, 7, theta)])
  c = spread(theta)
  c[0], c[-1] = np.inf, -np.inf
  cols.append(c)
  c = spread(theta)
  c[theta // 2] = np.nan
  cols.append(c)
  cols.append(FLT_MAX / 2. * rng.uniform(0.9, 1., theta))
  c = rng.uniform(-1., 1., theta)
  h = theta // 3
  c[:h], c[h:2 * h] = 1e30, -1e30
  cols.append(c)
  out = np.stack(cols, axis=1).astype(F32)
  return out[rng.permutation(theta)]
