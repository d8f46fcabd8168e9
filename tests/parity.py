# coding: utf-8
"""Parity rules shared by the oracle-vs-golden (CPU) and CUDA-vs-oracle/golden (GPU) tests.

Bars (BASELINE.json north_star; SURVEY.md §0.6-0.7, §7.3, Appendix A):
  * selection indices / orders: bit-exact (aliased Byzantine rows are one object in the
    reference, so indices >= n_honest are equivalent);
  * values that are a fixed-order fp32 reduction of selected rows (average, krum, brute,
    aksel, cge, bulyan stage 1) and values that are an input element (median): bit-exact
    (value equality: -0.0 == +0.0, NaN == NaN);
  * trmean: bit-exact, except the trailing partial 32-column block (`d mod 32` columns)
    where ATen's vectorised `mean(dim=0)` switches to another summation order on the
    AVX-512 box the goldens were generated on (<= 1e-6 relative there);
  * closest-m means (phocas, meamed, bulyan stage 2): the reference sums in `topk`'s
    unspecified order -> 1e-6 relative to the magnitude of the summed values wherever the
    chosen values are unique, non-finite ones included (`closest_ambiguous`).  Exempt: keys
    tied across the selection boundary between different values (any valid resolution is
    accepted), a NaN centre, and columns whose magnitudes add up past FLT_MAX (the overflow
    itself depends on the order).  There the oracle gets the column-range check, and the
    kernels are held to their restated order (tests/closest_columns.py for Phocas and MeaMed,
    tests/bulyan_columns.py for Bulyan's stage 2);
  * distances and norms (krum, bulyan, brute, cge scores; the clip norm; the study scalars):
    ATen's fp32 `norm()` / `dot()` -> +inf once the sum of squares passes FLT_MAX, squares
    below 2^-150 are 0.  Not pinned: a sum within an ulp of the overflow boundary, and sums
    whose squares are partly subnormal, where ATen's fp32 order and the kernels' FFMA
    (unrounded square) may round differently.  The golden stacks keep every sum of squares
    at least 2x away from FLT_MAX.
"""

import numpy as np

RTOL = 1e-6   # the tolerance BASELINE.json's north_star states for float reductions
FLT_MAX = float(np.finfo(np.float32).max)

def equal_values(a, b):
  """ Element-wise value equality with NaN == NaN (and -0.0 == +0.0). """
  a = np.asarray(a)
  b = np.asarray(b)
  return (a == b) | (np.isnan(a) & np.isnan(b))

def assert_bit_exact(got, ref, what=""):
  got = np.asarray(got)
  ref = np.asarray(ref)
  assert got.shape == ref.shape, f"{what}: shape {got.shape} vs {ref.shape}"
  ok = equal_values(got, ref)
  if not ok.all():
    bad = np.flatnonzero(~ok)
    j = int(bad[0])
    raise AssertionError(f"{what}: {bad.size}/{ok.size} values differ, first at {j}: got {got[j]!r} ref {ref[j]!r}")

def assert_close_scaled(got, ref, scale, what="", rtol=RTOL, exempt=None):
  """ |got - ref| <= rtol * max(|ref|, scale) wherever not exempt; NaN/inf must match. """
  got = np.asarray(got, dtype=np.float64)
  ref = np.asarray(ref, dtype=np.float64)
  scale = np.broadcast_to(np.asarray(scale, dtype=np.float64), ref.shape)
  fin = np.isfinite(ref) & np.isfinite(got)
  with np.errstate(all="ignore"):
    ok = np.where(fin, np.abs(got - ref) <= rtol * np.maximum(np.abs(ref), scale), equal_values(got, ref))
  if exempt is not None:
    ok = ok | exempt
  if not ok.all():
    bad = np.flatnonzero(~ok)
    j = int(bad[0])
    raise AssertionError(f"{what}: {bad.size}/{ok.size} values out of tolerance, first at {j}: got {got[j]!r} ref {ref[j]!r} scale {scale[j]!r}")

def column_scale(rows):
  """ Magnitude of the summed values: mean |x| over the finite entries of each column. """
  with np.errstate(invalid="ignore"):          # signalling NaN payloads
    rows = np.asarray(rows, dtype=np.float64)
  fin = np.isfinite(rows)
  cnt = np.maximum(fin.sum(axis=0), 1)
  return np.where(fin, np.abs(rows), 0.).sum(axis=0) / cnt

def assert_trmean(got, ref, rows, what=""):
  """ rows: the [n, d] inputs (tolerance on the tail columns is relative to the magnitude
  of the summed values, as the mean may cancel). """
  d = ref.shape[0]
  body = d - d % 32
  assert_bit_exact(got[:body], ref[:body], what + " [body]")
  if body < d:
    assert_close_scaled(got[body:], ref[body:], column_scale(np.asarray(rows)[:, body:]), what + " [ATen tail columns]")

def _magnitude_key(x):
  """ fl32|x| as ordered integers, every NaN (any sign or payload) largest. """
  x = np.asarray(x, dtype=np.float32)
  return np.where(np.isnan(x), np.int32(0x7fffffff), x.view(np.int32) & np.int32(0x7fffffff))

def _value_key(x):
  """ Integers equal exactly where the fp32 values are equal as values (-0 == +0, NaN == NaN). """
  x = np.asarray(x, dtype=np.float32)
  return np.where(np.isnan(x), np.int32(0x7fffffff), np.where(x == 0, np.int32(0), x.view(np.int32)))

def value_ambiguous(rows, m, center):
  """ Coordinates where the multiset of the m values with the smallest keys fl32|fl32(x - c)| (NaN
  keys largest) is not unique: keys tie across the selection boundary and the tied entries are not
  all the same value.  A tie among equal values (a plateau, aliased rows, NaN keys all from +inf)
  leaves the chosen values, hence the mean up to summation order, unique. """
  rows = np.asarray(rows, dtype=np.float32)
  n = rows.shape[0]
  if m >= n:
    return np.zeros(rows.shape[1], dtype=bool)
  with np.errstate(all="ignore"):
    key = _magnitude_key(rows - np.asarray(center, dtype=np.float32)[None, :])
  sk = np.sort(key, axis=0)
  tied = (key == sk[m - 1][None, :]) & (sk[m - 1] == sk[m])[None, :]
  val = _value_key(rows).astype(np.int64)
  lo = np.where(tied, val, np.int64(1) << 40).min(axis=0)
  hi = np.where(tied, val, -(np.int64(1) << 40)).max(axis=0)
  return tied.any(axis=0) & (lo != hi)

def closest_ambiguous(rows, m, center):
  """ Coordinates where the reference's closest-m mean is not pinned down, so that any valid
  resolution is accepted there: the chosen values are not unique (`value_ambiguous`), the centre is
  NaN (the reference then ranks every entry on NaN keys, so which m it averages is unspecified), or
  the column's magnitudes add up past FLT_MAX (the reference sums in `topk`'s unspecified order, so
  +inf, -inf or a finite mean are all possible there).  Everywhere else, infinities and NaN included,
  the chosen values are unique and the mean is compared. """
  rows = np.asarray(rows, dtype=np.float32)
  with np.errstate(all="ignore"):
    magnitude = np.where(np.isfinite(rows), np.abs(rows.astype(np.float64)), 0.).sum(axis=0)
  return value_ambiguous(rows, m, center) | np.isnan(np.asarray(center, dtype=np.float32)) | (magnitude > FLT_MAX)

def assert_in_hull(got, rows, mask, what=""):
  """ On exempt coordinates a mean of column entries must still lie within the column's
  finite range (or be non-finite when the column holds non-finite entries, or when its
  entries are large enough for an fp32 partial sum to overflow in some summation order). """
  with np.errstate(invalid="ignore"):          # signalling NaN payloads
    rows = np.asarray(rows, dtype=np.float64)
    got = np.asarray(got, dtype=np.float64)
  idx = np.flatnonzero(mask)
  for j in idx:
    col = rows[:, j]
    fin = col[np.isfinite(col)]
    if not np.isfinite(got[j]):
      assert fin.size < col.size or np.abs(fin).sum() > FLT_MAX, f"{what}: non-finite result at {j} from a finite column"
    elif fin.size:
      lo, hi = fin.min(), fin.max()
      tol = RTOL * max(abs(lo), abs(hi), 1e-30)
      assert lo - tol <= got[j] <= hi + tol, f"{what}: result {got[j]} at {j} outside column range [{lo}, {hi}]"
