# coding: utf-8
"""Phocas and MeaMed (trmean.py:35-109) column by column: a restatement of K1's closest epilogue
(`closest_pairs` / `closest_pairs_static` in k1_select.cuh) and an exact reference to check it with.
Test infrastructure only: plain NumPy, no GPU.

Both rules average the m = n - f values of each column whose keys fl32|fl32(x - c)| are smallest, c the
trimmed mean (Phocas) or the lower median (MeaMed), NaN keys largest.  `k1_closest` restates the kernel
step by step: the column sorted by float_to_key (-0 before +0, NaN last), for each l < f the closer of
s[l] and s[l + m] (compared as magnitude bits, a NaN key largest, ties to s[l]), those f values added in
fp32 from +0.0 in order l = 0..f-1, then the core s[f..m-1], one fp32 division by m, and NaN where the
centre is NaN.  Where the chosen values are unique (not `value_ambiguous`) the reference's mean differs
from it only by summation order; `sum_bound` states by how much.  Where the values are not unique the
kernel's choice is still a valid closest set (`closest_set_valid`), and the GPU tests hold the kernels to
`k1_closest` bit for bit on every column."""

import numpy as np

import bulyan_columns as bc
import parity
from oracle import byzoracle as orc

F32 = np.float32
U = 2. ** -24
MODES = ("phocas", "meamed")

to_key, from_key, abs_key = bc.to_key, bc.from_key, bc.abs_key
value_ambiguous = parity.value_ambiguous

def center(x, f, mode):
  """ The centre K1 computes (bit-exact with the oracle): trmean(x, f) or the lower median, NaN if the
  column holds a NaN. """
  x = np.asarray(x, dtype=F32)
  return orc.trmean(x, f) if mode == "phocas" else orc.median(x)

def k1_closest(x, f, mode, c=None):
  """ K1's closest epilogue on the [n, d] rows x: (out fp32 [d], chosen bool [n, d] in the rows' order).
  f = 0 (m = n) compares no pairs: the whole column summed in rank order. """
  x = np.asarray(x, dtype=F32)
  n, d = x.shape
  m = n - f
  assert 0 <= f < m, (n, f)
  c = center(x, f, mode) if c is None else np.asarray(c, dtype=F32)
  keys = to_key(x)
  order = np.argsort(keys, axis=0, kind="stable")
  s = from_key(np.take_along_axis(keys, order, axis=0))
  picked = np.zeros((n, d), dtype=bool)
  picked[f:m] = True
  acc = np.zeros(d, dtype=F32)
  with np.errstate(all="ignore"):
    for l in range(f):
      up = abs_key(s[l] - c) > abs_key(s[l + m] - c)
      acc = (acc + np.where(up, s[l + m], s[l])).astype(F32)
      picked[l], picked[l + m] = ~up, up
    for k in range(f, m):
      acc = (acc + s[k]).astype(F32)
    out = (acc / F32(m)).astype(F32)
  out[np.isnan(c)] = np.nan
  chosen = np.zeros((n, d), dtype=bool)
  np.put_along_axis(chosen, order, picked, axis=0)
  return out, chosen

def closest_set_valid(x, c, chosen):
  """ Per column: no chosen key exceeds an unchosen key (NaN keys largest). """
  return bc.closest_set_valid(x, c, chosen)

def chosen_values(x, chosen):
  """ The m chosen values of each column, [m, d], in row order. """
  x = np.asarray(x, dtype=F32)
  m = int(chosen[:, 0].sum()) if x.shape[1] else 0
  assert (chosen.sum(axis=0) == m).all()
  return x.T[chosen.T].reshape(x.shape[1], m).T

def exact_mean(values):
  """ The mean of each column of `values` [m, d], summed exactly (math.fsum): NaN if a value is NaN or the
  column holds +inf and -inf, else +-inf if it holds one (the rules of bulyan_columns.exact_mean). """
  return bc.exact_mean(values, np.asarray(values).shape[0])

def sum_bound(values, exact):
  """ A rigorous bound on |out - exact| for any fixed order of fp32 additions of the m values and one fp32
  division by m: the sum errs by at most gamma_{m-1} sum |v|, the division rounds once more (the exact mean
  itself is fsum / m in fp64, off by 2^-52 of it). """
  v = np.asarray(values, dtype=np.float64)
  m = v.shape[0]
  g = (m - 1) * U / (1 - (m - 1) * U)
  with np.errstate(invalid="ignore"):         # columns holding +-inf or NaN: the bound is NaN there
    mag = np.abs(v).sum(axis=0) / m
    return (1 + U) * g * mag + (U + 2. ** -50) * np.abs(exact) + 2. ** -149

def check_restatement(x, f, mode, what=""):
  """ `k1_closest` against the exact reference on every column of x: a valid closest set of m values
  around a live centre, NaN where the centre is NaN, and within `sum_bound` of the exact mean of its set
  (within the column's hull where the fp32 sum overflows and the exact mean does not).  Returns
  (out, chosen, centre). """
  x = np.asarray(x, dtype=F32)
  n = x.shape[0]
  m = n - f
  c = center(x, f, mode)
  out, chosen = k1_closest(x, f, mode, c)
  assert (chosen.sum(axis=0) == m).all(), what
  live = ~np.isnan(c)
  assert np.isnan(out[~live]).all(), what + " [NaN centre]"
  assert closest_set_valid(x, c, chosen)[live].all(), what + " [not a closest set]"
  vals = chosen_values(x, chosen)
  exact = exact_mean(vals)
  with np.errstate(invalid="ignore"):
    err = np.abs(out.astype(np.float64) - exact)
  fin = live & np.isfinite(exact)
  overflow = fin & ~np.isfinite(out)
  inside = fin & ~overflow
  bad = inside & ~(err <= sum_bound(vals, exact))
  assert not bad.any(), f"{what}: out of the summation bound at {np.flatnonzero(bad)[:5]}"
  nonfin = live & ~np.isfinite(exact)
  assert parity.equal_values(out[nonfin], exact[nonfin]).all(), what + " [non-finite means]"
  if overflow.any():
    parity.assert_in_hull(out, x, overflow, what + " [overflow]")
  return out, chosen, c

def check_kernel(got, x, f, mode, what="", want=None, c=None):
  """ A kernel's output against `k1_closest`, value for value (NaN == NaN) on every column, and, where the
  chosen values are unique, against the oracle within the scaled bar of tests/parity.py.  `c`: the centre,
  when the caller has it already. """
  x = np.asarray(x, dtype=F32)
  n = x.shape[0]
  c = center(x, f, mode) if c is None else np.asarray(c, dtype=F32)
  if want is None:
    want = k1_closest(x, f, mode, c)[0]
  parity.assert_bit_exact(np.asarray(got, dtype=F32), want, what + " [K1's closest epilogue]")
  ref = orc.closest_mean(x, n - f, c)
  parity.assert_close_scaled(got, ref, parity.column_scale(x), what + " [oracle]", rtol=parity.RTOL * max(1., (n - f) / 64),
                             exempt=parity.closest_ambiguous(x, n - f, c))

# ---------------------------------------------------------------------------------------------- #
# Constructed columns

FLT_MAX = float(np.finfo(F32).max)
NAN_BITS = np.array([0xffc00000, 0x7f800001, 0xffffffff, 0x7fc00000], dtype=np.uint32).view(F32)   # -NaN, payloads
CONSTRUCTED = ("+inf", "-inf", "+inf beyond f", "nan within f", "nan beyond f", "single nan", "+inf majority",
               "both infinities", "nan signs and payloads", "key ties", "plateau", "all equal",
               "signed zeros and subnormals", "overflow", "cancellation")

def constructed_columns(n, f, seed):
  """ n x len(CONSTRUCTED) fp32 rows, one column per case, rows shuffled (n >= 3, 1 <= f < n - f):
    +inf, -inf               one infinity among spread values;
    +inf beyond f            f + 1 entries +inf: Phocas' centre is +inf, finite keys +inf, +inf keys NaN;
    nan within f             f NaNs: Phocas' centre stays finite and its NaN keys are never chosen;
    nan beyond f             f + 1 NaNs: Phocas' centre is NaN;
    single nan               one NaN: MeaMed's centre is NaN;
    +inf majority            n - (n - 1) // 2 entries +inf: MeaMed's (and Phocas') centre is +inf;
    both infinities          f + 1 of +inf and of -inf where that leaves the median finite (n >= 2f + 4),
                             else one of each: MeaMed's core then holds both (NaN);
    nan signs and payloads   -NaN, signalling and all-ones NaNs, min(f, 4) of them;
    key ties                 values 3 +- k: keys tie across both window edges with different values;
    plateau                  m + 3 equal values (n when shorter): the boundary tie is between equal values;
    all equal                every value 0.75;
    signed zeros and subnormals  -0, +0 and +-2^-149 .. 2^-126 (subnormal keys);
    overflow                 values near FLT_MAX / 2, all positive: the fp32 sum overflows;
    cancellation             +-1e30 in equal numbers around small values. """
  rng = np.random.default_rng(seed)
  m = n - f
  spread = lambda: rng.uniform(-4., 4., n)
  cols = []
  for v in (np.inf, -np.inf):
    c = spread()
    c[0] = v
    cols.append(c)
  c = spread()
  c[: f + 1] = np.inf
  cols.append(c)
  for k in (f, f + 1, 1):
    c = spread()
    c[:k] = np.nan
    cols.append(c)
  c = spread()
  c[: n - (n - 1) // 2] = np.inf
  cols.append(c)
  c = spread()
  k = f + 1 if n >= 2 * f + 4 else 1
  c[:k], c[k:2 * k] = np.inf, -np.inf
  cols.append(c)
  c = spread().astype(F32)
  k = min(f, 4)
  c[:k] = NAN_BITS[:k]
  cols.append(c)
  k = np.arange(n) - (n - 1) // 2
  cols.append(3. + np.sign(k) * np.ceil(np.abs(k) / 2.))
  c = spread()
  c[: min(n, m + 3)] = 2.5
  cols.append(c)
  cols.append(np.full(n, 0.75))
  tiny = 2. ** -149
  cols.append(np.array([-0., 0., tiny, -tiny, 2. ** -130, -2. ** -127, 2. ** -126])[rng.integers(0, 7, n)])
  cols.append(FLT_MAX / 2. * rng.uniform(0.9, 1., n))
  c = rng.uniform(-1., 1., n)
  h = n // 3
  c[:h], c[h:2 * h] = 1e30, -1e30
  cols.append(c)
  out = np.stack([np.asarray(c, dtype=F32) for c in cols], axis=1)
  return out[rng.permutation(n)]

def stack(n, f, d, seed):
  """ [n, d] rows for the GPU: finite noise with exact ties, and copies of the constructed columns placed at
  strides 1 to 5 from the start of successive 128-column blocks, so that some VEC groups hold only finite
  columns (among them finite constructed ones, which then take the FMNMX network) and neighbouring ones
  mix finite and non-finite columns (the integer-key network, finite columns included). """
  rng = np.random.default_rng(seed)
  x = rng.standard_normal((n, d)).astype(F32)
  x[:, 1::5] = np.round(x[:, 1::5] * 2) / 2
  k = len(CONSTRUCTED)
  for copy, stride in enumerate((1, 2, 3, 4, 5)):
    j0 = 128 * copy + copy % 4
    cols = j0 + stride * np.arange(k)
    if cols[-1] >= d:
      break
    x[:, cols] = constructed_columns(n, f, seed * 8 + copy)
  return x
