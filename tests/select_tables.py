# coding: utf-8
"""Constructed tables of squared distances for the scoring / selection step (K5), and the
expectations the oracle derives from them.  Test infrastructure only: plain NumPy, no GPU.

A table is a stack of R fp64 blocks `[R][n*n]` (or `[R][n]` for row keys), the partial blocks R
ranks publish in the d-sharded path; only entries (i, j) with i < j carry values.  The selection
must be the oracle's on `fp32_norm(sum_parts(parts))`, where `sum_parts` adds the blocks in rank
order.  The builders aim at the places a kernel can be subtly wrong and random rows never reach:
  * straddling splits: R blocks whose sum lies within a few fp64 ulps of `mid**2`, `mid` the
    midpoint of two adjacent fp32 values, so that another summation order of the blocks gives
    another fp32 distance, and an order that hinges on that one distance;
  * a Neumaier corpus: scores whose order depends on CPython's compensated `sum()`;
  * non-finite and overflowing sums at the fp32 rounding point to +inf;
  * planted brute subsets at the edges of the threads' rank ranges;
  * Bulyan stacks at the exact boundary of its degenerate rule.
`interleaved_sum` restates the order an earlier K5 used (interleaved classes of blocks), so the
self-checks can show the straddling splits tell the two orders apart."""

import itertools
import math

import numpy as np

from oracle import byzoracle as orc

F32 = np.float32
FLT_MAX = float(np.finfo(F32).max)
# the fp64 sum of squares at which fp32 rounding reaches +inf (a tie, rounded to even: +inf)
INF_TIE = FLT_MAX + 2. ** 103
INF_BELOW = np.nextafter(INF_TIE, 0.)
K5_THREADS = 1024

def tail_threads(n):
  """ Threads of the ring kernel's CTA, which runs K5 in its tail (ring_shape in k2_ring.cu):
  6 warps up to 15 distinct rows, 12 warps up to 35, 16 warps beyond. """
  return 192 if n <= 15 else 384 if n <= 35 else 512

# ---------------------------------------------------------------------------------------------- #
# Summation orders

def pick_slices(n, nparts, threads=K5_THREADS, budget=48 * 1024):
  """ Number of interleaved classes of the earlier K5 (the order `interleaved_sum` restates). """
  s = max(1, min(budget // (n * n * 8), 8, nparts))
  while threads % s:
    s -= 1
  return s

def interleaved_sum(parts, slices):
  """ Blocks split into `slices` classes p mod slices, each class summed from 0.0 in ascending p,
  then the class sums added from 0.0 in ascending class: not rank order unless slices == 1, or
  slices == nparts with nparts a power of two. """
  parts = np.asarray(parts, dtype=np.float64)
  out = np.zeros(parts.shape[1:])
  with np.errstate(all="ignore"):
    for s in range(slices):
      acc = np.zeros(parts.shape[1:])
      for p in range(s, parts.shape[0], slices):
        acc = acc + parts[p]
      out = out + acc
  return out

def interleaved_differs(n, R):
  """ (n, R) where the earlier K5 (select / select_peers) did not add the blocks in rank order. """
  s = pick_slices(n, R)
  return s > 1 and not (s == R and R & (R - 1) == 0)

def naive_sum(v):
  acc = 0.
  for x in v:
    acc += x
  return acc

# ---------------------------------------------------------------------------------------------- #
# Straddling splits

def _fp32_sqrt(s):
  return float(orc.fp32_norm(s))

def reverse_sum(parts):
  """ The blocks added in reverse rank order, ((p[R-1] + p[R-2]) + ...) + p0. """
  return orc.sum_parts(np.asarray(parts)[::-1])

def pairwise_sum(parts):
  """ The blocks added as a pairwise tree: the sums of the two halves (the first one the larger) added. """
  parts = np.asarray(parts, dtype=np.float64)
  if parts.shape[0] == 1:
    return parts[0].copy()
  h = (parts.shape[0] + 1) // 2
  with np.errstate(all="ignore"):
    return pairwise_sum(parts[:h]) + pairwise_sum(parts[h:])

def other_orders(R):
  """ The alternative summers that can round R blocks differently from rank order: the reverse from 3 blocks
  on (two blocks commute), the pairwise tree from 4 on (with 3 it is rank order). """
  return ([reverse_sum] if R >= 3 else []) + ([pairwise_sum] if R >= 4 else [])

def straddle_split(R, rng, y, key=_fp32_sqrt, alt_slices=None, square=True, tries=200_000, alts=()):
  """ R non-negative fp64 blocks of one entry whose rank-order sum lies within a few ulps of the
  square of the midpoint between y and its upper fp32 neighbour (of the midpoint itself when not
  `square`).  With `alt_slices`, only a split whose rank-order and interleaved sums give different
  keys is accepted; with `alts` (summers of a [R][1] stack), only a split that every one of them
  rounds to another key.  Returns (blocks, key of the rank-order sum). """
  y = F32(y)
  mid = (float(y) + float(np.nextafter(y, F32(np.inf)))) / 2.      # exact in fp64
  target = mid * mid if square else mid
  for _ in range(tries):
    w = rng.uniform(0.05, 1., R)
    parts = w / w.sum() * target
    # a few ulps either side of the target, so that some order lands on each side
    parts[-1] += rng.integers(-4, 5) * math.ulp(target)
    parts = np.maximum(parts, 0.)
    got = key(orc.sum_parts(parts[:, None])[0])
    if any(got == key(alt(parts[:, None])[0]) for alt in alts):
      continue
    if alt_slices is None or R == 1:
      return parts, got
    if got != key(interleaved_sum(parts[:, None], alt_slices)[0]):
      return parts, got
  raise RuntimeError(f"no straddling split for R = {R}")

def straddle_table(n, R, seed, alt_slices=None, alts=()):
  """ n x n blocks in which the order of Krum / Bulyan rows 0-3 and brute's best pair hinge on one
  distance: d(0, 1) is the straddled y or its upper neighbour, d(2, 3) is exactly y, every other
  distance 3.0.  Rows 0 and 1 score d(0, 1) + c and rows 2 and 3 y + c (exact sums): a tie kept in
  index order when d(0, 1) = y, rows 2 and 3 first otherwise; brute with subsets of two picks
  {0, 1} or {2, 3} the same way.  Returns (parts [R][n*n], d01). """
  assert n >= 4
  rng = np.random.default_rng(seed)
  y = F32(rng.uniform(1., 2.))
  split, d01 = straddle_split(R, rng, y, alt_slices=alt_slices, alts=alts)
  table = np.full((n, n), 9.)
  table[2, 3] = float(y) * float(y)
  parts = np.zeros((R, n, n))
  w = rng.permutation(R)                       # the other pairs: exact shares of their square
  for r in range(R):
    parts[r] = np.triu(table, 1) / R if R & (R - 1) == 0 else (np.triu(table, 1) if r == w[0] else 0.)
  parts[:, 0, 1] = split
  return parts.reshape(R, n * n), d01

def straddle_keys(n, R, seed, sqrt_norm, alt_slices=None, alts=()):
  """ [R][n] row keys: key 0 straddles, key 1 is exactly y (its lower neighbour), the rest larger.
  The stable order starts [0, 1] when key 0 rounds to y, [1, 0] otherwise. """
  rng = np.random.default_rng(seed)
  y = F32(rng.uniform(1., 2.))
  if sqrt_norm:
    split, _ = straddle_split(R, rng, y, alt_slices=alt_slices, alts=alts)
    rest = (float(y) * float(y), 16.)
  else:
    split, _ = straddle_split(R, rng, y, key=lambda s: float(F32(s)), alt_slices=alt_slices, square=False, alts=alts)
    rest = (float(y), 4.)
  parts = np.zeros((R, n))
  parts[:, 0] = split
  if n > 1:
    parts[0, 1] = rest[0]
    parts[0, 2:] = rest[1] + np.arange(n - 2)
  return parts

# ---------------------------------------------------------------------------------------------- #
# The oracle on a stack of blocks

def distances(parts, n, map_nonfinite=True):
  """ The distance table the selection sees: fp32 norms of the rank-order sum, symmetric. """
  sq = orc.sum_parts(parts).reshape(n, n)
  D = np.triu(orc.fp32_norm(sq), 1)
  D = D + D.T
  if map_nonfinite:
    D = np.where(np.isfinite(D), D, np.inf)
  return D

def bulyan_status(scores, n, f, m):
  """ bulyan_stage1's degenerate rule: 2 when the reference fails on gradients[None]. """
  finite = sum(1 for s in scores if math.isfinite(s))
  mi = m
  for i in range(n - 2 * f - 2):
    mi = min(mi, n - f - 2 - i)
    if i >= 1 and finite - i < mi:
      return 2
  return 0

def expect_krum(parts, n, f):
  return orc.krum_order(distances(parts, n), f)[0]

def expect_bulyan(parts, n, f, m):
  order, scores = orc.bulyan_order(distances(parts, n), f, m)
  return order, bulyan_status(scores, n, f, m)

def expect_brute(parts, n, f):
  try:
    return orc.brute_selection(distances(parts, n, False), f), 0
  except AssertionError:
    return list(range(n - f)), 1

def expect_rowdist(parts, n, sqrt_norm):
  sq = orc.sum_parts(parts)
  with np.errstate(all="ignore"):
    key = orc.fp32_norm(sq) if sqrt_norm else sq.astype(F32).astype(np.float64)
  if sqrt_norm:
    key = np.where(np.isfinite(key), key, np.inf)
  return sorted(range(n), key=lambda i: (math.isnan(key[i]), 0. if math.isnan(key[i]) else float(key[i]), i))

# ---------------------------------------------------------------------------------------------- #
# Neumaier corpus

def _krum_scores(D, f, summer):
  n = D.shape[0]
  out = []
  for i in range(n):
    d = sorted(float(D[i, j]) for j in range(n) if j != i)
    out.append(summer(d[:n - f - 1]))
  return out

def neumaier_corpus(count=40, seed=0, max_tries=5_000):
  """ (n, f, D) tables of exact fp32 distances, n in 8..64, f in 0..(n-3)//2, kept when the naive
  left-to-right score order differs from the one Python's `sum()` gives.  Every distance is one
  huge power of two (2^24, 2^29, 2^53 or 2^60 per table) except a sparse set of small ones (1, 2, 3,
  5): rows of the same degree in that set tie on their huge part, the naive sum rounds their small
  parts away where the compensated one keeps them. """
  rng = np.random.default_rng(seed)
  out = []
  for _ in range(max_tries):
    n = int(rng.integers(8, 65))
    f = int(rng.integers(0, (n - 3) // 2 + 1))
    big = 2. ** int(rng.choice([24, 29, 53, 60]))
    small = np.array([1., 2., 3., 5.])[rng.integers(0, 4, (n, n))]
    D = np.where(rng.random((n, n)) < 3. / n, small, big)
    D = np.triu(D, 1)
    D = D + D.T
    if orc._stable_argsort(_krum_scores(D, f, sum)) != orc._stable_argsort(_krum_scores(D, f, naive_sum)):
      out.append((n, f, D))
      if len(out) == count:
        return out
  raise RuntimeError(f"only {len(out)} discriminating tables")

def neumaier_corpus_wide(count=24, seed=0, max_tries=200):
  """ (n, f, D) tables of exact fp32 distances, n in 65..128, f in 0..(n-3)//2 (Krum counts n - f - 1 up to 127
  terms), built rather than sampled: rows 2k and 2k + 1 are at a small integer distance s_k of each other and at
  one huge power of two B (2^53 or 2^60) of every other row.  A row's score is s_k + (count - 1) B: the naive sum
  rounds s_k at every power of two the partial sum crosses, the compensated one once, so some pairs the naive sum
  ties (or inverts) are strictly ordered by sum().  The s_k are drawn within a few ulps of (count - 1) B and put in
  descending order, so that a tie kept in index order is the inverse of the compensated order.  Only tables whose
  naive and compensated Krum orders differ are kept. """
  rng = np.random.default_rng(seed)
  out = []
  first = [(128, 0), (127, 0), (65, 31), (96, 1)]          # the longest counts, and the shortest
  for t in range(max_tries):
    n = first[t][0] if t < len(first) else int(rng.integers(65, 129))
    f = first[t][1] if t < len(first) else int(rng.choice([0, 1, int(rng.integers(0, (n - 3) // 2 + 1)), (n - 3) // 2]))
    big = 2. ** int(rng.choice([53, 60]))
    ulp = math.ulp((n - f - 2) * big)
    s = np.sort(rng.integers(1, int(4 * ulp) + 2, n // 2).astype(np.float64))[::-1]
    D = np.full((n, n), big)
    for k, v in enumerate(s):
      D[2 * k, 2 * k + 1] = D[2 * k + 1, 2 * k] = v
    np.fill_diagonal(D, 0.)
    if orc._stable_argsort(_krum_scores(D, f, sum)) != orc._stable_argsort(_krum_scores(D, f, naive_sum)):
      out.append((n, f, D))
      if len(out) == count:
        return out
  raise RuntimeError(f"only {len(out)} discriminating tables")

def square_blocks(D, R=1):
  """ [R][n*n] blocks whose rank-order sum is exactly D**2 above the diagonal (R a power of two:
  equal shares, each exact). """
  sq = np.triu(D * D, 1)
  return np.stack([sq / R] * R).reshape(R, -1)

def tie_table(n, seed, levels=(1., 2.)):
  """ n x n exact fp32 distances drawn from a few values: rows hold long runs of equal distances (ties in the
  row sort, broken by column index) and many rows score alike (ties in the stable argsort, kept in index
  order). """
  rng = np.random.default_rng(seed)
  D = np.asarray(levels, dtype=np.float64)[rng.integers(0, len(levels), (n, n))]
  D = np.triu(D, 1)
  return D + D.T

# ---------------------------------------------------------------------------------------------- #
# Brute: planted subsets

def unrank(rank, n, k):
  """ The rank-th k-subset of range(n) in lexicographic order, by the scheme of brute_from_table. """
  out, x, r = [], 0, rank
  for pos in range(k):
    while True:
      c = math.comb(n - 1 - x, k - 1 - pos)
      if c > r:
        break
      r -= c
      x += 1
    out.append(x)
    x += 1
  return out

def rank_of(sub, n):
  k = len(sub)
  r, prev = 0, -1
  for pos, x in enumerate(sub):
    for y in range(prev + 1, x):
      r += math.comb(n - 1 - y, k - 1 - pos)
    prev = x
  return r

def thread_of(rank, total, threads):
  per = -(-total // threads)
  return rank // per

def planted_targets(total, threads):
  """ (r1, r2, what): pairs of ranks r1 <= r2 at the edges of the threads' rank ranges, for
  `threads` threads each scanning `per = ceil(total / threads)` consecutive ranks. """
  per = -(-total // threads)
  last = (total - 1) // per                      # the last thread with ranks (idle ones follow)
  t = min(threads // 2 + 3, last - 1)            # a thread with a successor
  out = [(0, total - 1, "rank 0 and the last rank")]
  if t >= 0:
    out += [(t * per, t * per + per - 1, "first and last rank of one thread"),
            (t * per + per - 1, (t + 1) * per, "last rank of thread t, first of thread t + 1")]
  if per >= 2:
    out.append((t * per + 1, t * per + 2 if per > 2 else t * per + 1, "two ranks of one thread"))
  if last >= 40:
    out += [(33 * per, 34 * per + per - 1, "two threads of one warp"),
            (32 * per - 1, 32 * per, "last rank of warp 0, first of warp 1"),
            (5 * per, 40 * per, "different warps")]
  return [(a, b, w) for a, b, w in out if 0 <= a <= b < total]

def planted_table(n, f, r1, r2, strict=False):
  """ Distance 1.0 inside S1 = unrank(r1) and S2 = unrank(r2), 2.0 elsewhere (S2's diameter is
  nextafter(1, 2) when `strict`): the two only subsets of diameter <= 1 + ulp, so brute returns
  S1 (the first of a tie, or the strictly smaller).  Returns (D, S1, S2). """
  k = n - f
  S1, S2 = unrank(r1, n, k), unrank(r2, n, k)
  D = np.full((n, n), 2.)
  assert k >= 2
  # a pair of S1 and S2 both keeps 1.0; S2 still holds a pair outside S1 at its diameter
  for S, v in ((S2, float(np.nextafter(F32(1), F32(2))) if strict else 1.), (S1, 1.)):
    for a, b in itertools.combinations(S, 2):
      D[a, b] = D[b, a] = v
  np.fill_diagonal(D, 0.)
  return D, S1, S2

# ---------------------------------------------------------------------------------------------- #
# Non-finite and overflowing entries

NONFINITE_SUMS = [math.nan, math.inf, FLT_MAX, INF_BELOW, INF_TIE]

def nonfinite_table(n, R, seed):
  """ n x n blocks over R ranks with, above the diagonal, finite exact squares mixed with sums that
  are NaN, +inf, FLT_MAX, just below the fp32 rounding point to +inf, and at it (split over the
  blocks so that only the summed table reaches them). """
  rng = np.random.default_rng(seed)
  y = rng.uniform(1., 4., (n, n)).astype(F32).astype(np.float64)
  sq = np.triu(y * y, 1)
  iu = np.triu_indices(n, 1)
  pick = rng.choice(len(iu[0]), size=min(len(iu[0]), max(2, n // 2)), replace=False)
  for q, p in enumerate(pick):
    sq[iu[0][p], iu[1][p]] = NONFINITE_SUMS[q % len(NONFINITE_SUMS)]
  parts = np.zeros((R, n, n))
  parts[0] = sq
  if R > 1:
    # move exact halves of the big sums to the last block: the sum is reached only across blocks
    big = np.isfinite(sq) & (sq > 1e30)
    parts[0][big] = sq[big] / 2.
    parts[R - 1][big] = sq[big] / 2.
  return parts.reshape(R, n * n)

def special_keys(n, seed):
  """ [n] fp64 row sums for Aksel and CGE: NaN, +inf, sums at and just below the fp32 rounding point to +inf,
  FLT_MAX, 1e300, fp32 ties of different fp64 sums (y^2 and y^2 (1 +- 2^-40)), exact squares and 0, shuffled. """
  rng = np.random.default_rng(seed)
  y = float(F32(1.5))
  special = [math.nan, math.inf, INF_TIE, INF_BELOW, FLT_MAX, 1e300, y * y, y * y * (1 + 2. ** -40),
             y * y * (1 - 2. ** -40), 0.]
  rest = rng.integers(1, 6, max(0, n - 3 * len(special))).astype(np.float64) ** 2
  return rng.permutation(np.concatenate([special * 3, rest])[:n])

# ---------------------------------------------------------------------------------------------- #
# Bulyan: degenerate boundary

def bulyan_nan_rows(n, q, seed):
  """ One block: rows 0..q-1 all NaN (every distance to them +inf), the rest exact distances. """
  rng = np.random.default_rng(seed)
  y = rng.uniform(1., 4., (n, n)).astype(F32).astype(np.float64)
  sq = np.triu(y * y, 1)
  sq[:q, :] = math.nan
  sq[:, :q] = math.nan
  return np.triu(sq, 1).reshape(1, n * n)
