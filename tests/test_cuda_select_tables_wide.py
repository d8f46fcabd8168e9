# coding: utf-8
"""GPU tests of phase B above 64 rows (`bz_distance_select`) on constructed tables (tests/select_tables.py).

`k5_blocks_select_wide` adds the R gathered [n*n] blocks in rank order and scores them with
`score_from_floats`, the steps `k5_score_select_wide` (bz_distance's own scoring) shares; Aksel and CGE run
`k5_rowkeys_select_wide` over R [n] blocks.  Every selection is compared bit for bit (order, and Bulyan's
status) with the oracle on `fp32_norm(sum_parts(parts))`:
  * straddling splits that reverse rank order and a pairwise tree round to the other fp32 distance or key;
  * a Neumaier corpus whose Krum order needs CPython's compensated sum, with counts up to 127 terms;
  * NaN, +inf and overflowing sums at the fp32 rounding point to +inf, reached only across blocks;
  * Bulyan's degenerate boundary at every number of NaN rows;
  * row keys with NaN (last for Aksel), +inf, overflow and fp32 ties of different fp64 sums;
  * tables of few distinct distances, where the row sort and the stable argsort meet long runs of ties."""

import math

import numpy as np
import pytest

import select_tables as st
from oracle import byzoracle as orc
from test_cuda_distance_wide import CODES

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NS = [65, 66, 70, 96, 97, 111, 127, 128]

def _lib():
  from byzantinemomentum_b200 import _lib
  return _lib.lib()

def select(rule, parts, n, f=0, m=1):
  """ (order, status) of bz_distance_select on the blocks `parts` [R][n*n] or [R][n]; status -1 when the rule
  writes none. """
  lib = _lib()
  t = torch.tensor(np.ascontiguousarray(parts, dtype=np.float64), device=DEV)
  meta = torch.full((n + 1,), -1, dtype=torch.int32, device=DEV)
  rc = lib.bz_distance_select(CODES[rule], t.data_ptr(), t.shape[0], n, f, m, 0, meta.data_ptr(), meta.data_ptr() + 4 * n,
                              torch.cuda.current_stream().cuda_stream)
  assert rc == 0, lib.bz_last_error()
  torch.cuda.synchronize()
  out = meta.cpu().tolist()
  return out[:n], out[n]

def bulyan_f(n):
  return (n - 3) // 4

def expect_bulyan_sweep(parts, n, f, ms):
  """ {m: (order, status)} of the oracle, the distance table and its sorted rows computed once. """
  D = st.distances(parts, n)
  rows = []
  for i in range(n):
    r = [float(D[i, j]) if j != i else math.inf for j in range(n)]
    r.sort()
    rows.append(r)
  out = {}
  for m in ms:
    scores = [sum(r[:m]) for r in rows]
    out[m] = (orc._stable_argsort(scores), st.bulyan_status(scores, n, f, m))
  return out

def check_pairs(parts, n, what, f_krum=1, bulyan_ms=None):
  """ Krum (its order only: it writes no status) and Bulyan at the given m (default m_max) on the blocks. """
  assert select("krum", parts, n, f_krum)[0] == st.expect_krum(parts, n, f_krum), what
  f = bulyan_f(n)
  m_max = n - f - 2
  for m, want in expect_bulyan_sweep(parts, n, f, bulyan_ms or [m_max]).items():
    assert select("bulyan", parts, n, f, m) == want, (what, m)

@pytest.mark.parametrize("n", NS)
def test_straddling_splits_select_like_the_rank_order_sum(n):
  """ At every block count R in 1..24: the one straddled distance decides the order of rows 0-3; from three
  blocks on, the split is one that reverse rank order (and, from four, a pairwise tree) rounds to the other
  fp32 distance, so a kernel adding the blocks in either order selects other rows. """
  for R in range(1, 25):
    parts, d01 = st.straddle_table(n, R, seed=100 * n + R, alts=st.other_orders(R))
    check_pairs(parts, n, f"n={n} R={R} d01={d01!r}", bulyan_ms=[1, n - bulyan_f(n) - 2])

@pytest.mark.parametrize("sqrt_norm", [0, 1])
def test_rowkeys_straddle_at_every_block_count(sqrt_norm):
  rule = "cge" if sqrt_norm else "aksel"
  for n in NS:
    for R in range(1, 25):
      parts = st.straddle_keys(n, R, seed=R * 101 + n, sqrt_norm=sqrt_norm, alts=st.other_orders(R))
      assert select(rule, parts, n)[0] == st.expect_rowdist(parts, n, sqrt_norm), (n, R, sqrt_norm)

def test_neumaier_corpus():
  """ Krum on every table (f as drawn, counts up to 127 terms) and Bulyan at m = 1 and m_max, on one block and
  on two exact halves. """
  for k, (n, f, D) in enumerate(st.neumaier_corpus_wide()):
    for R in (1, 2):
      parts = st.square_blocks(D, R)
      assert select("krum", parts, n, f)[0] == orc.krum_order(D, f)[0], (k, n, f, R)
      fb = bulyan_f(n)
      for m, want in expect_bulyan_sweep(parts, n, fb, [1, n - fb - 2]).items():
        assert select("bulyan", parts, n, fb, m) == want, (k, n, fb, m, R)

@pytest.mark.parametrize("n", [65, 97, 128])
def test_nonfinite_and_overflowing_sums(n):
  """ NaN, +inf, FLT_MAX, just below and at the fp32 rounding point to +inf, reached only across the blocks:
  Krum and Bulyan map them to +inf. """
  for R in (1, 3, 16):
    parts = st.nonfinite_table(n, R, seed=n + R)
    check_pairs(parts, n, f"n={n} R={R}", bulyan_ms=[1, n - bulyan_f(n) - 2])

@pytest.mark.parametrize("n", [65, 97, 128])
def test_bulyan_degenerate_boundary(n):
  """ q all-NaN rows (their distances +inf) for every q in 0..n, m in {1, 2, m_max - 1, m_max}: the status and
  the order of the oracle and of bulyan_stage1's degenerate rule. """
  f = bulyan_f(n)
  m_max = n - f - 2
  seen = set()
  for q in range(n + 1):
    parts = st.bulyan_nan_rows(n, q, seed=q)
    for m, want in expect_bulyan_sweep(parts, n, f, [1, 2, m_max - 1, m_max]).items():
      assert select("bulyan", parts, n, f, m) == want, (n, q, m)
      seen.add(want[1])
  assert seen == {0, 2}

@pytest.mark.parametrize("n", [65, 100, 128])
def test_aksel_and_cge_special_keys(n):
  """ Row keys with NaN, +inf, sums at and below the fp32 rounding point to +inf, 1e300 and fp32 ties of
  different fp64 sums, split in exact halves over the first and last of R blocks: CGE maps every non-finite
  norm to +inf, Aksel keeps NaN and sorts it last; ties stay in index order. """
  sq = st.special_keys(n, seed=n)
  for R in (1, 2, 17):
    parts = np.zeros((R, n))
    parts[0] = sq / (2 if R > 1 else 1)
    if R > 1:
      parts[R - 1] = sq / 2
    for rule, sqrt_norm in (("aksel", 0), ("cge", 1)):
      want = st.expect_rowdist(parts, n, sqrt_norm)
      assert select(rule, parts, n)[0] == want, (n, R, rule)
  keys = orc.sum_parts(parts).astype(np.float32)
  assert np.isnan(keys).sum() == 3 and st.expect_rowdist(parts, n, 0)[-3:] == sorted(np.flatnonzero(np.isnan(keys)).tolist())

@pytest.mark.parametrize("n", [65, 96, 128])
def test_many_equal_scores(n):
  """ Distances from {1, 2} and from {1}: long runs of equal distances in every row and rows scoring alike, so
  the row sort and the stable argsort over up to 128 columns decide the order by index alone. """
  for seed, levels in ((n, (1., 2.)), (n + 1, (1., 2., 2., 2.)), (n + 2, (1.,))):
    D = st.tie_table(n, seed, levels)
    for R in (1, 4):
      check_pairs(st.square_blocks(D, R), n, f"n={n} levels={levels} R={R}", bulyan_ms=[1, 2, n - bulyan_f(n) - 2])
  D = st.tie_table(n, 0, (1.,))
  assert st.expect_krum(st.square_blocks(D), n, 1) == list(range(n))
