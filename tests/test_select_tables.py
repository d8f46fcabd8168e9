# coding: utf-8
"""CPU self-checks of the constructed selection tables (tests/select_tables.py): the corpus must
really discriminate, or the GPU tests built on it prove nothing."""

import math

import numpy as np
import pytest

import select_tables as st
from oracle import byzoracle as orc

# (n, R) where the earlier selection kernels did not add the blocks in rank order
DIFFERS = {5: [3, 5, 6, 7] + list(range(9, 17)), 11: [3, 5, 6, 7] + list(range(9, 17)),
           17: [3, 5, 6, 7] + list(range(9, 17)), 25: [3, 5, 6, 7] + list(range(9, 17)),
           30: [3] + list(range(5, 17)), 33: [3] + list(range(5, 17)),
           40: list(range(3, 17)), 51: list(range(3, 17)), 64: []}

def test_interleaved_order_differs_exactly_where_expected():
  for n, want in DIFFERS.items():
    assert [R for R in range(1, 17) if st.interleaved_differs(n, R)] == want, n

def test_sum_parts_is_rank_order():
  p = np.array([[1.], [2. ** 53], [1.]])
  assert orc.sum_parts(p)[0] == 2. ** 53                  # (1 + 2^53) + 1: both ties round to even
  assert orc.sum_parts(p[[0, 2, 1]])[0] == 2. ** 53 + 2.
  assert st.interleaved_sum(p, 2)[0] == 2. ** 53 + 2.     # (p0 + p2) + p1

@pytest.mark.parametrize("n", sorted(DIFFERS))
def test_straddling_splits_tell_the_orders_apart(n):
  for R in DIFFERS[n]:
    parts, d01 = st.straddle_table(n, R, seed=100 * n + R, alt_slices=st.pick_slices(n, R))
    alt = st.interleaved_sum(parts, st.pick_slices(n, R)).reshape(n, n)
    sq = orc.sum_parts(parts).reshape(n, n)
    assert orc.fp32_norm(sq[0, 1]) == d01 != orc.fp32_norm(alt[0, 1]), (n, R)
    # the order of rows 0-3 hinges on that distance
    want = st.expect_krum(parts, n, 1)
    D = st.distances(parts, n)
    D[0, 1] = D[1, 0] = float(orc.fp32_norm(alt[0, 1]))
    assert orc.krum_order(D, 1)[0] != want, (n, R)

def test_straddling_keys_beyond_sixteen_blocks():
  for sqrt_norm in (0, 1):
    for R in (17, 20, 24):
      parts = st.straddle_keys(11, R, seed=R, sqrt_norm=sqrt_norm, alt_slices=16)
      a = st.expect_rowdist(parts, 11, sqrt_norm)
      key = lambda s: float(orc.fp32_norm(s)) if sqrt_norm else float(np.float32(s))
      assert key(orc.sum_parts(parts)[0]) != key(st.interleaved_sum(parts, 16)[0]), (sqrt_norm, R)
      assert a[:2] in ([0, 1], [1, 0])

def test_neumaier_corpus_discriminates():
  corpus = st.neumaier_corpus()
  assert len(corpus) >= 20
  for n, f, D in corpus:
    assert 8 <= n <= 64 and 0 <= f <= (n - 3) // 2
    assert np.array_equal(D.astype(np.float32).astype(np.float64), D)          # fp32 distances
    blocks = st.square_blocks(D)
    assert np.array_equal(st.distances(blocks, n), D + np.diag(np.full(n, 0.)))
    py = orc.krum_order(D, f)[0]
    nv = orc._stable_argsort(st._krum_scores(D, f, st.naive_sum))
    assert py != nv

@pytest.mark.parametrize("threads", [st.K5_THREADS, 192, 384, 512])
@pytest.mark.parametrize("n,f", [(8, 4), (10, 5), (12, 4), (20, 10), (25, 12), (26, 13)])
def test_planted_subsets_land_on_thread_edges(n, f, threads):
  total = math.comb(n, n - f)
  per = -(-total // threads)
  targets = st.planted_targets(total, threads)
  whats = {w for _, _, w in targets}
  assert "rank 0 and the last rank" in whats
  if total > threads:
    assert "last rank of thread t, first of thread t + 1" in whats and "two ranks of one thread" in whats
  for r1, r2, what in targets:
    D, S1, S2 = st.planted_table(n, f, r1, r2)
    assert st.rank_of(S1, n) == r1 and st.rank_of(S2, n) == r2
    t1, t2 = st.thread_of(r1, total, threads), st.thread_of(r2, total, threads)
    if what == "first and last rank of one thread":
      assert t1 == t2 and r1 % per == 0 and r2 % per == per - 1
    if what.startswith("last rank of thread t"):
      assert t2 == t1 + 1 and r1 % per == per - 1 and r2 % per == 0
    if what == "two threads of one warp":
      assert t1 // 32 == t2 // 32 and t1 != t2
    if what.startswith("last rank of warp"):
      assert t2 // 32 == t1 // 32 + 1
    if total <= 3432:                              # the oracle's own scan, where it is quick
      assert orc.brute_selection(D, f) == S1
      Ds, _, _ = st.planted_table(n, f, r2, r1, strict=True) if r1 != r2 else (D, S1, S2)
      assert orc.brute_selection(Ds, f) == (S2 if r1 != r2 else S1)

def test_unrank_matches_itertools():
  import itertools
  for n, k in ((7, 3), (9, 5), (6, 6)):
    for r, sub in enumerate(itertools.combinations(range(n), k)):
      assert st.unrank(r, n, k) == list(sub) and st.rank_of(list(sub), n) == r

def test_nonfinite_sums_sit_at_the_rounding_point():
  with np.errstate(over="ignore"):
    assert np.isposinf(np.float32(st.INF_TIE))
  assert np.float32(st.INF_BELOW) == np.float32(st.FLT_MAX)
  for R in (1, 3):
    parts = st.nonfinite_table(11, R, seed=R)
    sq = orc.sum_parts(parts)
    for v in (st.FLT_MAX, st.INF_BELOW, st.INF_TIE):
      assert (sq == v).any() and (R == 1 or not (parts == v).any())
    assert np.isnan(sq).any() and np.isposinf(sq).any()

def test_bulyan_boundary_sweep_reaches_both_sides():
  n, f = 11, 2
  seen = set()
  for q in range(n + 1):
    for m in range(1, n - f - 1):
      seen.add(st.expect_bulyan(st.bulyan_nan_rows(n, q, q), n, f, m)[1])
  assert seen == {0, 2}
