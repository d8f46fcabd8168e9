# coding: utf-8
"""CPU self-checks of the constructed tables above 64 rows (tests/select_tables.py), which
test_cuda_select_tables_wide.py feeds to phase B: each must really discriminate, or the GPU tests built on it
prove nothing."""

import hashlib
import time

import numpy as np
import pytest

import select_tables as st
from oracle import byzoracle as orc

@pytest.mark.parametrize("n", [65, 97, 128])
def test_straddling_splits_tell_reverse_and_tree_orders_apart(n):
  for R in range(3, 25):
    parts, d01 = st.straddle_table(n, R, seed=100 * n + R, alts=st.other_orders(R))
    want = st.expect_krum(parts, n, 1)
    assert orc.fp32_norm(orc.sum_parts(parts)[1]) == d01
    for alt in st.other_orders(R):
      other = float(orc.fp32_norm(alt(parts)[1]))
      assert other != d01, (n, R, alt.__name__)
      D = st.distances(parts, n)
      D[0, 1] = D[1, 0] = other
      assert orc.krum_order(D, 1)[0] != want, (n, R, alt.__name__)        # the order of rows 0-3 hinges on it

def test_other_orders():
  p = np.array([[1.], [2. ** 53], [1.], [1.]])
  assert orc.sum_parts(p)[0] == 2. ** 53 and st.reverse_sum(p)[0] == 2. ** 53 + 4.    # (2 + 2^53) + 1: a tie, to even
  assert st.pairwise_sum(p)[0] == 2. ** 53 + 2.                          # (1 + 2^53) + (1 + 1)
  assert [a.__name__ for a in st.other_orders(2)] == [] and len(st.other_orders(3)) == 1 and len(st.other_orders(4)) == 2

def test_straddling_keys_tell_the_orders_apart():
  for sqrt_norm in (0, 1):
    key = (lambda s: float(orc.fp32_norm(s))) if sqrt_norm else (lambda s: float(np.float32(s)))
    for R in range(3, 25):
      parts = st.straddle_keys(128, R, seed=R * 101 + 128, sqrt_norm=sqrt_norm, alts=st.other_orders(R))
      for alt in st.other_orders(R):
        assert key(orc.sum_parts(parts)[0]) != key(alt(parts)[0]), (sqrt_norm, R, alt.__name__)

def test_existing_tables_are_unchanged():
  """ The 64-row tables (interleaved alternative, no `alts`) are the bits they were before the alternatives. """
  h = hashlib.sha256()
  for n, R in ((5, 3), (25, 9), (51, 16), (64, 24), (33, 5)):
    alt = st.pick_slices(n, R) if st.interleaved_differs(n, R) else None
    h.update(st.straddle_table(n, R, seed=100 * n + R, alt_slices=alt)[0].tobytes())
    for sq in (0, 1):
      h.update(st.straddle_keys(n, R, seed=R * 101 + n, sqrt_norm=sq, alt_slices=16 if R > 16 else None).tobytes())
  for _, _, D in st.neumaier_corpus():
    h.update(D.tobytes())
  assert h.hexdigest()[:16] == "1671bd625a72057b"

def test_wide_neumaier_corpus_discriminates_quickly():
  t0 = time.perf_counter()
  corpus = st.neumaier_corpus_wide()
  assert time.perf_counter() - t0 < 5.
  assert len(corpus) == 24
  counts = set()
  for n, f, D in corpus:
    assert 65 <= n <= 128 and 0 <= f <= (n - 3) // 2
    assert np.array_equal(D.astype(np.float32).astype(np.float64), D)
    for R in (1, 2):
      assert np.array_equal(st.distances(st.square_blocks(D, R), n), D)
    assert orc.krum_order(D, f)[0] != orc._stable_argsort(st._krum_scores(D, f, st.naive_sum))
    counts.add(n - f - 1)
  assert max(counts) == 127 and min(counts) <= 40

def test_special_keys_hold_every_case():
  for n in (65, 100, 128):
    sq = st.special_keys(n, seed=n)
    assert np.isnan(sq).sum() == 3 and np.isposinf(sq).sum() == 3
    for v in (st.INF_TIE, st.INF_BELOW, st.FLT_MAX, 1e300):
      assert (sq == v).sum() == 3
    y2 = float(np.float32(1.5)) ** 2
    assert (np.float32(sq[np.isfinite(sq) & (np.abs(sq - y2) < 1e-9)]) == np.float32(y2)).sum() == 9
    order = st.expect_rowdist(sq[None, :], n, 0)
    assert set(order[-3:]) == set(np.flatnonzero(np.isnan(sq)).tolist())       # Aksel: NaN keys last

def test_tie_tables_tie():
  D = st.tie_table(128, 0)
  assert set(np.unique(D).tolist()) == {0., 1., 2.}
  scores = orc.krum_order(D, 1)[1]
  assert len(set(scores)) < len(scores) // 2
  assert orc.krum_order(st.tie_table(128, 0, (1.,)), 1)[0] == list(range(128))

@pytest.mark.parametrize("n", [65, 128])
def test_bulyan_boundary_sweep_reaches_both_sides(n):
  f = (n - 3) // 4
  m_max = n - f - 2
  seen = set()
  for q in (0, f, f + 1, f + 2, n // 2, n):
    for m in (1, 2, m_max - 1, m_max):
      seen.add(st.expect_bulyan(st.bulyan_nan_rows(n, q, q), n, f, m)[1])
  assert seen == {0, 2}

def test_nonfinite_sums_reach_the_rounding_point_above_64_rows():
  for R in (1, 3, 16):
    parts = st.nonfinite_table(128, R, seed=128 + R)
    sq = orc.sum_parts(parts)
    for v in (st.FLT_MAX, st.INF_BELOW, st.INF_TIE):
      assert (sq == v).any() and (R == 1 or not (parts == v).any())
    assert np.isnan(sq).any() and np.isposinf(sq).any()
