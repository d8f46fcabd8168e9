# coding: utf-8
"""GPU tests of the scoring / selection step (K5) on constructed tables (tests/select_tables.py).

Every selection is compared, bit for bit (orders, subsets, status), with the oracle on
`fp32_norm(sum_parts(parts))`: the R blocks added in rank order.  The paths:
  * the phase-B entry points `bz_*_select` (strided blocks) and `bz_*_select_peers` (one pointer
    per block), at every block count the sharded path can have;
  * the tail of the distance pass: the fused exchange (`bz_krum_peers` / `bz_bulyan_peers`, ranks
    emulated on one GPU as in test_cuda_fused_exchange.py, the caller an empty shard), and the
    reuse calls (`bz_*_reuse`), whose tail reads the old pairs from a crafted `cache_in` and runs
    K5 with the ring CTA's own thread count."""

import ctypes
import math

import numpy as np
import pytest

import select_tables as st
from oracle import byzoracle as orc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NS = [1, 2, 3, 5, 11, 17, 25, 30, 33, 40, 51, 64]

def _lib():
  from byzantinemomentum_b200 import _lib
  return _lib.lib()

def _stream():
  return torch.cuda.current_stream().cuda_stream

def _ptrs(addrs):
  return (ctypes.c_void_p * len(addrs))(*addrs)

def _dev(a):
  return torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device=DEV)

def select(rule, parts, n, f=0, m=1, peers=False, sqrt_norm=0):
  """ (selection, status) of bz_<rule>_select[_peers] on the blocks `parts` [R][len]. """
  lib = _lib()
  t = _dev(parts)
  R = t.shape[0]
  src = _ptrs([t[r].data_ptr() for r in range(R)]) if peers else t.data_ptr()
  sfx = "_select_peers" if peers else "_select"
  out = torch.full((n,), -1, dtype=torch.int32, device=DEV)
  status = torch.full((1,), 7, dtype=torch.int32, device=DEV)
  if rule == "krum":
    rc = getattr(lib, "bz_krum" + sfx)(src, R, n, f, out.data_ptr(), _stream())
    status.zero_()
  elif rule == "bulyan":
    rc = getattr(lib, "bz_bulyan" + sfx)(src, R, n, f, m, out.data_ptr(), status.data_ptr(), _stream())
  elif rule == "brute":
    rc = getattr(lib, "bz_brute" + sfx)(src, R, n, f, out.data_ptr(), status.data_ptr(), _stream())
  else:
    rc = getattr(lib, "bz_rowdist" + sfx)(src, R, n, sqrt_norm, out.data_ptr(), _stream())
    status.zero_()
  assert rc == 0, lib.bz_last_error()
  torch.cuda.synchronize()
  k = n - f if rule == "brute" else n
  return out.cpu().tolist()[:k], int(status.item())

def _bulyan_f(n):
  return 0 if n < 7 else 1

def _small_table(n, R, seed):
  """ Exact fp32 distances, each square split into equal power-of-two shares (exact sums). """
  rng = np.random.default_rng(seed)
  D = rng.uniform(1., 4., (n, n)).astype(np.float32).astype(np.float64)
  D = np.triu(D, 1) + np.triu(D, 1).T
  shares = 1 << int(math.log2(R))
  blocks = np.zeros((R, n * n))
  blocks[:shares] = st.square_blocks(D, shares)
  return blocks

def _check_all(parts, n, tag, peers_too=True):
  """ Krum, Bulyan and brute (subsets of two) on the blocks, both entry points, against the oracle. """
  R = parts.shape[0]
  for peers in ((False, True) if peers_too and R <= 16 else (False,)):
    p = f"{tag} R={R} peers={peers}"
    if n >= 2:
      f = 1 if n >= 4 else 0
      assert select("krum", parts, n, f, peers=peers)[0] == st.expect_krum(parts, n, f), p
    if n >= 3:
      f = _bulyan_f(n)
      m = n - f - 2
      order, status = select("bulyan", parts, n, f, m, peers=peers)
      assert (order, status) == st.expect_bulyan(parts, n, f, m), p
    f = max(0, n - 2)
    assert select("brute", parts, n, f, peers=peers) == st.expect_brute(parts, n, f), p

@pytest.mark.parametrize("n", NS)
def test_straddling_splits_select_like_the_rank_order_sum(n):
  """ At every block count: the one straddled distance decides the order of rows 0-3 and brute's
  pair; where the earlier interleaved order gave the other fp32 distance, the split is chosen so. """
  for R in range(1, 25):
    if n < 4:
      _check_all(_small_table(n, R, 7 * n + R), n, f"n={n} exact")
      continue
    alt = st.pick_slices(n, R) if st.interleaved_differs(n, R) else None
    parts, d01 = st.straddle_table(n, R, seed=100 * n + R, alt_slices=alt)
    _check_all(parts, n, f"n={n} straddle d01={d01!r}")

@pytest.mark.parametrize("sqrt_norm", [0, 1])
def test_rowdist_keys_straddle_at_every_block_count(sqrt_norm):
  for n in NS:
    for R in range(1, 25):
      parts = st.straddle_keys(n, R, seed=R * 101 + n, sqrt_norm=sqrt_norm, alt_slices=16 if R > 16 else None)
      want = st.expect_rowdist(parts, n, sqrt_norm)
      assert select("rowdist", parts, n, sqrt_norm=sqrt_norm)[0] == want, (n, R, sqrt_norm)
      if R <= 16:
        assert select("rowdist", parts, n, sqrt_norm=sqrt_norm, peers=True)[0] == want, (n, R, sqrt_norm, "peers")

def test_neumaier_corpus():
  """ Scores whose order depends on CPython's compensated sum(): Krum on every table (f as drawn),
  Bulyan where n allows, on one block and on two exact halves. """
  for k, (n, f, D) in enumerate(st.neumaier_corpus()):
    for R in (1, 2):
      parts = st.square_blocks(D, R)
      assert select("krum", parts, n, f)[0] == orc.krum_order(D, f)[0], (k, n, f, R)
      fb = (n - 3) // 4
      for m in (1, n - fb - 2):
        assert select("bulyan", parts, n, fb, m) == st.expect_bulyan(parts, n, fb, m), (k, n, fb, m)

@pytest.mark.parametrize("n", [5, 11, 25, 51, 64])
def test_nonfinite_and_overflowing_sums(n):
  """ NaN, +inf, FLT_MAX, just below and at the fp32 rounding point to +inf, reached only across
  the blocks: Krum / Bulyan map them to +inf, brute skips every subset that holds one. """
  for R in (1, 3, 16):
    parts = st.nonfinite_table(n, R, seed=n + R)
    f = 1
    assert select("krum", parts, n, f)[0] == st.expect_krum(parts, n, f), (n, R)
    fb = (n - 3) // 4
    assert select("bulyan", parts, n, fb, n - fb - 2) == st.expect_bulyan(parts, n, fb, n - fb - 2), (n, R)
    for fr in (max(0, n - 3), max(0, n - 2)):
      if math.comb(n, n - fr) <= 50_000:
        assert select("brute", parts, n, fr) == st.expect_brute(parts, n, fr), (n, R, fr)

def test_brute_with_no_finite_subset():
  n, f = 6, 2
  parts = np.full((1, n * n), math.nan)
  assert select("brute", parts, n, f) == (list(range(n - f)), 1)

BRUTE_SIZES = [(5, 2), (8, 4), (10, 5), (12, 4), (20, 10), (25, 12), (26, 13)]

@pytest.mark.parametrize("n,f", BRUTE_SIZES)
def test_brute_planted_subsets_at_thread_edges(n, f):
  """ Two subsets of diameter 1 at ranks on the edges of the 1024 threads' rank ranges: the first
  in lexicographic order wins a tie, and the later one wins when the first is one ulp wider. """
  total = math.comb(n, n - f)
  for r1, r2, what in st.planted_targets(total, st.K5_THREADS):
    D, S1, S2 = st.planted_table(n, f, r1, r2)
    for R in (1, 4):
      assert select("brute", st.square_blocks(D, R), n, f) == (S1, 0), (n, f, what, R)
    if r1 != r2:
      Ds, _, _ = st.planted_table(n, f, r2, r1, strict=True)
      assert select("brute", st.square_blocks(Ds, 2), n, f, peers=True) == (S2, 0), (n, f, what, "strict")

@pytest.mark.parametrize("n", [7, 11, 15, 25, 51])
def test_bulyan_degenerate_boundary(n):
  """ q all-NaN rows (their distances +inf), every m: status and order as the oracle and the
  degenerate rule of bulyan_stage1. """
  f = (n - 3) // 4
  m_max = n - f - 2
  for q in range(n + 1):
    parts = st.bulyan_nan_rows(n, q, seed=q)
    for m in range(1, m_max + 1):
      assert select("bulyan", parts, n, f, m) == st.expect_bulyan(parts, n, f, m), (n, q, m)

def test_cge_and_aksel_keys():
  """ Row keys with +inf, overflowing sums and fp32 ties of different fp64 sums (index order). """
  n = 11
  y = float(np.float32(1.5))
  sq = np.array([st.INF_TIE, y * y, math.inf, st.FLT_MAX, st.INF_BELOW, y * y * (1 + 2. ** -40),
                 4., y * y, y * y * (1 - 2. ** -40), 1e300, 2.], dtype=np.float64)
  for R in (1, 2, 17):
    parts = np.zeros((R, n))
    parts[0] = sq / (2 if R > 1 else 1)
    if R > 1:
      parts[R - 1] = sq / 2
    for sqrt_norm in (0, 1):
      want = st.expect_rowdist(parts, n, sqrt_norm)
      assert select("rowdist", parts, n, sqrt_norm=sqrt_norm)[0] == want, (R, sqrt_norm)
  # aksel keys: fp32(sum), the ties of different fp64 sums stay in index order
  keys = [float(np.float32(x)) for x in orc.sum_parts(parts)]
  assert keys[1] == keys[5] == keys[7] == keys[8]

# ---------------------------------------------------------------------------------------------- #
# The tail of the distance pass

@pytest.mark.parametrize("rule", ["krum", "bulyan"])
@pytest.mark.parametrize("n", [5, 11, 17, 25, 33, 51, 64])
def test_fused_tail_sums_the_blocks_like_phase_b(rule, n):
  """ The caller (an empty shard) publishes a zero block at its rank; the other slots hold crafted
  blocks.  The fused order equals bz_*_select and bz_*_select_peers on the same blocks, and the
  oracle on their rank-order sum. """
  from test_cuda_fused_exchange import Call, Ranks, _s32
  epoch = 5
  s = epoch % 2
  for R in (2, 3, 5, 8, 16):
    rank = R // 2
    other, _ = st.straddle_table(n, R - 1, seed=1000 * n + R)
    parts = np.insert(other, rank, 0., axis=0)                # the caller's block is the zero one
    f = 1 if rule == "krum" else _bulyan_f(n)
    m = 1 if rule == "krum" else n - f - 2
    want = st.expect_krum(parts, n, f) if rule == "krum" else st.expect_bulyan(parts, n, f, m)
    ranks = Ranks(R, n)
    for p in range(R):
      ranks.slot(p, s).copy_(_dev(parts[p]))
      ranks.flags(p, s).fill_(_s32(epoch - 2))
    for t in range(R):
      if t != rank:
        ranks.flags(rank, s)[t] = _s32(epoch)
    call = Call(rule, n, f, m, 0)
    rows = [torch.empty(4, device=DEV)[:0] for _ in range(n)]
    assert call.peers(rows, rank, R, *ranks.tables(s), epoch) == 0, _lib().bz_last_error()
    assert not ranks.slot(rank, s).any(), "the empty shard publishes zeros"
    got = call.order.cpu().tolist()
    status = int(call.status.item())
    b = select(rule, parts, n, f, m)
    bp = select(rule, parts, n, f, m, peers=True)
    if rule == "krum":
      assert got == b[0] == bp[0] == want, (n, R)
    else:
      assert (got, status) == b == bp == want, (n, R)

def _reuse(rule, rows, n, f, m, cache_in):
  """ bz_<rule>_reuse with old_index = [0 .. n-2, -1] over the crafted n x n table `cache_in`. """
  lib = _lib()
  d = rows[0].numel()
  out = torch.empty(d, device=DEV)
  sel = torch.full((n,), -1, dtype=torch.int32, device=DEV)
  status = torch.full((1,), 7, dtype=torch.int32, device=DEV)
  old = (ctypes.c_int32 * n)(*(list(range(n - 1)) + [-1]))
  cin = _dev(cache_in.reshape(-1))
  cout = torch.zeros(64 * 64, dtype=torch.float64, device=DEV)
  mode = ctypes.c_int(7)
  nbytes = lib.bz_workspace_bytes(64)
  ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
  rp = _ptrs([r.data_ptr() for r in rows])
  common = (ctypes.addressof(old), cin.data_ptr(), n, cout.data_ptr(), ctypes.addressof(mode), ws.data_ptr(), nbytes, _stream())
  if rule == "krum":
    rc = lib.bz_krum_reuse(rp, n, f, m, d, out.data_ptr(), sel.data_ptr(), *common)
    status.zero_()
  elif rule == "bulyan":
    rc = lib.bz_bulyan_reuse(rp, n, f, m, d, out.data_ptr(), sel.data_ptr(), status.data_ptr(), *common)
  else:
    rc = lib.bz_brute_reuse(rp, n, f, d, out.data_ptr(), sel.data_ptr(), status.data_ptr(), *common)
  assert rc == 0, lib.bz_last_error()
  torch.cuda.synchronize()
  assert mode.value == 1, "the star pass did not run: the crafted table was not read"
  k = n - f if rule == "brute" else n
  return sel.cpu().tolist()[:k], int(status.item())

def _rows(n, d, last):
  rows = [torch.zeros(d, device=DEV) for _ in range(n - 1)]
  return rows + [torch.full((d,), last, device=DEV)]

@pytest.mark.parametrize("n", [5, 11, 17, 25, 33, 51])
def test_reuse_tail_scores_a_crafted_table(n):
  """ Krum and Bulyan in the ring tail on a straddled table (one block) whose new row is all NaN. """
  parts, _ = st.straddle_table(n, 1, seed=n)
  cache = parts.reshape(n, n)
  rows = _rows(n, 256, math.nan)
  D = st.distances(parts, n)
  D[:, n - 1] = D[n - 1, :] = math.inf
  np.fill_diagonal(D, 0.)
  f = 1
  assert _reuse("krum", rows, n, f, 1, cache)[0] == orc.krum_order(D, f)[0], n
  fb = _bulyan_f(n)
  m = n - fb - 2
  order, scores = orc.bulyan_order(D, fb, m)
  assert _reuse("bulyan", rows, n, fb, m, cache) == (order, st.bulyan_status(scores, n, fb, m)), n

def _nearest_without(rank, n, k, step, total):
  """ The nearest rank from `rank` in direction `step` whose subset leaves out row n - 1. """
  while 0 <= rank < total:
    if n - 1 not in st.unrank(rank, n, k):
      return rank
    rank += step
  return None

@pytest.mark.parametrize("n,f", [(8, 4), (12, 4), (15, 7), (20, 10), (25, 13), (26, 13)])
def test_reuse_tail_brute_at_its_thread_edges(n, f):
  """ Brute in the ring tail, whose CTA has 192, 384 or 512 threads: planted subsets at the edges of
  those threads' rank ranges (moved to the nearest subset without the new row, which is far away). """
  k = n - f
  total = math.comb(n, k)
  threads = st.tail_threads(n)
  d = 256
  rows = _rows(n, d, 1e4)
  far = float(orc.fp32_norm(d * 1e8))
  for r1, r2, what in st.planted_targets(total, threads):
    a, b = _nearest_without(r1, n, k, -1, total), _nearest_without(r2, n, k, 1, total)
    if a is None or b is None or a > b:
      continue
    for strict in (False, True):
      if strict and a == b:
        continue
      D, S1, S2 = st.planted_table(n, f, b, a, strict=True) if strict else st.planted_table(n, f, a, b)
      cache = np.triu(D * D, 1)
      got = _reuse("brute", rows, n, f, 0, cache)
      want = S1                                               # with `strict`, S1 = unrank(b) is the narrower
      Dfull = D.copy()
      Dfull[:, n - 1] = Dfull[n - 1, :] = far
      Dfull[n - 1, n - 1] = 0.
      assert got == (want, 0), (n, f, what, strict, a, b)
      if total <= 3432:
        assert orc.brute_selection(Dfull, f) == want
