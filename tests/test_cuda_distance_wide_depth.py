# coding: utf-8
"""`bz_distance` above 64 rows where its distance step can go wrong: at full depth, at every count u of
unique rows, and at the ends of the fp32 range.

  * Full depth: every K2 pass of Multi-Krum and Bulyan (36-64 rows each: the ring's 256-column tiles, 3
    stages, a flush every 8 tiles, test_cuda_depth.py) gets at least 17 full tiles per walker, and every
    thread of K2'-wide (Aksel, forward and reversed walk; CGE) at least 8 sweeps, even if 2 x SM-count CTAs
    ran.  The sizes are asserted from the SM count and these shapes, so a later change of the geometry fails
    here instead of quietly shrinking the coverage.
  * Every u in 65..128, and u in {1, 2, 16, 25, 26, 36, 64} at n = 65 and 128: alias groups (one tensor at
    several indices) scattered among the rows, in the first block of unique rows, in the last, and across
    blocks, some holding NaN or +-inf (their self distance is NaN: an infinite distance, as the reference's
    `(x - x).norm()`).  The rows are compared in a general alias-canonical form: the first index of their
    tensor.
  * Rows whose distances, norms and Aksel keys overflow (+inf ties keep index order), and 2^-80 rows whose
    every key is exactly 0 (the stable index order across blocks and alias groups).
  * The d-sharded phases on 3 emulated ranks at full depth, and on a stack whose sums are finite in every
    shard but overflow in total; the attack against CGE at 128 honest rows and full depth.

References are fp64 on the device or the NumPy oracle; a selection is compared where its margins are clear
or its ties exact."""

import numpy as np
import pytest

import bulyan_columns
import parity
from oracle import byzoracle as orc
from test_cuda_depth import D_EXACT, D_RAGGED, _assert_depth, _sm_count
from test_cuda_distance_wide import MIN_MARGIN, call
from test_cuda_distance_shards import emulate, phase_a, same_bits

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FLT_MAX = float(np.finfo(np.float32).max)
ORDER_RTOL = 1e-6         # finite keys closer than this may come out in either order (fp32-norm noise ~1e-7)
K2W_STRIDE = 256          # columns per CTA and sweep of K2'-wide (k2_rowdist_wide.cu), at most 2 CTAs per SM

# ---------------------------------------------------------------------------------------------------------- #
# Layouts: which tensor each original row is

def layout(n, u, seed):
  """ ids[i] = the tensor of original row i: u tensors, the n - u further rows copies of up to five sources
  spread over the unique rows: copies of tensor 0 inside the first fifth of the rows, copies of tensor u - 1 in
  the last fifth, the others anywhere (their group straddles the blocks of unique rows). """
  rng = np.random.default_rng(seed)
  ids = list(range(u))
  sources = sorted({0, u // 4, u // 2, (3 * u) // 4, u - 1})
  for k in range(n - u):
    s = sources[k % len(sources)]
    if s == 0:
      pos = int(rng.integers(1, max(2, n // 5)))
    elif s == u - 1 and u > 1:
      pos = int(rng.integers(len(ids) - min(len(ids) - 1, n // 5), len(ids) + 1))
    else:
      pos = int(rng.integers(1, len(ids) + 1))
    ids.insert(pos, s)
  return ids

def first_index(ids):
  """ The first original index of each row's tensor. """
  seen = {}
  return [seen.setdefault(t, i) for i, t in enumerate(ids)]

def canon(order, first):
  return [first[int(i)] for i in order]

def plan_blocks(u):
  """ The blocks of unique rows and the row count of each pass (plan_passes, api_distance.inc). """
  k = 1 if u <= 64 else (u + 31) // 32
  start = [b * u // k for b in range(k + 1)]
  if k == 1:
    return start, [u]
  return start, [start[a + 1] - start[a] + start[b + 1] - start[b] for a in range(k) for b in range(a + 1, k)]

def assert_full_depth(u, d):
  """ Every pass at the 36-64-row ring shape with full depth per walker; >= 8 sweeps per K2'-wide thread. """
  _, sizes = plan_blocks(u)
  for s in sizes:
    assert 36 <= s <= 64, (u, sizes)
    _assert_depth(s, d)
  sweeps = d // (2 * _sm_count() * K2W_STRIDE)
  assert sweeps >= 8, f"d={d}: {sweeps} K2'-wide sweeps per thread < 8"

# ---------------------------------------------------------------------------------------------------------- #
# Comparisons

def determined(a, b):
  """ Two keys that tie exactly at 0 or +inf: both stable sorts keep index order. """
  return a == b and (a == 0 or a == np.inf)

def clear(keys, order, upto, first):
  """ Whether the first upto + 1 keys in `order` are apart by MIN_MARGIN (relative) or tie exactly at 0 or
  +inf, ties inside an alias group aside. """
  for k in range(min(upto, len(order) - 1)):
    i, j = order[k], order[k + 1]
    if first[i] == first[j]:
      continue
    a, b = keys[i], keys[j]
    if determined(a, b):
      continue
    if np.isfinite(a) and np.isfinite(b):
      if (b - a) / max(abs(b), 1e-300) < MIN_MARGIN:
        return False
    elif a == b or np.isnan(a) or np.isnan(b):
      return False
  return True

def assert_order(got, want, keys, first, what, upto=None):
  """ The orders agree in canonical form, except that two different finite keys within ORDER_RTOL of each other
  may come out either way; +inf and exact 0 keys must be where index order puts them. """
  upto = len(want) if upto is None else upto
  g, w = canon(got[:upto], first), canon(want[:upto], first)
  for k in range(upto):
    if g[k] == w[k]:
      continue
    a, b = keys[got[k]], keys[want[k]]
    close = np.isfinite(a) and np.isfinite(b) and a != 0 and abs(a - b) <= ORDER_RTOL * abs(b)
    assert close, f"{what}: position {k}: row {got[k]} (key {a!r}) where the reference has row {want[k]} (key {b!r})"

def stable(keys):
  return sorted(range(len(keys)), key=lambda i: keys[i])

def check_rule(gar, x, first, got, order, status, f, m=None, mode="mid", what=""):
  """ `bz_distance`'s result against the oracle on host rows x: the status, the selection where clear(), the
  output bit for bit (Multi-Krum, Aksel, CGE) or, for Bulyan, within the closest-m bar and K4's order bit for
  bit.  Returns whether the selection was compared. """
  rows = [x[i] for i in range(x.shape[0])]
  n = len(rows)
  if gar == "bulyan":
    m = n - f - 2 if m is None else m
    try:
      ref, info = orc.bulyan(rows, f, m, return_info=True)
    except TypeError:
      assert status == 2 and np.isnan(got).all(), what
      return True
    assert status == 0, what
    parity.assert_close_scaled(got, ref, parity.column_scale(info["stage1"]), what, exempt=info["ambiguous"])
    if not clear(info["scores"], info["order"], n - f - 2, first):
      return False
    assert canon(order[:n - f - 2], first) == canon(info["order"][:n - f - 2], first), what
    bulyan_columns.check(got, info["stage1"], f, True, what)
    return True
  if gar == "krum":
    ref, info = orc.krum(rows, f, m, return_info=True)
    count, keys = n - f - 2 if m is None else m, info["scores"]
  elif gar == "aksel":
    ref, info = orc.aksel(rows, f, mode, return_info=True)
    count, keys = (n + 1) // 2 if mode == "mid" else n - f, info["distances"]
  else:
    ref, info = orc.cge(rows, f, return_info=True)
    count, keys = n - f, info["norms"]
  if not clear(keys, info["order"], count, first):
    return False
  assert canon(order[:count], first) == canon(info["order"][:count], first), what
  parity.assert_bit_exact(got, ref, what)
  return True

RULES = (("krum", None, 0), ("krum", 1, 0), ("bulyan", None, 0), ("aksel", None, 0), ("aksel", None, 1), ("cge", None, 0))

# ---------------------------------------------------------------------------------------------------------- #
# Device stacks

def padded(u, d):
  """ u rows of d floats, each starting on a 256-byte boundary (the ring's TMA path). """
  return torch.empty(u, (d + 63) // 64 * 64, device=DEV)[:, :d]

def device_stack(n, u, d, seed):
  """ u unique rows mu + sigma_k z_k (sigma spread over [0.5, 1.5] in shuffled order) of which the last is the
  Byzantine row -1.1 x the mean of the others, laid out over n rows by `layout`. """
  gen = torch.Generator(device=DEV).manual_seed(seed)
  uniq = padded(u, d)
  mu = torch.randn(d, device=DEV, generator=gen)
  sigma = np.random.default_rng(seed).permutation(np.linspace(0.5, 1.5, max(u - 1, 1)))
  for k in range(u - 1):
    uniq[k] = mu + float(sigma[k]) * torch.randn(d, device=DEV, generator=gen)
  uniq[u - 1] = uniq[:u - 1].mean(dim=0) * -1.1 if u > 1 else mu
  ids = layout(n, u, seed)
  return uniq, ids, [uniq[t] for t in ids]

def pair_sums(uniq):
  """ fp64 sums of the fp32 squares of fp32 differences between the unique rows, on the device; u x u, the
  diagonal the self distances (0, or NaN for a row holding NaN or inf). """
  u = uniq.shape[0]
  out = torch.empty(u, u, dtype=torch.float64, device=DEV)
  for i in range(u):
    out[i] = (uniq - uniq[i]).pow(2).double().sum(dim=1)
  return out.cpu().numpy()

def expand(table, ids):
  return table[np.ix_(ids, ids)]

def partial_block(gar, rows):
  """ Phase A (`bz_distance_partial`) on one rank over the whole rows: the n x n block of the pass tables or the
  n sums of K2'-wide. """
  from byzantinemomentum_b200 import _lib
  ws = torch.empty(_lib.lib().bz_distance_workspace_bytes(len(rows)), dtype=torch.uint8, device=DEV)
  return phase_a(gar, rows, ws).cpu().numpy()

def assert_pair_block(block, sums, n, what, rtol=5e-7):
  """ Phase A's n x n block against the fp64 sums of the original rows: entries i < j (for two rows of one tensor
  the self distance of its unique row, 0 or NaN) with the same non-finite pattern and the roots within rtol,
  the diagonal and the entries below it 0. """
  got = block.reshape(n, n)
  assert (got[np.tril_indices(n)] == 0).all(), what + ": entries on or below the diagonal"
  iu = np.triu_indices(n, 1)
  fin = np.isfinite(sums[iu])
  assert np.array_equal(np.isfinite(got[iu]), fin), what
  np.testing.assert_allclose(np.sqrt(got[iu][fin]), np.sqrt(sums[iu][fin]), rtol=rtol, err_msg=what)

def avg_in_order(rows, sel, zero_init=True):
  """ sum(rows[sel]) / len(sel) in fp32, left to right (from 0.0 or from a clone of the first). """
  acc = (torch.zeros_like(rows[0]) + rows[sel[0]]) if zero_init else rows[sel[0]].clone()
  for k in sel[1:]:
    acc = acc + rows[k]
  return acc / torch.full_like(acc, float(len(sel)))

# ---------------------------------------------------------------------------------------------------------- #
# Full depth

FULL = [(65, 100), (96, 128), (97, 110), (128, 128)]     # (u, n): 3 blocks (two sizes), 4 blocks, no alias

@pytest.mark.parametrize("d", [D_RAGGED, D_EXACT], ids=["ragged", "exact"])
@pytest.mark.parametrize("u,n", FULL)
def test_full_depth(u, n, d):
  assert_full_depth(u, d)
  seed = 11 * u + n + (d % 5)
  uniq, ids, rows = device_stack(n, u, d, seed)
  first = first_index(ids)
  f = (n - 3) // 4
  what = f"u={u} n={n} d={d}"
  # the pass tables, through phase A on one rank
  sq = expand(pair_sums(uniq), ids)
  assert_pair_block(partial_block("krum", rows), sq, n, what + " pairs")
  D = orc.fp32_norm(sq)
  D = np.where(np.isfinite(D), D, np.inf)
  np.fill_diagonal(D, 0.)
  # Multi-Krum at m = m_max and 1: the order, and the average in that order bit for bit
  korder, kscores = orc.krum_order(D, f)
  for m in (n - f - 2, 1):
    assert orc._margin([kscores[i] for i in korder], m) > 1e-5 or first[korder[m - 1]] == first[korder[m]], what
    out, order, _ = call("krum", rows, f, m)
    assert_order(order, korder, kscores, first, f"{what} krum m={m}")
    assert canon(order[:m], first) == canon(korder[:m], first), f"{what} krum m={m}: selection"
    want = avg_in_order(rows, order[:m].tolist()).cpu().numpy()
    assert same_bits(out, want), f"{what} krum m={m} values"
  # Bulyan: the order, and stage 2 on a column sample that ends with the last (ragged) columns
  m = n - f - 2
  border, bscores = orc.bulyan_order(D, f, m)
  out, order, status = call("bulyan", rows, f)
  assert status == 0, what
  assert_order(order, border, bscores, first, f"{what} bulyan")
  rng = np.random.default_rng(seed)
  cols = np.unique(np.concatenate([np.arange(64), rng.choice(d, 1500, replace=False), np.arange(d - 700, d)]))
  idx = torch.from_numpy(cols).to(DEV)
  host = torch.stack([r.index_select(0, idx) for r in rows]).cpu().numpy()
  s1 = bulyan_columns.stage1(host, order.tolist(), f, m)
  bulyan_columns.check(out[cols], s1, f, True, what + " bulyan columns")
  # Aksel (both modes: the reversed walk around the median) and CGE (forward walk around the origin)
  X = torch.stack(rows)
  med = X.median(dim=0).values
  asq = (X - med).pow(2).double().sum(dim=1).cpu().numpy()
  akeys = asq.astype(np.float32).astype(np.float64)
  del X, med
  # K2'-wide's fp64 sums themselves, through phase A on one rank: a walk that drops or repeats columns moves
  # every row's sum alike, which the orders below cannot see
  np.testing.assert_allclose(partial_block("aksel", rows), asq, rtol=1e-6, err_msg=what + " aksel sums")
  nsq = np.array([float(r.double().pow(2).sum()) for r in uniq])[ids]
  np.testing.assert_allclose(partial_block("cge", rows), nsq, rtol=1e-6, err_msg=what + " cge sums")
  aorder = stable(akeys)
  for mode, c in ((0, (n + 1) // 2), (1, n - f)):
    assert orc._margin([akeys[i] for i in aorder], c) > 1e-5 or first[aorder[c - 1]] == first[aorder[c]], what
    out, order, _ = call("aksel", rows, f, mode=mode)
    assert_order(order, aorder, akeys, first, f"{what} aksel mode={mode}")
    assert canon(order[:c], first) == canon(aorder[:c], first), f"{what} aksel mode={mode}: selection"
    assert same_bits(out, avg_in_order(rows, order[:c].tolist()).cpu().numpy()), f"{what} aksel mode={mode} values"
  norms = orc.fp32_norm(nsq)
  corder = stable(norms)
  c = n - f
  assert orc._margin([norms[i] for i in corder], c) > 1e-5 or first[corder[c - 1]] == first[corder[c]], what
  out, order, _ = call("cge", rows, f)
  assert_order(order, corder, norms, first, f"{what} cge")
  want = avg_in_order(rows, order[:c].tolist(), zero_init=False).cpu().numpy()
  assert same_bits(out, want), f"{what} cge values"
  if u == n:
    return
  # a NaN in the aliased tensor of block 0 and +inf in the aliased Byzantine tensor of the last block: their
  # self distances, NaN, come at depth from the passes (0, 1) and (0, K - 1); their Krum scores are +inf and
  # keep index order
  assert ids.count(0) > 1 and ids.count(u - 1) > 1
  uniq[0, d // 3] = float("nan")
  uniq[u - 1, d - 1] = float("inf")
  sq = expand(pair_sums(uniq), ids)
  assert_pair_block(partial_block("krum", rows), sq, n, what + " poisoned pairs")
  D = orc.fp32_norm(sq)
  D = np.where(np.isfinite(D), D, np.inf)
  np.fill_diagonal(D, 0.)
  korder, kscores = orc.krum_order(D, f)
  m = n - f - 2
  assert np.isinf(kscores).sum() >= 4 and orc._margin([kscores[i] for i in korder], m) > 1e-5, what
  out, order, _ = call("krum", rows, f)
  assert_order(order, korder, kscores, first, f"{what} poisoned krum")
  assert same_bits(out, avg_in_order(rows, order[:m].tolist()).cpu().numpy()), f"{what} poisoned krum values"

# ---------------------------------------------------------------------------------------------------------- #
# Every count of unique rows

EVERY_U = [(u, min(128, u + 1 + (7 * u) % 23)) for u in range(65, 129)] + \
          [(u, n) for u in (1, 2, 16, 25, 26, 36, 64) for n in (65, 128)]

def host_stack(n, u, d, seed, poison):
  """ u unique host rows (as device_stack) over n rows by `layout`; poison "nan": a NaN in the source of the
  group at u // 4, "inf": +inf there and -inf in the source at u // 2. """
  rng = np.random.default_rng(seed)
  mu = rng.standard_normal(d)
  sigma = rng.permutation(np.linspace(0.5, 1.5, max(u - 1, 1)))
  uniq = np.empty((u, d), dtype=np.float32)
  for k in range(u - 1):
    uniq[k] = mu + sigma[k] * rng.standard_normal(d)
  uniq[u - 1] = -1.1 * uniq[:u - 1].mean(axis=0) if u > 1 else mu
  if poison == "nan":
    uniq[u // 4, d // 3] = np.nan
  elif poison == "inf":
    uniq[u // 4, d // 3] = np.inf
    uniq[u // 2, (2 * d) // 3] = -np.inf
  ids = layout(n, u, seed)
  return uniq, ids

def put(uniq, ids):
  tensors = [torch.from_numpy(r.copy()).to(DEV) for r in uniq]
  return [tensors[t] for t in ids]

@pytest.mark.parametrize("u,n", EVERY_U)
def test_every_unique_row_count(u, n):
  poison = ("nan", "inf", None)[u % 3] if u >= 16 else None
  d = 2053
  uniq, ids = host_stack(n, u, d, 4000 + 131 * u + n, poison)
  x = uniq[ids]
  rows = put(uniq, ids)
  first = first_index(ids)
  f = (n - 3) // 4
  compared = 0
  for gar, m, mode in RULES:
    got, order, status = call(gar, rows, f, m, mode)
    what = f"{gar} m={m} mode={mode} u={u} n={n} poison={poison}"
    compared += check_rule(gar, x, first, got, order, status, f, m, "mid" if mode == 0 else "n-f", what)
  assert compared >= 2, (u, n)

# ---------------------------------------------------------------------------------------------------------- #
# The ends of the fp32 range

@pytest.mark.parametrize("n", [65, 100, 128])
def test_overflowing_pairs_norms_and_aksel_keys_order_like_the_reference(n):
  """ test_cuda_extremes.py's stack above 64 rows: rows s (mu + sigma_i z_i), d = 300,007, S = d s^2 = 1e38;
  every eighth row (in every block) has sigma in [3, 3.5], decreasing with the index, the others distinct
  sigma in [0.52, 0.75].  Pairs with a large row, the norms of the large rows and their squared distances to
  the median are past 2 FLT_MAX, everything else below FLT_MAX / 2: the large rows' Krum scores, CGE norms and
  Aksel keys ((float) of the sum) are +inf and keep their index order, which finite roots, or fp64 keys, of the
  sums would reverse. """
  d = 300_007
  f = (n - 3) // 4
  gen = torch.Generator(device=DEV).manual_seed(n)
  idx = torch.arange(n, device=DEV)
  sigma = torch.where(idx % 8 == 7, 3.0 + 0.5 * (1. - idx / n), 0.75 * (1. - 0.3 * idx / n))
  S = 1e38
  mu = torch.randn(d, device=DEV, generator=gen)
  uniq = padded(n, d)
  uniq.copy_((mu[None, :] + sigma[:, None] * torch.randn(n, d, device=DEV, generator=gen)) * float(np.sqrt(S / d)))
  rows = [uniq[i] for i in range(n)]
  ids = list(range(n))
  sq = pair_sums(uniq)
  iu = np.triu_indices(n, 1)
  small = sq[iu] < FLT_MAX / 2
  assert (small | (sq[iu] > 2 * FLT_MAX)).all() and small.any() and (~small).any()
  assert_pair_block(partial_block("krum", rows), sq, n, f"n={n} pairs", rtol=1e-6)
  D = orc.fp32_norm(sq)
  np.fill_diagonal(D, 0.)
  korder, kscores = orc.krum_order(D, f)
  assert np.isinf(kscores).sum() >= 2 and np.isfinite(kscores).sum() >= n - f - 2
  for m in (n - f - 2, 1):
    _, order, _ = call("krum", rows, f, m)
    assert_order(order, korder, kscores, ids, f"n={n} krum m={m}")
  norms_sq = uniq.double().pow(2).sum(dim=1).cpu().numpy()
  norms = orc.fp32_norm(norms_sq)
  assert np.isinf(norms).sum() >= 2 and (norms_sq[np.isfinite(norms)] < FLT_MAX / 2).all()
  assert (norms_sq[np.isinf(norms)] > 2 * FLT_MAX).all()
  _, order, _ = call("cge", rows, f)
  assert_order(order, stable(norms), norms, ids, f"n={n} cge")
  # Aksel: (float) of the fp64 sum of fp32 squares around the lower median
  med = uniq.median(dim=0).values
  asq = (uniq - med).pow(2).double().sum(dim=1).cpu().numpy()
  with np.errstate(over="ignore"):
    akeys = asq.astype(np.float32).astype(np.float64)          # +inf past FLT_MAX
  assert np.isinf(akeys).sum() >= 2 and (asq[np.isfinite(akeys)] < FLT_MAX / 2).all() and (asq[np.isinf(akeys)] > 2 * FLT_MAX).all()
  for mode in (0, 1):
    _, order, _ = call("aksel", rows, f, mode=mode)
    assert_order(order, stable(akeys), akeys, ids, f"n={n} aksel mode={mode}")

@pytest.mark.parametrize("u,n", [(100, 128), (40, 70), (65, 128)])
def test_tiny_rows_keep_index_order(u, n):
  """ Rows of 2^-80 z: every square, hence every distance, norm and Aksel key, is exactly 0 on both sides, so
  every rule's order is the index order across blocks and alias groups; outputs against the oracle. """
  d = 1031
  rng = np.random.default_rng(u + n)
  uniq = (rng.standard_normal((u, d)) * 2. ** -80).astype(np.float32)
  ids = layout(n, u, u * n)
  x = uniq[ids]
  rows = put(uniq, ids)
  first = first_index(ids)
  f = (n - 3) // 4
  assert not orc.pairwise_distances(x).any() and not orc.row_norms(x).any()
  for gar, m, mode in RULES:
    got, order, status = call(gar, rows, f, m, mode)
    what = f"tiny {gar} m={m} mode={mode} u={u} n={n}"
    assert order.tolist() == list(range(n)), what
    assert check_rule(gar, x, first, got, order, status, f, m, "mid" if mode == 0 else "n-f", what), what

# ---------------------------------------------------------------------------------------------------------- #
# The d-sharded phases

def test_three_ranks_at_full_depth():
  """ R = 3 emulated ranks whose shards are each at full depth: every rank's block against the fp64 sums of its
  columns, the selection and output those of one GPU, the selection the reference's. """
  from byzantinemomentum_b200 import sharded
  R, u, n = 3, 100, 128
  d = 3 * D_RAGGED + 2
  for r in range(R):
    lo, hi = sharded.shard_bounds(d, R, r)
    assert_full_depth(u, hi - lo)
  uniq, ids, rows = device_stack(n, u, d, 31337)
  first = first_index(ids)
  f = (n - 3) // 4
  shard_sq = [pair_sums(uniq[:, lo:hi]) for lo, hi in (sharded.shard_bounds(d, R, r) for r in range(R))]
  shard_norm = [uniq[:, lo:hi].double().pow(2).sum(dim=1).cpu().numpy() for lo, hi in (sharded.shard_bounds(d, R, r) for r in range(R))]
  shard_med = []
  for r in range(R):
    lo, hi = sharded.shard_bounds(d, R, r)
    X = torch.stack([g[lo:hi] for g in rows])
    shard_med.append((X - X.median(dim=0).values).pow(2).double().sum(dim=1).cpu().numpy())
    del X
  sq = orc.sum_parts([expand(s, ids) for s in shard_sq])
  D = orc.fp32_norm(sq)
  np.fill_diagonal(D, 0.)
  for gar, m, mode in RULES:
    what = f"R={R} {gar} m={m} mode={mode}"
    got, order, status, blocks = emulate(gar, rows, R, f, m, mode)
    blocks = blocks.cpu().numpy()
    for r in range(R):
      if gar in ("krum", "bulyan"):
        assert_pair_block(blocks[r], expand(shard_sq[r], ids), n, f"{what} rank {r}")
      else:
        want = (shard_med[r] if gar == "aksel" else shard_norm[r][ids])
        np.testing.assert_allclose(blocks[r], want, rtol=1e-6, err_msg=f"{what} rank {r}")
    one = call(gar, rows, f, m, mode)
    assert np.array_equal(order, one[1]) and status == one[2] and same_bits(got, one[0]), what
    if gar == "krum":
      want, keys = orc.krum_order(D, f)
    elif gar == "bulyan":
      want, keys = orc.bulyan_order(D, f, n - f - 2)
    elif gar == "aksel":
      keys = orc.sum_parts(shard_med).astype(np.float32).astype(np.float64)
      want = stable(keys)
    else:
      keys = orc.fp32_norm(orc.sum_parts([s[ids] for s in shard_norm]))
      want = stable(keys)
    assert_order(order, want, keys, first, what)

def test_shards_finite_but_the_rank_order_sum_overflows():
  """ R = 3: the large rows (every eighth, sigma = 3) against the small ones (sigma in [0.2, 0.3]): every pair
  sum, norm and Aksel key of a large row is below 0.9 FLT_MAX in every shard and above 1.2 FLT_MAX in total,
  so the overflow rule applies only after the ranks' blocks are added. """
  from byzantinemomentum_b200 import sharded
  R, n, d = 3, 100, 300_009
  f = (n - 3) // 4
  gen = torch.Generator(device=DEV).manual_seed(5)
  idx = torch.arange(n, device=DEV)
  sigma = torch.where(idx % 8 == 7, torch.full_like(idx, 3, dtype=torch.float32), 0.3 - 0.1 * idx / n)
  S = 0.14 * FLT_MAX
  mu = torch.randn(d, device=DEV, generator=gen)
  uniq = padded(n, d)
  uniq.copy_((mu[None, :] + sigma[:, None] * torch.randn(n, d, device=DEV, generator=gen)) * float(np.sqrt(S / d)))
  rows = [uniq[i] for i in range(n)]
  ids = list(range(n))
  bounds = [sharded.shard_bounds(d, R, r) for r in range(R)]
  shard_sq = [pair_sums(uniq[:, lo:hi]) for lo, hi in bounds]
  shard_norm = [uniq[:, lo:hi].double().pow(2).sum(dim=1).cpu().numpy() for lo, hi in bounds]
  med = uniq.median(dim=0).values
  shard_med = [(uniq[:, lo:hi] - med[lo:hi]).pow(2).double().sum(dim=1).cpu().numpy() for lo, hi in bounds]
  sq = orc.sum_parts(shard_sq)
  iu = np.triu_indices(n, 1)
  big = sq[iu] > 1.2 * FLT_MAX
  assert big.any() and (sq[iu][~big] < FLT_MAX / 2).all()
  for part in (shard_sq, shard_norm, shard_med):
    assert all(np.nanmax(p) < 0.9 * FLT_MAX for p in part)
  D = orc.fp32_norm(sq)
  np.fill_diagonal(D, 0.)
  norms = orc.fp32_norm(orc.sum_parts(shard_norm))
  with np.errstate(over="ignore"):
    akeys = orc.sum_parts(shard_med).astype(np.float32).astype(np.float64)
  assert np.isinf(norms).sum() >= 2 and np.isinf(akeys).sum() >= 2
  for gar, m, mode in RULES:
    what = f"overflow in total {gar} m={m} mode={mode}"
    got, order, status, blocks = emulate(gar, rows, R, f, m, mode)
    assert np.isfinite(blocks.cpu().numpy()).all(), what
    if gar == "krum":
      want, keys = orc.krum_order(D, f)
    elif gar == "bulyan":
      want, keys = orc.bulyan_order(D, f, n - f - 2)
    elif gar == "aksel":
      keys = akeys
      want = stable(keys)
    else:
      keys = norms
      want = stable(keys)
    assert np.isinf(keys).sum() >= 2, what
    assert_order(order, want, keys, ids, what)
    one = call(gar, rows, f, m, mode)
    assert np.array_equal(order, one[1]) and status == one[2] and same_bits(got, one[0]), what

# ---------------------------------------------------------------------------------------------------------- #
# The attack against CGE

def test_anticge_128_honest_rows_at_full_depth():
  """ `engine.AntiCGE` and the one-rank d-sharded stages at nh = 128: the order is the fp64 reference's, the
  unscaled sum s0 + s0 + s1 + ... + s(maxpos - 1) bit for bit the fp32 sum in that order. """
  import byzantinemomentum_b200 as bz
  from byzantinemomentum_b200 import sharded
  nh, f, d = 128, 31, D_RAGGED
  assert d // (2 * _sm_count() * K2W_STRIDE) >= 8
  gen = torch.Generator(device=DEV).manual_seed(128)
  uniq = padded(nh, d)
  uniq.copy_(torch.randn(nh, d, device=DEV, generator=gen) * (0.5 + torch.rand(nh, 1, device=DEV, generator=gen)))
  rows = [uniq[i] for i in range(nh)]
  norms = orc.fp32_norm(uniq.double().pow(2).sum(dim=1).cpu().numpy())
  want = stable(norms)
  assert orc._min_adjacent_gap([norms[i] for i in want], nh - 1) > 1e-6
  attack = bz.engine.AntiCGE(rows, f, f)
  attack()
  torch.cuda.synchronize()
  assert attack._ws[:4 * nh].view(torch.int32).cpu().tolist() == want
  one = sharded.ShardedAntiCGE(rows, f, f)
  one.sum(one.norms().unsqueeze(0))
  torch.cuda.synchronize()
  assert one.order.cpu().tolist() == want
  maxpos = nh - f
  presum = rows[want[0]].clone()
  for i in want[:maxpos]:
    presum = presum + rows[i]
  assert torch.equal(one.byz.view(torch.int32), presum.view(torch.int32))
