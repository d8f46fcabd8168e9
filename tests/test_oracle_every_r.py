# coding: utf-8
"""CPU: the oracle's trimmed mean against torch's own CPU `mean(dim=0)` at every count of kept rows.

`orc.aten_mean_dim0` restates the order in which ATen sums the rows of `values[f:-f].mean(dim=0)` (16-row
blocks folded into a cascade of levels).  The reference's recorded outputs pin that order only at the few
(n, f) they hold; here it must give torch's bits at every R = n - 2f from 1 to 1100 (R <= 16, the folds at 16,
256 and 512 rows and just around them) and at 4095, 4096 and 4097 (the fold of the 4096-row level).  d = 64, a
multiple of 32: the trailing `d mod 32` columns that the oracle leaves unmodelled do not arise.

Then `orc.trmean(x, f)` is `x.sort(dim=0).values[f:n-f].mean(dim=0)` for every f at a few n.  f = 0 keeps the
whole column (`values[0:n]`), which is the library's contract; the reference's `values[f:-f]` would be empty
there.  The data is finite and free of -0.0, since torch's sort does not pin the order of -0.0 and +0.0."""

import numpy as np
import pytest

from oracle import byzoracle as orc

torch = pytest.importorskip("torch")
F32 = np.float32
D = 64

@pytest.fixture(autouse=True)
def one_thread():
  """ ATen's reduction may split the work over threads; one thread keeps it to the order the oracle states. """
  before = torch.get_num_threads()
  torch.set_num_threads(1)
  yield
  torch.set_num_threads(before)

def _rows(r, seed):
  """ [r, D] fp32 rows: noise spread over magnitudes, so that the summation order shows in the last bits. """
  rng = np.random.default_rng(seed)
  return (rng.standard_normal((r, D)) * np.exp2(rng.integers(-8, 9, (r, D)))).astype(F32)

def _assert_same_bits(got, want, what):
  got, want = np.asarray(got, dtype=F32), np.asarray(want, dtype=F32)
  bad = got.view(np.int32) != want.view(np.int32)
  assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} columns differ, first at {np.flatnonzero(bad)[:5]}"

RS = list(range(1, 1101)) + [4095, 4096, 4097]

@pytest.mark.parametrize("lo", list(range(1, 1101, 100)) + [4095])
def test_aten_mean_dim0_is_torch_mean_at_every_r(lo):
  """ Every R in [lo, lo + 100) of RS, one stack of rows per R. """
  for r in [r for r in RS if lo <= r < lo + 100]:
    x = _rows(r, 7_000 + r)
    _assert_same_bits(orc.aten_mean_dim0(x), torch.from_numpy(x).mean(dim=0).numpy(), f"R={r}")

def test_the_orders_differ():
  """ The check has teeth: at R = 18 and R = 300 a plain sequential sum gives other bits than torch. """
  for r in (18, 300):
    x = _rows(r, 7_000 + r)
    acc = np.zeros(D, dtype=F32)
    for k in range(r):
      acc = (acc + x[k]).astype(F32)
    seq = (acc / F32(r)).astype(F32)
    assert (seq.view(np.int32) != torch.from_numpy(x).mean(dim=0).numpy().view(np.int32)).any(), r

@pytest.mark.parametrize("n", [17, 18, 33, 64, 129, 300, 1024])
def test_trmean_is_torch_sort_then_mean_at_every_f(n):
  x = _rows(n, 8_000 + n)
  x[:, ::4] = np.round(x[:, ::4])                  # ties
  x[x == 0] = 1.                                   # no -0.0 (nor +0.0) for torch's sort to place
  t = torch.from_numpy(x).sort(dim=0).values
  for f in range(0, (n - 1) // 2 + 1):
    _assert_same_bits(orc.trmean(x, f), t[f:n - f].mean(dim=0).numpy(), f"n={n} f={f}")
