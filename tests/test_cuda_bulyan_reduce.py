# coding: utf-8
"""Bulyan's reduce (`bz_distance_reduce`, rule bulyan) at every theta, against the column reference of
tests/bulyan_columns.py.  The caller chooses `order` and passes status 0, so stage 1 is known on the host
(`orc.bulyan_stage1`), and the output must be K4's order bit for bit, its window a valid closest set, and
within 1e-6 of the column's scale of the exact mean of that window.

  * K4-wide, one kernel per bucket of 8 theta values: every theta in 33..126, once with the largest f that
    keeps n <= 128 and n >= 4f + 3 (the window then moves over 2f places), once with f in {0, 1}; m in
    {1, 2, m_max / 2, m_max - 1, m_max}.  Rows are seeded stacks whose Byzantine rows are one aliased tensor.
  * The 64-row K4 (`k4_bulyan<THETA>`, and the compile-time kernels where (n, f) and m = m_max match one):
    every theta in 1..60 the same way at n <= 64, m in {1, m_max}; theta 61 and 62 (n = 63 and 64 with f = 0)
    run K4-wide.
  * Constructed columns at m = 1, where stage 1 is the rows in `order`: median ties, plateaus longer than
    beta, key ties across the window's edges, signed zeros and subnormals, +-inf, a NaN, overflowing sums.
  * A non-zero status fills the output with NaN."""

import ctypes

import numpy as np
import pytest

import bulyan_columns as bc
from test_cuda_distance_wide import CODES, device_rows, stack

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
D = 200          # one full CTA of 128 coordinates and a partial one

def _lib():
  from byzantinemomentum_b200 import _lib
  return _lib.lib()

def reduce(rows, f, m, order, status=0):
  n, d = len(rows), rows[0].numel()
  dev = rows[0].device
  lib = _lib()
  meta = torch.tensor(list(order) + [status], dtype=torch.int32, device=dev)
  out = torch.full((d,), 7., dtype=torch.float32, device=dev)
  ptrs = (ctypes.c_void_p * n)(*[r.data_ptr() for r in rows])
  rc = lib.bz_distance_reduce(CODES["bulyan"], ptrs, n, f, m, 0, meta.data_ptr(), meta.data_ptr() + 4 * n, d,
                              out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
  assert rc == 0, lib.bz_last_error()
  torch.cuda.synchronize(dev)
  return out.cpu().numpy()

def theta_sizes(theta, n_max):
  """ (n, f) reaching theta = n - 2f - 2: the largest f with n <= n_max and n >= 4f + 3, then f = 0 and 1. """
  big = min((theta - 1) // 2, (n_max - theta - 2) // 2)
  out = [(theta + 2 * f + 2, f) for f in sorted({big, 0, 1}) if f >= 0 and theta + 2 * f + 2 <= n_max and theta >= 2 * f + 1]
  return sorted(set(out), key=lambda nf: -nf[1])

def test_theta_sizes():
  assert theta_sizes(121, 128)[0] == (127, 2) and theta_sizes(112, 128)[0] == (128, 7)
  assert theta_sizes(73, 128)[0] == (127, 26) and theta_sizes(40, 128)[0] == (80, 19)
  assert theta_sizes(126, 128) == [(128, 0)]
  for theta in range(33, 127):
    assert any(n > 64 for n, _ in theta_sizes(theta, 128)), theta

def sweep(thetas, n_max, ms_of, seed):
  for theta in thetas:
    for n, f in theta_sizes(theta, n_max):
      x, nh = stack(n, n // 4, D, seed=seed + 131 * theta + f)
      rows = device_rows(x, nh)
      perm = np.random.default_rng(seed + theta).permutation(n)
      m_max = n - f - 2
      for m in sorted(set(ms_of(m_max))):
        got = reduce(rows, f, m, perm)
        bc.check(got, bc.stage1(x, perm, f, m), f, bc.uses_wide(n, f), f"theta={theta} n={n} f={f} m={m}")

@pytest.mark.parametrize("bucket", range(5, 17))
def test_wide_buckets_at_every_theta(bucket):
  thetas = [t for t in range(8 * bucket - 7, 8 * bucket + 1) if 33 <= t <= 126]
  sweep(thetas, 128, lambda mm: (1, 2, mm // 2, mm - 1, mm), seed=10_000)

@pytest.mark.parametrize("lo", [1, 21, 41])
def test_64_row_kernels_at_every_theta(lo):
  sweep(range(lo, lo + 22 if lo == 41 else lo + 20), 64, lambda mm: (1, mm), seed=20_000)

@pytest.mark.parametrize("n,f", [(7, 0), (11, 2), (25, 5), (64, 1), (64, 0), (65, 15), (66, 1), (97, 0), (127, 26),
                                 (128, 1), (128, 0)])
def test_constructed_columns(n, f):
  """ m = 1: stage 1 is rows order[0 .. theta-1] as they are; the constructed columns go there, the other rows
  are random. """
  m_max, theta, beta = bc.sizes(n, f)
  cols = bc.constructed_columns(theta, f, seed=n + f)
  rng = np.random.default_rng(n)
  x = rng.standard_normal((n, cols.shape[1])).astype(np.float32)
  perm = rng.permutation(n)
  x[perm[:theta]] = cols
  dev = torch.device("cuda", 0)
  rows = [torch.from_numpy(x[i].copy()).to(dev) for i in range(n)]
  got = reduce(rows, f, 1, perm)
  s = bc.stage1(x, perm, f, 1)
  assert np.array_equal(s, cols + np.float32(0.), equal_nan=True)        # the rows themselves, -0 added to +0
  bc.check(got, s, f, bc.uses_wide(n, f), f"n={n} f={f}")
  assert np.isnan(got[bc.CONSTRUCTED.index("nan")])
  assert np.isnan(reduce(rows, f, 1, perm, status=2)).all()
