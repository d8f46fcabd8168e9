# coding: utf-8
"""GPU parity of the coordinate-wise rules (K1) on the values sorting networks get wrong: NaN of
both signs and with non-canonical payloads, +-inf, +-0, subnormals and +-FLT_MAX, placed so that
some VEC groups of a row are all finite and others mixed.  Every n from 1 to 64 runs through the
generic `k1_median` / `k1_sorted` (16-byte aligned rows and mixed-offset views, which take the
scalar form even where n has a compile-time trimmed-mean network); shared-offset views take the
shifted vector path.  Median and trimmed mean are bit-exact against the oracle; phocas and meamed
are value for value K1's closest epilogue restated in tests/closest_columns.py, and meet the scaled
bar of tests/parity.py against the oracle wherever the chosen values are unique."""

import ctypes

import numpy as np
import pytest

import closest_columns as cc
import parity
from oracle import byzoracle as orc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"

SPECIALS = np.array([0x7fc00000, 0xffc00000, 0x7f800001, 0xff800001, 0x7fffffff,      # NaN: +/-, payloads
                     0x7f800000, 0xff800000, 0x00000000, 0x80000000,                  # +-inf, +-0
                     0x00000001, 0x80000001, 0x007fffff, 0x807fffff, 0x00400000,      # subnormals
                     0x7f7fffff, 0xff7fffff, 0x00800000, 0x80800000], dtype=np.uint32).view(np.float32)   # +-FLT_MAX, +-FLT_MIN

def _lib():
  from byzantinemomentum_b200 import _lib
  return _lib.lib()

def _ptrs(rows):
  return (ctypes.c_void_p * len(rows))(*[r.data_ptr() for r in rows])

def _stream():
  return torch.cuda.current_stream().cuda_stream

def _stack(n, d, seed, nonfinite=True):
  """ [n, d] rows: finite noise, ties, and the special values in every fourth 64-column block only
  (the other blocks' vector groups stay finite); blocks alternate between sparse and dense specials. """
  rng = np.random.default_rng(seed)
  x = rng.standard_normal((n, d)).astype(np.float32)
  x[:, 1::5] = np.round(x[:, 1::5] * 2) / 2                     # exact ties
  for b, j0 in enumerate(range(0, d, 256)):
    blk = slice(j0, min(j0 + 64, d))
    width = blk.stop - blk.start
    pool = SPECIALS if nonfinite else SPECIALS[np.isfinite(SPECIALS)]
    mask = rng.random((n, width)) < (0.05 if b % 2 else 0.4)
    vals = pool[rng.integers(0, pool.size, (n, width))]
    x[:, blk] = np.where(mask, vals, x[:, blk])
  return x

def _device_rows(x, offsets):
  n, d = x.shape
  rows = []
  for i in range(n):
    off = offsets[i % len(offsets)]
    buf = torch.empty(d + 8, device=DEV)
    buf[off:off + d] = torch.from_numpy(x[i])
    rows.append(buf[off:off + d])
  return rows

def _call(name, rows, d, f=None):
  lib = _lib()
  out = torch.full((d,), float("nan"), device=DEV)
  fn = getattr(lib, "bz_" + name)
  rc = fn(_ptrs(rows), len(rows), d, out.data_ptr(), _stream()) if f is None else fn(_ptrs(rows), len(rows), f, d, out.data_ptr(), _stream())
  assert rc == 0, lib.bz_last_error()
  return out.cpu().numpy()

def _check(x, rows, what, fs=None):
  n, d = x.shape
  host = [x[i] for i in range(n)]
  parity.assert_bit_exact(_call("median", rows, d), orc.median(host), f"median {what}")
  if fs is None:
    fs = sorted({1, (n - 1) // 4, (n - 1) // 2} - {0}) if n >= 3 else []
  for f in fs:
    parity.assert_bit_exact(_call("trmean", rows, d, f), orc.trmean(host, f), f"trmean {what} f={f}")
    for name in cc.MODES:
      cc.check_kernel(_call(name, rows, d, f), x, f, name, f"{name} {what} f={f}")

@pytest.mark.parametrize("n", list(range(1, 65)))
def test_special_values_every_n(n):
  d = 1031 + 4 * n
  x = _stack(n, d, 500 + n)
  _check(x, _device_rows(x, [0]), f"n={n} aligned")
  _check(x, _device_rows(x, [0, 1, 2, 3, 1]), f"n={n} mixed offsets")

@pytest.mark.parametrize("n", [11, 25, 51])
def test_compile_time_n_take_the_generic_kernel_on_mixed_offsets(n):
  """ n = 11, 25, 51 have one pruned trmean / phocas / meamed network per f; mixed offsets bypass them. """
  d = 2053
  x = _stack(n, d, 900 + n)
  _check(x, _device_rows(x, [1, 3, 0, 2]), f"n={n} mixed offsets", fs=list(range(1, (n - 1) // 2 + 1)))

@pytest.mark.parametrize("n", [11, 12, 25, 29, 33, 40, 51, 64])
@pytest.mark.parametrize("offset", [1, 2, 3])
def test_shared_offset_views(n, offset):
  """ All rows (and the output) at the same offset: the shifted vector path, VEC = 2 beyond n = 28. """
  d = 3001
  x = _stack(n, d, 1300 + 7 * n + offset)
  rows = _device_rows(x, [offset])
  _check(x, rows, f"n={n} offset={offset}")
  lib = _lib()
  outbig = torch.full((d + 8,), float("nan"), device=DEV)
  out = outbig[offset:offset + d]
  rc = lib.bz_median(_ptrs(rows), n, d, out.data_ptr(), _stream())
  assert rc == 0, lib.bz_last_error()
  parity.assert_bit_exact(out.cpu().numpy(), orc.median([x[i] for i in range(n)]), f"median n={n} offset output")
  assert torch.isnan(outbig[:offset]).all() and torch.isnan(outbig[offset + d:]).all()
