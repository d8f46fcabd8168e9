# coding: utf-8
"""Host-side argument validation (CPU suite).  `engine._validate` runs before anything touches
CUDA, and the C entry points check their arguments before the first CUDA call, so both are
testable without a GPU: invalid calls must fail with the documented error, never reach a kernel."""

import ctypes

import pytest

torch = pytest.importorskip("torch")

from byzantinemomentum_b200 import _lib, engine

def test_validate_rejects_malformed_gradient_lists():
  ok = [torch.zeros(8) for _ in range(3)]
  first, contiguous = engine._validate(ok)
  assert first is ok[0] and contiguous
  with pytest.raises(ValueError):
    engine._validate([])
  with pytest.raises(ValueError):
    engine._validate("not a list")
  with pytest.raises(TypeError):
    engine._validate([1.0, 2.0])
  with pytest.raises(TypeError):
    engine._validate([torch.zeros(8, dtype=torch.float64)] * 2)
  with pytest.raises(TypeError):
    engine._validate([torch.zeros(8), torch.zeros(8, dtype=torch.float16)])
  with pytest.raises(ValueError):
    engine._validate([torch.zeros(8), torch.zeros(9)])
  with pytest.raises(ValueError):
    engine._validate([torch.zeros(2, 4)])
  with pytest.raises(ValueError):
    engine._validate([torch.zeros(4)] * (_lib.MAX_N + 1))
  strided = torch.zeros(8, 3)[:, 0]
  assert engine._validate([strided, strided])[1] is False

def test_aksel_mode_is_checked_before_the_device_is_touched():
  with pytest.raises(NotImplementedError):
    engine.aksel([torch.zeros(4)] * 5, 1, mode="zzz")

def _rows(n, address=0x1000):
  return (ctypes.c_void_p * n)(*[address + 0x100 * i for i in range(n)])

def test_c_abi_rejects_bad_arguments_without_a_gpu():
  """ Every refusal below happens in the argument checks of api.cu, before any CUDA call; the
  pointers are never dereferenced (they are fake addresses). """
  lib = _lib.lib()
  out = ctypes.c_void_p(0x9000)
  def message():
    return lib.bz_last_error().decode()
  assert lib.bz_median(None, 3, 16, out, None) == -1 and "rows is NULL" in message()
  assert lib.bz_median(_rows(3), 0, 16, out, None) == -1
  assert lib.bz_median(_rows(3), 65, 16, out, None) == -2 and "BZ_MAX_N" in message()
  assert lib.bz_median(_rows(3), 3, -1, out, None) == -1
  assert lib.bz_median(_rows(3), 3, 16, None, None) == -1 and "output" in message()
  assert lib.bz_median(_rows(3, address=0x1002), 3, 16, out, None) == -1 and "aligned" in message()
  assert lib.bz_trmean(_rows(5), 5, 3, 16, out, None) == -1 and "n - 2f" in message()
  assert lib.bz_trmean(_rows(5), 5, -1, 16, out, None) == -1
  # d == 0 is a valid no-op for the coordinate-wise rules
  assert lib.bz_median(_rows(3), 3, 0, None, None) == 0
  assert lib.bz_trmean(_rows(5), 5, 2, 0, None, None) == 0
  # workspace: too small / misaligned
  need = lib.bz_workspace_bytes(7)
  assert need >= 7 * 7 * 8
  order = ctypes.c_void_p(0xA000)
  assert lib.bz_krum(_rows(7), 7, 2, 3, 16, out, order, ctypes.c_void_p(0xB000), need - 8, None) == -4 and "workspace" in message()
  assert lib.bz_krum(_rows(7), 7, 2, 3, 16, out, order, ctypes.c_void_p(0xB004), need, None) == -4
  assert lib.bz_avg_dev_max(_rows(7), 7, 16, out, None, ctypes.c_void_p(0xB000), need, None) == -1 and "stats" in message()
  assert lib.bz_aksel(_rows(7), 7, 2, 9, 16, out, order, ctypes.c_void_p(0xB000), need, None) == -1 and "mode" in message()

@pytest.mark.parametrize("name", ["bz_krum_peers", "bz_bulyan_peers"])
def test_fused_peer_calls_reject_bad_exchange_arguments_without_a_gpu(name):
  """ `bz_*_peers` check rank, nranks, status and the peer tables before any CUDA call (fake,
  never dereferenced addresses). """
  lib = _lib.lib()
  fn = getattr(lib, name)
  n, f, m, d = 11, 2, 3, 64
  need = lib.bz_workspace_bytes(n)
  table = lambda addrs: (ctypes.c_void_p * len(addrs))(*addrs)
  ok = dict(rank=1, nranks=3, status=0x9100, blocks=[0x10000 + 0x1000 * r for r in range(3)],
            flags=[0x20000 + 0x40 * r for r in range(3)])
  def call(**kw):
    a = dict(ok, **kw)
    status = None if a["status"] is None else ctypes.c_void_p(a["status"])
    blocks = None if a["blocks"] is None else table(a["blocks"])
    flags = None if a["flags"] is None else table(a["flags"])
    return fn(_rows(n), n, f, m, d, ctypes.c_void_p(0x9000), ctypes.c_void_p(0x9200), status, a["rank"], a["nranks"],
              blocks, flags, 7, ctypes.c_void_p(0xB000), need, None)
  message = lambda: lib.bz_last_error().decode()
  assert call(rank=3) == -1 and "rank 3 of 3" in message()
  assert call(rank=-1) == -1
  assert call(nranks=0, rank=0) == -1
  assert call(nranks=17, rank=0, blocks=ok["blocks"] * 6, flags=ok["flags"] * 6) == -1 and "of 17" in message()
  assert call(status=None) == -1 and "status" in message()
  assert call(blocks=None) == -1 and call(flags=None) == -1
  for bad in (0, 0x10004):                                        # NULL, not 8-byte aligned
    assert call(blocks=[ok["blocks"][0], bad, ok["blocks"][2]]) == -1 and "peer 1" in message()
  for bad in (0, 0x20002):                                        # NULL, not 4-byte aligned
    assert call(flags=[ok["flags"][0], ok["flags"][1], bad]) == -1 and "peer 2" in message()

def test_check_maps_codes_to_exceptions():
  lib = _lib.lib()
  code = lib.bz_median(None, 3, 16, None, None)
  with pytest.raises(ValueError):
    _lib.check(code, "bz_median")
  _lib.check(0, "anything")
