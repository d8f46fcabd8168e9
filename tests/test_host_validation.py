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

# Every distance-rule entry point with its parameters, in ABI order.  The defaults below pass every
# check; each case replaces a few of them so that exactly one check fails.
_PARAMS = {
  "bz_krum": "rows n f m d out order ws ws_bytes stream",
  "bz_krum_reuse": "rows n f m d out order old_index cache_in u_old cache_out mode_out ws ws_bytes stream",
  "bz_krum_peers": "rows n f m d out order status rank nranks blocks flags epoch ws ws_bytes stream",
  "bz_bulyan": "rows n f m d out order status ws ws_bytes stream",
  "bz_bulyan_reuse": "rows n f m d out order status old_index cache_in u_old cache_out mode_out ws ws_bytes stream",
  "bz_bulyan_peers": "rows n f m d out order status rank nranks blocks flags epoch ws ws_bytes stream",
  "bz_brute": "rows n f d out order status ws ws_bytes stream",
  "bz_brute_reuse": "rows n f d out order status old_index cache_in u_old cache_out mode_out ws ws_bytes stream",
  "bz_krum_select": "parts nparts n f order stream",
  "bz_bulyan_select": "parts nparts n f m order status stream",
  "bz_brute_select": "parts nparts n f order status stream",
  "bz_rowdist_select": "parts nparts n sqrt_norm order stream",
  "bz_krum_select_peers": "peers npeers n f order stream",
  "bz_bulyan_select_peers": "peers npeers n f m order status stream",
  "bz_brute_select_peers": "peers npeers n f order status stream",
  "bz_rowdist_select_peers": "peers npeers n sqrt_norm order stream",
  "bz_bulyan_reduce": "rows n f m order status d out stream",
}
_DEFAULTS = dict(rows=[0x1000 + 0x100 * i for i in range(64)], n=11, f=2, m=3, d=64, out=0x9000, order=0x9200,
                 status=0x9100, ws=0xB000, ws_bytes=None, stream=None, old_index=None, cache_in=None, u_old=0,
                 cache_out=0xC000, mode_out="int", rank=1, nranks=3, blocks=[0x10000 + 0x1000 * r for r in range(3)],
                 flags=[0x20000 + 0x40 * r for r in range(3)], epoch=7, parts=0x40000, nparts=2,
                 peers=[0x50000 + 0x1000 * r for r in range(16)], npeers=2, sqrt_norm=0)

def _whole(who, f_bad, f_text, m_bad=None, m_text=None):
  """ The checks of a whole rule after its own prologue: rows, rule, workspace. """
  cases = [(dict(rows=None), -1, f"{who}: rows is NULL"),
           (dict(n=0), -1, f"{who}: n = 0, expected n >= 1"),
           (dict(n=65), -2, f"{who}: n = 65 exceeds BZ_MAX_N"),
           (dict(out=None), -1, f"{who}: output pointer is NULL"),
           (dict(f=-1), -1, f"{who}: f = -1 not executable with n = 11"),
           (dict(f=f_bad), -1, f"{who}: f = {f_bad} not executable with n = 11{f_text}"),
           (dict(f=-1, ws_bytes=8), -1, f"{who}: f = -1"),                    # the rule before the workspace
           (dict(ws_bytes=-8), -4, f"{who}: workspace of"),                   # need - 8
           (dict(ws=0xB004), -4, f"{who}: workspace of")]
  if m_bad is not None:
    cases += [(dict(m=0), -1, f"{who}: m = 0, expected 1..{m_text}"),
              (dict(m=m_bad), -1, f"{who}: m = {m_bad}, expected 1..{m_text}")]
  return cases

_KRUM = _whole("bz_krum", 10, " (need n - f - 1 >= 1)", 12, 11)
_BULYAN = _whole("bz_bulyan", 3, " (need n >= 4f + 3)", 8, 7)
_BRUTE = _whole("bz_brute", 11, "") + [
  (dict(n=64, f=32), -2, "bz_brute: C(64, 32) subsets exceed the 2^31 limit"),
  (dict(n=64, f=32, ws_bytes=-8), -4, "bz_brute: workspace of"),            # the workspace before the subset count
  (dict(n=64, f=32, d=0), 0, None)]                                          # d == 0: nothing to select

def _reuse(who):
  return [(dict(cache_out=None), -1, f"{who}: cache_out / mode_out is NULL"),
          (dict(mode_out=None), -1, f"{who}: cache_out / mode_out is NULL"),
          (dict(cache_in=0xC000), -1, f"{who}: cache_in and cache_out must differ"),
          (dict(cache_in=0xD000, u_old=0), -1, f"{who}: u_old = 0"),
          (dict(cache_in=0xD000, u_old=65), -1, f"{who}: u_old = 65"),
          (dict(cache_out=None, rows=None, f=-1), -1, f"{who}: cache_out / mode_out is NULL")]

def _peers(who):
  return [(dict(rank=3), -1, f"{who}: rank 3 of 3"),
          (dict(status=None), -1, f"{who}: NULL peer table or status"),
          (dict(blocks=[0x10000, 0, 0x12000]), -1, f"{who}: peer 1: NULL or misaligned"),
          (dict(rank=3, rows=None, f=-1), -1, f"{who}: rank 3 of 3")]

def _phase_b(who, rule):
  """ Phase B: the gathered blocks or the peer table, n, then the rule (`rule`: its failing cases). """
  if who.endswith("_peers"):
    cases = [(dict(peers=None), -1, f"{who}: NULL argument"),
             (dict(npeers=0), -1, f"{who}: npeers = 0 outside 1..16"),
             (dict(npeers=17), -1, f"{who}: npeers = 17 outside 1..16"),
             (dict(peers=[0x50000, 0]), -1, f"{who}: peers[1] is NULL or misaligned"),
             (dict(peers=[0x50000, 0x51004]), -1, f"{who}: peers[1] is NULL or misaligned")]
  else:
    cases = [(dict(parts=None), -1, f"{who}: NULL argument or nparts < 1"),
             (dict(nparts=0), -1, f"{who}: NULL argument or nparts < 1")]
  cases += [(dict(order=None), -1, f"{who}: NULL argument"),
            (dict(n=0), -2, f"{who}: n = 0 outside 1..64"),
            (dict(n=65, f=-1), -2, f"{who}: n = 65 outside 1..64")]
  return cases + [(kw, code, f"{who}: {text}") for kw, code, text in rule]

_KRUM_B = [(dict(f=-1), -1, "f = -1 not executable"), (dict(f=10), -1, "f = 10 not executable with n = 11"),
           (dict(n=1, f=0), -1, "f = 0 not executable with n = 1")]
_BULYAN_B = [(dict(f=3), -1, "f = 3 not executable with n = 11 (need n >= 4f + 3)"),
             (dict(m=0), -1, "m = 0, expected 1..7"), (dict(m=8), -1, "m = 8, expected 1..7")]
_BRUTE_B = [(dict(f=-1), -1, "f = -1 not executable with n = 11"), (dict(f=11), -1, "f = 11 not executable"),
            (dict(n=64, f=32), -2, "C(64, 32) subsets exceed the 2^31 limit")]

_CASES = {
  "bz_krum": _KRUM,
  "bz_krum_reuse": _reuse("bz_krum_reuse") + _KRUM,
  "bz_krum_peers": _peers("bz_krum_peers") + _KRUM,
  "bz_bulyan": _BULYAN,
  "bz_bulyan_reuse": _reuse("bz_bulyan_reuse") + _BULYAN,
  "bz_bulyan_peers": _peers("bz_bulyan_peers") + _BULYAN,
  "bz_brute": _BRUTE,
  "bz_brute_reuse": _reuse("bz_brute_reuse") + _BRUTE,
  "bz_krum_select": _phase_b("bz_krum_select", _KRUM_B),
  "bz_bulyan_select": _phase_b("bz_bulyan_select", _BULYAN_B),
  "bz_brute_select": _phase_b("bz_brute_select", _BRUTE_B),
  "bz_rowdist_select": _phase_b("bz_rowdist_select", []),
  "bz_krum_select_peers": _phase_b("bz_krum_select_peers", _KRUM_B),
  "bz_bulyan_select_peers": _phase_b("bz_bulyan_select_peers", _BULYAN_B),
  "bz_brute_select_peers": _phase_b("bz_brute_select_peers", _BRUTE_B),
  "bz_rowdist_select_peers": _phase_b("bz_rowdist_select_peers", []),
  "bz_bulyan_reduce": [(dict(rows=None), -1, "bz_bulyan_reduce: rows is NULL"),
                       (dict(n=65), -2, "bz_bulyan_reduce: n = 65 exceeds BZ_MAX_N"),
                       (dict(order=None, f=3), -1, "bz_bulyan_reduce: order is NULL"),
                       (dict(f=3), -1, "bz_bulyan_reduce: f = 3 not executable with n = 11 (need n >= 4f + 3)"),
                       (dict(m=8), -1, "bz_bulyan_reduce: m = 8, expected 1..7")],
}

@pytest.mark.parametrize("name", sorted(_CASES))
def test_distance_rule_entry_points_check_every_argument_before_cuda(name):
  """ Each case fails one argument check of `name` (or, brute at d = 0, returns before any launch);
  the return code and the `bz_last_error` text, with the name of the entry point that reports it, are
  pinned.  The addresses are fake and never dereferenced.  The one exception is the status word of
  `bz_krum_peers`, which older builds zeroed before checking the rule: on a host with a GPU it is a
  real device buffer. """
  lib = _lib.lib()
  fn = getattr(lib, name)
  status_buf = None
  if name == "bz_krum_peers" and torch.cuda.is_available():
    status_buf = torch.zeros(1, dtype=torch.int32, device="cuda")
  for kw, code, text in _CASES[name]:
    a = dict(_DEFAULTS, **kw)
    if a["ws_bytes"] is None or a["ws_bytes"] < 0:
      a["ws_bytes"] = lib.bz_workspace_bytes(a["n"]) + (a["ws_bytes"] or 0)
    if status_buf is not None and a["status"] is not None:
      a["status"] = status_buf.data_ptr()
    mode_out = ctypes.c_int(5)
    args = []
    for p in _PARAMS[name].split():
      v = a[p]
      if p in ("rows", "blocks", "flags", "peers"):
        v = None if v is None else (ctypes.c_void_p * len(v))(*v)
      elif p == "mode_out":
        v = None if v is None else ctypes.byref(mode_out)
      elif p in ("out", "order", "status", "ws", "stream", "old_index", "cache_in", "cache_out", "parts"):
        v = None if v is None else ctypes.c_void_p(v)
      args.append(v)
    rc = fn(*args)
    case = f"{name}({kw})"
    assert rc == code, f"{case} returned {rc}, expected {code}: {lib.bz_last_error().decode()}"
    if text is not None:
      assert text in lib.bz_last_error().decode(), f"{case}: {lib.bz_last_error().decode()!r} lacks {text!r}"
    if "mode_out" in _PARAMS[name] and a["mode_out"] is not None:
      # the reuse calls report "no fused pass" once their own checks have passed
      reuse_failed = text is not None and text.startswith(name + ":")
      assert mode_out.value == (5 if reuse_failed else -1), case
  if status_buf is not None:
    torch.cuda.synchronize()

def test_check_maps_codes_to_exceptions():
  lib = _lib.lib()
  code = lib.bz_median(None, 3, 16, None, None)
  with pytest.raises(ValueError):
    _lib.check(code, "bz_median")
  _lib.check(0, "anything")
