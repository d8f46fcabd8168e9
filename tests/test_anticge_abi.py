# coding: utf-8
"""The attack against CGE (include/byzagg_anticge.h) on the CPU: the header and its binding, the argument checks
(before any CUDA call, with fake pointers), the register and stack budgets of K10 and K11, the NumPy oracle
against the reference's recorded outputs (`tests/golden/anticge/`), and which calls `plugin.install_attacks`
hands to the device.  No compute calls here."""

import ctypes
import math
import pathlib
import re
import shutil
import subprocess
import types

import numpy as np
import pytest

import anticge_oracle as aorc

ROOT = pathlib.Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden" / "anticge"
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
# The output's bound against the reference: maxnorm and attnorm come from fp32 norms that may differ from ATen's in
# their last bit, so the factor, and each coordinate, may differ by a few ulp.
RTOL = 2. ** -21

def declared_symbols():
  text = (ROOT / "include" / "byzagg_anticge.h").read_text()
  return sorted(set(re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", text)))

def goldens():
  return [pytest.param(path, id=path.stem) for path in sorted(GOLDEN.glob("anticge_*.npz"))]

def close(got, want, rtol=RTOL):
  """ Equal where the reference is not finite (NaN where NaN, same infinity), within rtol elsewhere. """
  got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
  same = (np.isnan(got) & np.isnan(want)) | (got == want)
  near = np.abs(got - want) <= rtol * np.abs(want)
  return bool(np.all(same | near))

def test_header_declares_the_calls_and_byzagg_h_includes_it():
  assert declared_symbols() == ["bz_anticge", "bz_anticge_partial", "bz_anticge_scale", "bz_anticge_workspace_bytes"]
  assert '#include "byzagg_anticge.h"' in (ROOT / "include" / "byzagg.h").read_text()
  assert "byzagg_anticge.h" in (ROOT / "byzantinemomentum_b200" / "csrc" / "Makefile").read_text()
  own = re.findall(r"BZ_API\s+[\w\s\*]+?\b(bz_\w+)\s*\(", (ROOT / "include" / "byzagg.h").read_text())
  assert not set(own) & set(declared_symbols())

def test_library_exports_the_calls_and_the_table_matches():
  from byzantinemomentum_b200 import _lib
  handle = ctypes.CDLL(str(_lib.library_path()))
  for name in declared_symbols():
    assert hasattr(handle, name), name
  assert sorted(_lib.ANTICGE_SIGNATURES) == declared_symbols()
  others = [_lib.SIGNATURES, _lib.SHARD_SIGNATURES, _lib.ATTACK_SIGNATURES, _lib.SEARCH_SHARD_SIGNATURES,
            _lib.SEARCH_PEER_SIGNATURES, _lib.COORDINATE_SIGNATURES, _lib.PEER_NEXT_SIGNATURES, _lib.DISTANCE_SIGNATURES,
            _lib.DISTANCE_SHARD_SIGNATURES]
  assert not set(_lib.ANTICGE_SIGNATURES) & set().union(*others)
  for name, (restype, argtypes) in _lib.ANTICGE_SIGNATURES.items():
    assert getattr(_lib.lib(), name).argtypes == argtypes

def test_workspace_sizes():
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  sizes = [lib.bz_anticge_workspace_bytes(n) for n in range(1, 129)]
  assert all(s % 256 == 0 for s in sizes) and sizes == sorted(sizes) and sizes[0] < sizes[-1]
  assert lib.bz_anticge_workspace_bytes(0) == sizes[0] and lib.bz_anticge_workspace_bytes(500) == sizes[-1]

def test_calls_reject_bad_arguments_before_touching_the_gpu():
  """ Only invalid calls here (and d = 0, which launches nothing): the pointers are fake addresses. """
  from byzantinemomentum_b200 import _lib
  lib = _lib.lib()
  rows = lambda n, address=0x1000: (ctypes.c_void_p * n)(*[address + 0x100 * i for i in range(n)])
  out, big = ctypes.c_void_p(0x90000), 1 << 40
  def call(table=None, nh=25, f_decl=5, f_real=5, d=16, dest=out, ws=0xc0000, ws_bytes=big):
    return lib.bz_anticge(rows(max(nh, 1)) if table is None else table, nh, f_decl, f_real, d, dest, ctypes.c_void_p(ws),
                          ws_bytes, None)
  def message():
    return lib.bz_last_error().decode()
  assert call(nh=0) == -1 and "n = 0" in message()
  assert call(nh=129) == -2 and "128" in message()
  for f_decl in (0, -1, 26):                             # maxpos = nh - f_decl outside 0..nh - 1
    assert call(f_decl=f_decl) == -1 and "f_decl" in message(), f_decl
  assert call(f_real=-1) == -1 and "f_real" in message()
  assert lib.bz_anticge(None, 25, 5, 5, 16, out, ctypes.c_void_p(0xc0000), big, None) == -1 and "rows is NULL" in message()
  assert call(dest=None) == -1 and "output" in message()
  assert call(table=rows(25, address=0x1002)) == -1 and "aligned" in message()
  with_null = rows(100)
  with_null[70] = None
  assert call(table=with_null, nh=100, f_decl=10) == -1 and "rows[70] is NULL" in message()
  need = lib.bz_anticge_workspace_bytes(25)
  assert call(ws_bytes=need - 1) == -4 and "workspace" in message()
  assert call(ws=0xc0004) == -4 and call(ws=0) == -4
  for nh in (1, 64, 65, 128):                            # d = 0: a no-op, the fill included
    assert call(nh=nh, f_decl=1, f_real=0, d=0, dest=None) == 0
    assert call(nh=nh, f_decl=1, f_real=3, d=0, dest=None) == 0
  # the d-sharded calls
  order, partial = ctypes.c_void_p(0xa0000), ctypes.c_void_p(0xb0000)
  assert lib.bz_anticge_partial(rows(25), 25, 0, order, 16, out, partial, ctypes.c_void_p(0xc0000), big, None) == -1
  assert lib.bz_anticge_partial(rows(25), 25, 5, None, 16, out, partial, ctypes.c_void_p(0xc0000), big, None) == -1
  assert lib.bz_anticge_partial(rows(25), 25, 5, order, 16, out, None, ctypes.c_void_p(0xc0000), big, None) == -1
  assert lib.bz_anticge_partial(rows(25), 25, 5, order, 16, out, partial, ctypes.c_void_p(0xc0000), 8, None) == -4
  blocks = ctypes.c_void_p(0xd0000)
  assert lib.bz_anticge_scale(None, order, partial, 1, 25, 5, 16, out, None) == -1
  assert lib.bz_anticge_scale(blocks, order, partial, 0, 25, 5, 16, out, None) == -1 and "nparts" in message()
  assert lib.bz_anticge_scale(blocks, order, partial, 2, 129, 5, 16, out, None) == -2
  assert lib.bz_anticge_scale(blocks, order, partial, 2, 25, 26, 16, out, None) == -1 and "f_decl" in message()
  assert lib.bz_anticge_scale(blocks, order, partial, 2, 25, 5, 16, None, None) == -1
  assert lib.bz_anticge_scale(blocks, order, partial, 2, 25, 5, -1, out, None) == -1
  assert lib.bz_anticge_scale(blocks, order, partial, 2, 25, 5, 0, None, None) == 0

@pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")
def test_k10_and_k11_fit_the_register_budget():
  """ K10 (both tables, both vector widths), K11 and the NaN fill: no stack, no spill. """
  from byzantinemomentum_b200 import _lib
  text = subprocess.run([CUOBJDUMP, "-res-usage", str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout
  usage = {name: (int(regs), int(stack)) for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text)}
  k10 = [name for name in usage if "k10_anticge_sum" in name]
  k11 = [name for name in usage if "k11_anticge_scale" in name]
  fill = [name for name in usage if "k_nan_fill" in name]
  assert len(k10) == 4 and len(k11) == 2 and len(fill) == 1
  for name in k10 + k11 + fill:
    regs, stack = usage[name]
    assert regs <= 255 and stack == 0, (name, regs, stack)

def test_goldens_cover_the_range_and_the_edge_cases():
  names = {path.stem[len("anticge_"):] for path in GOLDEN.glob("anticge_*.npz")}
  for nh in (1, 7, 25, 64, 65, 100, 128):
    assert f"n{nh}" in names, nh
  assert {"n25_maxpos0", "n25_fill", "n25_freal0", "n25_nan", "n25_inf", "n25_zero", "n25_overflow"} <= names
  assert sum(path.stat().st_size for path in GOLDEN.glob("*.npz")) < 1024 * 1024

@pytest.mark.parametrize("path", goldens())
def test_oracle_matches_the_reference(path):
  z = np.load(path)
  rows = [r for r in z["rows"]]
  f_decl, f_real = int(z["f_decl"]), int(z["f_real"])
  out, info = aorc.anticge(rows, f_decl, f_real, return_info=True)
  assert len(out) == int(z["count"]) == f_real and all(o is out[0] for o in out) and bool(z["aliased"])
  if f_real == 0:
    return
  if info["fill"]:
    assert np.isnan(out[0]).all() and np.isnan(z["out"]).all()
    return
  assert info["order"] == z["order"].tolist()
  assert np.array_equal(info["presum"].view(np.uint32), z["presum"].view(np.uint32))        # the sum: bit-exact
  ranked = [info["norms"][i] for i in info["order"]]
  assert close(ranked, z["norms"])
  assert close(out[0], z["out"]), np.max(np.abs(out[0] - z["out"]) / np.abs(z["out"]))

# ---- plugin.install_attacks(names=[... "anticge"]) ---------------------------------------------------------------

def _attacks():
  ns = types.SimpleNamespace(attacks={})
  def register(name, unchecked, check):
    if name in ns.attacks:
      raise KeyError(name)
    def checked(f_real, **kwargs):
      message = check(f_real=f_real, **kwargs)
      if message is not None:
        raise RuntimeError(message)
      return unchecked(f_real=f_real, **kwargs)
    checked.check, checked.checked, checked.unchecked = check, checked, unchecked
    ns.attacks[name] = checked
  ns.register = register
  for name in ("little", "empire", "bulyan", "empire-strict", "anticge", "nan"):
    register(name, (lambda name: lambda **kw: ("stock", name, kw))(name), lambda **kw: None)
  return ns

class OracleAttack:
  """ The device call replaced by the NumPy oracle; records its arguments. """
  def __init__(self):
    self.calls = []
  def anticge(self, grad_honests, f_decl, f_real):
    import torch
    self.calls.append((grad_honests, f_decl, f_real))
    out = aorc.anticge([g.numpy() for g in grad_honests], f_decl, f_real)
    row = torch.from_numpy(out[0]) if out else None
    return [row] * f_real

def test_install_attacks_keeps_its_default_and_takes_anticge_by_name(monkeypatch):
  torch = pytest.importorskip("torch")
  from byzantinemomentum_b200 import plugin
  attacks, backend = _attacks(), OracleAttack()
  assert plugin.install_attacks(_attacks(), backend=backend) == ["little", "empire", "bulyan", "empire-strict"]
  assert plugin.install_attacks(attacks, backend=backend, names=["anticge"]) == ["anticge"]
  assert attacks.attacks["little"].unchecked.__name__ == "<lambda>"          # untouched
  with pytest.raises(KeyError):
    plugin.install_attacks(_attacks(), backend=backend, names=["nan"])
  monkeypatch.setattr(plugin, "_is_cuda", lambda tensors: all(t.device.type == "cpu" for t in tensors))   # CPU rows stand for CUDA rows
  gen = torch.Generator().manual_seed(5)
  honest = [torch.randn(33, generator=gen) for _ in range(20)]
  run = lambda honest=honest, f_decl=4, f_real=4, **kw: attacks.attacks["anticge"].checked(grad_honests=honest, f_decl=f_decl,
                                                                                            f_real=f_real, **kw)
  def stock(result):
    return isinstance(result, tuple) and result[:2] == ("stock", "anticge")
  out = run(defense=None, model=None)
  assert backend.calls.pop() == (honest, 4, 4) and len(out) == 4 and all(o is out[0] for o in out)
  assert torch.equal(out[0], torch.from_numpy(aorc.anticge([g.numpy() for g in honest], 4, 4)[0]))
  for f_decl, f_real in ((20, 0), (1, 3), (3, 4)):       # maxpos = 0, f_real > f_decl (the fill), f_real = 0
    run(f_decl=f_decl, f_real=f_real)
    assert backend.calls.pop()[1:] == (f_decl, f_real)
  # every other case: the stock attack with its arguments unchanged
  assert stock(run(f_decl=0, f_real=0))                  # maxpos = nh: the reference raises IndexError
  assert stock(run(f_decl=0, f_real=1))                  # f_decl = 0 stays the reference's, its NaN fill included
  assert stock(run(f_decl=21))                           # maxpos < 0: the reference indexes from the end
  assert stock(run(f_decl=-2))
  assert stock(run(f_real=-1))
  assert stock(run(honest=honest * 7))                   # 140 rows > 128
  assert stock(run(honest=[g.double() for g in honest]))
  assert stock(run(honest=[g.view(3, 11) for g in honest]))
  assert stock(run(f_decl=4.))
  assert not backend.calls
  monkeypatch.setattr(plugin, "_is_cuda", lambda tensors: False)                # CPU tensors
  kind, name, kw = run(defense="x", model=None, extra=7)
  assert (kind, name) == ("stock", "anticge") and kw["extra"] == 7 and kw["f_decl"] == 4 and kw["grad_honests"] is honest
  assert not backend.calls
