# coding: utf-8
"""`sharded.aggregate` in-process, without a process group (a world of one rank), on the NumPy
stand-in `tests/fake_backend.py`: the phase chain of every distance-based rule must give the
single-process oracle's result, and it must refuse what the single-GPU call refuses."""

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import parity
from fake_backend import OracleBackend
from oracle import byzoracle as orc
from byzantinemomentum_b200 import sharded

CASES = [("krum", dict(f=3)), ("krum", dict(f=3, m=2)), ("bulyan", dict(f=2)), ("brute", dict(f=3)),
         ("aksel", dict(f=3)), ("aksel", dict(f=3, mode="n-f")), ("cge", dict(f=3))]

def _inputs(n=11, nb=3, d=601):
  gen = torch.Generator().manual_seed(2024)
  mu = torch.randn(d, generator=gen)
  honest = mu[None, :] + torch.linspace(0.5, 1.5, n - nb)[:, None] * torch.randn(n - nb, d, generator=gen)
  byz = honest.mean(dim=0).mul(-1.1)
  return [honest[i] for i in range(n - nb)] + [byz] * nb

@pytest.mark.parametrize("gar,params", CASES)
def test_distance_rules_on_one_rank_match_the_oracle(gar, params):
  rows = _inputs()
  np_rows = [r.numpy() for r in rows]
  got, sel = sharded.aggregate(gar, rows, backend=OracleBackend(), return_selection=True, **params)
  ref = orc.GARS[gar](np_rows, **params)
  if gar == "bulyan":
    parity.assert_close_scaled(got.numpy(), ref, parity.column_scale(np.stack(np_rows)), "bulyan on one rank")
  else:
    parity.assert_bit_exact(got.numpy(), ref, f"{gar} on one rank")
  assert sel.numel() == (len(rows) - params["f"] if gar == "brute" else len(rows))

def test_unknown_aksel_mode_is_refused():
  with pytest.raises(NotImplementedError):
    sharded.aggregate("aksel", _inputs(), f=2, mode="bogus", backend=OracleBackend())

def test_unknown_rule_is_refused():
  with pytest.raises(KeyError):
    sharded.aggregate("nope", _inputs(), f=2, backend=OracleBackend())
