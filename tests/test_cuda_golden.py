# coding: utf-8
"""GPU parity, part 1: the CUDA rules against the reference's recorded outputs
(`tests/golden/*.npz`) and against the NumPy oracle on the same inputs.
Calls go through the reference-facing plugin interface (`gars[name](gradients=..., f=...)`),
which is a thin shell over the C ABI."""

import numpy as np
import pytest

from conftest import golden_calls, canon_alias
import closest_columns as cc
import parity
from oracle import byzoracle as orc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

def _device_rows(g):
  """ Honest rows as separate CUDA tensors; the Byzantine rows are ONE tensor repeated. """
  dev = torch.device("cuda", 0)
  honests = [torch.from_numpy(g.rows[i].copy()).to(dev) for i in range(g.nh)]
  attacks = []
  if g.nb:
    byz = torch.from_numpy(g.rows[g.nh].copy()).to(dev)
    attacks = [byz] * g.nb
  return honests, attacks

@pytest.mark.parametrize("g,call", golden_calls())
def test_cuda_matches_reference(g, call):
  import byzantinemomentum_b200 as bz
  gar, params, tag = call["gar"], dict(call["params"]), call["tag"]
  honests, attacks = _device_rows(g)
  rows = honests + attacks
  rule = bz.gars[gar]
  assert rule.check(gradients=rows, **params) is None
  if "raises" in call:
    # brute with no finite subset -> AssertionError (brute.py:67); bulyan degenerate -> TypeError (bulyan.py:70)
    expected = {"AssertionError": AssertionError, "TypeError": TypeError}[call["raises"]]
    with pytest.raises(expected):
      rule.unchecked(gradients=rows, model=None, **params)
    return
  out = rule.unchecked(gradients=rows, model=None, **params)
  assert out.device == rows[0].device and out.dtype == torch.float32 and out.shape == rows[0].shape
  assert all(out.data_ptr() != r.data_ptr() for r in rows)
  got = out.cpu().numpy()
  ref_out = g.get(tag, "out")
  np_rows = [g.rows[i] for i in range(g.n)]
  if gar in ("average", "median"):
    parity.assert_bit_exact(got, ref_out, tag)
  elif gar == "trmean":
    parity.assert_trmean(got, ref_out, g.rows, tag)
    # and bit-exact against the oracle everywhere (same summation order, no ATen tail effect)
    parity.assert_bit_exact(got, orc.trmean(np_rows, **params), tag + " [oracle]")
  elif gar in ("phocas", "meamed"):
    f = params["f"]
    center = orc.trmean(np_rows, f) if gar == "phocas" else orc.median(np_rows)
    amb = parity.closest_ambiguous(g.rows, g.n - f, center)
    parity.assert_close_scaled(got, ref_out, parity.column_scale(g.rows), tag, exempt=amb)
    parity.assert_bit_exact(got, cc.k1_closest(g.rows, f, gar, center)[0], tag + " [K1's closest epilogue]")
  elif gar == "krum":
    m = params.get("m") or (g.n - params["f"] - 2)
    sel = bz.last_selection()
    assert canon_alias(sel[:m], g.nh) == canon_alias(g.get(tag, "order")[:m], g.nh), f"{tag}: selection differs"
    parity.assert_bit_exact(got, ref_out, tag)
  elif gar == "bulyan":
    _, info = orc.bulyan(np_rows, return_info=True, **params)
    scale = parity.column_scale(info["stage1"])
    parity.assert_close_scaled(got, ref_out, scale, tag, exempt=info["ambiguous"])
    parity.assert_in_hull(got, info["stage1"], info["ambiguous"], tag)
  elif gar == "brute":
    assert canon_alias(bz.last_selection(), g.nh) == canon_alias(g.get(tag, "selection"), g.nh), f"{tag}: selection differs"
    parity.assert_bit_exact(got, ref_out, tag)
  elif gar == "aksel":
    if np.isnan(g.get(tag, "dists")).any():
      return  # order undefined in the reference
    c = call["c"]
    assert canon_alias(bz.last_selection()[:c], g.nh) == canon_alias(g.get(tag, "order")[:c], g.nh), f"{tag}: selection differs"
    parity.assert_bit_exact(got, ref_out, tag)
  elif gar == "cge":
    m = g.n - params["f"]
    if m >= 1:
      assert canon_alias(bz.last_selection()[:m], g.nh) == canon_alias(g.get(tag, "order")[:m], g.nh), f"{tag}: selection differs"
    parity.assert_bit_exact(got, ref_out, tag)
  else:
    raise AssertionError(gar)
  if "influence" in call and rule.influence is not None and g.nb > 0:
    if gar == "aksel" and np.isnan(g.get(tag, "dists")).any():
      return
    ratio = rule.influence(honests, attacks, **params)
    assert abs(ratio - call["influence"]) < 1e-12, f"{tag}: influence {ratio} vs {call['influence']}"
