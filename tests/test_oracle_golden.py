# coding: utf-8
"""Pin the NumPy oracle (`oracle/byzoracle.py`) against outputs of the reference itself
(`tests/golden/*.npz`, produced by `tests/golden/make_golden.py` from the reference).
CPU-only; part of the `-m "not gpu"` suite."""

import math

import numpy as np
import pytest

from conftest import golden_calls, canon_alias
import parity
from oracle import byzoracle as orc

def _rows(g):
  return [g.rows[i] for i in range(g.n)]

@pytest.mark.parametrize("g,call", golden_calls())
def test_oracle_matches_reference(g, call):
  gar, params, tag = call["gar"], call["params"], call["tag"]
  rows = _rows(g)
  ref_out = g.get(tag, "out")
  if "raises" in call:
    # The reference itself raised on this input (non-finite rows in brute, degenerate bulyan, ...)
    with pytest.raises(Exception):
      orc.GARS[gar](rows, **params)
    return
  fn = orc.GARS[gar]
  if gar in ("average", "median"):
    parity.assert_bit_exact(fn(rows), ref_out, tag)
  elif gar == "trmean":
    parity.assert_trmean(fn(rows, **params), ref_out, g.rows, tag)
  elif gar in ("phocas", "meamed"):
    f = params["f"]
    center = orc.trmean(rows, f) if gar == "phocas" else orc.median(rows)
    amb = parity.closest_ambiguous(g.rows, g.n - f, center)
    got = fn(rows, **params)
    parity.assert_close_scaled(got, ref_out, parity.column_scale(g.rows), tag, exempt=amb)
    parity.assert_in_hull(got, g.rows, amb, tag)
  elif gar == "krum":
    got, info = fn(rows, return_info=True, **params)
    ref_order = g.get(tag, "order")
    m = params.get("m") or (g.n - params["f"] - 2)
    nan_rows = np.isnan(g.rows).any(axis=1)
    # Rows made of NaN have all-inf scores and tie among themselves: compare canonically
    assert canon_alias(info["order"][:m], g.nh) == canon_alias(ref_order[:m], g.nh), f"{tag}: selection differs (margin {info['margin']:.3g})"
    parity.assert_bit_exact(got, ref_out, tag)
    ref_scores = g.get(tag, "scores")
    ours = np.array(sorted(info["scores"]))
    fin = np.isfinite(ref_scores)
    assert np.array_equal(fin, np.isfinite(ours))
    np.testing.assert_allclose(ours[fin], ref_scores[fin], rtol=2e-6)
    del nan_rows
  elif gar == "bulyan":
    got, info = fn(rows, return_info=True, **params)
    scale = parity.column_scale(info["stage1"])
    parity.assert_close_scaled(got, ref_out, scale, tag, exempt=info["ambiguous"])
    parity.assert_in_hull(got, info["stage1"], info["ambiguous"], tag)
  elif gar == "brute":
    got, info = fn(rows, return_info=True, **params)
    assert canon_alias(info["selection"], g.nh) == canon_alias(g.get(tag, "selection"), g.nh), f"{tag}: selection differs (margin {info['margin']:.3g})"
    parity.assert_bit_exact(got, ref_out, tag)
  elif gar == "aksel":
    got, info = fn(rows, return_info=True, **params)
    c = call["c"]
    ref_order = g.get(tag, "order")
    if not np.isnan(g.get(tag, "dists")).any():   # NaN keys: order undefined in the reference
      assert canon_alias(info["order"][:c], g.nh) == canon_alias(ref_order[:c], g.nh), f"{tag}: selection differs (margin {info['margin']:.3g})"
      parity.assert_bit_exact(got, ref_out, tag)
  elif gar == "cge":
    got, info = fn(rows, return_info=True, **params)
    m = g.n - params["f"]
    assert canon_alias(info["order"][:m], g.nh) == canon_alias(g.get(tag, "order")[:m], g.nh), f"{tag}: selection differs (margin {info['margin']:.3g})"
    parity.assert_bit_exact(got, ref_out, tag)
  else:
    raise AssertionError(gar)
  # Influence (ratio of accepted Byzantine rows)
  if "influence" in call and not ("raises" in call):
    if gar == "aksel" and np.isnan(g.get(tag, "dists")).any():
      return
    got = orc.influence(gar, rows[:g.nh], rows[g.nh:], **params)
    assert math.isclose(got, call["influence"], rel_tol=0, abs_tol=1e-12), f"{tag}: influence {got} vs {call['influence']}"

def test_known_answers_appendix_b():
  """ SURVEY.md Appendix B: hand-checkable n=7, d=4 vectors (printed reference outputs). """
  rows = [[1.0, 2.0, -1.0, 0.5], [1.5, 1.0, -2.0, 0.0], [0.5, 3.0, -1.5, 1.0], [2.0, 2.5, -0.5, -0.5],
          [1.2, 1.8, -1.1, 0.4], [9.0, -9.0, 9.0, -9.0], [9.0, -9.0, 9.0, -9.0]]
  f32 = lambda xs: np.array(xs, dtype=np.float32)
  assert np.array_equal(orc.average(rows), f32([3.4571430683135986, -1.100000023841858, 1.6999999284744263, -2.3714287281036377]))
  assert np.array_equal(orc.median(rows), f32([1.5, 1.7999999523162842, -1.0, 0.0]))
  assert np.array_equal(orc.trmean(rows, 2), f32([1.566666603088379, 1.600000023841858, -0.8666666150093079, -0.03333333134651184]))
  common = f32([1.2400000095367432, 2.059999942779541, -1.2200000286102295, 0.2800000011920929])
  for name in ("phocas", "meamed", "brute", "cge"):
    assert np.array_equal(orc.GARS[name](rows, f=2), common), name
  assert np.array_equal(orc.aksel(rows, 2, mode="n-f"), common)
  assert np.array_equal(orc.krum(rows, 2), f32([1.2333333492279053, 1.600000023841858, -1.3666666746139526, 0.29999998211860657]))
  assert np.array_equal(orc.aksel(rows, 2), f32([1.4249999523162842, 1.8250000476837158, -1.149999976158142, 0.09999999403953552]))
  assert np.array_equal(orc.bulyan(rows, 1), f32([1.5, 1.8250000476837158, -1.1666666269302368, 0.0]))
  for name in ("krum", "brute", "aksel", "cge"):
    assert orc.influence(name, rows[:5], rows[5:], f=2) == 0.0
  assert orc.influence("average", rows[:5], rows[5:]) == 2 / 7
