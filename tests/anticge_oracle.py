# coding: utf-8
"""Restatement of the reference's attack against CGE (attacks/anticge.py:49-78) in NumPy, built on the oracle's
norms (`oracle.byzoracle.cge_order`: the fp32 rounding of fp64 sums of squares, as the kernels form them).
TEST INFRASTRUCTURE ONLY: the GPU tests (`tests/test_cuda_anticge.py`) cannot read the reference, so they
compare against this; `tests/test_anticge_abi.py` pins it against the reference's recorded outputs
(`tests/golden/anticge/`)."""

import math

import numpy as np

from oracle import byzoracle as orc

F32 = np.float32

def anticge(grad_honests, f_decl, f_real, return_info=False):
  """ attacks/anticge.py:49-78 for 0 <= maxpos = nh - f_decl < nh — a row of NaN f_real times when f_real > f_decl;
  else the rows ranked by `cge_order`, attack = σ0 + σ0 + σ1 + ... + σ(maxpos-1) in fp32 in that order, scaled by
  fl32(-maxnorm / attnorm) when attnorm = ||attack|| > 0, maxnorm = nextafter(norm of σ_maxpos, 0) in double.
  Returns the row f_real times (the same array); info: order, norms, maxnorm, the unscaled sum, attnorm. """
  g = orc.as_matrix(grad_honests)
  nh, d = g.shape
  if f_real > f_decl:
    row = np.full(d, np.nan, dtype=F32)
    return ([row] * f_real, dict(fill=True)) if return_info else [row] * f_real
  maxpos = nh - f_decl
  assert 0 <= maxpos < nh, "outside the device's range the reference indexes from the end or raises"
  order, nrm = orc.cge_order(g)
  maxnorm = math.nextafter(nrm[order[maxpos]], 0.)
  attack = g[order[0]].copy()
  with np.errstate(all="ignore"):
    for i in order[:maxpos]:
      attack = (attack + g[i]).astype(F32)
    presum = attack.copy()
    attnorm = float(orc.fp32_norm(orc.sum_squares(attack)))
    if attnorm > 0:
      attack = (attack * F32(-maxnorm / attnorm)).astype(F32)
  out = [attack] * f_real
  if return_info:
    return out, dict(fill=False, order=order, norms=nrm, maxnorm=maxnorm, presum=presum, attnorm=attnorm)
  return out
