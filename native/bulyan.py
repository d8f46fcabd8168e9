# coding: utf-8
"""native.bulyan — Bulyan over Multi-Krum on the GPU (binds aggregators/bulyan.py:86-100)."""

def aggregate(gradients, f, m=None):
  from byzantinemomentum_b200 import engine
  return engine.bulyan(gradients, f, engine._rule("bulyan", len(gradients), f, m).m)[0]
