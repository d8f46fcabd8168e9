# coding: utf-8
"""native.krum — Multi-Krum on the GPU (binds aggregators/krum.py:82-96)."""

def aggregate(gradients, f, m=None):
  from byzantinemomentum_b200 import engine
  return engine.krum(gradients, f, engine._rule("krum", len(gradients), f, m).m)[0]
