# coding: utf-8
"""byzantinemomentum_b200 — H100-native (sm_90a) Byzantine-robust gradient aggregation.

A drop-in for the aggregation hot path of LPD-EPFL/ByzantineMomentum (`aggregators/*.py` as
called from `attack.py:821-822`): same plugin interface, hand-written CUDA underneath.

    from byzantinemomentum_b200 import gars
    aggregated = gars["krum"](gradients=list_of_flat_fp32_cuda_tensors, f=5)

    plan = byzantinemomentum_b200.Plan("krum", gradients, f=5)   # prepared call: plan() is one C call, no sync

    import aggregators                              # the unmodified reference
    byzantinemomentum_b200.plugin.install(aggregators)   # registers "b200-<name>" rules

Importing this package never touches CUDA; the compiled library is loaded on first use and
its absence is an error (no CPU fallback).
"""

from . import _lib, engine, gars as _gars, hostmem, plugin, sharded
from .gars import gars, make_gar, register, UserException, last_selection
from .engine import config, Plan, compute_avg_dev_max, GradientStack

__all__ = ["gars", "make_gar", "register", "UserException", "last_selection", "config", "Plan", "GradientStack", "compute_avg_dev_max", "engine", "hostmem", "plugin", "sharded"]
__version__ = "0.1.0"
