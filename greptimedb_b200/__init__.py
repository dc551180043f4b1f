"""greptimedb_b200 — H100-native evaluator for GreptimeDB's PromQL range-query hot path.

The product is libb200promql.so (hand-written CUDA for sm_90a behind the C ABI of
include/b200promql.h); this package is the thin Python handle used by tests and bench.py.
Importing the package does not load the library; `engine.Context()` does, and fails loudly if the
library or a CUDA device is missing (there is no CPU fallback).
"""
from .engine import AGG_IDS, FN_IDS, B2PError, Context, make_params, num_steps, pack_ranges, valid_to_bool  # noqa: F401

__all__ = ["Context", "B2PError", "FN_IDS", "AGG_IDS", "make_params", "num_steps", "pack_ranges", "valid_to_bool"]
