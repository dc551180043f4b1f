#!/usr/bin/env python
"""Throughput of every range function on the BASELINE config-2 shape (device-resident inputs, K0 + K2 per pass).
usage (on an H100): python profiles/function_sweep.py [series]  -> markdown table on stdout"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from greptimedb_b200 import FN_IDS, Context, make_params  # noqa: E402

S = int(sys.argv[1]) if len(sys.argv) > 1 else 400_000
N, T0 = 1000, 1_700_000_000_000
dev = torch.device("cuda:0")
ctx = Context(0)
ctx.use_torch_stream()
ts = torch.empty(S * N, dtype=torch.int64, device=dev)
val = torch.empty(S * N, dtype=torch.float64, device=dev)
sid = torch.empty(S * N, dtype=torch.int32, device=dev)
off = torch.empty(S + 1, dtype=torch.int64, device=dev)
out = torch.empty(S * N, dtype=torch.float64, device=dev)
valid = torch.empty(S * 32, dtype=torch.int32, device=dev)
ctx.synth_fill_dev(0, S, N, T0, 15_000, 1000, 1, 0x5EED, ts, val, sid)
ctx.series_offsets_dev(sid, S * N, S, off)
ctx.sync()
params = {"predict_linear": (600.0, 0.0), "quantile_over_time": (0.9, 0.0), "holt_winters": (0.3, 0.1)}
print(f"| function | ms / pass ({S} series x {N} samples, reset-variant data) | G samples/s | slow-path series |")
print("|---|---|---|---|")
for fn in FN_IDS:
    p0, p1 = params.get(fn, (0.0, 0.0))
    p = make_params(fn, T0, T0 + 999 * 15_000, 15_000, 300_000, param0=p0, param1=p1)
    for _ in range(2):
        ctx.range_eval_dev(p, ts, val, off, S * N, S, out, valid)
    ctx.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        ctx.range_eval_dev(p, ts, val, off, S * N, S, out, valid)
    e1.record()
    ctx.sync()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 3
    print(f"| {fn} | {ms:.2f} | {S * N / ms / 1e6:.1f} | {ctx.last_slow_series()} |")
