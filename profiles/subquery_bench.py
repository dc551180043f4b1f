"""Times subqueries (K13 + the range tiers, b2p_subquery_dev) over the config-2 child grid: rate(x[5m]) of --series
synthetic series (default 1.25 M) x 1000 samples at a 15 s scrape, evaluated on 1000 steps (a device-resident
[series x 1000] grid, computed first), then

  a. max_over_time(<grid>[1h:1m]): the grid read as a 1 min inner grid, outer interval 1 min (941 outer steps)
  b. rate(<grid>[5m:15s]): the grid's own 15 s steps, outer interval 15 s (981 outer steps); every row whose cells are
     all valid is exactly regular at the outer interval, which the uniform-cadence first tier takes when the cadence
     probe says so

For each it prints one JSON line: the time of the call (host clock around the call and b2p_sync, median of --reps after
two warm-up calls: a grid of more than one scratch batch waits between batches), the bytes the call needs at least
(the child grid once, 8 B + 1 bit per cell, and the output once, 8 B + 1 bit per cell), that rate, the series the first
tier handed on in the last batch (b2p_last_warp_tier_series; 0 = the first tier took every series of the batch), and
the card's name and power limit read in the same run.

  python profiles/subquery_bench.py [--series N] [--reps R]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from binary_bench import PEAK_TBS, gpu_identity  # noqa: E402

N, T_IN, SCRAPE, T0 = 1000, 1000, 15_000, 1_700_000_000_000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_250_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch

    from greptimedb_b200 import Context, make_params, num_steps

    dev = torch.device("cuda:0")
    ctx = Context(0)
    ctx.use_torch_stream()
    ident = gpu_identity()
    S = args.series
    Tw_in = (T_IN + 31) // 32
    # the child grid: rate(x[5m]) over synthetic counters, in chunks of series
    grid = torch.empty(S * T_IN, dtype=torch.float64, device=dev)
    gvalid = torch.empty(S * Tw_in, dtype=torch.int32, device=dev)
    p_rate = make_params("rate", T0, T0 + (T_IN - 1) * SCRAPE, SCRAPE, 300_000)
    chunk = 250_000
    ts = torch.empty(chunk * N, dtype=torch.int64, device=dev)
    val = torch.empty(chunk * N, dtype=torch.float64, device=dev)
    sid = torch.empty(chunk * N, dtype=torch.int32, device=dev)
    offsets = torch.empty(chunk + 1, dtype=torch.int64, device=dev)
    for s0 in range(0, S, chunk):
        n = min(chunk, S - s0)
        ctx.synth_fill_dev(s0, n, N, T0, SCRAPE, 1000, 1, 0x5EED, ts, val, sid)
        ctx.series_offsets_dev(sid, n * N, n, offsets)
        ctx.range_eval_dev(p_rate, ts, val, offsets, n * N, n, grid[s0 * T_IN:], gvalid[s0 * Tw_in:])
        ctx.sync()
    del ts, val, sid, offsets
    torch.cuda.empty_cache()
    in_bytes = S * T_IN * 8 + S * T_IN // 8

    def out_bytes(T):
        return S * T * 8 + S * T // 8

    def report(query, T, ms, handed):
        b = in_bytes + out_bytes(T)
        print(json.dumps({"query": query, "series": S, "inner_steps": T_IN, "outer_steps": T, "call_ms": round(ms, 3),
                          "bytes": b, "tb_per_s": round(b / ms / 1e9, 3),
                          "fraction_of_3.35_tb_s": round(b / ms / 1e9 / PEAK_TBS, 3),
                          "first_tier_handed_on_last_batch": handed, **ident}), flush=True)

    def timed(call):
        ms = []
        for i in range(args.reps + 2):
            torch.cuda.synchronize()
            t = time.perf_counter()
            call()
            ctx.sync()
            torch.cuda.synchronize()
            if i >= 2:
                ms.append((time.perf_counter() - t) * 1e3)
        return float(np.median(ms))

    # a. max_over_time(<grid>[1h:1m])
    step_a, rng_a = 60_000, 3_600_000
    start_a = T0 + rng_a - step_a  # (the grid read as start' = T0 every 1 min)
    end_a = T0 + (T_IN - 1) * step_a
    pa_ = make_params("max_over_time", start_a, end_a, step_a, rng_a, filter_nan=False)
    T_a = num_steps(start_a, end_a, step_a)
    # b. rate(<grid>[5m:15s])
    rng_b = 300_000
    start_b = T0 + rng_b - SCRAPE
    end_b = T0 + (T_IN - 1) * SCRAPE
    pb = make_params("rate", start_b, end_b, SCRAPE, rng_b, filter_nan=False)
    T_b = num_steps(start_b, end_b, SCRAPE)
    out = torch.empty(S * max(T_a, T_b), dtype=torch.float64, device=dev)
    ov = torch.empty(S * ((max(T_a, T_b) + 31) // 32), dtype=torch.int32, device=dev)

    ms = timed(lambda: ctx.subquery_dev(pa_, T0, step_a, grid, gvalid, S, T_IN, out, ov))
    report("a. max_over_time(rate(x[5m])[1h:1m])", T_a, ms, ctx.last_warp_tier_series())
    ms = timed(lambda: ctx.subquery_dev(pb, T0, SCRAPE, grid, gvalid, S, T_IN, out, ov))
    report("b. rate(rate(x[5m])[5m:15s])", T_b, ms, ctx.last_warp_tier_series())

    ctx.close()


if __name__ == "__main__":
    main()
