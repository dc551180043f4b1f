"""Kernel time of the Int64 (BIGINT) device paths beside their Float64 twins, on device-resident data.

Pairs (each the same shape, the same bytes moved; only the value type differs):
  selector  the instant selector over --series series x 1000 samples scraped every 15 s, evaluated on 1000 steps with
            a 5 m lookback (the config-2 shape): Float64 b2p_instant_select_dev (K4) vs Int64
            b2p_instant_select_fields_i64_dev with one field (K17 without the stale test);
  sum by    b2p_group_aggregate_dev vs b2p_group_aggregate_i64_dev, sum over that [series x 1000] grid into 100 000
            groups (the config-3 shape);
  topk      topk(5) by 1 000 groups over the grid, b2p_topk_dev vs b2p_topk_i64_dev (rows grouped once by an index);
  sort      sort over the first --sort-rows rows of the grid, b2p_sort_cells_dev vs b2p_sort_cells_i64_dev.

Each call is timed with CUDA events on the context's stream (the torch stream), after one warm-up call of both
forms, the two forms alternating, median of --reps.  Every line carries the card's name and power limit, read in the
same run.

  python profiles/int64_bench.py [--series N] [--sort-rows R] [--reps K]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from binary_bench import gpu_identity  # noqa: E402

N, T, SCRAPE, T0, LOOKBACK = 1000, 1000, 15_000, 1_700_000_000_000, 300_000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_250_000)
    ap.add_argument("--sort-rows", type=int, default=125_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("int64_bench needs a CUDA device")
    from greptimedb_b200 import Context

    S = args.series
    ctx = Context(0)
    ctx.use_torch_stream()
    L = ctx._L
    p = lambda t: C.c_void_p(t.data_ptr())
    dev = torch.device("cuda:0")
    ident = gpu_identity()

    ts = (T0 + torch.arange(N, dtype=torch.int64, device=dev) * SCRAPE).repeat(S)
    offsets = torch.arange(S + 1, dtype=torch.int64, device=dev) * N
    ivals = torch.randint(-1_000_000, 1_000_000, (S * N,), dtype=torch.int64, device=dev)
    fvals = ivals.to(torch.float64)
    Tw = (T + 31) // 32
    out = torch.empty(S * T, dtype=torch.float64, device=dev)
    valid = torch.empty(S * Tw, dtype=torch.int32, device=dev)
    start, end = T0, T0 + (T - 1) * SCRAPE

    def timed(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        rc = fn()
        b.record()
        torch.cuda.synchronize()
        if rc != 0:
            raise RuntimeError(L.b2p_last_error().decode())
        return a.elapsed_time(b)

    def pair(name, f64, i64, bytes_moved):
        f64(), i64()  # warm-up
        tf, ti = [], []
        for _ in range(args.reps):
            tf.append(timed(f64))
            ti.append(timed(i64))
        mf, mi = float(np.median(tf)), float(np.median(ti))
        print(json.dumps({"path": name, "float64_ms": round(mf, 4), "int64_ms": round(mi, 4),
                          "int64_over_float64": round(mi / mf, 3), "bytes": bytes_moved,
                          "float64_tbs": round(bytes_moved / mf / 1e9, 3), "int64_tbs": round(bytes_moved / mi / 1e9, 3),
                          "series": S, "steps": T, **ident}), flush=True)

    # selector: reads the timestamps and values once, writes the grid and its bitmap
    outs_arr = (C.c_void_p * 1)(C.c_void_p(out.data_ptr()))
    vals_arr = (C.c_void_p * 1)(C.c_void_p(ivals.data_ptr()))
    pair("selector",
         lambda: L.b2p_instant_select_dev(ctx._h, start, end, SCRAPE, LOOKBACK, 0, p(ts), p(fvals), p(offsets), S * N, S,
                                          p(out), p(valid)),
         lambda: L.b2p_instant_select_fields_i64_dev(ctx._h, start, end, SCRAPE, LOOKBACK, 0, p(ts),
                                                     C.cast(vals_arr, C.c_void_p), None, 1, p(offsets), S * N, S,
                                                     C.cast(outs_arr, C.c_void_p), p(valid)),
         S * N * 16 + S * T * 8 + S * Tw * 4)
    # the grid both forms fold: the selector's bitmap (every cell valid) over the Float64 / Int64 values
    fgrid, igrid = fvals.view(S, N)[:, :T].contiguous().view(-1), ivals.view(S, N)[:, :T].contiguous().view(-1)
    del ts, fvals, ivals, out
    G = 100_000
    gid = (torch.arange(S, device=dev, dtype=torch.int64) * 2654435761 % G).to(torch.int32)
    gsum = torch.empty(G * T, dtype=torch.float64, device=dev)
    gcnt = torch.empty(G * T, dtype=torch.int32, device=dev)
    pair("sum by",
         lambda: L.b2p_group_aggregate_dev(ctx._h, 0, p(fgrid), p(valid), p(gid), S, G, T, p(gsum), p(gcnt)),
         lambda: L.b2p_group_aggregate_i64_dev(ctx._h, 0, p(igrid), p(valid), p(gid), S, G, T, p(gsum), p(gcnt)),
         S * T * 8 + S * Tw * 4 + G * T * 12)
    del gsum, gcnt
    G2 = 1000
    gid2 = (torch.arange(S, device=dev, dtype=torch.int32) % G2).contiguous()
    ix = ctx.group_index_create_dev(gid2, S, G2)
    tie = torch.arange(S, dtype=torch.int32, device=dev)
    kept = torch.empty_like(valid)
    pair("topk(5) by",
         lambda: L.b2p_topk_dev(ctx._h, 0, 5.0, p(fgrid), p(valid), ix, p(tie), T, p(kept)),
         lambda: L.b2p_topk_i64_dev(ctx._h, 0, 5.0, p(igrid), p(valid), ix, p(tie), T, p(kept)),
         S * T * 8 + 2 * S * Tw * 4 + S * 4)
    ctx.group_index_destroy(ix)
    R = min(args.sort_rows, S)
    cells = torch.empty(R * T, dtype=torch.int64, device=dev)
    n = torch.empty(1, dtype=torch.int64, device=dev)
    nv = R * T
    pair("sort",
         lambda: L.b2p_sort_cells_dev(ctx._h, 0, p(fgrid), p(valid), R, T, p(cells), p(n)),
         lambda: L.b2p_sort_cells_i64_dev(ctx._h, 0, p(igrid), p(valid), R, T, p(cells), p(n)),
         nv * 8 * 32 + R * T * 8 + 2 * R * Tw * 4 + nv * 16)
    ctx.close()


if __name__ == "__main__":
    main()
