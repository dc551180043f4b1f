"""Kernel time of the time functions beside the paths they are compared with, on device-resident data.

Pairs (the two forms alternate, CUDA events on the context's stream, one warm-up call of each, median of --reps):
  hour      hour(<rate grid>): K19 (b2p_step_fn_dev, B2P_STEP_HOUR) over the config-2 grid, --series rows x 1000 steps,
            every cell valid, against K9 abs (b2p_instant_fn_dev) in place on the same grid.  K19 writes 8 B per cell
            and reads the validity words; abs reads and writes 8 B per cell.  The same pair over --series rows of one
            step (an instant query, T = 1, where a K19 warp spans 32 rows).
  timestamp the timestamp leaf (b2p_instant_timestamp_dev, K4's timestamp mode) against the plain instant leaf
            (b2p_instant_select_dev) on int64_bench.py's instant shape: --series series x 1000 samples every 15 s,
            1000 steps, 5 m lookback.  The timestamp leaf reads no value column.

Every line carries the card's name and power limit, read in the same run.

  python profiles/time_fn_bench.py [--series N] [--reps K]
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
B2P_STEP_HOUR, B2P_IFN_ABS = 2, 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_250_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("time_fn_bench needs a CUDA device")
    from greptimedb_b200 import Context

    S = args.series
    ctx = Context(0)
    ctx.use_torch_stream()
    L = ctx._L
    p = lambda t: C.c_void_p(t.data_ptr())
    dev = torch.device("cuda:0")
    ident = gpu_identity()
    Tw = (T + 31) // 32
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

    def pair(name, new, old, new_bytes, old_bytes, labels, steps=T):
        new(), old()  # warm-up
        tn, to = [], []
        for _ in range(args.reps):
            tn.append(timed(new))
            to.append(timed(old))
        mn, mo = float(np.median(tn)), float(np.median(to))
        print(json.dumps({"path": name, f"{labels[0]}_ms": round(mn, 4), f"{labels[1]}_ms": round(mo, 4),
                          "ratio": round(mn / mo, 3), f"{labels[0]}_tbs": round(new_bytes / mn / 1e9, 3),
                          f"{labels[1]}_tbs": round(old_bytes / mo / 1e9, 3), "series": S, "steps": steps, **ident}),
              flush=True)

    # hour(<grid>) vs abs(<grid>) over one [S x T] grid, every cell valid
    grid = torch.rand(S * T, dtype=torch.float64, device=dev)
    valid = torch.full((S * Tw,), -1, dtype=torch.int32, device=dev)
    eval_ts = start + torch.arange(T, dtype=torch.int64, device=dev) * SCRAPE
    pair("hour vs abs",
         lambda: L.b2p_step_fn_dev(ctx._h, B2P_STEP_HOUR, p(eval_ts), p(valid), S, T, p(grid)),
         lambda: L.b2p_instant_fn_dev(ctx._h, B2P_IFN_ABS, 0.0, 0.0, p(grid), p(valid), S, T, p(grid), p(valid)),
         S * T * 8 + S * Tw * 4, S * T * 16 + S * Tw * 4, ("hour", "abs"))
    del grid
    torch.cuda.empty_cache()
    # the instant shape, one step per row: hour(<instant vector>) over --series rows against abs on the same column
    col = torch.rand(S, dtype=torch.float64, device=dev)
    cvalid = torch.full((S,), 1, dtype=torch.int32, device=dev)
    pair("hour vs abs, T = 1",
         lambda: L.b2p_step_fn_dev(ctx._h, B2P_STEP_HOUR, p(eval_ts), p(cvalid), S, 1, p(col)),
         lambda: L.b2p_instant_fn_dev(ctx._h, B2P_IFN_ABS, 0.0, 0.0, p(col), p(cvalid), S, 1, p(col), p(cvalid)),
         S * 12, S * 20, ("hour", "abs"), steps=1)
    del col, cvalid

    # timestamp leaf vs instant leaf
    ts = (T0 + torch.arange(N, dtype=torch.int64, device=dev) * SCRAPE).repeat(S)
    offsets = torch.arange(S + 1, dtype=torch.int64, device=dev) * N
    vals = torch.rand(S * N, dtype=torch.float64, device=dev)
    out = torch.empty(S * T, dtype=torch.float64, device=dev)
    pair("timestamp leaf vs instant leaf",
         lambda: L.b2p_instant_timestamp_dev(ctx._h, start, end, SCRAPE, LOOKBACK, 0, p(ts), p(offsets), S * N, S,
                                             p(out), p(valid)),
         lambda: L.b2p_instant_select_dev(ctx._h, start, end, SCRAPE, LOOKBACK, 0, p(ts), p(vals), p(offsets), S * N, S,
                                          p(out), p(valid)),
         S * N * 8 + S * T * 8 + S * Tw * 4, S * N * 16 + S * T * 8 + S * Tw * 4, ("timestamp", "instant"))
    ctx.close()


if __name__ == "__main__":
    main()
