"""Times the plan layer over a multi-field table and the multi-key sort.

  1. avg_over_time over a config-5-shaped table (32 Float64 field columns; --series series x --samples rows, 2 M rows
     by default, as config 5's 2 M rows x 32 columns) on --steps steps: one PromRangeExec over all 32 fields against 32
     single-field PromRangeExec nodes, one per field.  Host time of push + execute (each plan call is synchronous), the
     median of --reps after one warm-up.  Both read the same batch; the outputs are compared field by field.
  2. b2p_sort_cells_fields_dev (sort and sort_desc) on device-resident grids of --sort-rows x --sort-steps cells, about
     90 % valid, at F = 1, 2 and 8 fields: CUDA events around the call, the median of --reps after one warm-up.

Every line carries the card's name and power limit, read in the same run.  There is no target.

  python profiles/multifield_plan_bench.py [--series N] [--samples M] [--steps T] [--sort-rows R] [--sort-steps T] [--reps K]
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

from binary_bench import gpu_identity  # noqa: E402

T0, SCRAPE, F_TABLE = 1_700_000_000_000, 15_000, 32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=2000)
    ap.add_argument("--samples", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=250)
    ap.add_argument("--sort-rows", type=int, default=100_000)
    ap.add_argument("--sort-steps", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import pyarrow as pa
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("multifield_plan_bench needs a CUDA device")
    from greptimedb_b200 import Context
    from greptimedb_b200.plan import PromRangeExec

    ctx = Context(0)
    ident = gpu_identity()

    def report(**kw):
        print(json.dumps({**kw, **ident}), flush=True)

    def median_ms(fn):
        ms = []
        for i in range(args.reps + 1):
            t = time.perf_counter()
            out = fn()
            if i:
                ms.append((time.perf_counter() - t) * 1e3)
        return float(np.median(ms)), out

    # ---- 1. one node over 32 fields against 32 one-field nodes ------------------------------------------------------
    S, N = args.series, args.samples
    rng = np.random.default_rng(5)
    ts = (T0 + np.tile(np.arange(N) * SCRAPE, S)).astype(np.int64)
    fields = [f"f{f}" for f in range(F_TABLE)]
    cols = [pa.array(ts, pa.timestamp("ms"))] + [pa.array(rng.normal(0, 10, S * N)) for _ in fields]
    cols.append(pa.array(np.repeat([f"s{s:06d}" for s in range(S)], N)))
    batch = pa.record_batch(cols, names=["ts"] + fields + ["host"])
    end = T0 + (N - 1) * SCRAPE
    itv = max(1, (end - T0) // max(1, args.steps - 1))

    def node(names):
        ex = PromRangeExec(ctx, "prom_avg_over_time", T0, T0 + (args.steps - 1) * itv, itv, 300_000, "ts", names,
                           ["host"])
        ex.push(batch)
        return ex.execute()

    one_ms, multi = median_ms(lambda: node(fields))
    each_ms, singles = median_ms(lambda: [node([f]) for f in fields])
    for f, s in enumerate(singles):
        a = multi.column(1 + f).to_numpy()
        b = s.column(1).to_numpy()
        assert a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64)), f"field {f} differs"
    report(bench="multifield_plan", shape=f"{S}x{N} rows x {F_TABLE} fields, {args.steps} steps",
           one_node_ms=round(one_ms, 2), per_field_nodes_ms=round(each_ms, 2), rows_out=multi.num_rows)

    # ---- 2. the multi-key sort --------------------------------------------------------------------------------------
    R, T = args.sort_rows, args.sort_steps
    Tw = (T + 31) // 32
    ok = torch.rand(R, Tw * 32, device="cuda") < 0.9
    ok[:, T:] = False
    weights = (2 ** torch.arange(32, device="cuda", dtype=torch.int64)).view(1, 1, 32)
    valid = (ok.view(R, Tw, 32).to(torch.int64) * weights).sum(-1).to(torch.uint32).view(torch.int32).contiguous()
    grids = [torch.randint(0, 4, (R, T), device="cuda").to(torch.float64) for _ in range(8)]
    cells = torch.empty(R * T, dtype=torch.int64, device="cuda")
    n = torch.zeros(1, dtype=torch.int64, device="cuda")
    for F in (1, 2, 8):
        for desc in (False, True):
            ms = []
            for i in range(args.reps + 1):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                ctx.sort_cells_fields_dev(desc, grids[:F], valid, R, T, cells, n)
                b.record()
                torch.cuda.synchronize()
                if i:
                    ms.append(a.elapsed_time(b))
            report(bench="sort_cells_fields", fields=F, desc=desc, rows=R, steps=T, valid_cells=int(n.item()),
                   median_ms=round(float(np.median(ms)), 3))
    ctx.close()


if __name__ == "__main__":
    main()
