"""Times sort / sort_desc: K14 alone (b2p_sort_cells_dev) on device-resident grids, and end to end through SortPlan.

Shapes:
  1. the config-2 rate grid: rate(x[5m]) of --series synthetic counters (default 1.25 M) x 1000 samples at a 15 s scrape,
     evaluated on 1000 steps (nearly every cell valid);
  2. a grid of the same size with standard-normal values and about 50 % of the cells valid (random bits).

K14 alone: CUDA events around b2p_sort_cells_dev (count, scan, the read-back of the cell count, scatter, CUB's radix
sort), median of --reps after one warm-up, for sort and sort_desc.  The bytes it needs at least: every valid cell costs
8 radix passes x (16 B read + 16 B written) of (key, cell index), plus the compaction (the grid's values and its bitmap
read once, the bitmap a second time by the count, 16 B written per valid cell).  It prints that byte count, the achieved
rate and its fraction of the H100 SXM data-sheet 3.35 TB/s.

End to end: SortPlan over a leaf of --e2e-series series x 1000 steps (default 50 k; a plan node's result lives in host
memory), a __tsid-keyed range leaf of rate over counters for shape 1 and an instant leaf over standard-normal samples of
which about half are missing for shape 2: the host time of execute() of the sort node and of its child alone (median of
--reps after one warm-up; each plan call is synchronous).

Every line carries the card's name and power limit, read in the same run.

  python profiles/sort_bench.py [--series N] [--e2e-series M] [--reps R]
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

N, T, SCRAPE, T0, RANGE = 1000, 1000, 15_000, 1_700_000_000_000, 300_000


def k14_bytes(n_valid: int, rows: int, T: int) -> int:
    Tw = (T + 31) // 32
    return n_valid * 8 * 32 + rows * T * 8 + 2 * rows * Tw * 4 + n_valid * 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_250_000)
    ap.add_argument("--e2e-series", type=int, default=50_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import pyarrow as pa
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("sort_bench needs a CUDA device")
    from greptimedb_b200 import Context, make_params
    from greptimedb_b200.plan import PromRangeExec, SortPlan

    dev = torch.device("cuda:0")
    ctx = Context(0)
    ctx.use_torch_stream()
    ident = gpu_identity()
    S, Tw = args.series, (T + 31) // 32

    def report(**kw):
        print(json.dumps({**kw, **ident}), flush=True)

    def k14(shape, grid, gvalid):
        cells = torch.empty(S * T, dtype=torch.int64, device=dev)
        n = torch.zeros(1, dtype=torch.int64, device=dev)
        for desc in (False, True):
            ms = []
            for i in range(args.reps + 1):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                ctx.sort_cells_dev(desc, grid, gvalid, S, T, cells, n)
                b.record()
                torch.cuda.synchronize()
                if i:
                    ms.append(a.elapsed_time(b))
            nv = int(n.item())
            m = float(np.median(ms))
            byt = k14_bytes(nv, S, T)
            report(shape=shape, function="sort_desc" if desc else "sort", stage="k14", rows=S, steps=T, valid_cells=nv,
                   k14_ms=round(m, 3), k14_ms_min=round(min(ms), 3), k14_ms_max=round(max(ms), 3), bytes=byt,
                   tb_per_s=round(byt / m / 1e9, 3), **{"fraction_of_3.35_tb_s": round(byt / m / 1e9 / PEAK_TBS, 3)})
        del cells

    # shape 1: the config-2 rate grid
    grid = torch.empty(S * T, dtype=torch.float64, device=dev)
    gvalid = torch.empty(S * Tw, dtype=torch.int32, device=dev)
    p_rate = make_params("rate", T0, T0 + (T - 1) * SCRAPE, SCRAPE, RANGE)
    chunk = 250_000
    ts = torch.empty(chunk * N, dtype=torch.int64, device=dev)
    val = torch.empty(chunk * N, dtype=torch.float64, device=dev)
    sid = torch.empty(chunk * N, dtype=torch.int32, device=dev)
    offsets = torch.empty(chunk + 1, dtype=torch.int64, device=dev)
    for s0 in range(0, S, chunk):
        n = min(chunk, S - s0)
        ctx.synth_fill_dev(s0, n, N, T0, SCRAPE, 1000, 1, 0x5EED, ts, val, sid)
        ctx.series_offsets_dev(sid, n * N, n, offsets)
        ctx.range_eval_dev(p_rate, ts, val, offsets, n * N, n, grid[s0 * T:], gvalid[s0 * Tw:])
        ctx.sync()
    del ts, val, sid, offsets
    torch.cuda.empty_cache()
    k14("1. config-2 rate grid", grid, gvalid)
    # shape 2: random values, about half of the cells valid
    gen = torch.Generator(device=dev)
    gen.manual_seed(0x5EED)
    grid.normal_(generator=gen)
    gvalid.random_(generator=gen)  # (random 32-bit patterns over the int32 range's non-negative half ...)
    gvalid ^= torch.randint(0, 2, gvalid.shape, dtype=torch.int32, device=dev, generator=gen) << 31  # (... and the sign bit)
    k14("2. random values, 50 % valid", grid, gvalid)
    del grid, gvalid
    torch.cuda.empty_cache()

    # end to end through SortPlan
    E = args.e2e_series
    rng = np.random.default_rng(7)

    def timed(call):
        ms = []
        for i in range(args.reps + 1):
            t = time.perf_counter()
            out = call()
            if i:
                ms.append((time.perf_counter() - t) * 1e3)
        return float(np.median(ms)), out

    n1 = N + RANGE // SCRAPE
    ids = np.repeat(np.arange(E, dtype=np.uint64), n1)
    counters = np.cumsum(rng.random((E, n1)) * 10, axis=1).reshape(-1)
    b1 = pa.record_batch([pa.array(np.tile(T0 - RANGE + np.arange(n1, dtype=np.int64) * SCRAPE, E), pa.timestamp("ms")),
                          pa.array(counters), pa.array(ids, pa.uint64())], names=["ts", "val", "__tsid"])
    keep = rng.random(E * T) < 0.5
    b2 = pa.record_batch([pa.array(np.tile(T0 + np.arange(T, dtype=np.int64) * SCRAPE, E)[keep], pa.timestamp("ms")),
                          pa.array(rng.standard_normal(E * T)[keep]),
                          pa.array(np.repeat(np.arange(E, dtype=np.uint64), T)[keep], pa.uint64())],
                         names=["ts", "val", "__tsid"])
    del ids, counters, keep

    def leaf1():
        x = PromRangeExec(ctx, "prom_rate", T0, T0 + (T - 1) * SCRAPE, SCRAPE, RANGE, "ts", "val", ["__tsid"])
        x.push(b1)
        return x

    def leaf2():
        x = PromRangeExec(ctx, "", T0, T0 + (T - 1) * SCRAPE, SCRAPE, 0, "ts", "val", ["__tsid"], lookback_delta=1000)
        x.push(b2)
        return x

    for shape, leaf in (("1. rate grid (e2e)", leaf1), ("2. random values, 50 % valid (e2e)", leaf2)):
        child = leaf()
        child_ms, c_out = timed(child.execute)
        for function in ("sort", "sort_desc"):
            node = SortPlan(ctx, function, leaf())
            node_ms, out = timed(node.execute)
            assert out.num_rows == c_out.num_rows
            report(shape=shape, function=function, stage="end to end", rows=E, steps=T, exported_rows=out.num_rows,
                   child_execute_ms=round(child_ms, 3), sort_node_execute_ms=round(node_ms, 3),
                   sort_node_minus_child_ms=round(node_ms - child_ms, 3))
    ctx.close()


if __name__ == "__main__":
    main()
