"""Times count_values by label (K12, b2p_count_values_dev) on device-resident random grids, and K3 `count` beside it.

  a. one group of --rows rows (default 100 k) x 1000 steps, 16 distinct values
  b. --series rows (default 1.25 M) x 1000 steps in --groups groups (default 1000), 16 distinct values per group
  c. shape b with every value distinct (the worst case: one output row per cell)
  d. --rows rows x 1000 steps in groups of 8, 16 distinct values
  e. K3 count (b2p_group_aggregate_indexed_dev) on shape b, the floor: it reads the validity bits only (1 bit per cell)

Each input has 90 % of its cells valid.  For each shape it prints one JSON line: the CUDA-event time of the call
(median of --reps after two warm-up calls), the bytes one read of the input needs (8 B + 1 bit per cell; 1 bit for e),
that rate and its fraction of the H100 SXM data-sheet 3.35 TB/s, and the card's name and power limit read in the same
run.

  python profiles/count_values_bench.py [--rows N] [--series N] [--groups G] [--reps R]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from binary_bench import PEAK_TBS, gpu_identity  # noqa: E402

T = 1000


def read_bytes(rows: int) -> int:
    return rows * T * 8 + rows * T // 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--series", type=int, default=1_250_000)
    ap.add_argument("--groups", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    import numpy as np
    import torch

    from greptimedb_b200 import Context

    dev = torch.device("cuda:0")
    ctx = Context(0)
    ctx.use_torch_stream()
    ident = gpu_identity()
    Tw = (T + 31) // 32
    gen = torch.Generator(device=dev).manual_seed(0x5EED)

    def words(rows):
        shifts = torch.arange(32, device=dev, dtype=torch.int64)
        out = torch.empty((rows, Tw), dtype=torch.int32, device=dev)
        for w in range(Tw):
            ok = (torch.rand((rows, 32), device=dev, generator=gen) < 0.9) & (w * 32 + shifts < T)
            x = (ok.to(torch.int64) << shifts).sum(1)
            out[:, w] = torch.where(x >= 2 ** 31, x - 2 ** 32, x).to(torch.int32)
        return out.flatten()

    def sixteen(rows):
        return torch.randint(0, 16, (rows * T,), device=dev, generator=gen).to(torch.float64) * 0.5

    def run(query, rows, gid, n_groups, vals, valid, count=False):
        ix = ctx.group_index_create_dev(gid, rows, n_groups)
        out_rows = n_groups if count else rows
        out = torch.empty(out_rows * T, dtype=torch.float64, device=dev)
        cnt = torch.empty(out_rows * T, dtype=torch.int32, device=dev)
        ms = []
        for i in range(args.reps + 2):
            if count:
                ctx.group_aggregate_indexed_dev("count", vals, valid, ix, T, out, cnt)
            else:
                ctx.count_values_dev(vals, valid, ix, T, out, cnt)
            ctx.sync()
            if i >= 2:
                ms.append(ctx.kernel_ms(3))
        ctx.group_index_destroy(ix)
        del out, cnt
        m, b = float(np.median(ms)), rows * T // 8 if count else read_bytes(rows)  # count reads the validity bits only
        print(json.dumps({"query": query, "rows": rows, "groups": n_groups, "steps": T, "kernel_ms": round(m, 4),
                          "bytes": b, "tb_per_s": round(b / m / 1e9, 3),
                          "fraction_of_3.35_tb_s": round(b / m / 1e9 / PEAK_TBS, 3), **ident}), flush=True)

    N = args.rows
    vals, valid = sixteen(N), words(N)
    run("a. count_values, one group, 16 distinct values", N, torch.zeros(N, dtype=torch.int32, device=dev), 1, vals, valid)
    eights = torch.arange(N, dtype=torch.int32, device=dev) // 8
    run("d. count_values by (pair), groups of 8, 16 distinct values", N, eights, (N + 7) // 8, vals, valid)
    del vals, valid, eights
    S, G = args.series, args.groups
    valid = words(S)
    job = torch.randint(0, G, (S,), dtype=torch.int32, device=dev, generator=gen)
    vals = sixteen(S)
    run("b. count_values by (job), 16 distinct values per group", S, job, G, vals, valid)
    run("e. count(x) by (job) (K3)", S, job, G, vals, valid, count=True)
    del vals
    vals = torch.randn(S * T, dtype=torch.float64, device=dev, generator=gen)
    run("c. count_values by (job), every value distinct", S, job, G, vals, valid)
    ctx.close()


if __name__ == "__main__":
    main()
