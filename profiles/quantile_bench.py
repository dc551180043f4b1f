"""Times quantile by label (K11, b2p_group_quantile_dev) on device-resident random grids, and K3 `avg` beside it.

  a. one group of --rows rows (default 100 k) x 1000 steps, φ = 0.99 and 0.5 (the chunked path)
  b. --series rows (default 1.25 M) x 1000 steps in --groups groups (default 1000; the multi-pass path)
  c. --rows rows x 1000 steps in groups of 8 (the resident path)
  d. K3 avg (b2p_group_aggregate_indexed_dev) on shape b, for comparison

Each input has 90 % of its cells valid and distinct random values.  For each shape it prints one JSON line: the
CUDA-event time of the call (median of --reps), the bytes one read of the input needs (8 B + 1 bit per cell), that rate
and its fraction of the H100 SXM data-sheet 3.35 TB/s, and the card's name and power limit read in the same run.

  python profiles/quantile_bench.py [--rows N] [--series N] [--groups G] [--reps R]
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

    def grid(rows):
        vals = torch.randn(rows * T, dtype=torch.float64, device=dev, generator=gen)
        shifts = torch.arange(32, device=dev, dtype=torch.int64)
        words = torch.empty((rows, Tw), dtype=torch.int32, device=dev)
        for w in range(Tw):
            ok = (torch.rand((rows, 32), device=dev, generator=gen) < 0.9) & (w * 32 + shifts < T)
            x = (ok.to(torch.int64) << shifts).sum(1)
            words[:, w] = torch.where(x >= 2 ** 31, x - 2 ** 32, x).to(torch.int32)
        return vals, words.flatten()

    def run(query, rows, gid, n_groups, vals, words, phi=None):
        ix = ctx.group_index_create_dev(gid, rows, n_groups)
        out = torch.empty(n_groups * T, dtype=torch.float64, device=dev)
        cnt = torch.empty(n_groups * T, dtype=torch.int32, device=dev)
        ms = []
        for i in range(args.reps + 2):
            if phi is None:
                ctx.group_aggregate_indexed_dev("avg", vals, words, ix, T, out, cnt)
            else:
                ctx.group_quantile_dev(phi, vals, words, ix, T, out, cnt)
            ctx.sync()
            if i >= 2:
                ms.append(ctx.kernel_ms(3))
        ctx.group_index_destroy(ix)
        m, b = float(np.median(ms)), read_bytes(rows)
        print(json.dumps({"query": query, "rows": rows, "groups": n_groups, "steps": T, "phi": phi,
                          "kernel_ms": round(m, 4), "bytes": b, "tb_per_s": round(b / m / 1e9, 3),
                          "fraction_of_3.35_tb_s": round(b / m / 1e9 / PEAK_TBS, 3), **ident}), flush=True)

    N = args.rows
    vals, words = grid(N)
    one = torch.zeros(N, dtype=torch.int32, device=dev)
    run("a. quantile(0.99, x), one group", N, one, 1, vals, words, 0.99)
    run("a. quantile(0.5, x), one group", N, one, 1, vals, words, 0.5)
    eights = torch.arange(N, dtype=torch.int32, device=dev) // 8
    run("c. quantile(0.9, x) by (pair), groups of 8", N, eights, (N + 7) // 8, vals, words, 0.9)
    del vals, words, one, eights
    S, G = args.series, args.groups
    vals, words = grid(S)
    job = torch.randint(0, G, (S,), dtype=torch.int32, device=dev, generator=gen)
    run("b. quantile(0.9, x) by (job)", S, job, G, vals, words, 0.9)
    run("d. avg(x) by (job) (K3)", S, job, G, vals, words)
    ctx.close()


if __name__ == "__main__":
    main()
