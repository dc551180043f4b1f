"""Times topk / bottomk (K10, b2p_topk_dev) on device-resident random grids, in place.

  1. topk(10, ·): the config-3 aggregate shape, --rows rows (default 100 k) x 1000 steps in one group
  2. topk(5, ·) by (job): --series rows (default 1.25 M) x 1000 steps in --groups groups (default 1000)
  3. shape 1 with k = 100, which takes the general path (rounds of 32)
  4. shape 1 with k >= the group size: every valid cell is kept, a copy of the validity words

Each input has 90 % of its cells valid and distinct random values.  The validity words are restored from a copy
before every call (in place, a call leaves only the kept cells).  For each shape it prints one JSON line: the CUDA-event
time of the call (median of --reps), the algorithmic bytes (8 B + 1 bit read and 1 bit written per cell, plus 4 B per
row: the tie ordinal), that rate and its fraction of the H100 SXM data-sheet 3.35 TB/s, and the card's name and power
limit read in the same run.

  python profiles/topk_bench.py [--rows N] [--series N] [--groups G] [--reps R]
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


def topk_bytes(rows: int) -> int:
    return rows * T * 8 + 2 * rows * T // 8 + 4 * rows


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
        vals = torch.rand(rows * T, dtype=torch.float64, device=dev, generator=gen)
        shifts = torch.arange(32, device=dev, dtype=torch.int64)
        words = torch.empty((rows, Tw), dtype=torch.int32, device=dev)
        for w in range(Tw):
            ok = (torch.rand((rows, 32), device=dev, generator=gen) < 0.9) & (w * 32 + shifts < T)
            x = (ok.to(torch.int64) << shifts).sum(1)
            words[:, w] = torch.where(x >= 2 ** 31, x - 2 ** 32, x).to(torch.int32)
        tie = torch.randperm(rows, device=dev, generator=gen).to(torch.int32)
        return vals, words.flatten(), tie

    def run(query, op, k, rows, gid, n_groups, vals, words, tie):
        ix = ctx.group_index_create_dev(gid, rows, n_groups)
        work = words.clone()
        ms = []
        for i in range(args.reps + 2):
            work.copy_(words)
            ctx.topk_dev(op, k, vals, work, ix, tie, T, work)
            ctx.sync()
            if i >= 2:
                ms.append(ctx.kernel_ms(3))
        ctx.group_index_destroy(ix)
        m, b = float(np.median(ms)), topk_bytes(rows)
        print(json.dumps({"query": query, "rows": rows, "groups": n_groups, "steps": T, "k": k,
                          "kernel_ms": round(m, 4), "bytes": b, "tb_per_s": round(b / m / 1e9, 3),
                          "fraction_of_3.35_tb_s": round(b / m / 1e9 / PEAK_TBS, 3), **ident}), flush=True)

    N = args.rows
    vals, words, tie = grid(N)
    one = torch.zeros(N, dtype=torch.int32, device=dev)
    run("topk(10, sum by (pod)(rate(x[5m])))", "topk", 10.0, N, one, 1, vals, words, tie)
    del vals, words, tie, one
    S, G = args.series, args.groups
    vals, words, tie = grid(S)
    job = torch.randint(0, G, (S,), dtype=torch.int32, device=dev, generator=gen)
    run("topk(5, rate(x[5m])) by (job)", "topk", 5.0, S, job, G, vals, words, tie)
    del vals, words, tie, job
    torch.cuda.empty_cache()
    vals, words, tie = grid(N)
    one = torch.zeros(N, dtype=torch.int32, device=dev)
    run("topk(100, ·) one group (general path)", "topk", 100.0, N, one, 1, vals, words, tie)
    run("topk(k >= group size, ·) (copy)", "topk", float(N), N, one, 1, vals, words, tie)
    ctx.close()


if __name__ == "__main__":
    main()
