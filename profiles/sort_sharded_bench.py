"""Times the sharded sort (b2p_sort_shard_pack_dev, b2p_sort_shard_merge_dev, b2p_sort_cells_allgather_dev) on
device-resident grids on one GPU, with R ranks simulated by R contexts.

Shapes (standard-normal values, about 90 % of the cells valid):
  a. --rows1 rows (default 10 M) x 1 step: PromQL sort is mostly an instant-query function;
  b. --rows2 rows (default 100 k) x 1000 steps.
For each shape and R in 1, 2, 4, 8 (rows hashed to ranks by distributed.shard_of_series):
  - pack_ms: each rank's pack (K14 over its rows, then the pack kernel), the largest and the sum over ranks;
  - merge_ms: one rank's merge over every block laid back to back, against its HBM bound: rounds x 2 x N x 8 (F + 1)
    bytes (every round reads and writes every entry once), as an achieved rate and a share of the H100 SXM data sheet's
    3.35 TB/s; the merge kernels' device time from a torch.profiler run of its own;
  - sort_union_ms: b2p_sort_cells_dev over the whole grid, what a frontend does today after gathering the rows.
Then the composed call over a one-rank communicator beside b2p_sort_cells_dev, and the bytes the exchange moves
(16 B per valid cell) against the bytes gathering the grid moves (8 B per cell plus its validity words).

CUDA events around each call, median of --reps after one warm-up of every shape.  Every merged order is checked bit for
bit against b2p_sort_cells_dev.  Every line is one JSON object with the card's name and power limit read in the same run.
Multi-GPU runs are not made by this script.

  python profiles/sort_sharded_bench.py [--rows1 N] [--rows2 N] [--reps R]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from binary_bench import gpu_identity  # noqa: E402

HBM_BPS = 3.35e12


def median_ms(call, reps):
    import torch
    call()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def kernel_ms(call, needle):
    """device time (ms) of the kernels whose name holds `needle` in one call, from a torch.profiler run of its own"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    total = 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if needle in e.key:
            total += us / 1000.0
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows1", type=int, default=10_000_000)
    ap.add_argument("--rows2", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import numpy as np
    import torch
    from greptimedb_b200 import B2PError, Context
    from greptimedb_b200 import distributed as D
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    ident = gpu_identity()

    def report(**kw):
        print(json.dumps({**kw, **ident}), flush=True)

    for shape, R_rows, T in (("a", args.rows1, 1), ("b", args.rows2, 1000)):
        Tw = (T + 31) // 32
        g = torch.Generator(device="cuda").manual_seed(7)
        vals = torch.randn(R_rows * T, dtype=torch.float64, device="cuda", generator=g)
        bits = torch.rand((R_rows, Tw * 32), device="cuda", generator=g) < 0.9
        bits[:, T:] = False
        w = torch.zeros((R_rows, Tw), dtype=torch.int64, device="cuda")
        for b in range(32):
            w |= bits[:, b::32].to(torch.int64) << b
        valid = torch.where(w >= 1 << 31, w - (1 << 32), w).to(torch.int32).contiguous()
        one = Context(0)
        one.use_torch_stream()
        ref = torch.empty(R_rows * T, dtype=torch.int64, device="cuda")
        n_dev = torch.zeros(1, dtype=torch.int64, device="cuda")
        sort_union = median_ms(lambda: one.sort_cells_dev(False, vals, valid, R_rows, T, ref, n_dev), args.reps)
        torch.cuda.synchronize()
        N = int(n_dev.item())
        exp = ref[:N].clone()
        for n_ranks in (1, 2, 4, 8):
            owner = torch.from_numpy(D.shard_of_series(np.arange(R_rows, dtype=np.uint32), n_ranks)).cuda()
            ranks = []
            for r in range(n_ranks):
                rows = torch.nonzero(owner == r).flatten()
                ctx = Context(0)
                ctx.use_torch_stream()
                v = vals.view(R_rows, T)[rows].reshape(-1).contiguous()
                vw = valid[rows].contiguous()
                rid = rows.to(torch.int32).contiguous()
                cnt = int(ctx.sort_shard_counts_dev(vw, rows.numel(), T)[0])
                ranks.append((ctx, v, vw, rid, rows.numel(), cnt,
                              torch.empty(max(cnt * 2, 1), dtype=torch.int64, device="cuda")))
            counts = np.array([r[5] for r in ranks], np.uint64)
            pack = []
            for ctx, v, vw, rid, n, cnt, blk in ranks:
                pack.append(median_ms(lambda: ctx.sort_shard_pack_dev(False, v, vw, rid, n, T, cnt, blk), args.reps))
            laid = torch.cat([r[6][:r[5] * 2] for r in ranks])
            cells = torch.empty(N, dtype=torch.int64, device="cuda")
            out = torch.empty(N, dtype=torch.float64, device="cuda")
            m = ranks[0][0]
            merge = median_ms(lambda: m.sort_shard_merge_dev(False, counts, laid, cells, out), args.reps)
            merge_dev = kernel_ms(lambda: m.sort_shard_merge_dev(False, counts, laid, cells, out), "sort_shard_merge")
            torch.cuda.synchronize()
            ok = bool(torch.equal(cells, exp))
            runs = int((counts > 0).sum())
            rounds = max(1, int(np.ceil(np.log2(max(runs, 1)))))
            bound = rounds * 2 * N * 16
            report(shape=shape, rows=R_rows, T=T, valid_cells=N, ranks=n_ranks, pack_ms_max=round(max(pack), 3),
                   pack_ms_sum=round(sum(pack), 3), merge_ms=round(merge, 3), merge_kernels_ms=round(merge_dev, 3),
                   merge_rounds=rounds, merge_hbm_bytes=bound, merge_gbps=round(bound / merge / 1e6, 1),
                   merge_share_of_3_35_tbps=round(bound / (merge / 1e3) / HBM_BPS, 3),
                   sort_union_ms=round(sort_union, 3), bit_exact=ok)
            for r in ranks:
                r[0].close()
        # the composed call over a one-rank communicator, and the bytes against gathering the grid
        try:
            one.comm_init(one.comm_unique_id(), 1, 0)
            comm = True
        except B2PError:
            comm = False
        rid = torch.arange(R_rows, dtype=torch.int32, device="cuda")
        counts = one.sort_shard_counts_dev(valid, R_rows, T)
        cells = torch.empty(N, dtype=torch.int64, device="cuda")
        out = torch.empty(N, dtype=torch.float64, device="cuda")
        composed = median_ms(lambda: one.sort_cells_allgather_dev(False, vals, valid, rid, R_rows, T, counts, cells,
                                                                  out), args.reps)
        torch.cuda.synchronize()
        report(shape=shape, rows=R_rows, T=T, valid_cells=N, composed_ms=round(composed, 3),
               communicator="one-rank NCCL" if comm else "none (NCCL could not be loaded)",
               sort_union_ms=round(sort_union, 3), exchange_bytes=one.last_exchange_bytes(),
               gather_grid_bytes=R_rows * T * 8 + R_rows * Tw * 4, bit_exact=bool(torch.equal(cells, exp)))
        if comm:
            one.comm_destroy()
        one.close()
    report(multi_gpu="not measured")


if __name__ == "__main__":
    main()
