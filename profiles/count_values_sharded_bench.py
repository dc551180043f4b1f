"""Times the sharded count_values (b2p_count_values_shard_heights_dev + b2p_count_values_allgather_dev) on
device-resident random grids.

One GPU (plain `python`): over a one-rank communicator, the heights (one all-gather and a read-back) and the composed
call (per batch the rank's block, two all-gathers and the merge) against b2p_count_values_dev alone, which every rank
runs first over its own rows:
  a. --series rows (default 1.25 M) x 1000 steps in --groups groups (default 1000), 5 distinct values
  b. the same with all-distinct values
  c. --rows rows (default 100 k) x 1000 steps in groups of 8, 5 distinct values
What the exchange machinery costs when there is nothing to exchange with.  Without NCCL the calls run without a
communicator, and the line says so.

N GPUs (`torchrun --nproc-per-node N profiles/count_values_sharded_bench.py`): every rank holds --series rows of its own
grid and runs shape a; there is no single-GPU call to compare with.  With fewer than two GPUs visible that measurement
is not made, and a line says "not measured".

Each line is one JSON object: CUDA-event times (median of --reps) of b2p_count_values_dev, of the heights and of the
composed call; the bytes of this rank's blocks (b2p_last_exchange_bytes) against the bytes gathering the grid to one
rank would move per rank (8 B per cell plus the validity words); the device time of the count_values kernels (K12's
and the pack / merge ones), CUB's sort and scans, the NCCL kernels and the rest of one heights + composed call from a
torch.profiler run of its own; whether the merged rows equal the single-rank rows bit for bit; and the card's name and
power limit read in the same run.

  python profiles/count_values_sharded_bench.py [--rows N] [--series N] [--groups G] [--reps R]
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

T = 1000


def kernel_split(call):
    """device time (ms) of one call by kernel family, from a torch.profiler run of its own"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    split = {"count_values_kernels_ms": 0.0, "cub_ms": 0.0, "nccl_ms": 0.0, "other_device_ms": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0:
            continue
        name = e.key.lower()
        key = ("count_values_kernels_ms" if "count_values" in name else "nccl_ms" if "nccl" in name
               else "cub_ms" if "cub" in name else "other_device_ms")
        split[key] += us / 1000.0
    return {k: round(v, 4) for k, v in split.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--series", type=int, default=1_250_000)
    ap.add_argument("--groups", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    import numpy as np
    import torch

    from greptimedb_b200 import B2PError, Context

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    ctx = Context(local)
    ctx.use_torch_stream()
    ident = gpu_identity()
    Tw = (T + 31) // 32
    comm = "none"
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
        box = [ctx.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        ctx.comm_init(box[0], world, rank)
        comm = f"nccl x{world}"
    else:
        try:
            ctx.comm_init(ctx.comm_unique_id(), 1, 0)
            comm = "nccl x1"
        except B2PError as e:
            print(json.dumps({"note": f"no communicator: {e}"}), flush=True)
    gen = torch.Generator(device=dev).manual_seed(0x5EED + rank)

    def grid(rows, distinct):
        if distinct:
            vals = torch.randn(rows * T, dtype=torch.float64, device=dev, generator=gen)
        else:
            vals = torch.randint(0, 5, (rows * T,), device=dev, generator=gen).to(torch.float64)
        shifts = torch.arange(32, device=dev, dtype=torch.int64)
        words = torch.empty((rows, Tw), dtype=torch.int32, device=dev)
        for w in range(Tw):
            ok = (torch.rand((rows, 32), device=dev, generator=gen) < 0.9) & (w * 32 + shifts < T)
            x = (ok.to(torch.int64) << shifts).sum(1)
            words[:, w] = torch.where(x >= 2 ** 31, x - 2 ** 32, x).to(torch.int32)
        return vals, words.flatten()

    def timed(call):
        ms = []
        for i in range(args.reps + 2):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            call()
            b.record()
            torch.cuda.synchronize()
            if i >= 2:
                ms.append(a.elapsed_time(b))
        return float(np.median(ms))

    def run(query, rows, gid, n_groups, vals, words, single=True):
        ix = ctx.group_index_create_dev(gid, rows, n_groups)
        lv = torch.empty(rows * T, dtype=torch.float64, device=dev)
        lc = torch.empty(rows * T, dtype=torch.int32, device=dev)
        line = {"query": query, "ranks": world, "rows_per_rank": rows, "groups": n_groups, "steps": T,
                "communicator": comm}
        line["count_values_dev_ms"] = round(timed(lambda: ctx.count_values_dev(vals, words, ix, T, lv, lc)), 4)
        line["heights_ms"] = round(timed(lambda: ctx.count_values_shard_heights_dev(lc, ix, T, n_groups, world)), 4)
        H = ctx.count_values_shard_heights_dev(lc, ix, T, n_groups, world)
        out_goff = ctx.count_values_shard_rows(H)
        U = int(out_goff[-1])
        ov = torch.empty(max(U, 1) * T, dtype=torch.float64, device=dev)
        oc = torch.empty(max(U, 1) * T, dtype=torch.int32, device=dev)
        composed = lambda: ctx.count_values_allgather_dev(lv, lc, ix, T, H, ov, oc)  # noqa: E731
        line["allgather_ms"] = round(timed(composed), 4)
        line["output_rows"] = U
        line["batches"] = ctx.count_values_shard_plan(H, T)["n_batches"]
        line["exchange_bytes_per_rank"] = ctx.last_exchange_bytes()
        line["gather_grid_bytes_per_rank"] = rows * T * 8 + rows * Tw * 4
        line.update(kernel_split(lambda: (ctx.count_values_shard_heights_dev(lc, ix, T, n_groups, world), composed())))
        if single:
            torch.cuda.synchronize()
            goff = np.concatenate([[0], np.cumsum(np.bincount(gid.cpu().numpy(), minlength=n_groups))])
            keep = np.concatenate([np.arange(goff[g], goff[g] + out_goff[g + 1] - out_goff[g])
                                   for g in range(n_groups)])
            same = True
            for i in range(0, U, 100_000):  # in slices of rows: no second copy of the grid
                k = torch.from_numpy(keep[i:i + 100_000]).to(dev)
                n = k.numel()
                same = same and torch.equal(ov[i * T:(i + n) * T].view(torch.int64),
                                            lv.view(rows, T)[k].reshape(-1).view(torch.int64))
                same = same and torch.equal(oc[i * T:(i + n) * T], lc.view(rows, T)[k].reshape(-1))
            line["same_bits"] = bool(same)
        ctx.group_index_destroy(ix)
        if rank == 0:
            print(json.dumps({**line, **ident}), flush=True)

    if world == 1:
        S, G = args.series, args.groups
        job = torch.randint(0, G, (S,), dtype=torch.int32, device=dev, generator=gen)
        vals, words = grid(S, False)
        run("a. count_values(\"v\", x) by (job), 5 distinct values", S, job, G, vals, words)
        del vals, words
        torch.cuda.empty_cache()
        vals, words = grid(S, True)
        run("b. count_values(\"v\", x) by (job), all distinct", S, job, G, vals, words)
        del vals, words, job
        torch.cuda.empty_cache()
        N = args.rows
        vals, words = grid(N, False)
        eights = torch.arange(N, dtype=torch.int32, device=dev) // 8
        run("c. count_values(\"v\", x) by (pair), groups of 8", N, eights, (N + 7) // 8, vals, words)
        if torch.cuda.device_count() < 2:
            print(json.dumps({"multi_gpu": "not measured: one GPU visible", **ident}), flush=True)
    else:
        S, G = args.series, args.groups
        vals, words = grid(S, False)
        job = torch.randint(0, G, (S,), dtype=torch.int32, device=dev, generator=gen)
        run("a. count_values(\"v\", x) by (job), 5 distinct values", S, job, G, vals, words, single=False)
    if comm != "none":
        ctx.comm_destroy()
    ctx.close()
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
