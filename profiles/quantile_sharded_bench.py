"""Times the sharded quantile (b2p_quantile_allreduce_dev) on device-resident random grids.

One GPU (plain `python`): the composed call over a one-rank communicator (per batch and pass the rank's block, three
all-reduces and the advance, which reads back the cells left) against b2p_group_quantile_dev on the shapes of
profiles/quantile_bench.py: what the exchange machinery costs when there is nothing to exchange with.
  a. one group of --rows rows (default 100 k) x 1000 steps, φ = 0.99
  b. --series rows (default 1.25 M) x 1000 steps in --groups groups (default 1000), φ = 0.9
  c. --rows rows x 1000 steps in groups of 8, φ = 0.9
Without NCCL the composed call runs without a communicator, and the line says so.

N GPUs (`torchrun --nproc-per-node N profiles/quantile_sharded_bench.py`): every rank holds --series rows x 1000 steps
of its own grid and runs shape b and φ = 0.99 over one group; there is no single-GPU call to compare with.  With fewer
than two GPUs visible that measurement is not made, and a line says "not measured".

Each line is one JSON object: the CUDA-event time of the call (median of --reps, stage 3 of b2p_last_kernel_ms, which
spans the whole call, collectives included), the bytes of this rank's blocks (b2p_last_exchange_bytes) and the
(group, tile) unit-passes they stand for (bytes / 2 560; over the units, the mean passes run), the bytes gathering the
grid to one rank would move per rank (8 B per cell plus the validity words), the device time of the pass kernel, the
advance kernel, the NCCL kernels and the rest of one call from a torch.profiler run of its own, and the card's name
and power limit read in the same run.

  python profiles/quantile_sharded_bench.py [--rows N] [--series N] [--groups G] [--reps R]
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
UNIT_BYTES = 2560


def kernel_split(call):
    """device time (ms) of one call by kernel family, from a torch.profiler run of its own"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    split = {"pass_kernel_ms": 0.0, "advance_kernel_ms": 0.0, "nccl_ms": 0.0, "other_device_ms": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0:
            continue
        name = e.key.lower()
        key = ("pass_kernel_ms" if "quantile_pass_kernel" in name else "advance_kernel_ms"
               if "quantile_advance_kernel" in name else "nccl_ms" if "nccl" in name else "other_device_ms")
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

    def grid(rows):
        vals = torch.randn(rows * T, dtype=torch.float64, device=dev, generator=gen)
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
            call()
            ctx.sync()
            if i >= 2:
                ms.append(ctx.kernel_ms(3))
        return float(np.median(ms))

    def run(query, phi, rows, gid, n_groups, vals, words, single=True):
        ix = ctx.group_index_create_dev(gid, rows, n_groups)
        out = torch.empty(n_groups * T, dtype=torch.float64, device=dev)
        cnt = torch.empty(n_groups * T, dtype=torch.int32, device=dev)
        units = n_groups * Tw
        line = {"query": query, "phi": phi, "ranks": world, "rows_per_rank": rows, "groups": n_groups, "steps": T,
                "communicator": comm}
        sharded = lambda: ctx.quantile_allreduce_dev(phi, vals, words, ix, T, out, cnt)  # noqa: E731
        line["allreduce_ms"] = round(timed(sharded), 4)
        xb = ctx.last_exchange_bytes()
        line["exchange_bytes_per_rank"] = xb
        line["unit_passes"] = xb // UNIT_BYTES
        line["mean_passes"] = round(xb / UNIT_BYTES / units, 3)
        line["gather_grid_bytes_per_rank"] = rows * T * 8 + rows * Tw * 4
        line.update(kernel_split(sharded))
        if single:
            got = (out.clone(), cnt.clone())
            line["group_quantile_dev_ms"] = round(timed(lambda: ctx.group_quantile_dev(phi, vals, words, ix, T, out,
                                                                                       cnt)), 4)
            line["same_bits"] = bool(torch.equal(got[0].view(torch.int64), out.view(torch.int64))
                                     and torch.equal(got[1], cnt))
        ctx.group_index_destroy(ix)
        if rank == 0:
            print(json.dumps({**line, **ident}), flush=True)

    if world == 1:
        N = args.rows
        vals, words = grid(N)
        one = torch.zeros(N, dtype=torch.int32, device=dev)
        run("a. quantile(0.99, x), one group", 0.99, N, one, 1, vals, words)
        eights = torch.arange(N, dtype=torch.int32, device=dev) // 8
        run("c. quantile(0.9, x) by (pair), groups of 8", 0.9, N, eights, (N + 7) // 8, vals, words)
        del vals, words, one, eights
        torch.cuda.empty_cache()
        S, G = args.series, args.groups
        vals, words = grid(S)
        job = torch.randint(0, G, (S,), dtype=torch.int32, device=dev, generator=gen)
        run("b. quantile(0.9, x) by (job)", 0.9, S, job, G, vals, words)
        if torch.cuda.device_count() < 2:
            print(json.dumps({"multi_gpu": "not measured: one GPU visible", **ident}), flush=True)
    else:
        S, G = args.series, args.groups
        vals, words = grid(S)
        job = torch.randint(0, G, (S,), dtype=torch.int32, device=dev, generator=gen)
        run("b. quantile(0.9, x) by (job)", 0.9, S, job, G, vals, words, single=False)
        one = torch.zeros(S, dtype=torch.int32, device=dev)
        run("quantile(0.99, x), one group", 0.99, S, one, 1, vals, words, single=False)
    if comm != "none":
        ctx.comm_destroy()
    ctx.close()
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
