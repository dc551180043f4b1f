"""Times the sharded topk / bottomk (b2p_topk_allgather_dev) on device-resident random grids.

One GPU (plain `python`): the composed call over a one-rank communicator (the all-reduce of the group sizes, the
candidate blocks, three all-gathers per batch and round, the merge, the mark) against b2p_topk_dev on the shapes of
profiles/topk_bench.py: what the exchange machinery costs when there is nothing to exchange with.  Without NCCL the
composed call runs without a communicator, and the line says so.

N GPUs (`torchrun --nproc-per-node N profiles/topk_sharded_bench.py`): every rank holds --series rows (default 1.25 M) x
1000 steps of its own rate-like grid (90 % of the cells valid, uniform random values), and runs topk(10, ·) over one
group, topk(5, ·) by --groups groups (default 1000), and topk(100, ·) over one group (rounds).

Each line is one JSON object: the CUDA-event time of the call (median of --reps, stage 3 of b2p_last_kernel_ms, which
spans the whole call, collectives included), the bytes of this rank's candidate blocks (b2p_last_exchange_bytes), the
bytes gathering the grid to one rank would move per rank (8 B per cell plus the validity words), and the card's name
and power limit read in the same run.

  python profiles/topk_sharded_bench.py [--rows N] [--series N] [--groups G] [--reps R]
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
        vals = torch.rand(rows * T, dtype=torch.float64, device=dev, generator=gen)
        shifts = torch.arange(32, device=dev, dtype=torch.int64)
        words = torch.empty((rows, Tw), dtype=torch.int32, device=dev)
        for w in range(Tw):
            ok = (torch.rand((rows, 32), device=dev, generator=gen) < 0.9) & (w * 32 + shifts < T)
            x = (ok.to(torch.int64) << shifts).sum(1)
            words[:, w] = torch.where(x >= 2 ** 31, x - 2 ** 32, x).to(torch.int32)
        # distinct across ranks: this rank's rows take the ordinals [rank * rows, (rank + 1) * rows)
        tie = (torch.randperm(rows, device=dev, generator=gen) + rank * rows).to(torch.int32)
        return vals, words.flatten(), tie

    def timed(call, words):
        work = words.clone()
        ms = []
        for i in range(args.reps + 2):
            work.copy_(words)
            call(work)
            ctx.sync()
            if i >= 2:
                ms.append(ctx.kernel_ms(3))
        return float(np.median(ms)), work

    def run(query, k, rows, gid, n_groups, vals, words, tie, single=True):
        ix = ctx.group_index_create_dev(gid, rows, n_groups)
        line = {"query": query, "ranks": world, "rows_per_rank": rows, "groups": n_groups, "steps": T, "k": k,
                "communicator": comm}
        m, got = timed(lambda w: ctx.topk_allgather_dev("topk", k, vals, w, ix, tie, T, w), words)
        line["allgather_ms"] = round(m, 4)
        line["exchange_bytes_per_rank"] = ctx.last_exchange_bytes()
        line["gather_grid_bytes_per_rank"] = rows * T * 8 + rows * Tw * 4
        if single:
            m1, ref = timed(lambda w: ctx.topk_dev("topk", k, vals, w, ix, tie, T, w), words)
            line["topk_dev_ms"] = round(m1, 4)
            line["same_words"] = bool(torch.equal(got, ref))
        ctx.group_index_destroy(ix)
        if rank == 0:
            print(json.dumps({**line, **ident}), flush=True)

    if world == 1:
        N = args.rows
        vals, words, tie = grid(N)
        one = torch.zeros(N, dtype=torch.int32, device=dev)
        run("topk(10, sum by (pod)(rate(x[5m])))", 10.0, N, one, 1, vals, words, tie)
        del vals, words, tie, one
        S, G = args.series, args.groups
        vals, words, tie = grid(S)
        job = torch.randint(0, G, (S,), dtype=torch.int32, device=dev, generator=gen)
        run("topk(5, rate(x[5m])) by (job)", 5.0, S, job, G, vals, words, tie)
        del vals, words, tie, job
        torch.cuda.empty_cache()
        vals, words, tie = grid(N)
        one = torch.zeros(N, dtype=torch.int32, device=dev)
        run("topk(100, ·) one group (rounds)", 100.0, N, one, 1, vals, words, tie)
        run("topk(k >= group size, ·) (copy)", float(N), N, one, 1, vals, words, tie)
    else:
        S, G = args.series, args.groups
        vals, words, tie = grid(S)
        one = torch.zeros(S, dtype=torch.int32, device=dev)
        run("topk(10, rate(x[5m]))", 10.0, S, one, 1, vals, words, tie, single=False)
        job = torch.randint(0, G, (S,), dtype=torch.int32, device=dev, generator=gen)
        run("topk(5, rate(x[5m])) by (job)", 5.0, S, job, G, vals, words, tie, single=False)
        run("topk(100, rate(x[5m]))", 100.0, S, one, 1, vals, words, tie, single=False)
    if comm != "none":
        ctx.comm_destroy()
    ctx.close()
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
