"""Rank harnesses of the multi-rank tests: gloo worlds of CPU processes (spawn_gloo), a one-rank NCCL communicator on
one GPU (one_rank_comm), and the torchrun session of a multi-GPU check script (rank_session)."""
import contextlib
import os
import socket
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _gloo_rank(worker, rank, world, port, q, args):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    q.put((rank, worker(rank, world, *args)))
    dist.barrier()
    dist.destroy_process_group()


def spawn_gloo(worker, world=2, args=(), timeout=240):
    """worker(rank, world, *args) in `world` spawned processes joined in a gloo process group -> the workers' results
    in rank order.  Each result is waited for `timeout` seconds, each process must exit with 0."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_gloo_rank, args=(worker, r, world, port, q, args)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=timeout) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return [got[r] for r in range(world)]


@contextlib.contextmanager
def one_rank_comm(ctx):
    """ctx with a one-rank NCCL communicator (comm_init(id, 1, 0)), destroyed on exit; skips when NCCL cannot be
    loaded."""
    from greptimedb_b200 import B2PError
    try:
        uid = ctx.comm_unique_id()
    except B2PError as e:
        if "libnccl" in str(e):
            pytest.skip(f"NCCL cannot be loaded: {e}")
        raise
    ctx.comm_init(uid, 1, 0)
    try:
        yield ctx
    finally:
        ctx.comm_destroy()


def rank_session(tag, body):
    """A multi-GPU check script's rank under torchrun (one rank per GPU): set the device, join the NCCL process group,
    give a context the world's communicator, run body(s) with s.rank, s.world, s.dev and s.ctx, which returns its list
    of failures; then the verdict: the failures printed, every rank's verdict all-reduced with MIN, "<tag> world=<n>
    ok=<bool>" and s.note printed by rank 0, and the exit code.  torch.distributed carries the 128-byte communicator id
    and the verdict, and whatever the body sends itself."""
    import types

    import torch
    import torch.distributed as dist
    from greptimedb_b200 import Context
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    ctx = Context(local)
    ctx.use_own_stream()
    box = [ctx.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=0)
    ctx.comm_init(box[0], world, rank)
    s = types.SimpleNamespace(rank=rank, world=world, dev=dev, ctx=ctx, note="")
    bad = body(s)
    ctx.comm_destroy()
    ctx.close()
    verdict = torch.tensor([0.0 if bad else 1.0], device=dev)
    dist.all_reduce(verdict, op=dist.ReduceOp.MIN)
    for b in bad:
        print(b, flush=True)
    ok = bool(verdict.item() == 1.0)
    if rank == 0:
        print(f"{tag} world={world} ok={ok} {s.note}".rstrip(), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)
