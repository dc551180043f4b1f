"""World-size-2 gloo test (CPU) of the sharded topk / bottomk exchange: every rank holds whole series, the host mirror
of b2p_topk_allgather_dev (distributed.merge_topk_candidates) exchanges candidates, and the union of the ranks' kept
cells equals select_keys.topk over all rows.  The grids hold adversarial total-order keys (NaN payloads of both signs,
±0, ±inf, sentinel and equal-key columns) with value ties across ranks; the shards are hashed, uneven, and empty."""
import os
import socket
import sys

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KKS = (0, 1, 2, 5, 32, 33, 70)


def cases():
    """(name, vals, ok, gid, n_groups, tie, owner [R] rank of each row, slots_max)"""
    from greptimedb_b200 import distributed as D
    from tests import select_keys as sk
    out = []
    rng = np.random.default_rng(0x70B)
    classes = ("equal", "signed-zero", "payloads", "sentinel-lo0", "sentinel-onlymax", "ulps-inf", "depth3-adjacent",
               "depth7-last", "top")
    sizes = [300, 90, 40, 33, 6, 1, 0, 70]
    vals, ok, gid, n_groups, _ = sk.grid(sizes, 37, 0.5, rng, classes=classes, drop=0.2, gid_gap=2, stray=5)
    R = gid.size
    tie = rng.permutation(R).astype(np.uint32)
    hashed = D.shard_of_series(np.arange(R, dtype=np.uint32), 2)
    out.append(("hashed", vals, ok, gid, n_groups, tie, hashed, 32))
    out.append(("hashed-3-slots", vals, ok, gid, n_groups, tie, hashed, 3))
    uneven = (rng.random(R) < 0.1).astype(np.int64)          # rank 1 holds a tenth
    out.append(("uneven", vals, ok, gid, n_groups, tie, uneven, 32))
    out.append(("rank-1-empty", vals, ok, gid, n_groups, tie, np.zeros(R, np.int64), 32))
    # equal values on both ranks: only the tie decides
    vals2 = np.where(rng.random(vals.shape) < 0.7, 1.0, vals)
    out.append(("value-ties", vals2, ok, gid, n_groups, tie, hashed, 32))
    return out


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from greptimedb_b200 import distributed as D
    res = {}
    for name, vals, ok, gid, n_groups, tie, owner, slots in cases():
        mine = np.flatnonzero(owner == rank)
        for bottom in (False, True):
            largest = int(np.bincount(gid[gid < n_groups], minlength=n_groups).max())
            for kk in KKS + (largest,):
                kept, X, rounds, K = D.merge_topk_candidates(bottom, kk, vals[mine], ok[mine], gid[mine], n_groups,
                                                             tie[mine], slots_max=slots)
                res[(name, bottom, kk)] = (mine, kept, X, rounds, K)
    q.put((rank, res))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_topk_union_equals_the_unsharded_selection():
    from tests import select_keys as sk
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    checked = 0
    for name, vals, ok, gid, n_groups, tie, owner, slots in cases():
        sizes = np.bincount(gid[gid < n_groups], minlength=n_groups)
        for bottom in (False, True):
            for kk in KKS + (int(sizes.max()),):
                exp = sk.topk(bottom, kk, vals, ok, gid, n_groups, tie)
                union = np.zeros_like(exp)
                for r in range(world):
                    mine, kept, X, rounds, K = got[r][(name, bottom, kk)]
                    union[mine] |= kept
                    assert X == (int((sizes > kk).sum()) if 0 < kk < sizes.max() else 0), (name, kk)
                    assert rounds == (0 if X == 0 else -(-kk // slots)), (name, kk)
                assert (union == exp).all(), (name, bottom, kk)
                checked += 1
    assert checked == 5 * 2 * 8
