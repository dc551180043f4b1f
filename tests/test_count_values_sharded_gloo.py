"""World-size-2 gloo test (CPU) of the sharded count_values: every rank holds whole series and its own count_values
output (select_keys.count_values over its rows), the host mirror of b2p_count_values_allgather_dev
(distributed.merge_count_values) all-gathers the heights and each rank's (key, count) entries, and both ranks' merged
rows equal the first U_g rows of each group of select_keys.count_values over all rows, bit for bit; the rows past U_g
have count 0.  Classes: hashed, uneven and empty shards; the same values on both ranks and disjoint values; ±0.0 and NaN
payloads split across ranks; the largest positive NaN on one rank only; a group present on one rank only."""
import os
import socket
import sys

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_NAN = 0x7FFFFFFFFFFFFFFF


def _bits(x):
    return np.array(x, np.uint64).view(np.float64)


def cases():
    """(name, vals, ok, gid, n_groups, owner [R] rank of each row)"""
    from greptimedb_b200 import distributed as D
    from tests import select_keys as sk
    out = []
    rng = np.random.default_rng(0xC0)
    T = 37
    vals, ok, gid, n_groups, _ = sk.grid([70, 40, 33, 9, 2, 1, 0, 120], T, 0.5, rng, drop=0.2, gid_gap=2, stray=5)
    vals[rng.random(vals.shape) < 0.4] = 1.5                       # repeated values
    ok[rng.random(gid.size) < 0.05] = False                        # rows without a valid cell
    R = gid.size
    out.append(("hashed", vals, ok, gid, n_groups, D.shard_of_series(np.arange(R, dtype=np.uint32), 2)))
    out.append(("uneven", vals, ok, gid, n_groups, (rng.random(R) < 0.1).astype(np.int64)))
    out.append(("rank-1-empty", vals, ok, gid, n_groups, np.zeros(R, np.int64)))

    # the same few values on both ranks, and disjoint values (rank 0 negative, rank 1 positive)
    R, T = 60, 5
    gid = (np.arange(R) % 3).astype(np.uint32)
    own = (np.arange(R) // 3 % 2).astype(np.int64)
    same = rng.choice([-2.0, 0.5, 7.0, 1e300], (R, T))
    out.append(("same-values", same, np.ones((R, T), bool), gid, 3, own))
    disjoint = np.where(own[:, None] == 0, -1.0, 1.0) * rng.integers(1, 6, (R, T))
    out.append(("disjoint-values", disjoint, rng.random((R, T)) < 0.9, gid, 3, own))

    # ±0.0 and NaN payloads split across ranks, the largest positive NaN (the filler's key) on one rank only
    pay = [0x7FF0000000000001, 0x7FF8000000000000, 0xFFF8000000000000, 0xFFF0000000000123, 0x8000000000000000, 0]
    R, T = 40, 33
    gid = (np.arange(R) % 2).astype(np.uint32)
    own = (np.arange(R) // 2 % 2).astype(np.int64)
    nan = _bits(np.array(pay, np.uint64)[rng.integers(0, len(pay), (R, T))])
    out.append(("zeros-and-payloads", nan, rng.random((R, T)) < 0.8, gid, 2, own))
    top = nan.copy()
    top[(own == 1)[:, None] & (rng.random((R, T)) < 0.5)] = _bits(MAX_NAN)
    out.append(("largest-nan-one-rank", top, rng.random((R, T)) < 0.85, gid, 2, own))
    only = _bits(np.full((R, T), MAX_NAN, np.uint64))
    out.append(("only-largest-nan", only, rng.random((R, T)) < 0.5, gid, 2, own))

    # a group present on one rank only, and rows of no group
    R, T = 30, 7
    gid = np.array([0] * 10 + [1] * 10 + [2] * 6 + [9] * 4, np.uint32)
    own = np.array([0] * 10 + [0, 1] * 5 + [1] * 6 + [0, 1] * 2, np.int64)
    out.append(("group-on-one-rank", rng.integers(0, 4, (R, T)).astype(np.float64), rng.random((R, T)) < 0.7, gid, 3,
                own))
    return out


def local_heights(vals, ok, gid, n_groups, mine):
    """h_r(g) of the rows `mine`: 1 + the last row of each group in their count_values output with a count"""
    from tests import select_keys as sk
    _, cnt = sk.count_values(vals[mine], ok[mine], gid[mine], n_groups)
    _, goff = sk._groups(gid[mine], n_groups)
    h = np.zeros(n_groups, np.int64)
    for g in range(n_groups):
        rows = np.flatnonzero(cnt[goff[g]:goff[g + 1]].any(axis=1))
        h[g] = rows[-1] + 1 if rows.size else 0
    return h


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from greptimedb_b200 import distributed as D
    from tests import select_keys as sk
    res = []
    for name, vals, ok, gid, n_groups, owner in cases():
        mine = np.flatnonzero(owner == rank)
        lv, lc = sk.count_values(vals[mine], ok[mine], gid[mine], n_groups)
        res.append(D.merge_count_values(lv, lc, np.sort(gid[mine]), n_groups))
    q.put((rank, res))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_count_values_equals_the_unsharded_count():
    from greptimedb_b200 import distributed as D
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
    got = dict(q.get(timeout=600) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for i, (name, vals, ok, gid, n_groups, owner) in enumerate(cases()):
        exp, exp_cnt = sk.count_values(vals, ok, gid, n_groups)
        (o0, c0, u0, b0), (o1, c1, u1, b1) = got[0][i], got[1][i]
        assert sk.same_bits(o0, o1) and (c0 == c1).all() and (u0 == u1).all() and b0 == b1, name
        _, goff = sk._groups(gid, n_groups)
        for g in range(n_groups):
            U = u0[g + 1] - u0[g]
            assert U <= goff[g + 1] - goff[g], name
            assert sk.same_bits(o0[u0[g]:u0[g + 1]], exp[goff[g]:goff[g] + U]), (name, g)
            assert (c0[u0[g]:u0[g + 1]] == exp_cnt[goff[g]:goff[g] + U]).all(), (name, g)
            assert (exp_cnt[goff[g] + U:goff[g + 1]] == 0).all(), (name, g)
        assert (exp_cnt[goff[n_groups]:] == 0).all(), name
        heights = np.array([local_heights(vals, ok, gid, n_groups, owner == r) for r in range(world)])
        assert (u0 == np.concatenate([[0], np.cumsum(heights.sum(axis=0))])).all(), name
        assert b0 == heights.sum(axis=1).max() * vals.shape[1] * D.CV_ENTRY_BYTES, name
    names = [c[0] for c in cases()]
    assert "largest-nan-one-rank" in names and len(names) == 9
