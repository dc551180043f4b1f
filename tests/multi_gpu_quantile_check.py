"""Multi-rank check of the sharded quantile over the library's communicator (run under torchrun, one rank per GPU;
started by tests/test_multi_gpu.py when at least two GPUs are visible): rate() over series hash-sharded with
distributed.shard_rows, then b2p_quantile_allreduce_dev at several phi with one group and by 7 groups; every rank's
result == b2p_group_quantile_dev over the gathered rows (the oracle's full grid on one GPU), bit for bit, and the
counts == select_keys.quantile's.  torch.distributed only carries the 128-byte communicator id and the verdict."""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.ranks import rank_session  # noqa: E402


def main(s):
    rank, world, dev, ctx = s.rank, s.world, s.dev, s.ctx
    from greptimedb_b200 import make_params
    from greptimedb_b200 import distributed as D
    from oracle import oracle as orc
    from tests import select_keys as sk

    S, N, T0 = 1200, 300, 1_700_000_000_000
    ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, 1000, 1, 0x9A1)
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    owned, rows, loffs = D.shard_rows(offsets, world, rank)
    T = N
    p = make_params("rate", T0, T0 + (N - 1) * 15_000, 15_000, 300_000)
    full_out, full_valid = orc.range_query(orc.make_params("rate", T0, T0 + (N - 1) * 15_000, 15_000, 300_000),
                                           ts, val, sid, offsets, threads=4)
    full_ok = sk.bits_of(full_valid, T)
    ns = int(owned.size)
    Tw = (T + 31) // 32
    out = torch.zeros(max(ns, 1) * T, dtype=torch.float64, device=dev)
    valid = torch.zeros(max(ns, 1) * Tw, dtype=torch.int32, device=dev)
    if ns:
        d_ts, d_val = torch.from_numpy(ts[rows]).to(dev), torch.from_numpy(val[rows]).to(dev)
        d_off = torch.from_numpy(loffs.astype(np.int64)).to(dev)
        torch.cuda.synchronize()
        ctx.range_eval_dev(p, d_ts, d_val, d_off, rows.size, ns, out, valid)
        ctx.sync()
    # the gathered rows: the oracle's full grid on this GPU, one index over all of them
    g_vals = torch.from_numpy(np.ascontiguousarray(full_out)).to(dev)
    g_valid = torch.from_numpy(np.ascontiguousarray(full_valid).view(np.int32)).to(dev)
    torch.cuda.synchronize()
    bad = []
    for G in (1, 7):
        gid = (D.mix32(np.arange(S, dtype=np.uint32)) % np.uint32(G)).astype(np.uint32)
        d_gid = torch.from_numpy(gid[owned].view(np.int32).copy() if ns else np.zeros(1, np.int32)).to(dev)
        a_gid = torch.from_numpy(gid.view(np.int32).copy()).to(dev)
        torch.cuda.synchronize()
        ix = ctx.group_index_create_dev(d_gid, ns, G)
        ix_all = ctx.group_index_create_dev(a_gid, S, G)
        for phi in (0.0, 0.5, 0.9, 0.99, 1.0, math.nan):
            o = torch.full((G * T,), -1.0, dtype=torch.float64, device=dev)
            c = torch.full((G * T,), -1, dtype=torch.int32, device=dev)
            e = torch.full_like(o, -1.0)
            ec = torch.full_like(c, -1)
            torch.cuda.synchronize()
            ctx.quantile_allreduce_dev(phi, out, valid, ix, T, o, c)
            ctx.group_quantile_dev(phi, g_vals, g_valid, ix_all, T, e, ec)
            ctx.sync()
            torch.cuda.synchronize()
            _, exp_cnt = sk.quantile(phi, full_out, full_ok, gid, G)
            if not (sk.same_bits(o.cpu().numpy(), e.cpu().numpy()) and torch.equal(c, ec)
                    and (c.cpu().numpy().view(np.uint32).reshape(G, T) == exp_cnt).all()):
                bad.append(f"quantile({phi}) by {G} groups differs on rank {rank}")
        ctx.group_index_destroy(ix)
        ctx.group_index_destroy(ix_all)
    return bad


if __name__ == "__main__":
    rank_session("MULTI_GPU_QUANTILE_CHECK", main)
