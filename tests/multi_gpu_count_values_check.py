"""Multi-rank check of the sharded count_values over the library's communicator (run under torchrun, one rank per GPU;
started by tests/test_multi_gpu.py when at least two GPUs are visible): rate() over series hash-sharded
with distributed.shard_rows, rounded to a few distinct values, then b2p_count_values_dev over the rank's rows, the
heights' all-gather and b2p_count_values_allgather_dev with one group and by 7 groups; every rank's rows of group g ==
the first U_g rows of b2p_count_values_dev over the gathered rows (the oracle's full grid, rounded the same way, on one
GPU), bit for bit, and the rows past U_g have count 0.  After comm_destroy every rank runs the composed call over its
own rows as one rank of one, which must give b2p_count_values_dev's rows.  torch.distributed only carries the 128-byte
communicator id and the verdict."""
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

    S, N, T0 = 1200, 300, 1_700_000_000_000
    ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, 1000, 1, 0x9A1)
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    owned, rows, loffs = D.shard_rows(offsets, world, rank)
    T = N
    p = make_params("rate", T0, T0 + (N - 1) * 15_000, 15_000, 300_000)
    full_out, full_valid = orc.range_query(orc.make_params("rate", T0, T0 + (N - 1) * 15_000, 15_000, 300_000),
                                           ts, val, sid, offsets, threads=4)
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
    out = torch.round(out * 2.0) / 2.0  # a few distinct values per group and step
    g_vals = torch.round(torch.from_numpy(np.ascontiguousarray(full_out)).to(dev) * 2.0) / 2.0
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
        lv = torch.zeros(max(ns, 1) * T, dtype=torch.float64, device=dev)
        lc = torch.zeros(max(ns, 1) * T, dtype=torch.int32, device=dev)
        if ns:
            ctx.count_values_dev(out, valid, ix, T, lv, lc)
        H = ctx.count_values_shard_heights_dev(lc, ix, T, G, world)
        out_goff = ctx.count_values_shard_rows(H)
        U = int(out_goff[-1])
        o = torch.full((max(U, 1) * T,), -1.0, dtype=torch.float64, device=dev)
        c = torch.full((max(U, 1) * T,), -1, dtype=torch.int32, device=dev)
        e = torch.zeros(S * T, dtype=torch.float64, device=dev)
        ec = torch.zeros(S * T, dtype=torch.int32, device=dev)
        ctx.count_values_allgather_dev(lv, lc, ix, T, H, o, c)
        ctx.count_values_dev(g_vals, g_valid, ix_all, T, e, ec)
        ctx.sync()
        torch.cuda.synchronize()
        o, c = o.cpu().numpy()[:U * T].reshape(U, T), c.cpu().numpy().view(np.uint32)[:U * T].reshape(U, T)
        e, ec = e.cpu().numpy().reshape(S, T), ec.cpu().numpy().view(np.uint32).reshape(S, T)
        goff = np.searchsorted(np.sort(gid), np.arange(G + 1))
        sent = ctx.last_exchange_bytes()
        for g in range(G):
            u = out_goff[g + 1] - out_goff[g]
            if not (np.array_equal(o[out_goff[g]:out_goff[g + 1]].view(np.uint64), e[goff[g]:goff[g] + u].view(np.uint64))
                    and (c[out_goff[g]:out_goff[g + 1]] == ec[goff[g]:goff[g] + u]).all()
                    and (ec[goff[g] + u:goff[g + 1]] == 0).all()):
                bad.append(f"count_values by {G} groups differs in group {g} on rank {rank}")
        if sent <= 0:
            bad.append(f"exchange bytes {sent} on rank {rank}")
        ctx.group_index_destroy(ix)
        ctx.group_index_destroy(ix_all)
    # without a communicator every rank is rank 0 of one, whichever rank it had: the composed call over its own rows by
    # 7 groups gives count_values_dev's rows
    ctx.comm_destroy()
    G = 7
    gid = (D.mix32(np.arange(S, dtype=np.uint32)) % np.uint32(G)).astype(np.uint32)[owned]
    d_gid = torch.from_numpy(gid.view(np.int32).copy() if ns else np.zeros(1, np.int32)).to(dev)
    lv = torch.zeros(max(ns, 1) * T, dtype=torch.float64, device=dev)
    lc = torch.zeros(max(ns, 1) * T, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    ix = ctx.group_index_create_dev(d_gid, ns, G)
    if ns:
        ctx.count_values_dev(out, valid, ix, T, lv, lc)
    H = ctx.count_values_shard_heights_dev(lc, ix, T, G)
    out_goff = ctx.count_values_shard_rows(H)
    U = int(out_goff[-1])
    o = torch.full((max(U, 1) * T,), -1.0, dtype=torch.float64, device=dev)
    c = torch.full((max(U, 1) * T,), -1, dtype=torch.int32, device=dev)
    ctx.count_values_allgather_dev(lv, lc, ix, T, H, o, c)
    ctx.sync()
    torch.cuda.synchronize()
    ctx.group_index_destroy(ix)
    o, c = o.cpu().numpy()[:U * T].reshape(U, T), c.cpu().numpy().view(np.uint32)[:U * T].reshape(U, T)
    lv, lc = lv.cpu().numpy()[:ns * T].reshape(ns, T), lc.cpu().numpy().view(np.uint32)[:ns * T].reshape(ns, T)
    goff = np.searchsorted(np.sort(gid), np.arange(G + 1))
    for g in range(G):
        u = out_goff[g + 1] - out_goff[g]
        if not (np.array_equal(o[out_goff[g]:out_goff[g + 1]].view(np.uint64), lv[goff[g]:goff[g] + u].view(np.uint64))
                and (c[out_goff[g]:out_goff[g + 1]] == lc[goff[g]:goff[g] + u]).all()
                and (lc[goff[g] + u:goff[g + 1]] == 0).all()):
            bad.append(f"count_values without a communicator differs in group {g} on rank {rank}")
    return bad


if __name__ == "__main__":
    rank_session("MULTI_GPU_COUNT_VALUES_CHECK", main)
