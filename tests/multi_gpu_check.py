"""Multi-rank check of the library's own collective path (run under torchrun, one rank per GPU; started by
tests/test_multi_gpu.py when at least two GPUs are visible):

  * sum by (..)(rate(..)) with series hash-sharded over the ranks, through b2p_range_group_sum_allreduce_dev (fused
    partials, tiles all-reduced on the library's NCCL communicator) == the oracle on the unsharded data;
  * b2p_allreduce_partials_dev for min / max and for the (count, mean, M2) states of stddev / stdvar == the oracle.
torch.distributed only carries the 128-byte communicator id and the final verdict."""
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

    S, N, G, T0 = 2400, 500, 61, 1_700_000_000_000
    ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, 1000, 1, 0x5EED)
    val[77::4001] = np.nan
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    gid = (D.mix32(np.arange(S, dtype=np.uint32)) % np.uint32(G)).astype(np.uint32)
    owned, rows, loffs = D.shard_rows(offsets, world, rank)
    T = N
    p = make_params("rate", T0, T0 + (N - 1) * 15_000, 15_000, 300_000)
    op = orc.make_params("rate", T0, T0 + (N - 1) * 15_000, 15_000, 300_000)
    full_out, full_valid = orc.range_query(op, ts, val, sid, offsets, threads=4)
    ok, worst = True, 0.0

    d_ts, d_val = torch.from_numpy(ts[rows]).to(dev), torch.from_numpy(val[rows]).to(dev)
    d_off = torch.from_numpy(loffs.astype(np.int64)).to(dev)
    d_gid = torch.from_numpy(gid[owned].astype(np.int32)).to(dev)
    torch.cuda.synchronize()
    ns = int(owned.size)
    ix = ctx.group_index_create_dev(d_gid, ns, G)
    e_sum, e_cnt = orc.group_aggregate("sum", full_out, full_valid, gid, G)
    for tiles in (1, 3):
        gsum = torch.zeros(G * T, dtype=torch.float64, device=dev)
        gcnt = torch.zeros(G * T, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()   # the library runs on its own stream: the zero fills must land first
        ctx.range_group_sum_allreduce_dev(p, d_ts, d_val, d_off, rows.size, ns, ix, tiles, gsum, gcnt)
        ctx.sync()
        got, cnt = gsum.cpu().numpy().reshape(G, T), gcnt.cpu().numpy().view(np.uint32).reshape(G, T)
        ok = ok and bool((cnt == e_cnt).all())
        rel = np.abs(got - e_sum) / np.maximum(np.abs(e_sum), 1e-300)
        worst = max(worst, float(rel[e_cnt > 0].max()))
    ctx.group_index_destroy(ix)

    # min / max / stddev / stdvar: per-rank partial state from the by-label kernel, merged by the library
    out = torch.zeros(ns * T, dtype=torch.float64, device=dev)
    valid = torch.zeros(ns * ((T + 31) // 32), dtype=torch.int32, device=dev)
    ctx.range_eval_dev(p, d_ts, d_val, d_off, rows.size, ns, out, valid)
    ctx.sync()
    scale = float(np.abs(full_out).max())
    for agg in ("min", "max", "stddev", "stdvar", "avg"):
        e_val, e_c = orc.group_aggregate(agg, full_out, full_valid, gid, G)
        pv = torch.zeros(G * T, dtype=torch.float64, device=dev)
        pc = torch.zeros(G * T, dtype=torch.int32, device=dev)
        pm = torch.zeros(G * T, dtype=torch.float64, device=dev)
        var = agg in ("stddev", "stdvar")
        torch.cuda.synchronize()   # the library runs on its own stream: the zero fills must land first
        ctx.group_aggregate_partial_dev(agg, out, valid, d_gid, ns, G, T, pv, pc, pm if var else None)
        ctx.allreduce_partials_dev(agg, pv, pc, pm if var else None, G * T)
        if agg in ("stddev", "stdvar", "avg"):
            ctx.group_finalize_dev(agg, pv, pc, G * T)
        ctx.sync()
        got, cnt = pv.cpu().numpy().reshape(G, T), pc.cpu().numpy().view(np.uint32).reshape(G, T)
        ok = ok and bool((cnt == e_c).all())
        m = e_c > 0
        if agg in ("min", "max"):
            ok = ok and bool((got[m] == e_val[m]).all())
        else:
            err = np.abs(got[m] - e_val[m])
            bad = (err > 1e-9 * np.maximum(np.abs(e_val[m]), 1e-300)) & (err > 1e-9 * scale)
            ok = ok and not bool(bad.any())

    # min / max in the total order: NaN (both signs, with a payload) and +-0.0 members of one group on ranks 0 and 1 in
    # every placement order, groups absent on one rank or everywhere; other ranks hold no member.  Bit for bit.
    from tests.helpers import total_order_case
    tv, tvalid, tgid, TG = total_order_case()
    mine = slice(rank * TG, (rank + 1) * TG) if rank < 2 else slice(0, 0)
    n_mine = mine.stop - mine.start
    TT = tv.shape[1]
    d_tv = torch.from_numpy(np.ascontiguousarray(tv[mine]) if n_mine else np.zeros((1, TT))).to(dev)
    d_tvalid = torch.from_numpy((tvalid[mine] if n_mine else np.zeros((1, 1), np.uint32)).astype(np.int32)).to(dev)
    d_tgid = torch.from_numpy((tgid[mine] if n_mine else np.zeros(1, np.uint32)).astype(np.int32)).to(dev)
    torch.cuda.synchronize()
    for agg in ("min", "max"):
        e_val, e_c = orc.group_aggregate(agg, tv, tvalid, tgid, TG)
        pv = torch.zeros(TG * TT, dtype=torch.float64, device=dev)
        pc = torch.zeros(TG * TT, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()   # the library runs on its own stream: the zero fills must land first
        if n_mine:
            ctx.group_aggregate_partial_dev(agg, d_tv, d_tvalid, d_tgid, n_mine, TG, TT, pv, pc, None)
        ctx.allreduce_partials_dev(agg, pv, pc, None, TG * TT)
        ctx.sync()
        got, cnt = pv.cpu().numpy().reshape(TG, TT), pc.cpu().numpy().view(np.uint32).reshape(TG, TT)
        ok = ok and bool((cnt == e_c).all()) and bool((got.view(np.uint64) == e_val.view(np.uint64)).all())
    s.note = f"worst_rel={worst:.3e}"
    return [] if ok and worst <= 1e-9 else [f"rank {rank}: counts or values differ, worst_rel={worst:.3e}"]


if __name__ == "__main__":
    rank_session("MULTI_GPU_CHECK", main)
