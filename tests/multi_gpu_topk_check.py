"""Multi-rank check of the sharded topk / bottomk over the library's communicator (run under torchrun, one rank per
GPU; started by tests/test_multi_gpu.py when at least two GPUs are visible): rate() over series hash-sharded with
distributed.shard_rows, then b2p_topk_allgather_dev for k = 5 and k = 40 (rounds), with one group and by 7 groups; the
union of the ranks' kept cells == select_keys.topk over the oracle's full grid, bit for bit.  torch.distributed only
carries the 128-byte communicator id and the verdict."""
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
    ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, 1000, 1, 0x70B)
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    owned, rows, loffs = D.shard_rows(offsets, world, rank)
    T = N
    p = make_params("rate", T0, T0 + (N - 1) * 15_000, 15_000, 300_000)
    full_out, full_valid = orc.range_query(orc.make_params("rate", T0, T0 + (N - 1) * 15_000, 15_000, 300_000),
                                           ts, val, sid, offsets, threads=4)
    full_ok = sk.bits_of(full_valid, T)
    tie = np.random.default_rng(3).permutation(S).astype(np.uint32)   # distinct across every rank
    ns = int(owned.size)
    Tw = (T + 31) // 32
    out = torch.zeros(max(ns, 1) * T, dtype=torch.float64, device=dev)
    valid = torch.zeros(max(ns, 1) * Tw, dtype=torch.int32, device=dev)
    d_tie = torch.from_numpy(tie[owned].view(np.int32).copy() if ns else np.zeros(1, np.int32)).to(dev)
    torch.cuda.synchronize()
    if ns:
        d_ts, d_val = torch.from_numpy(ts[rows]).to(dev), torch.from_numpy(val[rows]).to(dev)
        d_off = torch.from_numpy(loffs.astype(np.int64)).to(dev)
        torch.cuda.synchronize()
        ctx.range_eval_dev(p, d_ts, d_val, d_off, rows.size, ns, out, valid)
        ctx.sync()
    bad = []
    for G in (1, 7):
        gid = (D.mix32(np.arange(S, dtype=np.uint32)) % np.uint32(G)).astype(np.uint32)
        d_gid = torch.from_numpy(gid[owned].view(np.int32).copy() if ns else np.zeros(1, np.int32)).to(dev)
        torch.cuda.synchronize()
        ix = ctx.group_index_create_dev(d_gid, ns, G)
        for op in ("topk", "bottomk"):
            for k in (5, 40):
                kept = torch.full_like(valid, -1)
                torch.cuda.synchronize()
                ctx.topk_allgather_dev(op, k, out, valid, ix, d_tie, T, kept)
                ctx.sync()
                exp = sk.words(sk.topk(op == "bottomk", k, full_out, full_ok, gid, G, tie))[owned]
                got = kept.cpu().numpy().view(np.uint32)[:ns]
                if not (got == exp).all():
                    bad.append(f"{op}({k}) by {G} groups: {int((got != exp).sum())} words differ on rank {rank}")
        ctx.group_index_destroy(ix)
    return bad


if __name__ == "__main__":
    rank_session("MULTI_GPU_TOPK_CHECK", main)
