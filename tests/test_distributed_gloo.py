"""World-size-2 gloo test (CPU) of the N>1 host logic: hash-sharding of series, per-rank partial
(sum, cnt), one all-reduce, finalize == unsharded result.  The per-shard compute is the oracle here
(the CUDA kernels need a GPU; tests/test_gpu_parity.py covers them)."""
import numpy as np
import torch

from tests.ranks import spawn_gloo


def _worker(rank, world):
    from greptimedb_b200 import distributed as D
    from oracle import oracle as orc
    S, N, G, T0 = 96, 200, 7, 1_700_000_000_000
    ts, val, sid = orc.synth_fill(0, S, N, T0, 15_000, 1000, 1, 0x5EED)
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    gid = (D.mix32(np.arange(S, dtype=np.uint32)) % np.uint32(G)).astype(np.uint32)
    p = orc.make_params("rate", T0, T0 + (N - 1) * 15_000, 15_000, 300_000)
    owned, rows, loffs = D.shard_rows(offsets, world, rank)
    out, valid = orc.range_query(p, ts[rows], val[rows], None, loffs)
    psum, pcnt = orc.group_aggregate("sum", out, valid, gid[owned], G)
    st, ct = torch.from_numpy(psum), torch.from_numpy(pcnt.astype(np.int64))
    D.allreduce_group_partials(st, ct)
    res = D.finalize_host("avg", st.numpy(), ct.numpy())
    full_out, full_valid = orc.range_query(p, ts, val, sid, offsets)
    worst = 0.0
    ok_all = True
    # min / max: groups missing on one rank must not poison the extreme; stddev / stdvar: (cnt, mean, M2) states merge
    for agg in ("min", "max", "stddev", "stdvar"):
        e_val, e_cnt = orc.group_aggregate(agg, full_out, full_valid, gid, G)
        if agg in ("min", "max"):
            pv, pc = orc.group_aggregate(agg, out, valid, gid[owned], G)
            vt, ctt = torch.from_numpy(pv.copy()), torch.from_numpy(pc.astype(np.int64))
            D.merge_partials(agg, vt, ctt)
            got = vt.numpy()
        else:
            m2, pc, mean = D.partial_state_host(agg, out, valid, gid[owned], G)
            vt, ctt, mt = torch.from_numpy(m2), torch.from_numpy(pc), torch.from_numpy(mean)
            D.merge_partials(agg, vt, ctt, mt)
            n = np.maximum(ctt.numpy(), 1)
            got = vt.numpy() / n if agg == "stdvar" else np.sqrt(vt.numpy() / n)
            got[ctt.numpy() == 0] = 0.0
        ok_all = ok_all and bool((ctt.numpy() == e_cnt).all())
        m = e_cnt > 0
        rel_a = np.abs(got[m] - e_val[m]) / np.maximum(np.abs(e_val[m]), 1e-300)
        # variance of near-constant samples cancels: compare absolutely against the scale of the data there
        scale = np.abs(full_out).max()
        bad = (rel_a > 1e-9) & (np.abs(got[m] - e_val[m]) > 1e-9 * scale)
        ok_all = ok_all and not bool(bad.any())
        if agg in ("min", "max"):
            ok_all = ok_all and bool((got[m] == e_val[m]).all())   # extremes are exact
    if rank == 0:
        e_avg, e_cnt = orc.group_aggregate("avg", full_out, full_valid, gid, G)
        ok_cnt = bool((ct.numpy() == e_cnt).all()) and ok_all
        rel = np.abs(res - e_avg) / np.maximum(np.abs(e_avg), 1e-300)
        return ok_cnt, float(rel[e_cnt > 0].max()), int(owned.size)
    return ok_all, 0.0, int(owned.size)


def _worker_total_order(rank, world):
    from greptimedb_b200 import distributed as D
    from oracle import oracle as orc
    from tests.helpers import total_order_case
    vals, valid, gid, G = total_order_case()
    mine = slice(rank * G, (rank + 1) * G)
    bad = []
    for agg in ("min", "max"):
        e_val, e_cnt = orc.group_aggregate(agg, vals, valid, gid, G)
        pv, pc = orc.group_aggregate(agg, vals[mine], valid[mine], gid[mine], G)
        vt, ct = torch.from_numpy(pv.copy()), torch.from_numpy(pc.astype(np.int64))
        D.merge_partials(agg, vt, ct)
        got = vt.numpy()
        if not (ct.numpy() == e_cnt).all():
            bad.append(f"{agg}: counts differ")
        diff = np.argwhere(got.view(np.uint64) != e_val.view(np.uint64))
        for g, k in diff[:4]:
            bad.append(f"{agg} group {g} step {k}: merged {got[g, k]!r} ({got[g, k:k + 1].view(np.uint64)[0]:#x}), "
                       f"single pass {e_val[g, k]!r} ({e_val[g, k:k + 1].view(np.uint64)[0]:#x})")
    return not bad, "; ".join(bad), 0


def test_min_max_merge_follows_the_total_order_across_ranks():
    """NaN (both signs, with and without payload), -0.0 and +0.0 members of one group on different ranks, in every
    placement order: the merged min / max equals the single-pass total-order aggregate bit for bit, and a group absent on
    one rank or on both merges like the single pass too (the neutral element, then 0.0)."""
    for ok, msg, _ in spawn_gloo(_worker_total_order):
        assert ok, msg


def test_sharded_partials_allreduce_equals_unsharded():
    world = 2
    results = spawn_gloo(_worker, world)
    assert all(r[0] for r in results)
    assert max(r[1] for r in results) <= 1e-9          # summation order differs across shards: 1e-9 rel, like the reference
    assert sum(r[2] for r in results) == 96              # every series owned exactly once


def test_shard_function_is_a_partition():
    from greptimedb_b200 import distributed as D
    ids = np.arange(10_000, dtype=np.uint32)
    for world in (1, 2, 4, 8):
        own = D.shard_of_series(ids, world)
        assert own.min() >= 0 and own.max() < world
        counts = np.bincount(own, minlength=world)
        assert counts.sum() == ids.size and counts.min() > 0.8 * ids.size / world
