"""Multi-rank check of the sharded histogram_quantile over the library's communicator (run under torchrun, one rank per
GPU; started by tests/test_multi_gpu_histogram.py when at least two GPUs are visible).  Bucket rows sharded by series
hash (histograms split across ranks) and by histogram (each whole on one rank), a rank without rows: every rank's
b2p_histogram_fold_allgather equals the host mirror (distributed.histogram_fold_sharded over torch.distributed) and
b2p_histogram_fold over every rank's rows in rank order on one GPU, bit for bit, and is the same on every rank.  By
histogram no bucket row moves.  Through the plan layer, a sharded HistogramQuantilePlan and a sharded leaf export the
same bytes on every rank; an Int64 rank beside a rank without rows is refused on every rank."""
import os
import sys
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.ranks import rank_session  # noqa: E402


def main(s):
    import pyarrow as pa
    import torch.distributed as dist
    from greptimedb_b200 import B2PError
    from greptimedb_b200 import distributed as D
    from greptimedb_b200.plan import HistogramQuantilePlan
    from tests.test_gpu_histogram_node import END, HISTS, LES, START, STEP, histograms, leaf
    from tests.test_gpu_histogram_sharded import bucket_rows, unsharded_fold

    rank, world, ctx = s.rank, s.world, s.ctx
    bad = []
    rates, words, hist, le = bucket_rows(np.random.default_rng(17), n_hist=60, T=200)
    H = int(hist.max()) + 1
    T = rates.shape[1]
    ok_bits = np.unpackbits(words.view(np.uint8), axis=1, bitorder="little")[:, :T].astype(bool)

    def same_everywhere(a):
        got = D._all_gather(np.ascontiguousarray(a).view(np.uint8).reshape(-1), None)
        return all(np.array_equal(g, got[0]) for g in got)

    for layout in ("series", "histogram"):
        rng = np.random.default_rng(5)
        rank_of_row = rng.integers(0, world, hist.size) if layout == "series" else rng.integers(0, world, H)[hist]
        if world > 2:
            rank_of_row[rank_of_row == 1] = 0  # rank 1 holds no rows
        mine = np.flatnonzero(rank_of_row == rank)
        order = np.argsort(rank_of_row, kind="stable")
        want_v, want_w = unsharded_fold(ctx, 0.9, rates[order], words[order], hist[order], le[order], H)
        got_v, got_w = ctx.histogram_fold_allgather(0.9, rates[mine], words[mine], hist[mine], le[mine], H)
        sent = ctx.last_exchange_bytes()
        m_v, m_ok, m_sent = D.histogram_fold_sharded(0.9, rates[mine], ok_bits[mine], hist[mine], le[mine], H)
        if not (np.array_equal(got_w, want_w) and np.array_equal(got_v.view(np.uint64), want_v.view(np.uint64))):
            bad.append(f"rank {rank} {layout}: differs from the fold over the concatenation")
        got_ok = np.unpackbits(got_w.view(np.uint8), axis=1, bitorder="little")[:, :T].astype(bool)
        if not (np.array_equal(got_ok, m_ok) and np.allclose(got_v[m_ok], m_v[m_ok], rtol=1e-12, equal_nan=True)):
            bad.append(f"rank {rank} {layout}: differs from the host mirror")
        if not (same_everywhere(got_v) and same_everywhere(got_w)):
            bad.append(f"rank {rank} {layout}: the ranks' results differ")
        if sent != m_sent:
            bad.append(f"rank {rank} {layout}: sent {sent} B, the mirror {m_sent} B")
        counts = np.stack([np.bincount(hist[rank_of_row == r], minlength=H) for r in range(world)])
        own = int(np.count_nonzero(D.histogram_owners(counts) == rank))
        if layout == "histogram" and sent != own * (8 * T + 4 * ((T + 31) // 32)):
            bad.append(f"rank {rank} histogram: bucket rows were sent")
        s.note += f"{layout}:rank{rank}_sent={sent} "

    # the plan layer: every rank's shard of the bucket series, one histogram split across ranks
    batch = histograms(np.random.default_rng(9), HISTS, LES, 90, missing=0.1)
    tags = ["job", "instance", "le"]
    labels = zip(*[batch.column(t).to_pylist() for t in tags])
    keep = [zlib.crc32("/".join(map(str, x)).encode()) % world == rank for x in labels]  # by series hash
    part = batch.filter(pa.array(keep))
    node = HistogramQuantilePlan(ctx, 0.9, leaf(ctx, part, tags, START, END, STEP)).sharded().execute()
    fused = leaf(ctx, part, tags, START, END, STEP, histogram_quantile=0.9).sharded().execute()
    for name, b in (("node", node), ("leaf", fused)):
        cols = [np.asarray(c.to_numpy(zero_copy_only=False), np.float64) for c in b.columns
                if pa.types.is_floating(c.type)]
        if b.num_rows == 0 or not all(same_everywhere(c) for c in cols):
            bad.append(f"rank {rank} plan {name}: the ranks' exports differ")
    # an Int64 rank beside a rank without rows: refused on every rank, none left in a collective
    from greptimedb_b200.plan import PromRangeExec
    ex = PromRangeExec(ctx, "", START, START, STEP, 0, "ts", "val", ["job", "le"], lookback_delta=STEP)
    if rank == 0:
        ex.push(pa.RecordBatch.from_pydict({"ts": pa.array([START, START], pa.timestamp("ms")),
                                            "val": pa.array([1, 2], pa.int64()), "job": ["a", "a"],
                                            "le": ["1", "+Inf"]}))
    try:
        HistogramQuantilePlan(ctx, 0.5, ex).sharded().execute()
        bad.append(f"rank {rank}: the Int64 rank was not refused")
    except B2PError as e:
        if "Int64" not in str(e):
            bad.append(f"rank {rank}: refused with {e}")
    dist.barrier()
    return bad


if __name__ == "__main__":
    rank_session("MULTI_GPU_HISTOGRAM_CHECK", main)
