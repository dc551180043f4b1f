"""Times histogram_quantile over any node (HistogramQuantilePlan, b2p_histogram_fold, K5) through the plan layer.

Data: --hists histograms (default 100 k, one job each, --instances per job) of 64 buckets, seeded counters scraped every
60 s, evaluated on --steps steps 60 s apart with a 5 m range, pushed as one Arrow batch.  It prints one JSON line per
query, with the card's name and power limit read in the same run.

A plan call is compute then export.  `compute_ms(x)` times the compute of x alone: it executes
histogram_quantile(x) with an le column x lacks, which runs x and returns an empty batch with no columns, so nothing is
exported.  The index build is then the compute of the node minus the compute of its child minus b2p_histogram_fold
over the child's grid and the node's index; the three terms cover the same work except the index build.  Each rep
takes the three in turn, and the difference is formed per rep (median, min and max over the reps are printed).

  1. histogram_quantile(0.99, sum by (le, job)(rate(x_bucket[5m]))):
     - k5_ms: the K5 fold kernel alone on the device-resident [64 H x T] child grid (CUDA events of the fold stage);
     - host_fold_call_ms: b2p_histogram_fold on the child's grid from host memory (copies and K5);
     - child_compute_ms, node_compute_ms: compute of the aggregate child, and of the node (child, index build, fold);
     - index_build_ms: node_compute - child_compute - host_fold_call, per rep;
     - node_ms: the node end to end (compute, the export of its [H x T] result and the import into pyarrow).
  2. histogram_quantile(0.99, rate(x_bucket[5m])) two ways, alternated in one loop: the fused leaf
     (b2p_range_histogram_fold: the [S x T] bucket grid never leaves the device) and the node over a plain range leaf
     (the grid comes to the host and goes back), both end to end; and the node's index build over the leaf's rows,
     measured as in 1.

The first rep of every loop is a warm-up and is not counted; host times end in a synchronise (each plan call is
synchronous).

  python profiles/histogram_bench.py [--hists H] [--instances I] [--steps T] [--reps R]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from binary_bench import gpu_identity  # noqa: E402

BUCKETS, SCRAPE, RANGE, PHI = 64, 60_000, 300_000, 0.99


def make_batch(np, pa, H, I, T, seed):
    """One batch, series after series (job, instance, le), each with the samples the T windows need"""
    n = RANGE // SCRAPE + T
    les = [f"{0.001 * 1.25 ** b:.4g}" for b in range(BUCKETS - 1)] + ["+Inf"]
    S = H * I * BUCKETS
    rng = np.random.default_rng(seed)
    inc = rng.random((H * I, BUCKETS)).cumsum(axis=1).reshape(S, 1)  # per-scrape increase, cumulative over le
    val = (inc * np.arange(1, n + 1)).reshape(-1)
    ts = np.tile(np.arange(n, dtype=np.int64) * SCRAPE, S)
    series = np.repeat(np.arange(S), n)
    job = pa.array([f"j{h}" for h in range(H)]).take(pa.array(series // (I * BUCKETS)))
    inst = pa.array([f"i{i}" for i in range(I)]).take(pa.array((series // BUCKETS) % I))
    le = pa.array(les).take(pa.array(series % BUCKETS))
    return pa.RecordBatch.from_arrays([pa.array(ts, pa.timestamp("ms")), pa.array(val), job, inst, le],
                                      ["ts", "val", "job", "instance", "le"]), n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hists", type=int, default=100_000)
    ap.add_argument("--instances", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import pyarrow as pa
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("histogram_bench needs a CUDA device")
    from greptimedb_b200 import Context
    from greptimedb_b200.plan import AggregatePlan, HistogramQuantilePlan, PromRangeExec
    from oracle import oracle as orc

    ident = gpu_identity()
    ctx = Context(0)
    H, I, T = args.hists, args.instances, args.steps
    batch, n = make_batch(np, pa, H, I, T, 0x5EED)
    start = RANGE
    end = start + (T - 1) * SCRAPE
    tags = ["job", "instance", "le"]

    def leaf(**kw):
        node = PromRangeExec(ctx, "prom_rate", start, end, SCRAPE, RANGE, "ts", "val", tags, **kw)
        node.push(batch)
        return node

    plain, fused = leaf(), leaf(histogram_quantile=PHI)
    del batch
    shape = {"histograms": H, "instances_per_job": I, "buckets": BUCKETS, "steps": T, "samples_per_series": n}

    def timed(call):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = call()
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3, out

    def report(query, **numbers):
        print(json.dumps({"query": query, **shape, **{k: round(v, 3) for k, v in numbers.items()}, **ident}), flush=True)

    def progress(msg):  # one line per timed call on stderr: a long run keeps showing that it is alive
        print(msg, file=sys.stderr, flush=True)

    def compute_only(x):  # histogram_quantile(x) over an le column x lacks: x's compute, an empty export
        return HistogramQuantilePlan(ctx, PHI, x, le="__absent__").execute

    def fold_inputs(b, value, le_col, group_cols):
        """An exported batch whose rows are the grid's rows, T cells each, all valid -> (grid, words, index) as the
        node builds its index: rows grouped by the tags without le, buckets by numeric le"""
        R = b.num_rows // T
        assert b.num_rows == R * T
        grid = np.asarray(b.column(b.schema.names.index(value))).reshape(R, T)
        words = np.packbits(np.ones((R, Tw * 32), bool) & (np.arange(Tw * 32) < T), axis=1, bitorder="little")
        words = np.ascontiguousarray(words).view(np.uint32)
        first = pa.array(np.arange(0, R * T, T))
        le_codes = b.column(b.schema.names.index(le_col)).take(first).dictionary_encode()
        le_num = np.array([orc.parse_f64_rust(x) for x in le_codes.dictionary.to_pylist()])[np.asarray(le_codes.indices)]
        keys = [np.asarray(b.column(b.schema.names.index(c)).take(first).dictionary_encode().indices) for c in group_cols]
        order = np.lexsort([le_num] + keys[::-1]).astype(np.uint32)
        G = R // BUCKETS
        return grid, words, (np.arange(G + 1) * BUCKETS).astype(np.uint32), order, le_num[order]

    def index_build(child_x, node_x, fold_call, extra=None):
        """per rep: compute of node_x - compute of child_x - fold_call; the first rep is a warm-up"""
        cc, nc, fc, diff = [], [], [], []
        for _ in range(args.reps + 1):
            if extra:
                extra()
            fc.append(timed(fold_call)[0])
            cc.append(timed(compute_only(child_x))[0])
            nc.append(timed(compute_only(node_x))[0])
            diff.append(nc[-1] - cc[-1] - fc[-1])
            progress(f"rep: fold call {fc[-1]:.1f} ms, child compute {cc[-1]:.1f} ms, node compute {nc[-1]:.1f} ms")
        d = diff[1:]
        return {"host_fold_call_ms": med(fc), "child_compute_ms": med(cc), "node_compute_ms": med(nc),
                "index_build_ms": float(np.median(d)), "index_build_ms_min": min(d), "index_build_ms_max": max(d)}

    med = lambda v: float(np.median(v[1:]))
    Tw = (T + 31) // 32

    # 1. histogram_quantile(0.99, sum by (le, job)(rate(x_bucket[5m])))
    child = AggregatePlan(ctx, "sum", plain, by=["le", "job"])
    node = HistogramQuantilePlan(ctx, PHI, child)
    progress(f"data pushed: {H} histograms x {BUCKETS} buckets x {n} samples")
    c_batch = child.execute()  # the child's grid: groups in (le, job) order, every cell valid
    assert c_batch.num_rows == H * BUCKETS * T
    grid, words, hist_off, order, bucket_le = fold_inputs(c_batch, "sum(prom_rate(ts_range,val))", "le", ["job"])
    del c_batch
    d = lambda a: torch.from_numpy(np.array(a.view(np.int32) if a.dtype == np.uint32 else a)).cuda()
    d_grid, d_words, d_off, d_bs, d_le = d(grid), d(words), d(hist_off), d(order), d(bucket_le)
    out = torch.empty((H, T), dtype=torch.float64, device="cuda")
    ov = torch.empty((H, Tw), dtype=torch.int32, device="cuda")
    k5 = []

    def k5_call():
        ctx.histogram_fold_dev(PHI, d_off, d_bs, d_le, H, d_grid, d_words, T, out, ov)
        ctx.sync()
        k5.append(ctx.kernel_ms(3))

    numbers = index_build(child, node, lambda: ctx.histogram_fold(PHI, hist_off, order, bucket_le, grid, words),
                          extra=k5_call)
    node_ms = []
    for _ in range(args.reps + 1):
        node_ms.append(timed(node.execute)[0])
        progress(f"node end to end {node_ms[-1]:.1f} ms")
    report("histogram_quantile(0.99, sum by (le, job)(rate(x_bucket[5m])))", k5_ms=med(k5), **numbers,
           node_ms=med(node_ms))
    del d_grid, d_words, grid, words, child, node
    torch.cuda.empty_cache()

    # 2. histogram_quantile(0.99, rate(x_bucket[5m])): the fused leaf and the node over a plain leaf, alternated
    over_leaf = HistogramQuantilePlan(ctx, PHI, plain)
    a_out, b_out = fused.execute(), over_leaf.execute()  # (warm-up; the two agree bit for bit)
    assert np.asarray(a_out.column(1)).view(np.uint64).tolist() == np.asarray(b_out.column(1)).view(np.uint64).tolist()
    fused_ms, node_leaf_ms = [], []
    for i in range(args.reps):
        fused_ms.append(timed(fused.execute)[0])
        node_leaf_ms.append(timed(over_leaf.execute)[0])
    l_batch = plain.execute()  # {ts, value, job, instance, le}: series in (job, instance, le) order, every cell valid
    grid, words, hist_off, order, bucket_le = fold_inputs(l_batch, "prom_rate(ts_range,val)", "le", ["job", "instance"])
    del l_batch
    numbers = index_build(plain, over_leaf, lambda: ctx.histogram_fold(PHI, hist_off, order, bucket_le, grid, words))
    report("histogram_quantile(0.99, rate(x_bucket[5m]))", fused_leaf_ms=float(np.median(fused_ms)),
           node_over_plain_leaf_ms=float(np.median(node_leaf_ms)),
           **{"node_over_plain_leaf_" + k: v for k, v in numbers.items()})
    ctx.close()


if __name__ == "__main__":
    main()
