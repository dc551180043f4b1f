"""Sharded plan nodes (b2p_plan_set_sharded) beside the unsharded ones, over a one-rank communicator: config 3's shape,
sum by (pod) over an instant leaf, through the leaf's aggregate stage and through an aggregate node.  Prints one JSON
line with, per route: the execute wall time of the sharded and the unsharded node (median of --reps), the agreement's
exchanged bytes (b2p_last_group_keys_bytes), the host time of the agreement's merge (b2p_group_keys_merge over this
rank's block), and the device time of the fold (K3 partials, stage 3) and of the merge (the all-reduce, stage 4) from
the context's CUDA events.  The card's name and power limit go beside the numbers.

The default size is config 3's group count (100 000 groups) over 200 000 series x 100 steps: the plan layer takes Arrow
batches on the host, and config 3's full rank (1.25 M series x 1000 steps) is 1.25 G rows of them.

    python profiles/plan_sharded_bench.py [--series 200000] [--steps 100] [--groups 100000] [--reps 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import pyarrow as pa

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def table(S, T, G):
    """S series of T samples, series s in pod s % G; rows sorted by (pod, sid, ts) as SeriesDivide requires (zero-padded
    names sort as their numbers)"""
    import pyarrow.compute as pc
    series = np.lexsort((np.arange(S), np.arange(S) % G))
    sid = np.repeat(series, T)
    pad = lambda x, w: pc.utf8_lpad(pa.array(x).cast(pa.utf8()), width=w, padding="0")  # noqa: E731
    rng = np.random.default_rng(3)
    return pa.record_batch([pa.array(np.tile(np.arange(T, dtype=np.int64) * 15_000, S), pa.timestamp("ms")),
                            pad(sid % G, 7), pad(sid, 8), pa.array(rng.random(S * T) * 100.0)],
                           names=["ts", "pod", "sid", "val"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=200_000)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--groups", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    from greptimedb_b200 import Context
    from greptimedb_b200 import distributed as D
    from greptimedb_b200.plan import AggregatePlan, PromRangeExec
    S, T, G = a.series, a.steps, a.groups
    batch = table(S, T, G)
    plain, comm = Context(0), Context(0)
    comm.comm_init(comm.comm_unique_id(), 1, 0)
    end = (T - 1) * 15_000

    def leaf(ctx, agg=None):
        ex = PromRangeExec(ctx, "", 0, end, 15_000, 0, "ts", "val", ["pod", "sid"], lookback_delta=30_000,
                           aggregate=agg, by_columns=["pod"] if agg else ())
        ex.push(batch)
        return ex

    routes = {
        "leaf_stage": lambda ctx, sharded: (leaf(ctx, "sum").sharded() if sharded else leaf(ctx, "sum")),
        "aggregate_node": lambda ctx, sharded: (AggregatePlan(ctx, "sum", leaf(ctx), by=["pod"]).sharded() if sharded
                                                else AggregatePlan(ctx, "sum", leaf(ctx), by=["pod"])),
    }
    out = {"series": S, "steps": T, "groups": G}
    for name, make in routes.items():
        res = {}
        for sharded, ctx in ((False, plain), (True, comm)):
            node = make(ctx, sharded)
            node.execute()  # warm-up
            times = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                r = node.execute()
                times.append(time.perf_counter() - t0)
            assert r.num_rows == G * T
            res["sharded_ms" if sharded else "unsharded_ms"] = 1e3 * float(np.median(times))
            if sharded:
                res["agreement_bytes"] = int(comm._L.b2p_last_group_keys_bytes(comm._h))
                res["fold_device_ms"] = float(comm._L.b2p_last_kernel_ms(comm._h, 3))
                res["merge_device_ms"] = float(comm._L.b2p_last_kernel_ms(comm._h, 4))
            node.close()
        out[name] = res
    # the agreement's host merge over this rank's block (G groups of one label)
    blk = D.serialize_group_keys([(str(g),) for g in sorted(map(str, range(G)))], 1)
    blocks = (C.c_void_p * 1)(C.cast(C.c_char_p(blk), C.c_void_p))
    sizes = (C.c_uint64 * 1)(len(blk))
    tbl = C.create_string_buffer(len(blk))
    nb, ng, l2g = C.c_uint64(), C.c_uint32(), (C.c_uint32 * G)()
    t0 = time.perf_counter()
    assert comm._L.b2p_group_keys_merge(blocks, sizes, 1, 0, tbl, C.byref(nb), C.byref(ng), l2g) == 0
    out["agreement_merge_host_ms"] = 1e3 * (time.perf_counter() - t0)
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                capture_output=True, text=True).stdout.strip()
    comm.comm_destroy()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
