"""Host time of label_replace and label_join nodes beside their child's own time, on the same run.

The child is the instant leaf over --series series (default 1.25 M, the config-2 row count) of one sample each, tags
(pod, inst), evaluated at one step.  pod takes the form "p<k>-x<k mod 7>"; two cases:
  distinct  every series has its own pod value (1.25 M regex evaluations)
  1000      pod takes 1000 distinct values (inst keeps the series apart), so the per-node cache evaluates 1000
For each case, the median of --reps executions of: the leaf alone, label_replace(leaf, "svc", "$1", "pod",
"(.*)-[^-]+") and label_join(leaf, "id", "/", "pod", "inst").  Every execution runs the whole sub-tree and exports its
Arrow batch, so a label node's own cost is its time minus the leaf's; both are printed.  The label nodes do no device
work; the card's name and power limit are printed with each line because the leaf's are part of the numbers.

  python profiles/label_bench.py [--series N] [--reps K]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_250_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import pyarrow as pa
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("label_bench needs a CUDA device")
    from greptimedb_b200 import Context
    from greptimedb_b200.plan import LabelJoinPlan, LabelReplacePlan, PromRangeExec

    S = args.series
    ctx = Context(0)
    ident = gpu_identity()

    def leaf(pods, insts):
        ex = PromRangeExec(ctx, "", 0, 0, 15_000, 0, "ts", "val", ["pod", "inst"], lookback_delta=300_000)
        ex.push(pa.record_batch([pa.array(np.zeros(S, np.int64), pa.timestamp("ms")), pods, insts,
                                 pa.array(np.arange(S, dtype=np.float64))], names=["ts", "pod", "inst", "val"]))
        return ex

    def median_s(node):
        node.execute()  # warm-up
        ts = []
        for _ in range(args.reps):
            t = time.perf_counter()
            node.execute()
            ts.append(time.perf_counter() - t)
        return float(np.median(ts))

    for case, n_pods in (("distinct", S), ("1000", 1000)):
        width = len(str(S))
        # sorted by (pod, inst): pod i * n_pods // S, zero-padded so byte order is numeric order
        idx = np.arange(S) * n_pods // S
        pods = pa.array([f"p{k:0{width}d}-x{k % 7}" for k in idx])
        insts = pa.array([f"i{i:0{width}d}" for i in range(S)])
        base = leaf(pods, insts)
        t_leaf = median_s(base)
        rep = LabelReplacePlan(ctx, base, "svc", "$1", "pod", "(.*)-[^-]+")
        t_rep = median_s(rep)
        join = LabelJoinPlan(ctx, base, "id", "/", "pod", "inst")
        t_join = median_s(join)
        for name, t in (("label_replace", t_rep), ("label_join", t_join)):
            print(json.dumps({"node": name, "case": case, "distinct_pods": n_pods, "series": S,
                              "leaf_ms": round(t_leaf * 1e3, 2), "with_node_ms": round(t * 1e3, 2),
                              "node_ms": round((t - t_leaf) * 1e3, 2), **ident}), flush=True)
        rep.close()
        join.close()
        base.close()
    ctx.close()


if __name__ == "__main__":
    main()
