"""Times absent(): K15 alone (b2p_absent_dev) on device-resident validity bitmaps, and end to end through AbsentPlan.

Shapes for K15 (only the bitmap exists: K15 never reads a value):
  1. the config-2 grid, --series rows (default 1.25 M) x 1000 steps (Tw = 32), every cell valid, no cell valid, and
     each bit random (about 50 % valid);
  2. T = 1 over --tall-rows rows (default 10 M; Tw = 1), with the same three fills.

K15 alone: CUDA events around b2p_absent_dev (the zeroing of the 4 B-per-word accumulator, the OR pass, the write pass),
median of --reps after one warm-up.  It prints the bitmap's size (rows x Tw x 4 B: what the OR pass reads at most), the
achieved rate over that size and its fraction of the H100 SXM data-sheet 3.35 TB/s.  A thread stops reading its word
once every step of it is present, so on a dense bitmap the pass reads much less than the bitmap and the rate over the
bitmap's size is not a bandwidth.

End to end: AbsentPlan over an instant leaf of --e2e-series series x 1000 steps (default 50 k) with about half of the
samples missing: the host time of execute() of the absent node and of its child alone (median of --reps after one
warm-up; each plan call is synchronous).  The child's execute() exports its cells to Arrow; under the absent node the
child only computes its grid, and the node sends the child's bitmap to the device, runs K15 and exports one row, so the
node's time is not the child's plus something.

Every line carries the card's name and power limit, read in the same run.

  python profiles/absent_bench.py [--series N] [--tall-rows M] [--e2e-series E] [--reps R]
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

from binary_bench import PEAK_TBS, gpu_identity  # noqa: E402

T, SCRAPE, T0 = 1000, 15_000, 1_700_000_000_000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_250_000)
    ap.add_argument("--tall-rows", type=int, default=10_000_000)
    ap.add_argument("--e2e-series", type=int, default=50_000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    import numpy as np
    import pyarrow as pa
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("absent_bench needs a CUDA device")
    from greptimedb_b200 import Context
    from greptimedb_b200.plan import AbsentPlan, PromRangeExec

    dev = torch.device("cuda:0")
    ctx = Context(0)
    ctx.use_torch_stream()
    ident = gpu_identity()

    def report(**kw):
        print(json.dumps({**kw, **ident}), flush=True)

    def k15(shape, rows, steps):
        Tw = (steps + 31) // 32
        valid = torch.empty(rows * Tw, dtype=torch.int32, device=dev)
        out = torch.empty(steps, dtype=torch.float64, device=dev)
        ov = torch.empty(Tw, dtype=torch.int32, device=dev)
        gen = torch.Generator(device=dev)
        gen.manual_seed(0x5EED)
        for fill in ("all valid", "none valid", "50 % random"):
            if fill == "all valid":
                valid.fill_(-1)
            elif fill == "none valid":
                valid.zero_()
            else:
                valid.random_(generator=gen)  # (the int32 range's non-negative half ...)
                valid ^= torch.randint(0, 2, valid.shape, dtype=torch.int32, device=dev, generator=gen) << 31  # (+ sign)
            ms = []
            for i in range(args.reps + 1):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                ctx.absent_dev(valid, rows, steps, out, ov)
                b.record()
                torch.cuda.synchronize()
                if i:
                    ms.append(a.elapsed_time(b))
            m = float(np.median(ms))
            byt = rows * Tw * 4
            report(shape=shape, fill=fill, stage="k15", rows=rows, steps=steps, absent_steps=int((out == 1.0).sum()),
                   k15_ms=round(m, 4), k15_ms_min=round(min(ms), 4), k15_ms_max=round(max(ms), 4), bitmap_bytes=byt,
                   tb_per_s_over_bitmap=round(byt / m / 1e9, 3),
                   **{"fraction_of_3.35_tb_s": round(byt / m / 1e9 / PEAK_TBS, 3)})
        del valid, out, ov
        torch.cuda.empty_cache()

    k15("1. config-2 grid", args.series, T)
    k15("2. T = 1", args.tall_rows, 1)

    # end to end through AbsentPlan over an instant leaf
    E = args.e2e_series
    rng = np.random.default_rng(7)
    keep = rng.random(E * T) < 0.5
    batch = pa.record_batch([pa.array(np.tile(T0 + np.arange(T, dtype=np.int64) * SCRAPE, E)[keep], pa.timestamp("ms")),
                             pa.array(rng.standard_normal(E * T)[keep]),
                             pa.array(np.repeat(np.arange(E, dtype=np.uint64), T)[keep], pa.uint64())],
                            names=["ts", "val", "__tsid"])
    del keep

    def leaf():
        x = PromRangeExec(ctx, "", T0, T0 + (T - 1) * SCRAPE, SCRAPE, 0, "ts", "val", ["__tsid"], lookback_delta=1000)
        x.push(batch)
        return x

    def timed(call):
        ms = []
        for i in range(args.reps + 1):
            t = time.perf_counter()
            out = call()
            if i:
                ms.append((time.perf_counter() - t) * 1e3)
        return float(np.median(ms)), out

    child_ms, _ = timed(leaf().execute)
    node = AbsentPlan(ctx, leaf(), T0, T0 + (T - 1) * SCRAPE, SCRAPE, "ts", "val", [("job", "api")])
    node_ms, out = timed(node.execute)
    report(shape="3. instant leaf, 50 % of the samples (e2e)", stage="end to end", rows=E, steps=T,
           exported_rows=out.num_rows, child_execute_ms=round(child_ms, 3), absent_node_execute_ms=round(node_ms, 3))
    ctx.close()


if __name__ == "__main__":
    main()
