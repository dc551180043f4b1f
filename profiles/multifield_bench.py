"""Times the selectors over several field columns (b2p_range_eval_fields_dev, b2p_instant_select_fields_dev) against F
separate single-field calls over the same columns, and K16 / K17 / K18 alone.

Workload: --series series (default 250 k) x 1000 samples, 15 s scrapes, regular (jitter 0) and jittered (up to 1 s),
F in {2, 4} Float64 fields (field f = field 0 x (f + 1), no NaN); the grid is 1000 steps of 15 s, rate over 5 min.
Why 250 k series and not config 2's 1.25 M: one series costs 8 kB of timestamps, 4 kB of ids, and per field 8 kB of
values, 8 kB of K16's copy and 8 kB of grid, so 108 kB at F = 4.  1.25 M series would need 135 GB; 250 k need 27 GB,
which leaves the 80 GB of an H100 room for the range tiers' scratch.  One size serves both F, so the two rows of a
workload compare like with like.

  * fields call: host time around the entry point and b2p_sync (the range entry synchronises once itself before K18);
    separate calls: F single-field calls into the same grids and one b2p_sync.  Median of --reps after one warm-up.
  * K16 / K18 / K17 alone: the context's stage timers of the last call (CUDA events around each kernel; stage 0 = K16,
    3 = K18 of the range entry, 1 = K17 of the instant entry).  Bytes: K16 reads 8F B per row (it writes none here:
    there is no NaN); K18 reads 4F B and writes 4 B per validity word; K17 writes 8F B per cell plus its bitmap and
    reads the timestamps of its searches (not counted).

Every line carries the card's name and power limit, read in the same run.

  python profiles/multifield_bench.py [--series N] [--reps R]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from binary_bench import PEAK_TBS, gpu_identity  # noqa: E402

N, T, SCRAPE, T0 = 1000, 1000, 15_000, 1_700_000_000_000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=250_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("multifield_bench needs a CUDA device")
    from greptimedb_b200 import Context, make_params

    ident = gpu_identity()
    dev = torch.device("cuda:0")
    ctx = Context(0)
    ctx.use_torch_stream()
    S, R = args.series, args.series * N
    Tw = (T + 31) // 32
    words = S * Tw
    ts = torch.empty(R, dtype=torch.int64, device=dev)
    v0 = torch.empty(R, dtype=torch.float64, device=dev)
    sid = torch.empty(R, dtype=torch.int32, device=dev)
    offsets = torch.empty(S + 1, dtype=torch.int64, device=dev)
    outs = [torch.empty((S, T), dtype=torch.float64, device=dev) for _ in range(4)]
    valid = torch.empty((S, Tw), dtype=torch.int32, device=dev)
    valids = [torch.empty((S, Tw), dtype=torch.int32, device=dev) for _ in range(4)]
    p = make_params("rate", T0 + 300_000, T0 + 300_000 + (T - 1) * SCRAPE, SCRAPE, 300_000)

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        xs = []
        for _ in range(args.reps):
            t = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            xs.append((time.perf_counter() - t) * 1e3)
        return statistics.median(xs)

    def emit(**kw):
        print(json.dumps({**kw, **ident}), flush=True)

    for jitter in (0, 1000):
        ctx.synth_fill_dev(0, S, N, T0, SCRAPE, jitter, 0, 0x5EED, ts, v0, sid)
        ctx.series_offsets_dev(sid, R, S, offsets)
        ctx.sync()
        fields = [v0] + [v0 * float(f + 1) for f in range(1, 4)]
        torch.cuda.synchronize()
        for F in (2, 4):
            vals = fields[:F]

            def fields_call():
                ctx.range_eval_fields_dev(p, ts, vals, offsets, R, S, outs[:F], valid)
                ctx.sync()

            def separate():
                for f in range(F):
                    ctx.range_eval_dev(p, ts, vals[f], offsets, R, S, outs[f], valids[f])
                ctx.sync()

            # the two alternate, so that both see the same neighbours on the machine
            a, b = [], []
            for _ in range(2):
                a.append(timed(fields_call))
                b.append(timed(separate))
            fields_call()
            k16, k18 = ctx.kernel_ms(0), ctx.kernel_ms(3)
            emit(what="range_fields", jitter_ms=jitter, F=F, series=S, steps=T, fields_ms=min(a), separate_ms=min(b))
            emit(what="K16", jitter_ms=jitter, F=F, rows=R, ms=k16, bytes=8 * F * R,
                 tb_s=8 * F * R / (k16 * 1e-3) / 1e12, peak_frac=8 * F * R / (k16 * 1e-3) / 1e12 / PEAK_TBS)
            emit(what="K18", jitter_ms=jitter, F=F, words=words, ms=k18, bytes=4 * (F + 1) * words,
                 tb_s=4 * (F + 1) * words / (k18 * 1e-3) / 1e12,
                 peak_frac=4 * (F + 1) * words / (k18 * 1e-3) / 1e12 / PEAK_TBS)

            def inst_fields():
                ctx.instant_select_fields_dev(p.start, p.end, p.interval, 300_000, 0, ts, vals, offsets, R, S,
                                              outs[:F], valid)
                ctx.sync()

            def inst_separate():
                for f in range(F):
                    ctx.instant_select_dev(p.start, p.end, p.interval, 300_000, 0, ts, vals[f], offsets, R, S,
                                           outs[f], valids[f])
                ctx.sync()

            a, b = [], []
            for _ in range(2):
                a.append(timed(inst_fields))
                b.append(timed(inst_separate))
            inst_fields()
            k17 = ctx.kernel_ms(1)
            wbytes = 8 * F * S * T + 4 * words
            emit(what="instant_fields", jitter_ms=jitter, F=F, series=S, steps=T, fields_ms=min(a),
                 separate_ms=min(b))
            emit(what="K17", jitter_ms=jitter, F=F, series=S, steps=T, ms=k17, written_bytes=wbytes,
                 tb_s=wbytes / (k17 * 1e-3) / 1e12)
        del fields
    ctx.close()


if __name__ == "__main__":
    main()
