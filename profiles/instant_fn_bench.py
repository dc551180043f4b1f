"""Times the instant-vector functions (K9, b2p_instant_fn_dev) and scalar() (b2p_scalar_calculate_dev) on
device-resident random grids.

  1. every function in place over --series rows x 1000 steps (default 1.25 M, the config-2 shape), and K7's scalar form
     (`x * 2`, b2p_scalar_op_dev) on the same grid, for comparison
  2. scalar() over --groups rows x 1000 steps (the config-3 aggregate shape): many series, so the NaN branch; and the
     same grid with one live row, so the copy branch

For each it prints one JSON line: the CUDA-event time of the call (median of --reps), the bytes it has to move (computed
from the shapes: 8 B read and 8 B written per cell plus the validity words read; scalar(): the validity words of every
row, the one series' cells and the [T] output), that traffic's rate and its fraction of the H100 SXM data-sheet
3.35 TB/s, and the card's name and power limit read in the same run.

  python profiles/instant_fn_bench.py [--series N] [--groups G] [--reps R]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from binary_bench import PEAK_TBS, gpu_identity  # noqa: E402

T = 1000
ARGS = {"round": (0.1, 0.0), "clamp": (-1.0, 1.0), "clamp_min": (0.0, 0.0), "clamp_max": (0.0, 0.0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_250_000)
    ap.add_argument("--groups", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    import numpy as np
    import torch

    from greptimedb_b200 import Context
    from greptimedb_b200.engine import IFN_IDS

    dev = torch.device("cuda:0")
    ctx = Context(0)
    ctx.use_torch_stream()
    ident = gpu_identity()
    Tw = (T + 31) // 32
    gen = torch.Generator(device=dev).manual_seed(0x5EED)

    def timed(fn):
        ms = []
        for i in range(args.reps + 2):
            fn()
            ctx.sync()
            if i >= 2:
                ms.append(ctx.kernel_ms(3))
        return float(np.median(ms))

    def report(query, rows, b, ms):
        print(json.dumps({"query": query, "rows": rows, "steps": T, "kernel_ms": round(ms, 4), "bytes": b,
                          "tb_per_s": round(b / ms / 1e9, 3), "fraction_of_3.35_tb_s": round(b / ms / 1e9 / PEAK_TBS, 3),
                          **ident}), flush=True)

    S, G = args.series, args.groups
    # values in [-0.9, 0.9] keep every function inside its domain; every cell valid
    x = (torch.rand(S * T, dtype=torch.float64, device=dev, generator=gen) - 0.5) * 1.8
    xv = torch.full((S * Tw,), -1, dtype=torch.int32, device=dev)
    cell_bytes = S * T * 16 + S * Tw * 4
    # ---- 1. every function in place, and K7's scalar form -------------------------------------------------------------
    ms = timed(lambda: ctx.scalar_op_dev("*", 2.0, x, xv, S, T, x, xv))
    report("x * 2 (K7 scalar form)", S, cell_bytes + S * Tw * 4, ms)
    for fn in IFN_IDS:
        a0, a1 = ARGS.get(fn, (0.0, 0.0))
        x.uniform_(-0.9, 0.9, generator=gen)
        ms = timed(lambda: ctx.instant_fn_dev(fn, x, xv, S, T, x, xv, a0, a1))
        report(f"{fn}(x)", S, cell_bytes, ms)
    del x, xv
    torch.cuda.empty_cache()
    # ---- 2. scalar() over the aggregate shape ---------------------------------------------------------------------------
    g = torch.randn(G * T, dtype=torch.float64, device=dev, generator=gen)
    gv = torch.full((G * Tw,), -1, dtype=torch.int32, device=dev)
    keys = torch.arange(G, dtype=torch.int32, device=dev)
    out = torch.empty(T, dtype=torch.float64, device=dev)
    out_v = torch.empty(Tw, dtype=torch.int32, device=dev)
    ms = timed(lambda: ctx.scalar_calculate_dev(g, gv, keys, G, T, out, out_v))
    report("scalar(sum by (pod)(x)), many series -> NaN", G, G * Tw * 4 + G * 4 + T * 8 + Tw * 4, ms)
    gv.zero_()
    gv[(G // 2) * Tw:(G // 2 + 1) * Tw] = -1
    ms = timed(lambda: ctx.scalar_calculate_dev(g, gv, keys, G, T, out, out_v))
    report("scalar(...), one live series -> copy", G, G * Tw * 4 + G * 4 + T * 16 + 2 * Tw * 4, ms)
    ctx.close()


if __name__ == "__main__":
    main()
