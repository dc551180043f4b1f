"""Times the set-operator kernels (K8, b2p_setop_dev) on device-resident random grids.

  1. x and y / x unless y, one to one: --series rows x 1000 steps (default 1.25 M, the config-2 shape), in place
  2. x unless on(pod) y: the same lhs against --groups aggregate rows (the config-3 shape)
  3. x or y, one to one
  4. x or on() y: one key, --wide lhs rows and --wide rhs rows, so the rhs-against-rhs dedupe walks one long member list

For each it prints one JSON line: the CUDA-event time of the whole call (key check, the key grouping's radix sort, the
mask / dedupe and copy kernels; median of --reps), the bytes the call has to move (computed from the shapes: 8 B read and
8 B written per kept-or-not output cell, the validity words each kernel reads and writes, 4 B per key), that traffic's
rate and its fraction of the H100 SXM data-sheet 3.35 TB/s, and the card's name and power limit read in the same run.

  python profiles/setop_bench.py [--series N] [--groups G] [--wide W] [--reps R]
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


def setop_bytes(op: str, n_lhs: int, n_rhs: int, n_keys: int) -> int:
    """and / unless: lhs values in and out, lhs words in and out, the mask written once and read per lhs row, the rhs
    words; or: both sides' values in and out, the lhs mask, the rhs words read twice (dedupe, copy) and written once."""
    Tw = (T + 31) // 32
    keys = 4 * (n_lhs + n_rhs)
    if op != "or":
        return n_lhs * T * 16 + (3 * n_lhs + n_rhs + n_keys) * Tw * 4 + keys
    return (n_lhs + n_rhs) * T * 16 + (3 * n_lhs + n_keys + 4 * n_rhs) * Tw * 4 + keys


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_250_000)
    ap.add_argument("--groups", type=int, default=100_000)
    ap.add_argument("--wide", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    import numpy as np
    import torch

    from greptimedb_b200 import Context

    dev = torch.device("cuda:0")
    ctx = Context(0)
    ctx.use_torch_stream()
    ident = gpu_identity()
    Tw = (T + 31) // 32
    gen = torch.Generator(device=dev).manual_seed(0x5EED)

    def grid(rows):
        vals = torch.randn(rows * T, dtype=torch.float64, device=dev, generator=gen)
        words = torch.randint(-2 ** 31, 2 ** 31 - 1, (rows * Tw,), dtype=torch.int32, device=dev, generator=gen)
        return vals, words

    def timed(fn):
        ms = []
        for i in range(args.reps + 2):
            fn()
            ctx.sync()
            if i >= 2:
                ms.append(ctx.kernel_ms(3))
        return float(np.median(ms))

    def report(query, op, n_lhs, n_rhs, n_keys, ms):
        b = setop_bytes(op, n_lhs, n_rhs, n_keys)
        print(json.dumps({"query": query, "lhs_rows": n_lhs, "rhs_rows": n_rhs, "keys": n_keys, "steps": T,
                          "kernel_ms": round(ms, 4), "bytes": b, "tb_per_s": round(b / ms / 1e9, 3),
                          "fraction_of_3.35_tb_s": round(b / ms / 1e9 / PEAK_TBS, 3), **ident}), flush=True)

    S, G = args.series, args.groups
    x, xv = grid(S)
    ident_keys = torch.arange(S, dtype=torch.int32, device=dev)
    _, yv = grid(S)
    # ---- 1. and / unless, one to one (in place: the lhs grid is overwritten, which does not change the traffic) -------
    for op in ("and", "unless"):
        ms = timed(lambda: ctx.setop_dev(op, x, xv, ident_keys, S, None, yv, ident_keys, S, S, T, x, xv))
        report(f"x {op} y", op, S, S, S, ms)
    # ---- 2. unless on(pod) against the aggregate rows -----------------------------------------------------------------
    pods = torch.randint(0, G, (S,), dtype=torch.int32, device=dev, generator=gen)
    _, gv = grid(G)
    gkeys = torch.arange(G, dtype=torch.int32, device=dev)
    ms = timed(lambda: ctx.setop_dev("unless", x, xv, pods, S, None, gv, gkeys, G, G, T, x, xv))
    report("x unless on(pod) sum by (pod)(y)", "unless", S, G, G, ms)
    del pods, gv, gkeys
    # ---- 3. or, one to one ---------------------------------------------------------------------------------------------
    y, _ = grid(S)
    out = torch.empty(2 * S * T, dtype=torch.float64, device=dev)
    out_v = torch.empty(2 * S * Tw, dtype=torch.int32, device=dev)
    ms = timed(lambda: ctx.setop_dev("or", x, xv, ident_keys, S, y, yv, ident_keys, S, S, T, out, out_v))
    report("x or y", "or", S, S, S, ms)
    del x, xv, y, yv, out, out_v, ident_keys
    torch.cuda.empty_cache()
    # ---- 4. x or on() y: one key ---------------------------------------------------------------------------------------
    W = args.wide
    a, av = grid(W)
    b, bv = grid(W)
    zero = torch.zeros(W, dtype=torch.int32, device=dev)
    out = torch.empty(2 * W * T, dtype=torch.float64, device=dev)
    out_v = torch.empty(2 * W * Tw, dtype=torch.int32, device=dev)
    ms = timed(lambda: ctx.setop_dev("or", a, av, zero, W, b, bv, zero, W, 1, T, out, out_v))
    report("x or on() y", "or", W, W, 1, ms)
    ctx.close()


if __name__ == "__main__":
    main()
