"""Times the binary-operator kernel (K7, b2p_binary_op_dev) on device-resident synthetic data.

  1. rate(a[5m]) / rate(b[5m]), one to one: --series pairs x 1000 steps (default 1.25 M, the config-2 shape)
  2. sum by (pod)(rate(err[5m])) / sum by (pod)(rate(req[5m])) at the config-3 shape (1.25 M series, --groups pods)

For each it prints one JSON line: the kernel's CUDA-event time (median of --reps), the bytes the kernel has to move
(computed from the shapes: two 8 B operands and one 8 B result per (pair, step), three validity words per 32 steps,
two row indices per pair), that traffic's rate and its fraction of the H100 SXM data-sheet 3.35 TB/s, and the card's
name and power limit read in the same run.

  python profiles/binary_bench.py [--series N] [--groups G] [--reps R]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T0, N_SAMPLES, SCRAPE, RANGE, SEED = 1_700_000_000_000, 1000, 15_000, 300_000, 0x5EED
PEAK_TBS = 3.35


def gpu_identity():
    info = {"gpu": None, "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        name, limit = r.stdout.strip().splitlines()[0].rsplit(",", 1)
        info = {"gpu": name.strip(), "power_limit_w": float(limit)}
    except Exception:
        pass
    return info


def binary_bytes(n_pairs: int, T: int) -> int:
    Tw = (T + 31) // 32
    return n_pairs * (T * 24 + Tw * 12 + 8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_250_000)
    ap.add_argument("--groups", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    import numpy as np
    import torch

    from greptimedb_b200 import Context, make_params
    from greptimedb_b200 import distributed as D

    dev = torch.device("cuda:0")
    ctx = Context(0)
    ctx.use_torch_stream()
    ident = gpu_identity()
    S, T = args.series, N_SAMPLES
    Tw = (T + 31) // 32
    n_rows = S * N_SAMPLES
    p = make_params("rate", T0, T0 + (N_SAMPLES - 1) * SCRAPE, SCRAPE, RANGE)

    def timed(fn):
        ms = []
        for i in range(args.reps + 2):
            fn()
            ctx.sync()
            if i >= 2:
                ms.append(ctx.kernel_ms(3))
        return float(np.median(ms))

    def report(query, n_pairs, ms, **extra):
        b = binary_bytes(n_pairs, T)
        print(json.dumps({"query": query, "pairs": n_pairs, "steps": T, "kernel_ms": round(ms, 4), "bytes": b,
                          "tb_per_s": round(b / ms / 1e9, 3), "fraction_of_3.35_tb_s": round(b / ms / 1e9 / PEAK_TBS, 3),
                          **extra, **ident}), flush=True)

    # ---- 1. rate(a) / rate(b), one to one ----------------------------------------------------------------------------
    ts = torch.empty(n_rows, dtype=torch.int64, device=dev)
    val = torch.empty(n_rows, dtype=torch.float64, device=dev)
    sid = torch.empty(n_rows, dtype=torch.int32, device=dev)
    offsets = torch.empty(S + 1, dtype=torch.int64, device=dev)
    grids = []
    for seed in (SEED, SEED + 1):
        out = torch.empty(S * T, dtype=torch.float64, device=dev)
        valid = torch.empty(S * Tw, dtype=torch.int32, device=dev)
        ctx.synth_fill_dev(0, S, N_SAMPLES, T0, SCRAPE, 1000, 1, seed, ts, val, sid)
        ctx.series_offsets_dev(sid, n_rows, S, offsets)
        ctx.range_eval_dev(p, ts, val, offsets, n_rows, S, out, valid)
        ctx.sync()
        grids.append((out, valid))
    del ts, val
    torch.cuda.empty_cache()
    rows = torch.arange(S, dtype=torch.int32, device=dev)
    q = torch.empty(S * T, dtype=torch.float64, device=dev)
    qv = torch.empty(S * Tw, dtype=torch.int32, device=dev)
    (a, av), (b, bv) = grids

    def one_to_one():
        ctx.binary_op_dev("/", a, av, rows, S, b, bv, rows, S, S, T, q, qv)

    report("rate(a[5m]) / rate(b[5m])", S, timed(one_to_one))
    del grids, a, av, b, bv, q, qv
    torch.cuda.empty_cache()

    # ---- 2. sum by (pod)(rate(err)) / sum by (pod)(rate(req)) ---------------------------------------------------------
    G = args.groups
    ts = torch.empty(n_rows, dtype=torch.int64, device=dev)
    val = torch.empty(n_rows, dtype=torch.float64, device=dev)
    gid = torch.from_numpy((D.mix32(np.arange(S, dtype=np.uint32)) % np.uint32(G)).astype(np.int32)).to(dev)
    ix = ctx.group_index_create_dev(gid, S, G)
    sides = []
    for seed in (SEED + 2, SEED + 3):
        gsum = torch.zeros(G * T, dtype=torch.float64, device=dev)
        gcnt = torch.zeros(G * T, dtype=torch.int32, device=dev)
        words = torch.empty(G * Tw, dtype=torch.int32, device=dev)
        ctx.synth_fill_dev(0, S, N_SAMPLES, T0, SCRAPE, 1000, 1, seed, ts, val, sid)
        ctx.series_offsets_dev(sid, n_rows, S, offsets)
        ctx.range_group_sum_indexed_dev(p, ts, val, offsets, n_rows, S, ix, 0, G, gsum, gcnt)
        ctx.count_valid_words_dev(gcnt, G, T, words)
        ctx.sync()
        sides.append((gsum, words))
    ctx.group_index_destroy(ix)
    grows = torch.arange(G, dtype=torch.int32, device=dev)
    q = torch.empty(G * T, dtype=torch.float64, device=dev)
    qv = torch.empty(G * Tw, dtype=torch.int32, device=dev)
    (e, ev), (r, rv) = sides

    def by_pod():
        ctx.binary_op_dev("/", e, ev, grows, G, r, rv, grows, G, G, T, q, qv)

    report("sum by (pod)(rate(err[5m])) / sum by (pod)(rate(req[5m]))", G, timed(by_pod), series=S)
    ctx.close()


if __name__ == "__main__":
    main()
