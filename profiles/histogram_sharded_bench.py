"""Times the sharded histogram_quantile (b2p_histogram_fold_allgather) and its row-move kernel.

One GPU (plain `python`), a reduced config-4 shape: --hists histograms (default 16 k) x --buckets buckets (default 64)
x --steps steps (default 128), all cells valid:
  a. the row-move kernel (b2p_row_move_dev) permuting every bucket row of the device grid, against its HBM bound
     (2 x (8 T + 4 Tw) B per row over 3.35 TB/s, the H100 SXM data sheet's figure);
  b. the composed call over a one-rank communicator beside b2p_histogram_fold on the same host rows.  Both stage the
     grid to the device; the composed call also builds the owner's index on the host and places the results;
  c. what a sharded leaf runs, b2p_range_histogram_fold_allgather (rate() over every bucket series of 128 samples into
     the fold's grid on the device), beside the unsharded leaf's fused b2p_range_histogram_fold.
Without NCCL the composed call runs without a communicator, and the line says so.

N GPUs (`torchrun --nproc-per-node N profiles/histogram_sharded_bench.py`): every rank holds 1/N of the rows, sharded
by series hash (histograms split) and by histogram (whole); per rank the composed call's time, its
b2p_last_exchange_bytes, and the bytes the `sum by (le, ...)` workaround would all-reduce (its [buckets x T] f64 partial
grid and u32 counts).  With fewer than two GPUs visible that measurement is not made.

Each line is one JSON object with CUDA-event or synchronised host times (median of --reps), and the card's name and
power limit read in the same run.

  python profiles/histogram_sharded_bench.py [--hists N] [--buckets B] [--steps T] [--reps R]
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

HBM_BPS = 3.35e12


def grid(H, B, T, seed=0):
    import numpy as np
    rng = np.random.default_rng(seed)
    rates = np.cumsum(rng.random((H * B, T)), axis=1)
    words = np.full((H * B, (T + 31) // 32), 0xFFFFFFFF, np.uint32)
    if T % 32:
        words[:, -1] = (1 << (T % 32)) - 1
    hist = np.repeat(np.arange(H, dtype=np.uint32), B)
    le = np.tile(np.r_[np.cumsum(np.ones(B - 1)), np.inf], H)
    return rates, words, hist, le


def median_ms(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return sorted(ts)[len(ts) // 2]


def one_gpu(a):
    import numpy as np
    import torch
    from greptimedb_b200 import B2PError, Context
    H, B, T = a.hists, a.buckets, a.steps
    Tw = (T + 31) // 32
    rates, words, hist, le = grid(H, B, T)
    n = H * B
    ctx = Context(0)
    ctx.use_torch_stream()  # the kernel on the stream the events are recorded on
    dev = torch.device("cuda", 0)
    d_in, d_inw = torch.from_numpy(rates.reshape(-1)).to(dev), torch.from_numpy(words.reshape(-1).view(np.int32)).to(dev)
    d_out, d_outw = torch.empty_like(d_in), torch.empty_like(d_inw)
    src = torch.arange(n, dtype=torch.int32, device=dev)
    dst = torch.from_numpy(np.random.default_rng(1).permutation(n).astype(np.int32)).to(dev)
    ctx.row_move_dev(d_in, d_inw, src, dst, n, T, d_out, d_outw)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(a.reps):
        e0.record()
        ctx.row_move_dev(d_in, d_inw, src, dst, n, T, d_out, d_outw)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    k_ms = sorted(ms)[len(ms) // 2]
    moved = 2 * n * (8 * T + 4 * Tw)
    ok = torch.equal(d_out.view(n, T)[dst.long()], d_in.view(n, T))
    print(json.dumps({"what": "row_move", "rows": n, "T": T, "ms": round(k_ms, 4), "bytes": moved,
                      "hbm_bound_ms": round(moved / HBM_BPS * 1e3, 4), "share_of_hbm_bound": round(moved / HBM_BPS * 1e3 / k_ms, 3),
                      "correct": bool(ok), **gpu_identity()}), flush=True)
    del d_in, d_inw, d_out, d_outw
    comm = "one-rank communicator"
    try:
        ctx.comm_init(ctx.comm_unique_id(), 1, 0)
    except B2PError as e:
        comm = f"no communicator ({e})"
    off = np.r_[0, np.cumsum(np.full(H, B))].astype(np.uint32)
    bs = np.arange(n, dtype=np.uint32)
    fold_ms = median_ms(lambda: ctx.histogram_fold(0.99, off, bs, le, rates, words), a.reps)
    sharded_ms = median_ms(lambda: ctx.histogram_fold_allgather(0.99, rates, words, hist, le, H), a.reps)
    v0, w0 = ctx.histogram_fold(0.99, off, bs, le, rates, words)
    v1, w1 = ctx.histogram_fold_allgather(0.99, rates, words, hist, le, H)
    same = bool(np.array_equal(w0, w1) and np.array_equal(v0.view(np.uint64), v1.view(np.uint64)))
    print(json.dumps({"what": "composed_vs_fold", "hists": H, "buckets": B, "T": T, "comm": comm,
                      "histogram_fold_ms": round(fold_ms, 3), "histogram_fold_allgather_ms": round(sharded_ms, 3),
                      "exchange_bytes": ctx.last_exchange_bytes(), "bit_identical": same, **gpu_identity()}), flush=True)
    # c. the leaf's calls: rate() over every bucket series (128 samples each) and the fold, the unsharded fused
    # b2p_range_histogram_fold beside the range form of the sharded call
    import ctypes as C
    from greptimedb_b200 import make_params
    N = 128
    ts = np.tile(15_000 * np.arange(N, dtype=np.int64), n)
    val = np.cumsum(np.random.default_rng(2).random((n, N)), axis=1).reshape(-1)
    offsets = (np.arange(n + 1, dtype=np.uint64) * N)
    p = make_params("rate", 300_000, 15_000 * (N - 1), 15_000, 300_000)
    Tr = (p.end - p.start) // p.interval + 1
    o0, w0 = np.zeros((H, Tr)), np.zeros((H, (Tr + 31) // 32), np.uint32)

    def fused():
        ctx._check(ctx._L.b2p_range_histogram_fold(ctx._h, C.byref(p), ts.ctypes.data, val.ctypes.data, None,
                                                   offsets.ctypes.data, ts.size, n, 0.99, off.ctypes.data,
                                                   bs.ctypes.data, le.ctypes.data, H, o0.ctypes.data, w0.ctypes.data))
    fused_ms = median_ms(fused, a.reps)
    range_ms = median_ms(lambda: ctx.range_histogram_fold_allgather(p, 0.99, ts, val, offsets, hist, le, H), a.reps)
    fused()
    o1, w1 = ctx.range_histogram_fold_allgather(p, 0.99, ts, val, offsets, hist, le, H)
    same = bool(np.array_equal(w0, w1) and np.array_equal(o0.view(np.uint64), o1.view(np.uint64)))
    print(json.dumps({"what": "leaf_range_form_vs_fused", "hists": H, "buckets": B, "samples": N, "T": int(Tr),
                      "comm": comm, "range_histogram_fold_ms": round(fused_ms, 3),
                      "range_histogram_fold_allgather_ms": round(range_ms, 3), "exchange_bytes": ctx.last_exchange_bytes(),
                      "bit_identical": same, **gpu_identity()}), flush=True)
    ctx.close()


def multi_gpu(a):
    import numpy as np
    import torch
    import torch.distributed as dist
    from greptimedb_b200 import Context
    from greptimedb_b200 import distributed as D
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ctx = Context(local)
    box = [ctx.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=0)
    ctx.comm_init(box[0], world, rank)
    H, B, T = a.hists, a.buckets, a.steps
    rates, words, hist, le = grid(H, B, T)
    for layout in ("series", "histogram"):
        owner = (D.shard_of_series(np.arange(H * B, dtype=np.uint32), world) if layout == "series"
                 else (hist % world))
        mine = np.flatnonzero(owner == rank)
        args = (0.99, rates[mine], words[mine], hist[mine], le[mine], H)
        dist.barrier()
        ms = median_ms(lambda: ctx.histogram_fold_allgather(*args), a.reps)
        sent = ctx.last_exchange_bytes()
        print(json.dumps({"what": "sharded", "layout": layout, "rank": rank, "world": world, "hists": H, "buckets": B,
                          "T": T, "rows": int(mine.size), "ms": round(ms, 3), "exchange_bytes": sent,
                          "sum_by_le_allreduce_bytes": H * B * T * 12, **gpu_identity()}), flush=True)
    ctx.comm_destroy()
    ctx.close()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hists", type=int, default=16384)
    ap.add_argument("--buckets", type=int, default=64)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing is measured")
    if "WORLD_SIZE" in os.environ and int(os.environ["WORLD_SIZE"]) > 1:
        multi_gpu(a)
    else:
        one_gpu(a)
        if torch.cuda.device_count() < 2:
            print(json.dumps({"what": "sharded", "note": "fewer than two GPUs visible: not measured"}), flush=True)


if __name__ == "__main__":
    main()
