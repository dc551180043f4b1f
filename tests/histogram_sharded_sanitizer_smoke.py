"""One small sharded histogram_quantile per path (the row-move kernel at aligned and unaligned rows, three simulated
ranks through the step entry points, and the composed call and its range form over one rank), for a compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck  python tests/histogram_sharded_sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/histogram_sharded_sanitizer_smoke.py

Paths: histograms split across ranks and whole on one, a rank with no rows, a histogram with no bucket, more than 64
buckets, a step count that is not a multiple of 32.  Each result is checked against b2p_histogram_fold over all rows."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from greptimedb_b200 import Context
    from tests.test_gpu_histogram_sharded import bucket_rows, simulate, unsharded_fold

    ctx = Context(0)
    rng = np.random.default_rng(3)
    rates, words, hist, le = bucket_rows(rng, n_hist=12, T=33)
    H = int(hist.max()) + 2
    for layout in ("series", "histogram"):
        rank_of_row = rng.integers(0, 3, hist.size) if layout == "series" else rng.integers(0, 3, H)[hist]
        rank_of_row[rank_of_row == 1] = 2
        order = np.argsort(rank_of_row, kind="stable")
        want_v, want_w = unsharded_fold(ctx, 0.9, rates[order], words[order], hist[order], le[order], H)
        got_v, got_w, _ = simulate(ctx, 0.9, rates, words, hist, le, H, rank_of_row, 3)
        assert np.array_equal(got_w, want_w) and np.array_equal(got_v.view(np.uint64), want_v.view(np.uint64))
    want_v, want_w = unsharded_fold(ctx, 0.5, rates, words, hist, le, H)
    got_v, got_w = ctx.histogram_fold_allgather(0.5, rates, words, hist, le, H)
    assert np.array_equal(got_w, want_w) and np.array_equal(got_v.view(np.uint64), want_v.view(np.uint64))
    from tests.test_gpu_histogram_sharded import bucket_series
    ts, val, offsets, shist, sle, p = bucket_series(rng, n_hist=8, n=40)
    grid, gw, _ = ctx.range_eval(p, ts, val, offsets=offsets)
    want_v, want_w = unsharded_fold(ctx, 0.9, grid, gw, shist, sle, int(shist.max()) + 1)
    got_v, got_w = ctx.range_histogram_fold_allgather(p, 0.9, ts, val, offsets, shist, sle, int(shist.max()) + 1)
    assert np.array_equal(got_w, want_w) and np.array_equal(got_v.view(np.uint64), want_v.view(np.uint64))
    ctx.close()
    print("HISTOGRAM_SHARDED_SANITIZER_SMOKE ok")


if __name__ == "__main__":
    main()
