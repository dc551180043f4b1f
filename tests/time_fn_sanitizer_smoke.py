"""One small call of every time-function entry point, for a compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck python tests/time_fn_sanitizer_smoke.py

K19 for every part over a grid with holes and a T that is not a multiple of 32 (and T = 1), K4's timestamp mode, unary
minus (K9), and the plan nodes above them: EmptyMetric, a calendar stage and the timestamp leaf.  Each result is checked
against tests/time_fn_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import pyarrow as pa

    from greptimedb_b200 import Context
    from greptimedb_b200.plan import EmptyMetricPlan, PromRangeExec
    from tests import time_fn_oracle as to
    from tests.binary_oracle import _words

    rng = np.random.default_rng(19)
    ctx = Context(0)
    for R, T in ((7, 45), (3, 1)):
        ets = rng.integers(-10**13, 10**13, T, dtype=np.int64)
        ok = rng.random((R, T)) < 0.6
        for part in to.PARTS:
            out = ctx.step_fn(part, ets, _words(ok))
            assert (out.view(np.int64) == to.step_fn(part, ets, ok).view(np.int64)).all(), part
    ts = np.array([0, 10_000, 10_000, 40_000, 5_000], np.int64)
    out, valid = ctx.instant_timestamp(ts, 0, 50_000, 7_000, 20_000, 1_000, offsets=np.array([0, 4, 5], np.uint64))
    want, ok = to.instant_timestamp(ts, [0, 4, 5], 0, 50_000, 7_000, 20_000, 1_000)
    assert (valid == _words(ok)).all() and (out == want).all()
    neg, _ = ctx.instant_fn("neg", np.array([[0.0, -2.5, 3.0]]), np.array([[7]], np.uint32))
    assert neg.view(np.int64).tolist() == np.array([[-0.0, 2.5, -3.0]]).view(np.int64).tolist()
    assert EmptyMetricPlan(ctx, 0, 4_000, 1_000, "none").function("day_of_week").execute().num_rows == 5
    b = pa.record_batch([pa.array([0, 10_000], pa.timestamp("ms")), pa.array([1.0, float("nan")])], names=["ts", "val"])
    ex = PromRangeExec(ctx, "", 0, 20_000, 5_000, 0, "ts", "val", [], lookback_delta=300_000)
    ex.push(b)
    assert ex.timestamp(300_000).execute().column(1).to_pylist() == [0.0, 0.0, 10.0, 10.0, 10.0]
    ctx.close()
    print("time_fn sanitizer smoke ok")


if __name__ == "__main__":
    main()
