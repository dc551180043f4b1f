"""One small call of every Int64 entry point, for a compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck python tests/int64_sanitizer_smoke.py

The instant selector with an Int64 field 0 (K17 without the staleness test), the by-label aggregate in its integer
and (double)i64 modes (K3), topk / bottomk (K10 with the Int64 key), count_values (K12), sort (K14) and the Float64
coercion, each over a grid with holes and a T that is not a multiple of 32.  Each result is checked against
tests/int64_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import pyarrow as pa

    from greptimedb_b200 import Context
    from greptimedb_b200.plan import PromRangeExec
    from tests import int64_oracle as io
    from tests.binary_oracle import _words

    rng = np.random.default_rng(64)
    R, T, G = 9, 45, 3
    vals = rng.integers(-3, 3, (R, T)).astype(np.int64)
    vals[0, ::5] = io.INT64_MAX
    vals[1, ::7] = np.array([np.nan], np.float64).view(np.int64)[0]
    ok = rng.random((R, T)) < 0.6
    gid = (np.arange(R) % G).astype(np.uint32)
    ctx = Context(0)
    for op in ("sum", "min", "max", "avg"):
        got, cnt = ctx.group_aggregate_i64(op, vals, _words(ok), gid, G)
        want, wcnt = io.group_aggregate(op, vals, ok, gid, G)
        assert (cnt == wcnt).all(), op
    for desc in (False, True):
        assert ctx.sort_cells_i64(desc, vals, _words(ok)).tolist() == io.value_order(vals, ok, desc)
    tie = np.arange(R, dtype=np.uint32)
    for op in ("topk", "bottomk"):
        assert (ctx.topk_i64(op, 2, vals, _words(ok), gid, G, tie) == _words(io.topk_keep(op == "bottomk", 2, vals, ok,
                                                                                          gid, G, tie))).all()
    out, cnt = ctx.count_values_i64(vals, _words(ok), gid, G)
    assert int(cnt.sum()) == int(ok.sum())
    assert ctx.i64_to_f64(vals[0]).tolist() == vals[0].astype(np.float64).tolist()
    b = pa.record_batch([pa.array([0, 5000, 0], pa.timestamp("ms")), pa.array(["a", "a", "b"]),
                         pa.array([int(vals[1, 0]), 2, 3], pa.int64())], names=["ts", "host", "val"])
    ex = PromRangeExec(ctx, "", 0, 10_000, 5_000, 0, "ts", "val", ["host"], lookback_delta=io.LOOKBACK)
    ex.push(b)
    assert ex.execute().num_rows == 6
    ctx.close()
    print("int64 sanitizer smoke ok")


if __name__ == "__main__":
    main()
