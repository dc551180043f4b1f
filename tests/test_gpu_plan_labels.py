"""GPU: how the plan layer stores, matches and orders label tuples.  A NULL label is its own state, never a string that
happens to look like one, and a tuple is never confused with another whose values concatenate to the same bytes."""
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu

NUL_NULL = "\x00null"   # a real Utf8 value: five bytes, the first a NUL


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def batch(tags, series, n=3):
    """One RecordBatch of `series` = [(label tuple, value)], each series n samples 1 s apart from ts 0."""
    ts, val, cols = [], [], {t: [] for t in tags}
    for labels, v in series:
        for i in range(n):
            ts.append(i * 1000)
            val.append(float(v))
            for t, lab in zip(tags, labels):
                cols[t].append(lab)
    return pa.record_batch([pa.array(ts, pa.timestamp("ms")), pa.array(val, pa.float64())] +
                           [pa.array(cols[t], pa.string()) for t in tags], names=["ts", "val"] + list(tags))


def node(ctx, tags, *batches, steps=2, **kw):
    """last_over_time over the batches, at `steps` steps ending at ts 2000 (every series has a cell at each)."""
    from greptimedb_b200.plan import PromRangeExec
    ex = PromRangeExec(ctx, "prom_last_over_time", 3000 - steps * 1000, 2000, 1000, 10_000, "ts", "val", tags, **kw)
    for b in batches:
        ex.push(b)
    return ex


def test_null_and_nul_string_label_are_two_series(ctx):
    null, nul = ((None,), 1.0), ((NUL_NULL,), 2.0)
    for batches in ([batch(["x"], [null, nul])], [batch(["x"], [null]), batch(["x"], [nul])]):  # one batch; a boundary
        ex = node(ctx, ["x"], *batches)
        out = ex.execute()
        assert ex.num_series() == 2
        assert out.column("x").to_pylist() == [None, None, NUL_NULL, NUL_NULL]
        assert out.column("x").null_count == 2
        assert out.column(1).to_pylist() == [1.0, 1.0, 2.0, 2.0]


def test_binary_and_set_operators_do_not_match_null_with_nul_string(ctx):
    from greptimedb_b200.plan import BinaryPlan, SetOpPlan
    lhs = lambda: node(ctx, ["x"], batch(["x"], [((None,), 1.0), (("a",), 1.0)]))
    rhs = lambda: node(ctx, ["x"], batch(["x"], [((NUL_NULL,), 2.0), (("a",), 2.0)]))
    out = BinaryPlan(ctx, "+", lhs(), rhs()).execute()
    assert out.column("x").to_pylist() == ["a", "a"] and out.column(2).to_pylist() == [3.0, 3.0]
    out = SetOpPlan(ctx, "and", lhs(), rhs()).execute()
    assert out.column("x").to_pylist() == ["a", "a"]


def test_scalar_of_one_nul_string_series_is_that_series(ctx):
    from greptimedb_b200.plan import ScalarPlan
    out = ScalarPlan(ctx, node(ctx, ["x"], batch(["x"], [((NUL_NULL,), 5.0)]))).execute()
    assert out.column(1).to_pylist() == [5.0, 5.0]


def hist_series(groups):
    return [(g + (le,), v) for g in groups for le, v in (("1", 1.0), ("+Inf", 2.0))]


def test_histogram_fold_keeps_tuples_apart_that_concatenate_alike(ctx):
    groups = [("a\x1f", "b"), ("a", "\x1fb")]
    out = node(ctx, ["x", "y", "le"], batch(["x", "y", "le"], hist_series(groups)), steps=1,
               histogram_quantile=0.5).execute()
    assert out.schema.names == ["ts", "prom_last_over_time(ts_range,val)", "x", "y"]
    assert list(zip(out.column("x").to_pylist(), out.column("y").to_pylist())) == [("a", "\x1fb"), ("a\x1f", "b")]


# ---- the order of sorted output: "" first, then NULL, then the other values --------------------------------------------
def test_sum_by_orders_empty_then_null_then_values(ctx):
    out = node(ctx, ["g"], batch(["g"], [(("a",), 1.0), ((None,), 2.0), (("",), 3.0)]), steps=1, aggregate="sum",
               by_columns=["g"]).execute()
    assert out.schema.names == ["g", "ts", "sum(prom_last_over_time)"]
    assert out.column("g").to_pylist() == ["", None, "a"] and out.column(2).to_pylist() == [3.0, 2.0, 1.0]


def test_histogram_fold_orders_empty_then_null_then_values(ctx):
    out = node(ctx, ["g", "le"], batch(["g", "le"], hist_series([("a",), (None,), ("",)])), steps=1,
               histogram_quantile=0.5).execute()
    assert out.column("g").to_pylist() == ["", None, "a"]


def test_sum_by_an_id_key_is_decimal_strings_in_string_order(ctx):
    from greptimedb_b200.plan import PromRangeExec
    b = pa.record_batch([pa.array([0, 1000, 0, 1000], pa.timestamp("ms")), pa.array([1.0, 2.0, 3.0, 4.0]),
                         pa.array([9, 9, 10, 10], pa.uint64())], names=["ts", "val", "__tsid"])
    ex = PromRangeExec(ctx, "prom_last_over_time", 1000, 1000, 1000, 10_000, "ts", "val", ["__tsid"], aggregate="sum",
                       by_columns=["__tsid"])
    ex.push(b)
    out = ex.execute()
    assert out.schema.field("__tsid").type == pa.string()
    assert out.column("__tsid").to_pylist() == ["10", "9"] and out.column(2).to_pylist() == [4.0, 2.0]


def test_or_has_real_nulls_where_a_side_lacks_a_tag(ctx):
    from greptimedb_b200.plan import SetOpPlan
    lhs = node(ctx, ["a"], batch(["a"], [(("x",), 1.0)]), steps=1)
    rhs = node(ctx, ["b"], batch(["b"], [(("y",), 2.0)]), steps=1)
    out = SetOpPlan(ctx, "or", lhs, rhs).execute()
    assert out.schema.names == ["ts", "a", "b", "prom_last_over_time(ts_range,val)"]
    assert out.column("a").to_pylist() == ["x", None] and out.column("b").to_pylist() == [None, "y"]
    assert out.column("a").null_count == 1 and out.column("b").null_count == 1
