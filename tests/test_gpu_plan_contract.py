"""GPU: what every plan node accepts from its child, in one table (DESIGN §1 a24-a27).

Each node over each kind of child either exports a batch (its column names, Arrow types and row count are pinned) or
refuses the child with a Plan error (its code and text are pinned).  The kinds are the shapes a node's contract speaks
of: one and two Float64 fields, an Int64 field, the Int32 of a calendar function, a count_values result and topk over
one, an id-keyed (__tsid) leaf, the EmptyMetric rows vector(1) and time(), and a child without columns.  Below the
table: the refusals with the texts the reference gives, and the paths each integer type is accepted on."""
import pyarrow as pa
import pytest

from tests import int64_oracle as io
from tests import multifield_plan_oracle as mp
from tests import test_gpu_int64 as t64
from tests import test_gpu_multifield_plan as tmf

pytestmark = pytest.mark.gpu

LOOKBACK = 300_000
START, END, STEP = 0, 120_000, 60_000
HOSTS = [("a", "1"), ("a", "+Inf"), ("b", "1"), ("b", "+Inf")]
VALUES = [[1, 1, 5], [2, 2, 2], [1, 3, 5], [3, 3, 3]]  # [series][step]: count_values has ties in its counts


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def _leaf(ctx, fields=("val",), val_type=pa.float64(), tsid=False):
    """the instant selector over four series on the grid START..END by STEP, tagged host and le (or a __tsid id)"""
    from greptimedb_b200.plan import PromRangeExec
    ts, cols = [], [[] for _ in fields]
    for s in range(len(HOSTS)):
        for k in range(3):
            ts.append(START + k * STEP)
            for f in range(len(fields)):
                cols[f].append(VALUES[s][k] * 10 ** f)
    arrays = [pa.array(ts, pa.timestamp("ms"))] + [pa.array(c, val_type) for c in cols]
    if tsid:
        tags = ["__tsid"]
        arrays.append(pa.array([7 * s + 3 for s in range(len(HOSTS)) for _ in range(3)], pa.uint64()))
    else:
        tags = ["host", "le"]
        arrays += [pa.array([h[i] for h in HOSTS for _ in range(3)]) for i in range(2)]
    ex = PromRangeExec(ctx, "", START, END, STEP, 0, "ts", list(fields), tags, lookback_delta=LOOKBACK)
    ex.push(pa.record_batch(arrays, names=["ts"] + list(fields) + tags))
    return ex


def children(ctx):
    from greptimedb_b200 import plan as P
    empty = lambda kind, **kw: P.EmptyMetricPlan(ctx, START, END, STEP, kind, **kw)
    return {
        "f64": lambda: _leaf(ctx),
        "f64x2": lambda: _leaf(ctx, ("val", "val2")),
        "i64": lambda: _leaf(ctx, val_type=pa.int64()),
        "hour": lambda: empty("none").function("hour"),
        "count_values": lambda: P.CountValuesPlan(ctx, "v", _leaf(ctx)),
        "topk_count_values": lambda: P.TopkPlan(ctx, "topk", 2, P.CountValuesPlan(ctx, "v", _leaf(ctx))),
        "tsid": lambda: _leaf(ctx, tsid=True),
        "vector1": lambda: empty("literal", literal=1.0),
        "time": lambda: empty("time"),
        "no_columns": lambda: P.HistogramQuantilePlan(ctx, 0.5, _leaf(ctx), le="nope"),
    }


def parents(ctx):
    from greptimedb_b200 import plan as P
    f64 = lambda: _leaf(ctx)
    return {
        "scalar": lambda c: P.ScalarPlan(ctx, c),
        "topk": lambda c: P.TopkPlan(ctx, "topk", 1, c),
        "sum": lambda c: P.AggregatePlan(ctx, "sum", c),
        "quantile": lambda c: P.AggregatePlan(ctx, "quantile", c, param=0.5),
        "group": lambda c: P.AggregatePlan(ctx, "group", c),
        "count_values": lambda c: P.CountValuesPlan(ctx, "w", c),
        "subquery": lambda c: P.SubqueryPlan(ctx, "prom_max_over_time", c, START, END, STEP, 2 * STEP),
        "histogram_quantile": lambda c: P.HistogramQuantilePlan(ctx, 0.5, c),
        "sort": lambda c: P.SortPlan(ctx, "sort", c),
        "sort_by_label": lambda c: P.SortPlan(ctx, "sort_by_label", c, ["host"]),
        "absent": lambda c: P.AbsentPlan(ctx, c, START, END, STEP, "ts", "value"),
        "label_replace": lambda c: P.LabelReplacePlan(ctx, c, "dst", "x$1", "host", "(.*)"),
        "label_join": lambda c: P.LabelJoinPlan(ctx, c, "dst", "-", "host", "le"),
        "fn_stage": lambda c: c.function("abs"),
        "arith_stage": lambda c: c.scalar_op("*", 2.0),
        "filter_stage": lambda c: c.scalar_op(">", 1.0),
        "unary_minus": lambda c: c.function("negative"),
        "arith_lhs": lambda c: P.BinaryPlan(ctx, "+", c, f64()),
        "arith_rhs": lambda c: P.BinaryPlan(ctx, "+", f64(), c),
        "filter_lhs": lambda c: P.BinaryPlan(ctx, ">", c, f64()),
        "filter_rhs": lambda c: P.BinaryPlan(ctx, ">", f64(), c),
        "and_lhs": lambda c: P.SetOpPlan(ctx, "and", c, f64()),
        "and_rhs": lambda c: P.SetOpPlan(ctx, "and", f64(), c),
        "or_lhs": lambda c: P.SetOpPlan(ctx, "or", c, f64()),
        "or_rhs": lambda c: P.SetOpPlan(ctx, "or", f64(), c),
        "unless_lhs": lambda c: P.SetOpPlan(ctx, "unless", c, f64()),
        "unless_rhs": lambda c: P.SetOpPlan(ctx, "unless", f64(), c),
    }


def outcome(make):
    """("error", code, text) of a refused plan, or ("ok", column names, Arrow types, rows) of its export"""
    from greptimedb_b200 import B2PError
    try:
        out = make().execute()
    except B2PError as e:
        return ("error", e.code, str(e).split(": ", 1)[1])
    return ("ok", out.schema.names, [str(t) for t in out.schema.types], out.num_rows)


# ---- the node x child table ---------------------------------------------------------------------------------------------
# Recorded from the plan layer before its child contracts were gathered into one place per node, and checked against
# DESIGN §1 a24-a27.  A cell missing here would fail the test: every node meets every kind of child.
OK, ERR = "ok", "error"
TS, F64, I64, I32, STR, U64 = "timestamp[ms]", "double", "int64", "int32", "string", "uint64"
EXPECTED = {
    ("scalar", "f64"): (OK, ["ts", "scalar(val)"], [TS, F64], 3),
    ("scalar", "f64x2"): (ERR, -1, "Multi fields calculation is not supported in scalar"),
    ("scalar", "i64"): (OK, ["ts", "scalar(val)"], [TS, F64], 3),
    ("scalar", "hour"): (ERR, -1, "GpuPromScalarExec: an Int32 value column is not supported by this node"),
    ("scalar", "count_values"): (ERR, -2, "scalar(): two rows of one series have a cell at the same step"),
    ("scalar", "topk_count_values"): (ERR, -2, "scalar(): two rows of one series have a cell at the same step"),
    ("scalar", "tsid"): (OK, ["ts", "scalar(val)"], [TS, F64], 3),
    ("scalar", "vector1"): (OK, ["time", "scalar(value)"], [TS, F64], 3),
    ("scalar", "time"): (OK, ["time", "scalar(time / Float64(1000))"], [TS, F64], 3),
    ("scalar", "no_columns"): (OK, ["ts", "scalar(val)"], [TS, F64], 3),
    ("topk", "f64"): (OK, ["val", "host", "le", "ts"], [F64, STR, STR, TS], 3),
    ("topk", "f64x2"): (ERR, -1, "Unsupported expr type: topk or bottomk on multi-value input"),
    ("topk", "i64"): (OK, ["val", "host", "le", "ts"], [I64, STR, STR, TS], 3),
    ("topk", "hour"): (OK, ["date_part(Utf8(\"hour\"),time)", "time"], [I32, TS], 3),
    ("topk", "count_values"): (OK, ["count(val)", "ts"], [F64, TS], 3),
    ("topk", "topk_count_values"): (OK, ["count(val)", "ts"], [F64, TS], 3),
    ("topk", "tsid"): (ERR, -1, "topk: an id-keyed (__tsid) child has no label values to order by"),
    ("topk", "vector1"): (OK, ["value", "time"], [F64, TS], 3),
    ("topk", "time"): (OK, ["time / Float64(1000)", "time"], [F64, TS], 3),
    ("topk", "no_columns"): (OK, ["val", "ts"], [F64, TS], 0),
    ("sum", "f64"): (OK, ["ts", "sum(val)"], [TS, F64], 3),
    ("sum", "f64x2"): (OK, ["ts", "sum(val)", "sum(val2)"], [TS, F64, F64], 3),
    ("sum", "i64"): (OK, ["ts", "sum(val)"], [TS, I64], 3),
    ("sum", "hour"): (ERR, -1, "GpuPromAggregateExec: an Int32 value column is not supported by this node"),
    ("sum", "count_values"): (OK, ["ts", "sum(count(val))"], [TS, F64], 3),
    ("sum", "topk_count_values"): (OK, ["ts", "sum(count(val))"], [TS, F64], 3),
    ("sum", "tsid"): (OK, ["ts", "sum(val)"], [TS, F64], 3),
    ("sum", "vector1"): (OK, ["time", "sum(value)"], [TS, F64], 3),
    ("sum", "time"): (OK, ["time", "sum(time / Float64(1000))"], [TS, F64], 3),
    ("sum", "no_columns"): (OK, ["ts", "sum(val)"], [TS, F64], 0),
    ("quantile", "f64"): (OK, ["ts", "quantile(Float64(0.5),val)"], [TS, F64], 3),
    ("quantile", "f64x2"): (OK, ["ts", "quantile(Float64(0.5),val)", "quantile(Float64(0.5),val2)"], [TS, F64, F64], 3),
    ("quantile", "i64"): (OK, ["ts", "quantile(Float64(0.5),val)"], [TS, F64], 3),
    ("quantile", "hour"): (ERR, -1, "GpuPromAggregateExec: an Int32 value column is not supported by this node"),
    ("quantile", "count_values"): (OK, ["ts", "quantile(Float64(0.5),count(val))"], [TS, F64], 3),
    ("quantile", "topk_count_values"): (OK, ["ts", "quantile(Float64(0.5),count(val))"], [TS, F64], 3),
    ("quantile", "tsid"): (OK, ["ts", "quantile(Float64(0.5),val)"], [TS, F64], 3),
    ("quantile", "vector1"): (OK, ["time", "quantile(Float64(0.5),value)"], [TS, F64], 3),
    ("quantile", "time"): (OK, ["time", "quantile(Float64(0.5),time / Float64(1000))"], [TS, F64], 3),
    ("quantile", "no_columns"): (OK, ["ts", "quantile(Float64(0.5),val)"], [TS, F64], 0),
    ("group", "f64"): (OK, ["ts", "max(Float64(1))"], [TS, F64], 3),
    ("group", "f64x2"): (ERR, -1, "Multi fields calculation is not supported in group()"),
    ("group", "i64"): (OK, ["ts", "max(Float64(1))"], [TS, F64], 3),
    ("group", "hour"): (ERR, -1, "GpuPromAggregateExec: an Int32 value column is not supported by this node"),
    ("group", "count_values"): (OK, ["ts", "max(Float64(1))"], [TS, F64], 3),
    ("group", "topk_count_values"): (OK, ["ts", "max(Float64(1))"], [TS, F64], 3),
    ("group", "tsid"): (OK, ["ts", "max(Float64(1))"], [TS, F64], 3),
    ("group", "vector1"): (OK, ["time", "max(Float64(1))"], [TS, F64], 3),
    ("group", "time"): (OK, ["time", "max(Float64(1))"], [TS, F64], 3),
    ("group", "no_columns"): (OK, ["ts", "max(Float64(1))"], [TS, F64], 0),
    ("count_values", "f64"): (OK, ["count(val)", "ts", "w"], [I64, TS, F64], 9),
    ("count_values", "f64x2"): (ERR, -1, "Unsupported expr type: count_values on multi-value input"),
    ("count_values", "i64"): (OK, ["count(val)", "ts", "w"], [I64, TS, I64], 9),
    ("count_values", "hour"): (ERR, -1, "GpuPromCountValuesExec: an Int32 value column is not supported by this node"),
    ("count_values", "count_values"): (OK, ["count(count(val))", "ts", "w"], [I64, TS, F64], 6),
    ("count_values", "topk_count_values"): (OK, ["count(count(val))", "ts", "w"], [I64, TS, F64], 6),
    ("count_values", "tsid"): (OK, ["count(val)", "ts", "w"], [I64, TS, F64], 9),
    ("count_values", "vector1"): (OK, ["count(value)", "time", "w"], [I64, TS, F64], 3),
    ("count_values", "time"): (OK, ["count(time / Float64(1000))", "time", "w"], [I64, TS, F64], 3),
    ("count_values", "no_columns"): (OK, ["count(val)", "ts", "w"], [I64, TS, F64], 0),
    ("subquery", "f64"): (OK, ["ts", "prom_max_over_time(ts_range,val)", "host", "le"], [TS, F64, STR, STR], 12),
    ("subquery", "f64x2"):
        (OK, ["ts", "prom_max_over_time(ts_range,val)", "prom_max_over_time(ts_range,val2)", "host", "le"], [TS, F64, F64, STR, STR], 12),
    ("subquery", "i64"): (ERR, -1, "GpuPromSubqueryExec: an Int64 value column is not supported by this node"),
    ("subquery", "hour"): (ERR, -1, "GpuPromSubqueryExec: an Int32 value column is not supported by this node"),
    ("subquery", "count_values"): (OK, ["ts", "prom_max_over_time(ts_range,count(val))"], [TS, F64], 9),
    ("subquery", "topk_count_values"): (OK, ["ts", "prom_max_over_time(ts_range,count(val))"], [TS, F64], 7),
    ("subquery", "tsid"): (OK, ["ts", "prom_max_over_time(ts_range,val)", "__tsid"], [TS, F64, U64], 12),
    ("subquery", "vector1"): (OK, ["time", "prom_max_over_time(time_range,value)"], [TS, F64], 3),
    ("subquery", "time"): (OK, ["time", "prom_max_over_time(time_range,time / Float64(1000))"], [TS, F64], 3),
    ("subquery", "no_columns"): (OK, ["ts", "prom_max_over_time(ts_range,val)"], [TS, F64], 0),
    ("histogram_quantile", "f64"): (OK, ["ts", "val", "host"], [TS, F64, STR], 6),
    ("histogram_quantile", "f64x2"):
        (ERR, -1, "GpuPromHistogramFoldExec: a multi-field child is not supported by this node"),
    ("histogram_quantile", "i64"):
        (ERR, -1, "GpuPromHistogramFoldExec: an Int64 value column is not supported by this node"),
    ("histogram_quantile", "hour"):
        (ERR, -1, "GpuPromHistogramFoldExec: an Int32 value column is not supported by this node"),
    ("histogram_quantile", "count_values"):
        (ERR, -1, "GpuPromHistogramFoldExec: a count_values child is not supported by this node"),
    ("histogram_quantile", "topk_count_values"): (OK, [], [], 0),
    ("histogram_quantile", "tsid"):
        (ERR, -1, "GpuPromHistogramFoldExec: an id-keyed (__tsid) child carries no le label"),
    ("histogram_quantile", "vector1"): (OK, [], [], 0),
    ("histogram_quantile", "time"): (OK, [], [], 0),
    ("histogram_quantile", "no_columns"): (OK, [], [], 0),
    ("sort", "f64"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 12),
    ("sort", "f64x2"): (OK, ["ts", "val", "val2", "host", "le"], [TS, F64, F64, STR, STR], 12),
    ("sort", "i64"): (OK, ["ts", "val", "host", "le"], [TS, I64, STR, STR], 12),
    ("sort", "hour"): (OK, ["time", "date_part(Utf8(\"hour\"),time)"], [TS, I32], 3),
    ("sort", "count_values"): (ERR, -1, "GpuPromSortExec: a count_values child is not supported by this node"),
    ("sort", "topk_count_values"): (OK, ["ts", "count(val)"], [TS, F64], 6),
    ("sort", "tsid"): (OK, ["ts", "val", "__tsid"], [TS, F64, U64], 12),
    ("sort", "vector1"): (OK, ["time", "value"], [TS, F64], 3),
    ("sort", "time"): (OK, ["time", "time / Float64(1000)"], [TS, F64], 3),
    ("sort", "no_columns"): (OK, [], [], 0),
    ("sort_by_label", "f64"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 12),
    ("sort_by_label", "f64x2"): (OK, ["ts", "val", "val2", "host", "le"], [TS, F64, F64, STR, STR], 12),
    ("sort_by_label", "i64"): (OK, ["ts", "val", "host", "le"], [TS, I64, STR, STR], 12),
    ("sort_by_label", "hour"): (ERR, -1, "GpuPromSortExec: No field named host"),
    ("sort_by_label", "count_values"): (ERR, -1, "GpuPromSortExec: a count_values child is not supported by this node"),
    ("sort_by_label", "topk_count_values"): (ERR, -1, "GpuPromSortExec: No field named host"),
    ("sort_by_label", "tsid"): (ERR, -1, "GpuPromSortExec: an id-keyed (__tsid) child has no label values to sort by"),
    ("sort_by_label", "vector1"): (ERR, -1, "GpuPromSortExec: No field named host"),
    ("sort_by_label", "time"): (ERR, -1, "GpuPromSortExec: No field named host"),
    ("sort_by_label", "no_columns"): (OK, [], [], 0),
    ("absent", "f64"): (OK, ["ts", "value"], [TS, F64], 0),
    ("absent", "f64x2"): (OK, ["ts", "value"], [TS, F64], 0),
    ("absent", "i64"): (OK, ["ts", "value"], [TS, F64], 0),
    ("absent", "hour"): (OK, ["ts", "value"], [TS, F64], 0),
    ("absent", "count_values"): (OK, ["ts", "value"], [TS, F64], 0),
    ("absent", "topk_count_values"): (OK, ["ts", "value"], [TS, F64], 0),
    ("absent", "tsid"): (OK, ["ts", "value"], [TS, F64], 0),
    ("absent", "vector1"): (OK, ["ts", "value"], [TS, F64], 0),
    ("absent", "time"): (OK, ["ts", "value"], [TS, F64], 0),
    ("absent", "no_columns"): (OK, ["ts", "value"], [TS, F64], 3),
    ("label_replace", "f64"): (OK, ["ts", "val", "dst", "host", "le"], [TS, F64, STR, STR, STR], 12),
    ("label_replace", "f64x2"): (OK, ["ts", "val", "val2", "dst", "host", "le"], [TS, F64, F64, STR, STR, STR], 12),
    ("label_replace", "i64"): (OK, ["ts", "val", "dst", "host", "le"], [TS, I64, STR, STR, STR], 12),
    ("label_replace", "hour"): (OK, ["time", "date_part(Utf8(\"hour\"),time)", "dst"], [TS, I32, STR], 3),
    ("label_replace", "count_values"):
        (ERR, -1, "GpuPromLabelExec: a count_values child is not supported by this node"),
    ("label_replace", "topk_count_values"): (OK, ["ts", "count(val)", "dst"], [TS, F64, STR], 6),
    ("label_replace", "tsid"): (ERR, -1, "GpuPromLabelExec: an id-keyed (__tsid) child has no label values to rewrite"),
    ("label_replace", "vector1"): (OK, ["time", "value", "dst"], [TS, F64, STR], 3),
    ("label_replace", "time"): (OK, ["time", "time / Float64(1000)", "dst"], [TS, F64, STR], 3),
    ("label_replace", "no_columns"): (OK, [], [], 0),
    ("label_join", "f64"): (OK, ["ts", "val", "dst", "host", "le"], [TS, F64, STR, STR, STR], 12),
    ("label_join", "f64x2"): (OK, ["ts", "val", "val2", "dst", "host", "le"], [TS, F64, F64, STR, STR, STR], 12),
    ("label_join", "i64"): (OK, ["ts", "val", "dst", "host", "le"], [TS, I64, STR, STR, STR], 12),
    ("label_join", "hour"): (OK, ["time", "date_part(Utf8(\"hour\"),time)", "dst"], [TS, I32, STR], 3),
    ("label_join", "count_values"): (ERR, -1, "GpuPromLabelExec: a count_values child is not supported by this node"),
    ("label_join", "topk_count_values"): (OK, ["ts", "count(val)", "dst"], [TS, F64, STR], 6),
    ("label_join", "tsid"): (ERR, -1, "GpuPromLabelExec: an id-keyed (__tsid) child has no label values to rewrite"),
    ("label_join", "vector1"): (OK, ["time", "value", "dst"], [TS, F64, STR], 3),
    ("label_join", "time"): (OK, ["time", "time / Float64(1000)", "dst"], [TS, F64, STR], 3),
    ("label_join", "no_columns"): (OK, [], [], 0),
    ("fn_stage", "f64"): (OK, ["ts", "abs(val)", "host", "le"], [TS, F64, STR, STR], 12),
    ("fn_stage", "f64x2"): (OK, ["ts", "abs(val)", "abs(val2)", "host", "le"], [TS, F64, F64, STR, STR], 12),
    ("fn_stage", "i64"): (OK, ["ts", "abs(val)", "host", "le"], [TS, F64, STR, STR], 12),
    ("fn_stage", "hour"): (OK, ["time", "abs(date_part(Utf8(\"hour\"),time))"], [TS, F64], 3),
    ("fn_stage", "count_values"): (OK, ["abs(count(val))", "ts", "v"], [F64, TS, F64], 9),
    ("fn_stage", "topk_count_values"): (OK, ["abs(count(val))", "ts"], [F64, TS], 6),
    ("fn_stage", "tsid"): (OK, ["ts", "abs(val)", "__tsid"], [TS, F64, U64], 12),
    ("fn_stage", "vector1"): (OK, ["time", "abs(value)"], [TS, F64], 3),
    ("fn_stage", "time"): (OK, ["time", "abs(time / Float64(1000))"], [TS, F64], 3),
    ("fn_stage", "no_columns"): (OK, [], [], 0),
    ("arith_stage", "f64"): (OK, ["ts", "val * Float64(2)", "host", "le"], [TS, F64, STR, STR], 12),
    ("arith_stage", "f64x2"):
        (OK, ["ts", "val * Float64(2)", "val2 * Float64(2)", "host", "le"], [TS, F64, F64, STR, STR], 12),
    ("arith_stage", "i64"): (OK, ["ts", "val * Float64(2)", "host", "le"], [TS, F64, STR, STR], 12),
    ("arith_stage", "hour"): (OK, ["time", "date_part(Utf8(\"hour\"),time) * Float64(2)"], [TS, F64], 3),
    ("arith_stage", "count_values"): (OK, ["count(val) * Float64(2)", "ts", "v"], [F64, TS, F64], 9),
    ("arith_stage", "topk_count_values"): (OK, ["count(val) * Float64(2)", "ts"], [F64, TS], 6),
    ("arith_stage", "tsid"): (OK, ["ts", "val * Float64(2)", "__tsid"], [TS, F64, U64], 12),
    ("arith_stage", "vector1"): (OK, ["time", "value * Float64(2)"], [TS, F64], 3),
    ("arith_stage", "time"): (OK, ["time", "time / Float64(1000) * Float64(2)"], [TS, F64], 3),
    ("arith_stage", "no_columns"): (OK, [], [], 0),
    ("filter_stage", "f64"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 9),
    ("filter_stage", "f64x2"): (ERR, -1, "Unsupported expr type: filter on multi-value input"),
    ("filter_stage", "i64"):
        (ERR, -1, "a filtering comparison over an Int64 value column is not supported by this node"),
    ("filter_stage", "hour"): (OK, ["time", "date_part(Utf8(\"hour\"),time)"], [TS, I32], 0),
    ("filter_stage", "count_values"): (OK, ["count(val)", "ts", "v"], [F64, TS, F64], 3),
    ("filter_stage", "topk_count_values"): (OK, ["count(val)", "ts"], [F64, TS], 3),
    ("filter_stage", "tsid"): (OK, ["ts", "val", "__tsid"], [TS, F64, U64], 9),
    ("filter_stage", "vector1"): (OK, ["time", "value"], [TS, F64], 0),
    ("filter_stage", "time"): (OK, ["time", "time / Float64(1000)"], [TS, F64], 2),
    ("filter_stage", "no_columns"): (OK, [], [], 0),
    ("unary_minus", "f64"): (OK, ["ts", "(- val)", "host", "le"], [TS, F64, STR, STR], 12),
    ("unary_minus", "f64x2"): (OK, ["ts", "(- val)", "(- val2)", "host", "le"], [TS, F64, F64, STR, STR], 12),
    ("unary_minus", "i64"): (ERR, -1, "unary minus over an integer value column is not supported by this node"),
    ("unary_minus", "hour"): (ERR, -1, "unary minus over an integer value column is not supported by this node"),
    ("unary_minus", "count_values"): (OK, ["(- count(val))", "ts", "v"], [F64, TS, F64], 9),
    ("unary_minus", "topk_count_values"): (OK, ["(- count(val))", "ts"], [F64, TS], 6),
    ("unary_minus", "tsid"): (OK, ["ts", "(- val)", "__tsid"], [TS, F64, U64], 12),
    ("unary_minus", "vector1"): (OK, ["time", "(- value)"], [TS, F64], 3),
    ("unary_minus", "time"): (OK, ["time", "(- time / Float64(1000))"], [TS, F64], 3),
    ("unary_minus", "no_columns"): (OK, [], [], 0),
    ("arith_lhs", "f64"): (OK, ["host", "le", "ts", "val + val"], [STR, STR, TS, F64], 12),
    ("arith_lhs", "f64x2"): (OK, ["host", "le", "ts", "val + val"], [STR, STR, TS, F64], 12),
    ("arith_lhs", "i64"): (OK, ["host", "le", "ts", "val + val"], [STR, STR, TS, F64], 12),
    ("arith_lhs", "hour"): (OK, ["host", "le", "ts", "date_part(Utf8(\"hour\"),time) + val"], [STR, STR, TS, F64], 12),
    ("arith_lhs", "count_values"): (OK, ["host", "le", "ts", "count(val) + val"], [STR, STR, TS, F64], 36),
    ("arith_lhs", "topk_count_values"): (OK, ["host", "le", "ts", "count(val) + val"], [STR, STR, TS, F64], 24),
    ("arith_lhs", "tsid"): (ERR, -1, "No field named host"),
    ("arith_lhs", "vector1"): (OK, ["host", "le", "ts", "value + val"], [STR, STR, TS, F64], 12),
    ("arith_lhs", "time"): (OK, ["host", "le", "ts", "time / Float64(1000) + val"], [STR, STR, TS, F64], 12),
    ("arith_lhs", "no_columns"): (OK, ["host", "le", "ts", "val + val"], [STR, STR, TS, F64], 0),
    ("arith_rhs", "f64"): (OK, ["host", "le", "ts", "val + val"], [STR, STR, TS, F64], 12),
    ("arith_rhs", "f64x2"): (OK, ["host", "le", "ts", "val + val"], [STR, STR, TS, F64], 12),
    ("arith_rhs", "i64"): (OK, ["host", "le", "ts", "val + val"], [STR, STR, TS, F64], 12),
    ("arith_rhs", "hour"): (OK, ["time", "val + date_part(Utf8(\"hour\"),time)"], [TS, F64], 12),
    ("arith_rhs", "count_values"): (OK, ["ts", "val + count(val)"], [TS, F64], 36),
    ("arith_rhs", "topk_count_values"): (OK, ["ts", "val + count(val)"], [TS, F64], 24),
    ("arith_rhs", "tsid"): (ERR, -1, "No field named __tsid"),
    ("arith_rhs", "vector1"): (OK, ["time", "val + value"], [TS, F64], 12),
    ("arith_rhs", "time"): (OK, ["time", "val + time / Float64(1000)"], [TS, F64], 12),
    ("arith_rhs", "no_columns"): (OK, ["ts", "val + val"], [TS, F64], 0),
    ("filter_lhs", "f64"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 0),
    ("filter_lhs", "f64x2"): (OK, ["ts", "val", "val2", "host", "le"], [TS, F64, F64, STR, STR], 0),
    ("filter_lhs", "i64"): (ERR, -1, "a filtering comparison over an Int64 value column is not supported by this node"),
    ("filter_lhs", "hour"): (OK, ["time", "date_part(Utf8(\"hour\"),time)"], [TS, I32], 0),
    ("filter_lhs", "count_values"): (OK, ["count(val)", "ts", "v"], [I64, TS, F64], 3),
    ("filter_lhs", "topk_count_values"): (OK, ["count(val)", "ts"], [F64, TS], 3),
    ("filter_lhs", "tsid"): (ERR, -1, "No field named host"),
    ("filter_lhs", "vector1"):
        (ERR, -1, "GpuPromBinaryExec: a filtering comparison with a literal EmptyMetric lhs against a vector is not supported by this node"),
    ("filter_lhs", "time"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 8),
    ("filter_lhs", "no_columns"): (OK, [], [], 0),
    ("filter_rhs", "f64"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 0),
    ("filter_rhs", "f64x2"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 0),
    ("filter_rhs", "i64"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 0),
    ("filter_rhs", "hour"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 12),
    ("filter_rhs", "count_values"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 24),
    ("filter_rhs", "topk_count_values"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 15),
    ("filter_rhs", "tsid"): (ERR, -1, "No field named __tsid"),
    ("filter_rhs", "vector1"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 9),
    ("filter_rhs", "time"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 4),
    ("filter_rhs", "no_columns"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 0),
    ("and_lhs", "f64"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 12),
    ("and_lhs", "f64x2"): (ERR, -1, "Multi fields calculation is not supported in AND operator"),
    ("and_lhs", "i64"): (OK, ["ts", "val", "host", "le"], [TS, I64, STR, STR], 12),
    ("and_lhs", "hour"): (ERR, -1, "set operator `and`: the key columns of the two sides differ: [] vs [host, le]"),
    ("and_lhs", "count_values"):
        (ERR, -1, "set operator `and`: the key columns of the two sides differ: [] vs [host, le]"),
    ("and_lhs", "topk_count_values"):
        (ERR, -1, "set operator `and`: the key columns of the two sides differ: [] vs [host, le]"),
    ("and_lhs", "tsid"): (ERR, -1, "set operator `and`: an id-keyed (__tsid) side has no label values to match"),
    ("and_lhs", "vector1"): (ERR, -1, "set operator `and`: the key columns of the two sides differ: [] vs [host, le]"),
    ("and_lhs", "time"): (ERR, -1, "set operator `and`: the key columns of the two sides differ: [] vs [host, le]"),
    ("and_lhs", "no_columns"):
        (ERR, -1, "set operator `and`: the key columns of the two sides differ: [] vs [host, le]"),
    ("and_rhs", "f64"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 12),
    ("and_rhs", "f64x2"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 12),
    ("and_rhs", "i64"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 12),
    ("and_rhs", "hour"): (ERR, -1, "set operator `and`: the key columns of the two sides differ: [host, le] vs []"),
    ("and_rhs", "count_values"):
        (ERR, -1, "set operator `and`: the key columns of the two sides differ: [host, le] vs []"),
    ("and_rhs", "topk_count_values"):
        (ERR, -1, "set operator `and`: the key columns of the two sides differ: [host, le] vs []"),
    ("and_rhs", "tsid"): (ERR, -1, "set operator `and`: an id-keyed (__tsid) side has no label values to match"),
    ("and_rhs", "vector1"): (ERR, -1, "set operator `and`: the key columns of the two sides differ: [host, le] vs []"),
    ("and_rhs", "time"): (ERR, -1, "set operator `and`: the key columns of the two sides differ: [host, le] vs []"),
    ("and_rhs", "no_columns"):
        (ERR, -1, "set operator `and`: the key columns of the two sides differ: [host, le] vs []"),
    ("or_lhs", "f64"): (OK, ["ts", "host", "le", "val"], [TS, STR, STR, F64], 12),
    ("or_lhs", "f64x2"):
        (ERR, -1, "Attempt to combine two tables with different column sets, left: [\"val\", \"val2\"], right: [\"val\"]"),
    ("or_lhs", "i64"): (ERR, -1, "set operator `or`: an Int64 value column is not supported by this node"),
    ("or_lhs", "hour"):
        (ERR, -1, "set operator `or`: an Int32 value column against another type is not supported by this node"),
    ("or_lhs", "count_values"): (OK, ["ts", "count(val)", "host", "le"], [TS, F64, STR, STR], 21),
    ("or_lhs", "topk_count_values"): (OK, ["ts", "count(val)", "host", "le"], [TS, F64, STR, STR], 18),
    ("or_lhs", "tsid"): (ERR, -1, "set operator `or`: an id-keyed (__tsid) side has no label values to match"),
    ("or_lhs", "vector1"): (OK, ["time", "host", "le", "value"], [TS, STR, STR, F64], 15),
    ("or_lhs", "time"): (OK, ["time", "host", "le", "time / Float64(1000)"], [TS, STR, STR, F64], 15),
    ("or_lhs", "no_columns"): (OK, ["ts", "host", "le", "val"], [TS, STR, STR, F64], 12),
    ("or_rhs", "f64"): (OK, ["ts", "host", "le", "val"], [TS, STR, STR, F64], 12),
    ("or_rhs", "f64x2"):
        (ERR, -1, "Attempt to combine two tables with different column sets, left: [\"val\"], right: [\"val\", \"val2\"]"),
    ("or_rhs", "i64"): (ERR, -1, "set operator `or`: an Int64 value column is not supported by this node"),
    ("or_rhs", "hour"):
        (ERR, -1, "set operator `or`: an Int32 value column against another type is not supported by this node"),
    ("or_rhs", "count_values"): (OK, ["ts", "host", "le", "val"], [TS, STR, STR, F64], 15),
    ("or_rhs", "topk_count_values"): (OK, ["ts", "host", "le", "val"], [TS, STR, STR, F64], 15),
    ("or_rhs", "tsid"): (ERR, -1, "set operator `or`: an id-keyed (__tsid) side has no label values to match"),
    ("or_rhs", "vector1"): (OK, ["ts", "host", "le", "val"], [TS, STR, STR, F64], 15),
    ("or_rhs", "time"): (OK, ["ts", "host", "le", "val"], [TS, STR, STR, F64], 15),
    ("or_rhs", "no_columns"): (OK, ["ts", "host", "le", "val"], [TS, STR, STR, F64], 12),
    ("unless_lhs", "f64"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 0),
    ("unless_lhs", "f64x2"): (ERR, -1, "Multi fields calculation is not supported in AND operator"),
    ("unless_lhs", "i64"): (OK, ["ts", "val", "host", "le"], [TS, I64, STR, STR], 0),
    ("unless_lhs", "hour"):
        (ERR, -1, "set operator `unless`: the key columns of the two sides differ: [] vs [host, le]"),
    ("unless_lhs", "count_values"):
        (ERR, -1, "set operator `unless`: the key columns of the two sides differ: [] vs [host, le]"),
    ("unless_lhs", "topk_count_values"):
        (ERR, -1, "set operator `unless`: the key columns of the two sides differ: [] vs [host, le]"),
    ("unless_lhs", "tsid"): (ERR, -1, "set operator `unless`: an id-keyed (__tsid) side has no label values to match"),
    ("unless_lhs", "vector1"):
        (ERR, -1, "set operator `unless`: the key columns of the two sides differ: [] vs [host, le]"),
    ("unless_lhs", "time"):
        (ERR, -1, "set operator `unless`: the key columns of the two sides differ: [] vs [host, le]"),
    ("unless_lhs", "no_columns"):
        (ERR, -1, "set operator `unless`: the key columns of the two sides differ: [] vs [host, le]"),
    ("unless_rhs", "f64"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 0),
    ("unless_rhs", "f64x2"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 0),
    ("unless_rhs", "i64"): (OK, ["ts", "val", "host", "le"], [TS, F64, STR, STR], 0),
    ("unless_rhs", "hour"):
        (ERR, -1, "set operator `unless`: the key columns of the two sides differ: [host, le] vs []"),
    ("unless_rhs", "count_values"):
        (ERR, -1, "set operator `unless`: the key columns of the two sides differ: [host, le] vs []"),
    ("unless_rhs", "topk_count_values"):
        (ERR, -1, "set operator `unless`: the key columns of the two sides differ: [host, le] vs []"),
    ("unless_rhs", "tsid"): (ERR, -1, "set operator `unless`: an id-keyed (__tsid) side has no label values to match"),
    ("unless_rhs", "vector1"):
        (ERR, -1, "set operator `unless`: the key columns of the two sides differ: [host, le] vs []"),
    ("unless_rhs", "time"):
        (ERR, -1, "set operator `unless`: the key columns of the two sides differ: [host, le] vs []"),
    ("unless_rhs", "no_columns"):
        (ERR, -1, "set operator `unless`: the key columns of the two sides differ: [host, le] vs []"),
}


def _cells():
    return [(p, c) for p in ("scalar", "topk", "sum", "quantile", "group", "count_values", "subquery",
                             "histogram_quantile", "sort", "sort_by_label", "absent", "label_replace", "label_join",
                             "fn_stage", "arith_stage", "filter_stage", "unary_minus", "arith_lhs", "arith_rhs",
                             "filter_lhs", "filter_rhs", "and_lhs", "and_rhs", "or_lhs", "or_rhs", "unless_lhs",
                             "unless_rhs")
            for c in ("f64", "f64x2", "i64", "hour", "count_values", "topk_count_values", "tsid", "vector1", "time",
                      "no_columns")]


@pytest.mark.parametrize("parent,child", _cells())
def test_node_over_child(ctx, parent, child):
    make_child, make_parent = children(ctx)[child], parents(ctx)[parent]
    got = outcome(lambda: make_parent(make_child()))
    assert got == EXPECTED[(parent, child)], got


def test_and_keeps_topk_rows_of_count_values_that_differ_in_the_counted_value(ctx):
    """`topk(3, count_values("v", x)) and on() vector(1)`: the rows share their (empty) label tuple and tie on some
    counts, but the counted value is a column of theirs, so left.distinct() keeps them all"""
    from greptimedb_b200 import plan as P
    top = P.TopkPlan(ctx, "topk", 3, P.CountValuesPlan(ctx, "v", _leaf(ctx)))
    alone = top.execute()
    top = P.TopkPlan(ctx, "topk", 3, P.CountValuesPlan(ctx, "v", _leaf(ctx)))
    out = P.SetOpPlan(ctx, "and", top, P.EmptyMetricPlan(ctx, START, END, STEP, "literal", literal=1.0), on=[]).execute()
    assert out.num_rows == alone.num_rows
    assert sorted(zip(out.column(1).cast(pa.int64()).to_pylist(), out.column(0).to_pylist())) == \
        sorted(zip(alone.column(1).cast(pa.int64()).to_pylist(), alone.column(0).to_pylist()))


# ---- the refusals by their texts, and the paths each integer type is accepted on ------------------------------------------
def test_int64_refusals(ctx):
    leaf, GOLDEN = t64.leaf, t64.GOLDEN
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import (BinaryPlan, HistogramQuantilePlan, SetOpPlan, SortPlan, SubqueryPlan)
    rows = GOLDEN["tables"]["sort"]["rows"]
    with pytest.raises(B2PError, match="field column val is not Float64"):
        leaf(ctx, rows, function="prom_rate")
    cases = [
        (lambda: BinaryPlan(ctx, "+", leaf(ctx, rows), leaf(ctx, rows)),
         "a binary operator between two Int64 value columns is not supported"),
        (lambda: BinaryPlan(ctx, ">", leaf(ctx, rows), leaf(ctx, rows, val_type=pa.float64())),
         "a filtering comparison over an Int64 value column is not supported"),
        (lambda: leaf(ctx, rows).scalar_op(">", 1.0), "a filtering comparison over an Int64 value column is not supported"),
        (lambda: SetOpPlan(ctx, "or", leaf(ctx, rows), leaf(ctx, rows)), "an Int64 value column is not supported"),
        (lambda: SubqueryPlan(ctx, "prom_max_over_time", leaf(ctx, rows), 0, 15_000, 5_000, 10_000),
         "GpuPromSubqueryExec: an Int64 value column is not supported"),
        (lambda: HistogramQuantilePlan(ctx, 0.5, leaf(ctx, rows), le="idc"),
         "GpuPromHistogramFoldExec: an Int64 value column is not supported"),
    ]
    for make, msg in cases:
        with pytest.raises(B2PError, match=msg):
            make().execute()
    # a mixed two-field node under sort
    from greptimedb_b200.plan import PromRangeExec
    b = pa.record_batch([pa.array([0], pa.timestamp("ms")), pa.array(["a"]), pa.array([1.0]), pa.array([1], pa.int64())],
                        names=["ts", "host", "f", "i"])
    ex = PromRangeExec(ctx, "", 0, 5000, 5000, 0, "ts", ["f", "i"], ["host"], lookback_delta=io.LOOKBACK)
    ex.push(b)
    with pytest.raises(B2PError, match="a multi-field child with an Int64 value column"):
        SortPlan(ctx, "sort", ex).execute()


def test_int32_refusals_and_accepted_paths(ctx):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import (AbsentPlan, AggregatePlan, BinaryPlan, CountValuesPlan, EmptyMetricPlan,
                                      HistogramQuantilePlan, ScalarPlan, SetOpPlan, SortPlan, SubqueryPlan, TopkPlan)

    def cal():
        return EmptyMetricPlan(ctx, 0, 120_000, 60_000, "none").function("hour")

    def f64():
        return EmptyMetricPlan(ctx, 0, 120_000, 60_000, "time")

    refused = {
        "GpuPromAggregateExec: an Int32": lambda: AggregatePlan(ctx, "sum", cal()),
        "GpuPromCountValuesExec: an Int32": lambda: CountValuesPlan(ctx, "v", cal()),
        "GpuPromScalarExec: an Int32": lambda: ScalarPlan(ctx, cal()),
        "GpuPromSubqueryExec: an Int32": lambda: SubqueryPlan(
            ctx, "prom_max_over_time", EmptyMetricPlan(ctx, -60_000, 120_000, 60_000, "none").function("hour"),
            0, 120_000, 60_000, 120_000),
        "GpuPromHistogramFoldExec: an Int32": lambda: HistogramQuantilePlan(ctx, 0.5, cal()),
        "an Int32 value column against another type": lambda: SetOpPlan(ctx, "or", cal(), f64()),
        "between two integer value columns": lambda: BinaryPlan(ctx, "+", cal(), cal()),
        "unary minus over an integer value column": lambda: cal().function("negative"),
    }
    for what, make in refused.items():
        with pytest.raises(B2PError) as ei:
            make().execute()
        assert ei.value.code == -1 and what in str(ei.value), (what, str(ei.value))
    hours = [0, 0, 0]
    typ = lambda out, name: out.schema.field(name).type
    val = 'date_part(Utf8("hour"),time)'
    # stages coerce to Float64; a filter keeps Int32
    assert typ(cal().scalar_op("+", 1.0).execute(), val + " + Float64(1)") == pa.float64()
    assert typ(cal().function("abs").execute(), "abs(" + val + ")") == pa.float64()
    assert typ(cal().scalar_op(">=", 0.0).execute(), val) == pa.int32()
    # against a Float64 side: arithmetic and `bool` give Float64, a vector-vector filter keeps the Int32 lhs
    assert typ(BinaryPlan(ctx, "*", cal(), f64()).execute(), val + " * time / Float64(1000)") == pa.float64()
    assert typ(BinaryPlan(ctx, "<=", cal(), f64(), return_bool=True).execute(), val + " <= time / Float64(1000)") == pa.float64()
    out = BinaryPlan(ctx, "<=", cal(), f64()).execute()
    assert typ(out, val) == pa.int32() and out.column(val).to_pylist() == hours
    # and / unless keep the lhs; `or` of two Int32 sides stays Int32
    assert typ(SetOpPlan(ctx, "and", cal(), f64()).execute(), val) == pa.int32()
    assert typ(SetOpPlan(ctx, "unless", cal(), f64()).execute(), val) == pa.int32()
    assert typ(SetOpPlan(ctx, "or", cal(), cal()).execute(), val) == pa.int32()
    # sort, topk / bottomk and absent
    out = SortPlan(ctx, "sort_desc", cal()).execute()
    assert typ(out, val) == pa.int32() and out.column(val).to_pylist() == hours
    for op in ("topk", "bottomk"):
        out = TopkPlan(ctx, op, 1, cal()).execute()
        assert typ(out, val) == pa.int32() and out.column(val).to_pylist() == hours, op
    assert AbsentPlan(ctx, cal(), 0, 120_000, 60_000, "time", "value").execute().num_rows == 0


def test_multi_field_refusals(ctx):
    Table, leaf = tmf.Table, tmf.leaf
    from greptimedb_b200 import B2PError
    from greptimedb_b200 import plan as P
    tab = Table(6, 80, 2, seed=80)
    one = Table(6, 80, 1, seed=80)
    cases = [
        (lambda: P.TopkPlan(ctx, "topk", 1, leaf(ctx, tab)), mp.REFUSALS["topk"]),
        (lambda: P.TopkPlan(ctx, "bottomk", 1, leaf(ctx, tab)), mp.REFUSALS["topk"]),
        (lambda: P.CountValuesPlan(ctx, "v", leaf(ctx, tab)), mp.REFUSALS["count_values"]),
        (lambda: P.AggregatePlan(ctx, "group", leaf(ctx, tab)), mp.REFUSALS["group"]),
        (lambda: P.ScalarPlan(ctx, leaf(ctx, tab)), mp.REFUSALS["scalar"]),
        (lambda: P.SetOpPlan(ctx, "and", leaf(ctx, tab), leaf(ctx, one)), mp.REFUSALS["and"]),
        (lambda: P.SetOpPlan(ctx, "unless", leaf(ctx, tab), leaf(ctx, tab)), mp.REFUSALS["unless"]),
        (lambda: P.SetOpPlan(ctx, "or", leaf(ctx, tab), leaf(ctx, tab)), mp.REFUSALS["or"]),
        (lambda: P.SetOpPlan(ctx, "or", leaf(ctx, one), leaf(ctx, tab)), "Attempt to combine two tables with different "
                                                                           "column sets"),
        (lambda: P.HistogramQuantilePlan(ctx, 0.5, leaf(ctx, tab)), "multi-field child"),
    ]
    for make, msg in cases:
        with pytest.raises(B2PError, match=msg.replace("(", r"\(").replace(")", r"\)")):
            make().execute()
    P.SetOpPlan(ctx, "and", leaf(ctx, one), leaf(ctx, tab)).execute()  # only the lhs's fields matter to `and`
