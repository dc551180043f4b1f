"""GPU: time(), the calendar functions, timestamp() and unary minus.  K19 bit for bit against tests/time_fn_oracle.py
for every part over T in {1, 31, 32, 33, 1000, 65 537} x rows in {0, 1, 5, 10 000}; K4's timestamp mode against the
oracle (a selected stale-NaN sample kept, offset, lookback edges, Int64 and multi-field tables); host and device forms
and NULL arguments; every golden of time_fn / timestamp_fn / binary_time_fn through the plan layer, the weekend query
end to end; a calendar stage and unary minus over every kind of node; and the Int32 refusals."""
import json
import math
import os

import numpy as np
import pyarrow as pa
import pytest

from tests import time_fn_oracle as to

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_time_fn_vectors.json")))
LOOKBACK = 300_000


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def words(ok):
    """bool [S,T] -> validity words [S,Tw] (bits past T zero)"""
    S, T = ok.shape
    Tw = (T + 31) // 32
    pad = np.zeros((S, Tw * 32), bool)
    pad[:, :T] = ok
    return np.packbits(pad, axis=1, bitorder="little").view(np.uint32).reshape(S, Tw)


def eval_steps(rng, T):
    """eval timestamps over the calendar's whole range, midnights and their neighbours, negative epochs included"""
    lo, hi = to.days_from_civil(-3000, 1, 1) * to.MS_PER_DAY, to.days_from_civil(12000, 1, 1) * to.MS_PER_DAY
    ts = rng.integers(lo, hi, T, dtype=np.int64)
    ts[::3] = (ts[::3] // to.MS_PER_DAY) * to.MS_PER_DAY + rng.integers(-1, 2, ts[::3].size)
    ts[:min(T, 4)] = [0, -1, 951_782_400_000, 4_107_542_400_000][:min(T, 4)]  # epoch, -1 ms, 2000-02-29, 2100-03-01
    return ts


def bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.int64)


# ---- K19 ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [1, 31, 32, 33, 1000, 65_537])
@pytest.mark.parametrize("rows", [0, 1, 5, 10_000])
def test_step_fn_every_part_bit_for_bit(ctx, T, rows):
    import torch
    rng = np.random.default_rng(T * 7 + rows)
    ets = eval_steps(rng, T)
    Tw = (T + 31) // 32
    dev = torch.device("cuda:0")
    d_ts = torch.from_numpy(ets).to(dev)
    d_valid = torch.randint(-2**31, 2**31 - 1, (max(rows, 1) * Tw,), dtype=torch.int32, device=dev)
    out = torch.full((max(rows, 1) * T,), 7.0, dtype=torch.float64, device=dev)
    k = torch.arange(T, device=dev)
    for part in to.PARTS:
        want = torch.from_numpy(to.step_value(part, ets)).to(dev)
        ctx.step_fn_dev(part, d_ts, d_valid, rows, T, out)
        ctx.sync()
        if rows == 0:
            assert (out == 7.0).all()
            continue
        for r0 in range(0, rows, 500):  # (row blocks keep the comparison's memory small)
            r1 = min(rows, r0 + 500)
            w = d_valid.view(-1, Tw)[r0:r1].to(torch.int64) & 0xFFFFFFFF
            ok = ((w[:, k >> 5] >> (k & 31)) & 1).bool()
            exp = torch.where(ok, want[None, :], torch.zeros((), dtype=torch.float64, device=dev))
            got = out.view(-1, T)[r0:r1]
            assert torch.equal(got.view(torch.int64), exp.view(torch.int64)), (part, T, rows, r0)


def test_step_fn_host_form_and_validity_untouched(ctx):
    rng = np.random.default_rng(19)
    ets = eval_steps(rng, 77)
    ok = rng.random((6, 77)) < 0.5
    valid = words(ok)
    before = valid.copy()
    for part in to.PARTS:
        out = ctx.step_fn(part, ets, valid)
        assert (bits(out) == bits(to.step_fn(part, ets, ok))).all(), part
    assert (valid == before).all()


def test_step_fn_refusals_without_fault(ctx):
    from greptimedb_b200 import B2PError
    valid = np.full((2, 1), 0xFFFFFFFF, np.uint32)
    far = to.days_from_civil(to.MAX_YEAR + 1, 1, 1) * to.MS_PER_DAY
    for part in to.PARTS[1:]:
        with pytest.raises(B2PError) as ei:
            ctx.step_fn(part, np.array([0, far], np.int64), valid)
        assert ei.value.code == -1 and "year" in str(ei.value)
    out = ctx.step_fn("time", np.array([0, far, np.iinfo(np.int64).min], np.int64), valid)  # time() has no bound
    assert out[0, 1] == float(far) / 1000.0 and out[0, 2] == float(np.iinfo(np.int64).min) / 1000.0
    edge = to.days_from_civil(to.MAX_YEAR + 1, 1, 1) * to.MS_PER_DAY - 1
    assert ctx.step_fn("year", np.array([edge], np.int64), valid[:, :1])[0, 0] == float(to.MAX_YEAR)
    for bad in (-1, 9, 100):
        with pytest.raises(B2PError):
            ctx.step_fn(bad, np.zeros(3, np.int64), valid)
    L = ctx._L
    assert L.b2p_step_fn_dev(ctx._h, 2, None, None, 3, 5, None) == -1
    assert L.b2p_step_fn_dev(ctx._h, 2, None, None, 0, 5, None) == 0  # nothing to do
    assert L.b2p_step_fn(None, 2, None, None, 0, 5, None) == -1
    out = ctx.step_fn("hour", np.array([3_600_000], np.int64), valid)  # the context works after the refusals
    assert out[0, 0] == 1.0


# ---- K4 timestamp mode ------------------------------------------------------------------------------------------------
def test_instant_timestamp_against_oracle(ctx):
    rng = np.random.default_rng(4)
    S = 40
    lens = rng.integers(0, 60, S)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    ts = np.concatenate([np.sort(rng.choice(np.arange(-50_000, 400_000, 500), n, replace=False)) for n in lens]).astype(np.int64)
    ts[offsets[1]:offsets[2]] = ts[offsets[1]] if lens[1] else ts[offsets[1]:offsets[2]]  # equal timestamps
    for start, end, step, lb, off in ((0, 300_000, 10_000, 30_000, 0), (-20_000, 350_000, 7_000, 1, 2_500),
                                      (0, 200_000, 1_000, 0, -500), (5_000, 5_000, 1, LOOKBACK, 0)):
        out, valid = ctx.instant_timestamp(ts, start, end, step, lb, off, offsets=offsets)
        want, ok = to.instant_timestamp(ts, offsets.astype(np.int64), start, end, step, lb, off)
        assert (valid == words(ok)).all(), (start, step, lb, off)
        assert (bits(out) == bits(want)).all(), (start, step, lb, off)


def test_instant_timestamp_keeps_a_stale_nan_sample_and_lookback_edges(ctx):
    ts = np.array([0, 10_000, 20_000], np.int64)
    val = np.array([1.0, float("nan"), 3.0])
    sid = np.zeros(3, np.uint32)
    plain, pv = ctx.instant_select(ts, val, 10_000, 10_000, 1, LOOKBACK, sid=sid)
    assert pv[0, 0] == 0  # the plain selector drops the stale NaN
    out, valid = ctx.instant_timestamp(ts, 10_000, 10_000, 1, LOOKBACK, sid=sid)
    assert valid[0, 0] == 1 and out[0, 0] == 10.0
    # lookback edges: t - lookback < ts <= t
    out, valid = ctx.instant_timestamp(ts, 29_999, 30_001, 1, 10_000, sid=sid)
    assert (valid[0, 0] & 7) == 0b001 and out[0, 0] == 20.0
    # device form
    import torch
    dev = torch.device("cuda:0")
    d_out = torch.empty(3, dtype=torch.float64, device=dev)
    d_valid = torch.empty(1, dtype=torch.int32, device=dev)
    offs = torch.tensor([0, 3], dtype=torch.int64, device=dev)
    ctx.instant_timestamp_dev(0, 20_000, 10_000, LOOKBACK, 0, torch.from_numpy(ts).to(dev), offs, 3, 1, d_out, d_valid)
    ctx.sync()
    assert d_out.cpu().tolist() == [0.0, 10.0, 20.0] and int(d_valid.item()) & 7 == 7
    L = ctx._L
    assert L.b2p_instant_timestamp_dev(ctx._h, 0, 10, 1, 5, 0, None, None, 3, 1, None, None) == -1
    assert L.b2p_instant_timestamp(ctx._h, 0, 10, 1, 5, 0, None, None, None, 3, 1, None, None) == -1


# ---- plan layer -------------------------------------------------------------------------------------------------------
def metric_batch(table):
    t = GOLDEN["tables"][table]
    return pa.record_batch([pa.array([r[0] for r in t["rows"]], pa.timestamp("ms")),
                            pa.array([r[1] for r in t["rows"]], pa.float64())], names=["ts", "val"])


def leaf(ctx, table, c, timestamp=False):
    from greptimedb_b200.plan import PromRangeExec
    ex = PromRangeExec(ctx, "", c["start_ms"], c["end_ms"], c["step_ms"], 0, "ts", "val", [], lookback_delta=LOOKBACK)
    ex.push(metric_batch(table))
    return ex.timestamp(LOOKBACK) if timestamp else ex


def empty(ctx, c, kind):
    from greptimedb_b200.plan import EmptyMetricPlan
    return EmptyMetricPlan(ctx, c["start_ms"], c["end_ms"], c["step_ms"], kind)


def plan_of(ctx, c):
    """the plan-layer form of a golden query (None: a query this layer does not express)"""
    from greptimedb_b200.plan import BinaryPlan
    q = c["query"]
    tstamp = lambda t: leaf(ctx, t, c, timestamp=True)
    simple = {
        "time()": lambda: empty(ctx, c, "time"),
        "time() + 1": lambda: empty(ctx, c, "time").scalar_op("+", 1.0),
        "1 + time()": lambda: empty(ctx, c, "time").scalar_op("+", 1.0, scalar_on_left=True),
        "time() < bool 1": lambda: empty(ctx, c, "time").scalar_op("<", 1.0, return_bool=True),
        "time() > bool 1": lambda: empty(ctx, c, "time").scalar_op(">", 1.0, return_bool=True),
        "timestamp(timestamp_test)": lambda: tstamp("timestamp_test"),
        "-timestamp(timestamp_test)": lambda: tstamp("timestamp_test").function("negative"),
        "timestamp(timestamp_test) + 1": lambda: tstamp("timestamp_test").scalar_op("+", 1.0),
        "timestamp(timestamp_test) > bool 30": lambda: tstamp("timestamp_test").scalar_op(">", 30.0, return_bool=True),
        "timestamp(timestamp_test) == 60": lambda: tstamp("timestamp_test").scalar_op("==", 60.0),
    }
    if q in simple:
        return simple[q]()
    if q.endswith("()") and q[:-2] in to.PARTS:
        return empty(ctx, c, "none").function(q[:-2])
    if q == "hour(metrics)":
        return leaf(ctx, "metrics", c).function("hour")
    parts = q.split(" ")  # `lhs op [bool] rhs` of two nodes
    if len(parts) in (3, 4) and (q.startswith("time()") or q.startswith("metrics") or q.startswith("timestamp(")):
        lhs_s, rhs_s = parts[0], parts[-1]
        op = parts[1]
        rb = len(parts) == 4
        if not all(s in ("time()", "metrics", "timestamp(timestamp_test)", "timestamp(timestamp_test2)") for s in (lhs_s, rhs_s)):
            return None
        node = lambda s: (empty(ctx, c, "time") if s == "time()" else leaf(ctx, "metrics", c) if s == "metrics"
                          else tstamp(s[len("timestamp("):-1]))
        return BinaryPlan(ctx, op, node(lhs_s), node(rhs_s), return_bool=rb)
    return None


def rows_of(out):
    cols = []
    for i in range(out.num_columns):
        col, typ = out.column(i), out.schema.field(i).type
        if pa.types.is_timestamp(typ):
            from tests.test_time_fn_oracle import stamp
            cols.append([stamp(v) for v in col.cast(pa.int64()).to_pylist()])
        elif pa.types.is_floating(typ):
            cols.append([repr(float(v)) for v in col.to_pylist()])
        else:
            cols.append([str(v) for v in col.to_pylist()])
    return [list(r) for r in zip(*cols)]


def unqualified(name):
    """a column name without DataFusion's table qualifiers (`metrics.val`, `.time`, `lhs.time` -> `val`, `time`): the
    plan API carries no table reference, so the binary node prints bare column names"""
    import re
    return re.sub(r"(^|[ (])[A-Za-z_0-9]*\.(?=[A-Za-z_])", r"\1", name)


def test_every_golden_through_the_plan_layer(ctx):
    ran = 0
    for c in GOLDEN["cases"]:
        if c["file"] == "binary_time_fn.result" or c["start_ms"] is None:
            continue
        plan = plan_of(ctx, c)
        if plan is None:
            assert c["query"].startswith("abs(")  # avg() of two timestamp() leaves over different tables: no rows
            continue
        out = plan.execute()
        assert sorted(rows_of(out)) == sorted(c["rows"]), c["query"]
        if c["rows"]:
            assert out.schema.names == [unqualified(n) for n in c["columns"]], c["query"]
        calendar = (c["query"].endswith("()") and c["query"][:-2] in to.PARTS[1:]) or c["query"] == "hour(metrics)"
        if c["rows"] and (calendar or c["query"] == "time()"):
            assert out.schema.names == c["columns"], c["query"]  # (single nodes: the names exactly)
            assert out.schema.field(1).type == (pa.int32() if calendar else pa.float64())
        ran += 1
    assert ran == len(GOLDEN["cases"]) - 4  # all but the weekend query, the two without a grid and abs(..)


def test_time_compared_with_a_tagged_vector_keeps_the_vector(ctx):
    """`time() > m` filters m (planner.rs:765-771 keeps the vector side): m's rows, labels, values and time index"""
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import BinaryPlan, EmptyMetricPlan
    inst = _leaves(ctx)["instant"]
    t = lambda: EmptyMetricPlan(ctx, 0, 120_000, 60_000, "time")
    for op, keep in ((">", {("a", 60_000, -2.0), ("a", 120_000, 0.0), ("b", 60_000, 5.0), ("b", 120_000, 6.0)}),
                     ("<", {("a", 0, 1.0), ("b", 0, 4.0)}), ("<=", {("a", 0, 1.0), ("b", 0, 4.0)}),
                     ("!=", {("a", 0, 1.0), ("a", 60_000, -2.0), ("a", 120_000, 0.0), ("b", 0, 4.0),
                             ("b", 60_000, 5.0), ("b", 120_000, 6.0)})):
        out = BinaryPlan(ctx, op, t(), inst()).execute()
        assert out.schema.names == ["ts", "val", "host", "le"], op
        got = set(zip(out.column("host").to_pylist(), out.column("ts").cast(pa.int64()).to_pylist(),
                      out.column("val").to_pylist()))
        assert got == keep, op
        # the mirrored form `m <op'> time()` keeps the same cells
        mirror = {">": "<", "<": ">", "<=": ">=", "!=": "!="}[op]
        m = BinaryPlan(ctx, mirror, inst(), t()).execute()
        assert set(zip(m.column("host").to_pylist(), m.column("ts").cast(pa.int64()).to_pylist(),
                       m.column("val").to_pylist())) == keep, op
    with pytest.raises(B2PError) as ei:  # vector(s) on the lhs: its matching is not modelled, so it is refused
        BinaryPlan(ctx, ">", EmptyMetricPlan(ctx, 0, 120_000, 60_000, "literal", literal=3.0), inst()).execute()
    assert "literal EmptyMetric" in str(ei.value)


def test_weekend_query_end_to_end(ctx):
    """max_over_time(test_metric[30s]) > 100 and on () (day_of_week() == 0 or day_of_week() == 6)"""
    from greptimedb_b200.plan import EmptyMetricPlan, PromRangeExec, SetOpPlan
    c = next(c for c in GOLDEN["cases"] if c["file"] == "binary_time_fn.result")
    t = GOLDEN["tables"]["test_metric"]
    rows = sorted(t["rows"], key=lambda r: (r[0], r[1], r[2], r[3]))
    b = pa.record_batch([pa.array([r[0] for r in rows]), pa.array([r[1] for r in rows]), pa.array([r[2] for r in rows]),
                         pa.array([r[3] for r in rows], pa.timestamp("ms")), pa.array([r[4] for r in rows], pa.float64())],
                        names=["asset", "attribute", "measurement", "timestamp", "value"])
    s, e, i = c["start_ms"], c["end_ms"], c["step_ms"]
    lhs = PromRangeExec(ctx, "prom_max_over_time", s, e, i, 30_000, "timestamp", "value",
                        ["asset", "attribute", "measurement"]).scalar_op(">", 100.0)
    lhs.push(b)
    sat = EmptyMetricPlan(ctx, s, e, i, "none").function("day_of_week").scalar_op("==", 0.0)
    sun = EmptyMetricPlan(ctx, s, e, i, "none").function("day_of_week").scalar_op("==", 6.0)
    weekend = SetOpPlan(ctx, "or", sat, sun)
    out = SetOpPlan(ctx, "and", lhs, weekend, on=[]).execute()
    assert out.schema.names == c["columns"]
    assert sorted(rows_of(out)) == sorted(c["rows"])
    w = weekend.execute()
    assert w.schema.field(1).type == pa.int32()  # `or` of two Int32 sides stays Int32


def _leaves(ctx):
    """one node of every kind over the same 3-step grid (0, 60 s, 120 s)"""
    from greptimedb_b200.plan import (AbsentPlan, AggregatePlan, BinaryPlan, CountValuesPlan, EmptyMetricPlan,
                                      HistogramQuantilePlan, PromRangeExec, ScalarPlan, SetOpPlan, SortPlan,
                                      SubqueryPlan, TopkPlan)
    b = pa.record_batch([pa.array([0, 60_000, 120_000, 0, 60_000, 120_000], pa.timestamp("ms")),
                         pa.array(["a", "a", "a", "b", "b", "b"]), pa.array(["1", "1", "1", "+Inf", "+Inf", "+Inf"]),
                         pa.array([1.0, -2.0, 0.0, 4.0, 5.0, 6.0])], names=["ts", "host", "le", "val"])

    def inst():
        ex = PromRangeExec(ctx, "", 0, 120_000, 60_000, 0, "ts", "val", ["host", "le"], lookback_delta=LOOKBACK)
        ex.push(b)
        return ex

    def rng():
        ex = PromRangeExec(ctx, "prom_rate", 0, 120_000, 60_000, 120_000, "ts", "val", ["host", "le"])
        ex.push(b)
        return ex

    def ts():
        ex = PromRangeExec(ctx, "", 0, 120_000, 60_000, 0, "ts", "val", ["host", "le"], lookback_delta=LOOKBACK)
        ex.push(b)
        return ex.timestamp(LOOKBACK)

    sub = PromRangeExec(ctx, "", -60_000, 120_000, 60_000, 0, "ts", "val", ["host", "le"], lookback_delta=LOOKBACK)
    sub.push(b)
    return {
        "instant": inst, "range": rng, "timestamp": ts,
        "empty": lambda: EmptyMetricPlan(ctx, 0, 120_000, 60_000, "time"),
        "binary": lambda: BinaryPlan(ctx, "+", inst(), inst()),
        "setop": lambda: SetOpPlan(ctx, "and", inst(), inst()),
        "scalar": lambda: ScalarPlan(ctx, AggregatePlan(ctx, "sum", inst())),
        "topk": lambda: TopkPlan(ctx, "topk", 1, inst()),
        "aggregate": lambda: AggregatePlan(ctx, "sum", inst(), by=["le"]),
        "count_values": lambda: CountValuesPlan(ctx, "v", inst()),
        "subquery": lambda: SubqueryPlan(ctx, "prom_max_over_time", sub, 0, 120_000, 60_000, 120_000),
        "histogram": lambda: HistogramQuantilePlan(ctx, 0.5, inst()),
        "sort": lambda: SortPlan(ctx, "sort", inst()),
        "absent": lambda: AbsentPlan(ctx, inst(), 0, 120_000, 60_000, "ts", "value"),
    }


@pytest.mark.parametrize("kind", ["instant", "range", "timestamp", "empty", "binary", "setop", "scalar", "topk",
                                  "aggregate", "count_values", "subquery", "histogram", "sort", "absent"])
def test_calendar_stage_and_unary_minus_over_every_node(ctx, kind):
    make = _leaves(ctx)[kind]
    base = make().execute()
    hour = make().function("hour").execute()
    minus = make().function("negative").execute()
    ti = [n for n in base.schema.names if pa.types.is_timestamp(base.schema.field(n).type)]
    if base.num_rows == 0:
        assert hour.num_rows == 0 and minus.num_rows == 0
        return
    t = hour.column(ti[0]).cast(pa.int64()).to_numpy()
    hcol = [n for n in hour.schema.names if n.startswith('date_part(Utf8("hour"),')]
    assert len(hcol) == 1 and hour.schema.field(hcol[0]).type == pa.int32(), hour.schema
    assert hour.num_rows == base.num_rows
    assert hour.column(hcol[0]).to_pylist() == [int(v) for v in to.step_value("hour", t)]
    vals = [n for n in base.schema.names if pa.types.is_floating(base.schema.field(n).type)]
    if kind == "count_values":  # the count (Int64 without a stage) is the value; the counted value is a label
        vals = [base.schema.names[0]]
    mvals = [n for n in minus.schema.names if n.startswith("(- ")]
    assert len(mvals) == len(vals) >= 1
    for a, m in zip(vals, mvals):
        x = base.column(a).to_numpy().astype(np.float64)
        assert (bits(minus.column(m).to_numpy()) == (bits(x) ^ np.int64(-2**63))).all()


def test_empty_metric_unit_vectors_and_create_errors(ctx):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import EmptyMetricPlan
    from tests.test_time_fn_oracle import stamp
    for v in GOLDEN["empty_metric"]:
        out = EmptyMetricPlan(ctx, v["start"], v["end"], v["interval"], "none" if v["field_expr"] is None else "time").execute()
        got = rows_of(out)
        assert [r[0] for r in got] == [r[0] for r in v["rows"]], v["name"]
        if v["field_expr"] is not None:
            assert [r[1] for r in got] == [r[1] for r in v["rows"]], v["name"]
        else:
            assert out.schema.names == ["time"]
    lit = EmptyMetricPlan(ctx, 0, 2000, 1000, "literal", literal=math.pi).execute()
    assert lit.schema.names == ["time", "value"] and lit.column(1).to_pylist() == [math.pi] * 3
    for bad in ((0, 10, 0), (0, 10, -5)):
        with pytest.raises(B2PError):
            EmptyMetricPlan(ctx, *bad)
    L = ctx._L
    assert not L.b2p_plan_empty_metric_create(ctx._h, 0, 10, 1, None, b"value", 1, 0.0)
    assert not L.b2p_plan_empty_metric_create(ctx._h, 0, 10, 1, b"time", b"value", 7, 0.0)
    assert stamp(0) == "1970-01-01T00:00:00"


def test_timestamp_leaf_over_int64_and_multi_field_tables(ctx):
    from greptimedb_b200.plan import PromRangeExec
    ts = [0, 10_000, 20_000, 0, 15_000]
    host = ["a", "a", "a", "b", "b"]
    nan_bits = int(np.array([np.nan]).view(np.int64)[0])
    for cols, names in (([pa.array([1, nan_bits, 3], pa.int64())], ["val"]),
                        ([pa.array([1.0, float("nan"), 3.0, 4.0, 5.0]), pa.array([7.0] * 5)], ["f1", "f2"])):
        n = len(cols[0])
        b = pa.record_batch([pa.array(ts[:n], pa.timestamp("ms")), pa.array(host[:n])] + cols,
                            names=["ts", "host"] + names)
        ex = PromRangeExec(ctx, "", 0, 20_000, 5_000, 0, "ts", names if len(names) > 1 else names[0], ["host"],
                           lookback_delta=LOOKBACK)
        ex.push(b)
        out = ex.timestamp(LOOKBACK).execute()
        assert out.schema.names == ["ts", "value", "host"] and out.schema.field(1).type == pa.float64()
        offs = [0, 3, n] if n == 5 else [0, 3]
        want, ok = to.instant_timestamp(np.array(ts[:n], np.int64), offs, 0, 20_000, 5_000, LOOKBACK)
        assert out.column(1).to_pylist() == want[ok].tolist()
