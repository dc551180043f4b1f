"""GPU: label_replace and label_join over any node.  Every query of the reference's label.result through the plan layer
(whole rows, column names and order, error texts); each node above a label node bit for bit against the same query
whose leaf was fed labels Python rewrote beforehand; multi-field, Int64 and vector(1) children; colliding rows and NULL
source values; and the refusals."""
import json
import os
import re

import numpy as np
import pyarrow as pa
import pytest

from greptimedb_b200 import B2PError

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_label_vectors.json")))
LOOKBACK = 300_000


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


# ---- the goldens ------------------------------------------------------------------------------------------------------
def table_leaf(ctx, c, table="test", keep=lambda row: True, f64=False):
    """the instant selector over a golden table (its BIGINT val through the Int64 leaf, or as Float64 with `f64`), fed
    the rows `keep` admits"""
    from greptimedb_b200.plan import PromRangeExec
    t = GOLDEN["tables"][table]
    rows = sorted((r for r in t["rows"] if keep(r)), key=lambda r: (r[1:1 + len(t["tags"])], r[0]))
    cols = [pa.array([r[0] for r in rows], pa.timestamp("ms"))]
    cols += [pa.array([r[1 + i] for r in rows], pa.utf8()) for i in range(len(t["tags"]))]
    cols.append(pa.array([r[-1] for r in rows], pa.float64() if f64 else pa.int64()))
    ex = PromRangeExec(ctx, "", c["start_ms"], c["end_ms"], c["step_ms"], 0, "ts", "val", t["tags"], lookback_delta=LOOKBACK)
    ex.push(pa.record_batch(cols, names=t["columns"][:1] + t["tags"] + ["val"]))
    return ex


def host(h):
    return lambda r: r[1] == h


def golden_plan(ctx, c, f64=False):
    """the plan-layer form of a golden query"""
    from greptimedb_b200.plan import BinaryPlan, EmptyMetricPlan, LabelJoinPlan, LabelReplacePlan
    q = c["query"]
    if c["table"] == "test2":  # matchers on a label no row has: every row reads it as ""
        m = re.fullmatch(r'test\{job(=~|=|!=)"(.*)"\}', q)
        op, pat = m.groups()
        hit = re.fullmatch(pat, "") is not None if op == "=~" else (pat == "") == (op == "=")
        return table_leaf(ctx, c, "test2", lambda r: hit)
    vec1 = lambda: EmptyMetricPlan(ctx, c["start_ms"], c["end_ms"], c["step_ms"], "literal", 1.0, "time", "greptime_value")
    m = re.fullmatch(r'\{__name__="test",host="host1"\} ([*+]) (label_replace\(vector\(1\), .*\))', q)
    if m:
        args = re.findall(r'"([^"]*)"', m.group(2))
        return BinaryPlan(ctx, m.group(1), table_leaf(ctx, c, keep=host("host1")), LabelReplacePlan(ctx, vec1(), *args))
    m = re.fullmatch(r'(label_replace|label_join)\((test\{host="(host\d)"\}|vector\(1\)), (.*)\)( == ([\d.]+))?', q)
    fn, child_s, h, rest, cmp_, lit = m.groups()
    args = re.findall(r'"([^"]*)"', rest)
    child = vec1() if child_s == "vector(1)" else table_leaf(ctx, c, keep=host(h), f64=f64)
    node = LabelReplacePlan(ctx, child, *args) if fn == "label_replace" else LabelJoinPlan(ctx, child, *args)
    return node.scalar_op("==", float(lit)) if cmp_ else node


def rows_of(out):
    from tests.test_time_fn_oracle import stamp
    cols = []
    for i in range(out.num_columns):
        col, typ = out.column(i), out.schema.field(i).type
        if pa.types.is_timestamp(typ):
            cols.append([stamp(v) for v in col.cast(pa.int64()).to_pylist()])
        elif pa.types.is_floating(typ):
            cols.append([repr(float(v)) for v in col.to_pylist()])
        else:
            cols.append([str(v) for v in col.to_pylist()])
    return [list(r) for r in zip(*cols)]


def unqualified(name):
    return re.sub(r"(^|[ (])[A-Za-z_0-9]*\.(?=[A-Za-z_])", r"\1", name)


def test_every_golden_through_the_plan_layer(ctx):
    from greptimedb_b200.plan import EmptyMetricPlan, LabelJoinPlan, LabelReplacePlan
    ran = 0
    for c in GOLDEN["cases"]:
        q = c["query"]
        if c["start_ms"] is None:  # over a table that does not exist: the planner's checks decide, on no rows
            c = dict(c, start_ms=0, end_ms=0, step_ms=1000)
            child = EmptyMetricPlan(ctx, 1, 0, 1000, "none")  # (no rows)
            args = re.findall(r'"([^"]*)"', q)
            if c.get("error"):
                with pytest.raises(B2PError, match=re.escape(c["error"])):
                    LabelReplacePlan(ctx, child, *args)
            else:
                assert LabelJoinPlan(ctx, child, *args).execute().num_rows == 0
            ran += 1
            continue
        if c.get("error"):
            with pytest.raises(B2PError) as e:
                golden_plan(ctx, c).execute()
            want = c["error"]
            if "No field named addr" in want:  # the binary node's own text: the reference adds the valid fields
                want = "No field named addr"
            assert want in str(e.value), q
            ran += 1
            continue
        f64 = " == " in q
        if f64:  # (issue 6438) the filter keeps the BIGINT column, which the stage refuses over Int64 (DESIGN §8):
            # pinned over the same values as Float64, the val column read back as integers
            with pytest.raises(B2PError, match="filtering comparison over an Int64 value column"):
                golden_plan(ctx, c).execute()
        out = golden_plan(ctx, c, f64=f64).execute()
        if c["table"] == "test2" and c["rows"]:  # a bare selector: the reference prints the scan's column order
            out = out.select(c["columns"])
        got = rows_of(out)
        if f64:
            iv = out.schema.names.index("val")
            got = [r[:iv] + [str(int(float(r[iv])))] + r[iv + 1:] for r in got]
        assert sorted(got) == sorted(c["rows"]), q
        if c["rows"]:
            names = out.schema.names
            want = c["columns"] if q.startswith("label_") else [unqualified(n) for n in c["columns"]]
            assert names == want, q
        ran += 1
    assert ran == len(GOLDEN["cases"])


# ---- composition, bit for bit ---------------------------------------------------------------------------------------
PODS = ["api-7f9c", "api-x1", "db-0", "web-a1", "web-b2", "web-c3"]
START, END, STEP, RANGE = 300_000, 900_000, 60_000, 300_000


def svc_of(pod):
    return re.fullmatch(r"(.*)-[^-]+", pod).group(1)


def samples(seed, n_series):
    rng = np.random.default_rng(seed)
    ts = np.arange(0, END + 1, 15_000, dtype=np.int64)
    return [(ts, np.cumsum(rng.integers(0, 50, ts.size)).astype(np.float64)) for _ in range(n_series)]


def range_leaf(ctx, tags, tag_rows, data, function="prom_rate", start=START, end=END, step=STEP, rng=RANGE):
    """a range (or, with function "", instant) leaf over series whose tag values are tag_rows[i], fed sorted by tags"""
    from greptimedb_b200.plan import PromRangeExec
    order = sorted(range(len(tag_rows)), key=lambda i: tuple((v is not None, v or "") for v in tag_rows[i]))
    ts = np.concatenate([data[i][0] for i in order])
    cols = [pa.array(ts, pa.timestamp("ms"))]
    for j in range(len(tags)):
        cols.append(pa.array([tag_rows[i][j] for i in order for _ in data[i][0]], pa.utf8()))
    cols.append(pa.array(np.concatenate([data[i][1] for i in order])))
    kw = {"lookback_delta": LOOKBACK} if function == "" else {}
    ex = PromRangeExec(ctx, function, start, end, step, rng, "ts", "val", tags, **kw)
    ex.push(pa.record_batch(cols, names=["ts"] + list(tags) + ["val"]))
    return ex


def by_name(out):
    return {n: out.column(i).to_pylist() for i, n in enumerate(out.schema.names)}


def same(a, b):
    """two batches equal column by column (by name, values by bits), row order included"""
    A, B = by_name(a), by_name(b)
    assert sorted(A) == sorted(B)
    for n in A:
        x, y = A[n], B[n]
        if a.schema.field(n).type == pa.float64():
            assert np.array_equal(np.array(x, np.float64).view(np.int64), np.array(y, np.float64).view(np.int64)), n
        else:
            assert x == y, n


def pods_replaced(ctx, data, **kw):
    from greptimedb_b200.plan import LabelReplacePlan
    leaf = range_leaf(ctx, ["pod"], [[p] for p in PODS], data, **kw)
    return LabelReplacePlan(ctx, leaf, "svc", "$1", "pod", "(.*)-[^-]+")


def pods_rewritten(ctx, data, **kw):
    return range_leaf(ctx, ["pod", "svc"], [[p, svc_of(p)] for p in PODS], data, **kw)


@pytest.mark.parametrize("shape", ["sum", "topk", "sort_by_label", "count_values", "eq", "absent", "subquery"])
def test_nodes_above_a_label_node_bit_for_bit(ctx, shape):
    from greptimedb_b200.plan import (AbsentPlan, AggregatePlan, CountValuesPlan, SortPlan, SubqueryPlan, TopkPlan)
    data = samples(7, len(PODS))
    if shape == "subquery":  # max_over_time(label_replace(rate(m[5m]))[4m:1m]) on the inner grid
        inner = dict(start=START - 240_000 + STEP)
        wrap = lambda n: SubqueryPlan(ctx, "prom_max_over_time", n, START, END, STEP, 240_000)
        same(wrap(pods_replaced(ctx, data, **inner)).execute(), wrap(pods_rewritten(ctx, data, **inner)).execute())
        return
    wrap = {
        "sum": lambda n: AggregatePlan(ctx, "sum", n, by=["svc"]),
        "topk": lambda n: TopkPlan(ctx, "topk", 1, n, by=["svc"]),
        "sort_by_label": lambda n: SortPlan(ctx, "sort_by_label", n, ["svc"]),
        "count_values": lambda n: CountValuesPlan(ctx, "v", n.function("prom_round"), by=["svc"]),
        "eq": lambda n: n.scalar_op(">", 1.0),
        "absent": lambda n: AbsentPlan(ctx, n.scalar_op(">", 1.7), START, END, STEP, "ts", "val", [("svc", "api")]),
    }[shape]
    got, want = wrap(pods_replaced(ctx, data)).execute(), wrap(pods_rewritten(ctx, data)).execute()
    same(got, want)
    if shape == "sum":
        assert got.num_rows > 0 and len(set(got.column("svc").to_pylist())) == 3  # six pods, three services
    if shape == "eq":  # the label node's own layout: dst right after the value
        assert got.schema.names[2:] == ["svc", "pod"] and want.schema.names[2:] == ["pod", "svc"]


def test_vector_matching_on_a_rewritten_label(ctx):
    from greptimedb_b200.plan import BinaryPlan, LabelReplacePlan
    svcs = ["api", "db", "web"]
    dx, dy = samples(1, 3), samples(2, 3)
    x = lambda: range_leaf(ctx, ["svc"], [[s] for s in svcs], dx)
    y_rw = lambda: range_leaf(ctx, ["service", "svc"], [[s, s] for s in svcs], dy)
    y_lr = lambda: LabelReplacePlan(ctx, range_leaf(ctx, ["service"], [[s] for s in svcs], dy), "svc", "$1", "service", "(.*)")
    got = BinaryPlan(ctx, "/", x(), y_lr(), on=["svc"]).execute()
    same(got, BinaryPlan(ctx, "/", x(), y_rw(), on=["svc"]).execute())
    assert got.num_rows > 0


# ---- children of every kind, rows, NULLs ------------------------------------------------------------------------------
def test_multi_field_int64_and_vector_children(ctx):
    from greptimedb_b200.plan import EmptyMetricPlan, LabelJoinPlan, LabelReplacePlan, PromRangeExec
    b = pa.record_batch([pa.array([0, 5000, 0], pa.timestamp("ms")), pa.array(["a-1", "a-1", "b-2"]),
                         pa.array([1.0, 2.0, 3.0]), pa.array([4.0, 5.0, 6.0]), pa.array([7.0, 8.0, 9.0])],
                        names=["ts", "host", "f1", "f2", "f3"])
    ex = PromRangeExec(ctx, "", 0, 5000, 5000, 0, "ts", ["f1", "f2", "f3"], ["host"], lookback_delta=LOOKBACK)
    ex.push(b)
    out = LabelReplacePlan(ctx, ex, "h", "$1", "host", "(.)-.*").execute()
    assert out.schema.names == ["ts", "f1", "f2", "f3", "h", "host"]
    assert out.column("h").to_pylist() == ["a", "a", "b", "b"] and out.column("f3").to_pylist() == [7.0, 8.0, 9.0, 9.0]
    bi = pa.record_batch([pa.array([0], pa.timestamp("ms")), pa.array(["x"]), pa.array([2**62 + 1], pa.int64())],
                         names=["ts", "host", "val"])
    ei = PromRangeExec(ctx, "", 0, 0, 5000, 0, "ts", "val", ["host"], lookback_delta=LOOKBACK)
    ei.push(bi)
    oi = LabelJoinPlan(ctx, ei, "j", ",", "host", "host").execute()
    assert oi.schema.field("val").type == pa.int64() and oi.column("val").to_pylist() == [2**62 + 1]
    assert oi.column("j").to_pylist() == ["x,x"]
    ov = LabelReplacePlan(ctx, EmptyMetricPlan(ctx, 0, 10_000, 5000, "literal", 1.0), "host", "h", "", "").execute()
    assert ov.schema.names == ["time", "value", "host"] and ov.column("host").to_pylist() == ["h"] * 3


def test_colliding_rows_stay_and_nulls_propagate(ctx):
    from greptimedb_b200.plan import LabelJoinPlan, LabelReplacePlan, PromRangeExec
    b = pa.record_batch([pa.array([0, 0, 0], pa.timestamp("ms")), pa.array([None, "a-1", "a-2"], pa.utf8()),
                         pa.array(["z", None, "z"], pa.utf8()), pa.array([1.0, 2.0, 3.0])], names=["ts", "pod", "zone", "val"])
    leaf = lambda: PromRangeExec(ctx, "", 0, 0, 5000, 0, "ts", "val", ["pod", "zone"], lookback_delta=LOOKBACK)
    e = leaf()
    e.push(b)
    out = LabelReplacePlan(ctx, e, "svc", "$1", "pod", "(.*)-.").execute()
    assert out.num_rows == 3 and out.schema.names == ["ts", "val", "svc", "pod", "zone"]
    assert out.column("svc").to_pylist() == [None, "a", "a"]  # NULL stays NULL; the two a rows stay two rows
    e = leaf()
    e.push(b)
    j = LabelJoinPlan(ctx, e, "j", "-", "missing", "pod", "", "zone").execute()
    assert j.column("j").to_pylist() == ["z", "a-1", "a-2-z"]  # NULLs and absent sources skipped
    e = leaf()
    e.push(b)
    assert LabelJoinPlan(ctx, e, "zone", "+", "pod").execute().schema.names == ["ts", "val", "zone", "pod"]


def test_refusals(ctx):
    from greptimedb_b200.plan import CountValuesPlan, LabelJoinPlan, LabelReplacePlan, PromRangeExec
    ids = PromRangeExec(ctx, "", 0, 0, 5000, 0, "ts", "val", ["__tsid"], lookback_delta=LOOKBACK)
    ids.push(pa.record_batch([pa.array([0], pa.timestamp("ms")), pa.array([1.0]), pa.array([7], pa.uint64())],
                             names=["ts", "val", "__tsid"]))
    with pytest.raises(B2PError, match="id-keyed"):
        LabelReplacePlan(ctx, ids, "d", "x", "__tsid", "(.*)").execute()
    data = samples(3, len(PODS))
    with pytest.raises(B2PError, match="time index or a value column"):
        LabelJoinPlan(ctx, pods_rewritten(ctx, data), "d", "-", "pod", "ts").execute()
    value = pods_rewritten(ctx, data).execute().schema.names[1]
    with pytest.raises(B2PError, match="time index or a value column"):
        LabelJoinPlan(ctx, pods_rewritten(ctx, data), "d", "-", value).execute()
    with pytest.raises(B2PError, match="time index or a value column"):
        LabelReplacePlan(ctx, pods_rewritten(ctx, data), value if value.isidentifier() else "ts", "x", "nope", "").execute()
    with pytest.raises(B2PError, match="count_values child"):
        LabelReplacePlan(ctx, CountValuesPlan(ctx, "v", pods_rewritten(ctx, data)), "d", "$1", "v", "(.*)").execute()
    with pytest.raises(B2PError, match="count_values child"):
        LabelJoinPlan(ctx, CountValuesPlan(ctx, "v", pods_rewritten(ctx, data)), "v", "-", "svc").execute()
    for rx in (r"\d+", "(?i)api"):
        with pytest.raises(B2PError, match="not supported by this node"):
            LabelReplacePlan(ctx, pods_rewritten(ctx, data), "d", "$1", "pod", rx)
    with pytest.raises(B2PError, match="Invalid regular expression in label_replace\\(\\): a\\{2,1\\}"):
        LabelReplacePlan(ctx, pods_rewritten(ctx, data), "d", "$1", "pod", "a{2,1}")
    with pytest.raises(B2PError, match="same labelset"):  # the literal branch checks it too (planner.rs:2339-2343)
        LabelReplacePlan(ctx, pods_rewritten(ctx, data), "svc", "x", "nope", "").execute()
