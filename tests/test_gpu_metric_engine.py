"""GPU: PromQL over metric-engine tables.  A leaf divides series on the UInt64 `__tsid` column with the Utf8 label
columns beside it (b2p_plan_set_label_columns); every node above reads the labels, and `__tsid` is exported where the
reference keeps it.  The reference's metric-engine goldens, a differential against the same rows keyed on the Utf8
labels over every node family, the `__tsid` schema of each node, and the leaf's refusals."""
import math

import numpy as np
import pyarrow as pa
import pytest

from tests.metric_engine_helpers import (build, expected_of, leaf, load_metric_engine, rows_of, table_batches,
                                         tsid_of)

pytestmark = pytest.mark.gpu
G = load_metric_engine()


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def case_labels(case):
    names = []
    for lab, _, _ in case["expected"]:
        names += [n for n in lab if n not in names]
    return names


def time_index_of(expr, tables):
    while expr[0] not in ("sel", "range"):
        expr = next(e for e in expr[1:] if isinstance(e, list))
    return tables[expr[1] if expr[0] == "sel" else expr[2]]["time_index"]


@pytest.mark.parametrize("case", G["cases"], ids=[c["name"] for c in G["cases"]])
def test_goldens_through_metric_engine_leaves(ctx, case):
    labels = case_labels(case)
    out = build(ctx, case["expr"], G["tables"], case, metric_engine=True).execute()
    ti = time_index_of(case["expr"], G["tables"])
    assert rows_of(out, ti, labels) == expected_of(case, labels)
    if "keeps_tsid" in case:   # whether the reference's printed plan keeps __tsid at this node
        assert ("__tsid" in out.schema.names) == case["keeps_tsid"], out.schema.names
    # the same plan over the Utf8-keyed leaves prints the same rows
    assert rows_of(build(ctx, case["expr"], G["tables"], case, metric_engine=False).execute(), ti, labels) == \
        expected_of(case, labels)


# ---- differential: seeded random metric-engine tables against the same rows keyed on the Utf8 labels ----------------
STEP, START, END = 10_000, 100_000, 400_000
LOOKBACK = 60_000


def random_table(seed, n_series=40, le=False):
    """Labels job / instance / region (NULL in some series) [+ le], integer-valued samples (sums are exact in any
    order), some missing, some NaN"""
    rng = np.random.default_rng(seed)
    series, seen = [], set()
    les = ["0.5", "1", "2", "+Inf"] if le else [None]
    for i in range(n_series):
        base = {"job": f"job{rng.integers(0, 3)}", "instance": f"i{i % 7}",
                "region": None if rng.random() < 0.3 else f"r{rng.integers(0, 2)}"}
        key = tuple(base.values())
        if key in seen:
            continue
        seen.add(key)
        cum = 0.0
        for b in les:
            ts = sorted(set(int(t) for t in rng.integers(0, END // 1000, size=rng.integers(0, 30)) * 1000))
            vals = [float(v) for v in rng.integers(-20, 40, size=len(ts))]
            if le:   # cumulative buckets
                cum += 1.0
                vals = [abs(v) * cum for v in vals]
            vals = [math.nan if rng.random() < 0.05 else v for v in vals]
            s = dict(base, ts=ts, val=vals)
            if le:
                s["le"] = b
            series.append(s)
    return {"time_index": "ts", "field": "val", "tags": ["job", "instance", "region"] + (["le"] if le else []),
            "series": series}


def value_bits_rows(batch):
    """-> the batch's rows without its __tsid column as a sorted list, every Float64 cell by its bits"""
    cols = []
    for n in batch.schema.names:
        if n == "__tsid":
            continue
        c = batch.column(n)
        if pa.types.is_timestamp(c.type):
            c = c.cast(pa.int64())
        vals = c.to_pylist()
        if pa.types.is_floating(c.type):
            vals = [int(np.array([v], np.float64).view(np.uint64)[0]) for v in vals]
        cols.append(vals)
    return sorted(zip(*cols), key=repr)


def sel(ctx, tab, me, **kw):
    return leaf(ctx, tab, me, START, END, STEP, lookback=LOOKBACK, splits=3, **kw)


def rng_(ctx, tab, me, fn="prom_max_over_time", **kw):
    return leaf(ctx, tab, me, START, END, STEP, fn=fn, range_ms=30_000, splits=3, **kw)


def shapes():
    from greptimedb_b200.plan import (AbsentPlan, AggregatePlan, BinaryPlan, CountValuesPlan, HistogramQuantilePlan,
                                      LabelJoinPlan, LabelReplacePlan, ScalarPlan, SetOpPlan, SortPlan, SubqueryPlan,
                                      TopkPlan)
    A, B, H = random_table(1), random_table(2), random_table(3, n_series=12, le=True)
    return {
        "range_leaf": lambda c, me: rng_(c, A, me),
        "instant_leaf": lambda c, me: sel(c, A, me),
        "fused_sum_by": lambda c, me: rng_(c, A, me, fn="prom_sum_over_time", aggregate="sum", by_columns=["job"]),
        "fused_max_instant": lambda c, me: sel(c, A, me, aggregate="max", by_columns=["region", "job"]),
        "fused_histogram": lambda c, me: leaf(c, H, me, START, END, STEP, fn="prom_max_over_time", range_ms=30_000,
                                              splits=2, histogram_quantile=0.7),
        "fn_stage": lambda c, me: sel(c, A, me).scalar_op("*", 2).function("abs").scalar_op(">", 10),
        "arith_filter_stages": lambda c, me: sel(c, A, me).scalar_op("-", 5).scalar_op(">", 10, return_bool=True)
                                                           .scalar_op("<", 1),
        "calendar": lambda c, me: sel(c, A, me).function("hour"),
        "unary_minus": lambda c, me: sel(c, A, me).function("negative"),
        "binary": lambda c, me: BinaryPlan(c, "-", sel(c, A, me), rng_(c, A, me)),
        "binary_on": lambda c, me: BinaryPlan(c, "/", sel(c, A, me), AggregatePlan(c, "sum", sel(c, B, me), by=["job"]),
                                              on=["job"], label_side="lhs"),
        "binary_ignoring_bool": lambda c, me: BinaryPlan(c, ">=", sel(c, A, me), sel(c, A, me), return_bool=True,
                                                         ignoring=["region"]),
        "binary_filter": lambda c, me: BinaryPlan(c, ">", sel(c, A, me), sel(c, B, me)),
        "and": lambda c, me: SetOpPlan(c, "and", sel(c, A, me), sel(c, B, me)),
        "or": lambda c, me: SetOpPlan(c, "or", sel(c, A, me), sel(c, B, me)),
        "unless_on": lambda c, me: SetOpPlan(c, "unless", sel(c, A, me), sel(c, B, me), on=["job"]),
        "scalar": lambda c, me: ScalarPlan(c, AggregatePlan(c, "sum", sel(c, A, me))),
        "topk_by": lambda c, me: TopkPlan(c, "topk", 2, sel(c, A, me), by=["job"]),
        "bottomk": lambda c, me: TopkPlan(c, "bottomk", 3, sel(c, A, me)),
        "sum_by": lambda c, me: AggregatePlan(c, "sum", sel(c, A, me), by=["job", "region"]),
        "avg_without": lambda c, me: AggregatePlan(c, "avg", sel(c, A, me), without=["instance"]),
        "quantile": lambda c, me: AggregatePlan(c, "quantile", sel(c, A, me), param=0.3, by=["region"]),
        "max_keep": lambda c, me: AggregatePlan(c, "max", sel(c, A, me), without=[]),
        "count_values": lambda c, me: CountValuesPlan(c, "v", sel(c, A, me), by=["job"]),
        "subquery": lambda c, me: SubqueryPlan(c, "prom_max_over_time",
                                               leaf(c, A, me, START - 30_000 + STEP, END, STEP, lookback=LOOKBACK,
                                                    splits=3), START, END, STEP, 30_000),
        "histogram_quantile": lambda c, me: HistogramQuantilePlan(c, 0.5, sel(c, H, me)),
        "sort_desc": lambda c, me: SortPlan(c, "sort_desc", sel(c, A, me)),
        "sort_by_label": lambda c, me: SortPlan(c, "sort_by_label", sel(c, A, me), ["region", "instance"]),
        "absent": lambda c, me: AbsentPlan(c, sel(c, A, me), START, END, STEP, "ts", "val", [("job", "x")]),
        "label_replace": lambda c, me: LabelReplacePlan(c, sel(c, A, me), "dst", "$1-x", "instance", "i(.*)"),
        "label_join": lambda c, me: LabelJoinPlan(c, sel(c, A, me), "dst", ",", "job", "region"),
    }


SHAPES = list(shapes())


@pytest.mark.parametrize("shape", SHAPES)
def test_differential_against_the_utf8_keyed_leaf(ctx, shape):
    make = shapes()[shape]
    got, exp = make(ctx, True).execute(), make(ctx, False).execute()
    names = [n for n in got.schema.names if n != "__tsid"]
    assert names == exp.schema.names
    assert value_bits_rows(got) == value_bits_rows(exp)
    assert got.num_rows == exp.num_rows
    # where the node orders its export, the order is the same in both forms (sort_desc: the values; sort_by_label: the
    # listed labels, rows of equal labels keeping the child's order, which differs; topk / bottomk: every column,
    # ties being ranked by the label tuple)
    order = {"sort_desc": [got.schema.names[1]], "sort_by_label": ["region", "instance"], "topk_by": names,
             "bottomk": names}.get(shape)
    if order:
        seq = lambda b: list(zip(*(b.column(n).to_pylist() for n in order)))
        assert seq(got) == seq(exp)


# ---- schema: where __tsid survives, with which values ----------------------------------------------------------------
# `binary` takes its labels from its rhs, a range leaf, which has dropped __tsid
KEEPS = {"instant_leaf", "arith_filter_stages", "unary_minus", "binary_on", "binary_ignoring_bool", "binary_filter",
         "and", "or", "unless_on", "topk_by", "bottomk", "max_keep"}


def id_by_labels(tab):
    return {tuple(s.get(t) for t in ("job", "instance", "region")): tsid_of(list(zip(tab["tags"], (s.get(t) for t in tab["tags"])))) for s in tab["series"]}


@pytest.mark.parametrize("shape", SHAPES)
def test_tsid_column_where_the_reference_keeps_it(ctx, shape):
    out = shapes()[shape](ctx, True).execute()
    has = "__tsid" in out.schema.names
    assert has == (shape in KEEPS), out.schema.names
    if not has:
        return
    assert out.schema.names[-1] == "__tsid" and out.schema.field("__tsid").type == pa.uint64()


def test_tsid_values(ctx):
    """A kept __tsid is the series' id, or the first member's id of a group over every label"""
    from greptimedb_b200.plan import AggregatePlan, BinaryPlan
    A = random_table(1)
    ids = id_by_labels(A)
    for node in (sel(ctx, A, True), sel(ctx, A, True).scalar_op("+", 1),
                 BinaryPlan(ctx, "+", sel(ctx, A, True), sel(ctx, A, True))):
        out = node.execute()
        for j, i, r, t in zip(*(out.column(n).to_pylist() for n in ("job", "instance", "region", "__tsid"))):
            assert ids[(j, i, r)] == t
    out = AggregatePlan(ctx, "max", sel(ctx, A, True), by=["region", "instance", "job"]).execute()
    for j, i, r, t in zip(*(out.column(n).to_pylist() for n in ("job", "instance", "region", "__tsid"))):
        assert ids[(j, i, r)] == t
    # a fused aggregate over every label keeps it too; over fewer labels it does not
    out = sel(ctx, A, True, aggregate="sum", by_columns=["job", "instance", "region"]).execute()
    assert out.schema.names[-1] == "__tsid"
    assert "__tsid" not in sel(ctx, A, True, aggregate="sum", by_columns=["job"]).execute().schema.names


def test_tsid_join_and_label_join(ctx):
    """Two sides that carry __tsid join on it without on / ignoring; with ignoring(host) they join on the labels and
    the rows differ (tsid_binary_join_regression.sql): host1 and host2 of one job then pair across series"""
    from greptimedb_b200.plan import BinaryPlan
    tab = {"time_index": "ts", "field": "v", "tags": ["host", "job"],
           "series": [{"host": "h1", "job": "j", "ts": [0], "val": [6.0]},
                      {"host": "h2", "job": "j", "ts": [0], "val": [3.0]}]}
    mk = lambda me: leaf(ctx, tab, me, 0, 0, 1000, lookback=LOOKBACK)
    by_id = BinaryPlan(ctx, "/", mk(True), mk(True)).execute()
    by_labels = BinaryPlan(ctx, "/", mk(False), mk(False)).execute()
    assert rows_of(by_id, "ts", ["host", "job"]) == rows_of(by_labels, "ts", ["host", "job"])
    assert sorted(by_id.column("__tsid").to_pylist()) == sorted(tsid_of([("host", h), ("job", "j")]) for h in ("h1", "h2"))
    ign = BinaryPlan(ctx, "/", mk(True), mk(True), ignoring=["host"]).execute()
    assert ign.num_rows == 4 and sorted(ign.column(ign.num_columns - 2).to_pylist()) == [0.5, 1.0, 1.0, 2.0]


def test_tsid_join_is_taken(ctx):
    """Where the two joins differ: the rhs carries a label the lhs lacks.  The label join then has a key column the lhs
    has no field for (a Plan error), while two sides that carry __tsid join on it, series by series, with the rhs's
    labels"""
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import BinaryPlan
    lhs = {"time_index": "ts", "field": "v", "tags": ["host"],
           "series": [{"host": "h1", "__tsid": 11, "ts": [0], "val": [6.0]},
                      {"host": "h2", "__tsid": 12, "ts": [0], "val": [3.0]}]}
    rhs = {"time_index": "ts", "field": "v", "tags": ["host", "dc"],
           "series": [{"host": "h1", "dc": "a", "__tsid": 11, "ts": [0], "val": [2.0]},
                      {"host": "h2", "dc": "b", "__tsid": 12, "ts": [0], "val": [1.0]}]}
    mk = lambda t, me: leaf(ctx, t, me, 0, 0, 1000, lookback=LOOKBACK)
    out = BinaryPlan(ctx, "/", mk(lhs, True), mk(rhs, True)).execute()
    assert rows_of(out, "ts", ["host", "dc"]) == [("h1", "a", 0, 3.0), ("h2", "b", 0, 3.0)]
    assert sorted(out.column("__tsid").to_pylist()) == [11, 12]
    with pytest.raises(B2PError, match="No field named dc"):
        BinaryPlan(ctx, "/", mk(lhs, False), mk(rhs, False)).execute()


# ---- refusals ----------------------------------------------------------------------------------------------------------
def test_refusals(ctx):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import PromRangeExec
    A = {"time_index": "ts", "field": "val", "tags": ["job"], "series": [{"job": "a", "ts": [0], "val": [1.0]}]}
    # label columns on a Utf8-keyed leaf: at the call, tag columns other than __tsid alone; at push, a Utf8 __tsid
    for tags in (["job"], ["a", "b"]):
        with pytest.raises(B2PError, match="label columns need the one tag column to be the UInt64 id __tsid") as ei:
            PromRangeExec(ctx, "", 0, 0, 1000, 0, "ts", "val", tags, lookback_delta=LOOKBACK, label_columns=["host"])
        assert ei.value.code == -1
    n = PromRangeExec(ctx, "", 0, 0, 1000, 0, "ts", "val", ["__tsid"], lookback_delta=LOOKBACK, label_columns=["job"])
    b = table_batches(A, False)[0]
    with pytest.raises(B2PError, match="label columns need the tag column __tsid to be a UInt64 id") as ei:
        n.push(b.append_column("__tsid", pa.array(["7"], pa.string())))
    assert ei.value.code == -1
    # a label column named like the time index or a field
    for bad in ("ts", "val", "__tsid"):
        with pytest.raises(B2PError, match="is named like the time index, a field column or the id column"):
            PromRangeExec(ctx, "", 0, 0, 1000, 0, "ts", "val", ["__tsid"], label_columns=[bad])
    # a missing label column (Plan) and a non-Utf8 one (Execution)
    n = PromRangeExec(ctx, "", 0, 0, 1000, 0, "ts", "val", ["__tsid"], lookback_delta=LOOKBACK, label_columns=["nope"])
    with pytest.raises(B2PError, match="No field named nope") as ei:
        n.push(table_batches(A, True)[0])
    assert ei.value.code == -1
    b = table_batches(A, True)[0]
    b = pa.RecordBatch.from_arrays([b.column(0), b.column(1), pa.array([1], pa.int64()), b.column(3)],
                                   names=["ts", "val", "job", "__tsid"])
    n = PromRangeExec(ctx, "", 0, 0, 1000, 0, "ts", "val", ["__tsid"], lookback_delta=LOOKBACK, label_columns=["job"])
    with pytest.raises(B2PError, match="label column job must be Utf8") as ei:
        n.push(b)
    assert ei.value.code != -1
    # by-columns and the le column name label columns
    n = PromRangeExec(ctx, "", 0, 0, 1000, 0, "ts", "val", ["__tsid"], lookback_delta=LOOKBACK, aggregate="sum",
                      by_columns=["job"], label_columns=["job"])
    assert n.execute().num_rows == 0
    with pytest.raises(B2PError, match="by-column host is not a tag column"):
        PromRangeExec(ctx, "", 0, 0, 1000, 0, "ts", "val", ["__tsid"], aggregate="sum", by_columns=["host"],
                      label_columns=["job"])
    # any other leaf still checks its by-columns at create
    with pytest.raises(B2PError, match="by-column host is not a tag column"):
        PromRangeExec(ctx, "", 0, 0, 1000, 0, "ts", "val", ["job"], aggregate="sum", by_columns=["host"])
