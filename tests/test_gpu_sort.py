"""GPU: sort / sort_desc (K14 in b2p_sort.cuh) against the oracle's permutation exactly, and the plan layer (SortPlan)
on the sqlness goldens, over every kind of child, with element-wise stages on top, under other nodes, and its
refusals."""
import numpy as np
import pyarrow as pa
import pytest

from tests import sort_oracle as so
from tests.binary_oracle import _words
from tests.test_sort_oracle import CASES, G, LOOKBACK, TOTAL_ORDER

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.uint64)


# ---- K14 ------------------------------------------------------------------------------------------------------------
def grid(rng, rows, T, kind):
    if kind == "special":
        vals = np.array(TOTAL_ORDER)[rng.integers(0, len(TOTAL_ORDER), (rows, T))]
    elif kind == "equal":
        vals = np.full((rows, T), 3.5)
    elif kind == "counter":  # monotone runs with resets: long runs of ties across rows
        vals = np.cumsum(rng.integers(0, 3, (rows, T)), axis=1).astype(np.float64)
        vals[:, T // 2:] -= vals[:, T // 2:T // 2 + 1] if T > 1 else 0.0
    else:
        vals = rng.standard_normal((rows, T))
    ok = rng.random((rows, T)) < 0.7
    return vals, ok


SHAPES = [(T, rows) for T in (1, 31, 32, 33, 1000) for rows in (0, 1, 5, 10_000)]


@pytest.mark.parametrize("T,rows", SHAPES)
def test_k14_equals_the_oracle(ctx, T, rows):
    rng = np.random.default_rng(T * 7919 + rows)
    kinds = ("special", "equal", "counter", "random") if rows * T <= 1_000_000 else ("special",)
    for kind in kinds:
        vals, ok = grid(rng, rows, T, kind)
        for desc in (False, True):
            got = ctx.sort_cells(desc, vals, _words(ok))
            assert got.dtype == np.uint64
            assert got.tolist() == so.value_order(vals, ok, desc).tolist(), (kind, desc)


def test_k14_all_invalid_and_stray_bits(ctx):
    rng = np.random.default_rng(3)
    vals, ok = grid(rng, 7, 45, "special")
    assert ctx.sort_cells(False, vals, np.zeros((7, 2), np.uint32)).size == 0
    words = _words(ok)
    words[:, -1] |= np.uint32(0xFFFFFFFF) << np.uint32(45 % 32)  # bits past T in each row's last word are ignored
    for desc in (False, True):
        assert ctx.sort_cells(desc, vals, words).tolist() == so.value_order(vals, ok, desc).tolist()


def test_device_form_equals_host_form(ctx):
    import torch
    rng = np.random.default_rng(5)
    R, T = 300, 97
    vals, ok = grid(rng, R, T, "special")
    words = _words(ok)
    d_vals = torch.from_numpy(vals).cuda()
    d_valid = torch.from_numpy(words.view(np.int32)).cuda()
    for desc in (False, True):
        cells = torch.full((R * T,), -1, dtype=torch.int64, device="cuda")
        n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        ctx.sort_cells_dev(desc, d_vals, d_valid, R, T, cells, n)
        ctx.sync()
        n = int(n.item())
        assert n == int(ok.sum())
        got = cells.cpu().numpy().view(np.uint64)
        assert got[:n].tolist() == ctx.sort_cells(desc, vals, words).tolist()
        assert (cells.cpu().numpy()[n:] == -1).all()  # nothing past the valid cells is written
    n = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    ctx.sort_cells_dev(False, None, None, 0, T, None, n)
    ctx.sync()
    assert int(n.item()) == 0


def test_k14_null_arguments(ctx):
    from greptimedb_b200.engine import _ptr
    L = ctx._L
    vals = np.zeros((2, 3))
    words = np.zeros((2, 1), np.uint32)
    out = np.zeros(6, np.uint64)
    n = np.zeros(1, np.uint64)
    assert L.b2p_sort_cells(ctx._h, 0, _ptr(vals), _ptr(words), 2, 3, _ptr(out), None) == -1
    assert L.b2p_sort_cells(ctx._h, 0, None, _ptr(words), 2, 3, _ptr(out), _ptr(n)) == -1
    assert L.b2p_sort_cells(ctx._h, 0, _ptr(vals), _ptr(words), 2, 3, None, _ptr(n)) == -1
    assert L.b2p_sort_cells_dev(None, 0, None, None, 0, 0, None, None) == -1
    with pytest.raises(ValueError):
        ctx.sort_cells(False, vals, np.zeros((2, 2), np.uint32))


# ---- plan layer -----------------------------------------------------------------------------------------------------
def table_batch(table, series):
    ts = [t for s in series for t in s["ts"]]
    val = [v for s in series for v in s["val"]]
    cols = [pa.array(ts, pa.timestamp("ms")), pa.array(val, pa.float64())]
    for t in table["tags"]:
        cols.append(pa.array([s[t] for s in series for _ in s["ts"]], pa.string()))
    return pa.record_batch(cols, names=[table["time_index"], table["field"]] + table["tags"])


def out_rows(b):
    """-> ([(value, {tag: label}, ts)] in the batch's order, tag names in column order)"""
    names = b.schema.names
    vi = next(i for i, f in enumerate(b.schema) if pa.types.is_floating(f.type))
    ti = next(i for i, f in enumerate(b.schema) if pa.types.is_timestamp(f.type))
    ts = b.column(ti).cast(pa.int64()).to_pylist()
    vals = b.column(vi).to_numpy(zero_copy_only=False)
    tags = [n for i, n in enumerate(names) if i not in (vi, ti)]
    cols = {t: b.column(names.index(t)).to_pylist() for t in tags}
    return [(vals[r], {t: cols[t][r] for t in tags}, ts[r]) for r in range(b.num_rows)], tags


def key(rows):
    return [(int(bits([v])[0]), sorted(lab.items(), key=lambda x: x[0]), ts) for v, lab, ts in rows]


def golden_child(ctx, case):
    from greptimedb_b200.plan import PromRangeExec
    t = G["tables"][case["input"]["table"]]
    series = [s for s in t["series"] if all(s[k] == v for k, v in case["input"]["match"].items())]
    ex = PromRangeExec(ctx, "", case["start"], case["end"], case["interval"], 0, t["time_index"], t["field"], t["tags"],
                       aggregate=case["input"]["aggregate"], by_columns=case["input"]["by"], lookback_delta=LOOKBACK)
    ex.push(table_batch(t, series))
    return ex


@pytest.mark.parametrize("name", sorted(CASES))
def test_plan_goldens(ctx, name):
    from greptimedb_b200.plan import SortPlan
    case = CASES[name]
    out = SortPlan(ctx, case["function"], golden_child(ctx, case), case["labels"]).execute()
    rows, _ = out_rows(out)
    got = [(lab, None if "ts" in case["masked"] else ts, None if "val" in case["masked"] else float(v))
           for v, lab, ts in rows]
    assert got == [(lab, ts, v) for lab, ts, v in case["expected"]]
    # {time index, value, tags..}; the reference qualifies the aggregate's value column (sum(test.val)), this layer
    # names it sum(val)
    names = list(case["columns"])
    if case["input"]["aggregate"]:
        names[1] = names[1].replace("test.", "")
    assert out.schema.names == names


# A table with ties, special values, "" and NULL labels, and an le tag: host x le, one sample every 5 s
HOSTS = ["a", "b", "", None]
LES = ["0.5", "1", "+Inf"]
STEP, START, END = 5000, 0, 60_000


def mixed_table(seed=11):
    rng = np.random.default_rng(seed)
    special = [float("inf"), float("-inf"), -0.0, 0.0, float("nan")]
    series = []
    for h in HOSTS:  # (grouped by series; SeriesDivide needs no particular order of the groups)
        for le in LES:
            n = 13
            v = rng.integers(0, 4, n).astype(np.float64)
            hit = rng.random(n) < 0.15
            v[hit] = np.array(special)[rng.integers(0, len(special), int(hit.sum()))]
            keep = rng.random(n) < 0.85
            series.append({"host": h, "le": le, "ts": [int(t) for t in np.arange(n)[keep] * STEP],
                           "val": v[keep].tolist()})
    return {"time_index": "ts", "field": "val", "tags": ["host", "le"], "series": series}


MIXED = mixed_table()


def leaf(ctx, function="", start=START, **match):
    from greptimedb_b200.plan import PromRangeExec
    series = [s for s in MIXED["series"] if all(s[k] == v for k, v in match.items())]
    if function:
        ex = PromRangeExec(ctx, function, start, END, STEP, 15_000, "ts", "val", MIXED["tags"])
    else:
        ex = PromRangeExec(ctx, "", start, END, STEP, 0, "ts", "val", MIXED["tags"], lookback_delta=20_000,
                           need_filter_out_nan=False)
    ex.push(table_batch(MIXED, series))
    return ex


def children(ctx):
    from greptimedb_b200.plan import (AggregatePlan, BinaryPlan, HistogramQuantilePlan, ScalarPlan, SetOpPlan,
                                      SubqueryPlan)
    return {
        "range": lambda: leaf(ctx, "prom_max_over_time"),
        "instant": lambda: leaf(ctx),
        "aggregate": lambda: AggregatePlan(ctx, "sum", leaf(ctx), by=["le"]),
        "binary": lambda: BinaryPlan(ctx, "-", leaf(ctx), leaf(ctx).scalar_op("*", 2.0)),
        "or": lambda: SetOpPlan(ctx, "or", leaf(ctx, le="1"), leaf(ctx)),
        "subquery": lambda: SubqueryPlan(ctx, "prom_max_over_time", leaf(ctx, start=20_000), 30_000, END, STEP, 15_000),
        "histogram_quantile": lambda: HistogramQuantilePlan(ctx, 0.5, leaf(ctx)),
        "scalar": lambda: ScalarPlan(ctx, leaf(ctx, host="a", le="1")),
    }


FUNCTIONS = [("sort", ()), ("sort_desc", ()), ("sort_by_label", ("le", "host")), ("sort_by_label_desc", ("host",)),
             ("sort_by_label_desc", ("le",))]
CHILDREN = ["range", "instant", "aggregate", "binary", "or", "subquery", "histogram_quantile", "scalar"]


def expected_columns(child_batch):
    """the sort node's columns over a child batch: time index, value, then the child's tags in its label order"""
    rows, tags = out_rows(child_batch)
    names = child_batch.schema.names
    vi = next(i for i, f in enumerate(child_batch.schema) if pa.types.is_floating(f.type))
    ti = next(i for i, f in enumerate(child_batch.schema) if pa.types.is_timestamp(f.type))
    return [names[ti], names[vi]] + tags


@pytest.mark.parametrize("child", CHILDREN)
def test_sort_over_every_child(ctx, child):
    from greptimedb_b200.plan import SortPlan
    make = children(ctx)[child]
    c_batch = make().execute()
    rows, tags = out_rows(c_batch)
    assert rows, child
    for function, labels in FUNCTIONS:
        if labels and not set(labels) <= set(tags):
            continue
        out = SortPlan(ctx, function, make(), labels).execute()
        got, _ = out_rows(out)
        assert key(got) == key(so.sort_rows(function, rows, labels)), (child, function)
        assert out.schema.names == expected_columns(c_batch), (child, function)
    if child == "or":  # its {time index, tags and value in name order} layout becomes {time index, value, tags..}
        assert c_batch.schema.names == ["ts", "host", "le", "val"]
        assert SortPlan(ctx, "sort", make()).execute().schema.names == ["ts", "val", "host", "le"]


def test_sort_over_topk(ctx):
    """topk's rank order is ignored: its kept cells in row-major order (the rows of its child) are what is sorted"""
    from greptimedb_b200.plan import SortPlan, TopkPlan
    child_rows, _ = out_rows(leaf(ctx).execute())
    kept = {(tuple(sorted(lab.items(), key=lambda x: x[0])), ts) for _, lab, ts in
            out_rows(TopkPlan(ctx, "topk", 2, leaf(ctx), by=["le"]).execute())[0]}
    rows = [r for r in child_rows if (tuple(sorted(r[1].items(), key=lambda x: x[0])), r[2]) in kept]
    assert len(rows) == len(kept)
    for function, labels in FUNCTIONS:
        out = SortPlan(ctx, function, TopkPlan(ctx, "topk", 2, leaf(ctx), by=["le"]), labels).execute()
        assert key(out_rows(out)[0]) == key(so.sort_rows(function, rows, labels)), function
        assert out.schema.names == ["ts", "val", "host", "le"]


def loose(rows):  # (a NaN's payload after arithmetic is the device's: every NaN compares alike here)
    return [("NaN" if v != v else v, sorted(lab.items(), key=lambda x: x[0]), ts) for v, lab, ts in rows]


def test_stages_apply_after_the_order(ctx):
    from greptimedb_b200.plan import SortPlan
    rows, _ = out_rows(leaf(ctx).execute())
    for function, labels in FUNCTIONS:
        exp = so.sort_rows(function, rows, labels)
        out = SortPlan(ctx, function, leaf(ctx), labels).scalar_op("*", -1.0).function("abs").execute()
        assert loose(out_rows(out)[0]) == loose([(abs(v), lab, ts) for v, lab, ts in exp]), function
        assert out.schema.names[1].startswith("abs(val * ")
        # a comparison filter clears bits: those cells are not exported, the others keep their places
        out = SortPlan(ctx, function, leaf(ctx), labels).scalar_op(">", 1.0).execute()
        assert key(out_rows(out)[0]) == key([r for r in exp if r[0] > 1.0]), function
        assert out.schema.names == ["ts", "val", "host", "le"]


def batches_equal(a, b):
    assert a.schema.names == b.schema.names
    for i in range(a.num_columns):
        x, y = a.column(i), b.column(i)
        if pa.types.is_floating(x.type):
            assert bits(x.to_numpy(zero_copy_only=False)).tolist() == bits(y.to_numpy(zero_copy_only=False)).tolist()
        else:
            assert x.to_pylist() == y.to_pylist()


def test_nodes_above_see_the_child(ctx):
    from greptimedb_b200.plan import AggregatePlan, BinaryPlan, SortPlan, TopkPlan
    for function, labels in FUNCTIONS:
        s = lambda: SortPlan(ctx, function, leaf(ctx), labels)
        batches_equal(AggregatePlan(ctx, "sum", s(), by=["host"]).execute(),
                      AggregatePlan(ctx, "sum", leaf(ctx), by=["host"]).execute())
        batches_equal(TopkPlan(ctx, "bottomk", 1, s(), by=["le"]).execute(),
                      TopkPlan(ctx, "bottomk", 1, leaf(ctx), by=["le"]).execute())
        batches_equal(BinaryPlan(ctx, "+", s(), leaf(ctx)).execute(), BinaryPlan(ctx, "+", leaf(ctx), leaf(ctx)).execute())
        batches_equal(BinaryPlan(ctx, "*", leaf(ctx), s()).execute(), BinaryPlan(ctx, "*", leaf(ctx), leaf(ctx)).execute())


def test_child_without_columns_and_id_keyed_child(ctx):
    from greptimedb_b200.plan import HistogramQuantilePlan, PromRangeExec, SortPlan
    for function, labels in FUNCTIONS:
        out = SortPlan(ctx, function, HistogramQuantilePlan(ctx, 0.5, leaf(ctx), le="__absent__"), labels).execute()
        assert out.num_rows == 0 and out.num_columns == 0
    ids = np.repeat(np.arange(3, dtype=np.uint64), 4)
    b = pa.record_batch([pa.array(np.tile(np.arange(4) * STEP, 3), pa.timestamp("ms")),
                         pa.array([2.0, 1.0, 3.0, 1.0, 0.0, -0.0, 5.0, 1.0, 2.0, 2.0, 9.0, -1.0]),
                         pa.array(ids, pa.uint64())], names=["ts", "val", "__tsid"])
    byid = lambda: PromRangeExec(ctx, "", 0, 3 * STEP, STEP, 0, "ts", "val", ["__tsid"], lookback_delta=LOOKBACK)
    child = byid()
    child.push(b)
    rows, _ = out_rows(child.execute())
    for function in ("sort", "sort_desc"):
        node = byid()
        node.push(b)
        out = SortPlan(ctx, function, node).execute()
        assert key(out_rows(out)[0]) == key(so.sort_rows(function, rows))
        assert out.schema.names == ["ts", "val", "__tsid"]


def test_refusals(ctx):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import CountValuesPlan, PromRangeExec, SortPlan
    for function, labels in [("sorted", ()), ("sort_by_label", ()), ("sort_by_label_desc", ()), ("sort", ("host",)),
                             ("sort_desc", ("host",)), ("", ())]:
        with pytest.raises(B2PError) as ei:
            SortPlan(ctx, function, leaf(ctx), labels)
        assert ei.value.code == -1, function
    with pytest.raises(B2PError) as ei:
        SortPlan(ctx, "sort_by_label", leaf(ctx), ["host", "nope"]).execute()
    assert ei.value.code == -1 and "nope" in str(ei.value)
    byid = PromRangeExec(ctx, "", 0, 3 * STEP, STEP, 0, "ts", "val", ["__tsid"], lookback_delta=LOOKBACK)
    byid.push(pa.record_batch([pa.array([0, STEP], pa.timestamp("ms")), pa.array([1.0, 2.0]),
                               pa.array([7, 7], pa.uint64())], names=["ts", "val", "__tsid"]))
    with pytest.raises(B2PError) as ei:
        SortPlan(ctx, "sort_by_label_desc", byid, ["__tsid"]).execute()
    assert ei.value.code == -1 and "__tsid" in str(ei.value)
    for function, labels in FUNCTIONS:
        with pytest.raises(B2PError) as ei:
            SortPlan(ctx, function, CountValuesPlan(ctx, "v", leaf(ctx)), labels).execute()
        assert ei.value.code == -1 and "count_values" in str(ei.value), function
