"""GPU: absent() (K15 in b2p_absent.cuh) against the numpy OR of the rows' validity words, and the plan layer
(AbsentPlan) on the sqlness goldens, over every kind of child, with element-wise stages on top, under other nodes, and
its refusals."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

from tests import absent_oracle as ao
from tests.test_absent_oracle import CASES, G, LOOKBACK, child_series, names

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


# ---- K15 ------------------------------------------------------------------------------------------------------------
def tail_mask(T):
    """[Tw] u32: the bits of each word that are steps < T"""
    Tw = (T + 31) // 32
    m = np.full(Tw, 0xFFFFFFFF, np.uint32)
    if T % 32:
        m[-1] = (1 << (T % 32)) - 1
    return m


def expect(words, T):
    """numpy: the OR over rows, inverted, masked to the grid -> (out [T] f64, words [Tw] u32)"""
    Tw = (T + 31) // 32
    any_row = np.bitwise_or.reduce(words, axis=0) if words.shape[0] else np.zeros(Tw, np.uint32)
    gone = ~any_row & tail_mask(T)
    bits = np.unpackbits(gone.view(np.uint8), bitorder="little")[:T]
    return np.where(bits == 1, 1.0, 0.0), gone


def grid_words(rng, rows, T, kind):
    Tw = (T + 31) // 32
    stray = ~tail_mask(T)  # bits past T
    if kind == "all_valid":
        return np.full((rows, Tw), 0xFFFFFFFF, np.uint32)
    w = np.zeros((rows, Tw), np.uint32)
    if kind == "last_cell" and rows:
        w[-1, (T - 1) // 32] = np.uint32(1 << ((T - 1) % 32))
    elif kind == "stray":  # only bits past T, and one real cell in the first row: the stray bits must be ignored
        w[:] = stray
        if rows:
            w[0, 0] |= np.uint32(1)
    elif kind == "random":  # half the steps live; each row holds a random part of the live steps (dense or sparse)
        live = rng.integers(0, 2**32, Tw, dtype=np.uint64).astype(np.uint32)
        w = rng.integers(0, 2**32, (rows, Tw), dtype=np.uint64).astype(np.uint32) & live
        if rows > 100:
            w &= rng.integers(0, 2**32, (rows, Tw), dtype=np.uint64).astype(np.uint32)
            w &= rng.integers(0, 2**32, (rows, Tw), dtype=np.uint64).astype(np.uint32)
            w[rng.random(rows) < 0.99] = 0  # most rows empty, so steps stay absent with 10 000 rows
        w |= stray  # stray bits too
    return w


SHAPES = [(T, rows) for T in (1, 31, 32, 33, 1000, 65_537) for rows in (0, 1, 5, 10_000)]
KINDS = ("random", "all_valid", "all_invalid", "last_cell", "stray")


@pytest.mark.parametrize("T,rows", SHAPES)
def test_k15_equals_the_numpy_or(ctx, T, rows):
    rng = np.random.default_rng(T * 31 + rows)
    for kind in KINDS:
        words = grid_words(rng, rows, T, kind)
        out, ov = ctx.absent(words, T)
        e_out, e_ov = expect(words, T)
        assert ov.tolist() == e_ov.tolist(), kind
        assert out.view(np.uint64).tolist() == e_out.view(np.uint64).tolist(), kind
        if kind == "all_valid" and rows:
            assert not out.any()
        if kind in ("all_invalid",) or rows == 0:
            assert (out == 1.0).all()


def test_device_form_equals_host_form(ctx):
    import torch
    rng = np.random.default_rng(15)
    for rows, T in ((300, 97), (7, 70_001), (100_000, 1), (0, 40)):
        words = grid_words(rng, rows, T, "random")
        Tw = (T + 31) // 32
        d_valid = torch.from_numpy(words.view(np.int32)).cuda() if rows else None
        out = torch.full((T,), -7.0, dtype=torch.float64, device="cuda")
        ov = torch.full((Tw,), -1, dtype=torch.int32, device="cuda")
        ctx.absent_dev(d_valid, rows, T, out, ov)
        ctx.sync()
        h_out, h_ov = ctx.absent(words, T)
        assert out.cpu().numpy().view(np.uint64).tolist() == h_out.view(np.uint64).tolist()
        assert ov.cpu().numpy().view(np.uint32).tolist() == h_ov.tolist()
    ctx.absent_dev(None, 0, 0, None, None)  # no step: nothing to write
    ctx.sync()


def test_k15_null_arguments(ctx):
    from greptimedb_b200.engine import _ptr
    L = ctx._L
    words = np.zeros((2, 1), np.uint32)
    out = np.full(3, -7.0)
    ov = np.full(1, 7, np.uint32)
    for f in (L.b2p_absent, L.b2p_absent_dev):
        assert f(None, None, 0, 3, _ptr(out), _ptr(ov)) == -1
        assert f(ctx._h, None, 2, 3, _ptr(out), _ptr(ov)) == -1
        assert f(ctx._h, _ptr(words), 2, 3, None, _ptr(ov)) == -1
        assert f(ctx._h, _ptr(words), 2, 3, _ptr(out), None) == -1
        assert f(ctx._h, None, 0, 0, None, None) == 0
    assert out.tolist() == [-7.0] * 3 and ov.tolist() == [7]  # a refused call writes nothing
    assert L.b2p_absent(ctx._h, None, 0, 3, _ptr(out), _ptr(ov)) == 0  # no rows: every step is absent
    assert out.tolist() == [1.0] * 3 and ov.tolist() == [7]
    with pytest.raises(ValueError):
        ctx.absent(np.zeros((2, 2), np.uint32), 3)


# ---- plan layer -----------------------------------------------------------------------------------------------------
def table_batch(table, series):
    ts = [t for s in series for t in s["ts"]]
    val = [v for s in series for v in s["val"]]
    cols = [pa.array(ts, pa.timestamp("ms")), pa.array(val, pa.float64())]
    for t in table["tags"]:
        cols.append(pa.array([s[t] for s in series for _ in s["ts"]], pa.string()))
    return pa.record_batch(cols, names=[table["time_index"], table["field"]] + table["tags"])


def out_rows(b):
    """-> [(ts, value, {label: value})] in the batch's order"""
    ti = next(i for i, f in enumerate(b.schema) if pa.types.is_timestamp(f.type))
    vi = next(i for i, f in enumerate(b.schema) if pa.types.is_floating(f.type))
    ts = b.column(ti).cast(pa.int64()).to_pylist()
    vals = b.column(vi).to_pylist()
    tags = {n: b.column(i).to_pylist() for i, n in enumerate(b.schema.names) if i not in (ti, vi)}
    return [(ts[r], vals[r], {t: tags[t][r] for t in tags}) for r in range(b.num_rows)]


def golden_child(ctx, case):
    from greptimedb_b200.plan import PromRangeExec
    ti, field = names(case)
    tags = G["tables"][case["table"]]["tags"] if case["table"] else []
    ex = PromRangeExec(ctx, "", case["start"], case["end"], case["interval"], 0, ti, field, tags,
                       lookback_delta=LOOKBACK)
    series = child_series(case)
    if series:
        ex.push(table_batch(G["tables"][case["table"]], series))
    return ex


@pytest.mark.parametrize("name", sorted(CASES))
def test_plan_goldens(ctx, name):
    from greptimedb_b200.plan import AbsentPlan
    case = CASES[name]
    ti, field = names(case)
    labels = [(n, v) for n, op, v in case["matchers"] if op == "="]
    out = AbsentPlan(ctx, golden_child(ctx, case), case["start"], case["end"], case["interval"], ti, field,
                     labels).execute()
    assert [[ts, v, lab] for ts, v, lab in out_rows(out)] == case["expected"]
    want = case["columns"] or [ti, field] + [n for n, _ in ao.fake_labels(case["matchers"])]
    assert out.schema.names == want
    assert out.schema.field(0).type == pa.timestamp("ms") and out.schema.field(1).type == pa.float64()
    assert all(f.type == pa.string() for f in list(out.schema)[2:])


def empty_leaf(ctx, start=0, end=20_000, step=5000):
    from greptimedb_b200.plan import PromRangeExec
    return PromRangeExec(ctx, "", start, end, step, 0, "ts", "val", ["host"], lookback_delta=LOOKBACK)


def test_label_handling(ctx):
    from greptimedb_b200.plan import AbsentPlan
    cases = [
        ([("job", "a"), ("job", "b")], ["job"], {"job": "b"}),                    # the last one wins
        ([("z", "1"), ("a", "2"), ("Z", "3"), ("ä", "4"), ("b", "")], ["Z", "a", "b", "z", "ä"],
         {"z": "1", "a": "2", "Z": "3", "ä": "4", "b": ""}),                      # byte order; "" kept
        ([], [], {}),                                                              # no labels
    ]
    for labels, order, want in cases:
        out = AbsentPlan(ctx, empty_leaf(ctx), 0, 20_000, 5000, "ts", "val", labels).execute()
        assert out.schema.names == ["ts", "val"] + order
        assert out_rows(out) == [(t, 1.0, want) for t in range(0, 20_001, 5000)]


# A sparse table: a sample is visible at one step only (lookback 4 s < step 5 s); some steps have no sample in any
# series, one has a sample in a single series
STEP, START, END, LB = 5000, 0, 60_000, 4000
HOSTS, LES = ["a", "b"], ["0.5", "+Inf"]
EMPTY_STEPS = {3, 7, 8, 12}
LONE_STEP = 5


def sparse_table():
    rng = np.random.default_rng(4)
    series = []
    for h in HOSTS:
        for le in LES:
            ks = [k for k in range(13) if k not in EMPTY_STEPS and (rng.random() < 0.6 or (h, le) == ("a", "+Inf"))]
            if (h, le) != ("a", "+Inf"):
                ks = [k for k in ks if k != LONE_STEP]
            series.append({"host": h, "le": le, "ts": [k * STEP - int(rng.integers(0, 3)) * 1000 for k in ks],
                           "val": [float(rng.integers(0, 9)) for _ in ks]})
    return {"time_index": "ts", "field": "val", "tags": ["host", "le"], "series": series}


SPARSE = sparse_table()


def leaf(ctx, function="", start=START, **match):
    from greptimedb_b200.plan import PromRangeExec
    series = [s for s in SPARSE["series"] if all(s[k] == v for k, v in match.items())]
    if function:
        ex = PromRangeExec(ctx, function, start, END, STEP, 5000, "ts", "val", SPARSE["tags"])
    else:
        ex = PromRangeExec(ctx, "", start, END, STEP, 0, "ts", "val", SPARSE["tags"], lookback_delta=LB,
                           need_filter_out_nan=False)
    ex.push(table_batch(SPARSE, series))
    return ex


def id_keyed(ctx):
    from greptimedb_b200.plan import PromRangeExec
    ex = PromRangeExec(ctx, "", START, END, STEP, 0, "ts", "val", ["__tsid"], lookback_delta=LB,
                       need_filter_out_nan=False)
    ts = [0, 5000, 20_000, 30_000, 0, 50_000]
    ex.push(pa.record_batch([pa.array(ts, pa.timestamp("ms")), pa.array([1.0, 2.0, float("nan"), 4.0, 5.0, 6.0]),
                             pa.array([1, 1, 1, 1, 2, 2], pa.uint64())], names=["ts", "val", "__tsid"]))
    return ex


def children(ctx):
    from greptimedb_b200.plan import (AggregatePlan, BinaryPlan, CountValuesPlan, HistogramQuantilePlan, ScalarPlan,
                                      SetOpPlan, SortPlan, SubqueryPlan, TopkPlan)
    return {  # name -> (make, the child's grid start)
        "range": (lambda: leaf(ctx, "prom_max_over_time"), START),
        "instant": (lambda: leaf(ctx), START),
        "nan_values": (lambda: leaf(ctx).scalar_op("*", float("nan")), START),  # every cell valid and NaN
        "aggregate": (lambda: AggregatePlan(ctx, "sum", leaf(ctx), by=["le"]), START),
        "binary": (lambda: BinaryPlan(ctx, "-", leaf(ctx), leaf(ctx).scalar_op("*", 2.0)), START),
        "or": (lambda: SetOpPlan(ctx, "or", leaf(ctx, le="0.5"), leaf(ctx, host="b")), START),
        "topk": (lambda: TopkPlan(ctx, "topk", 1, leaf(ctx), by=["host"]), START),
        "subquery": (lambda: SubqueryPlan(ctx, "prom_count_over_time", leaf(ctx, start=15_000), 20_000, END, STEP,
                                          10_000), 20_000),
        "histogram_quantile": (lambda: HistogramQuantilePlan(ctx, 0.5, leaf(ctx)), START),
        "scalar": (lambda: ScalarPlan(ctx, leaf(ctx, host="b", le="0.5")), START),
        "count_values": (lambda: CountValuesPlan(ctx, "v", leaf(ctx)), START),
        "sort": (lambda: SortPlan(ctx, "sort_desc", leaf(ctx)), START),
        "no_columns": (lambda: HistogramQuantilePlan(ctx, 0.5, leaf(ctx), le="__absent__"), START),
        "id_keyed": (lambda: id_keyed(ctx), START),
    }


def present(batch):
    """the timestamps at which the child's export has a row: the steps with a valid cell"""
    if batch.num_columns == 0:
        return set()
    ti = next(i for i, f in enumerate(batch.schema) if pa.types.is_timestamp(f.type))
    return set(batch.column(ti).cast(pa.int64()).to_pylist())


CHILDREN = ["range", "instant", "nan_values", "aggregate", "binary", "or", "topk", "subquery", "histogram_quantile", "scalar",
            "count_values", "sort", "no_columns", "id_keyed"]


@pytest.mark.parametrize("child", CHILDREN)
def test_absent_over_every_child(ctx, child):
    from greptimedb_b200.plan import AbsentPlan
    make, start = children(ctx)[child]
    c_batch = make().execute()
    seen = present(c_batch)
    grid = ao.grid(start, END, STEP)
    want = [t for t in grid if t not in seen]
    if child in ("instant", "nan_values"):  # the sparse table's empty steps; a NaN cell is present
        assert want == [k * STEP for k in sorted(EMPTY_STEPS)] and LONE_STEP * STEP in seen
    if child == "nan_values":
        assert all(v != v for _, v, _ in out_rows(c_batch))
    if child == "no_columns":
        assert want == grid
    out = AbsentPlan(ctx, make(), start, END, STEP, "ts", "value", [("job", "x")]).execute()
    assert out_rows(out) == [(t, 1.0, {"job": "x"}) for t in want], child
    assert out.schema.names == ["ts", "value", "job"]


def absent_node(ctx, labels=(("job", "x"),)):
    from greptimedb_b200.plan import AbsentPlan
    return AbsentPlan(ctx, leaf(ctx), START, END, STEP, "ts", "val", list(labels))


ABSENT_TS = [k * STEP for k in sorted(EMPTY_STEPS)]


def test_stages_on_the_node(ctx):
    out = absent_node(ctx).scalar_op("*", 2.0).function("clamp_max", 1.5).execute()
    assert out_rows(out) == [(t, 1.5, {"job": "x"}) for t in ABSENT_TS]
    assert out.schema.names == ["ts", "clamp_max(val * Float64(2),Float64(1.5))", "job"]
    assert absent_node(ctx).scalar_op(">", 1.0).execute().num_rows == 0  # a filter clears the node's one row
    out = absent_node(ctx).scalar_op("==", 1.0, return_bool=True).execute()
    assert out_rows(out) == [(t, 1.0, {"job": "x"}) for t in ABSENT_TS]


def test_nodes_above(ctx):
    from greptimedb_b200.plan import AggregatePlan, BinaryPlan, SetOpPlan
    out = AggregatePlan(ctx, "sum", absent_node(ctx)).execute()
    assert [(ts, v) for ts, v, _ in out_rows(out)] == [(t, 1.0) for t in ABSENT_TS]
    out = AggregatePlan(ctx, "count", absent_node(ctx), by=["job"]).execute()
    assert out_rows(out) == [(t, 1.0, {"job": "x"}) for t in ABSENT_TS]
    out = BinaryPlan(ctx, "+", absent_node(ctx), absent_node(ctx)).execute()
    assert out_rows(out) == [(t, 2.0, {"job": "x"}) for t in ABSENT_TS]
    # vector or absent(..): the leaf's rows, then the absent row (its labels differ from every leaf row's)
    lhs = out_rows(leaf(ctx).execute())
    out = out_rows(SetOpPlan(ctx, "or", leaf(ctx), absent_node(ctx)).execute())
    assert len(out) == len(lhs) + len(ABSENT_TS)
    assert [(ts, v, lab.get("job")) for ts, v, lab in out[len(lhs):]] == [(t, 1.0, "x") for t in ABSENT_TS]


def test_start_after_end(ctx):
    from greptimedb_b200.plan import AbsentPlan
    out = AbsentPlan(ctx, empty_leaf(ctx, 10_000, 0), 10_000, 0, STEP, "ts", "val", [("job", "x")]).execute()
    assert out.num_rows == 0 and out.schema.names == ["ts", "val", "job"]


def test_refusals(ctx):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import AbsentPlan, _cstr_array
    for kw in (dict(interval=0), dict(interval=-5000), dict(labels=[("ts", "a")]), dict(labels=[("val", "a")])):
        args = dict(start=START, end=END, interval=STEP, time_index="ts", value_column="val", labels=[("job", "x")])
        args.update(kw)
        with pytest.raises(B2PError) as ei:
            AbsentPlan(ctx, empty_leaf(ctx), **args)
        assert ei.value.code == -1, kw
    L = ctx._L
    child = empty_leaf(ctx)
    n, v = _cstr_array(["job"]), _cstr_array(["x"])
    nul = (C.c_char_p * 1)()  # one NULL string
    assert not L.b2p_plan_absent_create(None, 0, 10, 5, b"ts", b"val", n, v, 1, child._h)   # NULL ctx
    assert not L.b2p_plan_absent_create(ctx._h, 0, 10, 5, b"ts", b"val", n, v, 1, None)     # NULL child
    assert not L.b2p_plan_absent_create(ctx._h, 0, 10, 5, None, b"val", n, v, 1, child._h)  # NULL time index
    assert not L.b2p_plan_absent_create(ctx._h, 0, 10, 5, b"ts", None, n, v, 1, child._h)   # NULL value column
    assert not L.b2p_plan_absent_create(ctx._h, 0, 10, 5, b"ts", b"val", nul, v, 1, child._h)  # NULL label name
    assert not L.b2p_plan_absent_create(ctx._h, 0, 10, 5, b"ts", b"val", n, nul, 1, child._h)  # NULL label value
    assert not L.b2p_plan_absent_create(ctx._h, 0, 10, 5, b"ts", b"val", None, None, 1, child._h)
    assert not L.b2p_plan_absent_create(ctx._h, 0, 10, 5, b"ts", b"val", n, v, -1, child._h)  # n_labels < 0
    h = L.b2p_plan_absent_create(ctx._h, 0, 10, 5, b"ts", b"val", None, None, 0, child._h)
    assert h
    L.b2p_plan_destroy(h)
    # at execute: a child with rows on another grid
    for start, end, step in ((START + 1, END, STEP), (START, END, STEP * 2), (START, END - STEP, STEP)):
        with pytest.raises(B2PError) as ei:
            AbsentPlan(ctx, leaf(ctx), start, end, step, "ts", "val").execute()
        assert ei.value.code == -1 and "grid" in str(ei.value)
    # a child without rows is absent at every step of the node's grid, whatever grid it was built on
    out = AbsentPlan(ctx, empty_leaf(ctx, 0, 5, 1), START, END, STEP, "ts", "val").execute()
    assert [r[0] for r in out_rows(out)] == ao.grid(START, END, STEP)
