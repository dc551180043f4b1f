"""GPU: Int64 (BIGINT) value columns.  Every BIGINT golden table through the plan API with the reference's digits and
Arrow types; each Int64 entry point against tests/int64_oracle.py on random grids (50 % validity, INT64_MIN / INT64_MAX,
i64s whose bits are NaN doubles, ties, |v| > 2^53); a mixed [f64, i64] instant leaf; and the shapes the plan layer
leaves on the CPU, with their messages."""
import json
import os

import numpy as np
import pyarrow as pa
import pytest

from tests import int64_oracle as io
from tests.binary_oracle import _words

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_int64_vectors.json")))


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def batch(rows, pred=lambda r: True, val_type=pa.int64()):
    rows = sorted((r for r in rows if pred(r)), key=lambda r: (r[1], r[2], r[0]))
    return pa.record_batch([pa.array([r[0] for r in rows], pa.timestamp("ms")), pa.array([r[1] for r in rows], pa.utf8()),
                            pa.array([r[2] for r in rows], pa.utf8()), pa.array([r[3] for r in rows], val_type)],
                           names=["ts", "host", "idc", "val"])


def leaf(ctx, rows, pred=lambda r: True, function="", val_type=pa.int64()):
    from greptimedb_b200.plan import PromRangeExec
    if function:
        ex = PromRangeExec(ctx, function, 0, 15_000, 5_000, 10_000, "ts", "val", ["host", "idc"])
    else:
        ex = PromRangeExec(ctx, "", 0, 15_000, 5_000, 0, "ts", "val", ["host", "idc"], lookback_delta=io.LOOKBACK)
    ex.push(batch(rows, pred, val_type))
    return ex


def plan_of(ctx, case, rows):
    from greptimedb_b200.plan import AggregatePlan, CountValuesPlan, SortPlan, TopkPlan
    q = case["query"]
    if q.startswith("sort"):
        fn = "sort_desc" if q.startswith("sort_desc") else "sort"
        if "sum(" in q:
            return SortPlan(ctx, fn, AggregatePlan(ctx, "sum", leaf(ctx, rows, lambda r: r[1] == "host2"), by=["idc"]))
        return SortPlan(ctx, fn, leaf(ctx, rows, lambda r: r[1] == "host1"))
    if q.startswith("count_values"):
        return CountValuesPlan(ctx, "status_code", leaf(ctx, rows), by=["idc"] if q.endswith("by (idc)") else None)
    if q == "quantile(0.5, test)":
        return AggregatePlan(ctx, "quantile", leaf(ctx, rows), param=0.5)
    if q == "quantile(0.5, test) by (idc)":
        return AggregatePlan(ctx, "quantile", leaf(ctx, rows), param=0.5, by=["idc"])
    if q.startswith("quantile"):
        return AggregatePlan(ctx, "quantile", AggregatePlan(ctx, "sum", leaf(ctx, rows), by=["idc"]), param=0.5)
    if q.startswith("topk"):
        return TopkPlan(ctx, "topk", float(q[len("topk("):q.index(",")]), leaf(ctx, rows))
    raise KeyError(q)


def printed_rows(out, stamp_ts):
    cols = []
    for i in range(out.num_columns):
        col, typ = out.column(i), out.schema.field(i).type
        if pa.types.is_timestamp(typ):
            cols.append(["timestamp" if not stamp_ts else io.stamp(v) for v in col.cast(pa.int64()).to_pylist()])
        elif pa.types.is_int64(typ):
            cols.append([io.printed(v, "Int64") for v in col.to_pylist()])
        elif pa.types.is_floating(typ):
            cols.append([io.printed(v, "Float64") for v in col.to_pylist()])
        else:
            cols.append(col.to_pylist())
    return [list(r) for r in zip(*cols)]


def build(ctx, expr):
    """the plan of one golden expression (tests/int64_oracle.py `run` evaluates the same tree)"""
    from greptimedb_b200.plan import (AggregatePlan, BinaryPlan, PromRangeExec, ScalarPlan, TopkPlan)
    kind = expr[0]
    if kind == "sel":
        _, name, field, match = expr
        tab = GOLDEN["tables"][name]
        tags = tab["tags"]
        rows = [r for r in tab["rows"] if all(r[1 + tags.index(k)] == v for k, v in match.items())]
        rows.sort(key=lambda r: (tuple(r[1:1 + len(tags)]), r[0]))
        cols = [pa.array([r[0] for r in rows], pa.timestamp("ms"))] + \
            [pa.array([r[1 + i] for r in rows], pa.utf8()) for i in range(len(tags))] + \
            [pa.array([r[1 + len(tags) + i] for r in rows], pa.int64()) for i in range(len(tab["fields"]))]
        ex = PromRangeExec(ctx, "", 0, 15_000, 5_000, 0, "ts", field, tags, lookback_delta=io.LOOKBACK)
        ex.push(pa.record_batch(cols, names=["ts"] + tags + tab["fields"]))
        return ex
    if kind == "sum_by":
        return AggregatePlan(ctx, "sum", build(ctx, expr[2]), by=expr[1])
    if kind == "topk":
        return TopkPlan(ctx, "bottomk" if expr[2] else "topk", float(expr[1]), build(ctx, expr[3]))
    if kind == "scalar":
        return ScalarPlan(ctx, build(ctx, expr[1]))
    if kind == "op":
        return build(ctx, expr[4]).scalar_op(expr[1], expr[2], scalar_on_left=expr[3])
    if kind == "bin":
        return BinaryPlan(ctx, expr[1], build(ctx, expr[2]), build(ctx, expr[3]), label_side=expr[4])
    if kind == "fn":
        return build(ctx, expr[3]).function(expr[1], *expr[2])
    raise KeyError(kind)


EXPR_CASES = [c for c in GOLDEN["cases"] if "expr" in c]


@pytest.mark.parametrize("case", EXPR_CASES, ids=[c["query"] for c in EXPR_CASES])
def test_golden_expression_from_the_device(ctx, case):
    """topk / bottomk over Int64 and over sum of Int64 (one- and two-field tables), and the Float64 promotion of
    scalar(), arithmetic with a scalar or literal operand and clamp*, as the reference prints them"""
    out = build(ctx, case["expr"]).execute()
    got = printed_rows(out, True)
    want = case["rows"]
    if case["sorted"]:
        got, want = sorted(got), sorted(want)
    assert got == want
    col = 0 if case["expr"][0] == "topk" else [i for i in range(out.num_columns)
                                               if not pa.types.is_timestamp(out.schema.field(i).type)
                                               and out.schema.field(i).name not in ("host", "idc")][0]
    assert out.schema.field(col).type == (pa.int64() if case["expr"][0] == "topk" else pa.float64())


ROW_CASES = [c for c in GOLDEN["cases"] if "expr" not in c]


@pytest.mark.parametrize("case", ROW_CASES, ids=[c["query"] for c in ROW_CASES])
def test_golden_table_from_the_device(ctx, case):
    rows = GOLDEN["tables"][case["table"]]["rows"]
    out = plan_of(ctx, case, rows).execute()
    stamp_ts = case["rows"][0].count("timestamp") == 0
    assert printed_rows(out, stamp_ts) == case["rows"]
    # the value column's Arrow type is the reference's: Int64 except under quantile
    q = case["query"]
    val_col = 0 if q.startswith(("topk", "count_values")) else [
        i for i in range(out.num_columns) if not pa.types.is_timestamp(out.schema.field(i).type)
        and out.schema.field(i).name not in ("host", "idc")][0]
    want = pa.float64() if q.startswith("quantile") else pa.int64()
    assert out.schema.field(val_col).type == want
    if q.startswith("count_values"):
        assert out.schema.field(out.num_columns - 1).type == pa.int64()  # the label column


# ---- the entry points against the oracle ------------------------------------------------------------------------
NAN_BITS = np.array([np.nan, -np.nan], np.float64).view(np.int64)
SPECIAL = np.array([io.INT64_MIN, io.INT64_MAX, -1, 0, 1, 2, NAN_BITS[0], NAN_BITS[1], (1 << 53) + 1, -(1 << 53) - 1,
                    0x7FF0000000000000, 7, 7, 7], np.int64)


def random_grid(rng, R, T):
    vals = SPECIAL[rng.integers(0, len(SPECIAL), (R, T))]
    mix = rng.random((R, T)) < 0.3
    vals[mix] = rng.integers(-5, 5, int(mix.sum()))  # many ties
    ok = rng.random((R, T)) < 0.5
    return vals, ok


@pytest.mark.parametrize("R,T,G", [(1, 1, 1), (7, 33, 3), (40, 65, 5), (300, 32, 1)])
def test_group_aggregate_i64(ctx, R, T, G):
    rng = np.random.default_rng(R * 100 + T)
    vals, ok = random_grid(rng, R, T)
    gid = rng.integers(0, G, R).astype(np.uint32)
    for op in ("sum", "min", "max", "count", "avg", "stddev", "stdvar"):
        got, cnt = ctx.group_aggregate_i64(op, vals, _words(ok), gid, G)
        want, wcnt = io.group_aggregate(op, vals, ok, gid, G)
        assert (cnt == wcnt).all(), op
        for g in range(G):
            for k in range(T):
                if wcnt[g, k] == 0:
                    continue
                if op in ("sum", "min", "max"):
                    assert int(got[g, k]) == want[g][k], (op, g, k)
                else:
                    # the Float64 path over (double)i64: the same member order, so the same bits
                    assert np.float64(got[g, k]).tobytes() == np.float64(want[g][k]).tobytes(), (op, g, k)


def test_sum_wraps_on_the_device(ctx):
    vals = np.array([[io.INT64_MAX], [1], [io.INT64_MAX]], np.int64)
    got, _ = ctx.group_aggregate_i64("sum", vals, _words(np.ones((3, 1), bool)), np.zeros(3, np.uint32), 1)
    assert int(got[0, 0]) == io.wrap(2 * io.INT64_MAX + 1)


@pytest.mark.parametrize("R,T", [(1, 1), (5, 31), (64, 33), (500, 40)])
def test_sort_cells_i64(ctx, R, T):
    rng = np.random.default_rng(R + T)
    vals, ok = random_grid(rng, R, T)
    for desc in (False, True):
        assert ctx.sort_cells_i64(desc, vals, _words(ok)).tolist() == io.value_order(vals, ok, desc), desc


@pytest.mark.parametrize("R,T,G,kk", [(6, 5, 1, 1), (40, 33, 3, 2), (80, 9, 2, 40), (700, 3, 1, 5)])
def test_topk_i64(ctx, R, T, G, kk):
    rng = np.random.default_rng(R * 7 + kk)
    vals, ok = random_grid(rng, R, T)
    gid = rng.integers(0, G, R).astype(np.uint32)
    tie = rng.permutation(R).astype(np.uint32)
    for op in ("topk", "bottomk"):
        words = ctx.topk_i64(op, kk, vals, _words(ok), gid, G, tie)
        keep = io.topk_keep(op == "bottomk", kk, vals, ok, gid, G, tie)
        assert (words == _words(keep)).all(), op


@pytest.mark.parametrize("R,T,G", [(5, 3, 1), (60, 33, 4), (300, 7, 2)])
def test_count_values_i64(ctx, R, T, G):
    rng = np.random.default_rng(R * 3 + T)
    vals, ok = random_grid(rng, R, T)
    gid = rng.integers(0, G, R).astype(np.uint32)
    out, cnt = ctx.count_values_i64(vals, _words(ok), gid, G)
    want = io.count_values(vals, ok, gid, G)
    members = np.argsort(gid, kind="stable")
    first = {g: int(np.searchsorted(gid[members], g)) for g in range(G)}
    for (g, k), pairs in want.items():
        n = int((gid == g).sum())
        got = [(int(out[first[g] + j, k]), int(cnt[first[g] + j, k])) for j in range(n) if cnt[first[g] + j, k]]
        assert got == pairs, (g, k)


def test_i64_to_f64_rounds_to_nearest(ctx):
    vals = np.array([io.INT64_MIN, io.INT64_MAX, (1 << 53) + 1, -(1 << 53) - 3, NAN_BITS[0], 0, -7], np.int64)
    assert ctx.i64_to_f64(vals).tobytes() == vals.astype(np.float64).tobytes()


# ---- the instant leaf -------------------------------------------------------------------------------------------
def test_nan_pattern_int64_is_never_stale(ctx):
    rows = [(0, "a", "x", int(NAN_BITS[0])), (5000, "a", "x", int(NAN_BITS[1])), (0, "b", "x", (1 << 53) + 1)]
    out = leaf(ctx, rows).execute()
    assert out.schema.field("val").type == pa.int64()
    got = sorted(zip(out.column("host").to_pylist(), out.column("ts").cast(pa.int64()).to_pylist(),
                     out.column("val").to_pylist()))
    assert got == [("a", 0, int(NAN_BITS[0])), ("a", 5000, int(NAN_BITS[1])), ("a", 10000, int(NAN_BITS[1])),
                   ("a", 15000, int(NAN_BITS[1])), ("b", 0, (1 << 53) + 1), ("b", 5000, (1 << 53) + 1),
                   ("b", 10000, (1 << 53) + 1), ("b", 15000, (1 << 53) + 1)]


def test_mixed_float_and_int_fields(ctx):
    from greptimedb_b200.plan import PromRangeExec
    b = pa.record_batch([pa.array([0, 5000, 0], pa.timestamp("ms")), pa.array(["a", "a", "b"]),
                         pa.array([1.5, np.nan, 2.5]), pa.array([int(NAN_BITS[0]), 7, io.INT64_MIN], pa.int64())],
                        names=["ts", "host", "f", "i"])
    for fields, stale_at_5s in ((["f", "i"], True), (["i", "f"], False)):
        ex = PromRangeExec(ctx, "", 0, 5000, 5000, 0, "ts", fields, ["host"], lookback_delta=io.LOOKBACK)
        ex.push(b)
        out = ex.execute()
        assert out.schema.field("f").type == pa.float64() and out.schema.field("i").type == pa.int64()
        got = list(zip(out.column("host").to_pylist(), out.column("ts").cast(pa.int64()).to_pylist(),
                       out.column("i").to_pylist()))
        # field 0 Float64: its NaN at 5 s is stale, and the step keeps nothing; field 0 Int64: never stale
        a5 = ("a", 5000, 7)
        assert (a5 not in got) == stale_at_5s
        assert ("a", 0, int(NAN_BITS[0])) in got and ("b", 0, io.INT64_MIN) in got


def test_element_wise_and_scalar_give_float64(ctx):
    from greptimedb_b200.plan import ScalarPlan
    rows = GOLDEN["tables"]["sort"]["rows"]
    out = leaf(ctx, rows, lambda r: r[1] == "host1").scalar_op("+", 1.0).execute()
    assert out.schema.field(1).type == pa.float64()
    assert sorted(out.column(1).to_pylist()) == sorted(float(v) + 1 for v in [1, 1, 1, 1, 3, 3, 3, 5, 5, 7])
    s = ScalarPlan(ctx, leaf(ctx, rows, lambda r: r[1] == "host1" and r[2] == "idc1")).execute()
    assert s.schema.field(1).type == pa.float64() and s.column(1).to_pylist() == [1.0] * 4
    c = leaf(ctx, rows, lambda r: r[1] == "host1").function("clamp", 0.0, 4.0).execute()
    assert c.schema.field(1).type == pa.float64() and max(c.column(1).to_pylist()) == 4.0


def test_absent_and_and_keep_working(ctx):
    from greptimedb_b200.plan import AbsentPlan, SetOpPlan
    rows = GOLDEN["tables"]["sort"]["rows"]
    a = AbsentPlan(ctx, leaf(ctx, rows), 0, 15_000, 5_000, "ts", "value", []).execute()
    assert a.num_rows == 0
    both = SetOpPlan(ctx, "and", leaf(ctx, rows), leaf(ctx, rows, lambda r: r[1] == "host1")).execute()
    assert both.schema.field("val").type == pa.int64() and set(both.column("host").to_pylist()) == {"host1"}


# ---- the Int64 instant selector, the device forms, topk's general path, NULL slots ----------------------------------
@pytest.mark.parametrize("F", [1, 2])
def test_instant_select_fields_i64(ctx, F):
    rng = np.random.default_rng(17 + F)
    S, start, end, interval, lookback = 60, 10_000, 400_000, 7_000, 30_000
    lens = rng.integers(0, 40, S)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    ts = np.concatenate([np.cumsum(rng.integers(1, 25_000, n)) for n in lens]).astype(np.int64)
    vals = [SPECIAL[rng.integers(0, len(SPECIAL), ts.size)]]
    if F == 2:  # a Float64 second field with NaNs: moved bit for bit, never tested
        v = rng.standard_normal(ts.size)
        v[::3] = np.nan
        vals.append(v)
    outs, valid = ctx.instant_select_fields_i64(ts, vals, start, end, interval, lookback, offsets=offsets)
    want, ok = io.instant_select(ts, vals, offsets, start, end, interval, lookback)
    assert (valid == _words(ok)).all()
    assert (np.where(ok, outs, 0) == np.where(ok, want, 0)).all()
    # a NaN-pattern i64 in field 0 is selected, never treated as stale
    assert any(outs[0][ok] == NAN_BITS[0]) or not (vals[0] == NAN_BITS[0]).any()


def test_one_field_int64_null_slots_are_refused(ctx):
    from greptimedb_b200 import B2PError
    ts = np.array([0, 5000], np.int64)
    with pytest.raises(B2PError, match="Int64 field has NULL slots"):
        ctx.instant_select_fields_i64(ts, [np.array([1, 2], np.int64)], 0, 5000, 5000, io.LOOKBACK,
                                      offsets=np.array([0, 2], np.uint64), present=[np.array([True, False])])
    b = pa.record_batch([pa.array([0, 5000], pa.timestamp("ms")), pa.array(["a", "a"]), pa.array([1, None], pa.int64())],
                        names=["ts", "host", "val"])
    from greptimedb_b200.plan import PromRangeExec
    ex = PromRangeExec(ctx, "", 0, 5000, 5000, 0, "ts", "val", ["host"], lookback_delta=io.LOOKBACK)
    ex.push(b)
    with pytest.raises(B2PError, match="Int64 field has NULL slots"):
        ex.execute()


def test_device_forms(ctx):
    import torch
    rng = np.random.default_rng(23)
    R, T, G = 200, 45, 7
    vals, ok = random_grid(rng, R, T)
    words = _words(ok)
    d_vals = torch.from_numpy(vals).cuda()
    d_valid = torch.from_numpy(words.view(np.int32)).cuda()
    for desc in (False, True):
        cells = torch.full((R * T,), -1, dtype=torch.int64, device="cuda")
        n = torch.zeros(1, dtype=torch.int64, device="cuda")
        ctx.sort_cells_i64_dev(desc, d_vals, d_valid, R, T, cells, n)
        ctx.sync()
        assert cells[:int(n.item())].cpu().numpy().view(np.uint64).tolist() == io.value_order(vals, ok, desc)
    gid = rng.integers(0, G, R).astype(np.uint32)
    d_gid = torch.from_numpy(gid.view(np.int32)).cuda()
    out = torch.zeros(G * T, dtype=torch.int64, device="cuda")
    cnt = torch.zeros(G * T, dtype=torch.int32, device="cuda")
    ctx.group_aggregate_i64_dev("sum", d_vals, d_valid, d_gid, R, G, T, out, cnt)
    ctx.sync()
    want, wcnt = io.group_aggregate("sum", vals, ok, gid, G)
    got = out.cpu().numpy().reshape(G, T)
    assert (cnt.cpu().numpy().view(np.uint32).reshape(G, T) == wcnt).all()
    assert all(int(got[g, k]) == want[g][k] for g in range(G) for k in range(T) if wcnt[g, k])


@pytest.mark.parametrize("kk", [33, 40, 64])
def test_topk_i64_general_path(ctx, kk):
    """kk > 32 and below the group size: the rounds of 32 and topk_select_kernel<I64Key>"""
    rng = np.random.default_rng(kk)
    R, T = 150, 37
    vals, ok = random_grid(rng, R, T)
    gid = np.zeros(R, np.uint32)
    tie = rng.permutation(R).astype(np.uint32)
    for op in ("topk", "bottomk"):
        words = ctx.topk_i64(op, kk, vals, _words(ok), gid, 1, tie)
        assert (words == _words(io.topk_keep(op == "bottomk", kk, vals, ok, gid, 1, tie))).all(), op
