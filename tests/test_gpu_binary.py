"""GPU: the binary operators (K7 binary_op_kernel, count_valid_kernel) against the CPU oracle, the device-API
composition of anon_promql_ratio_repro, and the plan layer (scalar_op / BinaryPlan) on the sqlness goldens."""
import math
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import oracle as orc
from tests import binary_oracle as bor
from tests.binary_helpers import (LOOKBACK, count_rows, dense_rows, expected_rows, load_binary, oracle_node,
                                  sum_rate_table, table_arrays)
from tests.ulp_bounds import POW_ATAN2_ULPS   # pow / atan2 are CUDA's, not glibc's: DESIGN.md section 2

pytestmark = pytest.mark.gpu
G = load_binary()
CASES = {c["name"]: c for c in G["cases"]}
ARITH = ["+", "-", "*", "/", "%", "^", "atan2"]
CMP = ["==", "!=", ">", "<", ">=", "<="]


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.uint64)


# ±0, ±inf, NaN of both signs with payloads, subnormals, values that overflow or cancel, and ordinary numbers
VALS = np.concatenate([
    np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8000000000123, 0xFFF0000000000456, 0x8000000000000000,
              0x0000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 0x0000000000000001, 0x800FFFFFFFFFFFFF],
             np.uint64).view(np.float64),
    np.array([1.0, -1.0, 2.0, 3.0, 0.5, -2.5, 10.0, 1e308, -1.7e308, 1e-300, 7.25, -0.1, 1e-5, 123456.789, 2.0 ** 60]),
])
SPECIAL = {float(v) for v in VALS if not np.isfinite(v) or v in (0.0, 1.0, -1.0)}


def total_key(x):
    b = bits(x).view(np.int64)
    return b ^ ((b >> 63).view(np.uint64) >> np.uint64(1)).view(np.int64)


def grid(rng, rows, T, pattern):
    """values from VALS (every pair of them meets somewhere) and validity words of the given pattern"""
    vals = VALS[rng.integers(0, VALS.size, size=(rows, T))]
    Tw = (T + 31) // 32
    ok = np.zeros((rows, T), bool)
    if pattern == "all":
        ok[:] = True
    elif pattern == "holes":
        ok = rng.random((rows, T)) < 0.6
    elif pattern == "one":
        ok[:, T // 2] = True
    valid = np.zeros((rows, Tw), np.uint32)
    for k in range(T):
        valid[:, k // 32] |= ok[:, k].astype(np.uint32) << np.uint32(k % 32)
    return vals, valid


def check_cells(op, arith, got, gv, exp, ev):
    assert (gv == ev).all(), "validity differs from the oracle"
    T = got.shape[1]
    ok = np.zeros(got.shape, bool)
    for k in range(T):
        ok[:, k] = (ev[:, k // 32] >> np.uint32(k % 32)) & 1
    assert (bits(got[~ok]) == 0).all(), "an invalid cell does not hold 0.0"
    g, e = got[ok], exp[ok]
    if not arith:
        assert (bits(g) == bits(e)).all(), "comparison result differs from the oracle"
        return
    both_nan = np.isnan(g) & np.isnan(e)   # the sign / payload of a NaN that arithmetic produced is the hardware's
    assert (np.isnan(g) == np.isnan(e)).all(), f"{op}: NaN where the oracle has none (or the reverse)"
    g, e = g[~both_nan], e[~both_nan]
    if op in ("^", "atan2"):
        exact = ~np.isfinite(e) | (e == 0) | (np.abs(e) == 1.0)
        assert (bits(g[exact]) == bits(e[exact])).all(), f"{op}: a C99 Annex F special case differs from glibc"
        ulps = np.abs(total_key(g) - total_key(e))
        assert ulps.max(initial=0) <= POW_ATAN2_ULPS, f"{op}: {ulps.max()} ulps from glibc"
    else:
        assert (bits(g) == bits(e)).all(), f"{op} differs from the oracle"


OPS = [(op, False) for op in ARITH] + [(op, rb) for op in CMP for rb in (False, True)]


@pytest.mark.parametrize("form", ["vector", "scalar_left", "scalar_right"])
@pytest.mark.parametrize("op,return_bool", OPS)
def test_every_op_form_and_mode_matches_the_oracle(ctx, op, return_bool, form):
    rng = np.random.default_rng(zlib.crc32(f"{op} {return_bool} {form}".encode()))
    arith = op in ARITH
    for i, T in enumerate([1, 31, 32, 33, 200, 1000]):
        for pattern in ("all", "none", "holes", "one"):
            nl, nr = 5, 4
            lhs, lv = grid(rng, nl, T, pattern)
            rhs, rv = grid(rng, nr, T, "all" if pattern == "one" else "holes")   # holes on either side or both
            if form == "vector":
                P = [0, 1, 23][(i + len(pattern)) % 3]
                lrow = rng.integers(0, nl, P).astype(np.uint32)   # unsorted, rows repeat
                rrow = rng.integers(0, nr, P).astype(np.uint32)
                got, gv = ctx.binary_op(op, lhs, lv, lrow, rhs, rv, rrow, return_bool=return_bool)
                exp, ev = bor.binary_op(op, lhs, lv, lrow, rhs, rv, rrow, return_bool=return_bool)
            else:
                left = form == "scalar_left"
                for s in VALS[rng.integers(0, VALS.size, 3)]:
                    got, gv = ctx.scalar_op(op, s, lhs, lv, scalar_on_left=left, return_bool=return_bool)
                    exp, ev = bor.scalar_op(op, s, lhs, lv, scalar_on_left=left, return_bool=return_bool)
                    check_cells(op, arith, got, gv, exp, ev)
                continue
            check_cells(op, arith, got, gv, exp, ev)


def test_pow_and_atan2_special_cases_are_exact(ctx):
    """C99 Annex F: pow(x, ±0) = 1 for every x (NaN too), pow(1, y) = 1 for every y, pow(-1, ±inf) = 1; atan2 of zeros
    and infinities — every combination of the special values against glibc, bit for bit."""
    sp = np.array(sorted(SPECIAL, key=lambda v: (math.isnan(v), v)) + [-0.0, -1.0, 0.5, -2.0, 3.0], np.float64)
    lhs = np.repeat(sp, sp.size).reshape(1, -1)
    rhs = np.tile(sp, sp.size).reshape(1, -1)
    T = lhs.shape[1]
    v = np.full((1, (T + 31) // 32), 0xFFFFFFFF, np.uint32)
    edge = lambda x: ~np.isfinite(x) | (x == 0)
    for op in ("^", "atan2"):
        got, _ = ctx.binary_op(op, lhs, v, [0], rhs, v, [0])
        exp, _ = bor.binary_op(op, lhs, v, [0], rhs, v, [0])
        annex_f = edge(lhs[0]) | edge(rhs[0]) | (lhs[0] == 1.0) | edge(exp[0]) | (np.abs(exp[0]) == 1.0)
        nan = np.isnan(exp[0])
        assert (np.isnan(got[0]) == nan).all(), op
        ok = annex_f & ~nan
        assert (bits(got[0][ok]) == bits(exp[0][ok])).all(), (op, lhs[0][ok][bits(got[0][ok]) != bits(exp[0][ok])])
    assert ctx.binary_op("^", np.array([[math.nan, 5.0]]), v[:, :1], [0], np.array([[0.0, -0.0]]), v[:, :1], [0])[0].tolist() == [[1.0, 1.0]]
    assert ctx.binary_op("^", np.array([[1.0, -1.0]]), v[:, :1], [0], np.array([[math.nan, math.inf]]), v[:, :1], [0])[0].tolist() == [[1.0, 1.0]]


def test_total_order_comparisons_on_the_device(ctx):
    neg_nan = np.array([0xFFF8000000000000], np.uint64).view(np.float64)[0]
    lhs = np.array([[math.nan, math.nan, -0.0, -0.0, neg_nan]])
    rhs = np.array([[1.0, math.nan, 0.0, 0.0, -math.inf]])
    v = np.array([[0x1F]], np.uint32)
    _, gt = ctx.binary_op(">", lhs, v, [0], rhs, v, [0])
    _, eq = ctx.binary_op("==", lhs, v, [0], rhs, v, [0])
    _, lt = ctx.binary_op("<", lhs, v, [0], rhs, v, [0])
    assert gt[0, 0] == 0b00001 and eq[0, 0] == 0b00010 and lt[0, 0] == 0b11100


def test_unaligned_and_in_place_device_calls(ctx):
    """Even T with 8-byte-offset pointers takes the scalar path; the scalar form writes in place."""
    import torch
    rng = np.random.default_rng(7)
    T, n = 64, 6
    a, av = grid(rng, n, T, "holes")
    b, bv = grid(rng, n, T, "holes")
    dev = torch.device("cuda:0")
    buf = torch.zeros(2 * n * T + 2, dtype=torch.float64, device=dev)
    da = buf[1:1 + n * T]
    db = buf[1 + n * T:1 + 2 * n * T]
    da.copy_(torch.from_numpy(a.ravel()))
    db.copy_(torch.from_numpy(b.ravel()))
    dav, dbv = torch.from_numpy(av.view(np.int32)).to(dev), torch.from_numpy(bv.view(np.int32)).to(dev)
    rows = torch.arange(n, dtype=torch.int32, device=dev)
    out = torch.zeros(n * T + 1, dtype=torch.float64, device=dev)[1:]
    ov = torch.zeros(n * 2, dtype=torch.int32, device=dev)
    ctx.use_torch_stream()
    ctx.binary_op_dev("-", da, dav, rows, n, db, dbv, rows.flip(0), n, n, T, out, ov)
    ctx.sync()
    exp, ev = bor.binary_op("-", a, av, np.arange(n), b, bv, np.arange(n)[::-1])
    check_cells("-", True, out.cpu().numpy().reshape(n, T), ov.cpu().numpy().view(np.uint32).reshape(n, 2), exp, ev)
    ctx.scalar_op_dev("-", 3.0, da, dav, n, T, da, dav, scalar_on_left=True)   # 3 - x, in place
    ctx.sync()
    exp, ev = bor.scalar_op("-", 3.0, a, av, scalar_on_left=True)
    check_cells("-", True, da.cpu().numpy().reshape(n, T), dav.cpu().numpy().view(np.uint32).reshape(n, 2), exp, ev)
    ctx.use_own_stream()


def test_bad_arguments_return_invalid_without_a_fault(ctx):
    import torch
    from greptimedb_b200 import B2PError
    a = np.ones((2, 40))
    v = np.full((2, 2), 0xFFFFFFFF, np.uint32)
    for op, rb in ((13, False), (-1, False), ("+", True), ("atan2", True)):
        with pytest.raises(B2PError) as ei:
            ctx.binary_op(op, a, v, [0], a, v, [1], return_bool=rb)
        assert ei.value.code == -1
        with pytest.raises(B2PError) as ei:
            ctx.scalar_op(op, 1.0, a, v, return_bool=rb)
        assert ei.value.code == -1
    with pytest.raises(B2PError) as ei:   # rhs row 2 of 2 rows: found on the device, that pair written invalid
        ctx.binary_op("+", a, v, [0, 1], a, v, [1, 2])
    assert ei.value.code == -1
    dev = torch.device("cuda:0")
    da, dv = torch.ones(80, dtype=torch.float64, device=dev), torch.full((4,), -1, dtype=torch.int32, device=dev)
    out, ov = torch.full((80,), 7.0, dtype=torch.float64, device=dev), torch.full((4,), -1, dtype=torch.int32, device=dev)
    lrow = torch.tensor([5, 0], dtype=torch.int32, device=dev)
    rrow = torch.tensor([0, 1], dtype=torch.int32, device=dev)
    ctx.use_torch_stream()
    ctx.binary_op_dev("*", da, dv, lrow, 2, da, dv, rrow, 2, 2, 40, out, ov)
    with pytest.raises(B2PError) as ei:
        ctx.sync()
    assert ei.value.code == -1
    torch.cuda.synchronize()
    assert (out[:40] == 0).all() and (ov[:2] == 0).all() and (out[40:] == 1).all()
    ctx.binary_op_dev("*", da, dv, rrow, 2, da, dv, rrow, 2, 2, 40, out, ov)   # the context is still usable
    ctx.sync()
    assert (out == 1).all()
    ctx.use_own_stream()
    assert ctx.binary_op("+", a, v, [1, 0], a, v, [0, 1])[0].tolist() == (2 * a).tolist()


# ---- composition through the device API: anon_promql_ratio_repro end to end ----------------------------------------------
def test_ratio_repro_through_the_device_api(ctx):
    """rate(metric_a[3m]) / on(l3,l4) group_left metric_b > 0.5, counted (K3), the count turned into validity, divided
    by count(rate(..)) and * 100: 1, 1.5 and 33.33333333333333 as printed (anon_promql_ratio_repro.result:60,78,87)."""
    import torch
    from greptimedb_b200 import make_params
    dev = torch.device("cuda:0")
    c = CASES["ratio_filtered_count"]
    start, end, step, rng_ms = c["start"], c["end"], c["interval"], c["range"]
    T = orc.num_steps(start, end, step)
    Tw = (T + 31) // 32
    ctx.use_torch_stream()

    def upload(table):
        labels, ts, val, offsets = table_arrays(G["tables"][table])
        return labels, torch.from_numpy(ts).to(dev), torch.from_numpy(val).to(dev), torch.from_numpy(offsets.view(np.int64)).to(dev), ts.size

    la, ts_a, val_a, off_a, n_a = upload("metric_a")
    lb, ts_b, val_b, off_b, n_b = upload("metric_b")
    Sa, Sb = len(la), len(lb)
    rate = torch.zeros(Sa * T, dtype=torch.float64, device=dev)
    rate_v = torch.zeros(Sa * Tw, dtype=torch.int32, device=dev)
    ctx.range_eval_dev(make_params("rate", start, end, step, rng_ms), ts_a, val_a, off_a, n_a, Sa, rate, rate_v)
    inst = torch.zeros(Sb * T, dtype=torch.float64, device=dev)
    inst_v = torch.zeros(Sb * Tw, dtype=torch.int32, device=dev)
    ctx.instant_select_dev(start, end, step, LOOKBACK, 0, ts_b, val_b, off_b, n_b, Sb, inst, inst_v)
    # on(l3, l4): the host match of the plan layer (tags l1..l5 / l6, l1..l4)
    lrow, rrow = bor.binary_pairs(["l1", "l2", "l3", "l4", "l5"], la, ["l6", "l1", "l2", "l3", "l4"], lb, on=["l3", "l4"])
    P = lrow.size
    ratio = torch.zeros(P * T, dtype=torch.float64, device=dev)
    ratio_v = torch.zeros(P * Tw, dtype=torch.int32, device=dev)
    ctx.binary_op_dev("/", rate, rate_v, torch.from_numpy(lrow.view(np.int32)).to(dev), Sa, inst, inst_v,
                      torch.from_numpy(rrow.view(np.int32)).to(dev), Sb, P, T, ratio, ratio_v)
    ctx.scalar_op_dev(">", 0.50, ratio, ratio_v, P, T, ratio, ratio_v)   # the filter, in place: K3 reads it as it is

    def count(vals, valid, n):
        out = torch.zeros(T, dtype=torch.float64, device=dev)
        cnt = torch.zeros(T, dtype=torch.int32, device=dev)
        ctx.group_aggregate_dev("count", vals, valid, torch.zeros(n, dtype=torch.int32, device=dev), n, 1, T, out, cnt)
        words = torch.zeros(Tw, dtype=torch.int32, device=dev)
        ctx.count_valid_words_dev(cnt, 1, T, words)
        return out, words

    c_kept, w_kept = count(ratio, ratio_v, P)
    c_all, w_all = count(rate, rate_v, Sa)
    half = torch.zeros(T, dtype=torch.float64, device=dev)
    half_v = torch.zeros(Tw, dtype=torch.int32, device=dev)
    ctx.scalar_op_dev("/", 2.0, c_all, w_all, 1, T, half, half_v)
    pct = torch.zeros(T, dtype=torch.float64, device=dev)
    pct_v = torch.zeros(Tw, dtype=torch.int32, device=dev)
    zero = torch.zeros(1, dtype=torch.int32, device=dev)
    ctx.binary_op_dev("/", c_kept, w_kept, zero, 1, c_all, w_all, zero, 1, 1, T, pct, pct_v)
    ctx.scalar_op_dev("*", 100.0, pct, pct_v, 1, T, pct, pct_v)
    ctx.sync()
    torch.cuda.synchronize()
    ctx.use_own_stream()
    eval_ts = start + step * np.arange(T)

    def rows(v, w):
        return dense_rows([], [()], v.cpu().numpy().reshape(1, T), w.cpu().numpy().view(np.uint32).reshape(1, Tw), eval_ts)[1]

    assert rows(c_kept, w_kept) == expected_rows(CASES["ratio_filtered_count"], [])
    assert rows(half, half_v) == expected_rows(CASES["ratio_count_div_2"], [])
    assert rows(pct, pct_v) == expected_rows(CASES["ratio_times_100"], [])


# ---- plan layer -----------------------------------------------------------------------------------------------------------
def table_batch(table, id_column=None):
    """One sorted RecordBatch of a golden table; with id_column, the tags are replaced by one UInt64 id per series."""
    labels, ts, val, offsets = table_arrays(table)
    n = np.diff(offsets.astype(np.int64))
    cols = [pa.array(ts, pa.timestamp("ms")), pa.array(val, pa.float64())]
    names = [table["time_index"], table["field"]]
    if id_column:
        cols.append(pa.array(np.repeat(np.arange(len(labels), dtype=np.uint64) + 1000, n), pa.uint64()))
        names.append(id_column)
    else:
        for i, t in enumerate(table["tags"]):
            cols.append(pa.array(np.repeat(np.array([lab[i] for lab in labels], dtype=object), n).tolist(), pa.string()))
            names.append(t)
    return pa.record_batch(cols, names=names)


def node(ctx, table, case, fn=None, range_ms=None, aggregate=None, by=(), id_column=None):
    from greptimedb_b200.plan import PromRangeExec
    tags = [id_column] if id_column else table["tags"]
    ex = PromRangeExec(ctx, "prom_" + fn if fn else "", case["start"], case["end"], case["interval"], range_ms or 0,
                       table["time_index"], table["field"], tags, aggregate=aggregate, by_columns=by,
                       lookback_delta=None if fn else LOOKBACK)
    ex.push(table_batch(table, id_column))
    return ex


def batch_rows(b, tags):
    """-> sorted [(labels in `tags` order..., ts, value)]; the value is the float64 column, the time index the timestamp."""
    names = b.schema.names
    vi = next(i for i, f in enumerate(b.schema) if pa.types.is_float64(f.type))
    ti = next(i for i, f in enumerate(b.schema) if pa.types.is_timestamp(f.type))
    ts = b.column(ti).cast(pa.int64()).to_pylist()
    vals = b.column(vi).to_pylist()
    lab = [b.column(names.index(t)).to_pylist() for t in tags]
    return sorted(tuple(col[r] for col in lab) + (ts[r], vals[r]) for r in range(b.num_rows))


def same_rows(got, exp, rel=1e-12):
    """labels and timestamps exact; values within `rel` (the range functions are the oracle's to within ulps)"""
    key = lambda r: (tuple(str(x) for x in r[:-1]), -math.inf if math.isnan(r[-1]) else r[-1])
    got, exp = sorted(got, key=key), sorted(exp, key=key)
    assert len(got) == len(exp) and [r[:-1] for r in got] == [r[:-1] for r in exp]
    for x, y in zip(got, exp):
        assert (math.isnan(x[-1]) and math.isnan(y[-1])) or abs(x[-1] - y[-1]) <= rel * abs(y[-1]), (x, y)


def tag_names(b):
    return [f.name for f in b.schema if not (pa.types.is_float64(f.type) or pa.types.is_timestamp(f.type))]


def test_scalar_goldens_through_the_plan(ctx):
    c = CASES["sum_rate_times_100"]
    ex = node(ctx, sum_rate_table(), c, fn="rate", range_ms=60000, aggregate="sum").scalar_op("*", 100)
    out = ex.execute()
    assert out.schema.names == ["ts", "sum(prom_rate) * Float64(100)"]
    assert batch_rows(out, []) == expected_rows(c, [])
    c = CASES["sum_by_host_rate_times_60"]
    out = node(ctx, sum_rate_table(), c, fn="rate", range_ms=60000, aggregate="sum", by=("host",)).scalar_op("*", 60).execute()
    assert tag_names(out) == ["host"] and batch_rows(out, ["host"]) == expected_rows(c, ["host"])
    c = CASES["ratio_count_div_2"]
    out = node(ctx, G["tables"]["metric_a"], c, fn="rate", range_ms=c["range"], aggregate="count").scalar_op("/", 2).execute()
    assert batch_rows(out, []) == expected_rows(c, [])
    # chained: sum(rate) * 100 > 50 keeps nothing, >= 50 keeps every row with the value 50; 100 - x with x on the right
    ex = node(ctx, sum_rate_table(), CASES["sum_rate_times_100"], fn="rate", range_ms=60000, aggregate="sum")
    assert ex.scalar_op("*", 100).scalar_op(">", 50).execute().num_rows == 0
    ex = node(ctx, sum_rate_table(), CASES["sum_rate_times_100"], fn="rate", range_ms=60000, aggregate="sum")
    assert [r[-1] for r in batch_rows(ex.scalar_op("*", 100).scalar_op(">=", 50).execute(), [])] == [50.0] * 3
    ex = node(ctx, sum_rate_table(), CASES["sum_rate_times_100"], fn="rate", range_ms=60000, aggregate="sum")
    assert [r[-1] for r in batch_rows(ex.scalar_op("-", 100, scalar_on_left=True).execute(), [])] == [99.5] * 3
    ex = node(ctx, sum_rate_table(), CASES["sum_rate_times_100"], fn="rate", range_ms=60000, aggregate="sum")
    assert [r[-1] for r in batch_rows(ex.scalar_op(">", 0.25, return_bool=True).execute(), [])] == [1.0] * 3


@pytest.mark.parametrize("name,fn", [("selector_plus_selector_two_tables", None),
                                     ("avg_over_time_plus_avg_over_time_two_tables", "avg_over_time")])
def test_vector_goldens_through_the_plan(ctx, name, fn):
    from greptimedb_b200.plan import BinaryPlan
    c = CASES[name]
    lhs = node(ctx, G["tables"]["host_sec"], c, fn=fn, range_ms=c.get("range"))
    rhs = node(ctx, G["tables"]["host_micro"], c, fn=fn, range_ms=c.get("range"))
    out = BinaryPlan(ctx, "+", lhs, rhs, label_side="rhs").execute()
    assert tag_names(out) == ["host"] and batch_rows(out, ["host"]) == expected_rows(c, ["host"])


@pytest.mark.parametrize("id_keyed", [False, True])
def test_tsid_golden_through_the_plan(ctx, id_keyed):
    from greptimedb_b200.plan import BinaryPlan
    c = CASES["tsid_div"]
    idc = "__tsid" if id_keyed else None
    lhs = node(ctx, G["tables"]["tsid_binary_join_left"], c, id_column=idc)
    rhs = node(ctx, G["tables"]["tsid_binary_join_right"], c, id_column=idc)
    out = BinaryPlan(ctx, "/", lhs, rhs).execute()
    if id_keyed:   # ids 1000 (host1/job1) and 1001 (host2/job2) on both sides
        assert tag_names(out) == ["__tsid"]
        got = batch_rows(out, ["__tsid"])
        assert [r[1:] for r in got] == [r[2:] for r in expected_rows(c, ["host", "job"])]
        assert [r[0] for r in got] == [1000, 1000, 1001, 1001]
    else:
        assert batch_rows(out, ["host", "job"]) == expected_rows(c, ["host", "job"])


def test_ratio_repro_through_the_plan(ctx):
    """(rate(metric_a[3m]) / on(l3,l4) group_left metric_b) > 0.50: one kept row at 180 s, as count() prints."""
    from greptimedb_b200.plan import BinaryPlan
    c = CASES["ratio_filtered_count"]
    a = node(ctx, G["tables"]["metric_a"], c, fn="rate", range_ms=c["range"])
    b = node(ctx, G["tables"]["metric_b"], c)
    ratio = BinaryPlan(ctx, "/", a, b, on=["l3", "l4"], label_side="rhs")
    kept = ratio.scalar_op(">", 0.50).execute()
    assert count_rows(batch_rows(kept, [])) == expected_rows(c, [])
    # the same rows from the oracle's row-literal join
    ra = dense_rows(*oracle_node(G["tables"]["metric_a"], c["start"], c["end"], c["interval"], fn="rate", range_ms=c["range"]))
    rb = dense_rows(*oracle_node(G["tables"]["metric_b"], c["start"], c["end"], c["interval"]))
    tags, exp = bor.binary_rows(ra, rb, "/", on=["l3", "l4"], label_side="rhs")
    same_rows(batch_rows(kept, tags), sorted(bor.scalar_rows(exp, ">", 0.5)))


def _plan_vs_oracle(ctx, op, lhs_spec, rhs_spec, label_side="rhs", return_bool=False, **match):
    from greptimedb_b200.plan import BinaryPlan
    c = CASES["ratio_filtered_count"]
    kw = dict(start=c["start"], end=c["end"], interval=c["interval"])

    def make(spec):
        table, fn, agg, by = spec
        n = node(ctx, G["tables"][table], c, fn=fn, range_ms=c["range"] if fn else None, aggregate=agg, by=by)
        rows = dense_rows(*oracle_node(G["tables"][table], kw["start"], kw["end"], kw["interval"], fn=fn,
                                       range_ms=c["range"] if fn else None, agg=agg, by=by))
        return n, rows

    (ln, lr), (rn, rr) = make(lhs_spec), make(rhs_spec)
    out = BinaryPlan(ctx, op, ln, rn, return_bool=return_bool, label_side=label_side, **match).execute()
    tags, exp = bor.binary_rows(lr, rr, op, return_bool=return_bool, label_side=label_side, **match)
    assert sorted(tag_names(out)) == sorted(tags)
    same_rows(batch_rows(out, tags), exp)
    return out, tags


def test_label_side_rule_both_ways(ctx):
    """sum by (l4)(rate(a)) / sum(rate(a)): the rhs has no tags, so every row pairs with the one total row; the output
    keeps l4 when the caller names the lhs (one table) and has no labels when it names the rhs (two tables)."""
    spec_l, spec_r = ("metric_a", "rate", "sum", ("l4",)), ("metric_a", "rate", "sum", ())
    _, tags = _plan_vs_oracle(ctx, "/", spec_l, spec_r, label_side="lhs")
    assert tags == ["l4"]
    out, tags = _plan_vs_oracle(ctx, "/", spec_l, spec_r, label_side="rhs")
    assert tags == [] and out.num_rows == 2


def test_on_ignoring_and_one_to_many(ctx):
    a, b = ("metric_a", "rate", None, ()), ("metric_b", None, None, ())
    out, _ = _plan_vs_oracle(ctx, "/", a, b, on=["l3", "l4"])        # v5a and v5b both pair with one metric_b series
    assert out.num_rows == 3
    _plan_vs_oracle(ctx, "-", a, b, ignoring=["l6", "l5"])
    _plan_vs_oracle(ctx, "<", a, b, return_bool=True, on=["l3"])
    _plan_vs_oracle(ctx, "!=", b, a, on=["l4"])                         # a filter keeps the lhs rows and labels
    _plan_vs_oracle(ctx, "*", a, ("metric_a", "rate", "count", ()), label_side="lhs")   # rhs without tags: all pairs


def test_binary_node_as_child_and_missing_key_column(ctx):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import BinaryPlan
    c = CASES["ratio_filtered_count"]
    a = node(ctx, G["tables"]["metric_a"], c, fn="rate", range_ms=c["range"])
    b = node(ctx, G["tables"]["metric_b"], c)
    inner = BinaryPlan(ctx, "/", a, b, on=["l3", "l4"], label_side="lhs")
    outer = BinaryPlan(ctx, "*", inner, b, on=["l3", "l4"], label_side="lhs").scalar_op("atan2", 1.0)
    got = batch_rows(outer.execute(), ["l5"])
    ra = dense_rows(*oracle_node(G["tables"]["metric_a"], c["start"], c["end"], c["interval"], fn="rate", range_ms=c["range"]))
    rb = dense_rows(*oracle_node(G["tables"]["metric_b"], c["start"], c["end"], c["interval"]))
    t1 = bor.binary_rows(ra, rb, "/", on=["l3", "l4"], label_side="lhs")
    t2 = bor.binary_rows(t1, rb, "*", on=["l3", "l4"], label_side="lhs")
    exp = sorted(bor.scalar_rows([(r[4],) + r[-2:] for r in t2[1]], "atan2", 1.0))
    same_rows(got, exp)
    # metric_b's key column l6 is not a tag of metric_a: the reference fails to plan this join
    bad = BinaryPlan(ctx, "+", node(ctx, G["tables"]["metric_a"], c, fn="rate", range_ms=c["range"]), b)
    with pytest.raises(B2PError) as ei:
        bad.execute()
    assert ei.value.code == -1 and "l6" in str(ei.value)
    with pytest.raises(B2PError):
        BinaryPlan(ctx, "+", a, b, return_bool=True)
    with pytest.raises(B2PError):
        BinaryPlan(ctx, "+", a, b, label_side="both")
