"""GPU: the set operators (K8 in b2p_setop.cuh) against the dense oracle bit for bit, the device-API compositions of the
vector(1) and count(...) goldens, and the plan layer (SetOpPlan) on the sqlness goldens."""
import zlib

import numpy as np
import pyarrow as pa
import pytest

from tests import binary_oracle as bor
from tests import set_oracle as sor
from tests.binary_helpers import LOOKBACK, dense_rows, oracle_node, table_arrays
from tests.set_helpers import CASES, EXPRS, G, MAX_RATIO, expected_set_rows, oracle_rows, row_key, select

pytestmark = pytest.mark.gpu
OPS = ["and", "or", "unless"]


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.uint64)


# NaN payloads of both signs, ±0, ±inf and ordinary numbers: a kept cell must be a bit copy
VALS = np.concatenate([
    np.array([0x7FF8000000000001, 0xFFF800000000BEEF, 0x7FF4000000000000, 0x8000000000000000, 0x7FF0000000000000,
              0x0000000000000001], np.uint64).view(np.float64),
    np.array([0.0, 1.0, -2.5, 1e300]),
])


def grid(rng, rows, T, p=0.6):
    vals = VALS[rng.integers(0, VALS.size, size=(rows, T))]
    ok = rng.random((rows, T)) < p
    return vals, bor._words(ok)   # the values of invalid cells are left in place: the kernel must not copy them


def check(got, gv, exp, ev):
    assert got.shape == exp.shape and (gv == ev).all(), "validity differs from the oracle"
    assert (bits(got) == bits(exp)).all(), "a value differs from the oracle (kept cells are bit copies, others 0.0)"


def keys_for(rng, n_rows, n_keys, no_key_rate=0.1, big_group=0):
    k = rng.integers(0, max(n_keys, 1), n_rows).astype(np.uint32)
    if big_group:
        k[:big_group] = 0
    k[rng.random(n_rows) < no_key_rate] = sor.NO_KEY
    if n_keys == 0:
        k[:] = sor.NO_KEY
    return k


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("T", [1, 31, 32, 33, 64, 65, 200, 1000])
def test_device_api_matches_the_dense_oracle(ctx, op, T):
    rng = np.random.default_rng(zlib.crc32(f"{op} {T}".encode()))
    shapes = [(7, 9, 4), (0, 5, 3), (6, 0, 3), (8, 8, 0), (40, 60, 1), (300, 200, 37)]
    if T <= 65:
        shapes.append((500, 5000, 3))   # a key group of about 5 000 rhs rows (and `or` lhs rows)
    for nl, nr, n_keys in shapes:
        lhs, lv = grid(rng, nl, T)
        rhs, rv = grid(rng, nr, T)
        lk = keys_for(rng, nl, n_keys, big_group=nl // 2)
        rk = keys_for(rng, nr, n_keys, big_group=nr * 4 // 5)
        got, gv = ctx.setop(op, lhs, lv, lk, rhs, rv, rk, n_keys)
        exp, ev = sor.setop(op, lhs, lv, lk, rhs, rv, rk, n_keys)
        check(got, gv, exp, ev)


def test_or_keeps_the_first_rhs_row_per_key_and_step(ctx):
    """rhs rows of one key: each step goes to the first row (in row order) that has it, unless the lhs has it."""
    T = 40
    ok = np.zeros((4, T), bool)
    ok[0, [1, 2]] = True            # lhs, key 0
    ok[1, [2, 3, 35]] = True        # rhs row 0, key 0: 2 is the lhs's
    ok[2, [3, 4, 35, 39]] = True    # rhs row 1, key 0: 3 and 35 are row 0's
    ok[3, [1, 3]] = True            # rhs row 2, key 1: nobody else has key 1
    vals = np.arange(4 * T, dtype=np.float64).reshape(4, T)
    words = bor._words(ok)
    got, gv = ctx.setop("or", vals[:1], words[:1], [0], vals[1:], words[1:], [0, 0, 1], 2)
    steps = [np.flatnonzero(bor._bits(gv[r:r + 1], T)[0]).tolist() for r in range(4)]
    assert steps == [[1, 2], [3, 35], [4, 39], [1, 3]]


def test_in_place_and_unaligned_device_calls(ctx):
    """and / unless written over the lhs (128-bit path: T even and aligned), and an 8-byte-offset lhs (scalar path)."""
    import torch
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(11)
    T, nl, nr, n_keys = 64, 50, 70, 9
    Tw = T // 32
    ctx.use_torch_stream()
    for op in ("and", "unless"):
        for offset in (0, 1):
            lhs, lv = grid(rng, nl, T)
            rhs, rv = grid(rng, nr, T)
            lk, rk = keys_for(rng, nl, n_keys), keys_for(rng, nr, n_keys)
            exp, ev = sor.setop(op, lhs, lv, lk, rhs, rv, rk, n_keys)
            buf = torch.zeros(nl * T + 1, dtype=torch.float64, device=dev)
            dl = buf[offset:offset + nl * T]
            dl.copy_(torch.from_numpy(lhs.ravel()))
            dlv = torch.from_numpy(lv.view(np.int32).ravel()).to(dev)
            up = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int32).ravel()).to(dev)
            ctx.setop_dev(op, dl, dlv, up(lk), nl, None, up(rv), up(rk), nr, n_keys, T, dl, dlv)
            ctx.sync()
            torch.cuda.synchronize()
            check(dl.cpu().numpy().reshape(nl, T), dlv.cpu().numpy().view(np.uint32).reshape(nl, Tw), exp, ev)
    ctx.use_own_stream()


def test_a_bad_key_is_reported_and_its_row_written_invalid(ctx):
    from greptimedb_b200 import B2PError
    rng = np.random.default_rng(5)
    T = 33
    lhs, lv = grid(rng, 4, T, p=1.0)
    rhs, rv = grid(rng, 3, T, p=1.0)
    for op in OPS:
        with pytest.raises(B2PError) as ei:
            ctx.setop(op, lhs, lv, [0, 7, 1, sor.NO_KEY], rhs, rv, [0, 1, 1], 2)
        assert ei.value.code == -1 and "n_keys" in str(ei.value)
    with pytest.raises(B2PError):   # an rhs key out of range is reported too
        ctx.setop("and", lhs, lv, [0, 1, 1, 0], rhs, rv, [0, 2, 1], 2)
    with pytest.raises(B2PError):   # unknown operator
        ctx.setop(3, lhs, lv, [0, 1, 1, 0], rhs, rv, [0, 1, 1], 2)
    # through the device API: the row with key 7 is invalid, every other row is what the oracle computes
    import torch
    dev = torch.device("cuda:0")
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    lk = np.array([0, 7, 1, sor.NO_KEY], np.uint32)
    rk = np.array([0, 1, 1], np.uint32)
    out = torch.full((7 * T,), 9.0, dtype=torch.float64, device=dev)
    ov = torch.full((7 * 2,), -1, dtype=torch.int32, device=dev)
    ctx.use_torch_stream()
    ctx.setop_dev("or", up(lhs), up(lv.view(np.int32)), up(lk.view(np.int32)), 4, up(rhs), up(rv.view(np.int32)),
                  up(rk.view(np.int32)), 3, 2, T, out, ov)
    with pytest.raises(B2PError) as ei:
        ctx.sync()
    assert ei.value.code == -1
    torch.cuda.synchronize()
    ctx.use_own_stream()
    got, gv = out.cpu().numpy().reshape(7, T), ov.cpu().numpy().view(np.uint32).reshape(7, 2)
    assert (gv[1] == 0).all() and (bits(got[1]) == 0).all()
    lk_ok = lk.copy()
    lk_ok[1] = sor.NO_KEY
    exp, ev = sor.setop("or", lhs, lv, lk_ok, rhs, rv, rk, 2)
    keep = [0, 2, 3, 4, 5, 6]
    check(got[keep], gv[keep], exp[keep], ev[keep])
    assert ctx.setop("and", lhs, lv, [0, 1, 1, 0], rhs, rv, [0, 1, 1], 2)[1].shape == (4, 2)   # still usable


# ---- the device API composed: vector(1) and count(...) ------------------------------------------------------------------
def oracle_grid(table, case, agg=None, by=()):
    tags, labels, out, valid, eval_ts = oracle_node(table, case["start"], case["end"], case["interval"], agg=agg, by=by)
    return tags, labels, out, valid, eval_ts


@pytest.mark.parametrize("name,kw", [("and_on_dummy_vector1", {"on": ["dummy"]}),
                                     ("and_ignoring_all_vector1", {"ignoring": ["g", "instance", "job"]})])
def test_vector1_goldens_through_the_device_api(ctx, name, kw):
    case = CASES[name]
    tags, labels, out, valid, eval_ts = oracle_grid(G["tables"]["http_requests"], case)
    T = eval_ts.size
    one, one_v = np.ones((1, T)), bor._words(np.ones((1, T), bool))   # vector(1): no tags, a value at every step
    lk, rk, n_keys, _ = sor.setop_pairs("and", tags, labels, [], [()], **kw)
    got, gv = ctx.setop("and", out, valid, lk, one, one_v, rk, n_keys)
    rows = dense_rows(tags, labels, got, gv, eval_ts)[1]
    assert sorted(rows, key=row_key) == expected_set_rows(case, tags)


@pytest.mark.parametrize("name,op", [("count_and", "and"), ("count_unless", "unless")])
def test_count_goldens_through_the_device_api(ctx, name, op):
    """count(max by (namespace)(used) and / unless (max / max >= 0.8)): the set output feeds the by-label aggregate
    (K3) and its counts become validity words, all on the device."""
    import torch
    dev = torch.device("cuda:0")
    case = CASES[name]
    ltags, llab, lval, lvalid, eval_ts = oracle_grid(G["tables"]["stats_used_bytes"], case, agg="max", by=("namespace",))
    rtags, rrows = oracle_rows(MAX_RATIO, case)
    rlab = sorted({r[:-2] for r in rrows})
    T, Tw = eval_ts.size, (eval_ts.size + 31) // 32
    rok = np.zeros((len(rlab), T), bool)
    for r in rrows:
        rok[rlab.index(r[:-2]), list(eval_ts).index(r[-2])] = True
    rvalid = bor._words(rok)
    lk, rk, n_keys, _ = sor.setop_pairs(op, ltags, llab, rtags, rlab)
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    L = len(llab)
    d_l, d_lv = up(lval), up(lvalid.view(np.int32))
    ctx.use_torch_stream()
    ctx.setop_dev(op, d_l, d_lv, up(lk.view(np.int32)), L, None, up(rvalid.view(np.int32)), up(rk.view(np.int32)),
                  len(rlab), n_keys, T, d_l, d_lv)
    cnt_val = torch.zeros(T, dtype=torch.float64, device=dev)
    cnt = torch.zeros(T, dtype=torch.int32, device=dev)
    ctx.group_aggregate_dev("count", d_l, d_lv, torch.zeros(L, dtype=torch.int32, device=dev), L, 1, T, cnt_val, cnt)
    words = torch.zeros(Tw, dtype=torch.int32, device=dev)
    ctx.count_valid_words_dev(cnt, 1, T, words)
    ctx.sync()
    torch.cuda.synchronize()
    ctx.use_own_stream()
    rows = dense_rows([], [()], cnt_val.cpu().numpy().reshape(1, T), words.cpu().numpy().view(np.uint32).reshape(1, Tw),
                      eval_ts)[1]
    assert rows == expected_set_rows(case, [])


# ---- plan layer ---------------------------------------------------------------------------------------------------------
def table_batch(table):
    labels, ts, val, offsets = table_arrays(table)
    n = np.diff(offsets.astype(np.int64))
    cols = [pa.array(ts, pa.timestamp("ms")), pa.array(val, pa.float64())]
    names = [table["time_index"], table["field"]]
    for i, t in enumerate(table["tags"]):
        cols.append(pa.array(np.repeat(np.array([lab[i] for lab in labels], dtype=object), n).tolist(), pa.string()))
        names.append(t)
    return pa.record_batch(cols, names=names)


def plan_node(ctx, expr, case):
    from greptimedb_b200.plan import BinaryPlan, PromRangeExec, SetOpPlan
    kind = expr[0]
    if kind == "sel":
        _, table, match, agg, by = expr
        t = select(G["tables"][table], match)
        ex = PromRangeExec(ctx, "", case["start"], case["end"], case["interval"], 0, t["time_index"], t["field"],
                           t["tags"], aggregate=agg, by_columns=by, lookback_delta=LOOKBACK)
        if t["series"]:
            ex.push(table_batch(t))
        return ex
    if kind == "scalar":
        return plan_node(ctx, expr[1], case).scalar_op(expr[2], expr[3])
    lhs, rhs = plan_node(ctx, expr[2], case), plan_node(ctx, expr[3], case)
    if kind == "bin":
        return BinaryPlan(ctx, expr[1], lhs, rhs, **expr[4])
    return SetOpPlan(ctx, expr[1], lhs, rhs, **expr[4])


def batch_rows(b, tags):
    names = b.schema.names
    vi = next(i for i, f in enumerate(b.schema) if pa.types.is_float64(f.type))
    ti = next(i for i, f in enumerate(b.schema) if pa.types.is_timestamp(f.type))
    ts = b.column(ti).cast(pa.int64()).to_pylist()
    vals = b.column(vi).to_pylist()
    lab = [b.column(names.index(t)).to_pylist() for t in tags]
    return sorted((tuple(col[r] for col in lab) + (ts[r], vals[r]) for r in range(b.num_rows)), key=row_key)


PLAN_CASES = sorted(c["name"] for c in G["cases"] if "plan" in c["layers"])


@pytest.mark.parametrize("name", PLAN_CASES)
def test_plan_goldens(ctx, name):
    case = CASES[name]
    out = plan_node(ctx, EXPRS[name], case).execute()
    tags, _ = oracle_rows(EXPRS[name], case)
    assert sorted(n for n in out.schema.names if n in tags) == sorted(tags)
    assert batch_rows(out, tags) == expected_set_rows(case, tags)
    if EXPRS[name][:2] == ("set", "or") and "columns" in case:
        assert out.schema.names == case["columns"]


def test_or_schema_and_real_nulls(ctx):
    case = CASES["t1_or_t2"]
    out = plan_node(ctx, EXPRS["t1_or_t2"], case).execute()
    assert out.schema.names == ["ts", "greptime_value", "job"]
    job = out.column(2)
    assert job.null_count == 6 and job.is_null().to_pylist() == [False] * 3 + [True] * 6
    # a NULL label of an existing node's output is a real null too (it used to be the 5-byte string "\0null")
    c = CASES["null_label_div"]
    out = plan_node(ctx, EXPRS["null_label_div"], c).execute()
    nl = out.column(out.schema.names.index("null_label"))
    assert nl.null_count == out.num_rows == 4 and all(nl.is_null().to_pylist())


def test_set_node_as_child_and_scalar_on_top(ctx):
    """(a > b) or b or a, then * 2 on top; and an `unless` over an `or` node."""
    from greptimedb_b200.plan import SetOpPlan
    case = CASES["filter_or_fill"]
    got = batch_rows(plan_node(ctx, EXPRS["filter_or_fill"], case).scalar_op("*", 2.0).execute(), ["k"])
    assert [r[-1] for r in got] == [6.0, 4.0, 10.0]   # x, y, z
    inner = plan_node(ctx, EXPRS["filter_or_fill"], case)
    out = SetOpPlan(ctx, "unless", inner, plan_node(ctx, ("sel", "b", {}, None, ()), case)).execute()
    assert batch_rows(out, ["k"]) == [("z", 0, 5.0)]


def test_plan_errors(ctx):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import PromRangeExec, SetOpPlan
    case = CASES["and_selectors"]
    http = lambda: plan_node(ctx, ("sel", "http_requests", {}, None, ()), case)
    cases = [
        SetOpPlan(ctx, "and", http(), plan_node(ctx, ("sel", "vector_matching_a", {}, None, ()), case)),   # key sets differ
        SetOpPlan(ctx, "unless", http(), http(), on=["job", "nope"]),   # narrowed alike: [job] on both sides
        SetOpPlan(ctx, "or", http(), http(), on=["nope"]),                                                  # on label nowhere
    ]
    with pytest.raises(B2PError) as ei:
        cases[0].execute()
    assert ei.value.code == -1 and "key columns" in str(ei.value)
    assert cases[1].execute().num_rows == 0   # `on` labels a side lacks narrow both sides alike
    with pytest.raises(B2PError) as ei:
        cases[2].execute()
    assert ei.value.code == -1 and "nope" in str(ei.value)
    # different steps
    other = dict(case, start=case["start"] - 1000)
    with pytest.raises(B2PError) as ei:
        SetOpPlan(ctx, "or", http(), plan_node(ctx, ("sel", "http_requests", {}, None, ()), other)).execute()
    assert ei.value.code == -1 and "steps" in str(ei.value)
    # an id-keyed (__tsid) side
    t = G["tables"]["http_requests"]
    labels, ts, val, offsets = table_arrays(t)
    ids = np.repeat(np.arange(len(labels), dtype=np.uint64), np.diff(offsets.astype(np.int64)))
    b = pa.record_batch([pa.array(ts, pa.timestamp("ms")), pa.array(val), pa.array(ids, pa.uint64())],
                        names=["ts", "greptime_value", "__tsid"])
    byid = PromRangeExec(ctx, "", case["start"], case["end"], case["interval"], 0, "ts", "greptime_value", ["__tsid"],
                         lookback_delta=LOOKBACK)
    byid.push(b)
    with pytest.raises(B2PError) as ei:
        SetOpPlan(ctx, "and", byid, http()).execute()
    assert ei.value.code == -1 and "__tsid" in str(ei.value)
    with pytest.raises(B2PError):
        SetOpPlan(ctx, 7, http(), http())
