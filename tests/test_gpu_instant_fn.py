"""GPU: the instant-vector functions (K9 in b2p_instant.cuh) and scalar() against the oracle — bit for bit for the exact
set, within a measured ulp bound of glibc for the transcendental ones — their errors, the device-API and plan-layer
goldens, and both orders of a function / scalar-operator chain."""
import json
import math
import os
import zlib

import numpy as np
import pytest

from tests import instant_fn_oracle as ifo
from tests.binary_helpers import dense_rows, oracle_node
from tests.instant_fn_helpers import G, ORACLE_FN, check_rows, select
from tests.ulp_bounds import ULP_BOUND, ulp_distance   # every test of these functions holds the same bound

pytestmark = pytest.mark.gpu
EXACT = ["abs", "ceil", "floor", "sqrt", "round", "deg", "rad", "sgn", "clamp", "clamp_min", "clamp_max"]
ALL = EXACT + list(ifo.TRANSCENDENTAL)
ARGS = {"round": (0.1, 0.0), "clamp": (-2.0, 3.5), "clamp_min": (0.0, 0.0), "clamp_max": (1.0, 0.0)}


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.uint64)


SPECIAL = np.concatenate([
    np.array([0x7FF8000000000001, 0xFFF800000000BEEF, 0x7FF4000000000000, 0x8000000000000000, 0x7FF0000000000000,
              0xFFF0000000000000, 0x0000000000000001, 0x800FFFFFFFFFFFFF], np.uint64).view(np.float64),
    np.array([0.0, 1.0, -1.0, 0.5, -0.5, 2.5, -2.5, 0.49999999999999994, 1.5708, 90.0, 1e300, -1e300, 3e-310, 12.0,
              -17.3, 42.5, 0.999, -0.999, 710.0, -745.0]),
])


def operands(rng, fn, n):
    """n random operands spread over the function's domain (and beyond, for the domain edges)."""
    u = rng.random(n)
    logu = np.exp(rng.uniform(-690, 690, n)) * np.where(rng.random(n) < 0.5, -1.0, 1.0)
    if fn == "exp":
        return rng.uniform(-750, 712, n)
    if fn in ("ln", "log2", "log10"):
        return np.abs(logu)
    if fn in ("sin", "cos", "tan"):
        return np.where(u < 0.4, rng.uniform(-10, 10, n), np.where(u < 0.7, rng.uniform(-1e6, 1e6, n),
                                                                   np.exp(rng.uniform(-50, 690, n))))
    if fn in ("asin", "acos", "atanh"):
        return rng.uniform(-1, 1, n)
    if fn in ("sinh", "cosh"):
        return rng.uniform(-712, 712, n)
    if fn == "tanh":
        return rng.uniform(-25, 25, n)
    if fn == "acosh":
        return 1.0 + np.abs(logu)
    return logu   # atan, asinh


def grid(rng, rows, T, fn):
    vals = np.where(rng.random((rows, T)) < 0.3, SPECIAL[rng.integers(0, SPECIAL.size, (rows, T))],
                    operands(rng, fn if fn in ifo.TRANSCENDENTAL else "sin", rows * T).reshape(rows, T))
    ok = rng.random((rows, T)) < 0.7
    return vals, ifo._words(ok)   # invalid cells keep their values: the kernel must write 0.0 there


def check_fn(fn, vals, words, out, ov, a0, a1):
    exp, ev = ifo.instant_fn(fn, vals, words, a0, a1)
    assert (ov == ev).all(), f"{fn}: validity changed"
    ok = ifo._bits(words, vals.shape[1])
    assert (bits(out[~ok]) == 0).all(), f"{fn}: an invalid cell is not 0.0"
    if fn in EXACT:
        same = (bits(out) == bits(exp)) | (np.isnan(out) & np.isnan(exp))
        assert same.all(), f"{fn}: differs from the oracle at {np.argwhere(~same)[:5].tolist()}"
    else:
        d = ulp_distance(out[ok], exp[ok])
        assert d.max(initial=0) <= ULP_BOUND[fn], f"{fn}: {d.max()} ulp from glibc"


@pytest.mark.parametrize("fn", ALL)
@pytest.mark.parametrize("T", [1, 31, 32, 33, 64, 65, 1000])
def test_host_api_in_and_out_of_place(ctx, fn, T):
    rng = np.random.default_rng(zlib.crc32(f"{fn} {T}".encode()))
    a0, a1 = ARGS.get(fn, (0.0, 0.0))
    vals, words = grid(rng, 37, T, fn)
    out, ov = ctx.instant_fn(fn, vals, words, a0, a1)
    check_fn(fn, vals, words, out, ov, a0, a1)
    if fn == "round":   # round to an integer too (to_nearest 0)
        out, ov = ctx.instant_fn(fn, vals, words, 0.0)
        check_fn(fn, vals, words, out, ov, 0.0, 0.0)


@pytest.mark.parametrize("fn", ALL)
@pytest.mark.parametrize("T", [1, 33, 64, 1000])
def test_device_api_in_place_and_aligned_out_of_place(ctx, fn, T):
    import torch
    rng = np.random.default_rng(zlib.crc32(f"dev {fn} {T}".encode()))
    a0, a1 = ARGS.get(fn, (0.0, 0.0))
    vals, words = grid(rng, 19, T, fn)
    dv = torch.from_numpy(vals.copy()).cuda()
    dw = torch.from_numpy(words.view(np.int32).copy()).cuda()
    out = torch.full_like(dv, 7.0)
    ow = torch.zeros_like(dw)
    ctx.instant_fn_dev(fn, dv, dw, 19, T, out, ow, a0, a1)
    ctx.instant_fn_dev(fn, dv, dw, 19, T, dv, dw, a0, a1)   # in place: validity words left alone
    ctx.sync()
    check_fn(fn, vals, words, out.cpu().numpy(), ow.cpu().numpy().view(np.uint32), a0, a1)
    check_fn(fn, vals, words, dv.cpu().numpy(), dw.cpu().numpy().view(np.uint32), a0, a1)


def test_ulp_bound_over_a_million_operands(ctx):
    """The max ulp distance from glibc of each transcendental function over >= 1 M random operands (written as JSON to
    $B2P_ULP_REPORT when it is set; DESIGN.md section 2 quotes them)."""
    n, measured = 1 << 20, {}
    for fn in ifo.TRANSCENDENTAL:
        rng = np.random.default_rng(zlib.crc32(f"ulp {fn}".encode()))
        x = operands(rng, fn, n).reshape(1024, 1024)
        words = ifo._words(np.ones(x.shape, bool))
        out, _ = ctx.instant_fn(fn, x, words)
        exp = ifo.apply(fn, x)
        measured[fn] = float(ulp_distance(out, exp).max())
    if os.environ.get("B2P_ULP_REPORT"):
        with open(os.environ["B2P_ULP_REPORT"], "w") as f:
            json.dump(measured, f, indent=1)
    for fn, d in measured.items():
        assert d <= ULP_BOUND[fn], f"{fn}: {d} ulp from glibc"


def test_special_cases_exact(ctx):
    inf = math.inf
    cases = [("ln", 0.0, -inf), ("ln", 1.0, 0.0), ("atanh", 1.0, inf), ("atanh", -1.0, -inf), ("acos", 1.0, 0.0),
             ("exp", -inf, 0.0), ("exp", inf, inf), ("sqrt", -0.0, -0.0), ("tanh", inf, 1.0), ("atan", -inf, -math.pi / 2),
             ("asinh", -0.0, -0.0), ("acosh", 1.0, 0.0), ("sin", -0.0, -0.0), ("tan", 0.0, 0.0), ("cosh", 0.0, 1.0)]
    for fn, x, want in cases:
        out, _ = ctx.instant_fn(fn, np.array([[x]]), np.array([[1]], np.uint32))
        assert bits(out)[0, 0] == bits(np.float64(want)), (fn, x, out[0, 0])
    for fn, x in (("ln", -1.0), ("sqrt", -1.0), ("acosh", 0.5), ("asin", 2.0), ("sin", inf), ("atanh", 2.0)):
        out, _ = ctx.instant_fn(fn, np.array([[x]]), np.array([[1]], np.uint32))
        assert np.isnan(out[0, 0]), (fn, x)


def test_errors_without_fault(ctx):
    from greptimedb_b200 import B2PError
    vals, words = np.ones((2, 5)), np.full((2, 1), 31, np.uint32)
    for bad in (27, -1, 1000):
        with pytest.raises(B2PError) as ei:
            ctx.instant_fn(bad, vals, words)
        assert ei.value.code == -1
    for fn, a0, a1 in (("clamp", 12.0, 0.0), ("clamp_min", math.inf, 0.0), ("clamp_max", -math.inf, 0.0)):
        with pytest.raises(B2PError) as ei:
            ctx.instant_fn(fn, vals, words, a0, a1)
        assert ei.value.code == -1
    out, _ = ctx.instant_fn("clamp", vals, words, math.nan, 0.5)   # a NaN bound never binds and is no error
    assert (out[:, :5] == 0.5).all()
    with pytest.raises(B2PError) as ei:
        ctx.scalar_calculate(vals, words, [0, 7])   # key 7 >= n_rows
    assert ei.value.code == -1
    out, ov = ctx.scalar_calculate(vals, words, [0, 1])   # the context stays usable
    assert np.isnan(out).all()


def _sc(ctx, ok, key, vals=None):
    ok = np.asarray(ok, bool)
    vals = np.arange(ok.size, dtype=np.float64).reshape(ok.shape) if vals is None else vals
    words = ifo._words(ok)
    got, gv = ctx.scalar_calculate(vals, words, np.asarray(key, np.uint32))
    exp, ev = ifo.scalar_calculate(vals, words, key)
    assert (gv == ev).all() and ((bits(got) == bits(exp)) | (np.isnan(got) & np.isnan(exp))).all()
    return got, ifo._bits(gv[None, :], ok.shape[1])[0]


@pytest.mark.parametrize("T", [1, 31, 32, 33, 64, 65, 1000])
def test_scalar_branches(ctx, T):
    rng = np.random.default_rng(T)
    none = np.zeros((0, T), bool)
    got, cell = _sc(ctx, none, [])                                   # no rows: NaN everywhere
    assert np.isnan(got).all() and cell.all()
    got, cell = _sc(ctx, np.zeros((3, T), bool), [0, 1, 2])          # rows without cells: NaN everywhere
    assert np.isnan(got).all() and cell.all()
    one = np.zeros((1, T), bool)
    one[0, T - 1] = True
    got, cell = _sc(ctx, one, [0])                                   # one row, one cell
    assert cell.sum() == 1 and got[T - 1] == T - 1
    ok = rng.random((6, T)) < 0.5
    ok[:, -1] = False
    ok[2, -1] = True
    for r in range(6):                                               # one series spread over rows 1, 2, 4 (no overlap)
        if r not in (1, 2, 4):
            ok[r] = False
    ok[1] &= ~ok[2]
    ok[4] &= ~(ok[1] | ok[2])
    key = [3, 0, 0, 5, 0, 1]
    payload = np.full((6, T), np.array([0x7FF8000000000ABC], np.uint64).view(np.float64)[0])
    got, cell = _sc(ctx, ok, key, payload)                           # bit copies of NaN payloads
    assert (cell == ok.any(axis=0)).all()
    two = np.zeros((2, T), bool)
    two[0, 0] = two[1, T - 1] = True
    got, cell = _sc(ctx, two, [0, 1])                                # two series: NaN everywhere
    assert np.isnan(got).all() and cell.all()
    got, _ = _sc(ctx, one, [ifo.NO_KEY])                             # NULL label, one cell: that cell
    assert got[T - 1] == T - 1
    if T > 1:
        nul = np.zeros((1, T), bool)
        nul[0, :2] = True
        got, _ = _sc(ctx, nul, [ifo.NO_KEY])                         # NULL label, two cells: NaN
        assert np.isnan(got).all()


@pytest.mark.parametrize("T", [1, 31, 33, 65, 1000])
def test_scalar_ignores_validity_bits_past_T(ctx, T):
    """Only bits k < T of a row's last validity word are defined.  The one live series is the last row and its last word
    has every bit set; a row of another key has nothing but tail bits (not live); a B2P_NO_KEY row with one cell and a
    dirty tail is one series with that cell."""
    if T % 32 == 0:
        return
    Tw = (T + 31) // 32
    tail = np.uint32(~((1 << (T % 32)) - 1) & 0xFFFFFFFF)
    vals = np.arange(3 * T, dtype=np.float64).reshape(3, T)
    words = np.zeros((3, Tw), np.uint32)
    words[0, -1] = tail                       # key 1: tail bits only
    words[2, :] = 0xFFFFFFFF                  # key 0: every step, and every tail bit
    got, gv = ctx.scalar_calculate(vals, words, [1, ifo.NO_KEY, 0])
    assert (bits(got) == bits(vals[2])).all()
    assert (ifo._bits(gv[None, :], T)[0]).all() and gv[-1] & tail == 0
    words = np.zeros((2, Tw), np.uint32)
    words[0, -1] = tail                       # no cell at all
    words[1, -1] = tail | (1 << ((T - 1) % 32))   # NULL-label row: one cell (step T - 1) and a dirty tail
    got, gv = ctx.scalar_calculate(vals[:2], words, [0, ifo.NO_KEY])
    cell = ifo._bits(gv[None, :], T)[0]
    assert cell.sum() == 1 and cell[T - 1] and got[T - 1] == vals[1, T - 1]


def test_scalar_overlap_is_an_error(ctx):
    from greptimedb_b200 import B2PError
    ok = np.zeros((2, 40), bool)
    ok[0, [1, 35]] = ok[1, [2, 35]] = True
    with pytest.raises(B2PError) as ei:
        ctx.scalar_calculate(np.ones((2, 40)), ifo._words(ok), [1, 1])
    assert ei.value.code == -1 and "same step" in str(ei.value)


# ---- goldens -----------------------------------------------------------------------------------------------------
def device_node(ctx, expr, case):
    """Dense evaluation with the device API -> (tags, labels, out, valid, eval_ts); selectors come from the oracle."""
    kind = expr[0]
    if kind == "sel":
        t = select(expr[1], expr[2])
        return oracle_node(t, case["start"], case["end"], case["interval"])
    if kind == "fn":
        tags, labels, out, valid, ets = device_node(ctx, expr[3], case)
        args = list(expr[2]) + [0.0, 0.0]
        if out.shape[0]:
            out, valid = ctx.instant_fn(ORACLE_FN.get(expr[1], expr[1]), out, valid, args[0], args[1])
        return tags, labels, out, valid, ets
    if kind == "op":
        tags, labels, out, valid, ets = device_node(ctx, expr[4], case)
        if out.shape[0]:
            out, valid = ctx.scalar_op(expr[1], expr[2], out, valid, scalar_on_left=expr[3])
        return tags, labels, out, valid, ets
    if kind == "scalar":
        tags, labels, out, valid, ets = device_node(ctx, expr[1], case)
        ids = {}
        key = [ifo.NO_KEY if None in lab else ids.setdefault(tuple(lab), len(ids)) for lab in labels]
        s, sv = ctx.scalar_calculate(out.reshape(len(labels), ets.size), valid.reshape(len(labels), -1), key)
        return [], [()], s[None, :], sv[None, :], ets
    tags, labels, out, valid, ets = device_node(ctx, expr[-1], case)   # agg_by / count
    agg, by = (expr[1], expr[2]) if kind == "agg_by" else ("count", [])
    idx = [tags.index(b) for b in by]
    keys = sorted({tuple(lab[i] for i in idx) for lab in labels})
    gid = np.array([keys.index(tuple(lab[i] for i in idx)) for lab in labels], np.uint32)
    cnt_val, cnt = ctx.group_aggregate(agg, out, valid, gid, len(keys))
    words = ifo._words(cnt != 0)
    return list(by), keys, np.where(cnt != 0, cnt_val, 0.0), words, ets


DEVICE = [c for c in G["cases"] if "device" in c["layers"]]
PLAN = [c for c in G["cases"] if "plan" in c["layers"]]


@pytest.mark.parametrize("case", DEVICE, ids=[c["name"] for c in DEVICE])
def test_device_api_goldens(ctx, case):
    tags, rows = dense_rows(*device_node(ctx, case["expr"], case))
    check_rows(case, tags, rows)


def plan_node(ctx, expr, case):
    from greptimedb_b200.plan import BinaryPlan, PromRangeExec, ScalarPlan
    import pyarrow as pa
    kind = expr[0]
    if kind == "sel":
        t = select(expr[1], expr[2])
        node = PromRangeExec(ctx, "", case["start"], case["end"], case["interval"], 0, "ts", "val", t["tags"],
                             lookback_delta=300_000)
        series = sorted(t["series"], key=lambda s: tuple(s[k] for k in t["tags"]))
        cols = {"ts": pa.array([x for s in series for x in s["ts"]], pa.timestamp("ms")),
                "val": pa.array([x for s in series for x in s["val"]], pa.float64())}
        for k in t["tags"]:
            cols[k] = pa.array([s[k] for s in series for _ in s["ts"]], pa.utf8())
        if series:
            node.push(pa.RecordBatch.from_pydict(cols))
        return node
    if kind == "fn":
        return plan_node(ctx, expr[3], case).function(expr[1], *expr[2])
    if kind == "op":
        return plan_node(ctx, expr[4], case).scalar_op(expr[1], expr[2], scalar_on_left=expr[3])
    if kind == "scalar":
        return ScalarPlan(ctx, plan_node(ctx, expr[1], case))
    assert kind == "bin"
    return BinaryPlan(ctx, expr[1], plan_node(ctx, expr[2], case), plan_node(ctx, expr[3], case),
                      label_side=expr[4].get("label_side", "rhs"))


@pytest.mark.parametrize("case", PLAN, ids=[c["name"] for c in PLAN])
def test_plan_layer_goldens(ctx, case):
    batch = plan_node(ctx, case["expr"], case).execute()
    names = batch.schema.names
    value = [n for n in names if n not in ("ts",) and n not in _tag_names(case)]
    assert len(value) == 1
    # the reference's column order; the binary node names its value without the reference's lhs. / rhs. qualifiers
    assert [value[0] if n == case["value_column"] else n for n in case["columns"]] == names
    if "." not in case["value_column"]:
        assert value[0] == case["value_column"], (value[0], case["value_column"])
    tags = _tag_names(case)
    import pyarrow as pa
    d = batch.to_pydict()
    ts = batch.column("ts").cast(pa.int64()).to_pylist()
    rows = [tuple(d[t][i] for t in tags) + (ts[i], d[value[0]][i]) for i in range(batch.num_rows)]
    check_rows(case, tags, rows)


def _tag_names(case):
    return [c for c in case["columns"] if c in ("unit", "host", "job", "instance")]


ID_KEYED = [c for c in G["cases"] if "plan_id_keyed" in c["layers"]]


@pytest.mark.parametrize("case", ID_KEYED, ids=[c["name"] for c in ID_KEYED])
def test_plan_layer_goldens_on_an_id_keyed_node(ctx, case):
    """A function stage and scalar() over a node keyed by a UInt64 __tsid column: the node carries the id, not the
    labels, so the printed values, timestamps and value column are compared."""
    import pyarrow as pa
    from greptimedb_b200.plan import PromRangeExec, ScalarPlan

    t = G["tables"][case["table"]]

    def node():
        n = PromRangeExec(ctx, "", case["start"], case["end"], case["interval"], 0, "ts", "val", ["__tsid"],
                          lookback_delta=300_000)
        s = t["series"][0]
        n.push(pa.RecordBatch.from_pydict({"ts": pa.array(s["ts"], pa.timestamp("ms")),
                                           "val": pa.array(s["val"], pa.float64()),
                                           "__tsid": pa.array([t["tsid"]] * len(s["ts"]), pa.uint64())}))
        return n

    assert case["expr"][0] == "fn"
    want = sorted((ts, v) for _, ts, v in case["expected"])
    for plan, value in ((node().function(case["expr"][1]), case["value_column"]),
                        (ScalarPlan(ctx, node().function(case["expr"][1])), "scalar(" + case["value_column"] + ")")):
        b = plan.execute()
        assert value in b.schema.names
        got = sorted(zip(b.column("ts").cast(pa.int64()).to_pylist(), b.column(value).to_pylist()))
        assert [g[0] for g in got] == [w[0] for w in want]
        assert all(float(w[1]) == g[1] for g, w in zip(got, want))
    assert b.schema.names == ["ts", "scalar(abs(val))"]


def test_plan_clamp_error(ctx):
    from greptimedb_b200 import B2PError
    e = G["errors"][0]
    with pytest.raises(B2PError) as ei:
        plan_node(ctx, e["expr"], e).execute()
    assert e["message"] in str(ei.value)
    # the reference checks the bounds once per input batch: a node without rows gives an empty result, no error
    empty = plan_node(ctx, ["fn", "clamp", [12.0, 0.0], ["sel", e["table"], {"host": "nope"}]], e).execute()
    assert empty.num_rows == 0


def test_plan_chain_orders(ctx):
    """round(x * 60, 0.1) and clamp_min(x, 0) * 2: functions and scalar operators apply in call order."""
    case = {"start": 0, "end": 35000, "interval": 5000}
    a = plan_node(ctx, ["sel", "angles", {}], case).scalar_op("*", 60.0).function("prom_round", 0.1).execute()
    b = plan_node(ctx, ["sel", "angles", {}], case).function("clamp_min", 0.0).scalar_op("*", 2.0).execute()
    assert a.schema.names[1] == "prom_round(val * Float64(60),Float64(0.1))"
    assert b.schema.names[1] == "clamp_min(val,Float64(0)) * Float64(2)"
    tags, labels, out, valid, ets = oracle_node(select("angles", {}), 0, 35000, 5000)
    ok = ifo._bits(valid, ets.size)
    ea = ifo.apply("round", out * 60.0, 0.1)[ok]
    eb = (ifo.apply("clamp_min", out, 0.0) * 2.0)[ok]
    assert (bits(np.array(a.column(1).to_pylist())) == bits(ea)).all()
    assert (bits(np.array(b.column(1).to_pylist())) == bits(eb)).all()


def test_plan_argument_errors(ctx):
    from greptimedb_b200 import B2PError
    case = {"start": 0, "end": 5000, "interval": 5000}
    node = plan_node(ctx, ["sel", "angles", {}], case)
    for name, args in (("clamp", (1.0,)), ("abs", (1.0,)), ("prom_round", (1.0, 2.0)), ("rad", ()), ("nope", ())):
        with pytest.raises(B2PError) as ei:
            node.function(name, *args)
        assert ei.value.code == -1
