"""GPU: subqueries fn(<expr>[range:step]) — K13 (b2p_subquery.cuh) plus the range tiers — against the row-literal oracle
for every range function, bit for bit against a leaf range call over the same sample rows, on the reference's goldens
through the device API and the plan layer (SubqueryPlan), in compositions, across scratch batches and in its errors."""
import json
import os
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import oracle as orc
from tests import subquery_oracle as sqo
from tests.binary_oracle import _words
from tests.helpers import GOLDEN_DIR
from tests.test_gpu_parity import ALL_FNS, BIT_EXACT, FN_PARAMS, assert_close

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN_DIR, "reference_subquery_vectors.json")) as f:
    G = json.load(f)
CASES = {c["name"]: c for c in G["cases"]}


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def params(fn, start, end, interval, rng_ms, **kw):
    from greptimedb_b200 import make_params
    p0, p1 = FN_PARAMS.get(fn, (0.0, 0.0))
    return make_params(fn, start, end, interval, rng_ms, filter_nan=False, param0=p0, param1=p1, **kw)


def bits_equal(a, b):
    return np.ascontiguousarray(a, np.float64).view(np.uint64).tobytes() == \
        np.ascontiguousarray(b, np.float64).view(np.uint64).tobytes()


def run_dev(ctx, p, s, step, vals, valid):
    import torch
    R, T_in = vals.shape
    T = orc.num_steps(p.start, p.end, p.interval)
    out = torch.full((R, T), 12345.0, dtype=torch.float64, device="cuda")
    ov = torch.full((R, (T + 31) // 32), -1, dtype=torch.int32, device="cuda")
    ctx.subquery_dev(p, s, step, torch.from_numpy(vals).cuda(), torch.from_numpy(valid.view(np.int32)).cuda(), R, T_in,
                     out, ov)
    ctx.sync()
    return out.cpu().numpy(), ov.cpu().numpy().view(np.uint32)


# ---- goldens ------------------------------------------------------------------------------------------------------------
def golden_child(c):
    t = G["tables"]["metric_total"]
    s, step, _ = sqo.inner_grid(c["start"], c["end"], c["interval"], c["range"], c["step"])
    vals, valid = sqo.instant_child(t["ts"], t["val"], s, c["end"], step, G["lookback"])
    return s, step, vals, valid


@pytest.mark.parametrize("name", sorted(CASES))
def test_goldens_through_the_device_api(ctx, name):
    c = CASES[name]
    s, step, vals, valid = golden_child(c)
    p = params(c["function"][len("prom_"):], c["start"], c["end"], c["interval"], c["range"])
    for out, ov in (ctx.subquery(p, s, step, vals, valid), run_dev(ctx, p, s, step, vals, valid)):
        assert ov[0, 0] & 1 and repr(float(out[0, 0])) == repr(float(c["expected"][0][1])), (name, out[0, 0])


@pytest.mark.parametrize("name", sorted(CASES))
def test_goldens_through_the_plan_layer(ctx, name):
    from greptimedb_b200.plan import PromRangeExec, SubqueryPlan
    c = CASES[name]
    t = G["tables"]["metric_total"]
    s, step, _ = sqo.inner_grid(c["start"], c["end"], c["interval"], c["range"], c["step"])
    child = PromRangeExec(ctx, "", s, c["end"], step, 0, "ts", "val", [], lookback_delta=G["lookback"])
    child.push(pa.RecordBatch.from_pydict({"ts": pa.array(t["ts"], pa.timestamp("ms")), "val": pa.array(t["val"])}))
    b = SubqueryPlan(ctx, c["function"], child, c["start"], c["end"], c["interval"], c["range"]).execute()
    assert b.schema.names == ["ts", c["column"]]
    got = list(zip(b.column(0).cast(pa.int64()).to_pylist(), b.column(1).to_pylist()))
    assert [(ts, repr(v)) for ts, v in got] == [(ts, repr(float(v))) for ts, v in c["expected"]]


# ---- every range function over seeded child grids -----------------------------------------------------------------------
def child_grid(rng, R, T_in):
    """Counter-like rows with resets; row 0 all valid, row 1 empty, holes elsewhere, NaN and -0.0 cells"""
    vals = np.cumsum(rng.random((R, T_in)) * 5.0, axis=1)
    reset = rng.random((R, T_in)) < 0.02
    vals = np.where(np.cumsum(reset, axis=1) % 2 == 1, vals * 0.25, vals)
    ok = rng.random((R, T_in)) < 0.75
    ok[0, :] = True
    ok[1, :] = False
    if R > 3:
        vals[2, ::7] = np.nan
        vals[3, ::5] = -0.0
        ok[4, : T_in // 2] = False
    vals[~ok] = 7777.0  # never a sample
    return vals, _words(ok)


# (start, end, interval, range, step): start' < 0; T' < 32; T' >> range / step; step == interval on a long grid
SHAPES = {"neg_start": (0, 600_000, 60_000, 300_000, 15_000),
          "short": (100_000, 160_000, 10_000, 50_000, 10_000),
          "long": (3_600_000, 9_600_000, 60_000, 300_000, 15_000),
          "regular": (1_000_000, 1_000_000 + 299 * 60_000, 60_000, 3_600_000, 60_000)}


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("fn", ALL_FNS)
def test_every_function_matches_the_oracle_and_the_leaf(ctx, fn, shape):
    start, end, interval, rng_ms, step = SHAPES[shape]
    s, step, T_in = sqo.inner_grid(start, end, interval, rng_ms, step)
    rng = np.random.default_rng(zlib.crc32(f"{fn}/{shape}".encode()))
    vals, valid = child_grid(rng, 24, T_in)
    p = params(fn, start, end, interval, rng_ms)
    out, ov = run_dev(ctx, p, s, step, vals, valid)
    p0, p1 = FN_PARAMS.get(fn, (0.0, 0.0))
    e_out, e_ov = sqo.subquery(fn, start, end, interval, rng_ms, s, step, vals, valid, p0, p1)
    T = out.shape[1]
    gv, ev = orc.valid_to_bool(ov, T), orc.valid_to_bool(e_ov, T)
    assert_close(out, e_out, gv, ev, f"{fn}/{shape}", bit_exact=fn in BIT_EXACT | {"resets", "changes", "count_over_time"})
    # K13 only reshapes: the leaf over the same sample rows gives the same bits
    ts, val, offs = sqo.grid_to_rows(vals, valid, s, step)
    l_out, l_ov, _ = ctx.range_eval(p, ts, val, offsets=offs)
    assert bits_equal(out, l_out) and (ov == l_ov).all(), f"{fn}/{shape}: differs from the leaf"
    # the host-pointer form is the same call
    h_out, h_ov = ctx.subquery(p, s, step, vals, valid)
    assert bits_equal(out, h_out) and (ov == h_ov).all()


def test_no_inner_step_and_no_rows(ctx):
    p = params("sum_over_time", 0, 60_000, 10_000, 30_000)
    out, ov = ctx.subquery(p, 0, 10_000, np.zeros((3, 0)), np.zeros((3, 0), np.uint32))
    assert out.shape == (3, 7) and not ov.any() and not out.any()
    out, ov = ctx.subquery(p, 0, 10_000, np.zeros((0, 5)), np.zeros((0, 1), np.uint32))
    assert out.shape == (0, 7)


def test_grid_larger_than_one_scratch_batch(ctx):
    """2^27 grid cells per batch: 130 rows of 2^20 steps are two batches; the result equals the leaf over the rows"""
    R, T_in, step = 130, 1 << 20, 1000
    rng = np.random.default_rng(5)
    ok = rng.random((R, T_in)) < 0.9
    vals = rng.standard_normal((R, T_in))
    p = params("max_over_time", 0, (T_in - 1) * step, 600_000, 600_000)
    out, ov = run_dev(ctx, p, 0, step, vals, _words(ok))
    r, k = np.nonzero(ok)
    ts, val = (k * step).astype(np.int64), vals[r, k]
    offs = np.concatenate([[0], np.cumsum(ok.sum(axis=1))]).astype(np.uint64)
    l_out, l_ov, _ = ctx.range_eval(p, ts, val, offsets=offs)
    assert bits_equal(out, l_out) and (ov == l_ov).all()


# ---- compositions through the plan layer ---------------------------------------------------------------------------------
HOSTS = [("a", "h1"), ("a", "h2"), ("b", "h3"), ("b", "h4"), ("c", "h5")]


def counter_table(rng, t0, t1, scrape):
    ts = np.arange(t0, t1 + 1, scrape, dtype=np.int64)
    cols = {"ts": [], "val": [], "g": [], "host": []}
    series = []
    for g, h in HOSTS:
        keep = rng.random(ts.size) < 0.9
        v = np.cumsum(rng.random(ts.size) * 10)[keep]
        series.append((ts[keep], v))
        cols["ts"] += ts[keep].tolist()
        cols["val"] += v.tolist()
        cols["g"] += [g] * int(keep.sum())
        cols["host"] += [h] * int(keep.sum())
    batch = pa.RecordBatch.from_pydict({"ts": pa.array(cols["ts"], pa.timestamp("ms")), "val": pa.array(cols["val"]),
                                        "g": pa.array(cols["g"]), "host": pa.array(cols["host"])})
    return batch, series


def leaf(ctx, batch, fn, start, end, interval, rng_ms):
    from greptimedb_b200.plan import PromRangeExec
    ex = PromRangeExec(ctx, fn, start, end, interval, rng_ms, "ts", "val", ["g", "host"])
    ex.push(batch)
    return ex


def leaf_oracle(series, fn, start, end, interval, rng_ms):
    ts = np.concatenate([s[0] for s in series])
    val = np.concatenate([s[1] for s in series])
    offs = np.concatenate([[0], np.cumsum([s[0].size for s in series])]).astype(np.uint64)
    return orc.range_query(orc.make_params(fn, start, end, interval, rng_ms), ts, val, None, offs)


def grid_of(batch, T, start, interval):
    """the export of a {time index, value, tags..} node as a dense grid over HOSTS"""
    ts = batch.column(0).cast(pa.int64()).to_pylist()
    vals = batch.column(1).to_pylist()
    hosts = batch.column(batch.schema.names.index("host")).to_pylist()
    out = np.zeros((len(HOSTS), T))
    ok = np.zeros((len(HOSTS), T), bool)
    for t, v, h in zip(ts, vals, hosts):
        r = [x[1] for x in HOSTS].index(h)
        out[r, (t - start) // interval] = v
        ok[r, (t - start) // interval] = True
    return out, ok


START, END, INTERVAL = 7_200_000, 7_200_000 + 119 * 60_000, 60_000


def close(got, ok, e_out, e_ov):
    ev = orc.valid_to_bool(e_ov, got.shape[1])
    assert (ok == ev).all()
    assert np.allclose(got[ev], e_out[ev], rtol=1e-9, atol=0, equal_nan=True)


def test_max_over_time_of_rate(ctx):
    """max_over_time(rate(x[5m])[1h:1m])"""
    from greptimedb_b200.plan import SubqueryPlan
    batch, series = counter_table(np.random.default_rng(1), 0, END, 15_000)
    s, step, _ = sqo.inner_grid(START, END, INTERVAL, 3_600_000, 60_000)
    node = SubqueryPlan(ctx, "prom_max_over_time", leaf(ctx, batch, "prom_rate", s, END, step, 300_000), START, END,
                        INTERVAL, 3_600_000)
    b = node.execute()
    assert b.schema.names == ["ts", "prom_max_over_time(ts_range,prom_rate(ts_range,val))", "g", "host"]
    c_out, c_ov = leaf_oracle(series, "rate", s, END, step, 300_000)
    e_out, e_ov = sqo.subquery("max_over_time", START, END, INTERVAL, 3_600_000, s, step, c_out, c_ov)
    close(*grid_of(b, e_out.shape[1], START, INTERVAL), e_out, e_ov)


def test_avg_over_time_of_a_ratio_and_sum_by_over_it(ctx):
    """avg_over_time((rate(a[5m]) / rate(b[5m]))[30m:1m]) and sum by (g)(max_over_time(rate(a[5m])[30m:1m]))"""
    from greptimedb_b200.plan import AggregatePlan, BinaryPlan, SubqueryPlan
    ba, sa = counter_table(np.random.default_rng(2), 0, END, 15_000)
    bb, sb = counter_table(np.random.default_rng(3), 0, END, 15_000)
    s, step, _ = sqo.inner_grid(START, END, INTERVAL, 1_800_000, 60_000)
    ratio = BinaryPlan(ctx, "/", leaf(ctx, ba, "prom_rate", s, END, step, 300_000),
                       leaf(ctx, bb, "prom_rate", s, END, step, 300_000))
    b = SubqueryPlan(ctx, "prom_avg_over_time", ratio, START, END, INTERVAL, 1_800_000).execute()
    ra, va = leaf_oracle(sa, "rate", s, END, step, 300_000)
    rb, vb = leaf_oracle(sb, "rate", s, END, step, 300_000)
    T_in = ra.shape[1]
    both = orc.valid_to_bool(va, T_in) & orc.valid_to_bool(vb, T_in)
    e_out, e_ov = sqo.subquery("avg_over_time", START, END, INTERVAL, 1_800_000, s, step, np.where(both, ra / rb, 0.0),
                               _words(both))
    close(*grid_of(b, e_out.shape[1], START, INTERVAL), e_out, e_ov)

    sub = SubqueryPlan(ctx, "prom_max_over_time", leaf(ctx, ba, "prom_rate", s, END, step, 300_000), START, END,
                       INTERVAL, 1_800_000)
    agg = AggregatePlan(ctx, "sum", sub, by=["g"]).execute()
    m_out, m_ov = sqo.subquery("max_over_time", START, END, INTERVAL, 1_800_000, s, step, ra, va)
    gid = np.array([0, 0, 1, 1, 2], np.uint32)
    g_sum, g_cnt = orc.group_aggregate("sum", m_out, m_ov, gid, 3)
    ts = agg.column(agg.schema.names.index("ts")).cast(pa.int64()).to_pylist()
    gs = agg.column(agg.schema.names.index("g")).to_pylist()
    vs = agg.column(agg.schema.names.index("sum(prom_max_over_time(ts_range,prom_rate(ts_range,val)))")).to_pylist()
    got = {(g, t): v for g, t, v in zip(gs, ts, vs)}
    exp = {(g, START + k * INTERVAL): g_sum[i, k] for i, g in enumerate("abc") for k in range(g_sum.shape[1])
           if g_cnt[i, k]}
    assert got.keys() == exp.keys()
    assert all(np.isclose(got[k], exp[k], rtol=1e-9, atol=0) for k in got)


def test_subquery_over_a_subquery(ctx):
    """max_over_time(deriv(rate(x[5m])[10m:30s])[1h:1m]): the inner subquery runs on the outer one's inner grid"""
    from greptimedb_b200.plan import SubqueryPlan
    batch, series = counter_table(np.random.default_rng(4), 0, END, 15_000)
    s1, st1, _ = sqo.inner_grid(START, END, INTERVAL, 3_600_000, 60_000)
    s2, st2, _ = sqo.inner_grid(s1, END, st1, 600_000, 30_000)
    inner = SubqueryPlan(ctx, "prom_deriv", leaf(ctx, batch, "prom_rate", s2, END, st2, 300_000), s1, END, st1, 600_000)
    b = SubqueryPlan(ctx, "prom_max_over_time", inner, START, END, INTERVAL, 3_600_000).execute()
    assert b.schema.names[1] == "prom_max_over_time(ts_range,prom_deriv(ts_range,prom_rate(ts_range,val)))"
    c_out, c_ov = leaf_oracle(series, "rate", s2, END, st2, 300_000)
    d_out, d_ov = sqo.subquery("deriv", s1, END, st1, 600_000, s2, st2, c_out, c_ov)
    e_out, e_ov = sqo.subquery("max_over_time", START, END, INTERVAL, 3_600_000, s1, st1, d_out, d_ov)
    close(*grid_of(b, e_out.shape[1], START, INTERVAL), e_out, e_ov)


def test_elementwise_stage_and_parameter_names(ctx):
    from greptimedb_b200.plan import SubqueryPlan
    batch, _ = counter_table(np.random.default_rng(6), 0, END, 15_000)
    s, step, _ = sqo.inner_grid(START, END, INTERVAL, 600_000, 30_000)
    for fn, p0, p1, name in [("prom_quantile_over_time", 0.5, 0.0, "prom_quantile_over_time(ts_range,val,Float64(0.5))"),
                             ("prom_predict_linear", 3.0, 0.0, "prom_predict_linear(ts_range,val,Float64(3))"),
                             ("prom_holt_winters", 0.5, 0.1, "prom_holt_winters(ts_range,val,Float64(0.5),Float64(0.1))"),
                             ("prom_increase", 0.0, 0.0, "prom_increase(ts_range,val,ts,Int64(600000))")]:
        from greptimedb_b200.plan import PromRangeExec
        child = PromRangeExec(ctx, "", s, END, step, 0, "ts", "val", ["g", "host"], lookback_delta=300_000)
        child.push(batch)
        node = SubqueryPlan(ctx, fn, child, START, END, INTERVAL, 600_000, param0=p0, param1=p1)
        assert node.execute().schema.names[1] == name
    node.scalar_op("*", 2.0)
    assert node.execute().schema.names[1] == "prom_increase(ts_range,val,ts,Int64(600000)) * Float64(2)"


# ---- errors -------------------------------------------------------------------------------------------------------------
def test_plan_errors(ctx):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import PromRangeExec, SubqueryPlan
    child = PromRangeExec(ctx, "", 0, 60_000, 10_000, 0, "ts", "val", [], lookback_delta=300_000)
    for kw in [dict(function="prom_nope"), dict(interval=0), dict(range=0), dict(offset=5_000)]:
        args = dict(function="prom_sum_over_time", start=0, end=60_000, interval=10_000, range=30_000)
        args.update(kw)
        with pytest.raises(B2PError) as ei:
            SubqueryPlan(ctx, args.pop("function"), child, **args)
        assert ei.value.code == -1 and "GpuPromSubqueryExec" in str(ei.value), kw


def test_device_api_errors(ctx):
    from greptimedb_b200 import B2PError
    vals, valid = np.zeros((2, 5)), np.zeros((2, 1), np.uint32)
    for p, step in [(params(99, 0, 60_000, 10_000, 30_000), 10_000), (params("rate", 0, 60_000, 0, 30_000), 10_000),
                    (params("rate", 0, 60_000, 10_000, 0), 10_000), (params("rate", 0, 60_000, 10_000, 30_000, offset=1), 10_000),
                    (params("rate", 0, 60_000, 10_000, 30_000), 0)]:
        with pytest.raises(B2PError) as ei:
            ctx.subquery(p, 0, step, vals, valid)
        assert ei.value.code == -1
    from greptimedb_b200 import make_params
    with pytest.raises(B2PError):  # filter_nan must be 0
        ctx.subquery(make_params("rate", 0, 60_000, 10_000, 30_000), 0, 10_000, vals, valid)
