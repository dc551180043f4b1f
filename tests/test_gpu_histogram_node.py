"""GPU: histogram_quantile(φ, <any node>) — HistogramQuantilePlan over the host-pointer fold b2p_histogram_fold (K5) —
on the reference's goldens, bit for bit against the range leaf's fused fold, against the row-literal oracle over the
child's exported rows in compositions and at its edges, and in its errors."""
import json
import math
import os

import numpy as np
import pyarrow as pa
import pytest

from tests import histogram_node_oracle as hno
from tests import subquery_oracle as sqo
from tests.binary_oracle import _words
from tests.helpers import GOLDEN_DIR

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN_DIR, "reference_histogram_node_vectors.json")) as f:
    G = json.load(f)
CASES = {c["name"]: c for c in G["cases"]}
B2P_E_INVALID = -1


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def table_batch(series, tags, string_tags=True):
    """series [({tag: label or None}, ts list, val list)] -> one pyarrow batch, series after series"""
    cols = {"ts": [], "val": []}
    for t in tags:
        cols[t] = []
    for lab, ts, val in series:
        cols["ts"].extend(ts)
        cols["val"].extend(val)
        for t in tags:
            cols[t].extend([lab.get(t)] * len(ts))
    data = {"ts": pa.array(cols["ts"], pa.timestamp("ms")), "val": pa.array(cols["val"], pa.float64())}
    for t in tags:
        data[t] = pa.array(cols[t], pa.string() if string_tags else pa.uint64())
    return pa.RecordBatch.from_pydict(data)


def leaf(ctx, batch, tags, start, end, interval, fn="prom_rate", range_ms=300_000, instant=False, lookback=300_000,
         **kw):
    from greptimedb_b200.plan import PromRangeExec
    n = PromRangeExec(ctx, "" if instant else fn, start, end, interval, range_ms, "ts", "val", tags,
                      lookback_delta=lookback if instant else None, **kw)
    n.push(batch)
    return n


def rows_of(batch):
    """An exported batch -> (rows [(value, {tag: label}, ts)], tag names): tags are the Utf8 columns"""
    names = batch.schema.names
    tags = [n for n, t in zip(names, batch.schema.types) if pa.types.is_string(t)]
    ts = next(n for n, t in zip(names, batch.schema.types) if pa.types.is_timestamp(t))
    val = next(n for n, t in zip(names, batch.schema.types) if pa.types.is_floating(t))
    return hno.batch_rows(batch, tags, ts, val), tags


def keyed(rows):
    out = {}
    for v, lab, ts in rows:
        k = (tuple(sorted(lab.items())), ts)
        assert k not in out, f"two rows for {k}"
        out[k] = v
    return out


def same(a, b):
    return (math.isnan(a) and math.isnan(b)) or a == b or abs(a - b) <= 1e-12 * max(abs(a), abs(b))


def check_against_oracle(ctx, child, phi, what=""):
    """The node over `child` equals the oracle over the child's exported rows; returns the node's batch"""
    from greptimedb_b200.plan import HistogramQuantilePlan
    c_rows, c_tags = rows_of(child.execute())
    got_batch = HistogramQuantilePlan(ctx, phi, child).execute()
    e_rows, e_tags = hno.histogram_node(c_rows, c_tags, phi)
    if "le" not in c_tags:
        assert got_batch.num_rows == 0 and got_batch.num_columns == 0, what
        return got_batch
    g_rows, g_tags = rows_of(got_batch)
    assert sorted(g_tags) == sorted(e_tags), what
    g, e = keyed(g_rows), keyed(e_rows)
    assert g.keys() == e.keys(), what
    for k in g:
        assert same(g[k], e[k]), (what, k, g[k], e[k])
    return got_batch


def histograms(rng, hists, les, n, t0=0, scrape=15_000, tags=("job", "instance", "le"), missing=0.0):
    """Counter series of every (histogram, le): cumulative over le, increasing over time, seeded; `missing` drops that
    share of samples"""
    series = []
    for h in hists:
        w = rng.random(len(les)) * 3.0 + 0.1
        for b, le in enumerate(les):
            ts = t0 + scrape * np.arange(n, dtype=np.int64)
            val = np.cumsum(np.full(n, w[: b + 1].sum())) + rng.random(n) * 0.01
            keep = rng.random(n) >= missing
            lab = dict(h)
            lab[tags[-1]] = le
            series.append((lab, ts[keep].tolist(), val[keep].tolist()))
    return table_batch(series, list(tags))


LES = ["0.005", "0.01", "0.025", "0.05", "0.1", "0.25", "0.5", "1", "2.5", "5", "10", "+Inf"]
HISTS = [{"job": j, "instance": f"i{k}"} for j in ("api", "db", "web") for k in range(3)]
START, END, STEP = 600_000, 600_000 + 40 * 15_000, 15_000  # T = 41: one full 32-step tile and a partial one


def bucket_leaf(ctx, seed=1, instant=False, fn="prom_rate", hists=HISTS, les=LES, missing=0.0, **kw):
    batch = histograms(np.random.default_rng(seed), hists, les, 90, missing=missing)
    return leaf(ctx, batch, ["job", "instance", "le"], START, END, STEP, fn=fn, instant=instant, **kw)


# ---- goldens -------------------------------------------------------------------------------------------------------------
def golden_child(ctx, c):
    from greptimedb_b200.plan import AggregatePlan
    t = G["tables"][c["table"]]
    ch = c["child"]
    series = [({k: s[k] for k in t["tags"]}, s["ts"], s["val"]) for s in t["series"]
              if all(s[k] == v for k, v in ch.get("matchers", {}).items())]
    node = leaf(ctx, table_batch(series, t["tags"]), t["tags"], c["start"], c["end"], c["interval"],
                fn=ch.get("function", ""), range_ms=ch.get("range", 0), instant=ch["kind"] == "instant")
    if "aggregate" in ch:
        node = AggregatePlan(ctx, ch["aggregate"], node, by=ch["by"])
    return node


@pytest.mark.parametrize("name", sorted(CASES))
def test_goldens_through_the_plan_layer(ctx, name):
    from greptimedb_b200.plan import HistogramQuantilePlan, TopkPlan
    c = CASES[name]
    node = HistogramQuantilePlan(ctx, float(c["phi"]), golden_child(ctx, c))
    if "outer" in c:
        node = TopkPlan(ctx, c["outer"]["op"], c["outer"]["k"], node)
    b = node.execute()
    assert b.schema.names == c["columns"], (name, b.schema.names)
    assert b.num_rows == len(c["expected"])
    if not c["expected"]:
        return
    rows, _ = rows_of(b)
    for (v, lab, ts), (e_lab, e_ts, e_v) in zip(rows, c["expected"]):
        assert lab == e_lab and ts == e_ts, name
        assert repr(v) == repr(float(e_v)) or (math.isnan(v) and e_v == "NaN"), (name, v, e_v)


# ---- the node over a range leaf is the leaf's own fused fold ---------------------------------------------------------
@pytest.mark.parametrize("fn", ["prom_rate", "prom_increase", "prom_irate", "prom_delta", "prom_avg_over_time",
                                "prom_max_over_time"])
def test_node_over_a_range_leaf_equals_the_fused_leaf_bit_for_bit(ctx, fn):
    from greptimedb_b200.plan import HistogramQuantilePlan
    fused = bucket_leaf(ctx, seed=7, fn=fn, missing=0.1, histogram_quantile=0.9).execute()
    node = HistogramQuantilePlan(ctx, 0.9, bucket_leaf(ctx, seed=7, fn=fn, missing=0.1)).execute()
    assert node.schema.names == fused.schema.names
    assert node.num_rows == fused.num_rows > 0
    for i in range(fused.num_columns):
        a, b = node.column(i), fused.column(i)
        if pa.types.is_floating(a.type):
            assert np.asarray(a).view(np.uint64).tolist() == np.asarray(b).view(np.uint64).tolist(), fn
        else:
            assert a.equals(b), fn


# ---- compositions ----------------------------------------------------------------------------------------------------
def test_over_an_instant_selector(ctx):
    check_against_oracle(ctx, bucket_leaf(ctx, seed=2, instant=True), 0.75)


@pytest.mark.parametrize("by,without", [(["le", "job"], None), (None, ["instance"]), (["job"], None)])
def test_over_an_aggregate(ctx, by, without):
    from greptimedb_b200.plan import AggregatePlan
    child = AggregatePlan(ctx, "sum", bucket_leaf(ctx, seed=3, missing=0.05), by=by, without=without)
    check_against_oracle(ctx, child, 0.99, f"by={by} without={without}")


def test_over_binary_nodes(ctx):
    from greptimedb_b200.plan import BinaryPlan
    check_against_oracle(ctx, bucket_leaf(ctx, seed=4).scalar_op("*", 2.0), 0.5, "x * 2")
    a = bucket_leaf(ctx, seed=5, hists=[{"job": "api", "instance": "i0"}])
    b = bucket_leaf(ctx, seed=6, hists=[{"job": "api", "instance": "i9"}])
    child = BinaryPlan(ctx, "/", a, b, on=["le", "job"], label_side="rhs")
    check_against_oracle(ctx, child, 0.5, "a / on(le, job) b")


def test_over_or_topk_and_subquery(ctx):
    from greptimedb_b200.plan import SetOpPlan, SubqueryPlan, TopkPlan
    a = bucket_leaf(ctx, seed=8, hists=HISTS[:4])
    b = bucket_leaf(ctx, seed=9, hists=HISTS[2:6])
    check_against_oracle(ctx, SetOpPlan(ctx, "or", a, b), 0.9, "or")
    check_against_oracle(ctx, TopkPlan(ctx, "topk", 3, bucket_leaf(ctx, seed=10), by=["job", "le"]), 0.9, "topk")
    s, step, _ = sqo.inner_grid(START, END, STEP, 300_000, 15_000)
    batch = histograms(np.random.default_rng(11), HISTS[:3], LES, 120)
    inner = leaf(ctx, batch, ["job", "instance", "le"], s, END, step)
    sub = SubqueryPlan(ctx, "prom_max_over_time", inner, START, END, STEP, 300_000)
    check_against_oracle(ctx, sub, 0.9, "subquery")


def test_under_other_nodes_and_stages(ctx):
    from greptimedb_b200.plan import (AggregatePlan, BinaryPlan, HistogramQuantilePlan, ScalarPlan, TopkPlan)

    def node(seed=12):
        return HistogramQuantilePlan(ctx, 0.9, bucket_leaf(ctx, seed=seed))

    h_rows, h_tags = rows_of(node().execute())
    # stages on top: * 1000 then clamp_min
    b = node().scalar_op("*", 1000.0).function("clamp_min", 50.0).execute()
    got, _ = rows_of(b)
    assert keyed(got) == {k: max(v * 1000.0, 50.0) for k, v in keyed(h_rows).items()}
    assert b.schema.names[1] == "clamp_min(prom_rate(ts_range,val) * Float64(1000),Float64(50))"
    # topk over the node
    t = TopkPlan(ctx, "topk", 2, node(), by=["job"]).execute()
    got, _ = rows_of(t)
    for v, lab, ts in got:
        peers = sorted((hv for hv, hl, hts in h_rows if hl["job"] == lab["job"] and hts == ts), reverse=True)
        assert v in peers[:2]
    # the aggregate over the node
    a = AggregatePlan(ctx, "max", node(), by=["job"]).execute()
    got, _ = rows_of(a)
    for v, lab, ts in got:
        assert v == max(hv for hv, hl, hts in h_rows if hl["job"] == lab["job"] and hts == ts)
    # a binary node over two histogram nodes: node / node is 1 wherever the quantile is finite and non-zero
    d = BinaryPlan(ctx, "/", node(13), node(13)).execute()
    got, _ = rows_of(d)
    assert len(got) == len(h_rows) and all(v == 1.0 for v, _, _ in got)
    # scalar() over a one-histogram node is that histogram's row
    one = HistogramQuantilePlan(ctx, 0.5, bucket_leaf(ctx, seed=14, hists=HISTS[:1]))
    e_rows, _ = rows_of(HistogramQuantilePlan(ctx, 0.5, bucket_leaf(ctx, seed=14, hists=HISTS[:1])).execute())
    sc = ScalarPlan(ctx, one).execute()
    assert [r[0] for r in rows_of(sc)[0]] == [v for v, _, _ in e_rows]


# ---- edges -----------------------------------------------------------------------------------------------------------
def test_children_without_rows(ctx):
    from greptimedb_b200.plan import HistogramQuantilePlan
    empty = leaf(ctx, table_batch([], ["job", "le"]), ["job", "le"], START, END, STEP)
    b = HistogramQuantilePlan(ctx, 0.5, empty).execute()
    assert b.num_rows == 0 and b.schema.names == ["ts", "prom_rate(ts_range,val)", "job"]
    # a leaf whose windows are all empty
    far = leaf(ctx, histograms(np.random.default_rng(0), HISTS[:2], LES, 5, t0=10**9), ["job", "instance", "le"],
               START, END, STEP)
    assert HistogramQuantilePlan(ctx, 0.5, far).execute().num_rows == 0


@pytest.mark.parametrize("end", [START, START + 14 * STEP, START + 31 * STEP, START + 32 * STEP, START + 70 * STEP])
def test_step_counts(ctx, end):
    batch = histograms(np.random.default_rng(end % 97), HISTS[:4], LES, 120, missing=0.1)
    check_against_oracle(ctx, leaf(ctx, batch, ["job", "instance", "le"], START, end, STEP), 0.9, f"T={end}")


def literal_buckets(ctx, layout, n=40, phi=0.5, tags=("job", "le")):
    """layout {job: [(le label, value fn(k) or None to leave the series out at k)]}: one instant leaf, checked"""
    series = []
    for job, buckets in layout.items():
        for le, f in buckets:
            ks = [k for k in range(n) if f(k) is not None]
            series.append(({"job": job, "le": le}, [START + k * STEP for k in ks], [f(k) for k in ks]))
    # a lookback shorter than the step: a step sees only its own samples, so whole histograms can be absent
    child = leaf(ctx, table_batch(series, list(tags)), list(tags), START, START + (n - 1) * STEP, STEP, instant=True,
                 lookback=STEP - 1)
    return check_against_oracle(ctx, child, phi)


def test_layout_edges(ctx):
    nan = float("nan")
    layout = {
        # the first histogram in order lacks +Inf, so the reference folds everything in its safe mode
        "a_no_inf": [("0.5", lambda k: 1.0 + k), ("1", lambda k: 2.0 + k)],
        "b_one_bucket": [("+Inf", lambda k: 3.0)],
        "c_dup_le": [("1", lambda k: 2.0), ("1.0", lambda k: 4.0), ("2", lambda k: 6.0), ("+Inf", lambda k: 9.0)],
        "d_nan_values": [("0.1", lambda k: nan if k % 3 == 0 else 1.0), ("1", lambda k: -0.0 if k % 2 else 3.0),
                         ("5", lambda k: -2.0), ("+Inf", lambda k: 7.0)],
        "e_absent": [("1", lambda k: None if k % 4 == 0 else 2.0), ("+Inf", lambda k: None if k % 4 == 0 else 5.0)],
        "f_partial": [("0.1", lambda k: None if k % 2 else 1.0), ("1", lambda k: 3.0), ("3", lambda k: None if k % 5 else 3.5),
                      ("+Inf", lambda k: None if k % 7 == 0 else 4.0)],
        "g_neg": [("-1", lambda k: -5.0), ("0", lambda k: -1.0), ("+Inf", lambda k: 2.0 * k)],
    }
    for phi in (0.0, 0.25, 0.5, 0.99, 1.0):
        literal_buckets(ctx, layout, phi=phi)


def test_null_unparsable_le_and_null_tags(ctx):
    series = [({"job": "a", "le": "0.5"}, [START], [1.0]), ({"job": "a", "le": "1"}, [START], [2.0]),  # no +Inf
              ({"job": None, "le": "1"}, [START], [2.0]), ({"job": None, "le": "+Inf"}, [START], [4.0]),
              ({"job": "b", "le": "1"}, [START], [2.0]), ({"job": "b", "le": "+Inf"}, [START], [4.0]),
              ({"job": "b", "le": None}, [START], [5.0]), ({"job": "b", "le": "abc"}, [START], [6.0]),
              ({"job": "c", "le": "0x10"}, [START], [1.0]), ({"job": "c", "le": " 1"}, [START], [2.0]),
              ({"job": "c", "le": "inf"}, [START], [3.0]), ({"job": "", "le": "1"}, [START], [1.0]),
              ({"job": "", "le": "+Inf"}, [START], [3.0])]
    child = leaf(ctx, table_batch(series, ["job", "le"]), ["job", "le"], START, START, STEP, instant=True)
    b = check_against_oracle(ctx, child, 0.5)
    assert b.column(2).to_pylist() == ["", None, "a", "b", "c"]  # Labels::less: "" first, then NULL


def test_more_than_64_buckets(ctx):
    les = [repr(0.01 * (i + 1)) for i in range(99)] + ["+Inf"]
    for missing in (0.0, 0.2):
        batch = histograms(np.random.default_rng(31), HISTS[:3], les, 60, missing=missing)
        child = leaf(ctx, batch, ["job", "instance", "le"], START, END, STEP)
        check_against_oracle(ctx, child, 0.9, f"100 buckets, missing={missing}")


# ---- errors and the empty result ---------------------------------------------------------------------------------------
def test_plan_errors_and_the_empty_result(ctx):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import CountValuesPlan, HistogramQuantilePlan
    ids = leaf(ctx, table_batch([({"__tsid": 7}, [START], [1.0])], ["__tsid"], string_tags=False), ["__tsid"],
               START, START, STEP, instant=True)
    with pytest.raises(B2PError, match="id-keyed") as ei:
        HistogramQuantilePlan(ctx, 0.5, ids).execute()
    assert ei.value.code == B2P_E_INVALID
    cv = CountValuesPlan(ctx, "le", bucket_leaf(ctx, seed=41), by=["job"])
    with pytest.raises(B2PError, match="count_values") as ei:
        HistogramQuantilePlan(ctx, 0.5, cv).execute()
    assert ei.value.code == B2P_E_INVALID
    no_le = leaf(ctx, histograms(np.random.default_rng(42), HISTS[:2], LES, 60, tags=("job", "instance", "bucket")),
                 ["job", "instance", "bucket"], START, END, STEP)
    node = HistogramQuantilePlan(ctx, 0.5, no_le)
    b = node.execute()
    assert b.num_rows == 0 and b.num_columns == 0
    # nodes above see no rows over the child's steps
    from greptimedb_b200.plan import ScalarPlan
    sc = ScalarPlan(ctx, HistogramQuantilePlan(ctx, 0.5, no_le)).execute()
    assert sc.num_rows == 41 and all(math.isnan(v) for v in sc.column(1).to_pylist())
    # the le column can be named
    renamed = HistogramQuantilePlan(ctx, 0.5, no_le, le="bucket").execute()
    assert renamed.num_rows > 0 and "bucket" not in renamed.schema.names


# ---- the host-pointer fold -------------------------------------------------------------------------------------------
def fold_inputs(rng, R=70, T=45):
    rates = np.cumsum(rng.random((R, T)) * 3.0, axis=0)
    rates[rng.random((R, T)) < 0.05] = np.nan
    ok = rng.random((R, T)) < 0.9
    rates[~ok] = 0.0
    sizes = [1, 2, 5, 64, 65, 0, 3, 12]
    bs, les, off = [], [], [0]
    perm = rng.permutation(R)
    p = 0
    for n in sizes:
        take = [int(perm[(p + i) % R]) for i in range(n)]
        p += n
        bs += take
        les += sorted(rng.random(n - 1).tolist()) + [math.inf] if n else []
        off.append(len(bs))
    return (np.array(off, np.uint32), np.array(bs, np.uint32), np.array(les, np.float64), rates, _words(ok))


def test_host_fold_equals_the_device_fold_and_rejects_bad_indices(ctx):
    import torch
    off, bs, les, rates, words = fold_inputs(np.random.default_rng(51))
    H, T = off.size - 1, rates.shape[1]
    out, ov = ctx.histogram_fold(0.9, off, bs, les, rates, words)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int32) if a.dtype == np.uint32 else a).cuda()
    out_d = torch.zeros((H, T), dtype=torch.float64, device="cuda")
    ov_d = torch.zeros((H, (T + 31) // 32), dtype=torch.int32, device="cuda")
    ctx.histogram_fold_dev(0.9, d(off), d(bs), d(les), H, d(rates), d(words), T, out_d, ov_d)
    ctx.sync()
    assert out.view(np.uint64).tolist() == out_d.cpu().numpy().view(np.uint64).tolist()
    assert (ov == ov_d.cpu().numpy().view(np.uint32)).all() and ov.any()
    from greptimedb_b200 import B2PError
    bad = {"first offset": (np.concatenate([[1], off[1:]]).astype(np.uint32), bs),
           "decreasing": (np.array([0, 5, 3] + off[3:].tolist(), np.uint32), bs),
           "row out of range": (off, np.where(np.arange(bs.size) == 9, rates.shape[0], bs).astype(np.uint32))}
    for what, (o, b) in bad.items():
        before = ctx.launch_count()
        with pytest.raises(B2PError) as ei:
            ctx.histogram_fold(0.9, o, b, les, rates, words)
        assert ei.value.code == B2P_E_INVALID, what
        assert ctx.launch_count() == before, f"{what}: a kernel ran"
