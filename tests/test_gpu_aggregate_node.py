"""GPU: quantile by label (K11 in b2p_quantile.cuh) against the dense oracle bit for bit, a 1.25 M-row × 1000-step run
against numpy, and the aggregate node (AggregatePlan) on the goldens, against the leaf's aggregate, over other nodes and
in its errors."""
import json
import math
import os

import numpy as np
import pyarrow as pa
import pytest

from tests import aggregate_oracle as ago
from tests import binary_oracle as bor
from tests.binary_helpers import sum_rate_table
from tests.helpers import GOLDEN_DIR
from tests.test_aggregate_oracle import CASES, G, NAN_NEG, PHIS, SPECIAL

pytestmark = pytest.mark.gpu

RESIDENT = 64  # kQuantResident


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return bool(((np.isnan(a) & np.isnan(b)) | (a.view(np.uint64) == b.view(np.uint64))).all())


def shape(rng, T, sizes):
    """Groups of the given sizes, an empty group id between every two, 1 % of the rows with a group id out of range;
    values: normal numbers, NaNs of both signs, ±0, ±inf and many duplicates; some rows and steps without cells."""
    gid = np.concatenate([np.full(s, 2 * g, np.uint32) for g, s in enumerate(sizes)])
    n_groups = 2 * len(sizes)
    gid[rng.random(gid.size) < 0.01] = n_groups + 5
    rng.shuffle(gid)
    R = gid.size
    vals = rng.choice(np.array([1.0, 2.0, -3.0, 7.5]), (R, T))
    spread = rng.random((R, T)) < 0.5
    vals[spread] = rng.standard_normal(int(spread.sum())) * 10.0 ** rng.integers(-3, 4, int(spread.sum()))
    special = rng.random((R, T)) < 0.05
    vals[special] = SPECIAL[rng.integers(0, SPECIAL.size, int(special.sum()))]
    ok = rng.random((R, T)) < 0.85
    ok[rng.random(R) < 0.05] = False
    if T > 2:
        ok[:, 1] = False
    return vals, bor._words(ok), gid, n_groups


SIZES = [1, 2, 31, 32, 33, RESIDENT - 1, RESIDENT, RESIDENT + 1, 5000, 0, 3]


def run_dev(ctx, phi, vals, valid, gid, n_groups):
    import torch
    T = vals.shape[1]
    d_vals = torch.from_numpy(vals).cuda()
    d_valid = torch.from_numpy(valid.view(np.int32)).cuda()
    d_gid = torch.from_numpy(gid.view(np.int32)).cuda()
    out = torch.full((n_groups, T), 12345.0, dtype=torch.float64, device="cuda")  # overwritten
    cnt = torch.full((n_groups, T), 777, dtype=torch.int32, device="cuda")
    ix = ctx.group_index_create_dev(d_gid, gid.size, n_groups)
    try:
        ctx.group_quantile_dev(phi, d_vals, d_valid, ix, T, out, cnt)
        ctx.sync()
    finally:
        ctx.group_index_destroy(ix)
    return out.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("T", [1, 31, 32, 33, 64, 65, 200, 1000])
def test_device_api_matches_the_dense_oracle(ctx, T):
    rng = np.random.default_rng(T)
    vals, valid, gid, G_ = shape(rng, T, SIZES if T <= 200 else SIZES[:-3] + [0, 3])
    phis = PHIS + [NAN_NEG] if T in (1, 33) else [0.5, 0.99]
    for phi in phis:
        exp, ecnt = ago.group_quantile(phi, vals, valid, gid, G_)
        out, cnt = ctx.group_quantile(phi, vals, valid, gid, G_)
        assert (cnt == ecnt).all(), phi
        assert same_bits(out, exp), phi
        dout, dcnt = run_dev(ctx, phi, vals, valid, gid, G_)
        assert (dcnt == ecnt).all() and same_bits(dout, exp), phi
        again, _ = ctx.group_quantile(phi, vals, valid, gid, G_)
        assert (again.view(np.uint64) == out.view(np.uint64)).all()


def test_one_group_of_100k_rows_is_chunked(ctx):
    rng = np.random.default_rng(5)
    T = 33
    vals, valid, gid, _ = shape(rng, T, [100_000])
    gid[gid != 0] = 0  # one group (no row out of range)
    for phi in (0.0, 0.25, 0.5, 0.99, 1.0):
        exp, ecnt = ago.group_quantile(phi, vals, valid, gid, 1)
        out, cnt = ctx.group_quantile(phi, vals, valid, gid, 1)
        assert (cnt == ecnt).all() and same_bits(out, exp), phi
        again, _ = ctx.group_quantile(phi, vals, valid, gid, 1)
        assert (again.view(np.uint64) == out.view(np.uint64)).all()


def test_inf_times_zero_on_the_device(ctx):
    vals = np.array([[1.0], [math.inf]])
    valid = np.ones((2, 1), np.uint32)
    for phi in (0.0, 1.0):
        out, cnt = ctx.group_quantile(phi, vals, valid, np.zeros(2, np.uint32), 1)
        assert cnt[0, 0] == 2 and math.isnan(out[0, 0])


@pytest.mark.parametrize("u", [u for u in G["units"] if "device" in u["layers"]], ids=lambda u: u["name"])
def test_accumulator_unit_vectors_on_the_device(ctx, u):
    n = len(u["values"])
    vals = np.array(u["values"] or [0.0], np.float64).reshape(-1, 1)
    valid = np.full((max(n, 1), 1), 1 if n else 0, np.uint32)
    out, cnt = ctx.group_quantile(u["phi"], vals, valid, np.zeros(max(n, 1), np.uint32), 1)
    assert cnt[0, 0] == n
    if n:  # (no values: the reference's NaN, but an aggregate has no empty bucket; count 0 is no row here)
        assert out[0, 0] == u["expected"]


def test_1_25m_rows_1000_steps_1000_groups(ctx):
    """Counts on every cell; values on sampled (group, step) cells against numpy's sort-and-interpolate."""
    import torch
    R, T, G_ = 1_250_000, 1000, 1000
    gen = torch.Generator(device="cuda").manual_seed(11)
    vals = torch.randn((R, T), dtype=torch.float64, device="cuda", generator=gen)
    vals[:, 7] = 4.0  # a step of ties
    Tw = (T + 31) // 32
    valid = torch.randint(-2**31, 2**31, (R, Tw), dtype=torch.int32, device="cuda", generator=gen)
    lanes = torch.arange(32, device="cuda", dtype=torch.int32)

    def ok_of(w0, w1):  # [R, steps of words w0..w1) the validity bits, as int32
        return ((valid[:, w0:w1].unsqueeze(-1) >> lanes) & 1).reshape(R, -1)[:, :T - 32 * w0]

    gid_np = np.random.default_rng(3).integers(0, G_, R).astype(np.uint32)
    gid = torch.from_numpy(gid_np.view(np.int32)).cuda()
    out = torch.empty((G_, T), dtype=torch.float64, device="cuda")
    cnt = torch.empty((G_, T), dtype=torch.int32, device="cuda")
    ix = ctx.group_index_create_dev(gid, R, G_)
    try:
        ctx.group_quantile_dev(0.9, vals, valid, ix, T, out, cnt)
        ctx.sync()
    finally:
        ctx.group_index_destroy(ix)
    gidl = gid.to(torch.int64)
    for w0 in range(0, Tw, 4):
        ok = ok_of(w0, min(w0 + 4, Tw))
        exp_cnt = torch.zeros((G_, ok.shape[1]), dtype=torch.int32, device="cuda")
        exp_cnt.index_add_(0, gidl, ok)
        assert torch.equal(cnt[:, 32 * w0:32 * w0 + ok.shape[1]], exp_cnt), w0
    rng = np.random.default_rng(4)
    for k in [0, 7, 999] + list(rng.integers(0, T, 5)):
        col = vals[:, k].cpu().numpy()
        okc = ok_of(k // 32, k // 32 + 1)[:, k % 32].cpu().numpy().astype(bool)
        for g in rng.integers(0, G_, 20):
            s = np.sort(col[(gid_np == g) & okc])
            rank = 0.9 * (s.size - 1)
            lo = int(math.floor(rank))
            hi = min(s.size - 1, lo + 1)
            w = rank - math.floor(rank)
            assert out[g, k].item() == s[lo] * (1 - w) + s[hi] * w, (g, k)


# ---- plan layer ---------------------------------------------------------------------------------------------------------
def instant_node(ctx, table, case, select=None, id_column=None):
    from greptimedb_b200.plan import PromRangeExec
    series = sorted((s for s in table["series"] if all(s[k] == v for k, v in (select or {}).items())),
                    key=lambda s: tuple(s[t] for t in table["tags"]))
    tags = [id_column] if id_column else table["tags"]
    ex = PromRangeExec(ctx, "", case["start"], case["end"], case["interval"], 0, table["time_index"], table["field"], tags,
                       lookback_delta=case.get("lookback", 300_000))
    cols = {table["time_index"]: pa.array([t for s in series for t in s["ts"]], pa.timestamp("ms")),
            table["field"]: pa.array([v for s in series for v in s["val"]], pa.float64())}
    if id_column:
        cols[id_column] = pa.array([1000 + i for i, s in enumerate(series) for _ in s["ts"]], pa.uint64())
    else:
        for t in table["tags"]:
            cols[t] = pa.array([s[t] for s in series for _ in s["ts"]], pa.utf8())
    if series:
        ex.push(pa.RecordBatch.from_pydict(cols))
    return ex


def export_rows(b):
    """-> ([(value, {tag: label}, ts)] in the batch's order, tag names)"""
    names = b.schema.names
    vi = next(i for i, f in enumerate(b.schema) if pa.types.is_float64(f.type))
    ti = next(i for i, f in enumerate(b.schema) if pa.types.is_timestamp(f.type))
    ts = b.column(ti).cast(pa.int64()).to_pylist()
    vals = b.column(vi).to_pylist()
    tags = [n for i, n in enumerate(names) if i not in (vi, ti)]
    cols = {t: b.column(names.index(t)).to_pylist() for t in tags}
    return [(vals[r], {t: cols[t][r] for t in tags}, ts[r]) for r in range(b.num_rows)], tags


def agg(ctx, o, child):
    from greptimedb_b200.plan import AggregatePlan
    return AggregatePlan(ctx, o["op"], child, param=o.get("param"), by=o.get("by"), without=o.get("without"))


PLAN_CASES = sorted(c["name"] for c in G["cases"] if "plan" in c["layers"])


@pytest.mark.parametrize("name", PLAN_CASES)
def test_plan_goldens(ctx, name):
    c = CASES[name]
    node = instant_node(ctx, G["tables"][c["table"]], c, c["select"])
    for o in c["ops"]:
        node = agg(ctx, o, node)
    out = node.execute()
    rows, _ = export_rows(out)
    assert [(lab, ts, v) for v, lab, ts in rows] == [tuple(e) for e in c["expected"]]
    names = out.schema.names
    assert len(names) == len(c["columns"]) and names[:-1] == c["columns"][:-1]
    if "." not in c["columns"][-1]:
        assert names[-1] == c["columns"][-1]
    if c["ops"][-1]["op"] == "quantile":  # φ as a literal, the child's value column unqualified
        assert names[-1] == "quantile(%s,%s)" % ("Float64(0.5)", "sum(val)" if len(c["ops"]) > 1 else "val")


def test_scalar_count_of_an_aggregate(ctx):
    """scalar.result:128-164: ScalarPlan(AggregatePlan(count, AggregatePlan(op by (host))))."""
    from greptimedb_b200.plan import ScalarPlan
    with open(os.path.join(GOLDEN_DIR, "reference_instant_fn_vectors.json")) as f:
        g = json.load(f)
    for name in ("scalar:128", "scalar:140", "scalar:152", "scalar:164"):
        c = next(c for c in g["cases"] if c["name"] == name)
        _, (_, op, by, sel) = c["expr"][1]
        inner = agg(ctx, {"op": op, "by": by}, instant_node(ctx, g["tables"][sel[1]], c, sel[2]))
        out = ScalarPlan(ctx, agg(ctx, {"op": "count"}, inner)).execute()
        rows, _ = export_rows(out)
        assert [(lab, ts, v) for v, lab, ts in rows] == [(e[0], e[1], float(e[2])) for e in c["expected"]], name
        assert out.schema.names[-1] == c["value_column"].replace("host.", ""), name


def test_ratio_repro_without_hand_chained_calls(ctx):
    from greptimedb_b200.plan import BinaryPlan
    from tests.test_gpu_binary import CASES as BC
    from tests.test_gpu_binary import G as BG
    from tests.test_gpu_binary import node
    c = BC["ratio_filtered_count"]
    a = node(ctx, BG["tables"]["metric_a"], c, fn="rate", range_ms=c["range"])
    b = node(ctx, BG["tables"]["metric_b"], c)
    kept = BinaryPlan(ctx, "/", a, b, on=["l3", "l4"], label_side="rhs").scalar_op(">", 0.50)
    counted = agg(ctx, {"op": "count"}, kept)
    rows, _ = export_rows(counted.execute())
    assert [(lab, ts, v) for v, lab, ts in rows] == [tuple(e) for e in c["expected"]]
    pct = BinaryPlan(ctx, "/", counted, agg(ctx, {"op": "count"}, a)).scalar_op("*", 100.0)
    rows, _ = export_rows(pct.execute())
    assert [(lab, ts, v) for v, lab, ts in rows] == [tuple(e) for e in BC["ratio_times_100"]["expected"]]


OPS = ["sum", "avg", "count", "min", "max", "stddev", "stdvar"]


@pytest.mark.parametrize("op", OPS)
def test_same_as_the_leaf_aggregate(ctx, op):
    """AggregatePlan(op, by) over a bare range node == the leaf's aggregate=op: rows and value bits; only the value
    column's name differs."""
    from greptimedb_b200.plan import PromRangeExec
    from tests.test_gpu_binary import table_batch
    t = sum_rate_table()
    with open(os.path.join(GOLDEN_DIR, "reference_sum_rate_vectors.json")) as f:
        cases = json.load(f)["cases"]
    for c in cases:
        for by in ([], ["host"], ["service"], ["host", "service"]):
            def range_node(aggregate=None):
                ex = PromRangeExec(ctx, "prom_rate", c["start"], c["end"], c["interval"], c["range"], "ts", "val",
                                   t["tags"], aggregate=aggregate, by_columns=by if aggregate else [])
                ex.push(table_batch(t))
                return ex
            leaf = range_node(op).execute()
            node = agg(ctx, {"op": op, "by": by}, range_node()).execute()
            assert node.schema.names[:-1] == leaf.schema.names[:-1]
            assert leaf.schema.names[-1] == f"{op}(prom_rate)"
            df = {"stddev": "stddev_pop", "stdvar": "var_pop"}.get(op, op)
            assert node.schema.names[-1] == f"{df}(prom_rate(ts_range,val))"
            lr, _ = export_rows(leaf)
            nr, _ = export_rows(node)
            assert [r[1:] for r in lr] == [r[1:] for r in nr]
            assert same_bits([r[0] for r in lr], [r[0] for r in nr])


# ---- compositions: the node against the row-literal aggregate of its child's exported rows -----------------------------
JOB_TABLE = {
    "time_index": "ts", "field": "val", "tags": ["instance", "job"],
    "series": [{"instance": f"i{i}", "job": ["api", "db", "web"][i % 3], "ts": [0, 30000, 60000, 90000],
                "val": [float((i * 7) % 11) + 0.25 * k for k in range(4)]} for i in range(10)],
}
STEPS = {"start": 0, "end": 90000, "interval": 30000}


def check_over(ctx, child_factory, o, post=None):
    child_rows, tags = export_rows(child_factory().execute())
    exp, _ = ago.aggregate_rows(child_rows, tags, o["op"], o.get("param"), by=o.get("by"), without=o.get("without"))
    node = agg(ctx, o, child_factory())
    if post:
        node = post(node)
        exp = [(bor.binary_value(post.op, v, post.scalar), lab, ts) for v, lab, ts in exp]
    got, _ = export_rows(node.execute())
    assert [(lab, ts) for _, lab, ts in got] == [(lab, ts) for _, lab, ts in exp]
    assert same_bits([v for v, _, _ in got], [v for v, _, _ in exp])
    return got


def test_compositions(ctx):
    from greptimedb_b200.plan import BinaryPlan, SetOpPlan, TopkPlan
    x = lambda: instant_node(ctx, JOB_TABLE, STEPS)
    # sum by (job)(a / b)
    check_over(ctx, lambda: BinaryPlan(ctx, "/", x(), x().scalar_op("+", 1.0)), {"op": "sum", "by": ["job"]})
    # count(x > 5)
    got = check_over(ctx, lambda: x().scalar_op(">", 5.0), {"op": "count"})
    assert got and all(lab == {} for _, lab, _ in got)
    # max(topk(3, x))
    check_over(ctx, lambda: TopkPlan(ctx, "topk", 3, x()), {"op": "max"})
    # avg without (instance)(abs(x))
    check_over(ctx, lambda: x().scalar_op("-", 5.0).function("abs"), {"op": "avg", "without": ["instance"]})
    # quantile(0.9, x) by (job) * 2

    class Times2:
        op, scalar = "*", 2.0

        def __call__(self, node):
            return node.scalar_op("*", 2.0)

    check_over(ctx, x, {"op": "quantile", "param": 0.9, "by": ["job"]}, post=Times2())
    # over `or` with NULL labels: the rhs has a tag the lhs lacks
    other = {"time_index": "ts", "field": "val", "tags": ["instance", "job", "zone"],
             "series": [{"instance": "i99", "job": "api", "zone": "z1", "ts": [0, 30000], "val": [4.0, 8.0]}]}
    union = lambda: SetOpPlan(ctx, "or", x(), instant_node(ctx, other, STEPS))
    for o in ({"op": "sum", "by": ["zone"]}, {"op": "quantile", "param": 0.5, "by": ["zone", "job"]}, {"op": "group", "without": ["instance"]}):
        check_over(ctx, union, o)
    # an aggregate over an aggregate
    check_over(ctx, lambda: agg(ctx, {"op": "count", "by": ["job"]}, x()), {"op": "count"})
    check_over(ctx, lambda: agg(ctx, {"op": "stdvar", "by": ["job"]}, x()), {"op": "quantile", "param": 0.5})


def test_quantile_value_name_keeps_the_sign_of_zero(ctx):
    x = instant_node(ctx, JOB_TABLE, STEPS)
    assert agg(ctx, {"op": "quantile", "param": -0.0}, x).execute().schema.names[-1] == "quantile(Float64(-0),val)"
    assert agg(ctx, {"op": "quantile", "param": 0.0}, x).execute().schema.names[-1] == "quantile(Float64(0),val)"


def test_id_keyed_child_without_modifier(ctx):
    node = agg(ctx, {"op": "sum"}, instant_node(ctx, JOB_TABLE, STEPS, id_column="__tsid"))
    out = node.execute()
    rows, tags = export_rows(out)
    assert tags == []
    plain, _ = export_rows(agg(ctx, {"op": "sum"}, instant_node(ctx, JOB_TABLE, STEPS)).execute())
    assert [r[2] for r in rows] == [r[2] for r in plain] and same_bits([r[0] for r in rows], [r[0] for r in plain])


def test_plan_errors(ctx):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import AggregatePlan
    x = lambda: instant_node(ctx, JOB_TABLE, STEPS)
    with pytest.raises(B2PError, match="count_values is not supported by this node"):
        AggregatePlan(ctx, "count_values", x())
    for op in ("topk", "bottomk"):
        with pytest.raises(B2PError, match="b2p_plan_topk_create"):
            AggregatePlan(ctx, op, x())
    with pytest.raises(B2PError, match="unknown aggregator median"):
        AggregatePlan(ctx, "median", x())
    ided = lambda: instant_node(ctx, JOB_TABLE, STEPS, id_column="__tsid")
    for mod in ({"by": ["__tsid"]}, {"without": ["job"]}):
        with pytest.raises(B2PError, match="id-keyed"):
            AggregatePlan(ctx, "sum", ided(), **mod).execute()
