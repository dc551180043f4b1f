"""GPU: count_values by label (K12 in b2p_count_values.cuh) against the dense oracle bit for bit, at the batch
boundaries, and the count_values node (CountValuesPlan) on the goldens, over other nodes, under nodes and in its
errors."""
import json
import math
import os

import numpy as np
import pyarrow as pa
import pytest

from tests import binary_oracle as bor
from tests import count_values_oracle as cvo
from tests.helpers import GOLDEN_DIR
from tests.test_count_values_oracle import SPECIAL
from tests.test_gpu_aggregate_node import JOB_TABLE, STEPS, export_rows, instant_node

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN_DIR, "reference_count_values_vectors.json")) as f:
    G = json.load(f)
CASES = {c["name"]: c for c in G["cases"]}


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def same(a, b):
    return np.asarray(a, np.float64).view(np.uint64).tobytes() == np.asarray(b, np.float64).view(np.uint64).tobytes()


def shape(rng, T, sizes):
    """Groups of the given sizes, an empty group id between every two, 1 % of the rows with a group id out of range;
    values from a small pool with NaNs of both signs and several payloads, ±0, ±inf (many duplicates), or spread;
    some rows and steps without cells."""
    gid = np.concatenate([np.full(s, 2 * g, np.uint32) for g, s in enumerate(sizes)])
    n_groups = 2 * len(sizes)
    gid[rng.random(gid.size) < 0.01] = n_groups + 5
    rng.shuffle(gid)
    R = gid.size
    vals = rng.choice(np.concatenate([SPECIAL, np.array([1.0, 2.0, -3.0, 7.5])]), (R, T))
    spread = rng.random((R, T)) < 0.3
    vals[spread] = rng.standard_normal(int(spread.sum()))
    ok = rng.random((R, T)) < 0.85
    ok[rng.random(R) < 0.05] = False
    if T > 2:
        ok[:, 1] = False
    vals[~ok] = 12345.0  # never read
    return vals, bor._words(ok), gid, n_groups


SIZES = [1, 2, 64, 65, 1000, 0, 3]


def run_dev(ctx, vals, valid, gid, n_groups):
    import torch
    T = vals.shape[1]
    d_vals = torch.from_numpy(vals).cuda()
    d_valid = torch.from_numpy(valid.view(np.int32)).cuda()
    d_gid = torch.from_numpy(gid.view(np.int32)).cuda()
    out = torch.full(vals.shape, 12345.0, dtype=torch.float64, device="cuda")  # overwritten
    cnt = torch.full(vals.shape, 777, dtype=torch.int32, device="cuda")
    ix = ctx.group_index_create_dev(d_gid, gid.size, n_groups)
    try:
        ctx.count_values_dev(d_vals, d_valid, ix, T, out, cnt)
        ctx.sync()
    finally:
        ctx.group_index_destroy(ix)
    return out.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("T", [1, 31, 32, 33, 64, 65, 200, 1000])
def test_device_api_matches_the_dense_oracle(ctx, T):
    rng = np.random.default_rng(T)
    vals, valid, gid, G_ = shape(rng, T, SIZES if T <= 200 else [1, 2, 64, 65, 0, 3])
    exp, ecnt = cvo.count_values(vals, valid, gid, G_)
    out, cnt = ctx.count_values(vals, valid, gid, G_)
    assert (cnt == ecnt).all() and same(out, exp)
    dout, dcnt = run_dev(ctx, vals, valid, gid, G_)
    assert (dcnt == ecnt).all() and same(dout, exp)
    again, acnt = ctx.count_values(vals, valid, gid, G_)
    assert (acnt == cnt).all() and same(again, out)


def test_one_group_of_100k_rows(ctx):
    rng = np.random.default_rng(5)
    T = 33
    vals, valid, gid, _ = shape(rng, T, [100_000])
    gid[:] = 0
    exp, ecnt = cvo.count_values(vals, valid, gid, 1)
    out, cnt = ctx.count_values(vals, valid, gid, 1)
    assert (cnt == ecnt).all() and same(out, exp)


def test_no_group_in_range(ctx):
    vals = np.ones((5, 40))
    valid = bor._words(np.ones((5, 40), bool))
    out, cnt = ctx.count_values(vals, valid, np.full(5, 9, np.uint32), 2)
    assert not cnt.any() and not out.any()


def check_sampled(out, cnt, vals_np, ok_np, gid_np, n_groups, steps, groups):
    order, goff = cvo.member_order(gid_np, n_groups)
    for k in steps:
        for g in groups:
            rows = order[goff[g]:goff[g + 1]]
            cell = vals_np[rows[ok_np[rows, k]], k]
            keys = cell.view(np.int64) ^ ((cell.view(np.int64) >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))
            uniq, n = np.unique(keys, return_counts=True)
            b = (uniq ^ ((uniq >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))).view(np.float64)
            c = cnt[goff[g]:goff[g + 1], k]
            assert (c[:n.size] == n).all() and not c[n.size:].any(), (g, k)
            assert same(out[goff[g]:goff[g] + n.size, k], b), (g, k)


def test_several_batches_of_groups(ctx):
    """250 k rows x 1000 steps in 1000 groups: more cells than one batch holds, so the groups are cut into runs."""
    rng = np.random.default_rng(8)
    R, T, G_ = 250_000, 1000, 1000
    vals = rng.integers(0, 40, (R, T)).astype(np.float64)
    ok = rng.random((R, T)) < 0.9
    gid = rng.integers(0, G_, R).astype(np.uint32)
    out, cnt = ctx.count_values(vals, bor._words(ok), gid, G_)
    order, goff = cvo.member_order(gid, G_)
    assert (np.diff(goff) > 0).all()
    per_group = np.add.reduceat(cnt, goff[:-1], axis=0, dtype=np.int64)  # rows are in member order
    exp = np.add.reduceat(ok[order], goff[:-1], axis=0, dtype=np.int64)
    assert (per_group == exp).all()
    check_sampled(out, cnt, vals, ok, gid, G_, [0, 31, 32, 500, 999], [0, 1, 500, 998, 999])


def test_one_group_cut_into_step_windows(ctx):
    """One group of 2.2 M rows: its cells over 64 steps exceed a batch, so it runs in windows of 32 steps."""
    rng = np.random.default_rng(9)
    R, T = 2_200_000, 70
    vals = rng.integers(0, 3000, (R, T)).astype(np.float64)
    vals[:, 5] = -0.0
    vals[::2, 5] = 0.0
    ok = rng.random((R, T)) < 0.95
    gid = np.zeros(R, np.uint32)
    out, cnt = ctx.count_values(vals, bor._words(ok), gid, 1)
    assert (cnt.sum(axis=0, dtype=np.int64) == ok.sum(axis=0)).all()
    check_sampled(out, cnt, vals, ok, gid, 1, [0, 5, 31, 32, 63, 64, 69], [0])
    assert cnt[2:, 5].sum() == 0 and cnt[0, 5] and cnt[1, 5]  # -0.0 and +0.0, in that order
    assert math.copysign(1.0, out[0, 5]) < 0 and math.copysign(1.0, out[1, 5]) > 0


# ---- plan layer ---------------------------------------------------------------------------------------------------------
def cv_rows(b):
    """an exported count_values batch -> ([(count, {tag: label}, ts, value)], tag names)"""
    names = b.schema.names
    ti = next(i for i, f in enumerate(b.schema) if pa.types.is_timestamp(f.type))
    ts = b.column(ti).cast(pa.int64()).to_pylist()
    cnt, val = b.column(0).to_pylist(), b.column(len(names) - 1).to_pylist()
    tags = names[1:ti]
    cols = {t: b.column(names.index(t)).to_pylist() for t in tags}
    return [(cnt[r], {t: cols[t][r] for t in tags}, ts[r], val[r]) for r in range(b.num_rows)], tags


def cv(ctx, label, child, **kw):
    from greptimedb_b200.plan import CountValuesPlan
    return CountValuesPlan(ctx, label, child, **kw)


@pytest.mark.parametrize("name", sorted(c["name"] for c in G["cases"] if "plan" in c["layers"]))
def test_plan_goldens(ctx, name):
    c = CASES[name]
    node = cv(ctx, c["label"], instant_node(ctx, G["tables"][c["table"]], c, c["select"]), by=c.get("by"))
    out = node.execute()
    rows, _ = cv_rows(out)
    assert [(lab, ts, n, v) for n, lab, ts, v in rows] == [tuple(e) for e in c["expected"]]
    assert out.schema.names == [n.replace("http_requests.", "") for n in c["columns"]]
    assert [str(f.type) for f in out.schema] == c["types"]


def test_plan_schema(ctx):
    """planner.rs:6723: {count(<value>) Int64, group labels.., time index, <label> Float64}"""
    s = G["schema"]
    from greptimedb_b200.plan import PromRangeExec
    ex = PromRangeExec(ctx, "", 0, 10000, 5000, 0, s["time_index"], s["value_column"], s["tags"], lookback_delta=1000)
    ex.push(pa.RecordBatch.from_pydict({
        s["time_index"]: pa.array([0, 5000, 0], pa.timestamp("ms")),
        s["value_column"]: pa.array([1.0, 2.0, 1.0], pa.float64()),
        "ip": pa.array(["10.0.160.237:8080", "10.0.160.237:8080", "10.0.160.237:9090"], pa.utf8())}))
    out = cv(ctx, s["label"], ex, by=s["by"]).execute()
    assert out.schema.names == [n.replace("prometheus_tsdb_head_series.", "") for n in s["columns"]]
    assert [str(f.type) for f in out.schema] == ["int64", "string", "timestamp[ms]", "double"]
    rows, _ = cv_rows(out)
    assert [(n, lab["ip"][-4:], ts, v) for n, lab, ts, v in rows] == [(1, "8080", 0, 1.0), (1, "8080", 5000, 2.0),
                                                                   (1, "9090", 0, 1.0)]


def check_over(ctx, child_factory, **kw):
    child_rows, tags = export_rows(child_factory().execute())
    exp, _ = cvo.count_values_rows(child_rows, tags, **kw)
    got, _ = cv_rows(cv(ctx, "v", child_factory(), **kw).execute())
    assert [(n, lab, ts) for n, lab, ts, _ in got] == [(n, lab, ts) for n, lab, ts, _ in exp]
    assert same([v for *_, v in got], [v for *_, v in exp])
    return got


def test_compositions(ctx):
    from greptimedb_b200.plan import AggregatePlan, BinaryPlan
    x = lambda: instant_node(ctx, JOB_TABLE, STEPS)
    # count_values("v", x) by (job), over an instant selector; without (instance); no modifier
    assert check_over(ctx, x, by=["job"])
    check_over(ctx, x, without=["instance"])
    check_over(ctx, x)
    # over a binary node: count_values("v", floor(x / 2))
    check_over(ctx, lambda: BinaryPlan(ctx, "/", x(), x().scalar_op("*", 0.0).scalar_op("+", 2.0)).function("floor"),
               by=["job"])
    # count(count_values("v", x)): how many distinct values per step
    child_rows, tags = export_rows(x().execute())
    exp, _ = cvo.count_values_rows(child_rows, tags)
    per_ts = {}
    for _, _, ts, _ in exp:
        per_ts[ts] = per_ts.get(ts, 0) + 1
    got, _ = export_rows(AggregatePlan(ctx, "count", cv(ctx, "v", x())).execute())
    assert [(ts, v) for v, _, ts in got] == sorted((ts, float(n)) for ts, n in per_ts.items())
    # sum by (job)(count_values("v", x) by (job)) is the number of cells per job
    got, _ = export_rows(AggregatePlan(ctx, "sum", cv(ctx, "v", x(), by=["job"]), by=["job"]).execute())
    cells = {}
    for _, lab, ts in child_rows:
        cells[(lab["job"], ts)] = cells.get((lab["job"], ts), 0) + 1
    assert [((lab["job"], ts), v) for v, lab, ts in got] == sorted((k, float(n)) for k, n in cells.items())


def test_element_wise_stage_on_top(ctx):
    """count_values("v", x) > 1: the export keeps the layout and the label column; the count is Float64 there."""
    x = lambda: instant_node(ctx, JOB_TABLE, STEPS).scalar_op("/", 4.0).function("floor")  # repeated values
    child_rows, tags = export_rows(x().execute())
    exp, _ = cvo.count_values_rows(child_rows, tags, by=["job"])
    out = cv(ctx, "v", x(), by=["job"]).scalar_op(">", 1.0).execute()
    assert [str(f.type) for f in out.schema] == ["double", "string", "timestamp[ms]", "double"]
    assert out.schema.names == ["count(floor(val / Float64(4)))", "job", "ts", "v"]
    got, _ = cv_rows(out)
    assert got == [(float(n), lab, ts, v) for n, lab, ts, v in exp if n > 1] and got


def test_plan_errors(ctx):
    from greptimedb_b200 import B2PError
    x = lambda: instant_node(ctx, JOB_TABLE, STEPS)
    for label, kw in (("job", {"by": ["job"]}), ("instance", {"without": ["job"]}), ("ts", {})):
        with pytest.raises(B2PError, match="names another column"):
            cv(ctx, label, x(), **kw).execute()
    assert cv(ctx, "job", x(), by=["instance"]).execute().num_rows  # the child's tag, but not a group label
    ided = lambda: instant_node(ctx, JOB_TABLE, STEPS, id_column="__tsid")
    for mod in ({"by": ["__tsid"]}, {"without": ["job"]}):
        with pytest.raises(B2PError, match="id-keyed"):
            cv(ctx, "v", ided(), **mod).execute()
    got, tags = cv_rows(cv(ctx, "v", ided()).execute())
    assert tags == [] and got
