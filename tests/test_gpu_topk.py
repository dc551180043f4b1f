"""GPU: topk / bottomk (K10 in b2p_topk.cuh) against the dense oracle bit for bit, a 1.25 M-row one-group run, and the
plan layer (TopkPlan) on the sqlness goldens and over binary, set, function and scalar() compositions."""
import math

import numpy as np
import pyarrow as pa
import pytest

from tests import topk_oracle as tko
from tests.binary_helpers import LOOKBACK, table_arrays
from tests.test_topk_oracle import CASES, G, KS, NAN_NEG

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.uint64)


# NaN payloads of both signs, ±0, ±inf, repeated ordinary numbers (value ties)
VALS = np.concatenate([
    np.array([0x7FF8000000000001, 0xFFF800000000BEEF, 0x7FF4000000000000, 0x8000000000000000, 0x7FF0000000000000,
              0xFFF0000000000000, 0x0000000000000001], np.uint64).view(np.float64),
    np.array([0.0, 1.0, 1.0, -2.5, 1e300, 7.0]),
])


def shape(rng, T, big=2500, small=60):
    """One group of `big` rows (several chunks), one of 150 (one chunk, more than the fast path's largest k), `small`
    groups of 0..9 rows, empty group ids between them, rows with no valid cell, and rows whose group id is out of range."""
    sizes = [big, 150] + list(rng.integers(0, 10, small))
    gid = np.concatenate([np.full(s, 2 * g, np.uint32) for g, s in enumerate(sizes)])  # odd ids: empty groups
    n_groups = 2 * len(sizes)
    gid[rng.random(gid.size) < 0.01] = n_groups + 3
    rng.shuffle(gid)
    R = gid.size
    vals = VALS[rng.integers(0, VALS.size, (R, T))]
    spread = rng.random((R, T)) < 0.5  # half the cells distinct, the rest drawn from VALS (ties)
    vals[spread] = rng.standard_normal(int(spread.sum()))
    ok = rng.random((R, T)) < 0.8
    ok[rng.random(R) < 0.05] = False
    tie = rng.permutation(R).astype(np.uint32)
    return vals, tko._words(ok), gid, n_groups, tie


def kk_of(k, largest):
    return float(largest) if k == "largest" else float(k)


@pytest.mark.parametrize("T", [1, 31, 32, 33, 64, 65, 200, 1000])
def test_device_api_matches_the_dense_oracle(ctx, T):
    import torch
    rng = np.random.default_rng(T)
    vals, valid, gid, n_groups, tie = shape(rng, T, big=2500 if T <= 200 else 1200)
    R = gid.size
    dev = torch.device("cuda:0")
    d_vals = torch.from_numpy(vals.copy()).to(dev)
    d_valid = torch.from_numpy(valid.view(np.int32).copy()).to(dev)
    d_gid = torch.from_numpy(gid.view(np.int32)).to(dev)
    d_tie = torch.from_numpy(tie.view(np.int32)).to(dev)
    ix = ctx.group_index_create_dev(d_gid, R, n_groups)
    largest = int(np.bincount(gid[gid < n_groups]).max())
    try:
        for op in ("topk", "bottomk"):
            for k in KS + [100.0]:
                k = kk_of(k, largest)
                exp = tko.topk(op == "bottomk", k, vals, valid, gid, n_groups, tie)
                out = torch.full_like(d_valid, -1)
                ctx.topk_dev(op, k, d_vals, d_valid, ix, d_tie, T, out)
                again = torch.full_like(d_valid, -1)
                ctx.topk_dev(op, k, d_vals, d_valid, ix, d_tie, T, again)
                inplace = d_valid.clone()
                ctx.topk_dev(op, k, d_vals, inplace, ix, d_tie, T, inplace)
                ctx.sync()
                got = out.cpu().numpy().view(np.uint32)
                assert (got == exp).all(), (op, k)
                assert (again.cpu().numpy() == out.cpu().numpy()).all(), (op, k)
                assert (inplace.cpu().numpy().view(np.uint32) == exp).all(), (op, k)
                assert (bits(d_vals.cpu().numpy()) == bits(vals)).all(), "the value grid was written"
                assert (d_valid.cpu().numpy().view(np.uint32) == valid).all(), "the input words were written"
    finally:
        ctx.group_index_destroy(ix)


def test_host_api_and_errors(ctx):
    from greptimedb_b200 import B2PError
    rng = np.random.default_rng(5)
    vals, valid, gid, n_groups, tie = shape(rng, 70, big=700)
    for op, k in [("topk", 3), ("bottomk", 40), ("topk", math.inf), ("bottomk", NAN_NEG)]:
        exp = tko.topk(op == "bottomk", k, vals, valid, gid, n_groups, tie)
        assert (ctx.topk(op, k, vals, valid, gid, n_groups, tie) == exp).all(), (op, k)
    with pytest.raises(B2PError) as ei:
        ctx._check(ctx._L.b2p_topk(ctx._h, 0, 1.0, None, None, None, 3, 1, None, 4, None))
    assert ei.value.code == -1


def test_one_group_of_1_25m_rows(ctx):
    """topk(10) over 1.25 M rows x 1000 steps in one group: argpartition on sampled steps, kept counts on every step."""
    import torch
    R, T, kk = 1_250_000, 1000, 10
    Tw = (T + 31) // 32
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(7)
    vals = torch.rand((R, T), dtype=torch.float64, device=dev, generator=g)
    shifts = torch.arange(32, device=dev, dtype=torch.int64)
    valid = torch.empty((R, Tw), dtype=torch.int32, device=dev)
    for w in range(Tw):   # 90 % of the cells valid; no bit at or past T
        ok = (torch.rand((R, 32), device=dev, generator=g) < 0.9) & (w * 32 + shifts < T)
        x = (ok.to(torch.int64) << shifts).sum(1)
        valid[:, w] = torch.where(x >= 2 ** 31, x - 2 ** 32, x).to(torch.int32)
    tie = torch.randperm(R, device=dev, generator=g).to(torch.int32)
    gid = torch.zeros(R, dtype=torch.int32, device=dev)
    ix = ctx.group_index_create_dev(gid, R, 1)
    out = torch.empty_like(valid)
    try:
        ctx.topk_dev("topk", float(kk), vals, valid, ix, tie, T, out)
        ctx.sync()
    finally:
        ctx.group_index_destroy(ix)
    word_bits = lambda t, w: (t[:, w].to(torch.int64).unsqueeze(1) >> shifts) & 1   # [R, 32]
    sample = set(range(0, T, 97)) | {T - 1}
    for w in range(Tw):
        kept, ok = word_bits(out, w), word_bits(valid, w)
        assert (kept & (1 - ok)).sum().item() == 0, "a kept cell that was not valid"
        assert torch.equal(kept.sum(0), torch.clamp(ok.sum(0), max=kk)), w
        for b in range(32):
            k = w * 32 + b
            if k not in sample:
                continue
            col = torch.where(ok[:, b].bool(), vals[:, k], torch.tensor(-1.0, dtype=torch.float64, device=dev))
            top = np.argpartition(-col.cpu().numpy(), kk)[:kk]
            assert set(top.tolist()) == set(torch.nonzero(kept[:, b]).flatten().cpu().numpy().tolist()), k


# ---- plan layer ---------------------------------------------------------------------------------------------------------
def table_batch(table, series=None):
    table = dict(table, series=series if series is not None else table["series"])
    labels, ts, val, offsets = table_arrays(table)
    n = np.diff(offsets.astype(np.int64))
    cols = [pa.array(ts, pa.timestamp("ms")), pa.array(val, pa.float64())]
    names = [table["time_index"], table["field"]]
    for i, t in enumerate(table["tags"]):
        cols.append(pa.array(np.repeat(np.array([lab[i] for lab in labels], dtype=object), n).tolist(), pa.string()))
        names.append(t)
    return pa.record_batch(cols, names=names)


def input_node(ctx, case, **match):
    from greptimedb_b200.plan import PromRangeExec
    inp = case.get("input", {"table": "test"})
    t = G["tables"][inp["table"]]
    series = [s for s in t["series"] if all(s[k] == v for k, v in match.items())]
    if inp.get("histogram"):
        ex = PromRangeExec(ctx, "prom_rate", case["start"], case["end"], case["interval"], case["range"],
                           t["time_index"], t["field"], t["tags"], histogram_quantile=case["phi"], le_column="le")
    else:
        ex = PromRangeExec(ctx, "", case["start"], case["end"], case["interval"], 0, t["time_index"], t["field"],
                           t["tags"], aggregate=inp.get("aggregate"), by_columns=inp.get("by", []),
                           lookback_delta=LOOKBACK)
    ex.push(table_batch(t, series))
    return ex


def out_rows(b):
    """-> [(value, {tag: label}, ts)] in the batch's order"""
    names = b.schema.names
    vi = next(i for i, f in enumerate(b.schema) if pa.types.is_float64(f.type))
    ti = next(i for i, f in enumerate(b.schema) if pa.types.is_timestamp(f.type))
    ts = b.column(ti).cast(pa.int64()).to_pylist()
    vals = b.column(vi).to_pylist()
    tags = [n for i, n in enumerate(names) if i not in (vi, ti)]
    cols = {t: b.column(names.index(t)).to_pylist() for t in tags}
    return [(vals[r], {t: cols[t][r] for t in tags}, ts[r]) for r in range(b.num_rows)], tags


PLAN_CASES = sorted(c["name"] for c in G["cases"] if "plan" in c["layers"])


@pytest.mark.parametrize("name", PLAN_CASES)
def test_plan_goldens(ctx, name):
    from greptimedb_b200.plan import TopkPlan
    case = CASES[name]
    out = TopkPlan(ctx, case["op"], case["k"], input_node(ctx, case)).execute()
    rows, _ = out_rows(out)
    assert [(v, lab, ts) for v, lab, ts in rows] == [(v, lab, ts) for lab, ts, v in case["expected"]]
    # {value, tags.., time index}; the value column carries the child's name (the printed sum(test.val) and the q95
    # alias are names the reference's projection gives it)
    assert out.schema.names[1:] == case["columns"][1:]
    assert pa.types.is_float64(out.schema.field(0).type)
    if case["input"].get("aggregate") is None and not case["input"].get("histogram"):
        assert out.schema.names == case["columns"]


def test_the_issue_examples_print_in_order(ctx):
    from greptimedb_b200.plan import TopkPlan
    c3 = CASES["topk_3_test"]
    rows, _ = out_rows(TopkPlan(ctx, "topk", 3, input_node(ctx, c3)).execute())
    assert len(rows) == 12 and [(r[1]["host"], r[2]) for r in rows[:3]] == [("host3", 0), ("host2", 0), ("host1", 0)]
    cb = CASES["bottomk_2_test_sum_by_idc"]
    rows, _ = out_rows(TopkPlan(ctx, "bottomk", 2, input_node(ctx, cb)).execute())
    assert [(r[1]["idc"], r[2], r[0]) for r in rows] == [(l["idc"], ts, v) for l, ts, v in cb["expected"]]


def node_rows(node):
    rows, tags = out_rows(node.execute())
    return rows, tags


def check_over(ctx, child_factory, op, k, **mod):
    """topk over `child` through the plan layer == the row-literal oracle over the child's own output"""
    from greptimedb_b200.plan import TopkPlan
    rows, tags = node_rows(child_factory())
    mname, labels = next(iter(mod.items())) if mod else (None, ())
    exp = tko.topk_rows(op == "bottomk", k, rows, tags, mname, labels)
    got, _ = out_rows(TopkPlan(ctx, op, k, child_factory(), **mod).execute())
    key = lambda rs: [(bits([v])[0], sorted(lab.items(), key=lambda x: x[0]), ts) for v, lab, ts in rs]
    assert key(got) == key(exp)
    return got


def test_topk_over_binary_set_and_function_nodes(ctx):
    from greptimedb_b200.plan import BinaryPlan, SetOpPlan
    case = CASES["topk_3_test"]
    node = lambda **m: input_node(ctx, case, **m)
    check_over(ctx, lambda: BinaryPlan(ctx, "-", node(), node().scalar_op("*", 2.0)), "topk", 2)
    check_over(ctx, lambda: SetOpPlan(ctx, "or", node(idc="idc2"), node()), "bottomk", 1, by=["idc"])
    check_over(ctx, lambda: node().function("abs").scalar_op("*", -1.0), "topk", 1, without=["host"])
    check_over(ctx, lambda: node(), "bottomk", 2, by=["nope", "idc"])  # a `by` label the child lacks is ignored
    check_over(ctx, lambda: node(), "topk", 1, without=[])


def test_consumers_read_only_kept_cells(ctx):
    """The node leaves the child's values in place and clears bits: the export, K7 (binary), K8 (set), K9 (functions,
    scalar operators) and scalar() must all see only the kept cells."""
    from greptimedb_b200.plan import BinaryPlan, ScalarPlan, SetOpPlan, TopkPlan
    case = CASES["topk_1_test"]
    node = lambda: input_node(ctx, case)
    top1 = [(v, lab, ts) for lab, ts, v in case["expected"]]
    key = lambda rs: sorted((ts, tuple(sorted(lab.items())), v) for v, lab, ts in rs)
    # K9 / scalar operators on top: topk(1, test) * 2, then abs
    got, _ = out_rows(TopkPlan(ctx, "topk", 1, node()).scalar_op("*", -2.0).function("abs").execute())
    assert [(v, lab, ts) for v, lab, ts in got] == [(2 * v, lab, ts) for v, lab, ts in top1]
    # K7: topk(1, test) + test pairs only the kept cells
    got, _ = out_rows(BinaryPlan(ctx, "+", TopkPlan(ctx, "topk", 1, node()), node()).execute())
    assert key(got) == key([(2 * v, lab, ts) for v, lab, ts in top1])
    # K8: test and topk(1, test)
    got, _ = out_rows(SetOpPlan(ctx, "and", node(), TopkPlan(ctx, "topk", 1, node())).execute())
    assert key(got) == key(top1)
    # scalar(bottomk(1, test)): host1 at every step, one series
    got, _ = out_rows(ScalarPlan(ctx, TopkPlan(ctx, "bottomk", 1, node())).execute())
    assert [(v, ts) for v, _, ts in got] == [(v, ts) for lab, ts, v in CASES["bottomk_1_test"]["expected"]]


def test_plan_errors(ctx):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import PromRangeExec, TopkPlan
    case = CASES["topk_1_test"]
    t = G["tables"]["test"]
    labels, ts, val, offsets = table_arrays(t)
    ids = np.repeat(np.arange(len(labels), dtype=np.uint64), np.diff(offsets.astype(np.int64)))
    b = pa.record_batch([pa.array(ts, pa.timestamp("ms")), pa.array(val), pa.array(ids, pa.uint64())],
                        names=["ts", "val", "__tsid"])
    byid = PromRangeExec(ctx, "", case["start"], case["end"], case["interval"], 0, "ts", "val", ["__tsid"],
                         lookback_delta=LOOKBACK)
    byid.push(b)
    with pytest.raises(B2PError) as ei:
        TopkPlan(ctx, "topk", 1, byid).execute()
    assert ei.value.code == -1 and "__tsid" in str(ei.value)
    with pytest.raises(ValueError):
        TopkPlan(ctx, "topk", 1, byid, by=["a"], without=["b"])
    # k below one keeps nothing; +inf keeps everything
    assert TopkPlan(ctx, "topk", 0.5, input_node(ctx, case)).execute().num_rows == 0
    assert TopkPlan(ctx, "bottomk", math.inf, input_node(ctx, case)).execute().num_rows == 12
