"""GPU: sharded plan nodes (b2p_plan_set_sharded) over a one-rank communicator export the same bytes as the unsharded
nodes (every aggregate op, the leaf's aggregate stage, Float64 and Int64 columns, one and several fields, by / without,
__tsid kept); the Int64 partials of R simulated shards merged with the all-reduce's arithmetic equal
b2p_group_aggregate_i64 over the union; and the subtrees a sharded node refuses."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

from tests.binary_oracle import _words
from tests.ranks import one_rank_comm

pytestmark = pytest.mark.gpu

OPS = ["sum", "avg", "count", "min", "max", "stddev", "stdvar", "group", "quantile"]
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


@pytest.fixture(scope="module")
def ctxs():
    """(plain context, context with a one-rank communicator)"""
    from greptimedb_b200 import Context
    plain, comm = Context(0), Context(0)
    with one_rank_comm(comm):
        yield plain, comm
    comm.close()
    plain.close()


def table(seed, i64=False, fields=1, n_series=60):
    rng = np.random.default_rng(seed)
    hosts = [None, "", "h1", "h2", "é", "日本"]
    rows = []
    for s in range(n_series):
        host, idc = hosts[s % len(hosts)], f"dc{s % 4}"
        for t in range(0, 20_000, 1000):
            if rng.random() < 0.3:
                continue
            if i64:
                v = [int(rng.choice([I64_MIN, I64_MAX, -5, 7, 1 << 62, int(rng.integers(-1000, 1000))]))
                     for _ in range(fields)]
            else:
                v = [float(rng.choice([np.nan, -0.0, 1e300, 2.5, float(rng.normal())])) for _ in range(fields)]
            rows.append((t, host, idc, f"s{s}", v))
    rows.sort(key=lambda r: (r[1] is not None, r[1] or "", r[2], r[3], r[0]))
    typ = pa.int64() if i64 else pa.float64()
    cols = [pa.array([r[0] for r in rows], pa.timestamp("ms")), pa.array([r[1] for r in rows], pa.utf8()),
            pa.array([r[2] for r in rows], pa.utf8()), pa.array([r[3] for r in rows], pa.utf8())]
    cols += [pa.array([r[4][f] for r in rows], typ) for f in range(fields)]
    return pa.record_batch(cols, names=["ts", "host", "idc", "sid"] + [f"v{f}" for f in range(fields)])


def leaf(ctx, batch, fields, aggregate=None, by=()):
    from greptimedb_b200.plan import PromRangeExec
    ex = PromRangeExec(ctx, "", 0, 20_000, 1000, 0, "ts", [f"v{f}" for f in range(fields)], ["host", "idc", "sid"],
                       lookback_delta=3000, aggregate=aggregate, by_columns=by)
    ex.push(batch)
    return ex


def same_export(a, b):
    """one schema, equal non-float columns, NULLs in the same places and float columns of the same bits"""
    if a.schema != b.schema:
        return False
    for x, y in zip(a.columns, b.columns):
        if not pa.types.is_floating(x.type):
            if not x.equals(y):
                return False
            continue
        if not (x.is_null().to_numpy(zero_copy_only=False) == y.is_null().to_numpy(zero_copy_only=False)).all():
            return False
        xs = np.asarray(x.fill_null(0).to_numpy(zero_copy_only=False), np.float64).view(np.uint64)
        ys = np.asarray(y.fill_null(0).to_numpy(zero_copy_only=False), np.float64).view(np.uint64)
        if not (xs == ys).all():
            return False
    return True


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("i64", [False, True])
@pytest.mark.parametrize("mod", [None, ("by", ["idc"]), ("without", ["sid"]), ("by", ["host"])])
def test_aggregate_node_exports_the_unsharded_bytes(ctxs, op, i64, mod):
    from greptimedb_b200.plan import AggregatePlan
    plain, comm = ctxs
    fields = 1 if op == "group" else 2
    batch = table(7, i64, fields)
    kw = {} if mod is None else {mod[0]: mod[1]}
    param = 0.3 if op == "quantile" else None
    exp = AggregatePlan(plain, op, leaf(plain, batch, fields), param=param, **kw).execute()
    got = AggregatePlan(comm, op, leaf(comm, batch, fields), param=param, **kw).sharded().execute()
    same = AggregatePlan(plain, op, leaf(plain, batch, fields), param=param, **kw).sharded().execute()
    assert same_export(same, exp)  # without a communicator: the unsharded node
    # (stddev / stdvar too: the merge's (cnt * mean) / cnt could move M2 by cnt * ulp(mean)^2, which these tables do
    # not show)
    assert same_export(got, exp), (op, i64, mod)


@pytest.mark.parametrize("op", ["sum", "avg", "count", "min", "max", "stddev", "stdvar"])
def test_leaf_aggregate_stage_exports_the_unsharded_bytes(ctxs, op):
    plain, comm = ctxs
    batch = table(11, False, 1)
    exp = leaf(plain, batch, 1, op, ["idc", "host"]).execute()
    got = leaf(comm, batch, 1, op, ["idc", "host"]).sharded().execute()
    assert same_export(got, exp)
    assert comm._L.b2p_last_group_keys_bytes(comm._h) > 12


@pytest.mark.parametrize("i64", [False, True])
@pytest.mark.parametrize("mod", [None, ("by", ["idc"]), ("without", ["sid"])])
def test_count_values_node_exports_the_unsharded_bytes(ctxs, i64, mod):
    from greptimedb_b200.plan import CountValuesPlan
    plain, comm = ctxs
    batch = table(13, i64, 1)
    kw = {} if mod is None else {mod[0]: mod[1]}
    exp = CountValuesPlan(plain, "value", leaf(plain, batch, 1), **kw).execute()
    got = CountValuesPlan(comm, "value", leaf(comm, batch, 1), **kw).sharded().execute()
    assert exp.num_rows > 0 and same_export(got, exp), (i64, mod)
    same = CountValuesPlan(plain, "value", leaf(plain, batch, 1), **kw).sharded().execute()
    assert same_export(same, exp)


def test_sharded_leaf_needs_an_aggregate_stage(ctxs):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import SortPlan
    plain, _ = ctxs
    with pytest.raises(B2PError, match="has a sharded form"):
        leaf(plain, table(1), 1).sharded()
    with pytest.raises(B2PError, match="has a sharded form"):
        SortPlan(plain, "sort", leaf(plain, table(1), 1))._set_sharded()


def test_refused_subtrees(ctxs):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import (AbsentPlan, AggregatePlan, BinaryPlan, CountValuesPlan, EmptyMetricPlan,
                                      LabelReplacePlan, ScalarPlan, SortPlan, SubqueryPlan, TopkPlan)
    _, comm = ctxs
    b = table(3)

    def lf():
        return leaf(comm, b, 1)
    refused = {
        "a binary operator": BinaryPlan(comm, "+", lf(), lf()),
        "topk / bottomk": TopkPlan(comm, "topk", 2, lf()),
        "sort": SortPlan(comm, "sort", lf()),
        "absent()": AbsentPlan(comm, lf(), 0, 20_000, 1000, "ts", "value"),
        "scalar()": ScalarPlan(comm, lf()),
        "an aggregate": AggregatePlan(comm, "sum", lf(), by=["idc"]),
        "an aggregate stage": leaf(comm, b, 1, "sum", ["idc"]),
        "count_values": CountValuesPlan(comm, "v", lf()),
        "an EmptyMetric row": EmptyMetricPlan(comm, 0, 20_000, 1000, kind="literal", literal=1.0),
    }
    for what, child in refused.items():
        with pytest.raises(B2PError, match=what.replace("(", r"\(").replace(")", r"\)")):
            AggregatePlan(comm, "sum", child).sharded().execute()
    with pytest.raises(B2PError, match="below a sharded node"):
        AggregatePlan(comm, "sum", AggregatePlan(comm, "sum", lf(), by=["idc"]).sharded()).sharded().execute()
    with pytest.raises(B2PError, match="below a sharded node"):
        CountValuesPlan(comm, "v", AggregatePlan(comm, "sum", lf(), by=["idc"]).sharded()).sharded().execute()
    with pytest.raises(B2PError, match="an aggregate"):
        CountValuesPlan(comm, "v", AggregatePlan(comm, "sum", lf(), by=["idc"])).sharded().execute()
    # row-local subtrees are accepted: element-wise stages, label_replace, a subquery
    ok = LabelReplacePlan(comm, lf().function("abs"), "dst", "$1", "host", "(.*)")
    AggregatePlan(comm, "max", ok, by=["dst"]).sharded().execute()
    sq = SubqueryPlan(comm, "prom_max_over_time", lf(), 5000, 20_000, 1000, 5000)
    AggregatePlan(comm, "sum", sq).sharded().execute()


@pytest.mark.parametrize("R", [1, 2, 3, 8])
@pytest.mark.parametrize("op", ["sum", "min", "max"])
def test_int64_partials_of_simulated_shards_merge_to_the_union(ctxs, R, op):
    import torch
    from greptimedb_b200.engine import AGG_IDS
    plain, _ = ctxs
    L = plain._L
    rng = np.random.default_rng(R * 10 + len(op))
    n, G, T = 300, 9, 45
    vals = rng.choice(np.array([I64_MIN, I64_MAX, I64_MAX - 1, I64_MIN + 1, 1 << 62, -3, 0, 9], np.int64), (n, T))
    ok = rng.random((n, T)) < 0.6
    ok[:, 7] = False  # a step without any member
    gid = rng.integers(0, G, n).astype(np.uint32)
    gid[gid == 4] = 3  # a group without members
    words = _words(ok)
    exp_v, exp_c = np.zeros(G * T, np.int64), np.zeros(G * T, np.uint32)
    rc = L.b2p_group_aggregate_i64(plain._h, AGG_IDS[op], vals.ctypes.data, words.ctypes.data, gid.ctypes.data, n, G, T,
                                   exp_v.ctypes.data, exp_c.ctypes.data)
    assert rc == 0
    owner = rng.integers(0, R, n)
    acc_v = np.zeros(G * T, np.uint64) if op == "sum" else np.full(G * T, I64_MAX if op == "min" else I64_MIN, np.int64)
    acc_c = np.zeros(G * T, np.uint64)
    for r in range(R):
        mine = np.flatnonzero(owner == r)
        dv = torch.from_numpy(np.ascontiguousarray(vals[mine])).cuda()
        dw = torch.from_numpy(np.ascontiguousarray(_words(ok[mine])).view(np.int32)).cuda()
        dg = torch.from_numpy(np.ascontiguousarray(gid[mine]).view(np.int32)).cuda()
        ov = torch.zeros(G * T, dtype=torch.int64, device="cuda")
        oc = torch.zeros(G * T, dtype=torch.int32, device="cuda")
        assert L.b2p_group_aggregate_partial_i64_dev(plain._h, AGG_IDS[op], dv.data_ptr(), dw.data_ptr(), dg.data_ptr(),
                                                     mine.size, G, T, ov.data_ptr(), oc.data_ptr()) == 0
        plain.sync()
        pv, pc = ov.cpu().numpy(), oc.cpu().numpy().view(np.uint32)
        if op == "sum":
            acc_v += pv.view(np.uint64)
        else:
            pv = np.where(pc > 0, pv, I64_MAX if op == "min" else I64_MIN)
            acc_v = np.minimum(acc_v, pv) if op == "min" else np.maximum(acc_v, pv)
        acc_c += pc
    got_v = acc_v.view(np.int64) if op == "sum" else np.where(acc_c > 0, acc_v, 0)
    assert (got_v == exp_v).all() and (acc_c == exp_c).all()
    assert ((vals == I64_MIN) & ok).any() and ((vals == I64_MAX) & ok).any()


@pytest.mark.parametrize("op", ["sum", "min", "max"])
def test_int64_allreduce_over_one_rank(ctxs, op):
    import torch
    from greptimedb_b200.engine import AGG_IDS
    _, comm = ctxs
    L = comm._L
    v = torch.tensor([I64_MIN, 5, I64_MAX, 77], dtype=torch.int64, device="cuda")
    c = torch.tensor([1, 0, 2, 0], dtype=torch.int32, device="cuda")
    assert L.b2p_allreduce_partials_i64_dev(comm._h, AGG_IDS[op], v.data_ptr(), c.data_ptr(), 4) == 0
    comm.sync()
    # one rank: the sum is its own partial; min / max pass through the neutral values and read 0 where cnt is 0
    exp = [I64_MIN, 5, I64_MAX, 77] if op == "sum" else [I64_MIN, 0, I64_MAX, 0]
    assert v.cpu().tolist() == exp and c.cpu().tolist() == [1, 0, 2, 0]
    assert L.b2p_allreduce_partials_i64_dev(comm._h, AGG_IDS["avg"], v.data_ptr(), c.data_ptr(), 4) != 0


def test_group_keys_exchange_over_one_rank(ctxs):
    from greptimedb_b200 import distributed as D
    _, comm = ctxs
    L = comm._L
    rank = C.c_int32(-1)
    assert L.b2p_comm_ranks(comm._h, C.byref(rank)) == 1 and rank.value == 0
    blk = D.serialize_group_keys([("", None), (None, "é")], 2, n_rows=5, types=(1,))
    sizes = (C.c_uint64 * 1)()
    assert L.b2p_group_keys_sizes(comm._h, len(blk), sizes) == 0 and sizes[0] == len(blk)
    out = C.create_string_buffer(len(blk))
    assert L.b2p_group_keys_allgather(comm._h, blk, sizes, out) == 0
    assert out.raw == blk and L.b2p_last_group_keys_bytes(comm._h) == len(blk)
