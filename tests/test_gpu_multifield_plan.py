"""GPU: the plan layer over tables with several Float64 field columns (b2p_plan_range_create_fields and the nodes above
it) and the multi-key sort (b2p_sort_cells_fields[_dev]), against tests/multifield_plan_oracle.py and the single-field
nodes, bit for bit (a NaN matches a NaN only where arithmetic made it)."""
import ctypes as C
import os

import numpy as np
import pyarrow as pa
import pytest

from oracle import oracle as orc
from tests import multifield_oracle as mf
from tests import multifield_plan_oracle as mp
from tests import select_keys as sk
from tests import subquery_oracle as sq

pytestmark = pytest.mark.gpu

T0 = 1_700_000_000_000
STEP = 15_000
PARAMS = {"predict_linear": (600.0, 0.0), "quantile_over_time": (0.9, 0.0), "holt_winters": (0.3, 0.1)}
ITV, RNG, LOOKBACK = 20_000, 60_000, 45_000


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


TIERS = {"default": {}, "warp": {"B2P_DISABLE_LEAN_TIER": "1"}, "flags": {"B2P_LEAN_FORCE_FLAGS": "1",
                                                                          "B2P_LEAN_ADAPTIVE": "0"}}


@pytest.fixture(scope="module", params=list(TIERS))
def tier_ctx(request):
    from greptimedb_b200 import Context
    env = TIERS[request.param]
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        c = Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    yield c
    c.close()


# ---- tables -------------------------------------------------------------------------------------------------------------
class Table:
    """S series of about N rows (series 1 empty), F fields f0.., tag `host` (or a UInt64 __tsid), sorted by (tag, ts)"""

    def __init__(self, S, N, F, seed, nan_rate=0.02, jitter=4000, present=None, tsid=False, dc=False):
        rng = np.random.default_rng(seed)
        sizes = rng.integers(max(1, N // 2), N + 1, S)
        if S > 2:
            sizes[1] = 0
        self.offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
        n = int(self.offsets[-1])
        self.ts = np.concatenate([T0 + np.arange(m) * STEP + (rng.integers(0, jitter, m) if jitter else 0)
                                  for m in sizes]).astype(np.int64)
        self.vals = []
        for f in range(F):
            v = np.cumsum(rng.uniform(0, 5, n)) if f % 2 == 0 else rng.normal(0, 10, n)
            v[rng.random(n) < nan_rate / max(F, 1)] = np.nan
            self.vals.append(v)
        self.present = present(n, rng) if present else None
        if self.present is not None:
            for f, m in enumerate(self.present):
                if m is not None:
                    self.vals[f][~m] = 0.0
        self.S, self.F, self.tsid = S, F, tsid
        self.hosts = [f"h{s:03d}" for s in range(S)]
        self.dcs = [f"dc{s % 3}" for s in range(S)]
        self.dc = dc
        self.sizes = sizes

    def fields(self, F=None):
        return [f"f{f}" for f in range(self.F if F is None else F)]

    def tags(self):
        return ["__tsid"] if self.tsid else (["host", "dc"] if self.dc else ["host"])

    def batch(self):
        cols = [pa.array(self.ts, pa.timestamp("ms"))]
        for f in range(self.F):
            m = None if self.present is None or self.present[f] is None else ~self.present[f]
            cols.append(pa.array(self.vals[f], pa.float64(), mask=m))
        if self.tsid:
            cols.append(pa.array(np.repeat(np.arange(self.S, dtype=np.uint64) * 7 + 3, self.sizes), pa.uint64()))
        else:
            cols.append(pa.array(np.repeat(self.hosts, self.sizes)))
            if self.dc:
                cols.append(pa.array(np.repeat(self.dcs, self.sizes)))
        return pa.record_batch(cols, names=["ts"] + self.fields() + self.tags())

    def push(self, ex, cuts=()):
        """the batch, or its slices at the given row cuts (mid-series, odd offsets)"""
        b = self.batch()
        edges = [0] + [c for c in cuts if 0 < c < b.num_rows] + [b.num_rows]
        for a, z in zip(edges, edges[1:]):
            ex.push(b.slice(a, z - a))
        return ex

    def labels(self):
        return [(h, d) for h, d in zip(self.hosts, self.dcs)] if self.dc else [(h,) for h in self.hosts]


def grid(T):
    return T0, T0 + (T - 1) * ITV, ITV


def leaf(ctx, tab, fn="prom_rate", T=60, fields=None, cuts=(), instant=False, filter_nan=True, rng=RNG, **kw):
    from greptimedb_b200.plan import PromRangeExec
    start, end, itv = grid(T)
    p0, p1 = PARAMS.get(fn[5:], (0.0, 0.0))
    ex = PromRangeExec(ctx, fn, start, end, itv, rng, "ts", tab.fields() if fields is None else fields, tab.tags(),
                       need_filter_out_nan=filter_nan, param0=p0, param1=p1,
                       lookback_delta=LOOKBACK if instant else None, **kw)
    return tab.push(ex, cuts)


def expect_leaf(tab, fn="prom_rate", T=60, instant=False, filter_nan=True, rng=RNG, F=None):
    start, end, itv = grid(T)
    vals = tab.vals[:F] if F else tab.vals
    if instant:
        return mf.instant_query_fields(tab.ts, vals, tab.offsets, start, end, itv, LOOKBACK, present=tab.present)
    p0, p1 = PARAMS.get(fn[5:], (0.0, 0.0))
    op = orc.make_params(fn[5:], start, end, itv, rng, filter_nan=filter_nan, param0=p0, param1=p1)
    return mf.range_query_fields(op, tab.ts, vals, tab.offsets, present=tab.present, rescan=True)


def same(a, b, nan_as_nan=True):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape:
        return False
    if not nan_as_nan:
        return np.array_equal(a.view(np.uint64), b.view(np.uint64))
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64))


def cells(valid, T):
    """(row, step) of every valid cell, row-major"""
    ok = orc.valid_to_bool(np.ascontiguousarray(valid, np.uint32), T)
    return np.argwhere(ok)


def check_rows(out, names, outs, valid, T, labels=None, tag_names=None, order=None, nan_as_nan=True):
    """the export: one row per valid cell (row-major, or `order` as cell indices), ts, each named value column and the
    tags of the cell's row"""
    rc = cells(valid, T)
    if order is not None:
        order = np.asarray(order, np.int64)
        rc = np.stack([order // T, order % T], axis=1) if order.size else np.zeros((0, 2), np.int64)
    assert out.num_rows == len(rc)
    ts = out.column(out.schema.names.index("ts")).cast(pa.int64()).to_numpy()
    start = T0
    assert np.array_equal(ts, start + rc[:, 1] * ITV)
    for f, name in enumerate(names):
        got = out.column(name).to_numpy(zero_copy_only=False)
        assert same(got, outs[f][rc[:, 0], rc[:, 1]], nan_as_nan), f"field {f} ({name})"
    if labels is not None:
        for t, tn in enumerate(tag_names):
            assert out.column(tn).to_pylist() == [labels[r][t] for r in rc[:, 0]]


# ---- the leaf ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F", [1, 2, 3, 8, 64])
@pytest.mark.parametrize("instant", [False, True])
def test_leaf_fields_batches_and_schema(ctx, F, instant):
    tab = Table(12, 90, F, seed=F * 3 + instant, nan_rate=0.0 if instant else 0.05)
    n = int(tab.offsets[-1])
    ex = leaf(ctx, tab, instant=instant, cuts=(37, 38, n // 2 + 3, n - 5))  # mid-series, odd offsets
    out = ex.execute()
    names = mp.leaf_names("" if instant else "prom_rate", "ts", tab.fields())
    assert out.schema.names == ["ts"] + names + ["host"]
    assert ex.num_series() == 11  # series 1 has no rows
    outs, valid = expect_leaf(tab, instant=instant)
    S = tab.offsets.size - 1
    labels = [tab.labels()[s] for s in range(S) if tab.sizes[s]]
    keep = np.flatnonzero(tab.sizes)
    check_rows(out, names, outs[:, keep], valid[keep], 60, labels, ["host"], nan_as_nan=not instant)


@pytest.mark.parametrize("fn", list(orc.FN_IDS))
def test_every_function_on_every_tier(tier_ctx, fn):
    tab = Table(40, 400, 3, seed=5, nan_rate=0.03)
    for rng in (60_000, 600_000):
        out = leaf(tier_ctx, tab, fn="prom_" + fn, T=120, rng=rng, cuts=(1001, 2503)).execute()
        outs, valid = expect_leaf(tab, "prom_" + fn, T=120, rng=rng)
        keep = np.flatnonzero(tab.sizes)
        check_rows(out, mp.leaf_names("prom_" + fn, "ts", tab.fields()), outs[:, keep], valid[keep], 120)


@pytest.mark.parametrize("filter_nan", [True, False])
def test_nan_in_one_field(ctx, filter_nan):
    tab = Table(10, 200, 2, seed=9, nan_rate=0.2)
    out = leaf(ctx, tab, fn="prom_max_over_time", filter_nan=filter_nan).execute()
    outs, valid = expect_leaf(tab, "prom_max_over_time", filter_nan=filter_nan)
    keep = np.flatnonzero(tab.sizes)
    check_rows(out, mp.leaf_names("prom_max_over_time", "ts", tab.fields()), outs[:, keep], valid[keep], 60)


def _nulls(n, rng):
    m = rng.random(n) > 0.05
    return [None, m, None]


@pytest.mark.parametrize("fn", sorted(mf.BUFFER_FNS | mf.NULL_FNS) + ["instant"])
def test_null_slots(ctx, fn):
    from greptimedb_b200 import B2PError
    tab = Table(10, 300, 3, seed=31, nan_rate=0.0, present=_nulls)
    n = int(tab.offsets[-1])
    instant = fn == "instant"
    name = "" if instant else "prom_" + fn
    ex = leaf(ctx, tab, fn=name, instant=instant, cuts=(5, 13, n // 3 + 1))  # bitmaps at non-byte-aligned offsets
    if instant or fn in mf.NULL_FNS:
        with pytest.raises(B2PError, match="field 1 has NULL slots"):
            ex.execute()
        return
    out = ex.execute()
    outs, valid = expect_leaf(tab, name)
    keep = np.flatnonzero(tab.sizes)
    check_rows(out, mp.leaf_names(name, "ts", tab.fields()), outs[:, keep], valid[keep], 60)


def test_tsid_keyed_table(ctx):
    tab = Table(9, 120, 3, seed=4, tsid=True)
    out = leaf(ctx, tab, cuts=(77,)).execute()
    assert out.schema.names == ["ts"] + mp.leaf_names("prom_rate", "ts", tab.fields()) + ["__tsid"]
    outs, valid = expect_leaf(tab)
    keep = np.flatnonzero(tab.sizes)
    ids = [(int(s) * 7 + 3,) for s in keep]
    check_rows(out, mp.leaf_names("prom_rate", "ts", tab.fields()), outs[:, keep], valid[keep], 60, ids, ["__tsid"])


# ---- one field through the new entry is the old entry ---------------------------------------------------------------
def _old_leaf(ctx, tab, fn="prom_rate", T=60, instant=False):
    """the same node through b2p_plan_range_create"""
    from greptimedb_b200 import B2PError, make_params
    from greptimedb_b200.plan import PromRangeExec, _cstr_array
    ex = PromRangeExec.__new__(PromRangeExec)
    ex._L, ex._ctx = ctx._L, ctx
    start, end, itv = grid(T)
    p = make_params(0, start, end, itv, RNG)
    tags = _cstr_array(tab.tags())
    ex._h = ex._L.b2p_plan_range_create(ctx._h, fn.encode(), C.byref(p), b"ts", b"f0", tags, len(tab.tags()), b"",
                                        _cstr_array([]), 0)
    if not ex._h:
        raise B2PError(-1, ex._L.b2p_plan_last_error().decode())
    if instant:
        ex._L.b2p_plan_set_instant(ex._h, LOOKBACK)
    return tab.push(ex)


def _trees(ctx, make):
    from greptimedb_b200 import plan as P
    yield "leaf", make()
    yield "stages", make().function("abs").scalar_op("*", 2.0).scalar_op(">", 1.0)
    yield "binary", P.BinaryPlan(ctx, "-", make(), make(), on=["host"])
    yield "filter", P.BinaryPlan(ctx, ">", make(), make().scalar_op("/", 2.0))
    yield "aggregate", P.AggregatePlan(ctx, "avg", make(), by=["host"])
    yield "quantile", P.AggregatePlan(ctx, "quantile", make(), param=0.3)
    yield "group", P.AggregatePlan(ctx, "group", make())
    yield "topk", P.TopkPlan(ctx, "topk", 2, make())
    yield "count_values", P.CountValuesPlan(ctx, "v", make())
    yield "scalar", P.ScalarPlan(ctx, make())
    yield "and", P.SetOpPlan(ctx, "and", make(), make().scalar_op(">", 1.0))
    yield "or", P.SetOpPlan(ctx, "or", make(), make())
    yield "sort", P.SortPlan(ctx, "sort_desc", make())
    yield "sort_by_label", P.SortPlan(ctx, "sort_by_label", make(), ["host"])
    yield "absent", P.AbsentPlan(ctx, make(), T0, T0 + 59 * ITV, ITV, "ts", "value")


def test_one_field_through_the_new_entry_is_the_old_entry(ctx):
    """b2p_plan_range_create is the one-field call of b2p_plan_range_create_fields, so the two share the C++ path and
    this pins only the C wrapper and PromRangeExec's binding of a one-name list; what pins F = 1 against the reference
    is the existing single-field plan suite (test_gpu_plan.py and the node tests), which now runs through the new entry"""
    tab = Table(8, 90, 1, seed=12, nan_rate=0.05)
    for instant in (False, True):
        new = dict(_trees(ctx, lambda: leaf(ctx, tab, instant=instant)))
        old = dict(_trees(ctx, lambda: _old_leaf(ctx, tab, instant=instant)))
        for kind in new:
            a, b = new[kind].execute(), old[kind].execute()
            assert a.schema == b.schema, kind
            assert a.num_rows == b.num_rows, kind
            for ca, cb in zip(a.columns, b.columns):
                if pa.types.is_floating(ca.type):
                    assert same(ca.to_numpy(zero_copy_only=False), cb.to_numpy(zero_copy_only=False), False), kind
                else:
                    assert ca.equals(cb), kind


# ---- stages ---------------------------------------------------------------------------------------------------------------
def test_stages_per_field(ctx):
    from greptimedb_b200 import B2PError
    tab = Table(10, 200, 3, seed=7)
    outs, valid = expect_leaf(tab)
    ex = leaf(ctx, tab).function("clamp", -1.0, 1.0).scalar_op("-", 0.5, scalar_on_left=True) \
        .scalar_op("<", 0.2, return_bool=True)
    e, ev = mp.instant_fn("clamp", outs, valid, -1.0, 1.0)
    e, ev = mp.scalar_op("-", 0.5, e, ev, scalar_on_left=True)
    e, ev = mp.scalar_op("<", 0.2, e, ev, return_bool=True)
    names = [f"Float64(0.5) - clamp({n},Float64(-1),Float64(1)) < Float64(0.2)"
             for n in mp.leaf_names("prom_rate", "ts", tab.fields())]
    out = ex.execute()
    assert out.schema.names == ["ts"] + names + ["host"]
    keep = np.flatnonzero(tab.sizes)
    check_rows(out, names, e[:, keep], ev[keep], 60)
    with pytest.raises(B2PError, match="Unsupported expr type: filter on multi-value input"):
        leaf(ctx, tab).scalar_op(">", 1.0).execute()


# ---- binary ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("FL,FR", [(2, 2), (3, 2), (2, 3), (1, 3), (3, 1)])
@pytest.mark.parametrize("matching", ["on", "ignoring"])
@pytest.mark.parametrize("op,return_bool", [("*", False), ("/", False), (">=", True)])
def test_binary_zip(ctx, FL, FR, matching, op, return_bool):
    from greptimedb_b200.plan import BinaryPlan
    from tests import binary_oracle as bo
    L = Table(9, 150, FL, seed=FL * 10 + FR, dc=True)
    R = Table(6, 150, FR, seed=FL * 10 + FR + 1)
    kw = {"on": ["host"]} if matching == "on" else {"ignoring": ["dc"]}
    node = BinaryPlan(ctx, op, leaf(ctx, L), leaf(ctx, R), return_bool=return_bool, **kw)
    out = node.execute()
    lo, lv = expect_leaf(L)
    ro, rv = expect_leaf(R)
    lk, rk = np.flatnonzero(L.sizes), np.flatnonzero(R.sizes)
    lrow, rrow = bo.binary_pairs(["host", "dc"], [L.labels()[s] for s in lk], ["host"], [R.labels()[s] for s in rk],
                                 on=kw.get("on"), ignoring=kw.get("ignoring"))
    e, ev = mp.binary_op(op, lo[:, lk], lv[lk], lrow, ro[:, rk], rv[rk], rrow, return_bool)
    names = mp.binary_names(op, mp.leaf_names("prom_rate", "ts", L.fields()),
                            mp.leaf_names("prom_rate", "ts", R.fields()), return_bool)
    assert out.schema.names == ["host"] + ["ts"] + names
    labels = [R.labels()[rk[q]] for q in rrow]
    check_rows(out, names, e, ev, 60, labels, ["host"])


@pytest.mark.parametrize("FL,FR", [(3, 1), (1, 3), (2, 2)])
def test_binary_filter(ctx, FL, FR):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import BinaryPlan
    from tests import binary_oracle as bo
    L = Table(7, 150, FL, seed=FL + 40)
    R = Table(7, 150, FR, seed=FL + 41)
    node = BinaryPlan(ctx, ">", leaf(ctx, L), leaf(ctx, R))
    if min(FL, FR) > 1:
        with pytest.raises(B2PError, match="Unsupported expr type: filter on multi-value input"):
            node.execute()
        return
    out = node.execute()
    lo, lv = expect_leaf(L)
    ro, rv = expect_leaf(R)
    lk, rk = np.flatnonzero(L.sizes), np.flatnonzero(R.sizes)
    lrow, rrow = bo.binary_pairs(["host"], [L.labels()[s] for s in lk], ["host"], [R.labels()[s] for s in rk])
    e, ev = mp.binary_op(">", lo[:, lk], lv[lk], lrow, ro[:, rk], rv[rk], rrow)
    names = mp.leaf_names("prom_rate", "ts", L.fields())  # the lhs's fields, every one
    assert out.schema.names == ["ts"] + names + ["host"]
    check_rows(out, names, e, ev, 60, [L.labels()[lk[q]] for q in lrow], ["host"])


# ---- aggregates ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", ["sum", "avg", "count", "min", "max", "stddev", "stdvar", "quantile"])
@pytest.mark.parametrize("modifier", ["by", "without", None])
def test_aggregate_per_field_is_the_single_field_node(ctx, op, modifier):
    from greptimedb_b200.plan import AggregatePlan
    tab = Table(12, 150, 3, seed=17, nan_rate=0.0, dc=True)
    kw = {} if modifier is None else {modifier: ["dc"]}
    param = 0.75 if op == "quantile" else None
    multi = AggregatePlan(ctx, op, leaf(ctx, tab), param=param, **kw).execute()
    for f in range(3):
        one = AggregatePlan(ctx, op, leaf(ctx, tab, fields=[f"f{f}"]), param=param, **kw).execute()
        assert multi.num_rows == one.num_rows
        name = one.schema.names[-1]
        assert multi.schema.names[-3 + f] == name
        for c in one.schema.names[:-1]:
            assert multi.column(c).equals(one.column(c))
        assert same(multi.column(name).to_numpy(), one.column(name).to_numpy(), False)


def test_aggregate_against_the_oracle(ctx):
    from greptimedb_b200.plan import AggregatePlan
    tab = Table(12, 150, 4, seed=18, dc=True)
    out = AggregatePlan(ctx, "sum", leaf(ctx, tab), by=["dc"]).execute()
    outs, valid = expect_leaf(tab)
    keep = np.flatnonzero(tab.sizes)
    names = sorted(set(tab.dcs[s] for s in keep))
    gid = np.array([names.index(tab.dcs[s]) for s in keep], np.uint32)
    e, cnt = mp.aggregate("sum", outs[:, keep], valid[keep], gid, len(names))
    ev = sk.words(cnt != 0)
    vn = [f"sum({n})" for n in mp.leaf_names("prom_rate", "ts", tab.fields())]
    assert out.schema.names == ["dc", "ts"] + vn
    check_rows(out, vn, e, ev, 60, [(n,) for n in names], ["dc"], nan_as_nan=False)


# ---- sort -----------------------------------------------------------------------------------------------------------------
def adversarial(F, R, T, seed, last_only=False):
    """F fields over an R x T grid: field 0 (and every field but the last when last_only) takes a couple of values, so
    tuples tie there; the later fields take ±0.0, ±inf, NaN of both signs and two finite values"""
    rng = np.random.default_rng(seed)
    pool = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 1.5, -2.5])
    vals = np.empty((F, R, T))
    for f in range(F):
        ties = f < F - 1 if last_only else f == 0
        vals[f] = rng.choice([3.0, -1.0], (R, T)) if ties else rng.choice(pool, (R, T))
    ok = rng.random((R, T)) > 0.15
    return vals, ok


@pytest.mark.parametrize("F", [1, 2, 3, 8])
@pytest.mark.parametrize("desc", [False, True])
@pytest.mark.parametrize("last_only", [False, True])
def test_sort_cells_fields(ctx, F, desc, last_only):
    import torch
    vals, ok = adversarial(F, 37, 45, seed=F * 4 + desc * 2 + last_only, last_only=last_only)
    valid = sk.words(ok)
    expect = mp.sort(desc, vals, ok)
    got = ctx.sort_cells_fields(desc, vals, valid)
    assert np.array_equal(got, expect)
    if F == 1:
        assert np.array_equal(got, ctx.sort_cells(desc, vals[0], valid))
    d_vals = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in vals]
    d_valid = torch.from_numpy(valid.view(np.int32)).cuda()
    d_out = torch.zeros(37 * 45, dtype=torch.int64, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int64, device="cuda")
    before = ctx.launch_count()
    ctx.sort_cells_fields_dev(desc, d_vals, d_valid, 37, 45, d_out, d_n)
    ctx.sync()
    # K13's count and K14's scatter, then one rekey per field but the last (CUB's F radix sorts are not counted)
    assert ctx.launch_count() - before == 2 + (F - 1)
    n = int(d_n.item())
    assert np.array_equal(d_out.cpu().numpy()[:n].view(np.uint64), expect)


def test_sort_ties_in_every_field_keep_row_major_order(ctx):
    vals = np.full((3, 6, 40), 7.0)
    ok = np.ones((6, 40), bool)
    for desc in (False, True):
        assert ctx.sort_cells_fields(desc, vals, sk.words(ok)).tolist() == list(range(240))


def test_sort_empty_and_refused(ctx):
    from greptimedb_b200 import B2PError
    vals = np.zeros((2, 4, 40))
    assert ctx.sort_cells_fields(False, vals, np.zeros((4, 2), np.uint32)).size == 0
    with pytest.raises(B2PError, match="n_fields"):
        ctx.sort_cells_fields(False, [vals[0]] * 65, np.zeros((4, 2), np.uint32))
    assert ctx._L.b2p_sort_cells_fields(ctx._h, 0, None, 0, None, 4, 40, None, None) == -1
    assert "n_fields" in ctx._L.b2p_last_error().decode()


@pytest.mark.parametrize("F", [2, 3, 8])
@pytest.mark.parametrize("function", ["sort", "sort_desc"])
def test_sort_node(ctx, F, function):
    """sort over an instant leaf, whose cells are the fields' own values: field 0 ties, the later fields hold ±0, ±inf
    and NaN of both signs"""
    from greptimedb_b200.plan import SortPlan
    tab = Table(10, 80, F, seed=F + 60, nan_rate=0.0, jitter=0)
    rng = np.random.default_rng(F)
    n = tab.ts.size
    tab.vals[0] = rng.choice([1.0, 2.0], n)
    pool = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 1.5])
    for f in range(1, F):
        tab.vals[f] = rng.choice(pool, n)
    out = SortPlan(ctx, function, leaf(ctx, tab, instant=True)).execute()
    outs, valid = expect_leaf(tab, instant=True)
    keep = np.flatnonzero(tab.sizes)
    ok = orc.valid_to_bool(valid[keep], 60)
    order = mp.sort(function == "sort_desc", outs[:, keep], ok)
    check_rows(out, tab.fields(), outs[:, keep], valid[keep], 60, [tab.labels()[s] for s in keep], ["host"],
               order=order, nan_as_nan=False)


# ---- subquery and absent --------------------------------------------------------------------------------------------------
def test_subquery_over_a_multi_field_child(ctx):
    from greptimedb_b200.plan import PromRangeExec, SubqueryPlan
    tab = Table(8, 200, 3, seed=71)
    start, end = T0 + 30 * ITV, T0 + 59 * ITV
    s, step, T_in = sq.inner_grid(start, end, ITV, 200_000)
    child = tab.push(PromRangeExec(ctx, "prom_rate", s, end, step, RNG, "ts", tab.fields(), ["host"]))
    out = SubqueryPlan(ctx, "prom_max_over_time", child, start, end, ITV, 200_000).execute()
    op = orc.make_params("rate", s, end, step, RNG)
    co, cv = mf.range_query_fields(op, tab.ts, tab.vals, tab.offsets, rescan=True)
    keep = np.flatnonzero(tab.sizes)
    e, ev = mp.subquery("max_over_time", start, end, ITV, 200_000, s, step, co[:, keep], cv[keep])
    names = [f"prom_max_over_time(ts_range,{n})" for n in mp.leaf_names("prom_rate", "ts", tab.fields())]
    assert out.schema.names == ["ts"] + names + ["host"]
    T = orc.num_steps(start, end, ITV)
    rc = cells(ev, T)
    assert out.num_rows == len(rc)
    assert np.array_equal(out.column("ts").cast(pa.int64()).to_numpy(), start + rc[:, 1] * ITV)
    for f, name in enumerate(names):
        assert same(out.column(name).to_numpy(), e[f][rc[:, 0], rc[:, 1]])


def test_absent_over_a_multi_field_child(ctx):
    from greptimedb_b200.plan import AbsentPlan
    tab = Table(3, 20, 3, seed=72, jitter=0)
    start, end, itv = grid(60)
    out = AbsentPlan(ctx, leaf(ctx, tab), start, end, itv, "ts", "value", [("job", "x")]).execute()
    _, valid = expect_leaf(tab)
    present = orc.valid_to_bool(valid, 60).any(axis=0)
    assert out.schema.names == ["ts", "value", "job"]
    assert np.array_equal(out.column("ts").cast(pa.int64()).to_numpy(), start + np.flatnonzero(~present) * itv)


# ---- refusals -------------------------------------------------------------------------------------------------------------
def test_refusals_at_create_and_push(ctx):
    from greptimedb_b200 import B2PError, make_params
    from greptimedb_b200.plan import PromRangeExec, _cstr_array
    tab = Table(6, 80, 2, seed=81)
    with pytest.raises(B2PError, match="aggregate stage takes one field"):
        leaf(ctx, tab, aggregate="sum")
    with pytest.raises(B2PError, match="HistogramFold over several field columns"):
        leaf(ctx, tab, histogram_quantile=0.5, le_column="host")
    with pytest.raises(B2PError, match="f1 is given twice"):
        leaf(ctx, tab, fields=["f0", "f1", "f1"])
    with pytest.raises(B2PError, match="No field named nope"):
        leaf(ctx, tab, fields=["f0", "nope"])
    b = tab.batch()
    bad = b.set_column(2, "f1", pa.array(np.arange(b.num_rows), pa.int64()))
    ex = leaf(ctx, Table(1, 1, 2, seed=1), fields=["f0", "f1"])
    with pytest.raises(B2PError, match="field column f1 is not Float64"):
        ex.push(bad)
    L = ctx._L
    start, end, itv = grid(10)
    p = make_params(0, start, end, itv, RNG)
    for n in (0, 65):
        names = _cstr_array([f"g{i}" for i in range(max(n, 1))])
        h = L.b2p_plan_range_create_fields(ctx._h, b"prom_rate", C.byref(p), b"ts", names, n, _cstr_array(["host"]), 1,
                                           b"", _cstr_array([]), 0)
        assert not h and "n_fields" in L.b2p_plan_last_error().decode()
